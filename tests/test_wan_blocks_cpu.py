"""Wan2.1 fused block path, CPU side: the three wan_* entry points of the dense chains validate their
arguments before any CUDA call, install() patches the unmodified wan/modules/model_mul.py
WanAttentionBlock and WanT2VCrossAttention forwards without changing their signatures, and the
*_supported predicates refuse what the kernels do not take."""
import inspect
import sys
from pathlib import Path

import pytest
import torch

from jenga_b200._lib import JENGA_BF16, JENGA_F32, lib

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(ROOT))

E_INVALID, E_UNSUPPORTED, E_CUDA = -1, -2, -3
P = 0x10000   # never dereferenced on the validation paths


def _err():
    return lib.jenga_last_error().decode()


def _ln(**over):
    a = dict(x=P, dt=JENGA_F32, xs=5120, scale=P, shift=P, out=P, os=5120, rows=10, C=5120)
    a.update(over)
    return lib.jenga_wan_ln_modulate(a["x"], a["dt"], a["xs"], a["scale"], a["shift"], a["out"], a["os"], a["rows"],
                                     a["C"], 1e-6, None)


def _res(**over):
    a = dict(x=P, dt=JENGA_BF16, xs=5120, y=P, ys=5120, gate=P, res=P, rs=5120, va=P, vb=P, affine=1, out=P,
             os=5120, rows=10, C=5120)
    a.update(over)
    return lib.jenga_wan_residual_ln(a["x"], a["dt"], a["xs"], a["y"], a["ys"], a["gate"], a["res"], a["rs"], a["va"],
                                     a["vb"], a["affine"], a["out"], a["os"], a["rows"], a["C"], 1e-6, None)


def _gate(**over):
    a = dict(x=P, dt=JENGA_F32, xs=5120, y=P, ys=5120, gate=P, out=P, os=5120, rows=10, C=5120)
    a.update(over)
    return lib.jenga_wan_gate_residual(a["x"], a["dt"], a["xs"], a["y"], a["ys"], a["gate"], a["out"], a["os"],
                                       a["rows"], a["C"], None)


_COMMON = [
    (dict(x=None), E_INVALID, "null"),
    (dict(out=None), E_INVALID, "null"),
    (dict(dt=1), E_INVALID, "bf16 or f32"),
    (dict(C=5118), E_INVALID, "multiples of 8"),
    (dict(xs=5124), E_INVALID, "multiples of 8"),
    (dict(os=5116), E_INVALID, "multiples of 8"),
    (dict(xs=5112), E_INVALID, "shape"),
    (dict(rows=0), E_INVALID, "shape"),
    (dict(x=P + 8), E_INVALID, "aligned"),
    (dict(out=P + 2), E_INVALID, "aligned"),
    (dict(C=8192, xs=8192, os=8192), E_UNSUPPORTED, "6144"),
]


@pytest.mark.parametrize("over,code,needle", _COMMON + [
    (dict(scale=None), E_INVALID, "null"),
    (dict(shift=None), E_INVALID, "null"),
    (dict(scale=P + 4), E_INVALID, "aligned"),
])
def test_wan_ln_modulate_validates_before_cuda(over, code, needle):
    rc = _ln(**over)
    assert rc == code, (rc, _err())
    assert needle.lower() in _err().lower(), _err()


@pytest.mark.parametrize("over,code,needle", _COMMON + [
    (dict(y=None), E_INVALID, "null"),
    (dict(res=None), E_INVALID, "null"),
    (dict(va=None), E_INVALID, "null"),
    (dict(vb=None), E_INVALID, "null"),
    (dict(ys=5124), E_INVALID, "multiples of 8"),
    (dict(rs=5112), E_INVALID, "shape"),
    (dict(y=P + 8), E_INVALID, "aligned"),
    (dict(res=P + 4), E_INVALID, "aligned"),
    (dict(gate=P + 4), E_INVALID, "aligned"),
    (dict(vb=P + 8), E_INVALID, "aligned"),
])
def test_wan_residual_ln_validates_before_cuda(over, code, needle):
    rc = _res(**over)
    assert rc == code, (rc, _err())
    assert needle.lower() in _err().lower(), _err()


@pytest.mark.parametrize("over,code,needle", _COMMON[:-1] + [
    (dict(y=None), E_INVALID, "null"),
    (dict(gate=None), E_INVALID, "null"),
    (dict(ys=5116), E_INVALID, "multiples of 8"),
    (dict(y=P + 8), E_INVALID, "aligned"),
    (dict(gate=P + 4), E_INVALID, "aligned"),
])
def test_wan_gate_residual_validates_before_cuda(over, code, needle):
    rc = _gate(**over)
    assert rc == code, (rc, _err())
    assert needle.lower() in _err().lower(), _err()


def test_valid_arguments_without_a_device_report_a_cuda_error():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert _ln() == E_CUDA and _err()
    assert _res() == E_CUDA and _err()
    assert _res(gate=None, affine=0) == E_CUDA and _err()
    assert _gate() == E_CUDA and _err()


class WanLayerNorm(torch.nn.LayerNorm):
    """stand-in with the name and construction of wan/modules/model_mul.py:93-103"""

    def __init__(self, dim, eps=1e-6, elementwise_affine=False):
        super().__init__(dim, elementwise_affine=elementwise_affine, eps=eps)


def test_predicates_refuse_what_the_kernels_do_not_take():
    """CPU tensors, batch 2, a bf16 `e` and a call outside autocast are all refused; so are norms of
    the wrong class or affinity"""
    from jenga_b200 import dense as DN
    C = 64
    x = torch.zeros(1, 16, C)
    e = torch.zeros(1, 6, C)
    n, n3 = WanLayerNorm(C), WanLayerNorm(C, elementwise_affine=True)
    for ac in (False, True):
        # the CPU tensors are refused whatever the autocast state
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=ac):
            assert not DN.wan_ln_modulate_supported(x, n, e)
            assert not DN.wan_residual_ln_supported(x, n3, e, affine=True)
            assert not DN.wan_gate_residual_supported(x, e)
    # everything below but the device would do: each case fails on its own account
    cuda_x = torch.empty(1, 16, C, device="meta")
    cuda_e = torch.empty(1, 6, C, device="meta")
    assert not DN._wan_rows_ok(cuda_x, cuda_e)                     # not a CUDA tensor
    assert not DN._wan_rows_ok(torch.zeros(2, 16, C), torch.zeros(2, 6, C))
    assert not DN._wan_rows_ok(x, e.bfloat16())
    assert not DN._autocast_bf16()
    assert DN._wan_layer_norm(n, affine=False) and not DN._wan_layer_norm(n, affine=True)
    assert DN._wan_layer_norm(n3, affine=True) and not DN._wan_layer_norm(n3, affine=False)
    assert not DN._wan_layer_norm(torch.nn.LayerNorm(C, elementwise_affine=False), affine=False)
    assert not DN._wan_layer_norm(torch.nn.Identity(), affine=True)


def test_predicates_on_cuda_need_bf16_autocast_batch_1_and_fp32_e():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device to build CUDA tensors")
    from jenga_b200 import dense as DN
    C = 64
    x = torch.zeros(1, 16, C, device="cuda")
    e = torch.zeros(1, 6, C, device="cuda")
    n = WanLayerNorm(C)
    assert not DN.wan_ln_modulate_supported(x, n, e)               # no autocast
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert DN.wan_ln_modulate_supported(x, n, e)
        assert not DN.wan_ln_modulate_supported(x.expand(2, 16, C), n, e)
        assert not DN.wan_ln_modulate_supported(x, n, e.bfloat16())
        assert not DN.wan_gate_residual_supported(x.cpu(), e)


def _load_wan(product):
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    return R.load_blocks(product=product)[1]


def test_install_patches_wan_block_and_t2v_cross_attention_with_the_reference_signatures():
    from jenga_b200 import blocks
    ref = _load_wan(False)
    ours = _load_wan(True)
    try:
        for cls in ("WanAttentionBlock", "WanT2VCrossAttention"):
            orig = getattr(ref, cls).forward
            patched = getattr(ours, cls).forward
            assert not getattr(orig, "__jenga_b200__", False)
            assert patched.__jenga_b200__, cls
            assert inspect.signature(patched) == inspect.signature(orig), cls
            # the unpatched forward of the product-bound module is kept for the fall-back path
            assert inspect.signature(patched.__wrapped__) == inspect.signature(orig)
            assert not getattr(patched.__wrapped__, "__jenga_b200__", False)
            assert patched.__wrapped__.__qualname__ == f"{cls}.forward"
        assert not getattr(ours.WanI2VCrossAttention.forward, "__jenga_b200__", False)
        assert {"wan_block", "wan_cross"} <= set(blocks.STATS)
    finally:
        blocks.remove_gather_hook()


def test_install_without_fused_blocks_patches_neither_wan_class():
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    import importlib
    from jenga_b200 import blocks, install
    parked = [f for f in sys.meta_path if isinstance(f, blocks._PatchFinder)]
    for f in parked:
        sys.meta_path.remove(f)
    try:
        with R.reference_packages(product=False):
            install.install(fused_blocks=False, gather=False)
            m = importlib.import_module("wan.modules.model_mul")
        assert not getattr(m.WanAttentionBlock.forward, "__jenga_b200__", False)
        assert not getattr(m.WanT2VCrossAttention.forward, "__jenga_b200__", False)
        assert m.block_sparse_attention.__doc__ == "jenga_b200 drop-in (wan variant)"
    finally:
        for f in parked:
            sys.meta_path.insert(0, f)
