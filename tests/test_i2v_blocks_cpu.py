"""HunyuanVideo-I2V fused block path, CPU side: the token-replace entry points of the dense chains
validate their arguments before any CUDA call, and install() patches the unmodified
hyvideo_i2v/modules/models_mul.py block forwards without changing their signatures."""
import inspect
import sys
from pathlib import Path

import pytest
import torch

from jenga_b200._lib import lib

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(ROOT))

E_INVALID, E_UNSUPPORTED, E_CUDA = -1, -2, -3
P = 0x10000   # never dereferenced on the validation paths


def _err():
    return lib.jenga_last_error().decode()


def _ln(**over):
    a = dict(x=P, xs=3072, scale=P, shift=P, tr_scale=P, tr_shift=P, mask=P, out=P, os=3072, rows=10, C=3072)
    a.update(over)
    return lib.jenga_ln_modulate_tr(a["x"], a["xs"], a["scale"], a["shift"], a["tr_scale"], a["tr_shift"], a["mask"],
                                    a["out"], a["os"], a["rows"], a["C"], 1e-6, None)


def _gate(**over):
    a = dict(x=P, xs=3072, y=P, ys=3072, gate=P, tr_gate=P, mask=P, out=P, os=3072, rows=10, C=3072)
    a.update(over)
    return lib.jenga_gate_residual_tr(a["x"], a["xs"], a["y"], a["ys"], a["gate"], a["tr_gate"], a["mask"], a["out"],
                                      a["os"], a["rows"], a["C"], None)


@pytest.mark.parametrize("over,code,needle", [
    (dict(x=None), E_INVALID, "null"),
    (dict(tr_scale=None), E_INVALID, "null"),
    (dict(tr_shift=None), E_INVALID, "null"),
    (dict(mask=None), E_INVALID, "null"),
    (dict(C=3070), E_INVALID, "multiples of 8"),
    (dict(xs=3076), E_INVALID, "multiples of 8"),
    (dict(os=3068), E_INVALID, "multiples of 8"),
    (dict(rows=0), E_INVALID, "shape"),
    (dict(tr_scale=P + 8), E_INVALID, "aligned"),
    (dict(tr_shift=P + 2), E_INVALID, "aligned"),
    (dict(scale=P + 8), E_INVALID, "aligned"),
    (dict(C=8192, xs=8192, os=8192), E_UNSUPPORTED, "6144"),
])
def test_ln_modulate_tr_validates_before_cuda(over, code, needle):
    rc = _ln(**over)
    assert rc == code, (rc, _err())
    assert needle.lower() in _err().lower(), _err()


@pytest.mark.parametrize("over,code,needle", [
    (dict(y=None), E_INVALID, "null"),
    (dict(tr_gate=None), E_INVALID, "null"),
    (dict(mask=None), E_INVALID, "null"),
    (dict(C=3070), E_INVALID, "shape"),
    (dict(ys=3076), E_INVALID, "shape"),
    (dict(rows=0), E_INVALID, "shape"),
    (dict(tr_gate=P + 8), E_INVALID, "aligned"),
    (dict(gate=P + 4), E_INVALID, "aligned"),
])
def test_gate_residual_tr_validates_before_cuda(over, code, needle):
    rc = _gate(**over)
    assert rc == code, (rc, _err())
    assert needle.lower() in _err().lower(), _err()


def test_valid_arguments_without_a_device_report_a_cuda_error():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert _ln() == E_CUDA and _err()
    assert _gate() == E_CUDA and _err()


def test_predicates_refuse_token_replace_arguments_they_cannot_take():
    """the *_supported predicates are pure shape / dtype checks: CPU tensors are refused, and so
    are masks of the wrong length or dtype"""
    from jenga_b200 import dense as DN
    x = torch.zeros(1, 16, 64, dtype=torch.bfloat16)
    g = torch.zeros(1, 64, dtype=torch.bfloat16)
    m = torch.zeros(16, dtype=torch.bool)
    assert not DN.gate_residual_supported(x, x, g, tr=(g, m))            # not on a GPU
    assert not DN._tr_supported(x, (g,), m[:15])
    assert not DN._tr_supported(x, (g,), m.to(torch.uint8))
    assert not DN._tr_supported(x, (g.float(),), m)
    assert DN._tr_supported(x, (g, g), m)


def test_install_patches_i2v_blocks_with_the_reference_signatures():
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    pytest.importorskip("einops")
    from jenga_b200 import blocks
    from i2v_ref import load_i2v_blocks
    ref = load_i2v_blocks(product=False)
    ours = load_i2v_blocks(product=True)
    try:
        for cls in ("MMDoubleStreamBlock", "MMSingleStreamBlock"):
            orig = getattr(ref, cls).forward
            patched = getattr(ours, cls).forward
            assert not getattr(orig, "__jenga_b200__", False)
            assert patched.__jenga_b200__, cls
            assert inspect.signature(patched) == inspect.signature(orig), cls
            # the original forward of the product-bound module is kept for the fall-back path
            assert inspect.signature(patched.__wrapped__) == inspect.signature(orig)
            assert not getattr(patched.__wrapped__, "__jenga_b200__", False)
        assert ours.block_sparse_attention.__doc__ == "jenga_b200 drop-in (hyvideo_i2v variant)"
        assert "hyvideo_i2v.modules.models_mul" in blocks._PatchFinder.targets
        assert {"i2v_double", "i2v_single"} <= set(blocks.STATS)
    finally:
        blocks.remove_gather_hook()


def test_install_without_fused_blocks_leaves_i2v_on_the_operator_hook():
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    pytest.importorskip("einops")
    import importlib
    from jenga_b200 import blocks, install
    parked = [f for f in sys.meta_path if isinstance(f, blocks._PatchFinder)]
    for f in parked:
        sys.meta_path.remove(f)
    try:
        with R.reference_packages(product=False):
            install.install(fused_blocks=False, gather=False)
            m = importlib.import_module("hyvideo_i2v.modules.models_mul")
        assert not getattr(m.MMDoubleStreamBlock.forward, "__jenga_b200__", False)
        assert not getattr(m.MMSingleStreamBlock.forward, "__jenga_b200__", False)
        assert m.block_sparse_attention.__doc__ == "jenga_b200 drop-in (hyvideo_i2v variant)"
    finally:
        for f in parked:
            sys.meta_path.insert(0, f)
