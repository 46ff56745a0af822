"""Wan2.1-I2V fused cross-attention, CPU side: jenga_wan_i2v_cross_attn validates every argument before
any CUDA call and has no fallback, the fused block's I2V eligibility rules, and install() leaving
WanI2VCrossAttention.forward unpatched."""
import ctypes as C
import sys
from pathlib import Path

import pytest
import torch

from jenga_b200._lib import JENGA_BF16, JENGA_F16, JengaWanCrossArgs, lib

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(ROOT))

E_INVALID, E_CUDA = -1, -3
P = 0x10000   # never dereferenced on the validation paths
H = 40
ROW = H * 128


def _err():
    return lib.jenga_last_error().decode()


def _args(**over):
    a = JengaWanCrossArgs()
    for n, off in (("q", 0), ("k_img", 1), ("v_img", 2), ("k_txt", 3), ("v_txt", 4), ("out", 5)):
        setattr(a, n, P * (off + 1))
    a.dtype, a.batch, a.heads, a.head_dim = JENGA_BF16, 1, H, 128
    a.q_rows, a.img_rows, a.txt_rows = 1037, 257, 512
    for t, rows in (("q", 1037), ("ki", 257), ("vi", 257), ("kt", 512), ("vt", 512), ("o", 1037)):
        setattr(a, f"{t}_stride_b", rows * ROW)
        setattr(a, f"{t}_stride_s", ROW)
        setattr(a, f"{t}_stride_h", 128)
    a.sm_scale = 128 ** -0.5
    a.err_flag = None
    for k, v in over.items():
        setattr(a, k, v)
    return a


def _call(a):
    return lib.jenga_wan_i2v_cross_attn(C.byref(a), None)


_INVALID = [
    (dict(q=None), "null"), (dict(k_img=None), "null"), (dict(v_img=None), "null"),
    (dict(k_txt=None), "null"), (dict(v_txt=None), "null"), (dict(out=None), "null"),
    (dict(dtype=JENGA_F16), "bf16"), (dict(dtype=2), "bf16"),
    (dict(head_dim=64), "head_dim"), (dict(head_dim=256), "head_dim"),
    (dict(img_rows=0), "img_rows"), (dict(txt_rows=0), "txt_rows"), (dict(txt_rows=-3), "txt_rows"),
    (dict(q_rows=0), "empty"), (dict(batch=0), "empty"), (dict(heads=0), "empty"),
    (dict(sm_scale=0.0), "sm_scale"), (dict(sm_scale=-0.1), "sm_scale"), (dict(sm_scale=float("nan")), "sm_scale"),
    (dict(q_stride_s=ROW + 4), "16 bytes"), (dict(ki_stride_h=132), "16 bytes"), (dict(vi_stride_b=12), "16 bytes"),
    (dict(kt_stride_s=ROW - 2), "16 bytes"), (dict(vt_stride_h=0), "16 bytes"), (dict(o_stride_s=-ROW), "16 bytes"),
    (dict(q=P + 8), "aligned"), (dict(v_txt=P * 5 + 2), "aligned"), (dict(out=P * 6 + 4), "aligned"),
]


@pytest.mark.parametrize("over,needle", _INVALID, ids=[",".join(f"{k}={v}" for k, v in o.items()) for o, _ in _INVALID])
def test_every_invalid_argument_is_refused_before_cuda(over, needle):
    rc = _call(_args(**over))
    assert rc == E_INVALID, (rc, _err())
    assert needle.lower() in _err().lower(), _err()


def test_null_args_struct_is_refused():
    assert lib.jenga_wan_i2v_cross_attn(None, None) == E_INVALID
    assert "null" in _err().lower()


def test_valid_arguments_without_a_device_report_a_cuda_error():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    for over in ({}, dict(img_rows=1, txt_rows=1, q_rows=1)):
        assert _call(_args(**over)) == E_CUDA and _err()


def test_python_wrapper_has_no_cpu_path():
    from jenga_b200 import wan
    from jenga_b200._lib import JengaError
    t = torch.zeros(1, 4, 1, 128, dtype=torch.bfloat16)
    with pytest.raises(JengaError):
        wan.i2v_cross_attn(t, t, t, t, t)


# ------------------------------------------------------------------------------------------------
# eligibility of the fused I2V cross-attention inside the fused block
# ------------------------------------------------------------------------------------------------
class WanRMSNorm(torch.nn.Module):
    """stand-in with the name and parameters of wan/modules/model_mul.py:74-90"""

    def __init__(self, dim, eps=1e-6):
        super().__init__()
        self.eps = eps
        self.weight = torch.nn.Parameter(torch.ones(dim))


class _I2VCross(torch.nn.Module):
    def __init__(self, dim=256, heads=2, eps=1e-6):
        super().__init__()
        self.num_heads, self.head_dim = heads, dim // heads
        self.norm_q, self.norm_k, self.norm_k_img = WanRMSNorm(dim, eps), WanRMSNorm(dim, eps), WanRMSNorm(dim, eps)


def test_i2v_eligibility_rules():
    from jenga_b200 import blocks
    ok = blocks._wan_i2v_cross_shape_ok
    ca = _I2VCross()
    x = torch.zeros(1, 300, 256)
    ctx = torch.zeros(1, 257 + 512, 256)
    assert ok(ca, x, ctx, None)
    assert ok(ca, x, ctx[:, :258], None)                               # one text row is enough
    assert not ok(ca, x, ctx, torch.tensor([300]))                     # varlen context_lens
    assert not ok(ca, x, ctx[:, :257], None)                           # no text rows
    assert not ok(ca, x, ctx[:, :100], None)
    assert not ok(ca, x.expand(2, -1, -1), ctx.expand(2, -1, -1), None)  # batch 2
    assert not ok(ca, x, ctx.expand(2, -1, -1), None)
    assert not ok(ca, x[0], ctx, None)
    assert not ok(_I2VCross(dim=256, heads=4), x, ctx, None)          # head_dim 64
    for n in ("norm_q", "norm_k", "norm_k_img"):
        bad = _I2VCross()
        setattr(bad, n, torch.nn.Identity())                           # qk_norm=False
        assert not ok(bad, x, ctx, None), n
        bad = _I2VCross()
        getattr(bad, n).eps = 1e-5
        assert not ok(bad, x, ctx, None), n
    # on the CPU, and outside autocast, the full predicate always refuses
    from jenga_b200 import dense as DN
    assert not DN._autocast_bf16()
    assert not blocks.wan_i2v_cross_eligible(ca, x, ctx, None)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert not blocks.wan_i2v_cross_eligible(ca, x, ctx, None)


def _load_wan(product):
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    return R.load_blocks(product=product)[1]


def test_install_leaves_i2v_cross_attention_forward_unpatched():
    from jenga_b200 import blocks
    ref = _load_wan(False)
    ours = _load_wan(True)
    try:
        assert ours.WanAttentionBlock.forward.__jenga_b200__
        assert not getattr(ours.WanI2VCrossAttention.forward, "__jenga_b200__", False)
        assert ours.WanI2VCrossAttention.forward.__qualname__ == "WanI2VCrossAttention.forward"
        assert ours.WanI2VCrossAttention.forward.__code__.co_code == ref.WanI2VCrossAttention.forward.__code__.co_code
        assert {"wan_block", "wan_cross", "wan_i2v_cross"} <= set(blocks.STATS)
    finally:
        blocks.remove_gather_hook()
