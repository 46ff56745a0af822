"""Opt-in FP8 Linears (csrc/linear_fp8.cu, jenga_ln_modulate_fp8 in csrc/dense_fused.cu) without a GPU:
argument validation of the four new entry points, no fallback without a device, and the row
quantisation rule restated in torch (the oracle of tests/test_linear_fp8_gpu.py), pinned on hand-made rows.

The rule: scale = amax(|row|) / 448 (1 for an all-zero row), codes = e4m3(x / scale) rounded to
nearest-even and saturated at ±448 (what cvt.rn.satfinite does; torch's own cast makes NaN there)."""
import ctypes as C
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
from jenga_b200 import _lib  # noqa: E402
from jenga_b200._lib import JengaLinearFp8Args, lib  # noqa: E402
from test_cabi_validation_cpu import E_CUDA, E_INVALID, E_UNSUPPORTED, _err  # noqa: E402

P = 0x10000


def quantize_rows_ref(x: torch.Tensor):
    """torch restatement of jenga_quantize_rows_fp8: x bf16 [M, K] -> (codes float8_e4m3fn [M, K], scale f32 [M])"""
    xf = x.float()
    amax = xf.abs().amax(-1)
    scale = torch.where(amax > 0, amax / 448, torch.ones_like(amax))
    return (xf / scale[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn), scale


# ------------------------------------------------------------------ argument validation
def _lin(**over):
    a = JengaLinearFp8Args(a=P, a_stride=256, a_scale=P, w=P, w_scale=P, w_scale_stride=1, bias=None,
                           bias_dtype=_lib.JENGA_BF16, out=P, out_stride=128, m=100, n=128, k=256)
    for k, v in over.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("over,code,needle", [
    (dict(a=None), E_INVALID, "null"),
    (dict(w_scale=None), E_INVALID, "null"),
    (dict(out=None), E_INVALID, "null"),
    (dict(m=0), E_INVALID, "shape"),
    (dict(a_stride=128), E_INVALID, "shape"),
    (dict(k=120, a_stride=256), E_UNSUPPORTED, "multiple of 16"),
    (dict(n=100, out_stride=128), E_UNSUPPORTED, "multiple of 16"),
    (dict(w_scale_stride=2), E_INVALID, "w_scale_stride"),
    (dict(bias=P, bias_dtype=_lib.JENGA_F16), E_INVALID, "bias dtype"),
    (dict(a=P + 8), E_INVALID, "aligned"),
    (dict(a_stride=264), E_INVALID, "aligned"),
    (dict(bias=P + 4), E_INVALID, "aligned"),
])
def test_linear_fp8_argument_validation(over, code, needle):
    rc = lib.jenga_linear_fp8(C.byref(_lin(**over)), None)
    assert rc == code, (rc, _err())
    assert needle in _err().lower(), _err()
    assert lib.jenga_linear_fp8(None, None) == E_INVALID and "null" in _err()


@pytest.mark.parametrize("args,code,needle", [
    ((None, 256, 10, 256, P, 256, P), E_INVALID, "null"),
    ((P, 256, 10, 256, P, 256, None), E_INVALID, "null"),
    ((P, 256, 0, 256, P, 256, P), E_INVALID, "shape"),
    ((P, 256, 10, 264, P, 272, P), E_INVALID, "shape"),
    ((P, 264, 10, 264, P, 272, P), E_UNSUPPORTED, "multiple of 16"),
    ((P + 8, 256, 10, 256, P, 256, P), E_INVALID, "aligned"),
    ((P, 260, 10, 256, P, 256, P), E_INVALID, "aligned"),
    ((P, 256, 10, 256, P, 264, P), E_INVALID, "aligned"),
])
def test_quantize_rows_fp8_argument_validation(args, code, needle):
    rc = lib.jenga_quantize_rows_fp8(*args, None)
    assert rc == code, (rc, _err())
    assert needle in _err().lower(), _err()


@pytest.mark.parametrize("tr", [False, True])
@pytest.mark.parametrize("over,code,needle", [
    (dict(x=None), E_INVALID, "null"),
    (dict(a_scale=None), E_INVALID, "null"),
    (dict(channels=72, x_stride=72, out_stride=80), E_UNSUPPORTED, "multiple of 16"),
    (dict(out_stride=264), E_INVALID, "aligned"),
    (dict(x=P + 8), E_INVALID, "aligned"),
    (dict(channels=100), E_INVALID, "shape"),
])
def test_ln_modulate_fp8_argument_validation(tr, over, code, needle):
    a = dict(x=P, x_stride=256, scale=P, shift=P, out8=P, out_stride=256, a_scale=P, rows=10, channels=256)
    a.update(over)
    if tr:
        rc = lib.jenga_ln_modulate_tr_fp8(a["x"], a["x_stride"], a["scale"], a["shift"], P, P, P, a["out8"],
                                          a["out_stride"], a["a_scale"], a["rows"], a["channels"], 1e-6, None)
    else:
        rc = lib.jenga_ln_modulate_fp8(a["x"], a["x_stride"], a["scale"], a["shift"], a["out8"], a["out_stride"],
                                       a["a_scale"], a["rows"], a["channels"], 1e-6, None)
    assert rc == code, (rc, _err())
    assert needle in _err().lower(), _err()


def test_ln_modulate_tr_fp8_needs_its_token_replace_vectors():
    rc = lib.jenga_ln_modulate_tr_fp8(P, 256, P, P, None, P, P, P, 256, P, 10, 256, 1e-6, None)
    assert rc == E_INVALID and "null" in _err()


def test_without_a_device_every_entry_point_reports_cuda_error_not_a_fallback():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert lib.jenga_linear_fp8(C.byref(_lin()), None) == E_CUDA and _err()
    assert lib.jenga_quantize_rows_fp8(P, 256, 10, 256, P, 256, P, None) == E_CUDA and _err()
    assert lib.jenga_ln_modulate_fp8(P, 256, P, P, P, 256, P, 10, 256, 1e-6, None) == E_CUDA and _err()
    assert lib.jenga_ln_modulate_tr_fp8(P, 256, P, P, P, P, P, P, 256, P, 10, 256, 1e-6, None) == E_CUDA


# ------------------------------------------------------------------ the restatement, pinned
def test_row_quantisation_rule_on_hand_made_rows():
    x = torch.zeros(4, 16, dtype=torch.bfloat16)
    x[0, :4] = torch.tensor([896.0, -3.0, 0.5, 1.0])          # scale 2: 448, -1.5, 0.25, 0.5
    x[2, :3] = torch.tensor([-4.0, 1.0, 0.0136])              # scale 4/448; 0.0136 * 112 = 1.5232 -> 1.5
    x[3, :2] = torch.tensor([1.0, 2.0 ** -16])                # / fl(1/448), which rounds up: just under 3.5 * 2^-9 -> subnormal 3 * 2^-9
    codes, scale = quantize_rows_ref(x)
    assert scale[0].item() == 2.0 and scale[1].item() == 1.0   # row 1 is all zero
    assert scale[2].item() == torch.tensor(4.0) / 448
    assert codes[0, :4].float().tolist() == [448.0, -1.5, 0.25, 0.5]
    assert (codes[1].float() == 0).all()
    assert codes[2, :2].float().tolist() == [-448.0, 112.0] and codes[2, 2].float().item() == 1.5
    assert codes[3, 0].float().item() == 448.0 and codes[3, 1].float().item() == 3 * 2.0 ** -9
    assert codes.view(torch.uint8)[0, 0].item() == 0x7E       # 448 is the largest finite e4m3, never NaN


def test_restatement_saturates_instead_of_making_nan():
    x = torch.tensor([[448.0, 1.0]], dtype=torch.float32)
    big = (x * 1.2).clamp(-448, 448).to(torch.float8_e4m3fn)
    assert big.float()[0, 0].item() == 448.0
    codes, _ = quantize_rows_ref(x.bfloat16())
    assert codes.float().isfinite().all()


def test_dense_shape_rule_and_switch_default():
    from jenga_b200 import dense as DN
    assert DN.linear_fp8_shape_ok(3072, 9216) and DN.linear_fp8_shape_ok(16, 8)
    assert not DN.linear_fp8_shape_ok(3000, 9216) and not DN.linear_fp8_shape_ok(3072, 100)
    import os
    assert DN.LINEAR_FP8 == (os.environ.get("JENGA_LINEAR_FP8", "0") == "1")
