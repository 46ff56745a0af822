"""f-3 (opt-in) INT8 Q.K^T variant, without a GPU: argument validation of its two C-ABI entry points,
no fallback without a device, and a CPU model of its error that pins the tolerance row of the GPU
tests (tests/test_qk_int8_gpu.py).

The model quantises with `quantize_ref`, a torch restatement of jenga_quantize_int8 (the oracle of
the GPU quantiser test), and runs exact fp64 attention on the dequantised operands over a random
~30 % block mask of bench.synth_tokens (regime P) tokens: 2 heads, 6 query blocks, 96 key blocks.
Errors are relative to fp64 attention on the unquantised operands, in units of the output RMS:
  INT8 Q (per 64 rows) and K (per 128 keys), K smoothed   ~1e-2 mean, ~0.07 max
K with a common channel bias (8 channels offset by 3-8, times three, as DiT keys carry) leaves the
smoothed path there but pushes the unsmoothed one to ~5e-2 / ~0.3.  The GPU row, mean <= 2e-2 and
max <= 0.15, is about twice the smoothed model: it covers the kernel's own fp32 and bf16 roundings.
"""
import ctypes as C
import math
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
from jenga_b200 import _lib  # noqa: E402
from jenga_b200._lib import JengaQkInt8Args, lib  # noqa: E402
from test_cabi_validation_cpu import E_CUDA, E_INVALID, E_UNSUPPORTED, _attn_args, _err  # noqa: E402

TOL_MEAN, TOL_MAX = 2e-2, 0.15           # the qk_int8 row of the GPU tests
KBIAS = torch.zeros(128, dtype=torch.float64)
KBIAS[:8] = torch.tensor([6.0, -5, 4, 8, -7, 5, 3, -6])


def quantize_ref(x: torch.Tensor, group_rows: int, smooth: bool):
    """torch restatement of jenga_quantize_int8 in fp32.  x [B,S,H,128] -> (codes int8
    [B, round_up(S,128), H, 128], scale f32 [B*H, round_up(S,128) / group_rows], mean f32 [B*H,128])."""
    B, S, H, D = x.shape
    Sp = (S + 127) // 128 * 128
    xf = torch.zeros(B, Sp, H, D, dtype=torch.float32, device=x.device)
    xf[:, :S] = x.float()
    mean = (x.float().sum(1) / S) if smooth else torch.zeros(B, H, D, dtype=torch.float32, device=x.device)
    y = (xf - mean[:, None]).permute(0, 2, 1, 3).reshape(B * H, Sp // group_rows, group_rows, D)
    scale = y.abs().amax(dim=(2, 3)) / 127
    s = scale[:, :, None, None]
    codes = torch.where(s > 0, torch.round(y / s).clamp(-127, 127), torch.zeros_like(y))
    codes = codes.reshape(B, H, Sp, D).permute(0, 2, 1, 3).to(torch.int8).contiguous()
    return codes, scale, mean.reshape(B * H, D)


def dequantize_ref(codes, scale, group_rows):
    """codes [B,Sp,H,D] int8, scale [B*H, Sp/g] -> fp64 [B,Sp,H,D] of (x - mean)."""
    B, Sp, H, D = codes.shape
    s = scale.double().reshape(B, H, Sp // group_rows).repeat_interleave(group_rows, -1).permute(0, 2, 1)
    return codes.double() * s[..., None]


# ------------------------------------------------------------------ argument validation
def _qk_args(**over):
    x = JengaQkInt8Args()
    x.q_i8, x.q_scale, x.k_i8, x.k_scale = 0x20000, 0x30000, 0x40000, 0x50000
    x.q_rows_padded = x.kv_rows_padded = 256
    for k, v in over.items():
        setattr(x, k, v)
    return x


@pytest.mark.parametrize("attn,qk,code,needle", [
    ({}, dict(q_i8=None), E_INVALID, "null"),
    ({}, dict(k_scale=None), E_INVALID, "null"),
    (dict(lse_out=0x60000), {}, E_UNSUPPORTED, "lse"),
    (dict(v_fp8=0x60000, v_fp8_amax=0x70000, dtype=_lib.JENGA_F16, out_dtype=_lib.JENGA_F16), {}, E_UNSUPPORTED, "fp8"),
    ({}, dict(q_rows_padded=128), E_INVALID, "padded"),
    ({}, dict(kv_rows_padded=200), E_INVALID, "padded"),
    (dict(kv_rows=300), {}, E_INVALID, "padded"),
    ({}, dict(q_i8=0x20008), E_INVALID, "aligned"),
    ({}, dict(k_scale=0x50002), E_INVALID, "aligned"),
])
def test_qk_int8_entry_point_rejects_what_it_does_not_build(attn, qk, code, needle):
    rc = lib.jenga_carved_attn_fwd_qk_int8(C.byref(_attn_args(**attn)), C.byref(_qk_args(**qk)), None)
    assert rc == code, (rc, _err())
    assert needle in _err().lower(), _err()


def test_qk_int8_entry_point_rejects_null_args_and_the_ulysses_epilogue():
    assert lib.jenga_carved_attn_fwd_qk_int8(C.byref(_attn_args()), None, None) == E_INVALID and "null" in _err()
    peers = (C.c_uint64 * 2)(0x40000, 0x50000)
    a = _attn_args(sp_world=2, sp_rank=1, sp_heads_total=4, sp_rows=128, out_peers_host=C.addressof(peers))
    rc = lib.jenga_carved_attn_fwd_qk_int8(C.byref(a), C.byref(_qk_args()), None)
    assert rc == E_UNSUPPORTED and "ulysses" in _err().lower(), (rc, _err())


P = 0x10000


@pytest.mark.parametrize("args,code,needle", [
    ((None, 0, 1, 256, 2, 256 * 256, 256, 128, 64, 0, None, P, 256, P), E_INVALID, "null"),
    ((P, 0, 1, 256, 2, 256 * 256, 256, 128, 128, 1, None, P, 256, P), E_INVALID, "null"),    # smooth needs mean
    ((P, 0, 1, 256, 2, 256 * 256, 256, 128, 64, 0, None, None, 256, P), E_INVALID, "null"),
    ((P, _lib.JENGA_F32, 1, 256, 2, 256 * 256, 256, 128, 64, 0, None, P, 256, P), E_INVALID, "dtype"),
    ((P, 0, 1, 256, 2, 256 * 256, 256, 128, 32, 0, None, P, 256, P), E_UNSUPPORTED, "group_rows"),
    ((P, 0, 0, 256, 2, 256 * 256, 256, 128, 64, 0, None, P, 256, P), E_INVALID, "shape"),
    ((P, 0, 1, 300, 2, 256 * 256, 256, 128, 64, 0, None, P, 300, P), E_INVALID, "out_rows"),
    ((P, 0, 1, 300, 2, 256 * 256, 256, 128, 64, 0, None, P, 256, P), E_INVALID, "out_rows"),
    ((P, 0, 1, 256, 2, 256 * 256, 250, 128, 64, 0, None, P, 256, P), E_INVALID, "alignment"),
    ((P + 8, 0, 1, 256, 2, 256 * 256, 256, 128, 64, 0, None, P, 256, P), E_INVALID, "alignment"),
    ((P, 0, 1, 256, 2, 256 * 256, 256, 128, 64, 0, None, P + 8, 256, P), E_INVALID, "alignment"),
])
def test_quantize_int8_argument_validation(args, code, needle):
    rc = lib.jenga_quantize_int8(*args, None)
    assert rc == code, (rc, _err())
    assert needle in _err().lower(), _err()


def test_without_a_device_both_entry_points_report_cuda_error_not_a_fallback():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert lib.jenga_carved_attn_fwd_qk_int8(C.byref(_attn_args()), C.byref(_qk_args()), None) == E_CUDA and _err()
    assert lib.jenga_quantize_int8(P, 0, 1, 256, 2, 256 * 256, 256, 128, 128, 1, P, P, 256, P, None) == E_CUDA
    assert _err()


# ------------------------------------------------------------------ the restatement itself
def test_restatement_codes_scales_and_padding():
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(1, 200, 2, 128, generator=g) + 3.0).bfloat16()
    codes, scale, mean = quantize_ref(x, 128, True)
    assert codes.shape == (1, 256, 2, 128) and scale.shape == (2, 2)
    assert codes.abs().max().item() == 127
    assert torch.allclose(mean, x.float().mean(1).reshape(2, 128))
    back = dequantize_ref(codes, scale, 128)[:, :200]
    err = (back - (x.double() - mean.double().reshape(1, 1, 2, 128))).abs()
    assert err.max().item() <= scale.double().max().item() / 2 * (1 + 1e-6)
    pad = torch.round(-mean.reshape(1, 2, 128) / scale[:, 1].reshape(1, 2, 1)).clamp(-127, 127)
    assert torch.equal(codes[:, 200:].float(), pad[:, None].expand(1, 56, 2, 128))
    # no smoothing: scale = absmax / 127 of each 64-row group, exactly; pad rows are code 0
    q_codes, q_scale, _ = quantize_ref(x, 64, False)
    xg = torch.zeros(1, 256, 2, 128)
    xg[:, :200] = x.float()
    want = xg[0].permute(1, 0, 2).reshape(2, 4, 64 * 128).abs().amax(-1) / 127
    assert torch.equal(q_scale, want)
    assert (q_codes[:, 200:] == 0).all()


# ------------------------------------------------------------------ CPU error model
H_M, NQB, NKB = 2, 6, 96


def _model_inputs(kbias_gain):
    import bench
    dev = torch.device("cpu")
    S = NKB * 128
    q = bench.synth_tokens(S, H_M, dev, 11)[:, :NQB * 128]                              # [1, Sq, H, D] bf16
    k = (bench.synth_tokens(S, H_M, dev, 12).double() + kbias_gain * KBIAS).bfloat16()
    v = torch.randn(1, S, H_M, 128, generator=torch.Generator().manual_seed(13), dtype=torch.float64)
    blk = torch.rand(H_M, NQB, NKB, generator=torch.Generator().manual_seed(3)) < 0.3
    live = blk.repeat_interleave(128, 1).repeat_interleave(128, 2)                      # [H, Sq, S]
    return q, k, v, live


def _attn64(q, k, v, live):
    """q,k,v [1,S,H,D] (any float) -> fp64 [H, Sq, D]."""
    q, k, v = (t[0].transpose(0, 1).double() for t in (q, k, v))
    s = (q @ k.transpose(-1, -2) / math.sqrt(128)).masked_fill(~live, float("-inf"))
    return torch.softmax(s, -1) @ v


def _model_error(kbias_gain, smooth):
    q, k, v, live = _model_inputs(kbias_gain)
    truth = _attn64(q, k, v, live)
    qc, qs, _ = quantize_ref(q, 64, False)
    kc, ks, _ = quantize_ref(k, 128, smooth)
    got = _attn64(dequantize_ref(qc, qs, 64), dequantize_ref(kc, ks, 128), v, live)
    rms = truth.pow(2).mean().sqrt()
    e = (got - truth).abs() / rms
    return e.mean().item(), e.max().item()


@pytest.mark.parametrize("gain", [0.0, 1.0, 3.0])
def test_smoothed_int8_model_stays_inside_the_gpu_tolerance_row(gain):
    mean, mx = _model_error(gain, smooth=True)
    print(f"\n[int8 model, K bias x{gain:g}, smoothed] mean {mean:.2e} max {mx:.2e}")
    assert 5e-3 <= mean <= 1.5e-2 and mx <= 0.1           # the modelled ~1e-2 / ~0.07
    assert 2 * mean <= TOL_MEAN + 1e-3 and mx <= TOL_MAX


def test_unsmoothed_int8_model_leaves_the_row_on_biased_keys():
    mean0, max0 = _model_error(0.0, smooth=False)
    mean3, max3 = _model_error(3.0, smooth=False)
    print(f"\n[int8 model, no smoothing] unbiased mean {mean0:.2e} max {max0:.2e}; K bias x3 mean {mean3:.2e} max {max3:.2e}")
    assert mean0 <= 1.5e-2                                 # without a bias, smoothing changes little
    assert mean3 > TOL_MEAN and max3 > TOL_MAX             # with it, the unsmoothed path fails the row
