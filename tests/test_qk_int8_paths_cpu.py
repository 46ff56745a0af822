"""C-ABI validation of the INT8 Q.K^T entry points that build the LSE and the Ulysses epilogue
(jenga_carved_attn_fwd_qk_int8_ex, jenga_quantize_q_int8_lse_shift), without a GPU: every bad argument
is refused with a negative code and a message before any CUDA call, and everything the older entry
points refuse is refused here too, except the two things the new one exists to build."""
import ctypes as C
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
from jenga_b200 import _lib  # noqa: E402
from jenga_b200._lib import JengaAttnSched, JengaQkInt8ExArgs, lib  # noqa: E402
from test_cabi_validation_cpu import E_CUDA, E_INVALID, E_UNSUPPORTED, _attn_args, _err  # noqa: E402
from test_qk_int8_cpu import _qk_args  # noqa: E402

SHIFT = 0x80000
P = 0x10000


def _ex_args(shift=None, **qk):
    x = JengaQkInt8ExArgs()
    x.base = _qk_args(**qk)
    x.q_lse_shift = shift
    return x


def _ex(attn=None, sched=None, **kw):
    return lib.jenga_carved_attn_fwd_qk_int8_ex(C.byref(attn or _attn_args()), C.byref(_ex_args(**kw)),
                                                C.byref(sched) if sched is not None else None, None)


def test_lse_without_the_shift_is_refused():
    rc = _ex(_attn_args(lse_out=0x60000))
    assert rc == E_UNSUPPORTED and "lse" in _err().lower(), (rc, _err())


@pytest.mark.parametrize("shift", [SHIFT + 2, SHIFT + 1])
def test_a_misaligned_shift_pointer_is_invalid(shift):
    rc = _ex(_attn_args(lse_out=0x60000), shift=shift)
    assert rc == E_INVALID and "aligned" in _err().lower(), (rc, _err())


@pytest.mark.parametrize("attn,qk,code,needle", [
    ({}, dict(q_i8=None), E_INVALID, "null"),
    ({}, dict(q_scale=None), E_INVALID, "null"),
    ({}, dict(k_i8=None), E_INVALID, "null"),
    ({}, dict(k_scale=None), E_INVALID, "null"),
    (dict(q=None), {}, E_INVALID, "null"),
    (dict(v_fp8=0x60000, v_fp8_amax=0x70000, dtype=_lib.JENGA_F16, out_dtype=_lib.JENGA_F16), {}, E_UNSUPPORTED, "fp8"),
    (dict(v_fp8=0x60000, v_fp8_amax=None), {}, E_UNSUPPORTED, "fp8"),
    ({}, dict(q_rows_padded=128), E_INVALID, "padded"),
    ({}, dict(kv_rows_padded=200), E_INVALID, "padded"),
    (dict(kv_rows=300), {}, E_INVALID, "padded"),
    ({}, dict(q_i8=0x20008), E_INVALID, "aligned"),
    ({}, dict(k_i8=0x40004), E_INVALID, "aligned"),
    ({}, dict(q_scale=0x30002), E_INVALID, "aligned"),
    ({}, dict(k_scale=0x50002), E_INVALID, "aligned"),
    (dict(head_dim=64), {}, E_UNSUPPORTED, "head_dim"),
    (dict(q_stride_s=250), {}, E_INVALID, "strides"),
    (dict(sp_world=9), {}, E_INVALID, "ulysses"),
])
def test_every_other_refusal_of_the_old_entry_points_holds(attn, qk, code, needle):
    for shift in (None, SHIFT):
        rc = _ex(_attn_args(**attn), shift=shift, **qk)
        assert rc == code, (shift, rc, _err())
        assert needle in _err().lower(), _err()
    if "sp_world" not in attn:   # the old entry point refuses every sp_world > 0 before checking it
        rc = lib.jenga_carved_attn_fwd_qk_int8(C.byref(_attn_args(**attn)), C.byref(_qk_args(**qk)), None)
        assert rc == code, (rc, _err())


def test_null_args_and_a_bad_schedule_are_refused():
    assert lib.jenga_carved_attn_fwd_qk_int8_ex(C.byref(_attn_args()), None, None, None) == E_INVALID
    assert "null" in _err()
    s = JengaAttnSched()
    s.workspace, s.workspace_bytes = 0x90000, 3                  # 4 * 1 * 2 * 2 = 16 bytes needed
    assert _ex(sched=s) == -4 and "workspace" in _err()           # JENGA_E_WORKSPACE
    s.workspace, s.workspace_bytes = 0x90002, 1 << 20
    assert _ex(sched=s) == E_INVALID and "aligned" in _err()


def test_the_old_entry_points_still_refuse_what_the_new_one_builds():
    peers = (C.c_uint64 * 2)(0x40000, 0x50000)
    sp = dict(sp_world=2, sp_rank=1, sp_heads_total=4, sp_rows=128, out_peers_host=C.addressof(peers))
    s = JengaAttnSched()
    s.workspace, s.workspace_bytes = 0x90000, 1 << 20
    for attn, needle in ((dict(lse_out=0x60000), "lse"), (sp, "ulysses")):
        rc = lib.jenga_carved_attn_fwd_qk_int8(C.byref(_attn_args(**attn)), C.byref(_qk_args()), None)
        assert rc == E_UNSUPPORTED and needle in _err().lower(), (rc, _err())
        rc = lib.jenga_carved_attn_fwd_sched(C.byref(_attn_args(**attn)), C.byref(_qk_args()), C.byref(s), None)
        assert rc == E_UNSUPPORTED and needle in _err().lower(), (rc, _err())


def test_without_a_device_the_new_entry_points_report_cuda_error():
    """The Ulysses epilogue and the LSE pass validation and reach CUDA: no refusal, no fallback."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    peers = (C.c_uint64 * 2)(0x40000, 0x50000)
    sp = dict(sp_world=2, sp_rank=1, sp_heads_total=4, sp_rows=128, out_peers_host=C.addressof(peers))
    assert _ex(_attn_args(**sp)) == E_CUDA and _err()
    assert _ex(_attn_args(lse_out=0x60000), shift=SHIFT) == E_CUDA and _err()
    assert lib.jenga_quantize_q_int8_lse_shift(P, 0, 1, 256, 2, 256 * 256, 256, 128, P, P, 256, P, P, None) == E_CUDA


#       x  dtype batch rows heads  s_b        s_s  s_h  k_mean out  out_rows scale shift
GOOD = (P, 0,    1,    256, 2,     256 * 256, 256, 128, P,     P,   256,     P,    P)


def _q(**over):
    names = ["x", "dtype", "batch", "rows", "heads", "sb", "ss", "sh", "k_mean", "out", "out_rows", "scale", "shift"]
    a = dict(zip(names, GOOD))
    a.update(over)
    return lib.jenga_quantize_q_int8_lse_shift(*[a[n] for n in names], None)


@pytest.mark.parametrize("over,code,needle", [
    (dict(x=None), E_INVALID, "null"),
    (dict(k_mean=None), E_INVALID, "null"),
    (dict(shift=None), E_INVALID, "null"),
    (dict(out=None), E_INVALID, "null"),
    (dict(scale=None), E_INVALID, "null"),
    (dict(dtype=_lib.JENGA_F32), E_INVALID, "dtype"),
    (dict(batch=0), E_INVALID, "shape"),
    (dict(heads=70000), E_INVALID, "shape"),
    (dict(rows=300, out_rows=300), E_INVALID, "out_rows"),
    (dict(rows=300), E_INVALID, "out_rows"),
    (dict(ss=250), E_INVALID, "alignment"),
    (dict(x=P + 8), E_INVALID, "alignment"),
    (dict(out=P + 8), E_INVALID, "alignment"),
    (dict(k_mean=P + 2), E_INVALID, "alignment"),
    (dict(shift=P + 2), E_INVALID, "alignment"),
])
def test_the_shift_quantiser_rejects_bad_arguments_before_any_cuda_call(over, code, needle):
    rc = _q(**over)
    assert rc == code, (rc, _err())
    assert needle in _err().lower(), _err()
