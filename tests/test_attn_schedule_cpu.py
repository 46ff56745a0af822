"""Argument validation of jenga_carved_attn_fwd_sched, without a GPU: a missing, misaligned or too
small workspace is refused before any CUDA call, and valid arguments reach CUDA (JENGA_E_CUDA here)."""
import ctypes as C

import pytest

from jenga_b200 import _lib
from jenga_b200._lib import JengaAttnArgs, JengaAttnSched, lib

E_INVALID, E_CUDA, E_WORKSPACE = -1, -3, -4


def _err():
    return lib.jenga_last_error().decode()


def _args():
    a = JengaAttnArgs()
    a.q = a.k = a.v = a.out = 0x10000
    a.dtype = a.out_dtype = _lib.JENGA_BF16
    a.batch, a.heads, a.head_dim = 1, 2, 128
    a.q_rows = a.kv_rows = 256
    for t in "qkvo":
        setattr(a, f"{t}_stride_b", 256 * 256)
        setattr(a, f"{t}_stride_s", 256)
        setattr(a, f"{t}_stride_h", 128)
    a.nq_sparse, a.nq_dense = 1, 1
    a.mask_bits, a.mask_words = 0x20000, 1
    a.sm_scale = 0.1
    a.kv_limit_sparse = a.q_limit_sparse = a.kv_limit_dense = 256
    return a


def test_workspace_size_query():
    assert lib.jenga_carved_attn_sched_workspace_bytes(1, 24, 900, 2) == 4 * 24 * 902
    assert lib.jenga_carved_attn_sched_workspace_bytes(2, 3, 37, 2) == 4 * 6 * 39
    assert lib.jenga_carved_attn_sched_workspace_bytes(0, 24, 900, 2) == 0


@pytest.mark.parametrize("ws,nbytes,code,needle", [
    (None, 16, E_INVALID, "null workspace"),
    (0x30002, 16, E_INVALID, "aligned"),
    (0x30000, 15, E_WORKSPACE, "workspace"),
])
def test_bad_workspace_is_refused_before_cuda(ws, nbytes, code, needle):
    s = JengaAttnSched(ws, nbytes)
    rc = lib.jenga_carved_attn_fwd_sched(C.byref(_args()), None, C.byref(s), None)
    assert rc == code, (rc, _err())
    assert needle in _err()


def test_null_schedule_and_bad_attention_arguments_are_refused():
    assert lib.jenga_carved_attn_fwd_sched(C.byref(_args()), None, None, None) == E_INVALID
    assert "sched" in _err()
    a = _args()
    a.head_dim = 64
    s = JengaAttnSched(0x30000, 16)
    assert lib.jenga_carved_attn_fwd_sched(C.byref(a), None, C.byref(s), None) == -2 and "head_dim" in _err()


def test_without_a_device_reports_cuda_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    s = JengaAttnSched(0x30000, 16)
    assert lib.jenga_carved_attn_fwd_sched(C.byref(_args()), None, C.byref(s), None) == E_CUDA and _err()
