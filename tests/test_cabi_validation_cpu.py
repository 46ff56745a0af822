"""C-ABI argument validation and error reporting, exercised WITHOUT a GPU: every entry point
must reject bad arguments with a negative code and a message before it touches CUDA, and the
host-only entry points must work."""
import ctypes as C

import numpy as np
import pytest

from jenga_b200 import _lib
from jenga_b200._lib import JengaAttnArgs, JengaSelectArgs, lib

E_INVALID, E_UNSUPPORTED, E_CUDA = -1, -2, -3


def _err():
    return lib.jenga_last_error().decode()


def _attn_args(**over):
    a = JengaAttnArgs()
    a.q = a.k = a.v = a.out = 0x10000  # never dereferenced on the validation paths
    a.dtype = _lib.JENGA_BF16
    a.out_dtype = _lib.JENGA_BF16
    a.batch, a.heads, a.head_dim = 1, 2, 128
    a.q_rows = a.kv_rows = 256
    for t in "qkvo":
        setattr(a, f"{t}_stride_b", 256 * 256)
        setattr(a, f"{t}_stride_s", 256)
        setattr(a, f"{t}_stride_h", 128)
    a.nq_sparse, a.nq_dense = 0, 2
    a.sm_scale = 0.1
    a.kv_limit_sparse = a.q_limit_sparse = a.kv_limit_dense = 256
    for k, v in over.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("over,code,needle", [
    (dict(head_dim=64), E_UNSUPPORTED, "head_dim"),
    (dict(dtype=_lib.JENGA_F32), E_INVALID, "dtype"),
    (dict(q=None), E_INVALID, "null"),
    (dict(nq_sparse=0, nq_dense=0), E_INVALID, "query blocks"),
    (dict(nq_dense=3), E_INVALID, "exceed"),
    (dict(q_stride_s=250), E_INVALID, "strides"),
    (dict(q=0x10008), E_INVALID, "aligned"),
    (dict(sm_scale=0.0), E_INVALID, "sm_scale"),
    (dict(nq_sparse=1, nq_dense=1, mask_bits=None), E_INVALID, "mask_bits"),
    (dict(out_dtype=_lib.JENGA_F16), E_INVALID, "out_dtype"),
    (dict(sp_world=9), E_INVALID, "Ulysses"),
])
def test_attention_argument_validation(over, code, needle):
    a = _attn_args(**over)
    rc = lib.jenga_carved_attn_fwd(C.byref(a), None)
    assert rc == code, (rc, _err())
    assert needle.lower() in _err().lower(), _err()


def test_attention_without_a_device_reports_cuda_error_not_a_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    rc = lib.jenga_carved_attn_fwd(C.byref(_attn_args()), None)
    assert rc == E_CUDA and _err()


def test_select_and_pool_validation():
    s = JengaSelectArgs()
    assert lib.jenga_select_blocks(C.byref(s), None) == E_INVALID
    s.q_pool = s.k_pool = s.out_bits = 0x1000
    s.dtype, s.batch_heads, s.head_dim, s.nq, s.nk_pool, s.n_img, s.nb = 0, 1, 128, 4, 4, 4, 6
    s.mask_words = 0
    assert lib.jenga_select_blocks(C.byref(s), None) == E_INVALID and "mask_words" in _err()
    # score workspace: size query, and a too-small workspace is refused before anything launches
    assert lib.jenga_select_blocks_workspace_bytes(24, 900, 900) == 24 * 900 * 900 * 4
    assert lib.jenga_select_blocks_workspace_bytes(0, 900, 900) == 0
    s.mask_words, s.top_k, s.p_threshold = 1, 1, 0.5
    s.workspace, s.workspace_bytes = 0x2000, 4 * 4 * 4 - 1
    assert lib.jenga_select_blocks(C.byref(s), None) == -4 and "workspace" in _err()  # JENGA_E_WORKSPACE
    assert lib.jenga_block_pool(None, None, None, 0, 0, 1, 1, 128, 128, 0, 0, 0, 1, None) == E_INVALID
    # n_blocks beyond the rows
    assert lib.jenga_block_pool(0x1000, 0x1000, None, 0, 0, 1, 1, 128, 128, 16384, 128, 128, 2, None) == E_INVALID
    assert lib.jenga_gather_rows(0x1000, 0x1000, 0x1000, 4, 4, 24, 1, 96, 96, None) == E_INVALID  # row not x16
    assert lib.jenga_mask_onehot_to_bits(0x1000, 0x1000, 4, 40, 1, None) == E_INVALID            # words too small
    assert lib.jenga_copy2d_async(0x1000, 8, 0x1000, 16, 16, 4, 0, None) == E_INVALID               # pitch < width


def test_gilbert_host_entry_points_validate_and_run():
    assert lib.jenga_gilbert_mapping_host(0, 4, 4, 0, None, None) == E_INVALID
    a = np.zeros(8, dtype=np.int64)
    assert lib.jenga_gilbert_mapping_host(0, 2, 4, 0, a.ctypes.data, None) == E_INVALID and "empty" in _err()
    assert lib.jenga_gilbert_mapping_host(1, 2, 4, 0, a.ctypes.data, None) == 0
    assert sorted(a.tolist()) == list(range(8))
    assert lib.jenga_gilbert_xyz2d(5, 0, 0, 4, 4, 4) == -1  # out of bounds
    assert lib.jenga_gilbert_block_neighbors_host(1, 2, 4, 0, 0, a.ctypes.data) == E_INVALID


def _hy_args(**over):
    from jenga_b200._lib import JengaHyPrologueArgs
    a = JengaHyPrologueArgs()
    a.img_qkv = a.txt_qkv = a.q = a.k = a.v = 0x10000
    a.dtype, a.batch, a.heads, a.head_dim = _lib.JENGA_BF16, 1, 2, 128
    a.img_tokens, a.txt_tokens = 256, 64
    a.img_stride_b, a.img_stride_s, a.img_stride_w, a.img_stride_h = 256 * 768, 768, 256, 128
    a.txt_stride_b, a.txt_stride_s, a.txt_stride_w, a.txt_stride_h = 64 * 768, 768, 256, 128
    a.eps = 1e-6
    for k, v in over.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("over,code,needle", [
    (dict(q=None), E_INVALID, "null"),
    (dict(dtype=_lib.JENGA_F32), E_INVALID, "dtype"),
    (dict(head_dim=64), E_UNSUPPORTED, "head_dim"),
    (dict(img_tokens=0), E_INVALID, "shape"),
    (dict(txt_qkv=None), E_INVALID, "txt_qkv"),
    (dict(w_img_q=0x2000), E_INVALID, "norm weights"),
    (dict(rope_cos=0x2000), E_INVALID, "cos and sin"),
    (dict(q_pool=0x2000), E_INVALID, "q_pool"),
    (dict(img_stride_s=770), E_INVALID, "strides"),
])
def test_hy_prologue_argument_validation(over, code, needle):
    """jenga_hy_prologue (RMSNorm+RoPE+cat+pool) rejects bad arguments before any launch."""
    assert lib.jenga_hy_prologue(C.byref(_hy_args(**over)), None) == code
    assert needle in _err()


def test_wan_prologue_and_ulysses_scatter_validation():
    from jenga_b200._lib import JengaUlyssesScatterArgs, JengaWanPrologueArgs
    w = JengaWanPrologueArgs()
    assert lib.jenga_wan_prologue(C.byref(w), None) == E_INVALID and "null" in _err()
    w.x = w.out = 0x10000
    w.batch, w.heads, w.head_dim, w.tokens = 1, 12, 64, 128
    assert lib.jenga_wan_prologue(C.byref(w), None) == E_UNSUPPORTED and "head_dim" in _err()
    w.head_dim, w.tokens = 128, 0
    assert lib.jenga_wan_prologue(C.byref(w), None) == E_INVALID and "shape" in _err()
    w.tokens, w.x_dtype = 128, _lib.JENGA_F16
    assert lib.jenga_wan_prologue(C.byref(w), None) == E_INVALID and "dtypes" in _err()
    w.x_dtype, w.w_dtype = _lib.JENGA_F32, _lib.JENGA_BF16
    w.freqs, w.freq_rows, w.grid_f, w.grid_h, w.grid_w = 0x2000, 8, 21, 30, 52   # needs >= 52 rows
    assert lib.jenga_wan_prologue(C.byref(w), None) == E_INVALID and "frequency table" in _err()

    s = JengaUlyssesScatterArgs()
    assert lib.jenga_ulysses_scatter(C.byref(s), None) == E_INVALID and "null" in _err()


# ------------------------------------------------------------------ round-2 entry points
def test_round2_entry_points_validate_before_touching_cuda():
    """step cache, dense chains, FP8 quantisation, ProRes switch, device gilbert: bad arguments are
    rejected with a negative code and a message (no CUDA call is reached)."""
    P = 0x10000   # never dereferenced on the validation paths
    cases = [
        (lambda: lib.jenga_residual_apply(None, P, 16, _lib.JENGA_BF16, None), E_INVALID, "null"),
        (lambda: lib.jenga_residual_apply(P, P, 16, 7, None), E_INVALID, "dtype"),
        (lambda: lib.jenga_residual_apply(P + 8, P, 16, _lib.JENGA_BF16, None), E_INVALID, "aligned"),
        (lambda: lib.jenga_residual_store(P, P, None, 16, _lib.JENGA_F32, None), E_INVALID, "null"),
        (lambda: lib.jenga_ln_modulate(P, 3072, P, P, P, 3072, 10, 3070, 1e-6, None), E_INVALID, "multiples of 8"),
        (lambda: lib.jenga_ln_modulate(P, 3072, None, P, P, 3072, 10, 3072, 1e-6, None), E_INVALID, "null"),
        (lambda: lib.jenga_ln_modulate(P, 8192, P, P, P, 8192, 10, 8192, 1e-6, None), E_UNSUPPORTED, "6144"),
        (lambda: lib.jenga_gate_residual(P, 64, P, 64, P, P, 64, 0, 64, None), E_INVALID, "shape"),
        (lambda: lib.jenga_gelu_tanh(P, 64, P + 2, 64, 4, 64, None), E_INVALID, "aligned"),
        (lambda: lib.jenga_quantize_v_fp8(P, _lib.JENGA_F32, 1, 128, 2, 128 * 256, 256, 128, P, P, None), E_INVALID, "dtype"),
        (lambda: lib.jenga_quantize_v_fp8(P, _lib.JENGA_BF16, 1, 128, 2, 128 * 256, 250, 128, P, P, None), E_INVALID, "alignment"),
        (lambda: lib.jenga_prores_switch(P, P, None, P, 16, 4, 4, 4, 4, 8, 8, 0.1, 0.5, None), E_INVALID, "null"),
        (lambda: lib.jenga_prores_switch(P, P, P, P, 16, 4, 0, 4, 4, 8, 8, 0.1, 0.5, None), E_INVALID, "shape"),
        (lambda: lib.jenga_gilbert_mapping_device(0, 4, 4, 0, P, P, None), E_INVALID, "empty"),
        (lambda: lib.jenga_gilbert_mapping_device(2, 4, 4, 0, None, None, None), E_INVALID, "no output"),
        (lambda: lib.jenga_block_neighbor_bits_device(2, 4, 4, 128, P, P, 0, None), E_INVALID, "words"),
    ]
    for fn, code, needle in cases:
        rc = fn()
        assert rc == code, (rc, _err())
        assert needle.lower() in _err().lower(), (needle, _err())
    a = _lib.JengaTeaCacheArgs()
    assert lib.jenga_teacache_gate(C.byref(a), None) == E_INVALID and "null" in _err()
    a.cur = a.prev = a.state = a.flag = P
    a.n, a.n_coeff, a.dtype = 100, 9, _lib.JENGA_F32
    assert lib.jenga_teacache_gate(C.byref(a), None) == E_INVALID and "sizes" in _err()
    a.n_coeff, a.dtype = 5, _lib.JENGA_BF16
    assert lib.jenga_teacache_gate(C.byref(a), None) == E_UNSUPPORTED and "f32" in _err()


def test_fp8_and_head_group_arguments_of_the_attention_entry_point():
    """ABI 2 fields: the FP8 P.V variant needs its amax array, bf16 and the default generation; a
    Ulysses head sub-group must lie inside sp_heads_total."""
    a = _attn_args(v_fp8=0x20000)
    assert lib.jenga_carved_attn_fwd(C.byref(a), None) == E_UNSUPPORTED and "fp8" in _err().lower()
    a = _attn_args(v_fp8=0x20000, v_fp8_amax=0x30000, dtype=_lib.JENGA_F16, out_dtype=_lib.JENGA_F16)
    assert lib.jenga_carved_attn_fwd(C.byref(a), None) == E_UNSUPPORTED
    peers = (C.c_uint64 * 2)(0x40000, 0x50000)
    a = _attn_args(sp_world=2, sp_rank=1, sp_heads_total=4, sp_rows=128, out_peers_host=C.addressof(peers),
                   sp_head_base=3, sp_head_base_valid=1)       # heads [3, 5) of 4
    assert lib.jenga_carved_attn_fwd(C.byref(a), None) == E_INVALID and "head range" in _err()


def _peer_array(world, bad_rank, bad):
    """Host array of `world` plausible device addresses; entry `bad_rank` is NULL or 8 bytes off."""
    vals = [0x100000 * (r + 1) for r in range(world)]
    if bad_rank is not None:
        vals[bad_rank] = 0 if bad == "null" else vals[bad_rank] + 8
    return (C.c_uint64 * world)(*vals)


@pytest.mark.parametrize("world,bad_rank", [(1, 0), (2, 1), (8, 0), (8, 7)])
@pytest.mark.parametrize("bad", ["null", "misaligned"])
def test_ulysses_epilogue_rejects_bad_peer_entries(world, bad_rank, bad):
    """Every out_peers_host[0..sp_world) entry is checked before any CUDA call, with a NULL `out`
    as the fused Ulysses path passes it."""
    peers = _peer_array(world, bad_rank, bad)
    a = _attn_args(out=None, sp_world=world, sp_rank=world - 1, sp_heads_total=2 * world, sp_rows=128,
                   out_peers_host=C.addressof(peers))
    assert lib.jenga_carved_attn_fwd(C.byref(a), None) == E_INVALID, _err()
    assert f"out_peers_host[{bad_rank}]" in _err(), _err()
    sched = _lib.JengaAttnSched(0x20000, 1 << 20)
    assert lib.jenga_carved_attn_fwd_sched(C.byref(a), None, C.byref(sched), None) == E_INVALID, _err()
    assert f"out_peers_host[{bad_rank}]" in _err(), _err()


@pytest.mark.parametrize("world,bad_rank", [(1, 0), (2, 1), (8, 0), (8, 7)])
@pytest.mark.parametrize("bad", ["null", "misaligned"])
def test_ulysses_scatter_rejects_bad_peer_entries(world, bad_rank, bad):
    a = _lib.JengaUlyssesScatterArgs()
    P = 0x10000
    a.x = (C.c_void_p * 3)(P, P, P)
    a.x_stride_s = 24 * 128
    a.world, a.rank, a.heads, a.head_dim, a.n_loc, a.n_text = world, 0, 24, 128, 144, 0
    peers = _peer_array(world, bad_rank, bad)
    a.peer_qkv_host = C.addressof(peers)
    assert lib.jenga_ulysses_scatter(C.byref(a), None) == E_INVALID, _err()
    assert f"peer_qkv_host[{bad_rank}]" in _err(), _err()


def test_good_peer_entries_pass_validation_without_a_device():
    """Control for the two tests above: the same arguments with every entry good get past the
    validation and fail only at the first CUDA call."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the addresses are not real allocations")
    for world in (1, 8):
        peers = _peer_array(world, None, None)
        a = _attn_args(out=None, sp_world=world, sp_rank=0, sp_heads_total=2 * world, sp_rows=128,
                       out_peers_host=C.addressof(peers))
        assert lib.jenga_carved_attn_fwd(C.byref(a), None) == E_CUDA, _err()
        s = _lib.JengaUlyssesScatterArgs()
        s.x = (C.c_void_p * 3)(0x10000, 0x10000, 0x10000)
        s.x_stride_s = 24 * 128
        s.world, s.rank, s.heads, s.head_dim, s.n_loc, s.n_text = world, 0, 24, 128, 144, 0
        s.peer_qkv_host = C.addressof(peers)
        assert lib.jenga_ulysses_scatter(C.byref(s), None) == E_CUDA, _err()


def test_scatter_head_group_validation():
    a = _lib.JengaUlyssesScatterArgs()
    P = 0x10000
    a.x = (C.c_void_p * 3)(P, P, P)
    a.x_stride_s = 4 * 128
    a.world, a.rank, a.heads, a.head_dim, a.n_loc, a.n_text = 2, 0, 4, 128, 128, 0
    peers = (C.c_uint64 * 2)(P, P)
    a.peer_qkv_host = C.addressof(peers)
    a.head_begin, a.head_count = 1, 2                           # local heads [1, 3) of 2
    assert lib.jenga_ulysses_scatter(C.byref(a), None) == E_INVALID and "head group" in _err()
