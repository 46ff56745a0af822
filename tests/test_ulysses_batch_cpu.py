"""Several samples per call on the sequence-parallel paths, without a GPU.

* C-ABI validation of jenga_ulysses_scatter_batched, before any CUDA call: null pointers, the batch,
  the batch strides, and every rule of the two unbatched entry points it shares.
* hyi2v_sp.get_cu_seqlens builds the 2B+1 entries of hyvideo_i2v/modules/attenion.py:34-57.
* gloo ranks at world 2: UlyssesCarvedAttention with the oracle operator at B = 2 and 3, over the divisible
  and the ragged head split; every sample equals the single-process operator on that sample alone.
"""
import ctypes as C
import os
import sys
from pathlib import Path

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(HERE / "golden"))

E_INVALID, E_CUDA = -1, -3


# ------------------------------------------------------------------------------------------------
# C ABI
# ------------------------------------------------------------------------------------------------
def _batch_args(world=2, heads=4, batch=2):
    from jenga_b200._lib import JengaUlyssesScatterBatchArgs
    a = JengaUlyssesScatterBatchArgs()
    a.base.x = (C.c_void_p * 3)(0x10000, 0x20000, 0x30000)     # never dereferenced on the validation paths
    a.base.x_stride_s = heads * 128
    a.base.world, a.base.rank, a.base.heads, a.base.head_dim = world, 0, heads, 128
    a.base.n_loc, a.base.n_text = 128, 0
    peers = (C.c_uint64 * 9)(*[0x100000 * (i + 1) for i in range(9)])
    a.base.peer_qkv_host = C.addressof(peers)
    a.batch, a.x_stride_b, a.joint_stride_b = batch, 256 * heads * 128, 0
    return a, peers


@pytest.mark.parametrize("case,needle", [
    ("null_args", "null pointer"),
    ("null_x", "null pointer"),
    ("null_peers", "null pointer"),
    ("batch0", "batch 0"),
    ("batch_neg", "batch -2"),
    ("x_stride_b", "multiples of 8"),
    ("joint_stride_b", "multiples of 8"),
    ("world9", "bad shape"),
    ("heads_indivisible", "bad shape"),
    ("head_group", "head group"),
    ("peer_unaligned", "not 16-byte aligned"),
    ("joint_missing", "joint tensors missing"),
    ("ragged_start", "from 0 to heads"),
    ("ragged_decreasing", "decrease"),
    ("ragged_too_large", "exceeds the 2 slots"),
    ("ragged_world9", "bad shape"),
    ("ragged_slot_range", "slot range"),
])
def test_scatter_batched_validation(case, needle):
    from jenga_b200._lib import lib
    a, peers = _batch_args()
    off = None
    if case.startswith("ragged"):
        a, peers = _batch_args(world=3, heads=5)
        off = [0, 2, 4, 5]
    if case == "null_x":
        a.base.x[1] = None
    elif case == "null_peers":
        a.base.peer_qkv_host = None
    elif case == "batch0":
        a.batch = 0
    elif case == "batch_neg":
        a.batch = -2
    elif case == "x_stride_b":
        a.x_stride_b = 4 * 128 * 256 + 4
    elif case == "joint_stride_b":
        a.joint_stride_b = 12
    elif case == "world9":
        a.base.world, a.base.heads = 9, 18
    elif case == "heads_indivisible":
        a.base.heads = 5
    elif case == "head_group":
        a.base.head_begin, a.base.head_count = 1, 2
    elif case == "peer_unaligned":
        peers[1] = 0x100008
    elif case == "joint_missing":
        a.base.n_text = 256
    elif case == "ragged_start":
        off = [1, 2, 4, 5]
    elif case == "ragged_decreasing":
        off = [0, 2, 1, 5]
    elif case == "ragged_too_large":
        off = [0, 1, 2, 5]
    elif case == "ragged_world9":
        a.base.world, a.base.heads = 9, 12
        off = [0, 2, 4, 6, 7, 8, 9, 10, 11, 12]
    elif case == "ragged_slot_range":
        a.base.head_begin, a.base.head_count = 1, 2
    c_off = None if off is None else (C.c_int32 * len(off))(*off)
    rc = lib.jenga_ulysses_scatter_batched(None if case == "null_args" else C.byref(a), c_off, None)
    msg = lib.jenga_last_error().decode()
    assert rc == E_INVALID and needle in msg, (rc, msg)


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("batch", [1, 3])
def test_scatter_batched_accepts_valid_arguments_up_to_the_launch(ragged, batch):
    """Valid arguments pass validation; without a device the call fails at the launch (a CUDA error)."""
    if torch.cuda.is_available():
        pytest.skip("GPU present: the launch would dereference the dummy pointers")
    from jenga_b200._lib import lib
    a, peers = _batch_args(world=3, heads=5, batch=batch) if ragged else _batch_args(batch=batch)
    c_off = (C.c_int32 * 4)(0, 2, 4, 5) if ragged else None
    rc = lib.jenga_ulysses_scatter_batched(C.byref(a), c_off, None)
    assert rc == E_CUDA, (rc, lib.jenga_last_error().decode())


# ------------------------------------------------------------------------------------------------
# the sharded I2V forward's cu_seqlens
# ------------------------------------------------------------------------------------------------
def _ref_get_cu_seqlens(text_mask, img_len):
    """hyvideo_i2v/modules/attenion.py:34-57, restated on the CPU"""
    batch_size = text_mask.shape[0]
    text_len = text_mask.sum(dim=1)
    max_len = text_mask.shape[1] + img_len
    cu_seqlens = torch.zeros([2 * batch_size + 1], dtype=torch.int32)
    for i in range(batch_size):
        s = text_len[i] + img_len
        cu_seqlens[2 * i + 1] = i * max_len + s
        cu_seqlens[2 * i + 2] = (i + 1) * max_len
    return cu_seqlens


@pytest.mark.parametrize("B", [1, 2, 3])
def test_get_cu_seqlens_matches_the_reference(B):
    from jenga_b200.hyi2v_sp import get_cu_seqlens
    g = torch.Generator().manual_seed(B)
    T, img_len = 400, 1800
    valid = torch.randint(1, T + 1, (B,), generator=g)
    text_mask = (torch.arange(T)[None] < valid[:, None]).long()
    got = get_cu_seqlens(text_mask, img_len, "cpu")
    assert got.dtype == torch.int32 and got.shape == (2 * B + 1,)
    assert torch.equal(got, _ref_get_cu_seqlens(text_mask, img_len))


# ------------------------------------------------------------------------------------------------
# UlyssesCarvedAttention over gloo at B > 1
# ------------------------------------------------------------------------------------------------
T, VALID, TOP_K, N_IMG, P = 256, 180, 2, 384, 2     # n_loc = 192 straddles the second 128-row block


def _inputs(H, B):
    import synth
    nb = N_IMG // 128 + T // 128
    qs, ks, vs = [], [], []
    for b in range(B):
        s = 900 + 10 * b
        qs.append(synth.peaky(H, nb, 128, 2.0, s).transpose(1, 2).contiguous().bfloat16())   # [1, S, H, D]
        ks.append(synth.peaky(H, nb, 128, 2.0, s + 1).transpose(1, 2).contiguous().bfloat16())
        vs.append(synth.normal((1, nb * 128, H, 128), s + 2).bfloat16())
    return torch.cat(qs), torch.cat(ks), torch.cat(vs), synth.band_neighbours(N_IMG // 128)


def _oracle_attn(q, k, v, **kw):
    from oracle import attention_oracle as orc
    kw.pop("block_size_M", None)
    kw.pop("block_size_N", None)
    return orc.block_sparse_attention(q, k, v, variant="hyvideo", **kw)


def _worker(rank, world, H, B, ragged, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from jenga_b200 import ulysses as U
        from jenga_b200.hyi2v_sp import get_cu_seqlens
        U.RAGGED_HEADS = ragged
        q, k, v, nbr = _inputs(H, B)
        n = N_IMG // world
        sl = slice(rank * n, (rank + 1) * n)
        ql, kl, vl = (torch.cat([x[:, sl], x[:, N_IMG:]], 1) for x in (q, k, v))
        # what the sharded forward builds: 2B+1 local entries, every sample with the same prompt
        cu = get_cu_seqlens((torch.arange(T) < VALID).long().expand(B, T), n, "cpu")
        sp = U.UlyssesCarvedAttention(attn_fn=_oracle_attn)
        joint = U.my_parallel_attention(sp, ql, kl, vl, n, n, cu, cu, top_k=TOP_K, text_amp=0.3,
                                        block_neighbor_list=nbr, p_remain_rates=0.3)
        img = sp(None, q[:, sl], k[:, sl], v[:, sl], top_k=TOP_K, block_neighbor_list=nbr, p_remain_rates=0.3)
        ret[rank] = dict(joint=joint, img=img)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("B", [2, 3])
@pytest.mark.parametrize("H,ragged", [(4, False), (3, True)])
def test_carved_attention_each_sample_equals_it_alone(H, ragged, B):
    mgr = mp.Manager()
    ret = mgr.dict()
    port = 29500 + (os.getpid() + 71 * H + 7 * B) % 2000
    mp.spawn(_worker, args=(P, H, B, ragged, port, ret), nprocs=P, join=True)
    from jenga_b200.ulysses import head_offsets
    q, k, v, nbr = _inputs(H, B)
    cu = torch.tensor([0, N_IMG + VALID, N_IMG + T], dtype=torch.int32)
    off = head_offsets(H, P)
    n = N_IMG // P
    for b in range(B):
        # the single-process operator on sample b alone, over each rank's head group side by side (the
        # CPU oracle's fp32 GEMMs may round a one-head batch differently from a many-head one)
        full, img = [], []
        for p in range(P):
            qs, ks, vs = (x[b:b + 1, :, off[p]:off[p + 1]] for x in (q, k, v))
            full.append(_oracle_attn(qs, ks, vs, top_k=TOP_K, cu_seqlens_q=cu, cu_seqlens_kv=cu, text_amp=0.3,
                                     block_neighbor_list=nbr, p_remain_rates=0.3, text_blocks=T // 128,
                                     shape_xfuse=True))
            img.append(_oracle_attn(qs[:, :N_IMG], ks[:, :N_IMG], vs[:, :N_IMG], top_k=TOP_K,
                                    block_neighbor_list=nbr, p_remain_rates=0.3, text_blocks=0, shape_xfuse=True))
        full = torch.cat(full, dim=2).flatten(2)
        img = torch.cat(img, dim=2)
        for r in range(P):
            got = ret[r]
            assert got["joint"].shape == (B, n + T, H * 128)
            assert got["img"].shape == (B, n, H, 128)
            assert torch.equal(got["joint"][b, :n], full[0, r * n:(r + 1) * n]), (b, r)
            assert torch.equal(got["joint"][b, n:], full[0, N_IMG:]), (b, r)
            assert torch.equal(got["img"][b], img[0, r * n:(r + 1) * n]), (b, r)
