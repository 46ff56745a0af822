"""Several samples per call on the fused Ulysses exchange, emulated on one GPU.

The emulation of tests/test_ulysses_emulated_gpu.py (every rank's buffers on one device, their addresses in
the peer arrays, one Python thread per rank), with the batched buffers: qkv [3, B, N+T, slots, D] and result
buffers [B, n_loc+T, H, D], each between canary guard rows.

* Inbound: jenga_ulysses_scatter_batched writes exactly its region at B = 2 and 3, at every world size,
  head sub-group count, text length and slice kind, and under the ragged split (H = 24 at P = 5 and 7).
  At B = 1 it writes the bytes of jenga_ulysses_scatter / _ragged.
* Outbound: the peer-store epilogue stores exactly each owner's [B, n_loc+T, H, D] slab, through the plain,
  scheduled, INT8 Q.K^T and FP8 P.V launches; every sample is bit-identical to the single-GPU operator on
  that sample alone.
* UlyssesFusedAttention, unmodified, through my_parallel_attention: each sample of a B = 2 call equals its
  B = 1 call bit for bit (A, B, A: the double buffer holds); B = 1 and B = 2 calls interleave on separate
  buffers; the INT8 / FP8 switches at B = 2 equal their B = 1 results.  HY-720p at P = 8, B = 2.
* Blocks at B = 2 against each sample alone (the drop-in tolerance: cuBLAS may pick another GEMM algorithm
  for more rows): the unmodified HunyuanVideo double and single blocks under an emulated
  hybrid_seq_parallel_attn, and parallelize_i2v's sharded forward on a computed and a skipped step.
* Two GPUs (skipped on a one-GPU box): the real exchange at B = 2 equals the emulated run.
"""
import copy
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE / "golden"))
import synth  # noqa: E402
from test_ulysses_emulated_gpu import (BLOCK, D, DEV, GUARD, H, P_REMAIN, TOP_K, VARIANTS, WORLD_G, World,  # noqa: E402
                                       _FakeGroup, _Handle, _cu, _guarded, _guards_intact, _inputs, _n_img, _relaid,
                                       _run_ranks, _same, _single)

B_CASES = (2, 3)


def _offsets(H_, P):
    from jenga_b200.ulysses import head_offsets
    return head_offsets(H_, P)


class BatchWorld:
    """P emulated ranks' batched buffers: qkv[p] [3, B, N+T, slots, D] and n_out result buffers out[i][p]
    [B, n_loc+T, H, D], each in the middle of a canary-filled allocation"""

    def __init__(self, P, n, T, B, dtype=torch.bfloat16, n_out=1, heads=H, off=None):
        self.P, self.n, self.T, self.B, self.H, self.N = P, n, T, B, heads, P * n
        self.off = off or _offsets(heads, P)
        self.slots = max(self.off[p + 1] - self.off[p] for p in range(P))
        self.qkv_rows, self.out_rows = 3 * B * (self.N + T), B * (n + T)
        self.qkv_full, self.qkv = [], []
        for _ in range(P):
            full, mid = _guarded(self.qkv_rows, (self.slots, D), dtype)
            self.qkv_full.append(full)
            self.qkv.append(mid.view(3, B, self.N + T, self.slots, D))
        self.out_full, self.out = [], []
        for _ in range(n_out):
            fs = [_guarded(self.out_rows, (heads, D), dtype) for _ in range(P)]
            self.out_full.append([f for f, _ in fs])
            self.out.append([m.view(B, n + T, heads, D) for _, m in fs])
        self.p_qkv = (C.c_uint64 * P)(*[t.data_ptr() for t in self.qkv])
        self.p_out = [(C.c_uint64 * P)(*[o.data_ptr() for o in outs]) for outs in self.out]

    def guards_intact(self):
        return (all(_guards_intact(f, self.qkv_rows) for f in self.qkv_full) and
                all(_guards_intact(f, self.out_rows) for outs in self.out_full for f in outs))


def _batch_inputs(n_img, T, B, dtype=torch.bfloat16, seed=4100):
    """B samples [B, n_img+T, H, D], sample b from seed + 100 b (sample 0 is _inputs(seed))"""
    sets = [_inputs(n_img, T, dtype, seed + 100 * b) for b in range(B)]
    return [torch.cat([s[w] for s in sets]) for w in range(3)]


def _local(x, r, n, N):
    return torch.cat([x[:, r * n:(r + 1) * n], x[:, N:]], dim=1)


def _scatter_batched(xs, js, P, r, n, T, peers, head_begin, head_count, off=None, heads=H):
    """jenga_ulysses_scatter_batched as UlyssesFusedAttention calls it; xs / js: [B, n, H, D] / [B, T, H, D]"""
    from jenga_b200 import _lib
    from jenga_b200._lib import check, lib
    from jenga_b200.attention import _stream_ptr
    a = _lib.JengaUlyssesScatterBatchArgs()
    a.batch, a.x_stride_b = xs[0].shape[0], xs[0].stride(0)
    a.base.x = (C.c_void_p * 3)(*[t.data_ptr() for t in xs])
    a.base.x_stride_s = xs[0].stride(1)
    if T:
        a.base.joint = (C.c_void_p * 3)(*[t.data_ptr() for t in js])
        a.base.joint_stride_s, a.joint_stride_b = js[0].stride(1), js[0].stride(0)
    a.base.world, a.base.rank, a.base.heads, a.base.head_dim, a.base.n_loc, a.base.n_text = P, r, heads, D, n, T
    a.base.peer_qkv_host = C.addressof(peers)
    a.base.head_begin, a.base.head_count = head_begin, head_count
    c_off = None if off is None else (C.c_int32 * (P + 1))(*off)
    check(lib.jenga_ulysses_scatter_batched(C.byref(a), c_off, _stream_ptr(DEV)), "ulysses_scatter_batched")


# ------------------------------------------------------------------------------------------------
# (a) inbound exchange
# ------------------------------------------------------------------------------------------------
def _scatter_case(P, G, T, kind, B, heads=H, ragged=False):
    off = _offsets(heads, P)
    n_img = _n_img(P, kind)
    n, N = n_img // P, n_img
    world = BatchWorld(P, n, T, B, heads=heads, off=off)
    slots = world.slots
    g = torch.Generator(device=DEV).manual_seed(P * 100 + T + B)
    src = torch.randn(3, B, N + T, heads, D, generator=g, device=DEV).bfloat16()
    calls = [(0, 0)] if G == 0 else [(i * (slots // G), slots // G) for i in range(G)]
    expect = [f.clone() for f in world.qkv_full]
    for r in range(P):
        loc = [_local(src[w], r, n, N) for w in range(3)]              # [B, n+T, H, D] each
        for hb, hc in calls:
            _scatter_batched([t[:, :n] for t in loc], [t[:, n:] for t in loc], P, r, n, T, world.p_qkv, hb, hc,
                             off if ragged else None, heads)
            for p in range(P):
                e = expect[p][GUARD:GUARD + world.qkv_rows].view(3, B, N + T, slots, D)
                hi = min(hb + (hc or slots), off[p + 1] - off[p])
                for s in range(hb, hi):
                    e[:, :, r * n:(r + 1) * n, s] = src[:, :, r * n:(r + 1) * n, off[p] + s]
                    if p == r and T:
                        e[:, :, N:, s] = src[:, :, N:, off[r] + s]
        torch.cuda.synchronize()
        for p in range(P):
            assert _same(world.qkv_full[p], expect[p]), (r, p)
    assert world.guards_intact()


@pytest.mark.parametrize("B", B_CASES)
@pytest.mark.parametrize("kind", ["whole", "ragged"])
@pytest.mark.parametrize("T", [0, 256])
@pytest.mark.parametrize("P,G", WORLD_G)
def test_batched_scatter_writes_exactly_its_region(P, G, T, kind, B):
    _scatter_case(P, G, T, kind, B)


@pytest.mark.parametrize("B", B_CASES)
@pytest.mark.parametrize("T", [0, 256])
@pytest.mark.parametrize("P,G", [(5, 0), (5, 1), (5, 5), (7, 0), (7, 1), (7, 4)])
def test_batched_ragged_scatter_writes_exactly_its_region(P, G, T, B):
    """H = 24 over 5 (5, 5, 5, 5, 4 heads) and 7 (4, 4, 4, 3, 3, 3, 3) ranks; G counts slot groups"""
    _scatter_case(P, G, T, "whole", B, ragged=True)


@pytest.mark.parametrize("T", [0, 400])
@pytest.mark.parametrize("P,G,ragged", [(1, 1, False), (3, 2, False), (8, 3, False), (1, 1, True), (8, 3, True),
                                        (5, 1, True), (7, 4, True)])
def test_batched_scatter_at_batch_1_writes_the_unbatched_bytes(P, G, T, ragged):
    from jenga_b200._lib import check, lib
    from jenga_b200.attention import _stream_ptr
    from test_ulysses_ragged_gpu import _scatter_args
    off = _offsets(H, P)
    n_img = _n_img(P, "ragged")
    n, N = n_img // P, n_img
    q, k, v = _inputs(n_img, T, torch.bfloat16)
    worlds = [BatchWorld(P, n, T, 1), BatchWorld(P, n, T, 1)]
    slots = worlds[0].slots
    for r in range(P):
        loc = [_local(x, r, n, N) for x in (q, k, v)]
        xs, js = [t[:, :n] for t in loc], [t[:, n:] for t in loc]
        for i in range(G):
            hb, hc = i * (slots // G), slots // G
            _scatter_batched(xs, js, P, r, n, T, worlds[0].p_qkv, hb, hc, off if ragged else None)
            a = _scatter_args(xs, js, P, r, n, T, H, worlds[1].p_qkv)
            a.head_begin, a.head_count = hb, hc
            if ragged:
                check(lib.jenga_ulysses_scatter_ragged(C.byref(a), (C.c_int32 * (P + 1))(*off), _stream_ptr(DEV)), "r")
            else:
                check(lib.jenga_ulysses_scatter(C.byref(a), _stream_ptr(DEV)), "d")
    torch.cuda.synchronize()
    for p in range(P):
        assert _same(worlds[0].qkv_full[p], worlds[1].qkv_full[p]), p


# ------------------------------------------------------------------------------------------------
# (b) outbound exchange: the peer-store epilogue at B > 1
# ------------------------------------------------------------------------------------------------
def _restate(world, xs):
    """every rank's qkv as the inbound exchange leaves it, from the global [B, N+T, H, D] q, k, v"""
    for p in range(world.P):
        for w, x in enumerate(xs):
            world.qkv[p][w].copy_(x[:, :, world.off[p]:world.off[p] + world.slots])


def _epilogue_batch_case(P, G, name, B, dtype, launch):
    """launch: 'sched' (the operator's entry point), 'plain' (jenga_carved_attn_fwd), 'int8', 'fp8'"""
    from jenga_b200.attention import block_sparse_attention_variant
    variant, T, valid, amp = VARIANTS[name]
    n_img = _n_img(P, "ragged")
    n, N, h = n_img // P, n_img, H // P
    hg = h // G
    xs = _batch_inputs(n_img, T, B, dtype)
    nbr = synth.band_neighbours(n_img // BLOCK)
    sw = dict(qk_int8=launch == "int8", pv_fp8=launch == "fp8")
    cu = _cu(N, T, valid)
    kw = dict(cu_seqlens_q=cu, cu_seqlens_kv=cu, text_blocks=(T + BLOCK - 1) // BLOCK, text_amp=amp,
              block_neighbor_list=nbr, p_remain_rates=P_REMAIN)
    alone = [block_sparse_attention_variant(variant, *(x[b:b + 1] for x in xs), TOP_K, shape_xfuse=True, **kw, **sw)
             for b in range(B)]
    world = BatchWorld(P, n, T, B, dtype)
    _restate(world, xs)
    for r in range(P):
        for g in range(G):
            sl = slice(g * hg, (g + 1) * hg)
            sp = dict(world=P, rank=r, heads_total=H, rows=n, peers=world.p_out[0], head_base=r * h + g * hg)
            q, k, v = (world.qkv[r][w][:, :, sl] for w in range(3))
            block_sparse_attention_variant(variant, q, k, v, TOP_K, sp_out=sp, **kw, **sw)
    torch.cuda.synchronize()
    assert world.guards_intact()
    for p in range(P):
        for b in range(B):
            assert _same(world.out[0][p][b], _relaid(alone[b], p, n, T)), (p, b)
    if launch in ("int8", "fp8"):
        plain = block_sparse_attention_variant(variant, *(x[:1] for x in xs), TOP_K, shape_xfuse=True, **kw)
        assert not _same(plain, alone[0])                 # the opt-in path really ran


@pytest.mark.parametrize("B", B_CASES)
@pytest.mark.parametrize("launch", ["sched", "plain", "int8", "fp8"])
@pytest.mark.parametrize("P,G", [(1, 1), (2, 3), (8, 3)])
def test_epilogue_stores_each_owners_batch_slab(monkeypatch, P, G, launch, B):
    if launch == "plain":
        from jenga_b200 import attention
        lib = attention.lib
        plain = lib.jenga_carved_attn_fwd
        monkeypatch.setattr(lib, "jenga_carved_attn_fwd_sched", lambda a, qk, sched, stream: plain(a, stream))
    _epilogue_batch_case(P, G, "hy_amp", B, torch.bfloat16, launch)


@pytest.mark.parametrize("launch", ["sched", "plain"])
@pytest.mark.parametrize("name", ["hy_notext", "i2v"])
def test_epilogue_batch_fp16_and_other_text_lengths(monkeypatch, name, launch):
    if launch == "plain":
        from jenga_b200 import attention
        lib = attention.lib
        plain = lib.jenga_carved_attn_fwd
        monkeypatch.setattr(lib, "jenga_carved_attn_fwd_sched", lambda a, qk, sched, stream: plain(a, stream))
    _epilogue_batch_case(4, 2, name, 2, torch.float16 if name == "i2v" else torch.bfloat16, launch)


# ------------------------------------------------------------------------------------------------
# (c) the production class, one Python thread per emulated rank
# ------------------------------------------------------------------------------------------------
def _emulated_batch_fused(w1, wb, bar, r):
    """UlyssesFusedAttention whose symmetric buffers are the emulated ones: w1 (a batch-1 World or
    RaggedWorld) for B = 1 calls, which ask with the eight batch-1 arguments, and wb (a BatchWorld) for
    B > 1 calls"""
    from jenga_b200.ulysses import UlyssesFusedAttention

    class EmulatedFused(UlyssesFusedAttention):
        def _buffers(self, N, T, h, D_, n_loc, H_, dtype, dev, batch=1):
            w = w1 if batch == 1 else wb
            assert (N, T, n_loc) == (w.N, w.T, w.n) and batch == (1 if w is w1 else wb.B)
            hd = _Handle(bar)
            return w.qkv[r], hd, w.p_qkv, [(w.out[i][r], hd, w.p_out[i]) for i in range(2)]

    return EmulatedFused


def _patch_group(monkeypatch):
    from jenga_b200 import ulysses
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    monkeypatch.setattr(ulysses.dist, "get_world_size", lambda g=None: g.size)
    return ulysses


def _w1(P, n, T, heads, ragged):
    if ragged:
        from test_ulysses_ragged_gpu import RaggedWorld
        return RaggedWorld(P, n, heads, T=T)
    return World(P, n, T, torch.bfloat16, n_out=2)


@pytest.mark.parametrize("P,G,ragged", [(1, None, False), (2, 3, False), (4, None, False), (8, 3, False),
                                        (5, None, True)])
def test_production_class_batch_of_two_equals_its_batch_one_calls(monkeypatch, P, G, ragged):
    """B = 2 calls A, B, A, then B = 1 and B = 2 calls interleaved: every sample equals the single-GPU
    operator on that sample alone (what its batch-1 call returns); each result is intact after the next call;
    B = 1 and B = 2 calls never share a buffer"""
    ulysses = _patch_group(monkeypatch)
    if ragged:
        monkeypatch.setattr(ulysses, "RAGGED_HEADS", True)
    variant, T, valid, amp = VARIANTS["hy_amp"]
    n_img = _n_img(P, "whole")
    n, N = n_img // P, n_img
    nbr = synth.band_neighbours(n_img // BLOCK)
    A = _batch_inputs(n_img, T, 2, seed=4100)
    Bs = _batch_inputs(n_img, T, 2, seed=4300)
    refs = {(s, b): _single(variant, *(x[b:b + 1] for x in xs), T, valid, amp, nbr)[0]
            for s, xs in (("A", A), ("B", Bs)) for b in range(2)}
    calls = [("A", None), ("B", None), ("A", None), ("A", 0), ("B", None), ("A", 1), ("A", None)]
    cu1 = torch.tensor([0, n + valid, n + T], dtype=torch.int32, device=DEV)
    cu2 = torch.tensor([0, n + valid, n + T, 2 * (n + T) - T + valid, 2 * (n + T)], dtype=torch.int32, device=DEV)
    kw = dict(top_k=TOP_K, text_amp=amp, block_neighbor_list=nbr, p_remain_rates=P_REMAIN)
    w1, wb = _w1(P, n, T, H, ragged), BatchWorld(P, n, T, 2, n_out=2, off=_offsets(H, P))
    got = [dict() for _ in range(P)]

    def rank(r, bar):
        sp = _emulated_batch_fused(w1, wb, bar, r)(group=_FakeGroup(P, r), variant=variant, groups=G)
        outs = []
        for i, (s, b) in enumerate(calls):
            xs = A if s == "A" else Bs
            loc = [_local(x if b is None else x[b:b + 1], r, n, N) for x in xs]
            outs.append(ulysses.my_parallel_attention(sp, *loc, n, n, cu1 if b is not None else cu2,
                                                      cu1 if b is not None else cu2, **kw))
            torch.cuda.synchronize()
            got[r][i] = outs[-1].clone()
            if i:
                got[r][f"prev{i}"] = outs[-2].clone()
        got[r]["ptrs"] = [o.data_ptr() for o in outs]

    _run_ranks(P, rank)
    for r in range(P):
        for i, (s, b) in enumerate(calls):
            o = got[r][i].view(-1, n + T, H, D)
            samples = range(2) if b is None else [b]
            assert o.shape[0] == len(samples)
            for j, bb in enumerate(samples):
                assert _same(o[j], _relaid(refs[(s, bb)], r, n, T)), (r, i, bb)
        for i in range(1, len(calls)):
            assert _same(got[r][f"prev{i}"], got[r][i - 1]), (r, i)          # the double buffer
        ptrs = got[r]["ptrs"]
        assert ptrs[0] == ptrs[2] != ptrs[1], r
        assert not {ptrs[i] for i, c in enumerate(calls) if c[1] is None} & {ptrs[3], ptrs[5]}, r
    assert wb.guards_intact()
    if ragged:
        assert w1.guards_intact()
    else:
        assert all(_guards_intact(f, w1.qkv_rows) for f in w1.qkv_full)
        assert all(_guards_intact(f, w1.out_rows) for outs in w1.out_full for f in outs)


@pytest.mark.parametrize("switch", ["QK_INT8", "PV_FP8"])
@pytest.mark.parametrize("P,G,ragged", [(2, 3, False), (5, None, True)])
def test_production_class_switches_at_batch_two_equal_batch_one(monkeypatch, P, G, ragged, switch):
    from jenga_b200 import attention as A_
    ulysses = _patch_group(monkeypatch)
    monkeypatch.setattr(ulysses, "RAGGED_HEADS", ragged)
    monkeypatch.setattr(A_, switch, True)
    variant, T, valid, amp = VARIANTS["hy_amp"]
    n_img = _n_img(P, "whole")
    n, N = n_img // P, n_img
    nbr = synth.band_neighbours(n_img // BLOCK)
    xs = _batch_inputs(n_img, T, 2, seed=4500)
    cu1 = torch.tensor([0, n + valid, n + T], dtype=torch.int32, device=DEV)
    kw = dict(top_k=TOP_K, text_amp=amp, block_neighbor_list=nbr, p_remain_rates=P_REMAIN)
    w1, wb = _w1(P, n, T, H, ragged), BatchWorld(P, n, T, 2, n_out=2, off=_offsets(H, P))
    got = [dict() for _ in range(P)]

    def rank(r, bar):
        sp = _emulated_batch_fused(w1, wb, bar, r)(group=_FakeGroup(P, r), variant=variant, groups=G)
        loc = [_local(x, r, n, N) for x in xs]
        got[r]["B2"] = ulysses.my_parallel_attention(sp, *loc, n, n, cu1, cu1, **kw).clone()
        for b in range(2):
            got[r][b] = ulysses.my_parallel_attention(sp, *(t[b:b + 1] for t in loc), n, n, cu1, cu1, **kw).clone()
        torch.cuda.synchronize()

    _run_ranks(P, rank)
    monkeypatch.setattr(A_, switch, False)
    plain = _single(variant, *(x[:1] for x in xs), T, valid, amp, nbr)[0]
    for r in range(P):
        for b in range(2):
            assert _same(got[r]["B2"][b], got[r][b][0]), (r, b)
        assert not _same(got[r][0].view(n + T, H, D), _relaid(plain, r, n, T)), r   # the switch really ran


# ------------------------------------------------------------------------------------------------
# (d) full size, kernel layer
# ------------------------------------------------------------------------------------------------
def test_full_size_hy720p_batch_two_at_eight_ranks():
    """bench.py's HY-720p workload (n_loc = 14400 at P = 8) with a second sample from another seed, through
    the batched exchange and the head sub-groups UlyssesFusedAttention picks for B = 2"""
    import bench
    from jenga_b200.ulysses import UlyssesFusedAttention
    P, B = 8, 2
    wl = bench.workload("hy720p", 0.7)
    inps = [bench.build_inputs(wl, DEV, seed=1234 + 10 * b) for b in range(B)]
    S, N, T = inps[0]["S"], inps[0]["n_img"], wl["text_tokens"]
    n, h = N // P, H // P
    refs = [bench.run_operator(wl, inp).view(1, S, H, D) for inp in inps]
    assert not _same(refs[0], refs[1])
    xs = [torch.cat([inp[w] for inp in inps]) for w in ("q", "k", "v")]
    del inps[1:]
    G = UlyssesFusedAttention._n_groups(h, None, B * ((S + BLOCK - 1) // BLOCK))
    hg = h // G
    world = BatchWorld(P, n, T, B)
    for r in range(P):
        loc = [x[:, r * n:(r + 1) * n] for x in xs]
        for g in range(G):
            _scatter_batched(loc, [x[:, N:] for x in xs], P, r, n, T, world.p_qkv, g * hg, hg)
    torch.cuda.synchronize()
    for p in range(P):
        for w in range(3):
            assert _same(world.qkv[p][w], xs[w][:, :, p * h:(p + 1) * h]), (p, w)
    del xs
    from jenga_b200.attention import block_sparse_attention_variant
    cu = _cu(N, T, wl["text_valid"])
    for r in range(P):
        for g in range(G):
            sl = slice(g * hg, (g + 1) * hg)
            sp = dict(world=P, rank=r, heads_total=H, rows=n, peers=world.p_out[0], head_base=r * h + g * hg)
            block_sparse_attention_variant(wl["variant"], *(world.qkv[r][w][:, :, sl] for w in range(3)),
                                           inps[0]["top_k"], cu_seqlens_q=cu, cu_seqlens_kv=cu,
                                           text_blocks=(T + BLOCK - 1) // BLOCK, text_amp=wl["text_amp"],
                                           block_neighbor_list=inps[0]["nbr"], p_remain_rates=wl["p_remain"],
                                           sp_out=sp)
    torch.cuda.synchronize()
    assert world.guards_intact()
    for p in range(P):
        for b in range(B):
            assert _same(world.out[0][p][b], _relaid(refs[b], p, n, T)), (p, b)


# ------------------------------------------------------------------------------------------------
# (e) blocks
# ------------------------------------------------------------------------------------------------
from test_dropin_blocks_gpu import _compare, modules  # noqa: E402,F401
from test_hy_batch_gpu import _batch_args, _block  # noqa: E402


def _hy_block_sp(mod, blk, kind, seeds, P, monkeypatch):
    """the unmodified HunyuanVideo block on P emulated ranks under hybrid_seq_parallel_attn =
    UlyssesFusedAttention, as jenga_hyvideo_multigpu.py shards it: each rank's slice of the image rows and
    RoPE rows, the text rows replicated, the local cu_seqlens.  Returns the image rows of all ranks in rank
    order and rank 0's text rows, per output"""
    ulysses = _patch_group(monkeypatch)
    monkeypatch.setattr(mod, "get_sequence_parallel_world_size", lambda: P, raising=False)
    a, L, T = _batch_args(mod, kind, "hy", seeds)
    B, n = len(seeds), L // P
    text_mask = torch.zeros(B, T, dtype=torch.int64, device="cuda")
    text_mask[:, :180] = 1
    heads = blk.heads_num
    w1 = _w1(P, n, T, heads, True)                  # the batch-1 buffers at any head count
    wb = BatchWorld(P, n, T, B, n_out=2, heads=heads) if B > 1 else None
    got = {}
    import inspect
    names = list(inspect.signature(type(blk).forward.__wrapped__).parameters)[1:]

    def rank(r, bar):
        b_ = copy.copy(blk)
        b_.hybrid_seq_parallel_attn = _emulated_batch_fused(w1, wb, bar, r)(group=_FakeGroup(P, r), variant="hyvideo")
        loc = dict(a)
        sl = slice(r * n, (r + 1) * n)
        loc["freqs_cis"] = tuple(f[sl] for f in a["freqs_cis"])
        loc["cu_seqlens_q"] = loc["cu_seqlens_kv"] = mod.get_cu_seqlens(text_mask, n)
        loc["max_seqlen_q"] = loc["max_seqlen_kv"] = n + T
        if kind == "double":
            loc["img"] = a["img"][:, sl].contiguous()
        else:
            loc["x"] = torch.cat([a["x"][:, sl], a["x"][:, L:]], 1)
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            out = type(blk).forward(b_, *(loc[k] for k in names))
        torch.cuda.synchronize()
        got[r] = [o.clone() for o in (out if isinstance(out, tuple) else (out,))]

    _run_ranks(P, rank)
    if kind == "double":
        return torch.cat([got[r][0] for r in range(P)], 1), got[0][1]
    return torch.cat([got[r][0][:, :n] for r in range(P)], 1), got[0][0][:, n:]


@pytest.mark.parametrize("kind", ["double", "single"])
def test_hy_block_under_hybrid_seq_parallel_attn_batch_two(modules, monkeypatch, kind):
    from jenga_b200 import blocks
    mod = modules[2]
    blk = _block(mod, kind)
    P, seeds = 2, [41, 42]
    before = dict(blocks.STATS)
    img, txt = _hy_block_sp(mod, blk, kind, seeds, P, monkeypatch)
    assert blocks.STATS[f"hy_{kind}"] == before[f"hy_{kind}"] + P and blocks.STATS["fallback"] == before["fallback"]
    for b, s in enumerate(seeds):
        img1, txt1 = _hy_block_sp(mod, blk, kind, [s], P, monkeypatch)
        every = torch.ones(img1.shape[1], dtype=torch.bool, device="cuda")
        _compare(img1, img[b:b + 1], every, f"hy {kind} under SP, sample {b} image rows")
        _compare(txt1, txt[b:b + 1], torch.ones(txt1.shape[1], dtype=torch.bool, device="cuda"),
                 f"hy {kind} under SP, sample {b} text rows")


def test_sharded_i2v_forward_batch_two_equals_each_sample_alone(monkeypatch):
    """parallelize_i2v's forward over the patched I2V blocks of test_i2v_sp_forward_gpu.py at P = 2: two
    samples (the second from other latents and text) on a computed and a skipped step, each against its
    batch-1 run"""
    import test_i2v_sp_forward_gpu as F
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    from i2v_ref import load_i2v_blocks
    from jenga_b200 import blocks, hyi2v_sp
    mod = load_i2v_blocks(product=True)
    try:
        ulysses = _patch_group(monkeypatch)
        monkeypatch.setattr(ulysses.dist, "get_rank", lambda g=None: g.rank)
        monkeypatch.setattr(ulysses.dist, "is_initialized", lambda: True)
        monkeypatch.setattr(ulysses.dist, "all_gather", F._emulated_all_gather)
        P, dev = 2, torch.device("cuda", 0)
        L = F.GRID[0] * F.GRID[1] * F.GRID[2]
        base = F._Stack(mod, dev)
        monkeypatch.setattr(F._Stack, "unpatchify", lambda self, x, tt, th, tw: x.transpose(1, 2).reshape(
            x.shape[0], F.C, tt, th, tw))
        x0, t, txt0, mask0, txt20, cos, sin = F._inputs(dev)
        g = torch.Generator(device=dev).manual_seed(8)
        x1 = torch.randn(x0.shape, generator=g, device=dev).bfloat16()
        txt1 = torch.randn(txt0.shape, generator=g, device=dev).bfloat16()
        txt21 = torch.randn(txt20.shape, generator=g, device=dev).bfloat16()
        samples = [(x0, txt0, txt20), (x1, txt1, txt21)]

        def run(xs, txts, txt2s):
            B = xs.shape[0]
            n = L // P
            w1 = World(P, n, F.T, torch.bfloat16, n_out=2)
            wb = BatchWorld(P, n, F.T, B, n_out=2) if B > 1 else None
            models = [copy.deepcopy(base) for _ in range(P)]
            shared, got = {"rows": {}}, {}
            args = (xs, t.expand(B), txts, mask0.expand(B, -1), txt2s, cos, sin)

            def rank(r, bar):
                shared["bar"] = bar
                group = F._Group(P, r, shared)
                sp = _emulated_batch_fused(w1, wb, bar, r)(group=group, variant="hyvideo_i2v")
                hyi2v_sp.parallelize_i2v(models[r], group=group, attention=sp)
                got[r] = [o.clone() for o in F._two_steps(models[r], models[r], args)]

            _run_ranks(P, rank)
            for r in range(P):
                for s in range(2):
                    assert torch.equal(got[r][s], got[0][s]), r
            return got[0]

        before = dict(blocks.STATS)
        both = run(*(torch.cat(z) for z in zip(*samples)))
        assert blocks.STATS["i2v_double_sp"] == before["i2v_double_sp"] + P
        assert blocks.STATS["fallback"] == before["fallback"]
        every = torch.ones(L, dtype=torch.bool, device="cuda")
        for b, smp in enumerate(samples):
            alone = run(*smp)
            for step, what in enumerate(("computed step", "skipped step")):
                _compare(F._rows(alone[step]), F._rows(both[step][b:b + 1]), every,
                         f"sharded I2V forward B=2 sample {b}, {what}")
    finally:
        blocks.remove_gather_hook()


# ------------------------------------------------------------------------------------------------
# (f) two GPUs
# ------------------------------------------------------------------------------------------------
WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["JENGA_ROOT"]); sys.path.insert(0, os.path.join(os.environ["JENGA_ROOT"], "tests", "golden"))
import bench, synth
from jenga_b200.attention import block_sparse_attention_variant
from jenga_b200.ulysses import UlyssesFusedAttention, my_parallel_attention
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank); dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
variant, T, valid, amp, TOP_K, P_REMAIN, H, D = "hyvideo", 256, 180, 0.431, 2, 0.3, 24, 128
n_img = 9 * 128; n = n_img // world; N = n_img; S = N + T
nbr = synth.band_neighbours(n_img // 128)
def sample(seed):
    g = torch.Generator(device=dev).manual_seed(seed + 2)
    return [bench.synth_tokens(S, H, dev, seed).bfloat16(), bench.synth_tokens(S, H, dev, seed + 1).bfloat16(),
            torch.randn(1, S, H, D, generator=g, device=dev).bfloat16()]
sets = [sample(4100 + 100 * b) for b in range(2)]
xs = [torch.cat([s[w] for s in sets]) for w in range(3)]
cuf = torch.tensor([0, N + valid, S], dtype=torch.int32, device=dev)
loc = [torch.cat([x[:, rank * n:(rank + 1) * n], x[:, N:]], 1) for x in xs]
cu = torch.tensor([0, n + valid, n + T, 2 * n + T + valid, 2 * (n + T)], dtype=torch.int32, device=dev)
sp = UlyssesFusedAttention(variant=variant, groups=3)
ok = True
for _ in range(3):
    out = my_parallel_attention(sp, *loc, n, n, cu, cu, top_k=TOP_K, text_amp=amp, block_neighbor_list=nbr,
                                p_remain_rates=P_REMAIN)
    torch.cuda.synchronize()
    for b in range(2):
        ref = block_sparse_attention_variant(variant, *(x[b:b + 1] for x in xs), TOP_K, cu_seqlens_q=cuf,
                                             cu_seqlens_kv=cuf, text_blocks=2, text_amp=amp, block_neighbor_list=nbr,
                                             p_remain_rates=P_REMAIN, shape_xfuse=True)
        want = torch.cat([ref[0, rank * n:(rank + 1) * n], ref[0, N:]]).reshape(n + T, H * D)
        ok = ok and torch.equal(out[b].view(torch.int16), want.view(torch.int16))
t = torch.tensor([1 if ok else 0], device=dev); dist.all_reduce(t, op=dist.ReduceOp.MIN)
if rank == 0: print("BATCH_OK" if t.item() == 1 else "BATCH_MISMATCH")
dist.destroy_process_group()
'''


def test_two_gpus_real_exchange_batch_two(tmp_path):
    """UlyssesFusedAttention over NVLink at B = 2, three calls: every sample equals the single-GPU operator
    on that sample alone, as the emulated runs above do"""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, JENGA_ROOT=str(HERE.parent))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", "2",
                        str(script)], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "BATCH_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
