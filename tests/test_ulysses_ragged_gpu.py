"""The ragged Ulysses head split on the fused exchange, emulated on one GPU.

The ranks are emulated as tests/test_ulysses_emulated_gpu.py does: every rank's buffers on one device in
the middle of GUARD canary rows, UlyssesFusedAttention unmodified, one Python thread per rank with host
barriers.  Degrees that do not divide the head count, with ulysses.RAGGED_HEADS on:
(H, P) in {(12, 5), (12, 7), (12, 8), (24, 5), (24, 7), (40, 3), (40, 6), (40, 7)}, over every head
sub-group count G <= 3 that divides the slot count ceil(H/P).

* Inbound exchange: every jenga_ulysses_scatter_ragged call writes exactly its region of every rank's
  [3, N+T, slots, D] buffer (slot s of rank p = global head off[p] + s, the slots past a short group
  untouched), with and without text rows, whole and ragged row counts.  With P | H it writes the same
  bytes as jenga_ulysses_scatter.
* The production class through my_parallel_attention: HunyuanVideo with text rows (whole and, at even
  P, rows straddling blocks) and HunyuanVideo-I2V with 400 text tokens; every rank's rows equal the
  single-GPU operator bit for bit, on two consecutive calls (both result buffers), guards intact.
* The Wan self-attention section (tests/test_wan_sp_gpu.py), with seq_len pad rows where P does not divide L: the carved call, the
  dense-class call, and one JENGA_QK_INT8 point.
* Real model forwards: parallelize_wan on the patched 12-head Wan model at P = 5 and 8, and the sharded
  HunyuanVideo-I2V forward at 24 heads, P = 5 (tests/test_wan_sp_forward_gpu.py,
  tests/test_i2v_sp_forward_gpu.py, on emulated ranks).
* With three GPUs or more, a real NCCL run at P = 3 with 12 and with 14 heads (skipped otherwise).
"""
import ctypes as C
import os
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
import test_ulysses_emulated_gpu as UE  # noqa: E402
from test_ulysses_emulated_gpu import (BLOCK, CANARY, D, P_REMAIN, TOP_K, VARIANTS, _FakeGroup, _guarded,  # noqa: E402
                                       _guards_intact, _Handle, _mid, _run_ranks, _same)

DEV = torch.device("cuda", 0)
HP = [(12, 5), (12, 7), (12, 8), (24, 5), (24, 7), (40, 3), (40, 6), (40, 7)]


def _slots(H, P):
    return -(-H // P)


HPG = [(H, P, G) for H, P in HP for G in (1, 2, 3) if _slots(H, P) % G == 0]


@pytest.fixture
def ragged_on(monkeypatch):
    from jenga_b200 import ulysses
    monkeypatch.setattr(ulysses, "RAGGED_HEADS", True)
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    monkeypatch.setattr(ulysses.dist, "get_world_size", lambda g=None: g.size)


def _offsets(H, P):
    from jenga_b200.ulysses import head_offsets
    return head_offsets(H, P)


class RaggedWorld:
    """P ranks' buffers as UlyssesFusedAttention allocates them under the ragged split: qkv[p]
    [3, N+T, slots, D] and n_out result buffers out[b][p] [n_loc+T, H, D], each between canary guards."""

    def __init__(self, P, n, H, T=0, dtype=torch.bfloat16, n_out=2, off=None):
        self.P, self.n, self.H, self.T, self.N = P, n, H, T, P * n
        self.off = off or _offsets(H, P)
        self.slots = max(self.off[p + 1] - self.off[p] for p in range(P))
        self.qkv_rows, self.out_rows = 3 * (self.N + T), n + T
        self.qkv_full, self.qkv = [], []
        for _ in range(P):
            full, mid = _guarded(self.qkv_rows, (self.slots, D), dtype)
            self.qkv_full.append(full)
            self.qkv.append(mid.view(3, self.N + T, self.slots, D))
        self.out_full, self.out = [], []
        for _ in range(n_out):
            fs = [_guarded(self.out_rows, (H, D), dtype) for _ in range(P)]
            self.out_full.append([f for f, _ in fs])
            self.out.append([m for _, m in fs])
        self.p_qkv = (C.c_uint64 * P)(*[t.data_ptr() for t in self.qkv])
        self.p_out = [(C.c_uint64 * P)(*[o.data_ptr() for o in outs]) for outs in self.out]

    def fused(self, bar, r, G=None, variant="hyvideo", group=None):
        from jenga_b200.ulysses import UlyssesFusedAttention
        world = self

        class EmulatedFused(UlyssesFusedAttention):
            def _buffers(self, N, T, h, D_, n_loc, H_, dtype, dev):
                assert (N, T, h, n_loc, H_) == (world.N, world.T, world.slots, world.n, world.H)
                hd = _Handle(bar)
                return world.qkv[r], hd, world.p_qkv, [(world.out[b][r], hd, world.p_out[b]) for b in range(2)]

        return EmulatedFused(group=group or _FakeGroup(self.P, r), variant=variant, groups=G)

    def guards_intact(self):
        return (all(_guards_intact(f, self.qkv_rows) for f in self.qkv_full) and
                all(_guards_intact(f, self.out_rows) for b in self.out_full for f in b))


def _inputs(n_img, T, H, seed=4100):
    import bench
    S = n_img + T
    q = bench.synth_tokens(S, H, DEV, seed).bfloat16()
    k = bench.synth_tokens(S, H, DEV, seed + 1).bfloat16()
    g = torch.Generator(device=DEV).manual_seed(seed + 2)
    v = torch.randn(1, S, H, D, generator=g, device=DEV).bfloat16()
    return q, k, v


def _scatter_args(xs, js, P, r, n, T, H, peers):
    from jenga_b200 import _lib
    xs = [t[0] for t in xs]
    a = _lib.JengaUlyssesScatterArgs()
    a.x = (C.c_void_p * 3)(*[t.data_ptr() for t in xs])
    a.x_stride_s = xs[0].stride(0)
    if T:
        js = [t[0] for t in js]
        a.joint = (C.c_void_p * 3)(*[t.data_ptr() for t in js])
        a.joint_stride_s = js[0].stride(0)
    a.world, a.rank, a.heads, a.head_dim, a.n_loc, a.n_text = P, r, H, D, n, T
    a.peer_qkv_host = C.addressof(peers)
    return a


def _scatter(ragged, xs, js, P, r, n, T, H, peers, off, head_begin, head_count):
    from jenga_b200._lib import check, lib
    from jenga_b200.attention import _stream_ptr
    a = _scatter_args(xs, js, P, r, n, T, H, peers)
    a.head_begin, a.head_count = head_begin, head_count
    if ragged:
        c_off = (C.c_int32 * (P + 1))(*off)
        check(lib.jenga_ulysses_scatter_ragged(C.byref(a), c_off, _stream_ptr(DEV)), "ulysses_scatter_ragged")
    else:
        check(lib.jenga_ulysses_scatter(C.byref(a), _stream_ptr(DEV)), "ulysses_scatter")


# ------------------------------------------------------------------------------------------------
# (a) inbound exchange
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["whole", "ragged"])
@pytest.mark.parametrize("T", [0, 400])
@pytest.mark.parametrize("H,P,G", HPG)
def test_scatter_ragged_writes_exactly_its_region(H, P, G, T, kind):
    n = 256 if kind == "whole" else 200
    N = P * n
    q, k, v = _inputs(N, T, H)
    src = torch.stack([q[0], k[0], v[0]])                                  # [3, N+T, H, D]
    world = RaggedWorld(P, n, H, T, n_out=0)
    off, slots = world.off, world.slots
    hg = slots // G
    expect = [f.clone() for f in world.qkv_full]
    for r in range(P):
        loc = [torch.cat([x[:, r * n:(r + 1) * n], x[:, N:]], dim=1) for x in (q, k, v)]
        for g in range(G):
            _scatter(True, [t[:, :n] for t in loc], [t[:, n:] for t in loc], P, r, n, T, H, world.p_qkv, off,
                     g * hg, hg)
            torch.cuda.synchronize()
            for p in range(P):
                s0, s1 = g * hg, min((g + 1) * hg, off[p + 1] - off[p])
                if s0 >= s1:
                    continue
                e = _mid(expect[p], world.qkv_rows).view(3, N + T, slots, D)
                e[:, r * n:(r + 1) * n, s0:s1] = src[:, r * n:(r + 1) * n, off[p] + s0:off[p] + s1]
                if p == r and T:
                    e[:, N:, s0:s1] = src[:, N:, off[r] + s0:off[r] + s1]
            for p in range(P):
                assert _same(world.qkv_full[p], expect[p]), (r, g, p)
    for p in range(P):
        hp = off[p + 1] - off[p]
        assert _guards_intact(world.qkv_full[p], world.qkv_rows)
        assert _same(world.qkv[p][:, :, :hp], src[:, :, off[p]:off[p + 1]]), p
        assert bool((world.qkv[p][:, :, hp:].view(torch.int16) == CANARY).all()), p


@pytest.mark.parametrize("H,P,G", [(24, 4, 1), (24, 4, 2), (40, 8, 1), (12, 3, 2), (24, 1, 3)])
def test_divisible_split_writes_the_bytes_of_the_plain_exchange(H, P, G):
    n, T = 200, 400
    N = P * n
    q, k, v = _inputs(N, T, H, seed=4300)
    off = tuple(r * H // P for r in range(P + 1))
    worlds = [RaggedWorld(P, n, H, T, n_out=0, off=off) for _ in range(2)]
    hg = H // P // G
    for ragged, world in zip((False, True), worlds):
        for r in range(P):
            loc = [torch.cat([x[:, r * n:(r + 1) * n], x[:, N:]], dim=1) for x in (q, k, v)]
            for g in range(G):
                _scatter(ragged, [t[:, :n] for t in loc], [t[:, n:] for t in loc], P, r, n, T, H, world.p_qkv, off,
                         g * hg, hg)
    torch.cuda.synchronize()
    for p in range(P):
        assert _same(worlds[0].qkv_full[p], worlds[1].qkv_full[p]), p
        assert _same(worlds[1].qkv[p], torch.stack([q[0], k[0], v[0]])[:, :, off[p]:off[p + 1]]), p


# ------------------------------------------------------------------------------------------------
# (b) the production class, HunyuanVideo and HunyuanVideo-I2V
# ------------------------------------------------------------------------------------------------
def _single(variant, q, k, v, T, valid, amp, nbr):
    from jenga_b200.attention import block_sparse_attention_variant
    N = q.shape[1] - T
    cu = UE._cu(N, T, valid)
    return block_sparse_attention_variant(variant, q, k, v, TOP_K, cu_seqlens_q=cu, cu_seqlens_kv=cu,
                                          text_blocks=(T + BLOCK - 1) // BLOCK, text_amp=amp,
                                          block_neighbor_list=nbr, p_remain_rates=P_REMAIN, shape_xfuse=True)


PROD = [(H, P, G, name, kind) for H, P, G in HPG for name, kind in (("hy_amp", "whole"), ("i2v", "whole"))] + \
       [(H, P, G, "hy_amp", "ragged") for H, P, G in HPG if P % 2 == 0]


@pytest.mark.parametrize("H,P,G,name,kind", PROD)
def test_production_class_equals_single_gpu(ragged_on, H, P, G, name, kind):
    from jenga_b200 import ulysses
    variant, T, valid, amp = VARIANTS[name]
    n_img = 256 * P if kind == "whole" else 9 * BLOCK
    n, N = n_img // P, n_img
    assert n * P == N and (kind == "whole") == (n % BLOCK == 0)
    nbr = synth.band_neighbours(n_img // BLOCK)
    sets = [_inputs(n_img, T, H, seed) for seed in (4100, 4200)]
    refs = [_single(variant, *x, T, valid, amp, nbr) for x in sets]
    cu = torch.tensor([0, n + valid, n + T], dtype=torch.int32, device=DEV)
    kw = dict(top_k=TOP_K, text_amp=amp, block_neighbor_list=nbr, p_remain_rates=P_REMAIN)
    world = RaggedWorld(P, n, H, T)
    got = [dict() for _ in range(P)]

    def rank(r, bar):
        sp = world.fused(bar, r, G, variant)
        for i, s in enumerate(sets):
            ql, kl, vl = (torch.cat([x[:, r * n:(r + 1) * n], x[:, N:]], dim=1) for x in s)
            got[r][i] = ulysses.my_parallel_attention(sp, ql, kl, vl, n, n, cu, cu, **kw)
            torch.cuda.synchronize()

    _run_ranks(P, rank)
    for r in range(P):
        for i in range(len(sets)):
            assert _same(got[r][i].view(n + T, H, D), UE._relaid(refs[i], r, n, T)), (r, i)
    assert world.guards_intact()


# ------------------------------------------------------------------------------------------------
# (c) the Wan self-attention section: seq_len pad rows, the dense class, JENGA_QK_INT8
# ------------------------------------------------------------------------------------------------
class _WanWorld(RaggedWorld):
    """tests/test_wan_sp_gpu.py's _World interface over the ragged buffers"""

    def __init__(self, P, n, H):
        super().__init__(P, n, H)

    def fused(self, bar, P, r, G):
        return RaggedWorld.fused(self, bar, r, G, "wan")


@pytest.fixture
def wan_ragged(ragged_on, monkeypatch):
    import test_wan_sp_gpu as WS
    monkeypatch.setattr(WS, "_World", _WanWorld)
    return WS


@pytest.mark.parametrize("H,P,G", HPG)
def test_wan_section_equals_single_gpu(wan_ragged, H, P, G):
    WS = wan_ragged
    c = WS._section_case(H, WS.GRIDS["ragged"])
    for drop in (WS.CARVED, WS.DENSE):
        single, bits = WS._single(H, c, drop)
        got, per_rank, n = WS._sharded(H, P, G, c, drop)
        WS._check(H, P, c, drop, got, per_rank, n, single, bits)


def test_wan_section_qk_int8(wan_ragged, monkeypatch):
    from jenga_b200 import attention as A
    monkeypatch.setattr(A, "QK_INT8", True)
    WS = wan_ragged
    H, P = 12, 8
    c = WS._section_case(H, WS.GRIDS["ragged"], seed=5400)
    for drop in (WS.CARVED, WS.DENSE):
        single, bits = WS._single(H, c, drop)
        got, per_rank, n = WS._sharded(H, P, None, c, drop)
        WS._check(H, P, c, drop, got, per_rank, n, single, bits)


# ------------------------------------------------------------------------------------------------
# (d) real model forwards on emulated ranks
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def wan_module():
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    ours = R.load_blocks(product=True)[1]
    assert ours.WanSelfAttention.forward.__jenga_b200__
    yield ours
    from jenga_b200 import blocks
    blocks.remove_gather_hook()


@pytest.mark.parametrize("P", [5, 8])
def test_wan_forward_12_heads_matches_single_gpu(wan_module, ragged_on, monkeypatch, P):
    """parallelize_wan on the patched 12-head Wan model (2,2,2,2,1,1,1,1 heads at P = 8): the steps of
    tests/test_wan_sp_forward_gpu.py, a dense warm-up, carved, TeaCache-skipped and turbo-swap steps"""
    import test_wan_sp_forward_gpu as WF
    from jenga_b200 import blocks
    assert WF.HEADS == 12
    monkeypatch.setattr(WF, "_World", _WanWorld)
    ref, model = WF._single_gpu(wan_module)
    before = dict(blocks.STATS)
    got = WF._emulated(P, monkeypatch, model)
    assert blocks.STATS["wan_self_sp"] == before["wan_self_sp"] + 6 * P
    assert blocks.STATS["wan_self_dense_sp"] == before["wan_self_dense_sp"] + 2 * P
    assert blocks.STATS["fallback"] == before["fallback"]
    for i, (name, *_rest) in enumerate(WF._steps()):
        for r in range(P):
            assert torch.equal(got[r][i], got[0][i]), (r, name)
        rows = WF._rows(ref[i])
        WF._compare(rows, WF._rows(got[0][i]), torch.ones(rows.shape[1], dtype=torch.bool, device="cuda"),
                    f"sharded Wan forward, 12 heads, P={P}, {name}")


@pytest.fixture(scope="module")
def i2v_module():
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    from i2v_ref import load_i2v_blocks
    ours = load_i2v_blocks(product=True)
    assert ours.MMDoubleStreamBlock.forward.__jenga_b200__
    yield ours
    from jenga_b200 import blocks
    blocks.remove_gather_hook()


def test_i2v_forward_24_heads_at_5_ranks_matches_single_gpu(i2v_module, ragged_on, monkeypatch):
    import test_i2v_sp_forward_gpu as IF
    from jenga_b200 import blocks
    P = 5
    monkeypatch.setattr(IF, "GRID", (8, 16, 20))                   # L = 2560, 512 image rows per rank
    assert IF.H == 24

    def world(P_, n, T, dtype, n_out=2):
        return RaggedWorld(P_, n, IF.H, T, dtype, n_out)

    def emulated_fused(w, bar):
        def make(group, variant):
            return w.fused(bar, group.rank, None, variant, group=group)
        return make

    monkeypatch.setattr(IF, "World", world)
    monkeypatch.setattr(IF, "_emulated_fused", emulated_fused)
    ref, single_model = IF._single_gpu(i2v_module)
    before = dict(blocks.STATS)
    got = IF._emulated(i2v_module, P, monkeypatch, single_model)
    assert blocks.STATS["i2v_double_sp"] == before["i2v_double_sp"] + P
    assert blocks.STATS["i2v_single_sp"] == before["i2v_single_sp"] + P
    assert blocks.STATS["fallback"] == before["fallback"]
    L = 8 * 16 * 20
    every_row = torch.ones(L, dtype=torch.bool, device="cuda")
    for step, what in enumerate(("computed step", "skipped step")):
        for r in range(P):
            assert torch.equal(got[r][step], got[0][step]), (r, what)
        IF._compare(IF._rows(ref[step]), IF._rows(got[0][step]), every_row,
                    f"sharded I2V forward, 24 heads, P={P}, {what}")


# ------------------------------------------------------------------------------------------------
# (e) three GPUs: the real exchange over NCCL and NVLink peer memory
# ------------------------------------------------------------------------------------------------
def _nccl_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        import bench
        from jenga_b200 import ulysses
        from jenga_b200.hyi2v_sp import default_attention
        ulysses.RAGGED_HEADS = True
        variant, T, valid, amp = VARIANTS["hy_amp"]
        dev = torch.device("cuda", rank)
        n_img = 256 * world
        n = n_img // world
        nbr = synth.band_neighbours(n_img // BLOCK)
        res = {}
        for H in (12, 14):                       # 4 heads each, then 5, 5, 4 at P = 3
            q, k = (bench.synth_tokens(n_img + T, H, dev, s).bfloat16() for s in (4100, 4101))
            v = torch.randn(1, n_img + T, H, D, generator=torch.Generator(device=dev).manual_seed(4102),
                            device=dev).bfloat16()
            from jenga_b200.attention import block_sparse_attention_variant
            cu = torch.tensor([0, n_img + valid, n_img + T], dtype=torch.int32, device=dev)
            ref = block_sparse_attention_variant(variant, q, k, v, TOP_K, cu_seqlens_q=cu, cu_seqlens_kv=cu,
                                                 text_blocks=T // BLOCK, text_amp=amp, block_neighbor_list=nbr,
                                                 p_remain_rates=P_REMAIN, shape_xfuse=True)
            sp = default_attention(None, variant)
            cu_l = torch.tensor([0, n + valid, n + T], dtype=torch.int32, device=dev)
            ql, kl, vl = (torch.cat([x[:, rank * n:(rank + 1) * n], x[:, n_img:]], dim=1) for x in (q, k, v))
            out = ulysses.my_parallel_attention(sp, ql, kl, vl, n, n, cu_l, cu_l, top_k=TOP_K, text_amp=amp,
                                                block_neighbor_list=nbr, p_remain_rates=P_REMAIN)
            torch.cuda.synchronize()
            res[H] = (type(sp).__name__, _same(out.view(n + T, H, D), UE._relaid(ref, rank, n, T)))
        ret[rank] = res
    finally:
        dist.destroy_process_group()


def test_three_gpus_real_exchange_equals_single_gpu():
    if torch.cuda.device_count() < 3:
        pytest.skip("needs three GPUs")
    import torch.multiprocessing as mp
    P = 3
    ret = mp.Manager().dict()
    mp.spawn(_nccl_worker, args=(P, 29500 + os.getpid() % 2000, ret), nprocs=P, join=True)
    for r in range(P):
        for H, (kind, same) in ret[r].items():
            assert same, (r, H, kind)
