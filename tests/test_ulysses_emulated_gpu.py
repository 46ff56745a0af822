"""The fused Ulysses exchange at world sizes 1-8, emulated on one GPU.

A peer pointer is only a device address.  With every rank's buffers on one device and their
addresses in the peer arrays, `jenga_ulysses_scatter` (the inbound exchange) and the peer-store
epilogue of the carved-attention kernel (the outbound exchange) do exactly the arithmetic they do
over NVLink.  The exchange is pure data movement and attention is computed per head, so every
emulated result must equal the single-GPU operator bit for bit; the single-GPU operator is itself
checked against fp64 (refutil.fp64_truth) on the query blocks that straddle two owners.

Every emulated buffer sits in the middle of a larger allocation with GUARD rows before and after,
and all of it starts as a 16-bit NaN pattern the kernels never produce.  After each single call the
whole allocation is compared with the expected state, so a store that is missing, lands in the
wrong place, or leaves the buffer is seen.

The emulation serialises the ranks with host barriers, so ordering and races between ranks are out
of its reach; tests/test_ulysses_gpu.py runs the real exchange over NVLink on two GPUs.
"""
import ctypes as C
import functools
import sys
import threading
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE / "golden"))
import refutil  # noqa: E402
import synth  # noqa: E402
from test_attn_gpu import assert_close  # noqa: E402

DEV = torch.device("cuda", 0)
BLOCK, D, H = 128, 128, 24
GUARD = 128                        # rows of canary before and after every buffer
CANARY = 0x7FA5                    # a NaN in both bf16 and fp16
TOP_K, P_REMAIN = 2, 0.3
BARRIER_TIMEOUT_S = 120.0

# (world, head sub-groups G): G divides the H/world heads of a rank
WORLD_G = [(P, G) for P in (1, 2, 3, 4, 8) for G in (1, 2, 3) if (H // P) % G == 0]


def _n_img(P, kind):
    """Image tokens: 'whole' gives n_loc = 256 (two 128-row blocks per rank); 'ragged' gives
    9 blocks in all, so n_loc = 1152 / P (576, 288 and 144 rows straddle owners at P = 2, 4, 8)."""
    return 256 * P if kind == "whole" else 9 * BLOCK


def _bits16(t):
    return t.view(torch.int16)


def _same(a, b):
    return torch.equal(_bits16(a), _bits16(b))


def _guarded(rows, inner, dtype):
    """(allocation, middle): a [rows, *inner] tensor between GUARD canary rows on each side,
    itself canary-filled."""
    full = torch.empty((GUARD + rows + GUARD, *inner), dtype=dtype, device=DEV)
    _bits16(full).fill_(CANARY)
    return full, full[GUARD:GUARD + rows]


def _mid(full, rows):
    return full[GUARD:GUARD + rows]


def _guards_intact(full, rows):
    g = _bits16(full)
    return bool((g[:GUARD] == CANARY).all()) and bool((g[GUARD + rows:] == CANARY).all())


class World:
    """The buffers of P emulated ranks on one device, laid out as UlyssesFusedAttention allocates
    them: qkv[p] [3, N+T, h, D] and n_out result buffers out[b][p] [n_loc+T, H, D], with the peer
    arrays of their addresses."""

    def __init__(self, P, n_loc, T, dtype, n_out=1):
        self.P, self.n, self.T, self.h, self.N = P, n_loc, T, H // P, P * n_loc
        self.qkv_rows, self.out_rows = 3 * (self.N + T), n_loc + T
        self.qkv_full, self.qkv = [], []
        for _ in range(P):
            full, mid = _guarded(self.qkv_rows, (self.h, D), dtype)
            self.qkv_full.append(full)
            self.qkv.append(mid.view(3, self.N + T, self.h, D))
        self.out_full, self.out = [], []
        for _ in range(n_out):
            fs = [_guarded(self.out_rows, (H, D), dtype) for _ in range(P)]
            self.out_full.append([f for f, _ in fs])
            self.out.append([m for _, m in fs])
        self.p_qkv = (C.c_uint64 * P)(*[t.data_ptr() for t in self.qkv])
        self.p_out = [(C.c_uint64 * P)(*[o.data_ptr() for o in outs]) for outs in self.out]

    def restate_qkv(self, q, k, v):
        """Rank p's qkv as the inbound exchange leaves it: all image rows in rank order, then the
        text rows, of its heads [p*h, (p+1)*h)."""
        for p in range(self.P):
            for w, x in enumerate((q, k, v)):
                self.qkv[p][w].copy_(x[0, :, p * self.h:(p + 1) * self.h])


def _relaid(o, p, n, T):
    """Rank p's [n_loc+T, H, D] result: its n_loc image rows and all T text rows of the single-GPU
    output o [1, P*n_loc+T, H, D]."""
    N = o.shape[1] - T
    return torch.cat([o[0, p * n:(p + 1) * n], o[0, N:]], dim=0)


@functools.lru_cache(maxsize=24)
def _inputs(n_img, T, dtype, seed=4100):
    """Model-like q, k (per-block centroids along the token order) and normal v, [1, n_img+T, H, D]."""
    import bench
    S = n_img + T
    q = bench.synth_tokens(S, H, DEV, seed).to(dtype)
    k = bench.synth_tokens(S, H, DEV, seed + 1).to(dtype)
    g = torch.Generator(device=DEV).manual_seed(seed + 2)
    v = torch.randn(1, S, H, D, generator=g, device=DEV).to(dtype)
    return q, k, v


def _cu(N, T, valid):
    return torch.tensor([0, N + valid, N + T], dtype=torch.int32, device=DEV) if T else None


def _single(variant, q, k, v, T, valid, amp, nbr):
    """The single-GPU operator on all H heads: (out [1, S, H, D], mask bits)."""
    from jenga_b200.attention import block_sparse_attention_variant
    N = q.shape[1] - T
    cu = _cu(N, T, valid)
    return block_sparse_attention_variant(variant, q, k, v, TOP_K, cu_seqlens_q=cu, cu_seqlens_kv=cu,
                                          text_blocks=(T + BLOCK - 1) // BLOCK, text_amp=amp,
                                          block_neighbor_list=nbr, p_remain_rates=P_REMAIN, shape_xfuse=True,
                                          return_mask_bits=True)


def _scatter(xs, js, P, r, n, T, peers, head_begin, head_count):
    """jenga_ulysses_scatter with the arguments UlyssesFusedAttention builds; xs / js are the
    [1, n, H, D] / [1, T, H, D] q, k, v views of rank r."""
    from jenga_b200 import _lib
    from jenga_b200._lib import check, lib
    from jenga_b200.attention import _stream_ptr
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
    a.head_begin, a.head_count = head_begin, head_count
    check(lib.jenga_ulysses_scatter(C.byref(a), _stream_ptr(DEV)), "ulysses_scatter")


def _attend(world, r, g, hg, variant, valid, amp, nbr, peers, top_k=TOP_K, p_remain=P_REMAIN):
    """Head sub-group g of rank r through the operator with sp_out, as UlyssesFusedAttention calls it."""
    from jenga_b200.attention import block_sparse_attention_variant
    qkv, sl, T = world.qkv[r], slice(g * hg, (g + 1) * hg), world.T
    cu = _cu(world.N, T, valid)
    sp = dict(world=world.P, rank=r, heads_total=H, rows=world.n, peers=peers, head_base=r * world.h + g * hg)
    block_sparse_attention_variant(variant, qkv[0][None, :, sl], qkv[1][None, :, sl], qkv[2][None, :, sl], top_k,
                                   cu_seqlens_q=cu, cu_seqlens_kv=cu, text_blocks=(T + BLOCK - 1) // BLOCK,
                                   text_amp=amp, block_neighbor_list=nbr, p_remain_rates=p_remain, sp_out=sp)


# ------------------------------------------------------------------------------------------------
# (a) inbound exchange
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["whole", "ragged"])
@pytest.mark.parametrize("T", [0, 256, 400])
@pytest.mark.parametrize("P,G", WORLD_G + [(P, 0) for P in (1, 2, 3, 4, 8)])
def test_scatter_writes_exactly_its_region(P, G, T, kind):
    """G = 0 is one call with head_count = 0 (all of a rank's heads)."""
    n_img = _n_img(P, kind)
    n, N, h = n_img // P, n_img, H // P
    q, k, v = _inputs(n_img, T, torch.bfloat16)
    src = torch.stack([q[0], k[0], v[0]])                               # [3, N+T, H, D]
    world = World(P, n, T, torch.bfloat16)
    expect = [f.clone() for f in world.qkv_full]
    calls = [(0, 0)] if G == 0 else [(g * (h // G), h // G) for g in range(G)]
    for r in range(P):
        # rank r's activations: its image slice and the replicated text rows, [1, n+T, H, D]
        loc = [torch.cat([x[:, r * n:(r + 1) * n], x[:, N:]], dim=1) for x in (q, k, v)]
        for hb, hc in calls:
            _scatter([t[:, :n] for t in loc], [t[:, n:] for t in loc], P, r, n, T, world.p_qkv, hb, hc)
            torch.cuda.synchronize()
            hs = slice(hb, hb + (hc or h))
            for p in range(P):
                e = _mid(expect[p], world.qkv_rows).view(3, N + T, h, D)
                e[:, r * n:(r + 1) * n, hs] = src[:, r * n:(r + 1) * n, p * h + hs.start:p * h + hs.stop]
                if p == r and T:
                    e[:, N:, hs] = src[:, N:, r * h + hs.start:r * h + hs.stop]
            for p in range(P):
                assert _same(world.qkv_full[p], expect[p]), (r, hb, hc, p)
    for p in range(P):
        assert _guards_intact(world.qkv_full[p], world.qkv_rows)
        assert _same(world.qkv[p], src[:, :, p * h:(p + 1) * h]), p


# ------------------------------------------------------------------------------------------------
# (b) outbound exchange: the peer-store epilogue
# ------------------------------------------------------------------------------------------------
VARIANTS = {   # name: (variant, T, valid text tokens, text_amp)
    "hy": ("hyvideo", 256, 180, 0.0),
    "hy_amp": ("hyvideo", 256, 180, 0.431),
    "hy_notext": ("hyvideo", 0, 0, 0.0),
    "i2v": ("hyvideo_i2v", 400, 300, 0.0),
}


def _fp64_blocks(P, n, N, T, nb):
    """Query blocks to check against fp64: those straddling two owners (or the first block of rank 1
    when n_loc is whole), the first text block and the last (ragged for I2V) block."""
    straddle = [r * n // BLOCK for r in range(1, P) if (r * n) % BLOCK]
    qb = [straddle[0], straddle[-1]] if straddle else ([n // BLOCK] if P > 1 else [0])
    if T:
        qb += [N // BLOCK, nb - 1]
    return sorted(set(qb))


def _check_fp64(q, k, v, out, bits, variant, T, valid, amp, P, n, dtype):
    from jenga_b200.attention import bits_to_onehot
    S = q.shape[1]
    N, nb = S - T, (S + BLOCK - 1) // BLOCK
    ns = nb - (T + BLOCK - 1) // BLOCK
    truth = refutil.fp64_truth(q, k, v, bits_to_onehot(bits, nb), _fp64_blocks(P, n, N, T, nb),
                               n_img_blocks=ns, seqlen=N + valid if T else S, text_amp=amp)
    for qb, t in truth.items():
        r0, r1 = qb * BLOCK, min((qb + 1) * BLOCK, S)
        assert_close(out[0, r0:r1].transpose(0, 1), t[:, :r1 - r0], dtype)


def _epilogue_case(P, G, kind, name, dtype):
    variant, T, valid, amp = VARIANTS[name]
    n_img = _n_img(P, kind)
    n, N, h = n_img // P, n_img, H // P
    hg = h // G
    q, k, v = _inputs(n_img, T, dtype)
    nbr = synth.band_neighbours(n_img // BLOCK)
    ref, bits = _single(variant, q, k, v, T, valid, amp, nbr)
    world = World(P, n, T, dtype)
    world.restate_qkv(q, k, v)
    expect = [f.clone() for f in world.out_full[0]]
    for r in range(P):
        for g in range(G):
            _attend(world, r, g, hg, variant, valid, amp, nbr, world.p_out[0])
            torch.cuda.synchronize()
            hs = slice(r * h + g * hg, r * h + (g + 1) * hg)
            for p in range(P):
                _mid(expect[p], world.out_rows)[:, hs] = _relaid(ref, p, n, T)[:, hs]
            for p in range(P):
                assert _same(world.out_full[0][p], expect[p]), (r, g, p)
    for p in range(P):
        assert _guards_intact(world.out_full[0][p], world.out_rows)
        assert _same(world.out[0][p], _relaid(ref, p, n, T)), p
    _check_fp64(q, k, v, ref, bits, variant, T, valid, amp, P, n, dtype)


@pytest.mark.parametrize("name", list(VARIANTS))
@pytest.mark.parametrize("kind", ["whole", "ragged"])
@pytest.mark.parametrize("P,G", WORLD_G)
def test_epilogue_stores_exactly_its_slab(P, G, kind, name):
    _epilogue_case(P, G, kind, name, torch.bfloat16)


def test_epilogue_fp16():
    _epilogue_case(8, 3, "ragged", "hy_amp", torch.float16)


@pytest.mark.parametrize("P,G", [(1, 1), (8, 3)])
def test_epilogue_through_the_plain_entry_point(monkeypatch, P, G):
    """The same launches through jenga_carved_attn_fwd (no work order) instead of the scheduled
    entry point the operator uses."""
    from jenga_b200 import attention
    lib = attention.lib
    plain = lib.jenga_carved_attn_fwd
    calls = []

    def unscheduled(args, qk, sched, stream):
        assert qk is None
        calls.append(1)
        return plain(args, stream)

    monkeypatch.setattr(lib, "jenga_carved_attn_fwd_sched", unscheduled)
    _epilogue_case(P, G, "ragged", "hy_amp", torch.bfloat16)
    assert len(calls) == 1 + P * G


# ------------------------------------------------------------------------------------------------
# (c) FP8 P.V under the Ulysses epilogue
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,G,kind", [(1, 1, "whole"), (2, 3, "ragged"), (8, 3, "ragged")])
def test_fp8_pv_with_sp_out_equals_the_plain_fp8_launch(P, G, kind):
    from jenga_b200.attention import _launch, quantize_v_fp8
    variant, T, valid, amp = VARIANTS["hy_amp"]
    n_img = _n_img(P, kind)
    n, N, h = n_img // P, n_img, H // P
    hg = h // G
    q, k, v = _inputs(n_img, T, torch.bfloat16)
    nbr = synth.band_neighbours(n_img // BLOCK)
    ref, bits = _single(variant, q, k, v, T, valid, amp, nbr)
    S = N + T
    nb = S // BLOCK
    ns, nt = nb - T // BLOCK, T // BLOCK
    seqlen = _cu(N, T, valid)[1:2]
    full8 = torch.empty_like(ref)
    _launch(q, k, v, bits, ns, nt, D ** -0.5, amp, ns, S, S, nb * BLOCK, full8, seqlen, q.dtype,
            v_fp8=quantize_v_fp8(v))
    torch.cuda.synchronize()
    assert not _same(full8, ref)                      # the FP8 path really ran
    world = World(P, n, T, torch.bfloat16)
    world.restate_qkv(q, k, v)
    for r in range(P):
        for g in range(G):
            qs, ks, vs = (world.qkv[r][w][None, :, g * hg:(g + 1) * hg] for w in range(3))
            hb = r * h + g * hg
            sp = dict(world=P, rank=r, heads_total=H, rows=n, peers=world.p_out[0], head_base=hb)
            _launch(qs, ks, vs, bits[:, hb:hb + hg].contiguous(), ns, nt, D ** -0.5, amp, ns, S, S, nb * BLOCK,
                    None, seqlen, q.dtype, sp_out=sp, v_fp8=quantize_v_fp8(vs))
    torch.cuda.synchronize()
    for p in range(P):
        assert _guards_intact(world.out_full[0][p], world.out_rows)
        assert _same(world.out[0][p], _relaid(full8, p, n, T)), p


# ------------------------------------------------------------------------------------------------
# (d) the production classes, one Python thread per emulated rank
# ------------------------------------------------------------------------------------------------
class _FakeGroup:
    def __init__(self, size, rank):
        self.size, self.rank = size, rank


class _Handle:
    """Stands in for a symmetric-memory handle: barrier() waits for the device, then for every rank."""

    def __init__(self, bar):
        self._bar = bar

    def barrier(self, channel=0):
        torch.cuda.synchronize()
        self._bar.wait(timeout=BARRIER_TIMEOUT_S)


def _emulated_fused(world, bar):
    from jenga_b200.ulysses import UlyssesFusedAttention

    class EmulatedFused(UlyssesFusedAttention):
        def _buffers(self, N, T, h, D_, n_loc, H_, dtype, dev):
            assert (N, T, h, n_loc, H_) == (world.N, world.T, world.h, world.n, H)
            r, hd = self.group.rank, _Handle(bar)
            return world.qkv[r], hd, world.p_qkv, [(world.out[b][r], hd, world.p_out[b]) for b in range(2)]

    return EmulatedFused


def _run_ranks(P, body):
    """body(rank, barrier) in P threads; the first exception of any rank breaks the barrier for
    the others and is raised here."""
    bar = threading.Barrier(P)
    errors = []

    def run(r):
        try:
            body(r, bar)
        except BaseException as e:   # noqa: BLE001
            errors.append((r, e))
            bar.abort()

    threads = [threading.Thread(target=run, args=(r,), daemon=True) for r in range(P)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=4 * BARRIER_TIMEOUT_S)
    assert not any(t.is_alive() for t in threads), "a rank thread did not finish"
    if errors:
        real = [e for e in errors if not isinstance(e[1], threading.BrokenBarrierError)] or errors
        raise AssertionError(f"rank {real[0][0]} failed") from real[0][1]


@pytest.mark.parametrize("P,G", [(1, None), (2, 1), (2, 3), (4, None), (8, None), (8, 3)])
def test_production_classes_on_emulated_ranks(monkeypatch, P, G):
    """UlyssesFusedAttention and HostPipelinedUlysses, unmodified, called three times (inputs A, B, A)
    by P threads; only the process-group plumbing is substituted."""
    from jenga_b200 import ulysses
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    monkeypatch.setattr(ulysses.dist, "get_world_size", lambda g=None: g.size)
    variant, T, valid, amp = VARIANTS["hy_amp"]
    n_img = _n_img(P, "ragged")
    n, N = n_img // P, n_img
    nbr = synth.band_neighbours(n_img // BLOCK)
    sets = [_inputs(n_img, T, torch.bfloat16, seed) for seed in (4100, 4200)]
    refs = [_single(variant, *x, T, valid, amp, nbr)[0] for x in sets]
    assert not _same(refs[0], refs[1])
    order = (0, 1, 0)
    cu = torch.tensor([0, n + valid, n + T], dtype=torch.int32, device=DEV)   # as each rank builds it
    kw = dict(top_k=TOP_K, text_amp=amp, block_neighbor_list=nbr, p_remain_rates=P_REMAIN)

    def local(x, r):
        return torch.cat([x[:, r * n:(r + 1) * n], x[:, N:]], dim=1)

    # UlyssesFusedAttention, through my_parallel_attention as the DiT blocks call it
    world = World(P, n, T, torch.bfloat16, n_out=2)
    got = [dict() for _ in range(P)]

    def fused_rank(r, bar):
        sp = _emulated_fused(world, bar)(group=_FakeGroup(P, r), variant=variant, groups=G)
        outs = []
        for i, s in enumerate(order):
            ql, kl, vl = (local(x, r) for x in sets[s])
            outs.append(ulysses.my_parallel_attention(sp, ql, kl, vl, n, n, cu, cu, **kw))
            torch.cuda.synchronize()
            got[r][f"call{i}"] = outs[-1].clone()
            if i == 1:
                got[r]["call0_after_call1"] = outs[0].clone()
        got[r]["reuse"] = outs[2].data_ptr() == outs[0].data_ptr() != outs[1].data_ptr()

    _run_ranks(P, fused_rank)
    for r in range(P):
        for i, s in enumerate(order):
            assert _same(got[r][f"call{i}"].view(n + T, H, D), _relaid(refs[s], r, n, T)), (r, i)
        assert _same(got[r]["call0_after_call1"], got[r]["call0"]), r      # the double buffer
        assert got[r]["reuse"], r
    for b in range(2):
        for p in range(P):
            assert _guards_intact(world.out_full[b][p], world.out_rows)
    for p in range(P):
        assert _guards_intact(world.qkv_full[p], world.qkv_rows)

    # HostPipelinedUlysses on pinned host activations, on fresh buffers
    world2 = World(P, n, T, torch.bfloat16, n_out=2)
    host = [[local(x, r).cpu().pin_memory() for x in s] for r in range(P) for s in sets]
    hout = [[torch.empty((1, n + T, H, D), dtype=torch.bfloat16).pin_memory() for _ in order] for _ in range(P)]

    def host_rank(r, bar):
        fused = _emulated_fused(world2, bar)(group=_FakeGroup(P, r), variant=variant, groups=G)
        hp = ulysses.HostPipelinedUlysses(n, T, H, D, dtype=torch.bfloat16, device=DEV, fused=fused)
        for i, s in enumerate(order):
            hq, hk, hv = host[r * len(sets) + s]
            hp(hq, hk, hv, hout[r][i], cu_seqlens_q=cu, cu_seqlens_kv=cu, **kw)
        torch.cuda.synchronize()

    _run_ranks(P, host_rank)
    for r in range(P):
        for i in range(len(order)):
            assert _same(hout[r][i].to(DEV), got[r][f"call{i}"].view(1, n + T, H, D)), (r, i)
    for b in range(2):
        for p in range(P):
            assert _guards_intact(world2.out_full[b][p], world2.out_rows)


# ------------------------------------------------------------------------------------------------
# (e) full size, kernel layer
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,P", [("hy720p", 8), ("hy_i2v", 8), ("hy_turbo_s0", 2)])
def test_full_size_emulated_ranks_equal_single_gpu(name, P):
    """bench.py's workloads at the world sizes they run on: n_loc = 14400 (112.5 blocks) at HY-720p
    on 8 GPUs, 31680 (247.5 blocks) at HY-Turbo stage 0 on 2.  The inbound exchange runs on views
    of the global tensors, the attention with the head sub-groups UlyssesFusedAttention picks."""
    import bench
    from jenga_b200.ulysses import UlyssesFusedAttention
    wl = bench.workload(name, 0.7)
    inp = bench.build_inputs(wl, DEV)
    q, k, v = inp["q"], inp["k"], inp["v"]
    S, N, T = inp["S"], inp["n_img"], wl["text_tokens"]
    n, h = N // P, H // P
    assert n * P == N
    ref = bench.run_operator(wl, inp).view(1, S, H, D)
    G = UlyssesFusedAttention._n_groups(h, None, (S + BLOCK - 1) // BLOCK)
    hg = h // G
    world = World(P, n, T, torch.bfloat16)
    for r in range(P):
        xs = [x[:, r * n:(r + 1) * n] for x in (q, k, v)]
        for g in range(G):
            _scatter(xs, [x[:, N:] for x in (q, k, v)], P, r, n, T, world.p_qkv, g * hg, hg)
    torch.cuda.synchronize()
    for p in range(P):
        assert _guards_intact(world.qkv_full[p], world.qkv_rows)
        for w, x in enumerate((q, k, v)):
            assert _same(world.qkv[p][w], x[0, :, p * h:(p + 1) * h]), (p, w)
    for r in range(P):
        for g in range(G):
            _attend(world, r, g, hg, wl["variant"], wl["text_valid"], wl["text_amp"], inp["nbr"], world.p_out[0],
                    top_k=inp["top_k"], p_remain=wl["p_remain"])
    torch.cuda.synchronize()
    for p in range(P):
        assert _guards_intact(world.out_full[0][p], world.out_rows)
        assert _same(world.out[0][p], _relaid(ref, p, n, T)), p
