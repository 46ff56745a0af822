"""Sequence-parallel Wan2.1 self-attention (blocks._wan_self under `jenga_sp`), emulated on one GPU.

The ranks are emulated as tests/test_ulysses_emulated_gpu.py does: every rank's exchange buffers on
one device (here at the Wan head counts, each result buffer filled with a 16-bit NaN pattern first),
UlyssesFusedAttention unmodified, one Python thread per rank with host barriers.

* Attention section: each rank runs the norm + RoPE prologue on its Hilbert rows, the exchange, and the
  operator over the first L exchanged rows.  Its real rows equal, bit for bit, the single-GPU result:
  WAN.self_attention for carved calls (sa_drop_rate 0.7), the flash_attn_varlen_func shim over the same
  bf16 q / k / v for dense calls (0.2, the warm-up steps); every selection of the ranks' head groups
  equals the single-GPU one.  The pad rows of the last rank are zero.  40 heads at P = 1, 2, 4, 8 and 12
  heads at P = 3, 6, over every head sub-group count of 1-3 that divides; the whole grid 21x8x16 and the
  ragged grid 21x9x14 (first_frame_blocks 1 in both).  Wan-14B 21x45x80 and its turbo grid 21x33x60
  (41 580 rows, ragged over 8) at P = 8, and JENGA_QK_INT8 at P = 4.
* Blocks: an unmodified T2V WanAttentionBlock at P = 2 and 4, against the single-GPU fused forward,
  within the tolerance of tests/test_wan_blocks_gpu.py on rows whose selections are equal.
"""
import copy
import ctypes as C
import sys
import threading
import types
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
from test_ulysses_emulated_gpu import CANARY, _FakeGroup, _Handle, _run_ranks  # noqa: E402
from test_wan_blocks_gpu import _compare, _make_blocks, _structured_tokens  # noqa: E402

DEV = torch.device("cuda", 0)
D, BLOCK = 128, 128
P_REMAIN = 0.8
CARVED, DENSE = 0.7, 0.2
GRIDS = {"whole": (21, 8, 16), "ragged": (21, 9, 14)}
CASES = [(H, P, G) for H, Ps in ((40, (1, 2, 4, 8)), (12, (3, 6))) for P in Ps for G in (1, 2, 3)
         if (H // P) % G == 0]


@pytest.fixture
def emulated_groups(monkeypatch):
    from jenga_b200 import ulysses
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    monkeypatch.setattr(ulysses.dist, "get_world_size", lambda g=None: g.size)


class _World:
    """P ranks' buffers as UlyssesFusedAttention allocates them for T = 0: qkv [3, N, h, D] and two
    result buffers [n, H, D] each, the result buffers canary-filled"""

    def __init__(self, P, n, H):
        self.P, self.n, self.H, self.N, self.h = P, n, H, P * n, H // P
        self.qkv = [torch.empty((3, self.N, self.h, D), dtype=torch.bfloat16, device=DEV) for _ in range(P)]
        self.out = [[torch.empty((n, H, D), dtype=torch.bfloat16, device=DEV) for _ in range(P)] for _ in range(2)]
        for b in self.out:
            for o in b:
                o.view(torch.int16).fill_(CANARY)
        self.p_qkv = (C.c_uint64 * P)(*[t.data_ptr() for t in self.qkv])
        self.p_out = [(C.c_uint64 * P)(*[o.data_ptr() for o in b]) for b in self.out]

    def fused(self, bar, P, r, G):
        from jenga_b200.ulysses import UlyssesFusedAttention
        world = self

        class EmulatedFused(UlyssesFusedAttention):
            def _buffers(self, N, T, h, D_, n_loc, H_, dtype, dev):
                assert (N, T, h, n_loc, H_) == (world.N, 0, world.h, world.n, world.H)
                hd = _Handle(bar)
                return world.qkv[r], hd, world.p_qkv, [(world.out[b][r], hd, world.p_out[b]) for b in range(2)]

        return EmulatedFused(group=_FakeGroup(P, r), variant="wan", groups=G)


class _Capture(list):
    """attention.MASK_CAPTURE that records which emulated rank appended each selection"""
    local = threading.local()

    def append(self, item):
        super().append((getattr(self.local, "rank", None), item))


class WanRMSNorm(torch.nn.Module):
    """the two attributes of the reference WanRMSNorm the fused forward reads"""

    def __init__(self, weight, eps=1e-6):
        super().__init__()
        self.weight, self.eps = weight, eps


def _module(H, wq, wk, jsp):
    """a WanSelfAttention whose q / k / v Linears are slices of one [1, n, 3C] input and whose o is the
    identity: the section under test is everything between them"""
    Cc = H * D
    return types.SimpleNamespace(num_heads=H, head_dim=D, norm_q=WanRMSNorm(wq), norm_k=WanRMSNorm(wk), jenga_sp=jsp,
                                 q=lambda x: x[..., :Cc], k=lambda x: x[..., Cc:2 * Cc], v=lambda x: x[..., 2 * Cc:],
                                 o=lambda t: t)


def _section_case(H, grid, seed=5200):
    from jenga_b200 import gilbert
    f, h, w = grid
    L = f * h * w
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = (_structured_tokens(L, 3 * H * D, seed) * 0.5).contiguous()
    wq, wk = ((1.0 + 0.2 * torch.randn(H * D, generator=g, device=DEV)) for _ in range(2))
    _, h2l = gilbert.mapping_tensors(f, h, w, sliced=True)
    return dict(L=L, qkv=qkv, wq=wq, wk=wk, h2l=h2l.to(DEV), nbr=gilbert.block_neighbor_mapping(f, h, w, sliced=True),
                grid=torch.tensor([[f, h, w]]), freqs=_freqs())


def _freqs():
    from jenga_b200.wan import rope_freqs
    return rope_freqs(D)


def _single(H, c, drop):
    """the single-GPU result [1, L, H*D] fp32 and its selection (None for dense calls)"""
    from jenga_b200 import attention as A, wan as WAN
    from jenga_b200.flash_attn_shim import flash_attn_varlen_func
    Cc = H * D
    x = c["qkv"]
    q_lin, k_lin, v = x[..., :Cc], x[..., Cc:2 * Cc], x[..., 2 * Cc:].view(1, c["L"], H, D)
    grid = c["grid"][0].tolist()
    A.MASK_CAPTURE = []
    try:
        if drop > 0.25:
            out = WAN.self_attention(q_lin, k_lin, v, c["wq"], c["wk"], H, grid, c["freqs"], drop,
                                     p_remain_rates=P_REMAIN, freq_remap=c["h2l"], block_neighbor_list=c["nbr"])
            bits = A.MASK_CAPTURE[0][0]
        else:
            q = WAN.norm_rope(q_lin, c["wq"], H, grid, c["freqs"], c["h2l"])
            k = WAN.norm_rope(k_lin, c["wk"], H, grid, c["freqs"], c["h2l"])
            cu = torch.tensor([0, c["L"]], dtype=torch.int32, device=DEV)
            out = flash_attn_varlen_func(q[0], k[0], v[0].contiguous(), cu, cu, c["L"], c["L"])[None]
            bits = None
    finally:
        A.MASK_CAPTURE = None
    return out.flatten(2).float(), bits


def _sharded(H, P, G, c, drop):
    """every emulated rank's [1, n, H*D] result and its selections, in rank order"""
    from jenga_b200 import attention as A, blocks
    from jenga_b200.sharding import shard
    n = -(-c["L"] // P)
    world = _World(P, n, H)
    got, cap = {}, _Capture()

    def rank(r, bar):
        _Capture.local.rank = r
        m = _module(H, c["wq"], c["wk"], world.fused(bar, P, r, G))
        with torch.no_grad():
            out = blocks._wan_self(m, shard(c["qkv"], 1, P, r), torch.tensor([c["L"]]), c["grid"], c["freqs"],
                                   sa_drop_rate=drop, p_remain_rates=P_REMAIN, freq_remap=shard(c["h2l"], 0, P, r),
                                   block_neighbor_list=c["nbr"])
        torch.cuda.synchronize()
        got[r] = out.clone()

    A.MASK_CAPTURE = cap
    try:
        before = dict(blocks.STATS)
        _run_ranks(P, rank)
    finally:
        A.MASK_CAPTURE = None
    key = "wan_self_dense_sp" if drop <= 0.25 else "wan_self_sp"
    assert blocks.STATS[key] == before[key] + P and blocks.STATS["fallback"] == before["fallback"]
    per_rank = {}
    for r, (bits, _) in cap:
        per_rank.setdefault(r, []).append(bits)
    return [got[r] for r in range(P)], per_rank, n


def _check(H, P, c, drop, got, per_rank, n, single, single_bits):
    L = c["L"]
    for r in range(P):
        lo, hi = min(r * n, L), min((r + 1) * n, L)
        assert got[r].shape == (1, n, H * D)
        assert torch.equal(got[r][:, :hi - lo].view(torch.int32), single[:, lo:hi].view(torch.int32)), (r, lo, hi)
        assert bool((got[r][:, hi - lo:] == 0).all()), f"rank {r}: pad rows are not zero"
    if single_bits is None:
        assert not per_rank, "a dense call ran a selection"
    else:
        sp_bits = torch.cat([b for r in range(P) for b in per_rank[r]], dim=1)    # rank order, then sub-groups
        assert torch.equal(sp_bits, single_bits)


@pytest.mark.parametrize("grid", ["whole", "ragged"])
@pytest.mark.parametrize("H,P,G", CASES)
def test_sharded_self_attention_equals_single_gpu(emulated_groups, H, P, G, grid):
    c = _section_case(H, GRIDS[grid])
    assert -(-c["L"] // BLOCK) // 21 == 1                                       # first_frame_blocks 1
    for drop in (CARVED, DENSE):
        single, bits = _single(H, c, drop)
        got, per_rank, n = _sharded(H, P, G, c, drop)
        _check(H, P, c, drop, got, per_rank, n, single, bits)


@pytest.mark.parametrize("name,grid", [("Wan-14B", (21, 45, 80)), ("Wan-14B turbo", (21, 33, 60))])
def test_full_size_at_eight_ranks(emulated_groups, name, grid):
    H, P = 40, 8
    c = _section_case(H, grid, seed=5300)
    single, bits = _single(H, c, CARVED)
    got, per_rank, n = _sharded(H, P, None, c, CARVED)
    print(f"\n[wan sp] {name}: L = {c['L']}, {n} rows per rank, {P * n - c['L']} pad rows")
    _check(H, P, c, CARVED, got, per_rank, n, single, bits)


def test_qk_int8_equals_single_gpu(emulated_groups, monkeypatch):
    from jenga_b200 import attention as A
    monkeypatch.setattr(A, "QK_INT8", True)
    H, P = 40, 4
    c = _section_case(H, GRIDS["ragged"], seed=5400)
    for drop in (CARVED, DENSE):
        single, bits = _single(H, c, drop)
        got, per_rank, n = _sharded(H, P, None, c, drop)
        _check(H, P, c, drop, got, per_rank, n, single, bits)


# ------------------------------------------------------------------------------------------------
# the unmodified T2V block
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def wan_module():
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    ours = R.load_blocks(product=True)[1]
    assert ours.WanAttentionBlock.forward.__jenga_b200__ and ours.WanSelfAttention.forward.__jenga_b200__
    yield ours
    from jenga_b200 import blocks
    blocks.remove_gather_hook()


@pytest.mark.parametrize("P", [2, 4])
def test_unmodified_block_under_sp_matches_single_gpu(emulated_groups, wan_module, P):
    from jenga_b200 import attention as A, blocks, gilbert
    from jenga_b200.attention import bits_to_onehot
    from jenga_b200.sharding import shard
    f, h, w = GRIDS["ragged"]
    L, dim, H = f * h * w, 1536, 12
    blk = _make_blocks(wan_module, 1, dim=dim, H=H)[0]
    _, h2l = gilbert.mapping_tensors(f, h, w, sliced=True)
    g = torch.Generator(device="cuda").manual_seed(41)
    x = _structured_tokens(L, dim, 41)
    e = 0.3 * torch.randn(1, 6, dim, generator=g, device="cuda")
    ctx = torch.randn(1, 512, dim, generator=g, device="cuda").bfloat16()
    d = dim // H
    freqs = torch.cat([wan_module.rope_params(1024, d - 4 * (d // 6)), wan_module.rope_params(1024, 2 * (d // 6)),
                       wan_module.rope_params(1024, 2 * (d // 6))], dim=1).cuda()
    nbr = gilbert.block_neighbor_mapping(f, h, w, sliced=True)
    grid = torch.tensor([[f, h, w]])

    def call(b, xx, remap):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            return b(xx, e, torch.tensor([L]), grid, freqs, ctx, None, sa_drop_rate=0.75, freq_remap=remap,
                     block_neighbor_list=nbr, p_remain_rates=0.9)

    cap = _Capture()
    A.MASK_CAPTURE = cap
    try:
        before = dict(blocks.STATS)
        ref = call(blk, x, h2l.cuda())
        torch.cuda.synchronize()
        assert blocks.STATS["wan_self"] == before["wan_self"] + 1
        n = -(-L // P)
        world = _World(P, n, H)
        ranks = [copy.deepcopy(blk) for _ in range(P)]
        got = {}

        def rank(r, bar):
            _Capture.local.rank = r
            ranks[r].self_attn.jenga_sp = world.fused(bar, P, r, None)
            got[r] = call(ranks[r], shard(x, 1, P, r), shard(h2l, 0, P, r).cuda()).clone()
            torch.cuda.synchronize()

        before = dict(blocks.STATS)
        _run_ranks(P, rank)
    finally:
        A.MASK_CAPTURE = None
    assert blocks.STATS["wan_self_sp"] == before["wan_self_sp"] + P and blocks.STATS["wan_block"] == before["wan_block"] + P
    assert blocks.STATS["fallback"] == before["fallback"] and blocks.STATS["wan_self"] == before["wan_self"]
    single = [b for r, (b, _) in cap if r is None]
    per_rank = {r: b for r, (b, _) in cap if r is not None}
    nb = -(-L // BLOCK)
    sp_bits = torch.cat([per_rank[r] for r in range(P)], dim=1)
    same = (bits_to_onehot(single[0], nb) == bits_to_onehot(sp_bits, nb)).all(-1).all(1)[0]
    row_ok = same.repeat_interleave(BLOCK)[:L]
    got_rows = torch.cat([got[r][:, :max(0, min(n, L - r * n))] for r in range(P)], 1)
    _compare(ref, got_rows, row_ok, f"T2V block under SP, P={P}")
