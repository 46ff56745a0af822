"""Sequence-parallel Wan2.1-I2V on the GPU: blocks._wan_i2v_self under `jenga_sp`, the unmodified
wan/modules/model.py blocks, and parallelize_wan_i2v's forward.

The ranks are emulated on one device as tests/test_wan_sp_gpu.py and tests/test_wan_sp_forward_gpu.py do
(every rank's exchange buffers on one device, result buffers canary-filled, UlyssesFusedAttention
unmodified, one thread per rank).

* Attention section: each rank runs the norm + RoPE prologue on its raster rows, the exchange, and the
  dense class over the first L exchanged rows.  Its real rows equal, bit for bit, the single-GPU dense
  self-attention of the same rows (the prologue over all L rows, then the flash_attn_varlen_func shim);
  its pad rows are zero.  40 heads at P = 1, 2, 4, 8 on the grid 21x8x16 and the ragged 21x9x14, and
  Wan-I2V-14B 720p (21x45x80, 9 450 rows per rank) at P = 8.
* Blocks: two unmodified I2V WanAttentionBlocks of wan/modules/model.py at P = 2 and 4, against the
  single-GPU original forward (the reference block, self-attention and cross-attention forwards through
  the flash_attn shim), within the drop-in tolerance of tests/test_wan_blocks_gpu.py.
* Forward: parallelize_wan_i2v over a small random-init I2V WanModel at P = 2 and 4 against the
  single-GPU I2V TeaCache forward, on two computed steps and a skipped step; on two GPUs (skipped on a
  one-GPU box) the real exchange against the emulated run.
"""
import copy
import os
import sys
import types
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
from test_ulysses_emulated_gpu import _run_ranks  # noqa: E402
from test_wan_blocks_gpu import _compare, _reinit, _structured_tokens  # noqa: E402
from test_wan_i2v_gpu import _i2v_context  # noqa: E402
from test_wan_i2v_sp_cpu import _i2v_teacache_single, load_plain_wan  # noqa: E402
from test_wan_sp_forward_gpu import _emulated_all_gather, _emulated_broadcast, _Group, _rows  # noqa: E402
from test_wan_sp_gpu import WanRMSNorm, _World  # noqa: E402

DEV = torch.device("cuda", 0)
D = 128
GRIDS = {"whole": (21, 8, 16), "ragged": (21, 9, 14)}
CASES = [(P, G) for P in (1, 2, 4, 8) for G in (1, 2) if (40 // P) % G == 0]


@pytest.fixture
def emulated_groups(monkeypatch):
    from jenga_b200 import ulysses
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    monkeypatch.setattr(ulysses.dist, "get_world_size", lambda g=None: g.size)


@pytest.fixture(scope="module")
def plain_wan():
    mod = load_plain_wan(wan_sp=True)
    if mod is None:
        pytest.skip("reference files not staged (oracle/_ref/, oracle/_ref_wan_model/)")
    assert mod.WanAttentionBlock.forward.__jenga_b200__ and mod.WanSelfAttention.forward.__jenga_b200__
    return mod


# ------------------------------------------------------------------------------------------------
# the attention section
# ------------------------------------------------------------------------------------------------
def _section_case(H, grid, seed):
    from jenga_b200.wan import rope_freqs
    f, h, w = grid
    L = f * h * w
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = (_structured_tokens(L, 3 * H * D, seed) * 0.5).contiguous()
    wq, wk = ((1.0 + 0.2 * torch.randn(H * D, generator=g, device=DEV)) for _ in range(2))
    return dict(L=L, qkv=qkv, wq=wq, wk=wk, grid=torch.tensor([[f, h, w]]), freqs=rope_freqs(D))


def _single(H, c):
    """the single-GPU dense self-attention [1, L, H*D] fp32: the prologue over all L rows in raster
    order, then the flash_attn_varlen_func shim"""
    from jenga_b200 import wan as WAN
    from jenga_b200.flash_attn_shim import flash_attn_varlen_func
    Cc, L = H * D, c["L"]
    x = c["qkv"]
    grid = c["grid"][0].tolist()
    q = WAN.norm_rope(x[..., :Cc], c["wq"], H, grid, c["freqs"])
    k = WAN.norm_rope(x[..., Cc:2 * Cc], c["wk"], H, grid, c["freqs"])
    v = x[..., 2 * Cc:].view(1, L, H, D)
    cu = torch.tensor([0, L], dtype=torch.int32, device=DEV)
    return flash_attn_varlen_func(q[0], k[0], v[0].contiguous(), cu, cu, L, L)[None].flatten(2).float()


def _sharded(H, P, G, c):
    from jenga_b200 import blocks
    from jenga_b200.sharding import shard
    Cc = H * D
    n = -(-c["L"] // P)
    world = _World(P, n, H)
    got = {}

    def rank(r, bar):
        m = types.SimpleNamespace(num_heads=H, head_dim=D, norm_q=WanRMSNorm(c["wq"]), norm_k=WanRMSNorm(c["wk"]),
                                  jenga_sp=world.fused(bar, P, r, G), q=lambda x: x[..., :Cc],
                                  k=lambda x: x[..., Cc:2 * Cc], v=lambda x: x[..., 2 * Cc:], o=lambda t: t)
        with torch.no_grad():
            out = blocks._wan_i2v_self(m, shard(c["qkv"], 1, P, r), torch.tensor([c["L"]]), c["grid"], c["freqs"])
        torch.cuda.synchronize()
        got[r] = out.clone()

    before = dict(blocks.STATS)
    _run_ranks(P, rank)
    assert blocks.STATS["wan_i2v_self_sp"] == before["wan_i2v_self_sp"] + P
    assert blocks.STATS["fallback"] == before["fallback"]
    return [got[r] for r in range(P)], n


def _check(H, P, c, got, n, single):
    L = c["L"]
    for r in range(P):
        lo, hi = min(r * n, L), min((r + 1) * n, L)
        assert got[r].shape == (1, n, H * D)
        assert torch.equal(got[r][:, :hi - lo].view(torch.int32), single[:, lo:hi].view(torch.int32)), (r, lo, hi)
        assert bool((got[r][:, hi - lo:] == 0).all()), f"rank {r}: pad rows are not zero"


@pytest.mark.parametrize("grid", ["whole", "ragged"])
@pytest.mark.parametrize("P,G", CASES)
def test_sharded_self_attention_equals_single_gpu_dense(emulated_groups, P, G, grid):
    H = 40
    c = _section_case(H, GRIDS[grid], 6100)
    got, n = _sharded(H, P, G, c)
    _check(H, P, c, got, n, _single(H, c))


def test_wan_i2v_14b_720p_at_eight_ranks(emulated_groups):
    H, P = 40, 8
    c = _section_case(H, (21, 45, 80), 6200)
    got, n = _sharded(H, P, None, c)
    print(f"\n[wan i2v sp] 21x45x80: L = {c['L']}, {n} rows per rank")
    _check(H, P, c, got, n, _single(H, c))


# ------------------------------------------------------------------------------------------------
# the unmodified wan/modules/model.py blocks
# ------------------------------------------------------------------------------------------------
def _freqs(mod, dim, H):
    d = dim // H
    return torch.cat([mod.rope_params(1024, d - 4 * (d // 6)), mod.rope_params(1024, 2 * (d // 6)),
                      mod.rope_params(1024, 2 * (d // 6))], dim=1).cuda()


@pytest.mark.parametrize("P", [2, 4])
def test_unmodified_i2v_blocks_under_sp_match_the_original_forward(emulated_groups, plain_wan, P):
    from jenga_b200 import blocks
    from jenga_b200.sharding import shard
    f, h, w = GRIDS["ragged"]
    L, dim, H = f * h * w, 1536, 12
    blks = [plain_wan.WanAttentionBlock("i2v_cross_attn", dim, 8960, H, (-1, -1), True, True, 1e-6).cuda()
            for _ in range(2)]
    for i, b in enumerate(blks):
        _reinit(b, 80 + i)
    g = torch.Generator(device="cuda").manual_seed(81)
    x = _structured_tokens(L, dim, 81)
    e = 0.3 * torch.randn(1, 6, dim, generator=g, device="cuda")
    ctx = _i2v_context(dim, 82)
    freqs = _freqs(plain_wan, dim, H)
    grid = torch.tensor([[f, h, w]])
    original = type(blks[0]).forward.__wrapped__

    def chain(bs, xx, fwd):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            for b in bs:
                xx = fwd(b, xx, e, torch.tensor([L]), grid, freqs, ctx, None)
        return xx

    ref = chain(blks, x, original)
    torch.cuda.synchronize()
    n = -(-L // P)
    world = _World(P, n, H)
    ranks = [copy.deepcopy(blks) for _ in range(P)]
    got = {}

    def rank(r, bar):
        sp = world.fused(bar, P, r, None)
        for b in ranks[r]:
            b.self_attn.jenga_sp = sp
        got[r] = chain(ranks[r], shard(x, 1, P, r), lambda b, *a: b(*a)).clone()
        torch.cuda.synchronize()

    before = dict(blocks.STATS)
    _run_ranks(P, rank)
    for k, v in dict(wan_i2v_self_sp=2 * P, wan_i2v_cross_sp=2 * P, wan_block=2 * P, fallback=0, wan_i2v_cross=0).items():
        assert blocks.STATS[k] - before[k] == v, k
    got_rows = torch.cat([got[r][:, :max(0, min(n, L - r * n))] for r in range(P)], 1)
    _compare(ref, got_rows, torch.ones(L, dtype=torch.bool, device="cuda"), f"I2V blocks under SP, P={P}")


# ------------------------------------------------------------------------------------------------
# parallelize_wan_i2v's forward
# ------------------------------------------------------------------------------------------------
DIM, HEADS, LAYERS, TEXT_LEN, TEXT_DIM = 1536, 12, 2, 64, 256
GRID = GRIDS["ragged"]
STEPS = 3                       # cnt 0 and 1 computed, cnt 2 (even, rel-L1 0) skipped


def _model(mod, dev):
    torch.manual_seed(0)
    m = mod.WanModel(model_type="i2v", patch_size=(1, 2, 2), text_len=TEXT_LEN, in_dim=36, dim=DIM, ffn_dim=2048,
                     freq_dim=256, text_dim=TEXT_DIM, out_dim=16, num_heads=HEADS, num_layers=LAYERS).to(dev).eval()
    with torch.cuda.device(dev):
        _reinit(m, 5)                   # init_weights zeroes the head: the output would be all zero
    # the I2V TeaCache attributes of jenga_wan.py:1188-1213
    m.enable_teacache, m.cnt, m.num_steps, m.teacache_thresh = True, 0, 80, 0.5
    m.accumulated_rel_l1_distance_even = m.accumulated_rel_l1_distance_odd = 0
    m.previous_e0_even = m.previous_e0_odd = m.previous_residual_even = m.previous_residual_odd = None
    m.use_ref_steps, m.use_cache = False, False
    m.coefficients, m.ret_steps, m.cutoff_steps = [1.0, 0.0], 2, 78
    return m


def _inputs(dev, seed=7):
    g = torch.Generator(device=dev).manual_seed(seed)
    f, h, w = GRID
    x = [torch.randn(16, f, 2 * h, 2 * w, generator=g, device=dev)]
    y = [torch.randn(20, f, 2 * h, 2 * w, generator=g, device=dev)]
    ctx = [torch.randn(TEXT_LEN - 9, TEXT_DIM, generator=g, device=dev)]
    clip = torch.randn(1, 257, 1280, generator=g, device=dev)
    return x, ctx, clip, y


def _run(model, fwd, dev, P=1):
    x, ctx, clip, y = _inputs(dev)
    L = GRID[0] * GRID[1] * GRID[2]
    outs, used = [], []
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for _ in range(STEPS):
            outs.append(fwd(x, torch.tensor([900.0], device=dev), ctx, -(-L // P) * P, clip_fea=clip, y=y)[0].clone())
            used.append(model.use_cache)
    assert used == [False, False, True]
    return outs


def _emulated(P, monkeypatch, single_model):
    from jenga_b200 import ulysses, wan_sp
    dist = ulysses.dist
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    monkeypatch.setattr(dist, "get_world_size", lambda g=None: g.size)
    monkeypatch.setattr(dist, "get_rank", lambda g=None: g.rank)
    monkeypatch.setattr(dist, "get_global_rank", lambda g, r: r)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "all_gather", _emulated_all_gather)
    monkeypatch.setattr(dist, "broadcast", _emulated_broadcast)
    models = [copy.deepcopy(single_model) for _ in range(P)]
    L = GRID[0] * GRID[1] * GRID[2]
    world = _World(P, -(-L // P), HEADS)
    shared = {"rows": {}}
    got = {}

    def rank(r, bar):
        shared["bar"] = bar
        wan_sp.parallelize_wan_i2v(models[r], group=_Group(P, r, shared), attention=world.fused(bar, P, r, None))
        got[r] = _run(models[r], models[r].forward, DEV, P)

    _run_ranks(P, rank)
    return got


def _single_gpu(mod):
    model = _model(mod, DEV)
    ref_model = copy.deepcopy(model)
    return _run(ref_model, lambda *a, **k: _i2v_teacache_single(ref_model, *a, **k), DEV), model


@pytest.mark.parametrize("P", [2, 4])
def test_sharded_i2v_forward_matches_single_gpu(plain_wan, monkeypatch, P):
    from jenga_b200 import blocks
    ref, model = _single_gpu(plain_wan)
    before = dict(blocks.STATS)
    got = _emulated(P, monkeypatch, model)
    # per rank: 2 computed steps x 2 blocks
    assert blocks.STATS["wan_i2v_self_sp"] - before["wan_i2v_self_sp"] == 4 * P
    assert blocks.STATS["wan_i2v_cross_sp"] - before["wan_i2v_cross_sp"] == 4 * P
    assert blocks.STATS["fallback"] == before["fallback"]
    for i, name in enumerate(["computed", "computed", "skipped"]):
        for r in range(P):
            assert torch.equal(got[r][i], got[0][i]), (r, i)
        rows = _rows(ref[i])
        _compare(rows, _rows(got[0][i]), torch.ones(rows.shape[1], dtype=torch.bool, device="cuda"),
                 f"sharded Wan I2V forward P={P}, step {i} ({name})")


def _two_gpu_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        from jenga_b200 import blocks, wan_sp
        mod = load_plain_wan(wan_sp=True)
        dev = torch.device("cuda", rank)
        model = _model(mod, dev)
        sp = wan_sp.parallelize_wan_i2v(model)
        outs = _run(model, model.forward, dev, world)
        torch.cuda.synchronize()
        ret[rank] = dict(outs=[o.cpu() for o in outs], exchange=type(sp).__name__, fallback=blocks.STATS["fallback"])
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_gpus_real_exchange_matches_the_emulated_run(plain_wan, monkeypatch):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_two_gpu_worker, args=(world, 29500 + (os.getpid() + 3) % 2000, ret), nprocs=world, join=True)
    emu = _emulated(world, monkeypatch, _model(plain_wan, DEV))
    for r in range(world):
        got = ret[r]
        print(f"\n[two GPUs] rank {r}: exchange {got['exchange']}")
        assert got["fallback"] == 0
        for i in range(STEPS):
            rows = _rows(got["outs"][i].to("cuda"))
            _compare(_rows(emu[0][i]), rows, torch.ones(rows.shape[1], dtype=torch.bool, device="cuda"),
                     f"two GPUs rank {r} vs emulated, step {i}")
