"""parallelize_wan's sharded TeaCache forward over a real, patched Wan2.1 T2V model.

A small random-init WanModel from wan/modules/model_mul.py (two blocks at 12 heads of 128 channels,
patched by install()), with the Jenga curve and TeaCache attributes jenga_wan.py sets.  The reference
is the single-GPU restatement of teacache_forward (tests/test_wan_sp_cpu.py) over the same model without
jenga_sp, i.e. the single-GPU fused forward.  The steps are those of the CPU test: a dense warm-up
step, a carved step, a TeaCache-skipped step and the two calls after the turbo curve / grid swap, on
the ragged grids 21x9x14 and 21x7x10.

* Emulated ranks (every GPU box): UlyssesFusedAttention on one device, one thread per rank, the
  process-group calls the sharded forward makes (rank, size, broadcast, all_gather) answered by the
  threads.  Every rank's output equals the others' bit for bit and the single-GPU forward within the
  tolerance of tests/test_wan_blocks_gpu.py, at P = 2 and 4.
* Two GPUs (skipped on a one-GPU box): two NCCL processes, parallelize_wan with its default attention,
  real peer stores; every rank's output matches the emulated run at P = 2 within the same tolerance.
"""
import copy
import os
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))

from test_ulysses_emulated_gpu import BARRIER_TIMEOUT_S, _run_ranks  # noqa: E402
from test_wan_blocks_gpu import _compare, _reinit  # noqa: E402
from test_wan_sp_cpu import _steps, _teacache_single  # noqa: E402
from test_wan_sp_gpu import _World  # noqa: E402

DIM, HEADS, LAYERS, TEXT_LEN, TEXT_DIM = 1536, 12, 2, 64, 256


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


def _model(mod, dev):
    from jenga_b200 import gilbert
    torch.manual_seed(0)
    m = mod.WanModel(model_type="t2v", patch_size=(1, 2, 2), text_len=TEXT_LEN, in_dim=16, dim=DIM, ffn_dim=2048,
                     freq_dim=256, text_dim=TEXT_DIM, out_dim=16, num_heads=HEADS, num_layers=LAYERS).to(dev).eval()
    with torch.cuda.device(dev):
        _reinit(m, 3)                   # init_weights zeroes the head: the output would be all zero
    m.enable_teacache = True
    m.curve_sels = []
    for _, _, _, grid, _ in (_steps()[0], _steps()[3]):
        l2h, h2l = gilbert.mapping_tensors(*grid, sliced=True)
        m.curve_sels.append([[l2h, h2l, gilbert.block_neighbor_mapping(*grid, sliced=True)]])
    # jenga_wan.py:1066-1098
    m.cnt, m.num_steps, m.teacache_thresh = 0, 100, 0.5
    m.accumulated_rel_l1_distance_even = m.accumulated_rel_l1_distance_odd = 0
    m.previous_e0_even = m.previous_e0_odd = m.previous_residual_even = m.previous_residual_odd = None
    m.use_ref_steps, m.use_cache, m.stage_start = False, False, False
    m.coefficients, m.ret_steps, m.cutoff_steps = [1.0, 0.0], 2, 98
    m.p_remain_rates = 0.8
    m.set_curve = lambda i: [setattr(m, a, v) for a, v in
                             zip(("linear_to_hilbert", "hilbert_order", "block_neighbor_list"), m.curve_sels[i][0])]
    m.set_curve(0)
    return m


def _inputs(grid, dev, seed=7):
    g = torch.Generator(device=dev).manual_seed(seed)
    f, h, w = grid
    x = [torch.randn(16, f, 2 * h, 2 * w, generator=g, device=dev)]
    ctx = [torch.randn(TEXT_LEN - 9, TEXT_DIM, generator=g, device=dev)]
    return x, ctx


def _run(model, fwd, dev):
    outs = []
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for _, drop, t, grid, before in _steps():
            if before is not None:
                before(model)
            x, ctx = _inputs(grid, dev)
            L = grid[0] * grid[1] * grid[2]
            outs.append(fwd(x, torch.tensor([t], device=dev), ctx, L + 3, sa_drop_rate=drop)[0].clone())
    return outs


def _rows(o):
    return o.reshape(1, o.shape[0], -1).transpose(1, 2)          # [16, f, H, W] -> [1, f*H*W, 16]


class _Group:
    def __init__(self, size, rank, shared):
        self.size, self.rank, self.shared = size, rank, shared


def _emulated_all_gather(parts, t, group=None):
    torch.cuda.synchronize()
    group.shared["rows"][group.rank] = t
    group.shared["bar"].wait(timeout=BARRIER_TIMEOUT_S)
    for i, p in enumerate(parts):
        p.copy_(group.shared["rows"][i])
    torch.cuda.synchronize()
    group.shared["bar"].wait(timeout=BARRIER_TIMEOUT_S)


def _emulated_broadcast(t, src=0, group=None):
    torch.cuda.synchronize()
    if group.rank == src:
        group.shared["value"] = t.clone()
    group.shared["bar"].wait(timeout=BARRIER_TIMEOUT_S)
    t.copy_(group.shared["value"])
    torch.cuda.synchronize()
    group.shared["bar"].wait(timeout=BARRIER_TIMEOUT_S)


def _emulated(P, monkeypatch, single_model):
    """the sharded forward on P emulated ranks; returns {rank: [outputs per step]}"""
    from jenga_b200 import ulysses, wan_sp
    dist = ulysses.dist
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    monkeypatch.setattr(dist, "get_world_size", lambda g=None: g.size)
    monkeypatch.setattr(dist, "get_rank", lambda g=None: g.rank)
    monkeypatch.setattr(dist, "get_global_rank", lambda g, r: r)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "all_gather", _emulated_all_gather)
    monkeypatch.setattr(dist, "broadcast", _emulated_broadcast)
    dev = torch.device("cuda", 0)
    models = [copy.deepcopy(single_model) for _ in range(P)]
    for m in models:
        m.set_curve = (lambda mm: lambda i: [setattr(mm, a, v) for a, v in zip(
            ("linear_to_hilbert", "hilbert_order", "block_neighbor_list"), mm.curve_sels[i][0])])(m)
        m.set_curve(0)
        m.cnt, m.stage_start = 0, False
        m.previous_e0_even = m.previous_e0_odd = m.previous_residual_even = m.previous_residual_odd = None
    worlds = {}
    for _, _, _, grid, _ in _steps():
        L = grid[0] * grid[1] * grid[2]
        worlds.setdefault(L, _World(P, -(-L // P), HEADS))
    shared = {"rows": {}}
    got = {}

    def rank(r, bar):
        shared["bar"] = bar
        group = _Group(P, r, shared)
        world_of = {L: w.fused(bar, P, r, None) for L, w in worlds.items()}

        class _ByLength:
            """one emulated exchange per grid (the emulated buffers have one shape each)"""

            def __call__(self, attn, q, *a, seq_len=None, **k):
                return world_of[seq_len](attn, q, *a, seq_len=seq_len, **k)

        wan_sp.parallelize_wan(models[r], group=group, attention=_ByLength())
        got[r] = _run(models[r], models[r].forward, dev)

    _run_ranks(P, rank)
    return got


def _single_gpu(mod):
    dev = torch.device("cuda", 0)
    model = _model(mod, dev)
    ref_model = copy.deepcopy(model)
    ref_model.set_curve = lambda i: [setattr(ref_model, a, v) for a, v in zip(
        ("linear_to_hilbert", "hilbert_order", "block_neighbor_list"), ref_model.curve_sels[i][0])]
    ref = _run(ref_model, lambda *a, **k: _teacache_single(ref_model, *a, **k), dev)
    return ref, model


@pytest.mark.parametrize("P", [2, 4])
def test_sharded_forward_over_a_wan_model_matches_single_gpu(wan_module, monkeypatch, P):
    from jenga_b200 import blocks
    ref, model = _single_gpu(wan_module)
    before = dict(blocks.STATS)
    got = _emulated(P, monkeypatch, model)
    # per rank: 4 computed steps x 2 blocks, one of them dense
    assert blocks.STATS["wan_self_sp"] == before["wan_self_sp"] + 6 * P
    assert blocks.STATS["wan_self_dense_sp"] == before["wan_self_dense_sp"] + 2 * P
    assert blocks.STATS["fallback"] == before["fallback"]
    for i, (name, *_rest) in enumerate(_steps()):
        for r in range(P):
            assert torch.equal(got[r][i], got[0][i]), (r, name)
        rows = _rows(ref[i])
        _compare(_rows(ref[i]), _rows(got[0][i]), torch.ones(rows.shape[1], dtype=torch.bool, device="cuda"),
                 f"sharded Wan forward P={P}, {name}")


# ------------------------------------------------------------------------------------------------
# two GPUs: the real exchange
# ------------------------------------------------------------------------------------------------
def _two_gpu_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        from oracle import ref_loader as R
        from jenga_b200 import blocks, wan_sp
        mod = R.load_blocks(product=True)[1]
        blocks.remove_gather_hook()
        dev = torch.device("cuda", rank)
        model = _model(mod, dev)
        sp = wan_sp.parallelize_wan(model)
        outs = _run(model, model.forward, dev)
        torch.cuda.synchronize()
        ret[rank] = dict(outs=[o.cpu() for o in outs], exchange=type(sp).__name__, fallback=blocks.STATS["fallback"])
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_gpus_real_exchange_matches_the_emulated_run(wan_module, monkeypatch):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_two_gpu_worker, args=(world, 29500 + os.getpid() % 2000, ret), nprocs=world, join=True)
    _, model = _single_gpu(wan_module)
    emu = _emulated(world, monkeypatch, model)
    for r in range(world):
        got = ret[r]
        print(f"\n[two GPUs] rank {r}: exchange {got['exchange']}")
        assert got["fallback"] == 0
        for i, (name, *_rest) in enumerate(_steps()):
            real = got["outs"][i].to("cuda")
            rows = _rows(real)
            _compare(_rows(emu[0][i]), rows, torch.ones(rows.shape[1], dtype=torch.bool, device="cuda"),
                     f"two GPUs rank {r} vs emulated, {name}")
