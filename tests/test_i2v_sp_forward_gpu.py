"""parallelize_i2v's sharded forward over the real, patched HunyuanVideo-I2V blocks.

A two-block stack — one unmodified hyvideo_i2v/modules/models_mul.py MMDoubleStreamBlock and one
MMSingleStreamBlock at the HunyuanVideo width, patched by install() — inside a transformer whose
embedders and final layer are elementwise stand-ins.  The forward under test is the one
parallelize_i2v installs: Hilbert gather, each rank's slice of image rows, RoPE rows and first-frame
masks (a device mask into the double block, the CPU mask of n_loc + 400 rows into the single block),
the fused I2V forwards under jenga_sp, the image-row all-gather and the inverse scatter.  The reference
is a single-GPU restatement of jenga_hyi2v.py's ra_forward over the same blocks without jenga_sp
(tests/test_i2v_sp_cpu.py), i.e. the single-GPU fused forward.

* Emulated ranks (every GPU box): UlyssesFusedAttention on one device, one thread per rank, the
  process-group calls parallelize_i2v makes (rank, size, all_gather) answered by the threads.  Every
  rank's output equals the others' bit for bit and the single-GPU forward within the drop-in tolerance
  of tests/test_dropin_blocks_gpu.py, on a computed step and on a skipped step.
* Two GPUs (skipped on a one-GPU box): two NCCL processes, parallelize_i2v with its default attention
  (the all-ranks symmetric-memory agreement), real peer stores and barriers; every rank's output
  matches the emulated run at P = 2 within the same tolerance.
"""
import copy
import os
import sys
import threading
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))

from test_dropin_blocks_gpu import _compare, _reinit  # noqa: E402
from test_i2v_sp_cpu import _ra_forward_single  # noqa: E402
from test_ulysses_emulated_gpu import BARRIER_TIMEOUT_S, H, World, _emulated_fused, _run_ranks  # noqa: E402

D = 128
C = H * D
GRID = (8, 16, 16)                 # L = 2048 image tokens
T, VALID = 400, 300
DROP, P_REMAIN = 0.7, 0.3


class _Elementwise(torch.nn.Module):
    def __init__(self, seed, dev):
        super().__init__()
        g = torch.Generator(device=dev).manual_seed(seed)
        self.w = (1.0 + 0.3 * torch.randn(C, generator=g, device=dev)).bfloat16()

    def forward(self, x, *a):
        if x.dim() == 5:                      # the latent [1, C, t, h, w] -> tokens (patch size 1)
            x = x.flatten(2).transpose(1, 2)
        return x * self.w


class _Final(_Elementwise):
    def forward(self, x, vec):
        return x * self.w + vec[:, None]


class _Stack(torch.nn.Module):
    """The attributes and sub-modules ra_forward reads; the blocks are the real patched ones."""
    patch_size = (1, 1, 1)
    i2v_condition_type = "token_replace"
    guidance_embed = False
    text_projection = "linear"
    heads_num = H

    def __init__(self, mod, dev):
        super().__init__()
        from jenga_b200 import gilbert
        self.img_in, self.txt_in, self.vector_in = (_Elementwise(s, dev) for s in (1, 2, 3))
        self.final_layer = _Final(4, dev)
        self.t_w = _Elementwise(5, dev).w
        kw = dict(mlp_width_ratio=4.0, dtype=torch.bfloat16, device=dev)
        self.double_blocks = torch.nn.ModuleList([mod.MMDoubleStreamBlock(C, H, **kw)])
        self.single_blocks = torch.nn.ModuleList([mod.MMSingleStreamBlock(C, H, **kw)])
        with torch.cuda.device(dev):
            _reinit(self.double_blocks[0], 11)
            _reinit(self.single_blocks[0], 12)
        t, h, w = GRID
        l2h, h2l = gilbert.mapping_tensors(t, h, w)          # CPU, as jenga_hyi2v.py builds them
        self.curve_sel = [[l2h, h2l, gilbert.block_neighbor_mapping(t, h, w).to(dev)]]
        self.linear_to_hilbert, self.hilbert_order = l2h, h2l
        self.sa_drop_rate, self.p_remain_rates, self.text_amp = DROP, P_REMAIN, 0.0
        self.cnt, self.num_steps, self.start_stage, self.previous_residual = 0, 50, True, None

    def time_in(self, t):
        return (t[:, None] * 1e-3 * self.t_w).bfloat16()

    def unpatchify(self, x, tt, th, tw):
        return x.transpose(1, 2).reshape(1, C, tt, th, tw)


def _inputs(dev):
    g = torch.Generator(device=dev).manual_seed(7)
    t, h, w = GRID
    x = torch.randn(1, C, t, h, w, generator=g, device=dev).bfloat16()
    txt = torch.randn(1, T, C, generator=g, device=dev).bfloat16()
    mask = torch.zeros(1, T, dtype=torch.int64, device=dev)
    mask[:, :VALID] = 1
    txt2 = torch.randn(1, C, generator=g, device=dev).bfloat16()
    ang = torch.rand(t * h * w, D // 2, generator=g, device=dev) * 6.2831853
    cos = torch.cos(ang).repeat_interleave(2, 1).contiguous()
    sin = torch.sin(ang).repeat_interleave(2, 1).contiguous()
    return x, torch.tensor([900.0], device=dev), txt, mask, txt2, cos, sin


def _two_steps(fwd, model, args):
    """a computed step, then a skipped one (step 4 is not in jenga_hyi2v.py's step_calc)"""
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        a = fwd(*args)
        model.cnt = 4
        b = fwd(*args)
    return [o if isinstance(o, torch.Tensor) else o["x"] for o in (a, b)]


def _rows(o):
    return o.flatten(2).transpose(1, 2)                      # [1, C, t, h, w] -> [1, L, C]


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


def _single_gpu(mod):
    dev = torch.device("cuda", 0)
    model = _Stack(mod, dev)
    args = _inputs(dev)
    return _two_steps(lambda *a: _ra_forward_single(model, *a), model, args), model


class _Group:
    """The process group of one emulated rank; all_gather is answered through `shared`."""

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


def _emulated(mod, P, monkeypatch, single_model):
    """parallelize_i2v's forward on P emulated ranks; returns {rank: [computed, skipped]}"""
    from jenga_b200 import hyi2v_sp, ulysses
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    monkeypatch.setattr(ulysses.dist, "get_world_size", lambda g=None: g.size)
    monkeypatch.setattr(ulysses.dist, "get_rank", lambda g=None: g.rank)
    monkeypatch.setattr(ulysses.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(ulysses.dist, "all_gather", _emulated_all_gather)
    dev = torch.device("cuda", 0)
    L = GRID[0] * GRID[1] * GRID[2]
    world = World(P, L // P, T, torch.bfloat16, n_out=2)
    models = [copy.deepcopy(single_model) for _ in range(P)]
    for m in models:
        m.cnt, m.start_stage, m.previous_residual = 0, True, None
    args = _inputs(dev)
    shared = {"rows": {}}
    got = {}

    def rank(r, bar):
        shared["bar"] = bar
        group = _Group(P, r, shared)
        sp = _emulated_fused(world, bar)(group=group, variant="hyvideo_i2v")
        assert hyi2v_sp.parallelize_i2v(models[r], group=group, attention=sp) is sp
        got[r] = [o.clone() for o in _two_steps(models[r], models[r], args)]

    _run_ranks(P, rank)
    return got


@pytest.mark.parametrize("P", [2, 4])
def test_sharded_forward_over_patched_blocks_matches_single_gpu(i2v_module, monkeypatch, P):
    from jenga_b200 import blocks
    ref, single_model = _single_gpu(i2v_module)
    before = dict(blocks.STATS)
    got = _emulated(i2v_module, P, monkeypatch, single_model)
    assert blocks.STATS["i2v_double_sp"] == before["i2v_double_sp"] + P      # one computed step per rank
    assert blocks.STATS["i2v_single_sp"] == before["i2v_single_sp"] + P
    assert blocks.STATS["fallback"] == before["fallback"]
    assert blocks.STATS["i2v_double"] == before["i2v_double"]
    L = GRID[0] * GRID[1] * GRID[2]
    every_row = torch.ones(L, dtype=torch.bool, device="cuda")
    for step, what in enumerate(("computed step", "skipped step")):
        for r in range(P):
            assert torch.equal(got[r][step], got[0][step]), (r, what)          # replicated after the gather
        _compare(_rows(ref[step]), _rows(got[0][step]), every_row, f"sharded I2V forward P={P}, {what}")


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
        from i2v_ref import load_i2v_blocks
        from jenga_b200 import blocks, hyi2v_sp
        mod = load_i2v_blocks(product=True)
        blocks.remove_gather_hook()
        dev = torch.device("cuda", rank)
        model = _Stack(mod, dev)
        sp = hyi2v_sp.parallelize_i2v(model)
        outs = _two_steps(model, model, _inputs(dev))
        torch.cuda.synchronize()
        ret[rank] = dict(outs=[o.cpu() for o in outs], exchange=type(sp).__name__,
                         sp_calls=blocks.STATS["i2v_double_sp"] + blocks.STATS["i2v_single_sp"],
                         fallback=blocks.STATS["fallback"])
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_gpus_real_exchange_matches_the_emulated_run(i2v_module, monkeypatch):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_two_gpu_worker, args=(world, 29500 + os.getpid() % 2000, ret), nprocs=world, join=True)
    _, single_model = _single_gpu(i2v_module)
    emu = _emulated(i2v_module, world, monkeypatch, single_model)
    L = GRID[0] * GRID[1] * GRID[2]
    every_row = torch.ones(L, dtype=torch.bool, device="cuda")
    for r in range(world):
        got = ret[r]
        print(f"\n[two GPUs] rank {r}: exchange {got['exchange']}")
        assert got["sp_calls"] == 2 and got["fallback"] == 0
        for step, what in enumerate(("computed step", "skipped step")):
            real = got["outs"][step].to("cuda")
            print(f"[two GPUs] rank {r} {what}: bit-identical to the emulated run: "
                  f"{torch.equal(real, emu[0][step])}")
            _compare(_rows(emu[0][step]), _rows(real), every_row, f"two GPUs rank {r} vs emulated, {what}")
