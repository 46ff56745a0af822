"""Sequence-parallel Wan2.1 T2V (jenga_b200/wan_sp.py) without a GPU.

* The sharded forward at world sizes 2 and 4 (gloo), on a small model whose embeddings, blocks and head
  are elementwise stand-ins and whose self-attention is the oracle operator (or the oracle dense
  attention) through UlyssesCarvedAttention with seq_len / dense / first_frame_blocks.  Ragged grids
  (P * n > L), so the last rank holds zero pad rows.  The gathered, inverse-scattered output equals a
  single-process restatement of jenga_wan.py's teacache_forward bit for bit on a dense warm-up step, a
  carved step, a TeaCache-skipped step and a carved step after the turbo curve / grid swap; every rank's
  block input is its slice of the single-process Hilbert-ordered rows.
* The TeaCache agreement: rank-dependent rel-L1 values still give every rank rank 0's decision.
* The errors: no process group, heads % P, P > 8, a rank without a real row, batch > 1, an unpatched
  self-attention.
* install(wan_sp=True): wan.distributed.xdit_context_parallel's usp_dit_forward / usp_attn_forward are
  swapped only with the switch on, a model without the Jenga curve attributes gets the reference
  functions, and turning the switch off puts them back.
"""
import datetime
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(ROOT))

GRID = (21, 9, 14)                 # L = 2646: 21 blocks (first_frame_blocks 1), ragged over 4 ranks
GRID_TURBO = (21, 7, 10)           # L = 1470 after the turbo swap (12 blocks), ragged over 4 ranks
HEADS, D = 8, 128                  # two heads per rank at P = 4 (see test_i2v_sp_cpu.py)
C = HEADS * D
C_IN, OUT, TEXT_LEN = 4, 4, 16
P_REMAIN = 0.3


def sinusoidal_embedding_1d(dim, position):
    """stands in for model_mul.py's (the sharded forward calls the model module's own)"""
    return torch.sin(position.float()[:, None] * (torch.arange(dim) + 1) * 1e-3)


def _vec(seed, n=C, s=0.5):
    g = torch.Generator().manual_seed(seed)
    return 1.0 + s * torch.randn(n, generator=g)


def _oracle_attn(q, k, v, **kw):
    from oracle import attention_oracle as orc
    return orc.block_sparse_attention(q, k, v, variant="wan", **kw)


def _oracle_dense(q, k, v):
    from oracle import attention_oracle as orc
    t = lambda x: x.transpose(1, 2)   # noqa: E731
    return t(orc.dense_attention_rows(t(q), t(k), t(v), q.shape[-1] ** -0.5))


class _SelfAttn(torch.nn.Module):
    """Stand-in WanSelfAttention: elementwise q / k / v, a position table indexed by freq_remap in place
    of RoPE, the attention through jenga_sp or, without it, the oracle over all rows; the block counts
    and the dense rule of model_mul.py:153-164.  Records its calls."""

    def __init__(self, seed, log):
        super().__init__()
        self.w = [_vec(seed + i) for i in range(4)]
        self.log = log

    def forward(self, x, seq_lens, grid_sizes, freqs, sa_drop_rate=0.0, per_block_tokens=128, p_remain_rates=0.8,
                freq_remap=None, block_neighbor_list=None):
        from jenga_b200.wan import block_counts
        f, h, w = grid_sizes[0].tolist()
        L = f * h * w
        self.log.append(dict(x=x.clone(), remap=freq_remap.clone(), drop=sa_drop_rate))
        pos = freqs[freq_remap]
        n = x.shape[1]
        q, k, v = ((x * self.w[0] + pos), (x * self.w[1] - pos), x * self.w[2])
        q, k, v = (t.view(1, n, HEADS, D).bfloat16() for t in (q, k, v))
        dense = sa_drop_rate <= 0.25
        top_k, ff = (0, 0) if dense else block_counts(L, sa_drop_rate)
        sp = getattr(self, "jenga_sp", None)
        if sp is not None:
            out = sp(None, q, k, v, top_k=top_k, block_neighbor_list=None if dense else block_neighbor_list,
                     p_remain_rates=p_remain_rates, first_frame_blocks=ff, dense=dense, seq_len=L)
        elif dense:
            out = _oracle_dense(q, k, v)
        else:
            out = _oracle_attn(q, k, v, top_k=top_k, text_blocks=0, block_neighbor_list=block_neighbor_list,
                               p_remain_rates=p_remain_rates, first_frame_blocks=ff, shape_xfuse=True)
        return out.flatten(2).float() * self.w[3]

    # the stand-in routes jenga_sp itself, as the fused WanSelfAttention forward of blocks.py does
    forward.__jenga_b200__ = True


class _Block(torch.nn.Module):
    def __init__(self, seed, log):
        super().__init__()
        self.self_attn = _SelfAttn(seed, log)
        self.w = _vec(seed + 9)

    def forward(self, x, e, seq_lens, grid_sizes, freqs, context, context_lens, sa_drop_rate=0.0, freq_remap=None,
                block_neighbor_list=None, p_remain_rates=0.0):
        y = self.self_attn(x * (1 + e[:, 1]) + e[:, 0], seq_lens, grid_sizes, freqs, sa_drop_rate=sa_drop_rate,
                           freq_remap=freq_remap, block_neighbor_list=block_neighbor_list,
                           p_remain_rates=p_remain_rates)
        return x + y * e[:, 2] * self.w + context.mean(1)


class _Scale(torch.nn.Module):
    def __init__(self, seed, n=C):
        super().__init__()
        self.weight = torch.nn.Parameter(_vec(seed, n), requires_grad=False)

    def forward(self, x):
        return x * self.weight


class _PatchEmbed(_Scale):
    def forward(self, x):                                  # [1, C_in, f, h, w] -> [1, C, f, h, w]
        return x.repeat(1, C // C_IN, 1, 1, 1) * self.weight[None, :, None, None, None]


class _Proj(_Scale):
    def forward(self, e):                                  # [1, C] -> [1, 6C]
        return e.repeat(1, 6) * self.weight


class _Head(_Scale):
    def forward(self, x, e):                               # row-local, as Head is
        return x[..., :OUT] * self.weight[:OUT] + e[:, None, :OUT]


class _Model(torch.nn.Module):
    """The attributes and sub-modules teacache_forward reads (patch size 1)."""
    model_type = "t2v"
    patch_size = (1, 1, 1)
    enable_teacache = True

    def __init__(self, log, n_blocks=2):
        super().__init__()
        from jenga_b200 import gilbert
        self.dim, self.freq_dim, self.text_len, self.num_heads, self.out_dim = C, C, TEXT_LEN, HEADS, OUT
        self.patch_embedding = _PatchEmbed(1)
        self.time_embedding = _Scale(2)
        self.time_projection = _Proj(3, 6 * C)
        self.text_embedding = _Scale(4)
        self.head = _Head(5)
        self.blocks = torch.nn.ModuleList([_Block(10 + 10 * i, log) for i in range(n_blocks)])
        self.freqs = torch.randn(4096, C, generator=torch.Generator().manual_seed(6))
        self.curve_sels = []
        for grid in (GRID, GRID_TURBO):
            l2h, h2l = gilbert.mapping_tensors(*grid)
            self.curve_sels.append([[l2h, h2l, gilbert.block_neighbor_mapping(*grid)]])
        self.reset()

    def reset(self):
        """the per-prompt reset of jenga_wan.py:1066-1098 (set on the instance here)"""
        self.cnt, self.num_steps, self.teacache_thresh = 0, 100, 0.5
        self.accumulated_rel_l1_distance_even = self.accumulated_rel_l1_distance_odd = 0
        self.previous_e0_even = self.previous_e0_odd = None
        self.previous_residual_even = self.previous_residual_odd = None
        self.use_ref_steps, self.use_cache = False, False
        self.coefficients, self.ret_steps, self.cutoff_steps = [1.0, 0.0], 2, 98
        self.stage_start = False
        self.set_curve(0)
        self.p_remain_rates = P_REMAIN

    def set_curve(self, i):
        self.linear_to_hilbert, self.hilbert_order, self.block_neighbor_list = self.curve_sels[i][0]

    def unpatchify(self, x, grid_sizes):
        return [u[:f * h * w].view(f, h, w, OUT).permute(3, 0, 1, 2) for u, (f, h, w) in zip(x, grid_sizes.tolist())]


def _teacache_single(self, x, t, context, seq_len, sa_drop_rate=0.0):
    """jenga_wan.py:503-664 (teacache_forward) in one process, batch 1, t2v; the model module's own
    sinusoidal_embedding_1d"""
    import numpy as np
    device = self.patch_embedding.weight.device
    if self.freqs.device != device:
        self.freqs = self.freqs.to(device)
    x = [self.patch_embedding(u.unsqueeze(0)) for u in x]
    grid_sizes = torch.stack([torch.tensor(u.shape[2:], dtype=torch.long) for u in x])
    x = [u.flatten(2).transpose(1, 2) for u in x]
    seq_lens = torch.tensor([u.size(1) for u in x], dtype=torch.long)
    x = torch.cat([torch.cat([u, u.new_zeros(1, seq_len - u.size(1), u.size(2))], dim=1) for u in x])
    x = x[:, self.hilbert_order]
    with torch.autocast("cuda", dtype=torch.float32, enabled=x.is_cuda):
        e = self.time_embedding(type(self).unpatchify.__globals__["sinusoidal_embedding_1d"](self.freq_dim, t).float())
        e0 = self.time_projection(e).unflatten(1, (6, self.dim))
    context = self.text_embedding(torch.stack([torch.cat([u, u.new_zeros(self.text_len - u.size(0), u.size(1))])
                                               for u in context]))
    kwargs = dict(e=e0, seq_lens=seq_lens, grid_sizes=grid_sizes, freqs=self.freqs, context=context,
                  context_lens=None, sa_drop_rate=sa_drop_rate, freq_remap=self.hilbert_order,
                  block_neighbor_list=self.block_neighbor_list, p_remain_rates=self.p_remain_rates)
    modulated_inp = e0 if self.use_ref_steps else e
    if self.cnt % 2 == 0:
        self.is_even = True
        if self.cnt < self.ret_steps or self.cnt >= self.cutoff_steps or self.stage_start:
            should_calc_even = True
            self.accumulated_rel_l1_distance_even = 0
        else:
            rescale_func = np.poly1d(self.coefficients)
            self.accumulated_rel_l1_distance_even += rescale_func(((modulated_inp - self.previous_e0_even).abs().mean()
                                                                   / self.previous_e0_even.abs().mean()).cpu().item())
            if self.accumulated_rel_l1_distance_even < self.teacache_thresh:
                should_calc_even = False
            else:
                should_calc_even = True
                self.accumulated_rel_l1_distance_even = 0
        self.previous_e0_even = modulated_inp.clone()
    else:
        self.is_even = False
        if self.cnt < self.ret_steps or self.cnt >= self.cutoff_steps or self.stage_start:
            should_calc_odd = True
            self.accumulated_rel_l1_distance_odd = 0
        else:
            rescale_func = np.poly1d(self.coefficients)
            self.accumulated_rel_l1_distance_odd += rescale_func(((modulated_inp - self.previous_e0_odd).abs().mean()
                                                                  / self.previous_e0_odd.abs().mean()).cpu().item())
            if self.accumulated_rel_l1_distance_odd < self.teacache_thresh:
                should_calc_odd = False
            else:
                should_calc_odd = True
                self.accumulated_rel_l1_distance_odd = 0
        self.previous_e0_odd = modulated_inp.clone()
    calc = should_calc_even if self.is_even else should_calc_odd
    sfx = "even" if self.is_even else "odd"
    if not calc:
        x += getattr(self, "previous_residual_" + sfx)
        self.use_cache = True
    else:
        ori_x = x.clone()
        for block in self.blocks:
            x = block(x, **kwargs)
        setattr(self, "previous_residual_" + sfx, x - ori_x)
        self.use_cache = False
    x = x[:, self.linear_to_hilbert]
    x = self.head(x, e)
    x = self.unpatchify(x, grid_sizes)
    self.cnt += 1
    if self.cnt >= self.num_steps:
        self.cnt = 0
    return [u.float() for u in x]


def _inputs(grid, seed=7):
    g = torch.Generator().manual_seed(seed)
    x = [torch.randn(C_IN, *grid, generator=g)]
    ctx = [torch.randn(TEXT_LEN - 3, C, generator=g)]
    return x, ctx


# the four step kinds: (name, sa_drop_rate, t, grid, before the call); cnt runs 0..4
def _steps():
    def turbo(m):
        m.set_curve(1)      # jenga_wan.py:241-245: curve and grid swapped, and both calls of the next step computed
        m.stage_start = True

    return [("dense warm-up", 0.2, 900.0, GRID, None),
            ("carved", 0.7, 900.0, GRID, None),
            ("teacache skip", 0.7, 900.0, GRID, None),       # even step 2: rel-L1 0, reuses step 0's residual
            ("turbo swap, uncond", 0.7, 860.0, GRID_TURBO, turbo),
            ("turbo swap, cond", 0.7, 860.0, GRID_TURBO, None)]


def _run(model, fwd):
    outs = []
    for name, drop, t, grid, before in _steps():
        if before is not None:
            before(model)
        x, ctx = _inputs(grid)
        L = grid[0] * grid[1] * grid[2]
        outs.append((fwd(x, torch.tensor([t]), ctx, L + 5, sa_drop_rate=drop)[0], model.use_cache))
    return outs


def _init(rank, world, port):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))


def _worker(rank, world, port, ret):
    _init(rank, world, port)
    try:
        from jenga_b200 import wan_sp
        from jenga_b200.ulysses import UlyssesCarvedAttention
        log = []
        model = _Model(log)
        sp = UlyssesCarvedAttention(attn_fn=_oracle_attn, dense_fn=_oracle_dense, variant="wan")
        assert wan_sp.parallelize_wan(model, attention=sp) is sp
        assert all(b.self_attn.jenga_sp is sp for b in model.blocks)
        with torch.no_grad():
            outs = _run(model, model.forward)
        ret[rank] = dict(outs=outs, log=log)
        # the errors every rank raises before any collective
        with pytest.raises(ValueError, match="runs batch 1, got 2 videos"):
            model.forward(_inputs(GRID)[0] * 2, torch.tensor([1.0]), _inputs(GRID)[1], 3000)
        if world == 4:
            tiny = _Model([])
            tiny.hilbert_order = tiny.linear_to_hilbert = torch.arange(5)
            wan_sp.parallelize_wan(tiny, attention=sp)
            with pytest.raises(ValueError, match="5 tokens over 4 ranks leave the last rank without a real row"):
                tiny.forward([torch.randn(C_IN, 1, 1, 5)], torch.tensor([1.0]), _inputs(GRID)[1], 8)
        if world == 2:
            odd = _Model([])
            odd.num_heads = 3
            with pytest.raises(ValueError, match="sequence-parallel Wan2.1: 3 attention heads do not split over 2"):
                wan_sp.parallelize_wan(odd, attention=sp)
            plain = _Model([])
            plain.blocks[1].self_attn = torch.nn.Linear(2, 2)
            with pytest.raises(RuntimeError, match="Linear.forward is not the fused jenga_b200 forward"):
                wan_sp.parallelize_wan(plain, attention=sp)
            assert not hasattr(plain.blocks[0].self_attn, "jenga_sp") and "forward" not in plain.__dict__
            bound = _Model([])
            bound.blocks[0].self_attn.forward = lambda *a: None      # what WanT2V(use_usp=True) binds
            with pytest.raises(RuntimeError, match="instance forward"):
                wan_sp.parallelize_wan(bound, attention=sp)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_forward_equals_single_process(world):
    mgr = mp.Manager()
    ret = mgr.dict()
    port = 29500 + (os.getpid() + 41 * world) % 2000
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)

    log = []
    model = _Model(log)
    with torch.no_grad():
        ref = _run(model, lambda *a, **k: _teacache_single(model, *a, **k))
    assert [u for _, u in ref] == [False, False, True, False, False], "the steps are not the four kinds"
    assert model.block_neighbor_list is model.curve_sels[1][0][2]
    per_step_calls = [2, 2, 0, 2, 2]           # self-attention calls per step (two blocks)
    for r in range(world):
        got = ret[r]
        for i, ((o, used), (o_ref, used_ref)) in enumerate(zip(got["outs"], ref)):
            assert used == used_ref, (r, i)
            assert torch.equal(o, o_ref), (r, _steps()[i][0])
        assert len(got["log"]) == len(log) == sum(per_step_calls)
        j = 0
        for i, (_, _, _, grid, _) in enumerate(_steps()):
            L = grid[0] * grid[1] * grid[2]
            n = -(-L // world)
            lo, hi = min(r * n, L), min((r + 1) * n, L)
            for _ in range(per_step_calls[i]):
                g, e = got["log"][j], log[j]
                assert g["x"].shape[1] == n and g["drop"] == e["drop"]
                assert torch.equal(g["x"][:, :hi - lo], e["x"][:, lo:hi]), (r, i)
                assert torch.equal(g["remap"][:hi - lo], e["remap"][lo:hi]), (r, i)
                j += 1
    # the grids really are ragged over four ranks
    assert (21 * 9 * 14) % 4 and (21 * 7 * 10) % 4


def _agree_worker(rank, world, port, ret):
    _init(rank, world, port)
    try:
        from jenga_b200 import wan_sp

        class _Local:
            """attends nothing and exchanges nothing: a rank that took the other branch shows up as a
            different use_cache, not as a wait"""

            def __call__(self, attn, q, *a, **k):
                return torch.zeros_like(q)

        model = _Model([])
        wan_sp.parallelize_wan(model, attention=_Local())
        x, ctx = _inputs(GRID)
        with torch.no_grad():
            model.forward(x, torch.tensor([900.0]), ctx, 3000, sa_drop_rate=0.7)       # cnt 0: computed
            model.forward(x, torch.tensor([900.0]), ctx, 3000, sa_drop_rate=0.7)       # cnt 1: computed
            # rank 0's rel-L1 at cnt 2 is 0.1 (below the threshold 0.5: skip); the others see 1.0
            model.previous_e0_even = model.previous_e0_even / (1.1 if rank == 0 else 2.0)
            model.forward(x, torch.tensor([900.0]), ctx, 3000, sa_drop_rate=0.7)
        ret[rank] = dict(use_cache=model.use_cache, acc=model.accumulated_rel_l1_distance_even)
    finally:
        dist.destroy_process_group()


def test_ranks_take_rank_zeros_teacache_decision():
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_agree_worker, args=(world, 29500 + (os.getpid() + 7) % 2000, ret), nprocs=world, join=True)
    assert ret[0]["use_cache"] and ret[1]["use_cache"]
    assert ret[0]["acc"] == ret[1]["acc"] and abs(ret[0]["acc"] - 0.1) < 1e-6


def test_errors_outside_a_process_group():
    from jenga_b200 import wan_sp
    assert not dist.is_initialized()
    with pytest.raises(RuntimeError, match="needs an initialised process group"):
        wan_sp.parallelize_wan(_Model([]))
    with pytest.raises(ValueError, match="9 ranks; the Ulysses exchange is built for at most 8"):
        wan_sp._check_world(72, 9)
    with pytest.raises(ValueError, match="40 attention heads do not split over 3 ranks"):
        wan_sp._check_world(40, 3)
    for P in (1, 2, 4, 5, 8):
        wan_sp._check_world(40, P)


@pytest.mark.parametrize("L,P", [(75600, 8), (41580, 8), (2646, 4), (1470, 4), (7, 4), (9, 3)])
def test_shard_layout(L, P):
    """rows [r*n, min((r+1)*n, L)) with n = ceil(L/P), zero-padded to n; together they are 0..L-1"""
    from jenga_b200 import hyi2v_sp, wan_sp
    order = torch.randperm(L, generator=torch.Generator().manual_seed(L)) + 1
    n = -(-L // P)
    parts = []
    for r in range(P):
        got_n, real = wan_sp.shard_rows(L, P, r)
        s = hyi2v_sp.shard(order, 0, P, r)
        assert got_n == n and s.shape == (n,) and real == max(0, min(n, L - r * n))
        assert bool((s[real:] == 0).all())
        parts.append(s[:real])
    assert torch.equal(torch.cat(parts), order)


@pytest.mark.parametrize("L,P", [(5, 4), (6, 4), (1, 2)])
def test_a_rank_without_a_real_row_is_refused(L, P):
    from jenga_b200 import wan_sp
    with pytest.raises(ValueError, match="leave the last rank without a real row"):
        wan_sp.shard_rows(L, P, 0)


# ------------------------------------------------------------------------------------------------
# install(): the switch
# ------------------------------------------------------------------------------------------------
_STUB = '''
def usp_dit_forward(self, x, t, context, seq_len, clip_fea=None, y=None):
    return "reference usp_dit_forward"


def usp_attn_forward(self, x, seq_lens, grid_sizes, freqs, dtype=None):
    return "reference usp_attn_forward"
'''

_PROBE = '''
import os, sys, types, json
import torch
import torch.distributed as dist
sys.path.insert(0, {root!r})
sys.path.insert(0, {stub!r})
from jenga_b200 import install
done = install.install(flash_attn=False, gilbert=False, ulysses=False, gather=False, **{kw})
import wan.distributed.xdit_context_parallel as xdit
if {then_off!r}:
    install.install(flash_attn=False, gilbert=False, ulysses=False, gather=False, wan_sp=False)
    done = []
from jenga_b200 import blocks as jb, wan_sp
# the sharded forward itself is tested elsewhere: here it reports that it was reached
wan_sp._forward_factory = lambda group: (lambda self, *a, **k: ["sharded forward", k.get("sa_drop_rate")])
os.environ["MASTER_ADDR"] = "127.0.0.1"
os.environ["MASTER_PORT"] = {port!r}
dist.init_process_group("gloo", rank=0, world_size=1)
class SelfAttn(torch.nn.Module):   # stands in for the WanSelfAttention class the fused-forward hook patched
    def forward(self, *a, **k):
        return ["patched class forward", k.get("sa_drop_rate")]
    forward.__jenga_b200__ = True
def model(jenga):
    m = torch.nn.Module()
    m.num_heads = 40
    m.blocks = torch.nn.ModuleList([torch.nn.Module()])
    m.blocks[0].self_attn = SelfAttn()
    if jenga:
        m.hilbert_order = m.linear_to_hilbert = torch.arange(4)
    # what WanT2V(use_usp=True) does (text2video.py:88-99)
    for b in m.blocks:
        b.self_attn.forward = types.MethodType(xdit.usp_attn_forward, b.self_attn)
    m.forward = types.MethodType(xdit.usp_dit_forward, m)
    return m
res = {{}}
for jenga in (True, False):
    m = model(jenga)
    sa = m.blocks[0].self_attn
    if jenga:
        # t2v_generate passes sa_drop_rate (jenga_wan.py:210-213); the reference usp_dit_forward has no such
        # parameter
        try:
            first = m(None, None, None, 4, sa_drop_rate=0.7)
            second = m(None, None, None, 4, sa_drop_rate=0.2)
        except TypeError as e:
            first = second = "TypeError" if "sa_drop_rate" in str(e) else str(e)
    else:
        first = second = m(None, None, None, 4)
    res["jenga" if jenga else "plain"] = dict(
        first=first, second=second,
        attn=sa(None, None, None, None, **({{"sa_drop_rate": 0.7}} if hasattr(sa, "jenga_sp") else {{}})),
        jenga_sp=type(getattr(sa, "jenga_sp", None)).__name__,
        variant=getattr(getattr(sa, "jenga_sp", None), "variant", None))
print(json.dumps(dict(res=res, swapped=bool(getattr(xdit.usp_dit_forward, "__jenga_b200__", False)),
                      attn_swapped=bool(getattr(xdit.usp_attn_forward, "__jenga_b200__", False)),
                      route="sequence-parallel Wan route" in done, flag=jb.WAN_SP)))
dist.destroy_process_group()
'''


def _probe(tmp_path, kw, env_switch, then_off=False):
    import json
    stub = tmp_path / "stub"
    (stub / "wan" / "distributed").mkdir(parents=True)
    (stub / "wan" / "__init__.py").write_text("")
    (stub / "wan" / "distributed" / "__init__.py").write_text("")
    (stub / "wan" / "distributed" / "xdit_context_parallel.py").write_text(_STUB)
    env = {k: v for k, v in os.environ.items() if k != "JENGA_WAN_SP"}
    if env_switch is not None:
        env["JENGA_WAN_SP"] = env_switch
    code = _PROBE.format(root=str(ROOT), stub=str(stub), kw=repr(kw), port=str(33000 + os.getpid() % 2000),
                         then_off=then_off)
    r = subprocess.run([sys.executable, "-s", "-c", code], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


_REFERENCE = dict(first="reference usp_dit_forward", second="reference usp_dit_forward",
                  attn="reference usp_attn_forward", jenga_sp="NoneType", variant=None)
# the reference route under jenga_wan.py: its call with sa_drop_rate fails
_REFERENCE_JENGA = dict(_REFERENCE, first="TypeError", second="TypeError")


@pytest.mark.parametrize("kw,env_switch", [({}, None), ({}, "0"), ({"wan_sp": False}, "1")])
def test_without_the_switch_the_reference_functions_stay(tmp_path, kw, env_switch):
    got = _probe(tmp_path, kw, env_switch)
    assert not got["swapped"] and not got["attn_swapped"] and not got["route"] and not got["flag"]
    assert got["res"]["jenga"] == _REFERENCE_JENGA and got["res"]["plain"] == _REFERENCE


@pytest.mark.parametrize("kw,env_switch", [({}, "1"), ({"wan_sp": True}, None)])
def test_with_the_switch_usp_forwards_run_the_sharded_route(tmp_path, kw, env_switch):
    got = _probe(tmp_path, kw, env_switch)
    assert got["swapped"] and got["attn_swapped"] and got["route"] and got["flag"]
    jenga = got["res"]["jenga"]
    assert jenga["first"] == ["sharded forward", 0.7] and jenga["second"] == ["sharded forward", 0.2]
    assert jenga["attn"] == ["patched class forward", 0.7]
    # gloo has no symmetric memory: the all-ranks agreement picks the NCCL-style exchange
    assert jenga["jenga_sp"] == "UlyssesCarvedAttention" and jenga["variant"] == "wan"
    # a model without the Jenga curve attributes (WanI2V) runs the reference functions
    assert got["res"]["plain"] == _REFERENCE


def test_install_without_the_switch_turns_the_route_back_off(tmp_path):
    got = _probe(tmp_path, {"wan_sp": True}, None, then_off=True)
    assert not got["swapped"] and not got["attn_swapped"] and got["flag"] is False
    assert got["res"]["jenga"] == _REFERENCE_JENGA and got["res"]["plain"] == _REFERENCE


def test_wan_sp_needs_the_fused_blocks():
    from jenga_b200 import install
    with pytest.raises(ValueError, match="fused_blocks"):
        install.install(flash_attn=False, gilbert=False, ulysses=False, fused_blocks=False, gather=False,
                        wan_sp=True)
