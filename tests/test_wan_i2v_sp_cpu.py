"""Sequence-parallel Wan2.1-I2V (jenga_b200/wan_sp.py, parallelize_wan_i2v) without a GPU.

* The sharded forward at world sizes 2 and 4 (gloo), on a small I2V model whose embeddings, blocks and
  head are elementwise stand-ins and whose self-attention is the oracle dense attention through
  UlyssesCarvedAttention with dense / seq_len.  Ragged grids (P * n > L), so the last rank holds zero
  pad rows.  The gathered output equals a single-process restatement of the I2V TeaCache forward bit
  for bit, on computed steps and on a TeaCache-skipped step; every rank's block input is its raster
  slice of the single-process rows, and its RoPE index that slice with the pad rows at row 0.
* The errors: no process group, heads % P, P > 8, a rank without a real row, batch > 1, no clip_fea / y,
  an unpatched or shadowed self-attention, and (on the unmodified wan/modules/model.py blocks) a
  cross-attention the fused I2V kernel does not take.
* install(wan_sp=True): wan.modules.model is hooked only with the switch on, and turning it off puts the
  original forwards back; usp_dit_forward sends an I2V model to parallelize_wan_i2v, a Jenga T2V model
  to parallelize_wan, and any other model to the reference function.
"""
import datetime
import importlib
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
sys.path.insert(0, str(HERE))

from test_wan_sp_cpu import _Head, _Proj, _Scale, _vec  # noqa: E402

GRIDS = [(21, 9, 14), (3, 7, 11)]    # L = 2646 (ragged over 4) and 231 (ragged over 2 and 4)
HEADS, D = 8, 128
C = HEADS * D
C_IN, OUT, TEXT_LEN, CLIP_TOKENS = 4, 4, 16, 257


def sinusoidal_embedding_1d(dim, position):
    """stands in for model.py's (the sharded forward calls the model module's own)"""
    return torch.sin(position.float()[:, None] * (torch.arange(dim) + 1) * 1e-3)


def _oracle_dense(q, k, v):
    from oracle import attention_oracle as orc
    t = lambda x: x.transpose(1, 2)   # noqa: E731
    return t(orc.dense_attention_rows(t(q), t(k), t(v), q.shape[-1] ** -0.5))


def raster_remap(L, n, rank):
    """the RoPE index of rank `rank`'s n rows: its raster slice, pad rows at row 0"""
    rows = torch.arange(rank * n, (rank + 1) * n)
    return torch.where(rows < L, rows, torch.zeros_like(rows))


class _SelfAttn(torch.nn.Module):
    """Stand-in for the WanSelfAttention of wan/modules/model.py, (x, seq_lens, grid_sizes, freqs):
    elementwise q / k / v, a position table indexed by the row's raster position in place of RoPE, and a
    dense attention through jenga_sp over the first L exchanged rows or, without it, the oracle over all
    rows.  Records its calls."""

    def __init__(self, seed, log):
        super().__init__()
        self.w = [_vec(seed + i) for i in range(4)]
        self.log = log

    def forward(self, x, seq_lens, grid_sizes, freqs):
        f, h, w = grid_sizes[0].tolist()
        L = f * h * w
        sp = getattr(self, "jenga_sp", None)
        n = x.shape[1]
        remap = raster_remap(L, n, dist.get_rank(sp.group)) if sp is not None else torch.arange(L)
        self.log.append(dict(x=x.clone(), remap=remap))
        pos = freqs[remap]
        q, k, v = ((x * self.w[0] + pos), (x * self.w[1] - pos), x * self.w[2])
        q, k, v = (t.view(1, n, HEADS, D).bfloat16() for t in (q, k, v))
        out = sp(None, q, k, v, dense=True, seq_len=L) if sp is not None else _oracle_dense(q, k, v)
        return out.flatten(2).float() * self.w[3]

    forward.__jenga_b200__ = True


class _Block(torch.nn.Module):
    def __init__(self, seed, log):
        super().__init__()
        self.self_attn = _SelfAttn(seed, log)
        self.w = _vec(seed + 9)

    def forward(self, x, e, seq_lens, grid_sizes, freqs, context, context_lens):
        assert context.shape[1] == CLIP_TOKENS + TEXT_LEN and context_lens is None
        y = self.self_attn(x * (1 + e[:, 1]) + e[:, 0], seq_lens, grid_sizes, freqs)
        return x + y * e[:, 2] * self.w + context[:, :CLIP_TOKENS].mean(1) - context[:, CLIP_TOKENS:].mean(1)


class _PatchEmbed(_Scale):
    def forward(self, x):                                  # [1, 2*C_in, f, h, w] -> [1, C, f, h, w]
        return x.repeat(1, C // (2 * C_IN), 1, 1, 1) * self.weight[None, :, None, None, None]


class _ImgEmb(_Scale):
    def forward(self, clip_fea):                           # [1, 257, C] -> [1, 257, C]
        return clip_fea * self.weight


class _Model(torch.nn.Module):
    """The attributes and sub-modules the I2V forward reads (patch size 1), with the TeaCache attributes
    jenga_wan.py:1188-1213 sets on the I2V class; no stage_start and no curve (WanI2V has neither)."""
    model_type = "i2v"
    patch_size = (1, 1, 1)
    enable_teacache = True

    def __init__(self, log, n_blocks=2):
        super().__init__()
        self.dim, self.freq_dim, self.text_len, self.num_heads, self.out_dim = C, C, TEXT_LEN, HEADS, OUT
        self.patch_embedding = _PatchEmbed(1)
        self.time_embedding = _Scale(2)
        self.time_projection = _Proj(3, 6 * C)
        self.text_embedding = _Scale(4)
        self.img_emb = _ImgEmb(8)
        self.head = _Head(5)
        self.blocks = torch.nn.ModuleList([_Block(10 + 10 * i, log) for i in range(n_blocks)])
        self.freqs = torch.randn(4096, C, generator=torch.Generator().manual_seed(6))
        self.reset()

    def reset(self):
        self.cnt, self.num_steps, self.teacache_thresh = 0, 80, 0.5
        self.accumulated_rel_l1_distance_even = self.accumulated_rel_l1_distance_odd = 0
        self.previous_e0_even = self.previous_e0_odd = None
        self.previous_residual_even = self.previous_residual_odd = None
        self.use_ref_steps, self.use_cache = False, False
        self.coefficients, self.ret_steps, self.cutoff_steps = [1.0, 0.0], 2, 78

    def unpatchify(self, x, grid_sizes):
        return [u[:f * h * w].view(f, h, w, OUT).permute(3, 0, 1, 2) for u, (f, h, w) in zip(x, grid_sizes.tolist())]


def _i2v_teacache_single(self, x, t, context, seq_len, clip_fea=None, y=None):
    """jenga_wan.py:503-664 (teacache_forward) for an I2V model of wan/modules/model.py in one process,
    batch 1: raster order, the plain block arguments, stage_start False"""
    import numpy as np
    device = self.patch_embedding.weight.device
    if self.freqs.device != device:
        self.freqs = self.freqs.to(device)
    x = [torch.cat([u, v], dim=0) for u, v in zip(x, y)]
    x = [self.patch_embedding(u.unsqueeze(0)) for u in x]
    grid_sizes = torch.stack([torch.tensor(u.shape[2:], dtype=torch.long) for u in x])
    x = [u.flatten(2).transpose(1, 2) for u in x]
    seq_lens = torch.tensor([u.size(1) for u in x], dtype=torch.long)
    x = torch.cat([torch.cat([u, u.new_zeros(1, seq_len - u.size(1), u.size(2))], dim=1) for u in x])
    with torch.autocast("cuda", dtype=torch.float32, enabled=x.is_cuda):
        e = self.time_embedding(type(self).unpatchify.__globals__["sinusoidal_embedding_1d"](self.freq_dim, t).float())
        e0 = self.time_projection(e).unflatten(1, (6, self.dim))
    context = self.text_embedding(torch.stack([torch.cat([u, u.new_zeros(self.text_len - u.size(0), u.size(1))])
                                               for u in context]))
    context = torch.concat([self.img_emb(clip_fea), context], dim=1)
    kwargs = dict(e=e0, seq_lens=seq_lens, grid_sizes=grid_sizes, freqs=self.freqs, context=context,
                  context_lens=None)
    modulated_inp = e0 if self.use_ref_steps else e
    sfx = "even" if self.cnt % 2 == 0 else "odd"
    prev = getattr(self, "previous_e0_" + sfx)
    if self.cnt < self.ret_steps or self.cnt >= self.cutoff_steps:
        calc = True
        setattr(self, "accumulated_rel_l1_distance_" + sfx, 0)
    else:
        acc = getattr(self, "accumulated_rel_l1_distance_" + sfx) + np.poly1d(self.coefficients)(
            ((modulated_inp - prev).abs().mean() / prev.abs().mean()).cpu().item())
        calc = acc >= self.teacache_thresh
        setattr(self, "accumulated_rel_l1_distance_" + sfx, 0 if calc else acc)
    setattr(self, "previous_e0_" + sfx, modulated_inp.clone())
    if not calc:
        x += getattr(self, "previous_residual_" + sfx)
        self.use_cache = True
    else:
        ori_x = x.clone()
        for block in self.blocks:
            x = block(x, **kwargs)
        setattr(self, "previous_residual_" + sfx, x - ori_x)
        self.use_cache = False
    x = self.head(x, e)
    x = self.unpatchify(x, grid_sizes)
    self.cnt += 1
    if self.cnt >= self.num_steps:
        self.cnt = 0
    return [u.float() for u in x]


def _inputs(grid, seed=7):
    g = torch.Generator().manual_seed(seed)
    x = [torch.randn(C_IN, *grid, generator=g)]
    y = [torch.randn(C_IN, *grid, generator=g)]
    ctx = [torch.randn(TEXT_LEN - 3, C, generator=g)]
    clip = torch.randn(1, CLIP_TOKENS, C, generator=g)
    return x, ctx, clip, y


STEPS = 3          # per grid: cnt 0 and 1 computed, cnt 2 (even, rel-L1 0) reuses cnt 0's residual


def _run(model, fwd, P=1):
    outs = []
    for grid in GRIDS:
        model.reset()
        x, ctx, clip, y = _inputs(grid)
        L = grid[0] * grid[1] * grid[2]
        seq_len = -(-L // P) * P                      # WanI2V.generate's sp_size-rounded max_seq_len
        for _ in range(STEPS):
            outs.append((fwd(x, torch.tensor([900.0]), ctx, seq_len, clip_fea=clip, y=y)[0], model.use_cache))
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
        sp = UlyssesCarvedAttention(dense_fn=_oracle_dense, variant="wan")
        assert wan_sp.parallelize_wan_i2v(model, attention=sp) is sp
        assert all(b.self_attn.jenga_sp is sp for b in model.blocks)
        with torch.no_grad():
            outs = _run(model, model.forward, world)
        ret[rank] = dict(outs=outs, log=log)
        # the errors every rank raises before any collective
        x, ctx, clip, y = _inputs(GRIDS[1])
        with pytest.raises(ValueError, match="runs batch 1, got 2 videos"):
            model.forward(x * 2, torch.tensor([1.0]), ctx, 3000, clip_fea=clip, y=y * 2)
        with pytest.raises(ValueError, match="needs clip_fea and y"):
            model.forward(x, torch.tensor([1.0]), ctx, 3000, y=y)
        if world == 4:
            with pytest.raises(ValueError, match="5 tokens over 4 ranks leave the last rank without a real row"):
                model.forward([torch.randn(C_IN, 1, 1, 5)], torch.tensor([1.0]), ctx, 8, clip_fea=clip,
                              y=[torch.randn(C_IN, 1, 1, 5)])
        if world == 2:
            odd = _Model([])
            odd.num_heads = 3
            with pytest.raises(ValueError, match="sequence-parallel Wan2.1: 3 attention heads do not split over 2"):
                wan_sp.parallelize_wan_i2v(odd, attention=sp)
            plain = _Model([])
            plain.blocks[1].self_attn = torch.nn.Linear(2, 2)
            with pytest.raises(RuntimeError, match=r"Linear.forward is not the fused jenga_b200 forward: "
                                                   r"install\(wan_sp=True\)"):
                wan_sp.parallelize_wan_i2v(plain, attention=sp)
            assert not hasattr(plain.blocks[0].self_attn, "jenga_sp") and "forward" not in plain.__dict__
            bound = _Model([])
            bound.blocks[0].self_attn.forward = lambda *a: None      # the reference usp_attn_forward, bound
            with pytest.raises(RuntimeError, match="instance forward"):
                wan_sp.parallelize_wan_i2v(bound, attention=sp)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_i2v_forward_equals_single_process(world):
    mgr = mp.Manager()
    ret = mgr.dict()
    port = 29500 + (os.getpid() + 53 * world) % 2000
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)

    log = []
    model = _Model(log)
    with torch.no_grad():
        ref = _run(model, lambda *a, **k: _i2v_teacache_single(model, *a, **k))
    assert [u for _, u in ref] == [False, False, True] * len(GRIDS), "no computed and skipped steps"
    calls = [2, 2, 0] * len(GRIDS)                  # self-attention calls per step (two blocks)
    for r in range(world):
        got = ret[r]
        for i, ((o, used), (o_ref, used_ref)) in enumerate(zip(got["outs"], ref)):
            assert used == used_ref, (r, i)
            assert torch.equal(o, o_ref), (r, i)
        assert len(got["log"]) == len(log) == sum(calls)
        j = 0
        for i, c in enumerate(calls):
            f, h, w = GRIDS[i // STEPS]
            L = f * h * w
            n = -(-L // world)
            lo, hi = min(r * n, L), min((r + 1) * n, L)
            for _ in range(c):
                g, e = got["log"][j], log[j]
                assert g["x"].shape[1] == n
                assert torch.equal(g["x"][:, :hi - lo], e["x"][:, lo:hi]), (r, i)
                assert torch.equal(g["remap"], raster_remap(L, n, r))
                j += 1
    for f, h, w in GRIDS:
        assert (f * h * w) % 4, "the grids are not ragged over four ranks"
    assert (3 * 7 * 11) % 2


def test_errors_outside_a_process_group(monkeypatch):
    from jenga_b200 import wan_sp
    assert not dist.is_initialized()
    with pytest.raises(RuntimeError, match="needs an initialised process group"):
        wan_sp.parallelize_wan_i2v(_Model([]))
    monkeypatch.setattr(wan_sp.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(wan_sp.dist, "get_world_size", lambda g=None: 9)
    m = _Model([])
    m.num_heads = 72
    with pytest.raises(ValueError, match="9 ranks; the Ulysses exchange is built for at most 8"):
        wan_sp.parallelize_wan_i2v(m)
    monkeypatch.setattr(wan_sp.dist, "get_world_size", lambda g=None: 3)
    with pytest.raises(ValueError, match="8 attention heads do not split over 3 ranks"):
        wan_sp.parallelize_wan_i2v(_Model([]))
    assert "forward" not in m.__dict__


# ------------------------------------------------------------------------------------------------
# the unmodified wan/modules/model.py
# ------------------------------------------------------------------------------------------------
def load_plain_wan(wan_sp=True, then_off=False):
    """wan/modules/model.py, unmodified, imported after install() with the switch `wan_sp` (and, with
    then_off, the switch turned off again while the module is imported); None when the reference is not
    available.  The switch is restored to what it was; the module's classes keep what the hook did."""
    from jenga_b200 import blocks
    from oracle import make_ref_wan_model
    from oracle import ref_loader as R
    root = R.ref_root()
    if root is None:
        return None
    extra = None
    if not (root / "wan" / "modules" / "model.py").is_file():
        extra = make_ref_wan_model.staged()
        if extra is None:
            return None
    prev = blocks.WAN_SP
    try:
        with R.reference_packages(product=True):
            blocks.set_wan_sp(wan_sp)
            if extra is not None:
                sys.modules["wan.modules"].__path__.append(str(extra / "wan" / "modules"))
            mod = importlib.import_module("wan.modules.model")
            if then_off:
                blocks.set_wan_sp(False)
    finally:
        blocks.set_wan_sp(prev)
        blocks.remove_gather_hook()
    return mod


def _patched(mod):
    return {c: bool(getattr(getattr(mod, c).forward, "__jenga_b200__", False))
            for c in ("WanSelfAttention", "WanAttentionBlock", "WanI2VCrossAttention", "WanT2VCrossAttention")}


@pytest.fixture(scope="module")
def plain_wan():
    mod = load_plain_wan(wan_sp=True)
    if mod is None:
        pytest.skip("reference files not staged (oracle/_ref/, oracle/_ref_wan_model/)")
    return mod


def test_the_switch_hooks_the_plain_model_module(plain_wan):
    assert _patched(plain_wan) == dict(WanSelfAttention=True, WanAttentionBlock=True, WanI2VCrossAttention=False,
                                       WanT2VCrossAttention=False)
    off = load_plain_wan(wan_sp=False)
    assert _patched(off) == dict.fromkeys(_patched(off), False), "the module was touched without the switch"
    back_off = load_plain_wan(wan_sp=True, then_off=True)
    assert _patched(back_off) == dict.fromkeys(_patched(back_off), False)
    assert back_off.WanAttentionBlock.forward.__qualname__ == "WanAttentionBlock.forward"


class _Group:
    """a one-rank group for the checks that run before the exchange"""
    def __init__(self):
        self.group = None

    def __call__(self, *a, **k):
        raise AssertionError("the exchange was reached")


@pytest.mark.parametrize("case", ["context_lens", "clip_rows_only", "t2v_cross", "cpu_input"])
def test_a_block_under_sp_refuses_what_the_fused_i2v_path_does_not_take(plain_wan, case):
    torch.manual_seed(0)
    dim, H, L = 256, 2, 40
    blk = plain_wan.WanAttentionBlock("t2v_cross_attn" if case == "t2v_cross" else "i2v_cross_attn", dim, 512, H,
                                      (-1, -1), True, True, 1e-6)
    blk.self_attn.jenga_sp = _Group()
    x = torch.randn(1, L, dim)
    e = torch.randn(1, 6, dim)
    ctx = torch.randn(1, 257 if case == "clip_rows_only" else 300, dim)
    lens = torch.tensor([300]) if case == "context_lens" else None
    what = "not one the fused block takes" if case == "cpu_input" else "cross-attention is not one the fused I2V"
    with pytest.raises(RuntimeError, match=what):
        blk(x, e, torch.tensor([L]), torch.tensor([[1, 5, 8]]), torch.randn(1024, 64, dtype=torch.complex128),
            ctx, lens)


# ------------------------------------------------------------------------------------------------
# install(): usp_dit_forward's routes
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
install.install(flash_attn=False, gilbert=False, ulysses=False, gather=False, wan_sp=True)
import wan.distributed.xdit_context_parallel as xdit
from jenga_b200 import wan_sp
# the sharded forwards themselves are tested elsewhere: here they report that they were reached
wan_sp._forward_factory = lambda group: (lambda self, *a, **k: "T2V sharded forward")
wan_sp._i2v_forward_factory = lambda group: (lambda self, *a, **k: "I2V sharded forward")
os.environ["MASTER_ADDR"] = "127.0.0.1"
os.environ["MASTER_PORT"] = {port!r}
dist.init_process_group("gloo", rank=0, world_size=1)
class SelfAttn(torch.nn.Module):
    def forward(self, *a, **k):
        return "patched class forward"
    forward.__jenga_b200__ = True
def model(kind):
    m = torch.nn.Module()
    m.num_heads = 40
    m.blocks = torch.nn.ModuleList([torch.nn.Module()])
    m.blocks[0].self_attn = SelfAttn()
    if kind == "t2v":
        m.model_type = "t2v"
        m.hilbert_order = m.linear_to_hilbert = torch.arange(4)
    elif kind == "i2v":
        m.model_type = "i2v"
    # what WanI2V / WanT2V(use_usp=True) do (image2video.py:105-114, text2video.py:88-99)
    for b in m.blocks:
        b.self_attn.forward = types.MethodType(xdit.usp_attn_forward, b.self_attn)
    m.forward = types.MethodType(xdit.usp_dit_forward, m)
    return m
res = {{}}
for kind in ("t2v", "i2v", "plain"):
    m = model(kind)
    sa = m.blocks[0].self_attn
    res[kind] = dict(first=m(None, None, None, 4), second=m(None, None, None, 4),
                     attn=sa(None, None, None, None),
                     jenga_sp=type(getattr(sa, "jenga_sp", None)).__name__)
print(json.dumps(res))
dist.destroy_process_group()
'''


def test_usp_dit_forward_routes_i2v_t2v_and_other_models(tmp_path):
    import json
    stub = tmp_path / "stub"
    (stub / "wan" / "distributed").mkdir(parents=True)
    (stub / "wan" / "__init__.py").write_text("")
    (stub / "wan" / "distributed" / "__init__.py").write_text("")
    (stub / "wan" / "distributed" / "xdit_context_parallel.py").write_text(_STUB)
    code = _PROBE.format(root=str(ROOT), stub=str(stub), port=str(35000 + os.getpid() % 2000))
    env = {k: v for k, v in os.environ.items() if k != "JENGA_WAN_SP"}
    r = subprocess.run([sys.executable, "-s", "-c", code], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    for kind in ("t2v", "i2v"):
        assert got[kind] == dict(first=f"{kind.upper()} sharded forward", second=f"{kind.upper()} sharded forward",
                                 attn="patched class forward", jenga_sp="UlyssesCarvedAttention"), kind
    assert got["plain"] == dict(first="reference usp_dit_forward", second="reference usp_dit_forward",
                                attn="reference usp_attn_forward", jenga_sp="NoneType")
