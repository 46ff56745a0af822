"""The single-GPU Wan2.1-I2V forward and the opt-in carved I2V self-attention (jenga_b200/wan_sp.py) on
the GPU.

A small random-init I2V WanModel of the unmodified wan/modules/model.py (two blocks at 12 heads of 128
channels, latent grid 21x9x14, 257 CLIP + 64 text context rows, bf16 autocast), as in
tests/test_wan_i2v_sp_gpu.py.

* Dense (the default): bind_wan_i2v's forward matches the model's own unpatched forward (model.py's
  WanModel.forward through the flash_attn shim) within the tolerance of tests/test_wan_blocks_gpu.py, and
  equals parallelize_wan_i2v's output at P = 1 bit for bit on two computed steps and a skipped step.
* Carved (I2V_SA_DROP_RATES set): the single-GPU forward matches its restatement, which is what
  teacache_forward computes on I2V: the Hilbert gather, the same weights in model_mul.py
  WanAttentionBlock("i2v_cross_attn") blocks driven with sa_drop_rate / freq_remap /
  block_neighbor_list / p_remain_rates through the installed operator, the head and the scatter.  The
  steps cover the dense warm-up, a partly warmed-up carved step, a full carved step and the second rate.
* Sharded carving, emulated ranks on one GPU: the self-attention section on every rank's Hilbert rows
  equals the single-GPU carved section bit for bit at P = 1..8 (40 heads; P = 3, 6, 7 under the ragged
  head split), on carved and dense warm-up calls; the whole carved forward at P = 2 and at P = 5 (ragged,
  12 heads) matches the single-GPU carved forward within the same tolerance, every rank alike.
* No route falls back (blocks.STATS["fallback"]).
"""
import copy
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
from test_ulysses_ragged_gpu import RaggedWorld  # noqa: E402
from test_wan_blocks_gpu import _compare, _structured_tokens  # noqa: E402
from test_wan_i2v_carve_cpu import restated_schedule  # noqa: E402
from test_wan_i2v_sp_cpu import load_plain_wan  # noqa: E402
from test_wan_i2v_sp_gpu import GRID, HEADS, _inputs, _model, _run  # noqa: E402
from test_wan_sp_forward_gpu import _emulated_all_gather, _emulated_broadcast, _Group, _rows  # noqa: E402
from test_wan_sp_gpu import WanRMSNorm  # noqa: E402

DEV = torch.device("cuda", 0)
D = 128
L = GRID[0] * GRID[1] * GRID[2]
RATES = (0.7, 0.8)
NUM_STEPS = 100                 # 50 sampling steps
# model calls: cnt 0 dense (d = 0), cnt 3 dense warm-up (d = 0.143), cnt 7 warm-up carved (0.429), cnt 20
# carved (0.7), cnt 61 the second rate (0.8, an unconditional call)
CNTS = (0, 3, 7, 20, 61)


def _ones(o):
    return torch.ones(_rows(o).shape[1], dtype=torch.bool, device="cuda")


@pytest.fixture
def plain():
    """a fresh, untouched import of wan/modules/model.py per test (bind_wan_i2v patches its classes)"""
    mod = load_plain_wan(wan_sp=False)
    if mod is None:
        pytest.skip("reference files not staged (oracle/_ref/, oracle/_ref_wan_model/)")
    assert not getattr(mod.WanAttentionBlock.forward, "__jenga_b200__", False)
    return mod


@pytest.fixture
def carving(monkeypatch):
    from jenga_b200 import wan_sp
    monkeypatch.setattr(wan_sp, "I2V_SA_DROP_RATES", RATES)
    monkeypatch.setattr(wan_sp, "I2V_P_REMAIN", 0.8)


def _bound(mod):
    from jenga_b200 import wan_sp
    m = _model(mod, DEV)
    wan_sp.bind_wan_i2v(m)
    assert m.forward.__func__.__qualname__.startswith("_i2v_forward_factory")
    return m


def _call(m, x, ctx, clip, y):
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        return m(x, torch.tensor([900.0], device=DEV), ctx, L, clip_fea=clip, y=y)[0].clone()


def _stats():
    from jenga_b200 import blocks
    return dict(blocks.STATS)


def _delta(before):
    from jenga_b200 import blocks
    return {k: v - before[k] for k, v in blocks.STATS.items() if v != before[k]}


# ------------------------------------------------------------------------------------------------
# dense
# ------------------------------------------------------------------------------------------------
def test_dense_forward_matches_the_unpatched_model_forward(plain):
    from jenga_b200 import wan_sp
    m = _model(plain, DEV)
    m.enable_teacache = False
    x, ctx, clip, y = _inputs(DEV)
    ref = _call(m, x, ctx, clip, y)                          # model.py's WanModel.forward, flash_attn shim
    assert "forward" not in m.__dict__
    wan_sp.bind_wan_i2v(m)
    before = _stats()
    got = _call(m, x, ctx, clip, y)
    delta = _delta(before)
    assert {k: v for k, v in delta.items() if k.startswith(("wan_i2v", "fallback"))} == \
        dict(wan_i2v_self_dense=2, wan_i2v_cross=2), delta
    _compare(_rows(ref), _rows(got), _ones(ref), "single-GPU dense I2V forward vs model.py's forward")


def test_dense_forward_equals_the_sharded_route_at_one_rank(plain, monkeypatch):
    from jenga_b200 import ulysses, wan_sp
    from test_wan_sp_gpu import _World
    fresh = _model(plain, DEV)
    single = copy.deepcopy(fresh)
    wan_sp.bind_wan_i2v(single)
    before = _stats()
    got_single = _run(single, single.forward, DEV)           # computed, computed, skipped
    assert _delta(before).get("fallback", 0) == 0
    assert _delta(before)["wan_i2v_self_dense"] == 4
    dist = ulysses.dist
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    for name, fn in dict(get_world_size=lambda g=None: g.size, get_rank=lambda g=None: g.rank,
                         get_global_rank=lambda g, r: r, is_initialized=lambda: True,
                         all_gather=_emulated_all_gather, broadcast=_emulated_broadcast).items():
        monkeypatch.setattr(dist, name, fn)
    shared = {"rows": {}}
    got = {}

    def rank(r, bar):
        shared["bar"] = bar
        wan_sp.parallelize_wan_i2v(fresh, group=_Group(1, 0, shared), attention=_World(1, L, HEADS).fused(bar, 1, 0, None))
        got[r] = _run(fresh, fresh.forward, DEV, 1)

    _run_ranks(1, rank)
    for i in range(3):
        assert torch.equal(got[0][i], got_single[i]), i


# ------------------------------------------------------------------------------------------------
# carved, one GPU: against the restatement
# ------------------------------------------------------------------------------------------------
def _mul_blocks(model):
    """model_mul.py WanAttentionBlock("i2v_cross_attn") blocks with the model's block weights, bound to the
    installed operator"""
    from oracle import ref_loader as R
    from jenga_b200 import blocks
    mm = R.load_blocks(product=True)[1]
    blocks.remove_gather_hook()
    out = []
    for b in model.blocks:
        nb = mm.WanAttentionBlock("i2v_cross_attn", b.dim, b.ffn_dim, b.num_heads, b.window_size, b.qk_norm,
                                  b.cross_attn_norm, b.eps).to(DEV).eval()
        nb.load_state_dict(b.state_dict())
        out.append(nb)
    assert getattr(type(out[0]).forward, "__jenga_b200__", False)
    return out


def _restated(model, mul, x, t, context, seq_len, clip_fea, y, sa_drop_rate, curve):
    """jenga_wan.py:503-664 (teacache_forward, TeaCache off) over an I2V model: Hilbert gather, the
    model_mul blocks with the Jenga arguments, the scatter; embeddings and head are the model's"""
    l2h, h2l, nbr = curve
    sin = type(model).unpatchify.__globals__["sinusoidal_embedding_1d"]
    x = [torch.cat([u, v], dim=0) for u, v in zip(x, y)]
    x = [model.patch_embedding(u.unsqueeze(0)) for u in x]
    grid_sizes = torch.stack([torch.tensor(u.shape[2:], dtype=torch.long) for u in x])
    x = [u.flatten(2).transpose(1, 2) for u in x]
    seq_lens = torch.tensor([u.size(1) for u in x], dtype=torch.long)
    x = torch.cat([torch.cat([u, u.new_zeros(1, seq_len - u.size(1), u.size(2))], dim=1) for u in x])
    x = x[:, h2l]
    with torch.autocast("cuda", dtype=torch.float32):
        e = model.time_embedding(sin(model.freq_dim, t).float())
        e0 = model.time_projection(e).unflatten(1, (6, model.dim))
    context = model.text_embedding(torch.stack([torch.cat([u, u.new_zeros(model.text_len - u.size(0), u.size(1))])
                                                for u in context]))
    context = torch.concat([model.img_emb(clip_fea), context], dim=1)
    freqs = model.freqs.to(DEV)
    for b in mul:
        x = b(x, e=e0, seq_lens=seq_lens, grid_sizes=grid_sizes, freqs=freqs, context=context, context_lens=None,
              sa_drop_rate=sa_drop_rate, freq_remap=h2l, block_neighbor_list=nbr, p_remain_rates=0.8)
    x = x[:, l2h]
    return model.unpatchify(model.head(x, e), grid_sizes)[0].float()


def test_carved_forward_matches_the_restatement(plain, monkeypatch):
    from jenga_b200 import wan_sp
    m = _bound(plain)
    m.enable_teacache, m.num_steps = False, NUM_STEPS
    mul = _mul_blocks(m)                 # its install() sets the switches from the environment again
    monkeypatch.setattr(wan_sp, "I2V_SA_DROP_RATES", RATES)
    monkeypatch.setattr(wan_sp, "I2V_P_REMAIN", 0.8)
    curve = wan_sp.i2v_curve(*GRID)
    x, ctx, clip, y = _inputs(DEV)
    schedule = restated_schedule(NUM_STEPS // 2, RATES)
    kinds = set()
    for cnt in CNTS:
        d = schedule[cnt]
        m.cnt = cnt
        before = _stats()
        got = _call(m, x, ctx, clip, y)
        delta = _delta(before)
        assert delta.get("fallback", 0) == 0, cnt
        key = "wan_i2v_self_dense" if d <= 0.25 else "wan_i2v_self"
        assert delta[key] == 2 and delta["wan_i2v_cross"] == 2, (cnt, delta)
        kinds.add(key)
        assert m.cnt == cnt + 1
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            ref = _restated(m, mul, x, torch.tensor([900.0], device=DEV), ctx, L, clip, y, d, curve)
        _compare(_rows(ref), _rows(got), _ones(ref), f"carved I2V forward, call {cnt} (drop rate {d:.3f})")
    assert kinds == {"wan_i2v_self_dense", "wan_i2v_self"}


# ------------------------------------------------------------------------------------------------
# carved, sharded
# ------------------------------------------------------------------------------------------------
def _section_module(c, H, jsp=None):
    Cc = H * D
    return types.SimpleNamespace(num_heads=H, head_dim=D, norm_q=WanRMSNorm(c["wq"]), norm_k=WanRMSNorm(c["wk"]),
                                 jenga_sp=jsp, q=lambda x: x[..., :Cc], k=lambda x: x[..., Cc:2 * Cc],
                                 v=lambda x: x[..., 2 * Cc:], o=lambda t: t)


@pytest.mark.parametrize("P", range(1, 9))
def test_sharded_carved_section_equals_single_gpu(monkeypatch, P):
    from jenga_b200 import blocks, ulysses, wan_sp
    from jenga_b200.sharding import shard
    from jenga_b200.wan import rope_freqs
    H = 40
    ragged = H % P != 0
    monkeypatch.setattr(ulysses, "RAGGED_HEADS", ragged)
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    monkeypatch.setattr(ulysses.dist, "get_world_size", lambda g=None: g.size)
    l2h, h2l, nbr = wan_sp.i2v_curve(*GRID)
    g = torch.Generator(device=DEV).manual_seed(6300 + P)
    c = dict(qkv=(_structured_tokens(L, 3 * H * D, 6300 + P) * 0.5)[:, h2l.to(DEV)].contiguous(),
             wq=1.0 + 0.2 * torch.randn(H * D, generator=g, device=DEV),
             wk=1.0 + 0.2 * torch.randn(H * D, generator=g, device=DEV))
    grid, freqs = torch.tensor([list(GRID)]), rope_freqs(D)
    n = -(-L // P)
    for d in (0.7, 0.2):                                     # a carved call and a dense warm-up call
        kw = dict(sa_drop_rate=d, block_neighbor_list=nbr, p_remain_rates=0.8)
        with torch.no_grad():
            single = blocks._wan_i2v_self(_section_module(c, H), c["qkv"], torch.tensor([L]), grid, freqs,
                                          freq_remap=h2l.to(DEV), **kw)
        world = RaggedWorld(P, n, H)
        got = {}

        def rank(r, bar):
            m = _section_module(c, H, world.fused(bar, r, variant="wan"))
            with torch.no_grad():
                out = blocks._wan_i2v_self(m, shard(c["qkv"], 1, P, r), torch.tensor([L]), grid, freqs,
                                           freq_remap=shard(h2l, 0, P, r).to(DEV), **kw)
            torch.cuda.synchronize()
            got[r] = out.clone()

        before = _stats()
        _run_ranks(P, rank)
        delta = _delta(before)
        assert delta == {("wan_i2v_self_sp" if d <= 0.25 else "wan_i2v_self_carved_sp"): P}, delta
        for r in range(P):
            lo, hi = min(r * n, L), min((r + 1) * n, L)
            assert torch.equal(got[r][:, :hi - lo].view(torch.int32), single[:, lo:hi].view(torch.int32)), (d, r)
            assert bool((got[r][:, hi - lo:] == 0).all()), f"rank {r}: pad rows are not zero"
        assert world.guards_intact()
    print(f"\n[wan i2v carve sp] P = {P}{' (ragged heads)' if ragged else ''}: {n} rows per rank")


@pytest.mark.parametrize("P", [2, 5])
def test_sharded_carved_forward_matches_single_gpu(plain, carving, monkeypatch, P):
    from jenga_b200 import ulysses, wan_sp
    fresh = _model(plain, DEV)
    fresh.enable_teacache, fresh.num_steps = False, NUM_STEPS
    single = copy.deepcopy(fresh)
    wan_sp.bind_wan_i2v(single)
    x, ctx, clip, y = _inputs(DEV)
    cnts = (3, 20)                                           # dense warm-up, carved
    ref = []
    for cnt in cnts:
        single.cnt = cnt
        ref.append(_call(single, x, ctx, clip, y))
    monkeypatch.setattr(ulysses, "RAGGED_HEADS", HEADS % P != 0)
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    dist = ulysses.dist
    for name, fn in dict(get_world_size=lambda g=None: g.size, get_rank=lambda g=None: g.rank,
                         get_global_rank=lambda g, r: r, is_initialized=lambda: True,
                         all_gather=_emulated_all_gather, broadcast=_emulated_broadcast).items():
        monkeypatch.setattr(dist, name, fn)
    models = [copy.deepcopy(fresh) for _ in range(P)]
    world = RaggedWorld(P, -(-L // P), HEADS)
    shared = {"rows": {}}
    got = {}

    def rank(r, bar):
        shared["bar"] = bar
        wan_sp.parallelize_wan_i2v(models[r], group=_Group(P, r, shared), attention=world.fused(bar, r, variant="wan"))
        outs = []
        for cnt in cnts:
            models[r].cnt = cnt
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                outs.append(models[r](x, torch.tensor([900.0], device=DEV), ctx, -(-L // P) * P, clip_fea=clip,
                                      y=y)[0].clone())
        got[r] = outs

    before = _stats()
    _run_ranks(P, rank)
    delta = _delta(before)
    assert delta.get("fallback", 0) == 0
    assert delta["wan_i2v_self_sp"] == 2 * P and delta["wan_i2v_self_carved_sp"] == 2 * P, delta
    assert delta["wan_i2v_cross_sp"] == 4 * P
    for i, cnt in enumerate(cnts):
        for r in range(P):
            assert torch.equal(got[r][i], got[0][i]), (r, cnt)
        _compare(_rows(ref[i]), _rows(got[0][i]), _ones(ref[i]), f"sharded carved I2V forward P={P}, call {cnt}")
