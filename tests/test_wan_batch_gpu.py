"""Several videos per call on the fused Wan2.1 and Wan2.1-I2V paths, on an H100.

* Chains: wan_ln_modulate, wan_residual_ln (both forms), wan_gate_residual and the FP8 producers at B = 2
  and 3, C = 1536 and 5120, bf16 and fp32 x, a ragged L, shared and per-sample vectors (the [B, 1, C]
  views of e6.chunk) and strided batches: every sample is bit-identical to the batch-1 call on it.
* Kernels: the Wan prologue, the carved Wan operator (first_frame_blocks at the Wan-1.3B 480p and
  Wan-14B 720p block counts), the dense class (T2V cross-attention) and jenga_wan_i2v_cross_attn at B = 2
  and 3 with distinct samples: every sample is bit-identical to the call on it alone; a NaN canary
  after the last sample's output stays untouched.
* Blocks: the unmodified model_mul.py WanAttentionBlock (T2V) at B = 2 with per-sample t, e and context
  runs the fused block once (blocks.STATS: one wan_block, no fallback) and matches each sample alone and
  the original forward within the drop-in tolerance of tests/test_wan_blocks_gpu.py, with the FP8
  Linears off and forced on for every Wan shape.
* Forwards: bind_wan_i2v's forward at B = 2, dense and carved, on computed and TeaCache-skipped steps,
  against each sample alone; the sharded T2V and I2V forwards on emulated ranks at P = 1 and 2 and
  B = 2, every rank's output bit-identical to the others' and each sample within the drop-in tolerance of
  the one-GPU route on the same batch.  On two GPUs (skipped on a one-GPU box) the real exchange at B = 2.
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
from test_ulysses_batch_gpu import BatchWorld  # noqa: E402
from test_ulysses_emulated_gpu import _Handle, _run_ranks  # noqa: E402
from test_wan_blocks_gpu import _compare, _reinit, _structured_tokens, _Unpatched  # noqa: E402

DEV = torch.device("cuda", 0)


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape)
    assert torch.equal(a.view(torch.uint8) if a.dtype == torch.float8_e4m3fn else a,
                       b.view(torch.uint8) if b.dtype == torch.float8_e4m3fn else b), what


# ------------------------------------------------------------------------------------------------
# chains
# ------------------------------------------------------------------------------------------------
def _batch(B, L, C, dtype, strided, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    full = (torch.randn(B, L + (24 if strided else 0), C, generator=g, device=DEV) * 2).to(dtype)
    return full[:, 3:L + 3] if strided else full


@pytest.mark.parametrize("B", [2, 3])
@pytest.mark.parametrize("C", [1536, 5120])
@pytest.mark.parametrize("x_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("shared", [False, True])
def test_chains_give_each_sample_its_batch_one_result(B, C, x_dtype, shared):
    from jenga_b200 import dense as DN
    L = 1000 + 37                                          # ragged
    x = _batch(B, L, C, x_dtype, strided=not shared, seed=B * C)
    y = _batch(B, L, C, torch.bfloat16, strided=shared, seed=B * C + 1)
    g = torch.Generator(device=DEV).manual_seed(5)
    e6 = 0.3 * torch.randn(1 if shared else B, 6, C, generator=g, device=DEV)
    e = e6.chunk(6, dim=1)
    w3 = 1 + 0.1 * torch.randn(C, generator=g, device=DEV)
    b3 = 0.1 * torch.randn(C, generator=g, device=DEV)
    row = (lambda v, b: v) if shared else (lambda v, b: v[b:b + 1])

    def calls(x, y, b=None):
        pick = (lambda v: v) if b is None else (lambda v: row(v, b))
        return {
            "ln_modulate": DN.wan_ln_modulate(x, pick(e[0]), pick(e[1])),
            "ln_modulate_fp8": DN.wan_ln_modulate_fp8(x, pick(e[0]), pick(e[1])),
            "residual_ln affine": DN.wan_residual_ln(x, y, pick(e[2]), weight=w3, bias=b3),
            "residual_ln modulate": DN.wan_residual_ln(x, y, None, shift=pick(e[3]), scale=pick(e[4])),
            "residual_ln_fp8 affine": DN.wan_residual_ln_fp8(x, y, pick(e[2]), weight=w3, bias=b3),
            "residual_ln_fp8 modulate": DN.wan_residual_ln_fp8(x, y, None, shift=pick(e[3]), scale=pick(e[4])),
            "gate_residual": DN.wan_gate_residual(x, y, pick(e[5])),
        }

    with torch.autocast("cuda", dtype=torch.bfloat16):
        both = calls(x, y)
        alone = [calls(x[b:b + 1], y[b:b + 1], b) for b in range(B)]
    torch.cuda.synchronize()

    def flat(v, b):
        """sample b of one result: [B, L, C] tensors by batch, the FP8 [B*L, C] rows by row range"""
        if isinstance(v, tuple):
            return tuple(flat(t, b) for t in v)
        return v[b * L:(b + 1) * L] if v.dim() <= 2 else v[b:b + 1]

    for name, v in both.items():
        for b in range(B):
            got, want = flat(v, b), alone[b][name]
            got = got if isinstance(got, tuple) else (got,)
            want = want if isinstance(want, tuple) else (want,)
            for i, (gg, ww) in enumerate(zip(_leaves(got), _leaves(want))):
                _same(gg.reshape(ww.shape), ww, (name, b, i))


def _leaves(t):
    for v in t:
        if isinstance(v, tuple):
            yield from _leaves(v)
        else:
            yield v


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------
def _tokens(B, L, C, seed):
    return torch.cat([_structured_tokens(L, C, seed + 17 * b) for b in range(B)])


@pytest.mark.parametrize("B", [2, 3])
@pytest.mark.parametrize("x_dtype", [torch.bfloat16, torch.float32])
def test_prologue_per_sample(B, x_dtype):
    from jenga_b200 import gilbert
    from jenga_b200.wan import norm_rope, rope_freqs
    f, h, w, H = 21, 9, 14, 12
    L = f * h * w
    x = _tokens(B, L, H * 128, 3).to(x_dtype)
    wq = 1 + 0.1 * torch.randn(H * 128, device=DEV)
    remap = gilbert.mapping_tensors(f, h, w, sliced=True)[1].to(DEV)
    freqs = rope_freqs()
    for fr in (None, remap):
        got = norm_rope(x, wq, H, (f, h, w), freqs, fr)
        for b in range(B):
            _same(got[b:b + 1], norm_rope(x[b:b + 1], wq, H, (f, h, w), freqs, fr), ("prologue", b))


@pytest.mark.parametrize("B", [2, 3])
def test_t2v_cross_attention_per_sample(B):
    """the dense class of the attention kernel with each sample's own 512 context rows"""
    from jenga_b200 import wan as WAN
    H, L, Lc = 12, 4032 + 77, 512
    C = H * 128
    q = _tokens(B, L, C, 5)
    k = _tokens(B, Lc, C, 6)
    v = torch.randn(B, Lc, H, 128, device=DEV).bfloat16()
    wq, wk = 1 + 0.1 * torch.randn(C, device=DEV), 1 + 0.1 * torch.randn(C, device=DEV)
    got = WAN.cross_attention(q, k, v, wq, wk, H)
    for b in range(B):
        _same(got[b:b + 1], WAN.cross_attention(q[b:b + 1], k[b:b + 1], v[b:b + 1], wq, wk, H), ("cross", b))
    assert not torch.equal(got[0], got[1])


@pytest.mark.parametrize("B", [2, 3])
def test_i2v_cross_attn_per_sample_with_canary(B):
    from jenga_b200 import wan as WAN
    H, L, Li, Lt = 40, 3000 + 5, 257, 512
    g = torch.Generator(device=DEV).manual_seed(9)
    r = lambda S: torch.randn(B, S, H, 128, generator=g, device=DEV).bfloat16()   # noqa: E731
    q, ki, vi, kt, vt = r(L), r(Li), r(Li), r(Lt), r(Lt)
    full = torch.full((B + 1, L, H, 128), float("nan"), dtype=torch.bfloat16, device=DEV)
    got = WAN.i2v_cross_attn(q, ki, vi, kt, vt, out=full[:B])
    assert torch.isnan(full[B]).all(), "rows after the last sample were written"
    for b in range(B):
        s = slice(b, b + 1)
        _same(got[s], WAN.i2v_cross_attn(q[s], ki[s], vi[s], kt[s], vt[s]), ("i2v cross", b))


@pytest.mark.parametrize("grid,H", [((21, 30, 52), 12), ((21, 45, 80), 40)], ids=["wan-1.3b-480p", "wan-14b-720p"])
def test_carved_wan_operator_per_sample(grid, H):
    """WAN.self_attention at B = 2: top_k and first_frame_blocks of the single-GPU rule over L; selection
    per (sample, head)"""
    from jenga_b200 import gilbert
    from jenga_b200 import wan as WAN
    f, h, w = grid
    L, C, B = f * h * w, H * 128, 2
    top_k, ff = WAN.block_counts(L, 0.7)
    assert ff >= 1
    l2h, h2l = gilbert.mapping_tensors(f, h, w, sliced=True)
    nbr = gilbert.block_neighbor_mapping(f, h, w, sliced=True)
    q, k = _tokens(B, L, C, 11), _tokens(B, L, C, 12)
    v = torch.randn(B, L, H, 128, device=DEV).bfloat16()
    wq, wk = 1 + 0.1 * torch.randn(C, device=DEV), 1 + 0.1 * torch.randn(C, device=DEV)
    kw = dict(p_remain_rates=0.8, freq_remap=h2l.to(DEV), block_neighbor_list=nbr)
    got = WAN.self_attention(q, k, v, wq, wk, H, grid, WAN.rope_freqs(), 0.7, **kw)
    for b in range(B):
        s = slice(b, b + 1)
        _same(got[s], WAN.self_attention(q[s], k[s], v[s], wq, wk, H, grid, WAN.rope_freqs(), 0.7, **kw),
              ("carved", grid, b))


# ------------------------------------------------------------------------------------------------
# the T2V block
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def wan_modules():
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    ours = R.load_blocks(product=True)[1]
    assert ours.WanAttentionBlock.forward.__jenga_b200__
    yield ours
    from jenga_b200 import blocks
    blocks.remove_gather_hook()


def _fp8_everything(monkeypatch, dim, ffn):
    from jenga_b200 import dense as DN
    monkeypatch.setattr(DN, "LINEAR_FP8", True)
    monkeypatch.setattr(DN, "FP8_ROUTED", frozenset({("fp32", dim, dim), ("fp32", dim, ffn), ("fp32", ffn, dim)}))


@pytest.mark.parametrize("fp8", [False, True], ids=["fp8-off", "fp8-all"])
def test_t2v_block_batch_two(wan_modules, monkeypatch, fp8):
    from jenga_b200 import blocks, gilbert
    mod = wan_modules
    dim, H, ffn, f, h, w = 1536, 12, 8960, 21, 12, 16
    L = f * h * w
    if fp8:
        _fp8_everything(monkeypatch, dim, ffn)
    blk = mod.WanAttentionBlock("t2v_cross_attn", dim, ffn, H, (-1, -1), True, True, 1e-6).cuda()
    _reinit(blk, 61)
    d = dim // H
    freqs = torch.cat([mod.rope_params(1024, d - 4 * (d // 6)), mod.rope_params(1024, 2 * (d // 6)),
                       mod.rope_params(1024, 2 * (d // 6))], dim=1).cuda()
    h2l = gilbert.mapping_tensors(f, h, w, sliced=True)[1].cuda()
    nbr = gilbert.block_neighbor_mapping(f, h, w, sliced=True)
    g = torch.Generator(device="cuda").manual_seed(62)
    B = 2
    x = _tokens(B, L, dim, 63).float()
    e = 0.3 * torch.randn(B, 6, dim, generator=g, device="cuda")              # per-sample t
    ctx = torch.randn(B, 512, dim, generator=g, device="cuda").bfloat16()       # per-sample prompt
    kw = dict(sa_drop_rate=0.75, freq_remap=h2l, block_neighbor_list=nbr, p_remain_rates=0.9)

    def run(xx, ee, cc, unpatched=False):
        before = dict(blocks.STATS)
        n = xx.shape[0]
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            if unpatched:
                with _Unpatched(mod):
                    out = blk(xx, ee, torch.tensor([L] * n), torch.tensor([[f, h, w]] * n), freqs, cc, None, **kw)
            else:
                out = blk(xx, ee, torch.tensor([L] * n), torch.tensor([[f, h, w]] * n), freqs, cc, None, **kw)
        return out, {k: blocks.STATS[k] - before[k] for k in blocks.STATS}

    both, st = run(x, e, ctx)
    assert st["wan_block"] == 1 and st["wan_self"] == 1 and st["wan_cross"] == 1 and st["fallback"] == 0, st
    assert (st["linear_fp8"] > 0) == fp8, st
    every = torch.ones(L, dtype=torch.bool, device="cuda")
    for b in range(B):
        s = slice(b, b + 1)
        alone, sa = run(x[s], e[s], ctx[s])
        assert sa["wan_block"] == 1 and sa["fallback"] == 0
        _compare(alone, both[s], every, f"T2V block B=2 sample {b} vs alone ({'fp8' if fp8 else 'bf16'} Linears)")
    if not fp8:
        orig, so = run(x, e, ctx, unpatched=True)
        assert so["wan_block"] == 0
        for b in range(B):
            s = slice(b, b + 1)
            _compare(orig[s], both[s], every, f"T2V block B=2 sample {b} vs original forward")
    # samples on two grids are not the fused block's: the block body declines them (the original forward
    # would run), and the fused self-attention hands them back to the original forward too
    grids = torch.tensor([[f, h, w], [f, h, w - 1]])
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        assert blocks._wan_block_body(blk, x, e, torch.tensor([L, L]), grids, freqs, ctx, None, kw, False) is None
        assert blocks._wan_self_fused(blk.self_attn, None, x.bfloat16(), grids, freqs, 0.75, 128, 0.9, h2l, nbr,
                                      ("wan_self", None), fallback=True) is None


# ------------------------------------------------------------------------------------------------
# bind_wan_i2v's forward, one GPU
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def plain_wan():
    from test_wan_i2v_sp_cpu import load_plain_wan
    mod = load_plain_wan(wan_sp=True)
    if mod is None:
        pytest.skip("reference files not staged (oracle/_ref/, oracle/_ref_wan_model/)")
    return mod


def _i2v_inputs(B, seed=7, dev=DEV):
    from test_wan_i2v_sp_gpu import GRID, TEXT_DIM, TEXT_LEN
    f, h, w = GRID
    xs, ys, cs, clips = [], [], [], []
    for b in range(B):
        g = torch.Generator(device=dev).manual_seed(seed + 13 * b)
        xs.append(torch.randn(16, f, 2 * h, 2 * w, generator=g, device=dev))
        ys.append(torch.randn(20, f, 2 * h, 2 * w, generator=g, device=dev))
        cs.append(torch.randn(TEXT_LEN - 9, TEXT_DIM, generator=g, device=dev))
        clips.append(torch.randn(1, 257, 1280, generator=g, device=dev))
    return xs, cs, torch.cat(clips), ys


def _i2v_steps(model, fwd, xs, cs, clip, ys, ts, seq_len):
    outs, used = [], []
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for _ in range(3):                      # cnt 0 and 1 computed, cnt 2 (even, rel-L1 0) skipped
            outs.append(torch.stack(fwd(xs, ts, cs, seq_len, clip_fea=clip, y=ys)))
            used.append(model.use_cache)
    assert used == [False, False, True], used
    return outs


def _rows(o):
    """[B, 16, f, H, W] -> [B, f*H*W, 16]"""
    return o.reshape(o.shape[0], o.shape[1], -1).transpose(1, 2)


def _every(o):
    """_compare's row mask over every output row of o"""
    return torch.ones(_rows(o).shape[1], dtype=torch.bool, device="cuda")


@pytest.mark.parametrize("carved", [False, True], ids=["dense", "carved"])
def test_single_gpu_i2v_forward_batch_two(plain_wan, monkeypatch, carved):
    from test_wan_i2v_sp_gpu import GRID, _model
    from jenga_b200 import blocks, wan_sp
    L = GRID[0] * GRID[1] * GRID[2]
    B = 2
    base = _model(plain_wan, DEV)
    xs, cs, clip, ys = _i2v_inputs(B)
    ts = torch.tensor([900.0, 870.0], device=DEV)
    # the first sampling steps of the schedule are dense warm-up steps: hold the carved rate from the start
    monkeypatch.setattr(wan_sp, "sa_drop_schedule", lambda cnt, num_steps, rates: 0.7)
    try:
        wan_sp.set_i2v_carving("0.7" if carved else None)
        m = copy.deepcopy(base)
        wan_sp.bind_wan_i2v(m)
        before = dict(blocks.STATS)
        both = _i2v_steps(m, m.forward, xs, cs, clip, ys, ts, L)
        assert m.previous_residual_even.shape[0] == B            # the stored residual is the batch's
        assert blocks.STATS["fallback"] == before["fallback"]
        key = "wan_i2v_self" if carved else "wan_i2v_self_dense"
        # two computed steps x two blocks
        assert blocks.STATS["wan_i2v_cross"] - before["wan_i2v_cross"] == 4
        assert blocks.STATS[key] - before[key] == 4
        for b in range(B):
            m1 = copy.deepcopy(base)
            wan_sp.bind_wan_i2v(m1)
            alone = _i2v_steps(m1, m1.forward, [xs[b]], [cs[b]], clip[b:b + 1], [ys[b]], ts[b:b + 1], L)
            for i, what in enumerate(("computed", "computed", "skipped")):
                _compare(_rows(alone[i]), _rows(both[i][b:b + 1]), _every(alone[i]),
                         f"one-GPU I2V forward ({'carved' if carved else 'dense'}) B=2 sample {b}, {what}")
    finally:
        wan_sp.set_i2v_carving(None)


# ------------------------------------------------------------------------------------------------
# the sharded forwards on emulated ranks
# ------------------------------------------------------------------------------------------------
def _emulated_fused(wb, bar, r, P):
    from jenga_b200.ulysses import UlyssesFusedAttention

    class EmulatedFused(UlyssesFusedAttention):
        def _buffers(self, N, T, h, D_, n_loc, H_, dtype, dev, batch=1):
            assert (N, T, n_loc, batch) == (wb.N, 0, wb.n, wb.B)
            hd = _Handle(bar)
            return wb.qkv[r], hd, wb.p_qkv, [(wb.out[i][r], hd, wb.p_out[i]) for i in range(2)]

    return EmulatedFused


def _patch_dist(monkeypatch):
    from test_wan_sp_forward_gpu import _emulated_all_gather, _emulated_broadcast
    from jenga_b200 import ulysses
    dist = ulysses.dist
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    monkeypatch.setattr(dist, "get_world_size", lambda g=None: g.size)
    monkeypatch.setattr(dist, "get_rank", lambda g=None: g.rank)
    monkeypatch.setattr(dist, "get_global_rank", lambda g, r: r)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "all_gather", _emulated_all_gather)
    monkeypatch.setattr(dist, "broadcast", _emulated_broadcast)


@pytest.mark.parametrize("P", [1, 2])
def test_sharded_i2v_forward_batch_two(plain_wan, monkeypatch, P):
    from test_wan_i2v_sp_gpu import GRID, HEADS, _model
    from test_wan_sp_forward_gpu import _Group
    from jenga_b200 import blocks, wan_sp
    L = GRID[0] * GRID[1] * GRID[2]
    B, n = 2, -(-L // P)
    base = _model(plain_wan, DEV)
    xs, cs, clip, ys = _i2v_inputs(B)
    ts = torch.tensor([900.0, 870.0], device=DEV)
    single = copy.deepcopy(base)
    wan_sp.bind_wan_i2v(single)
    want = _i2v_steps(single, single.forward, xs, cs, clip, ys, ts, n * P)
    _patch_dist(monkeypatch)
    wb = BatchWorld(P, n, 0, B, n_out=2, heads=HEADS)
    models = [copy.deepcopy(base) for _ in range(P)]
    shared, got = {"rows": {}}, {}
    before = dict(blocks.STATS)

    def rank(r, bar):
        shared["bar"] = bar
        group = _Group(P, r, shared)
        wan_sp.parallelize_wan_i2v(models[r], group=group, attention=_emulated_fused(wb, bar, r, P)(
            group=group, variant="wan"))
        got[r] = _i2v_steps(models[r], models[r].forward, xs, cs, clip, ys, ts, n * P)

    _run_ranks(P, rank)
    assert blocks.STATS["fallback"] == before["fallback"]
    assert blocks.STATS["wan_i2v_self_sp"] - before["wan_i2v_self_sp"] == 4 * P
    for i in range(3):
        for r in range(P):
            assert torch.equal(got[r][i], got[0][i]), (r, i)
        for b in range(B):
            _compare(_rows(want[i][b:b + 1]), _rows(got[0][i][b:b + 1]), _every(want[i]),
                     f"sharded I2V forward P={P} B=2 sample {b}, step {i} vs one-GPU route")


@pytest.mark.parametrize("P", [1, 2])
def test_sharded_t2v_forward_batch_two(monkeypatch, P):
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    from test_wan_sp_cpu import _steps, _teacache_single
    from test_wan_sp_forward_gpu import HEADS, TEXT_DIM, TEXT_LEN, _Group, _model
    from jenga_b200 import blocks, wan_sp
    mod = R.load_blocks(product=True)[1]
    base = _model(mod, DEV)
    B = 2
    worlds = {}

    def inputs(grid):
        f, h, w = grid
        xs, cs = [], []
        for b in range(B):
            g = torch.Generator(device=DEV).manual_seed(7 + 13 * b)
            xs.append(torch.randn(16, f, 2 * h, 2 * w, generator=g, device=DEV))
            cs.append(torch.randn(TEXT_LEN - 9, TEXT_DIM, generator=g, device=DEV))
        return xs, cs

    def run(model, fwd):
        outs = []
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            for _, drop, t, grid, before in _steps():
                if before is not None:
                    before(model)
                xs, cs = inputs(grid)
                L = grid[0] * grid[1] * grid[2]
                ts = torch.tensor([t, t - 20.0], device=DEV)
                outs.append((torch.stack(fwd(xs, ts, cs, L + 3, sa_drop_rate=drop)), model.use_cache))
        return outs

    def fresh(m):
        m.set_curve = (lambda mm: lambda i: [setattr(mm, a, v) for a, v in zip(
            ("linear_to_hilbert", "hilbert_order", "block_neighbor_list"), mm.curve_sels[i][0])])(m)
        m.set_curve(0)
        return m

    ref_model = fresh(copy.deepcopy(base))
    want = run(ref_model, lambda *a, **k: _teacache_single(ref_model, *a, **k))
    assert [u for _, u in want] == [False, False, True, False, False]
    _patch_dist(monkeypatch)
    for _, _, _, grid, _ in _steps():
        L = grid[0] * grid[1] * grid[2]
        worlds.setdefault(L, BatchWorld(P, -(-L // P), 0, B, n_out=2, heads=HEADS))
    models = [fresh(copy.deepcopy(base)) for _ in range(P)]
    shared, got = {"rows": {}}, {}
    before = dict(blocks.STATS)

    def rank(r, bar):
        shared["bar"] = bar
        group = _Group(P, r, shared)
        by_len = {L: _emulated_fused(w, bar, r, P)(group=group, variant="wan") for L, w in worlds.items()}

        class _ByLength:
            def __call__(self, attn, q, *a, seq_len=None, **k):
                return by_len[seq_len](attn, q, *a, seq_len=seq_len, **k)

        wan_sp.parallelize_wan(models[r], group=group, attention=_ByLength())
        got[r] = run(models[r], models[r].forward)

    _run_ranks(P, rank)
    assert blocks.STATS["wan_self_sp"] == before["wan_self_sp"] + 6 * P
    assert blocks.STATS["fallback"] == before["fallback"]
    for i, (name, *_r) in enumerate(_steps()):
        assert [got[r][i][1] for r in range(P)] == [want[i][1]] * P
        for r in range(P):
            assert torch.equal(got[r][i][0], got[0][i][0]), (r, name)
        for b in range(B):
            o, o_ref = got[0][i][0][b:b + 1], want[i][0][b:b + 1]
            _compare(_rows(o_ref), _rows(o), torch.ones(o.shape[2] * o.shape[3] * o.shape[4], dtype=torch.bool,
                                                         device="cuda"),
                     f"sharded T2V forward P={P} B=2 sample {b}, {name} vs one-GPU fused forward")


# ------------------------------------------------------------------------------------------------
# two GPUs
# ------------------------------------------------------------------------------------------------
def _two_gpu_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        from test_wan_i2v_sp_cpu import load_plain_wan
        from test_wan_i2v_sp_gpu import GRID, _model
        from jenga_b200 import blocks, wan_sp
        mod = load_plain_wan(wan_sp=True)
        dev = torch.device("cuda", rank)
        model = _model(mod, dev)
        wan_sp.parallelize_wan_i2v(model)
        L = GRID[0] * GRID[1] * GRID[2]
        xs, cs, clip, ys = _i2v_inputs(2, dev=dev)
        outs = _i2v_steps(model, model.forward, xs, cs, clip, ys, torch.tensor([900.0, 870.0], device=dev),
                          -(-L // world) * world)
        torch.cuda.synchronize()
        ret[rank] = dict(outs=[o.cpu() for o in outs], fallback=blocks.STATS["fallback"])
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_gpus_real_exchange_batch_two(plain_wan):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    from test_wan_i2v_sp_gpu import GRID, _model
    from jenga_b200 import wan_sp
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_two_gpu_worker, args=(world, 29500 + (os.getpid() + 11) % 2000, ret), nprocs=world, join=True)
    L = GRID[0] * GRID[1] * GRID[2]
    single = _model(plain_wan, DEV)
    wan_sp.bind_wan_i2v(single)
    xs, cs, clip, ys = _i2v_inputs(2)
    want = _i2v_steps(single, single.forward, xs, cs, clip, ys, torch.tensor([900.0, 870.0], device=DEV),
                      -(-L // world) * world)
    for r in range(world):
        assert ret[r]["fallback"] == 0
        for i in range(3):
            o = ret[r]["outs"][i].to("cuda")
            for b in range(2):
                _compare(_rows(want[i][b:b + 1]), _rows(o[b:b + 1]), _every(o),
                         f"two GPUs rank {r}, step {i}, sample {b}")
