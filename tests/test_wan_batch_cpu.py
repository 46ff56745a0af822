"""Several videos per call on the Wan2.1 paths, without a GPU.

* The shape rules of the Wan chains and FP8 producers at B > 1: a vector batch that is neither 1 nor B, a
  misaligned batch stride and a y unlike x raise ValueError before any device check; well-shaped CPU
  arguments get past the shape checks and stop at the device check (JengaError: no CPU path).
* The block rules: a context batch unlike x's is not taken by the fused cross-attentions, and samples on
  different latent grids raise ValueError on the routes without a fall-back.
* The sharded T2V and I2V forwards (gloo, world 2) at B = 2 and 3 on the batched stand-in models below,
  built on those of tests/test_wan_sp_cpu.py and tests/test_wan_i2v_sp_cpu.py: every rank's output equals
  the single-process restatement of teacache_forward on the same batch, on computed, TeaCache-skipped and
  turbo-swap steps; on a computed step each sample equals that sample run alone.  The batch rules raise
  before any collective.
"""
import os
import sys
from pathlib import Path

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))

import test_wan_i2v_sp_cpu as I2V  # noqa: E402
import test_wan_sp_cpu as T2V  # noqa: E402
from jenga_b200 import dense as DN  # noqa: E402
from jenga_b200._lib import JengaError  # noqa: E402

B, L, C = 3, 16, 64


# ------------------------------------------------------------------------------------------------
# the chains
# ------------------------------------------------------------------------------------------------
def _x(b=B, dtype=torch.float32):
    return torch.zeros(b, L, C, dtype=dtype)


def _y(b=B):
    return torch.zeros(b, L, C, dtype=torch.bfloat16)


def _e6(b):
    """the six [b, 1, C] vectors of e6.chunk(6, dim=1): batch stride 6 C"""
    return torch.zeros(b, 6, C).chunk(6, dim=1)


def _calls(x, v, y=None):
    """every Wan chain with `v` as each of its per-sample vectors in turn, the others well-shaped"""
    ok = _e6(x.shape[0])[0]
    y = _y(x.shape[0]) if y is None else y
    w = torch.zeros(C)
    return [
        lambda: DN.wan_ln_modulate(x, v, ok),
        lambda: DN.wan_ln_modulate(x, ok, v),
        lambda: DN.wan_ln_modulate_fp8(x, v, ok),
        lambda: DN.wan_residual_ln(x, y, v, weight=w, bias=w),
        lambda: DN.wan_residual_ln(x, y, None, shift=v, scale=ok),
        lambda: DN.wan_residual_ln(x, y, None, shift=ok, scale=v),
        lambda: DN.wan_residual_ln_fp8(x, y, v, weight=w, bias=w),
        lambda: DN.wan_residual_ln_fp8(x, y, None, shift=ok, scale=v),
        lambda: DN.wan_gate_residual(x, y, v),
    ]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", ["chunk", (B, C), (1, C), (C,), (1, 1, C)])
def test_per_sample_and_shared_vectors_pass_the_shape_checks(shape, dtype):
    v = _e6(B)[3] if shape == "chunk" else torch.zeros(*shape)
    for call in _calls(_x(dtype=dtype), v):
        with pytest.raises(JengaError, match="no CPU path"):
            call()


@pytest.mark.parametrize("shape", [(B - 1, C), (B + 1, C), (B, C // 2), (1, B * C), (B * C,), (B, C + 8),
                                   (B - 1, 1, C)])
def test_a_vector_batch_neither_one_nor_b_raises_value_error(shape):
    for call in _calls(_x(), torch.zeros(*shape)):
        with pytest.raises(ValueError, match="one value per channel"):
            call()


def test_batch_one_takes_c_values_only():
    for call in _calls(_x(1), torch.zeros(2, C)):
        with pytest.raises(ValueError, match="one value per channel"):
            call()


def test_norm3_parameters_are_shared_by_every_sample():
    """weight / bias of the affine norm3 hold C values, never one row per sample"""
    x, y, g = _x(), _y(), _e6(B)[2]
    for fn in (DN.wan_residual_ln, DN.wan_residual_ln_fp8):
        with pytest.raises(ValueError, match="weight must hold one value per channel"):
            fn(x, y, g, weight=torch.zeros(B, C), bias=torch.zeros(C))


def test_a_misaligned_batch_stride_raises_value_error():
    """samples start 8-element aligned: a [B, L, C] view of rows L + 1 apart (batch stride (L+1) C is
    aligned, so the pitch is made odd by a 4-channel offset)"""
    full = torch.zeros(B, L * C + 4)
    x = full[:, :L * C].view(B, L, C)
    assert x.stride(0) % 8 == 4
    v = _e6(B)[0]
    yb = torch.zeros(B, L * C + 4, dtype=torch.bfloat16)[:, :L * C].view(B, L, C)
    for call in (lambda: DN.wan_ln_modulate(x, v, v), lambda: DN.wan_ln_modulate_fp8(x, v, v),
                 lambda: DN.wan_gate_residual(x, _y(), v), lambda: DN.wan_gate_residual(_x(), yb, v),
                 lambda: DN.wan_residual_ln(_x(), yb, v, weight=torch.zeros(C), bias=torch.zeros(C)),
                 lambda: DN.wan_residual_ln_fp8(x, _y(), None, shift=v, scale=v)):
        with pytest.raises(ValueError, match="batch stride"):
            call()


def test_y_unlike_x_raises_value_error():
    v = _e6(B)[0]
    for y in (_y(B - 1), torch.zeros(B, L, C)):
        with pytest.raises(ValueError, match="y must be a bf16 tensor shaped like x"):
            DN.wan_gate_residual(_x(), y, v)


def test_the_predicates_take_a_batch_but_not_an_expanded_one():
    """an expanded batch (stride 0) is one sample seen B times: the fused Wan path does not take it"""
    x = torch.zeros(B, L, C)
    assert DN.distinct_samples(x) and DN.distinct_samples(x[:1].expand(1, L, C))
    assert not DN.distinct_samples(x[:1].expand(B, L, C))
    assert not DN._wan_rows_ok(x, torch.zeros(B, 6, C))             # not a CUDA tensor


# ------------------------------------------------------------------------------------------------
# the block rules
# ------------------------------------------------------------------------------------------------
def test_one_grid_rule():
    from jenga_b200 import blocks
    g = torch.tensor([[21, 9, 14]] * 3)
    assert blocks._one_grid(g) and blocks._one_grid(g[:1])
    g2 = g.clone()
    g2[1, 2] = 16
    assert not blocks._one_grid(g2)
    with pytest.raises(ValueError, match="share one latent grid"):
        blocks._check_one_grid(g2, "WanAttentionBlock")
    blocks._check_one_grid(g, "WanAttentionBlock")


def test_a_context_batch_unlike_x_is_not_taken():
    from jenga_b200 import blocks
    ca = I2V_CROSS()
    x = torch.zeros(2, 300, 256)
    ctx = torch.zeros(2, 257 + 512, 256)
    assert blocks._wan_i2v_cross_shape_ok(ca, x, ctx, None)
    assert not blocks._wan_i2v_cross_shape_ok(ca, x, ctx[:1], None)
    assert not blocks._wan_i2v_cross_shape_ok(ca, x[:1], ctx, None)
    assert not blocks._wan_i2v_cross_shape_ok(ca, x, ctx[:1].expand(2, -1, -1), None)


def I2V_CROSS():
    sys.path.insert(0, str(HERE))
    from test_wan_i2v_cpu import _I2VCross
    return _I2VCross()


def test_the_sharded_block_raises_on_several_grids():
    """a plain block on curve-ordered rows (freq_remap set) has no fall-back: several grids raise
    ValueError before anything runs"""
    from jenga_b200 import blocks

    class _Blk:
        self_attn = object()
    g = torch.tensor([[3, 4, 5], [3, 4, 6]])
    with pytest.raises(ValueError, match="share one latent grid"):
        blocks._wan_block(True, _Blk(), torch.zeros(2, 60, 8), torch.zeros(2, 6, 8), torch.tensor([60, 72]), g,
                          None, torch.zeros(2, 3, 8), None, sa_drop_rate=0.7, freq_remap=torch.arange(60))


# ------------------------------------------------------------------------------------------------
# the sharded forwards on batched stand-in models
# ------------------------------------------------------------------------------------------------
class _T2VSelfAttn(T2V._SelfAttn):
    """test_wan_sp_cpu's stand-in on [B, n, C] rows"""

    def forward(self, x, seq_lens, grid_sizes, freqs, sa_drop_rate=0.0, per_block_tokens=128, p_remain_rates=0.8,
                freq_remap=None, block_neighbor_list=None):
        from jenga_b200.wan import block_counts
        assert bool((grid_sizes == grid_sizes[:1]).all())
        f, h, w = grid_sizes[0].tolist()
        Lg = f * h * w
        self.log.append(dict(x=x.clone(), remap=freq_remap.clone(), drop=sa_drop_rate))
        b, n = x.shape[:2]
        pos = freqs[freq_remap]
        q, k, v = ((x * self.w[0] + pos), (x * self.w[1] - pos), x * self.w[2])
        q, k, v = (t.view(b, n, T2V.HEADS, T2V.D).bfloat16() for t in (q, k, v))
        dense = sa_drop_rate <= 0.25
        top_k, ff = (0, 0) if dense else block_counts(Lg, sa_drop_rate)
        sp = getattr(self, "jenga_sp", None)
        if sp is not None:
            out = sp(None, q, k, v, top_k=top_k, block_neighbor_list=None if dense else block_neighbor_list,
                     p_remain_rates=p_remain_rates, first_frame_blocks=ff, dense=dense, seq_len=Lg)
        elif dense:
            out = T2V._oracle_dense(q, k, v)
        else:
            out = T2V._oracle_attn(q, k, v, top_k=top_k, text_blocks=0, block_neighbor_list=block_neighbor_list,
                                   p_remain_rates=p_remain_rates, first_frame_blocks=ff, shape_xfuse=True)
        return out.flatten(2).float() * self.w[3]

    forward.__jenga_b200__ = True


class _T2VBlock(T2V._Block):
    def __init__(self, seed, log):
        super().__init__(seed, log)
        self.self_attn = _T2VSelfAttn(seed, log)

    def forward(self, x, e, seq_lens, grid_sizes, freqs, context, context_lens, sa_drop_rate=0.0, freq_remap=None,
                block_neighbor_list=None, p_remain_rates=0.0):
        y = self.self_attn(x * (1 + e[:, 1:2]) + e[:, 0:1], seq_lens, grid_sizes, freqs, sa_drop_rate=sa_drop_rate,
                           freq_remap=freq_remap, block_neighbor_list=block_neighbor_list,
                           p_remain_rates=p_remain_rates)
        return x + y * e[:, 2:3] * self.w + context.mean(1, keepdim=True)


class _T2VModel(T2V._Model):
    def __init__(self, log, n_blocks=2):
        super().__init__(log, n_blocks)
        self.blocks = torch.nn.ModuleList([_T2VBlock(10 + 10 * i, log) for i in range(n_blocks)])


class _I2VSelfAttn(I2V._SelfAttn):
    def forward(self, x, seq_lens, grid_sizes, freqs):
        f, h, w = grid_sizes[0].tolist()
        Lg = f * h * w
        sp = getattr(self, "jenga_sp", None)
        b, n = x.shape[:2]
        remap = I2V.raster_remap(Lg, n, dist.get_rank(sp.group)) if sp is not None else torch.arange(Lg)
        pos = freqs[remap]
        q, k, v = ((x * self.w[0] + pos), (x * self.w[1] - pos), x * self.w[2])
        q, k, v = (t.view(b, n, I2V.HEADS, I2V.D).bfloat16() for t in (q, k, v))
        out = sp(None, q, k, v, dense=True, seq_len=Lg) if sp is not None else I2V._oracle_dense(q, k, v)
        return out.flatten(2).float() * self.w[3]

    forward.__jenga_b200__ = True


class _I2VBlock(I2V._Block):
    def __init__(self, seed, log):
        super().__init__(seed, log)
        self.self_attn = _I2VSelfAttn(seed, log)

    def forward(self, x, e, seq_lens, grid_sizes, freqs, context, context_lens):
        y = self.self_attn(x * (1 + e[:, 1:2]) + e[:, 0:1], seq_lens, grid_sizes, freqs)
        n = I2V.CLIP_TOKENS
        return (x + y * e[:, 2:3] * self.w + context[:, :n].mean(1, keepdim=True)
                - context[:, n:].mean(1, keepdim=True))


class _I2VModel(I2V._Model):
    def __init__(self, log, n_blocks=2):
        super().__init__(log, n_blocks)
        self.blocks = torch.nn.ModuleList([_I2VBlock(10 + 10 * i, log) for i in range(n_blocks)])


def _t2v_inputs(grid, nb):
    xs, cs = [], []
    for b in range(nb):
        x, c = T2V._inputs(grid, seed=7 + 31 * b)
        xs += x
        cs += c
    return xs, cs


def _t2v_steps(nb):
    """test_wan_sp_cpu's step kinds with nb videos and one timestep per video"""
    return [(name, drop, torch.tensor([t - 3.0 * b for b in range(nb)]), grid, before)
            for name, drop, t, grid, before in T2V._steps()]


def _t2v_run(model, fwd, nb):
    outs = []
    for name, drop, t, grid, before in _t2v_steps(nb):
        if before is not None:
            before(model)
        x, ctx = _t2v_inputs(grid, nb)
        Lg = grid[0] * grid[1] * grid[2]
        outs.append((torch.stack(fwd(x, t, ctx, Lg + 5, sa_drop_rate=drop)), model.use_cache))
    return outs


def _i2v_inputs(grid, nb):
    xs, cs, clips, ys = [], [], [], []
    for b in range(nb):
        x, c, clip, y = I2V._inputs(grid, seed=7 + 31 * b)
        xs += x
        cs += c
        clips.append(clip)
        ys += y
    return xs, cs, torch.cat(clips), ys


def _i2v_run(model, fwd, nb, P=1):
    outs = []
    for grid in I2V.GRIDS:
        model.reset()
        x, ctx, clip, y = _i2v_inputs(grid, nb)
        Lg = grid[0] * grid[1] * grid[2]
        seq_len = -(-Lg // P) * P
        for _ in range(I2V.STEPS):
            t = torch.tensor([900.0 - 5 * b for b in range(nb)])
            outs.append((torch.stack(fwd(x, t, ctx, seq_len, clip_fea=clip, y=y)), model.use_cache))
    return outs


def _worker(rank, world, port, nb, ret):
    T2V._init(rank, world, port)
    try:
        from jenga_b200 import wan_sp
        from jenga_b200.ulysses import UlyssesCarvedAttention
        model = _T2VModel([])
        sp = UlyssesCarvedAttention(attn_fn=T2V._oracle_attn, dense_fn=T2V._oracle_dense, variant="wan")
        wan_sp.parallelize_wan(model, attention=sp)
        with torch.no_grad():
            t2v = _t2v_run(model, model.forward, nb)
        i2v_model = _I2VModel([])
        sp2 = UlyssesCarvedAttention(dense_fn=I2V._oracle_dense, variant="wan")
        wan_sp.parallelize_wan_i2v(i2v_model, attention=sp2)
        with torch.no_grad():
            i2v = _i2v_run(i2v_model, i2v_model.forward, nb, world)
        ret[rank] = dict(t2v=t2v, i2v=i2v)
        # the batch rules, raised alike on every rank before any collective
        x, ctx = _t2v_inputs(T2V.GRID, nb)
        with pytest.raises(ValueError, match=f"runs batch {nb - 1}, got {nb} videos"):
            model.forward(x, torch.tensor([1.0]), ctx[1:], 3000)
        with pytest.raises(ValueError, match="one timestep per video"):
            model.forward(x, torch.ones(nb + 1), ctx, 3000)
        other = [torch.randn(T2V.C_IN, *T2V.GRID_TURBO)] + x[1:]
        with pytest.raises(ValueError, match="share one latent grid"):
            model.forward(other, torch.tensor([1.0]), ctx, 3000)
        xi, ci, clip, yi = _i2v_inputs(I2V.GRIDS[1], nb)
        with pytest.raises(ValueError, match="clip_fea holds 1 samples"):
            i2v_model.forward(xi, torch.tensor([1.0]), ci, 3000, clip_fea=clip[:1], y=yi)
        with pytest.raises(ValueError, match=f"y holds {nb - 1} conditions"):
            i2v_model.forward(xi, torch.tensor([1.0]), ci, 3000, clip_fea=clip, y=yi[1:])
        odd = [torch.randn(I2V.C_IN, *I2V.GRIDS[0])] + xi[1:]
        with pytest.raises(ValueError, match="share one latent grid"):
            i2v_model.forward(odd, torch.tensor([1.0]), ci, 3000, clip_fea=clip,
                              y=[torch.randn(I2V.C_IN, *I2V.GRIDS[0])] + yi[1:])
    finally:
        dist.destroy_process_group()


def _single_t2v(nb):
    model = _T2VModel([])
    with torch.no_grad():
        return _t2v_run(model, lambda *a, **k: T2V._teacache_single(model, *a, **k), nb)


def _single_i2v(nb):
    model = _I2VModel([])
    with torch.no_grad():
        return _i2v_run(model, lambda *a, **k: I2V._i2v_teacache_single(model, *a, **k), nb)


def _alone(steps_out, kinds, b, run_alone):
    """sample b of every computed step against the same step run with sample b alone"""
    for i, ((o, used), (o1, used1)) in enumerate(zip(steps_out, run_alone)):
        if kinds[i]:
            assert not used and not used1
            assert torch.equal(o[b], o1[0]), (b, i)


@pytest.mark.parametrize("nb", [2, 3])
def test_sharded_forwards_batch_equals_single_process_and_each_sample_alone(nb):
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    port = 29500 + (os.getpid() + 53 * nb) % 2000
    mp.spawn(_worker, args=(world, port, nb, ret), nprocs=world, join=True)

    t2v_ref, i2v_ref = _single_t2v(nb), _single_i2v(nb)
    assert [u for _, u in t2v_ref] == [False, False, True, False, False]
    assert [u for _, u in i2v_ref] == [False, False, True] * len(I2V.GRIDS)
    for r in range(world):
        for name, ref in (("t2v", t2v_ref), ("i2v", i2v_ref)):
            for i, ((o, used), (o_ref, used_ref)) in enumerate(zip(ret[r][name], ref)):
                assert used == used_ref and o.shape[0] == nb, (name, r, i)
                assert torch.equal(o, o_ref), (name, r, i)
    # computed steps: each sample is that sample run alone (its own video, context and timestep)
    for b in range(nb):
        m = _T2VModel([])
        with torch.no_grad():
            alone = []
            for name, drop, t, grid, before in _t2v_steps(nb):
                if before is not None:
                    before(m)
                x, ctx = _t2v_inputs(grid, nb)
                Lg = grid[0] * grid[1] * grid[2]
                alone.append((torch.stack(T2V._teacache_single(m, [x[b]], t[b:b + 1], [ctx[b]], Lg + 5,
                                                               sa_drop_rate=drop)), m.use_cache))
        # the skipped step depends on the batch's rel-L1 (one decision per call); steps 0, 1, 3, 4 are computed
        _alone(t2v_ref, [True, True, False, True, True], b, alone)
        mi = _I2VModel([])
        with torch.no_grad():
            alone = []
            for grid in I2V.GRIDS:
                mi.reset()
                x, ctx, clip, y = _i2v_inputs(grid, nb)
                Lg = grid[0] * grid[1] * grid[2]
                for _ in range(I2V.STEPS):
                    t = torch.tensor([900.0 - 5 * b])
                    alone.append((torch.stack(I2V._i2v_teacache_single(mi, [x[b]], t, [ctx[b]], Lg,
                                                                       clip_fea=clip[b:b + 1], y=[y[b]])),
                                  mi.use_cache))
        _alone(i2v_ref, [True, True, False] * len(I2V.GRIDS), b, alone)
