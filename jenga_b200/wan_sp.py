"""Sequence-parallel Wan2.1 T2V forward on the carved path.

The reference's Wan sequence parallelism (`WanT2V(use_usp=True)`, wan/text2video.py:88-99) binds
usp_dit_forward / usp_attn_forward (wan/distributed/xdit_context_parallel.py:66-147) to the model and
to every self-attention module.  Those instance attributes shadow the TeaCache forward jenga_wan.py
installs on the class, usp_dit_forward has no `sa_drop_rate`, and the tokens are chunked in raster
order for a dense attention: no curve order, no carving, no TeaCache.  `parallelize_wan` replaces the
model's forward with a restatement of jenga_wan.py:503-664 (`teacache_forward`) sharded over the
Hilbert order:

  embeddings (replicated) -> rank r gathers its Hilbert rows [r*n, min((r+1)*n, L)), n = ceil(L/P),
  zero-padded to n rows; `freq_remap` is the same slice of hilbert_order -> TeaCache decision (rank
  0's rel-L1 value, broadcast) -> blocks, whose self-attention (blocks._wan_self) routes through
  `block.self_attn.jenga_sp`, a Ulysses object, over the first L exchanged rows -> head on the rank's
  rows -> one all_gather of the [1, n, out_dim] rows in rank order -> [:L], inverse Hilbert scatter,
  unpatchify.

The result is the single-GPU Jenga Wan forward's: the same selection over the global L, the same
dense warm-up steps, the same TeaCache decisions.  Only the Linears run on a rank's rows.

Wan2.1-I2V loads the plain model of wan/modules/model.py (image2video.py:21,99), whose blocks take no
Jenga arguments and whose self-attention is dense in every step.  `parallelize_wan_i2v` replaces its
forward with a restatement of usp_dit_forward (xdit_context_parallel.py:66-146) plus the TeaCache
state machine of teacache_forward:

  embeddings, CLIP + text context (replicated) -> rank r takes the raster rows [r*n, min((r+1)*n, L)),
  zero-padded to n (no curve: the attention is dense, and raster order keeps RoPE a plain slice) ->
  TeaCache decision (rank 0's rel-L1 value) -> blocks, whose self-attention (blocks._wan_i2v_self) runs
  the dense class over the first L exchanged rows and whose cross-attention is the fused I2V kernel on
  the rank's rows -> head on the rank's rows -> one all_gather -> [:L], unpatchify.

Unlike the reference's USP, which attends to the zero pad rows of seq_len (its TODO at
xdit_context_parallel.py:172-187), the pad keys are excluded, as the single-GPU
flash_attention(k_lens=seq_lens) excludes them.

On one GPU (`bind_wan_i2v`, which install()'s hook calls for WanI2V(use_usp=False)) the same I2V forward
runs with group LOCAL: one rank, no exchange.  jenga_wan.py binds teacache_forward to the I2V model too,
which cannot run on it (no curve attributes, and model.py's blocks take no Jenga arguments); the
instance attribute shadows it.  Its self-attention is the fused prologue and the dense class over the L
raster rows.

Carving (opt-in, I2V_SA_DROP_RATES: install(wan_i2v_sa_drop_rates=...) / JENGA_WAN_I2V_SA_DROP) makes
both I2V forwards follow teacache_forward's T2V rules: the rows in the sliced Gilbert order of the
forward's own grid (i2v_curve; on P ranks each rank takes its slice, as parallelize_wan does),
freq_remap = that order in every step, the drop rate of t2v_generate's schedule (sa_drop_schedule), the
Wan operator with first_frame_blocks above 0.25 and the dense class below; then the head, the inverse
scatter and unpatchify.  Both T2V and I2V forwards run one body, _sharded_forward.
"""
from __future__ import annotations

import functools
import types

import numpy as np
import torch
import torch.distributed as dist

from . import sharding
from .sharding import LOCAL, check_fused_blocks, default_attention, gather_rows, shard, world

MODEL = "Wan2.1"
# the Wan degree rule, (heads, world), and the rows per rank, (L, world, rank) -> (n, real)
_check_world = functools.partial(sharding.check_world, model=MODEL)
shard_rows = functools.partial(sharding.shard_rows, model=MODEL)


def _route(group) -> str:
    return "single-GPU " if group is LOCAL else "sequence-parallel "


def _sinusoidal_embedding_1d(model):
    """model_mul.py:16-27, the reference forward's time embedding: the function in the globals of the
    model class's own unpatchify (which jenga_wan.py never replaces)"""
    return type(model).unpatchify.__globals__["sinusoidal_embedding_1d"]


def _rel_l1_from_rank0(value: torch.Tensor, group) -> float:
    """Rank 0's rel-L1 scalar on every rank.  Each rank computes its own (the modulated inputs are
    replicated, but nothing guarantees bit-equal reductions across devices); all ranks then accumulate
    the same number and take the same branch, so no rank skips the blocks while another enters the
    exchange."""
    if group is LOCAL:
        return value.cpu().item()
    v = value.reshape(1).clone()
    dist.broadcast(v, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    return v.cpu().item()


def parallelize_wan(model, group=None, attention=None):
    """Replaces `model.forward` (an instance attribute, as WanT2V(use_usp=True) binds usp_dit_forward)
    with the sharded TeaCache forward and sets `block.self_attn.jenga_sp = attention` on every block.
    attention: a Ulysses object with the hybrid_seq_parallel_attn call contract and the seq_len /
    dense / first_frame_blocks keywords; None means default_attention(group, "wan").  Returns it."""
    return _parallelize(model, group, attention, "install() (fused_blocks=True)", _forward_factory)


def _parallelize(model, group, attention, install_call: str, forward_factory):
    """The checks (the degree, and a fused, unshadowed self-attention in every block), then jenga_sp on
    every block and the forward of forward_factory(group) on the model"""
    if not dist.is_initialized():
        raise RuntimeError(f"sequence-parallel {MODEL} needs an initialised process group")
    _check_world(int(model.num_heads), dist.get_world_size(group))
    check_fused_blocks([block.self_attn for block in model.blocks], "Wan", install_call)
    sp = attention if attention is not None else default_attention(group, "wan")
    for block in model.blocks:
        block.self_attn.jenga_sp = sp
    model.forward = types.MethodType(forward_factory(group), model)
    return sp


def _teacache(self, x, e, e0, run_blocks, group):
    """jenga_wan.py:595-652: the TeaCache step decision around `run_blocks` (x -> x after every block),
    with rank 0's rel-L1 value on every rank.  Each rank keeps the residual of its own rows.  stage_start
    is read as False where the model has none (jenga_wan.py sets it on the T2V model only)."""
    if not getattr(self, "enable_teacache", False):     # a model jenga_wan.py has not set up
        return run_blocks(x)
    # :595-626
    modulated_inp = e0 if self.use_ref_steps else e
    even = self.cnt % 2 == 0
    self.is_even = even
    sfx = "even" if even else "odd"
    prev = getattr(self, "previous_e0_" + sfx)
    if self.cnt < self.ret_steps or self.cnt >= self.cutoff_steps or getattr(self, "stage_start", False):
        should_calc = True
        setattr(self, "accumulated_rel_l1_distance_" + sfx, 0)
    else:
        rescale_func = np.poly1d(self.coefficients)
        rel = _rel_l1_from_rank0((modulated_inp - prev).abs().mean() / prev.abs().mean(), group)
        acc = getattr(self, "accumulated_rel_l1_distance_" + sfx) + rescale_func(rel)
        setattr(self, "accumulated_rel_l1_distance_" + sfx, acc)
        if acc < self.teacache_thresh:
            should_calc = False
        else:
            should_calc = True
            setattr(self, "accumulated_rel_l1_distance_" + sfx, 0)
    setattr(self, "previous_e0_" + sfx, modulated_inp.clone())
    # :628-648
    if not should_calc:
        x += getattr(self, "previous_residual_" + sfx)
        self.use_cache = True
    else:
        ori_x = x.clone()
        x = run_blocks(x)
        setattr(self, "previous_residual_" + sfx, x - ori_x)
        self.use_cache = False
    return x


def _forward_factory(group):
    def forward(self, x, t, context, seq_len, clip_fea=None, y=None, sa_drop_rate=0.0):
        """jenga_wan.py:503-664 (teacache_forward) on this rank's Hilbert rows; returns the full output
        on every rank"""
        for name in ("hilbert_order", "linear_to_hilbert"):
            if getattr(self, name, None) is None:
                raise RuntimeError(f"sequence-parallel {MODEL}: model.{name} is not set (jenga_wan.py sets "
                                   "the Jenga curve attributes before sampling)")
        if self.model_type == 'i2v':
            assert clip_fea is not None and y is not None
        curve = (self.hilbert_order, self.linear_to_hilbert, self.block_neighbor_list)
        return _sharded_forward(self, group, x, t, context, seq_len, clip_fea, y, lambda grid: curve,
                                dict(sa_drop_rate=sa_drop_rate, p_remain_rates=self.p_remain_rates))
    return forward


def _sharded_forward(self, group, x, t, context, seq_len, clip_fea, y, curve_of, block_kw):
    """The body both Wan forwards share.  curve_of(grid) -> (hilbert_order, linear_to_hilbert,
    block_neighbor_list) or None: rank r takes the curve's rows [r*n, min((r+1)*n, L)) and `freq_remap`
    is that slice, or, without a curve, the raster rows.  block_kw: what the blocks get besides the
    arguments of model.py's WanAttentionBlock.forward (with a curve, also freq_remap and
    block_neighbor_list).  group LOCAL: one GPU, no exchange."""
    P, r = world(group)
    if len(x) != 1:
        raise ValueError(f"{_route(group)}{MODEL} runs batch 1, got {len(x)} videos")
    device = self.patch_embedding.weight.device
    if self.freqs.device != device:
        self.freqs = self.freqs.to(device)
    if y is not None:
        x = [torch.cat([u, v], dim=0) for u, v in zip(x, y)]
    # embeddings (replicated)
    x = [self.patch_embedding(u.unsqueeze(0)) for u in x]
    grid_sizes = torch.stack([torch.tensor(u.shape[2:], dtype=torch.long) for u in x])
    x = [u.flatten(2).transpose(1, 2) for u in x]
    seq_lens = torch.tensor([u.size(1) for u in x], dtype=torch.long)
    assert seq_lens.max() <= seq_len
    x = x[0]
    # rows past L (the reference's zero pad to seq_len, which the Hilbert gather drops again,
    # jenga_wan.py:554-559) are neither attended nor returned
    L = int(seq_lens[0])
    curve = curve_of(tuple(grid_sizes[0].tolist()))
    kwargs = dict(block_kw)
    if curve is None:
        shard_rows(L, P, r)                                  # raises when a rank holds no real row
        x = shard(x, 1, P, r)
    else:
        order = curve[0]
        if len(order) != L:
            raise ValueError(f"sequence-parallel {MODEL}: hilbert_order has {len(order)} entries for a latent "
                             f"of {L} tokens (curve and grid out of step)")
        n, real = shard_rows(L, P, r)
        rows = shard(order.to(torch.long), 0, P, r)          # pad entries point at row 0 (any valid row)
        x = x[:, rows.to(x.device)]
        if real < n:
            x[:, real:] = 0
        kwargs.update(freq_remap=rows.to(device), block_neighbor_list=curve[2])
    e, e0, context = _time_and_context(self, t, context, clip_fea)
    kwargs.update(e=e0, seq_lens=seq_lens, grid_sizes=grid_sizes, freqs=self.freqs, context=context,
                  context_lens=None)
    x = _teacache(self, x, e, e0, lambda x: _blocks(self, x, kwargs), group)
    # head on the rank's rows (row-local, as usp_dit_forward runs it before its gather), then the
    # [1, n, out] rows of every rank in rank order
    x = gather_rows(self.head(x, e), L, P, group)
    if curve is not None:
        x = x[:, curve[1]]                                                    # :655
    x = self.unpatchify(x, grid_sizes)
    if getattr(self, "num_steps", None) is not None:     # the TeaCache step counter, where jenga_wan.py set one
        self.cnt += 1
        if self.cnt >= self.num_steps:
            self.cnt = 0
    return [u.float() for u in x]


def _blocks(self, x, kwargs):
    for block in self.blocks:
        x = block(x, **kwargs)
    return x


def _time_and_context(self, t, context, clip_fea):
    """(e, e0, context) of jenga_wan.py:561-579, replicated on every rank"""
    device = self.patch_embedding.weight.device
    with torch.autocast("cuda", dtype=torch.float32, enabled=device.type == "cuda"):
        e = self.time_embedding(_sinusoidal_embedding_1d(self)(self.freq_dim, t).float())
        e0 = self.time_projection(e).unflatten(1, (6, self.dim))
        assert e.dtype == torch.float32 and e0.dtype == torch.float32
    context = self.text_embedding(torch.stack([
        torch.cat([u, u.new_zeros(self.text_len - u.size(0), u.size(1))]) for u in context]))
    if clip_fea is not None:
        context = torch.concat([self.img_emb(clip_fea), context], dim=1)
    return e, e0, context


# ------------------------------------------------------------------------------------------------
# Wan2.1-I2V: carving (opt-in), the single-GPU forward, the sharded forward
# ------------------------------------------------------------------------------------------------
I2V_P_REMAIN_DEFAULT = 0.8      # model_mul.py's WanSelfAttention.forward default
# the carved self-attention of Wan2.1-I2V: () is dense (the default), else the rates of
# jenga_wan.py --sa_drop_rates; set by install() (JENGA_WAN_I2V_SA_DROP / JENGA_WAN_I2V_P_REMAIN)
I2V_SA_DROP_RATES: tuple = ()
I2V_P_REMAIN = I2V_P_REMAIN_DEFAULT


def parse_sa_drop_rates(value) -> tuple:
    """"d0[,d1]" (or a sequence of one or two numbers) -> (d0[, d1]); "" or None -> () (dense).  Each
    rate is a drop rate in [0, 1): a rate of 1 would keep no key block."""
    if value is None:
        return ()
    parts = [p.strip() for p in value.split(",")] if isinstance(value, str) else list(value)
    if parts == [""]:
        return ()
    try:
        rates = tuple(float(p) for p in parts)
    except (TypeError, ValueError):
        raise ValueError(f"Wan2.1-I2V sa_drop_rates {value!r}: expected one or two numbers, 'd0[,d1]'") from None
    if not 1 <= len(rates) <= 2 or not all(0.0 <= d < 1.0 for d in rates):
        raise ValueError(f"Wan2.1-I2V sa_drop_rates {value!r}: expected one or two drop rates in [0, 1), 'd0[,d1]'")
    return rates


def parse_p_remain(value) -> float:
    """The p_remain_rates of the carved steps: a number in (0, 1]; "" or None -> 0.8."""
    if value is None or (isinstance(value, str) and not value.strip()):
        return I2V_P_REMAIN_DEFAULT
    try:
        p = float(value)
    except (TypeError, ValueError):
        raise ValueError(f"Wan2.1-I2V p_remain {value!r}: expected a number in (0, 1]") from None
    if not 0.0 < p <= 1.0:
        raise ValueError(f"Wan2.1-I2V p_remain {value!r}: expected a number in (0, 1]")
    return p


def set_i2v_carving(sa_drop_rates=None, p_remain=None) -> None:
    """Turns the carved Wan2.1-I2V self-attention on (rates given) or off (None / "") for every I2V
    forward of this module, on one GPU and sharded.  Malformed values raise and change nothing."""
    global I2V_SA_DROP_RATES, I2V_P_REMAIN
    rates, p = parse_sa_drop_rates(sa_drop_rates), parse_p_remain(p_remain)
    I2V_SA_DROP_RATES, I2V_P_REMAIN = rates, p


def sa_drop_schedule(cnt: int, num_steps: int, rates) -> float:
    """The drop rate of t2v_generate (jenga_wan.py:189-206) for model call `cnt` of `num_steps`
    (TeaCache counts the conditional and the unconditional call: sampling step cnt // 2 of
    num_steps // 2): d0 up to step 25, then d1 (d0 with one rate), warmed up as
    min(d, step / (steps - 1) * 10 * d).  The blocks run the dense class at <= 0.25."""
    steps, idx = num_steps // 2, cnt // 2
    if steps < 2:
        raise ValueError(f"the Wan drop-rate schedule needs at least two sampling steps, got {steps}")
    d = rates[0] if idx <= 25 or len(rates) == 1 else rates[1]
    return min(d, idx / (steps - 1) * 10 * d)


@functools.lru_cache(maxsize=8)
def i2v_curve(f: int, h: int, w: int):
    """(linear_to_hilbert, hilbert_order, block_neighbor_list) of the latent grid f x h x w: the sliced
    Gilbert curve and its 128-token block adjacency that jenga_wan.py builds for T2V (:1013-1035) from
    sliced_gilbert_mapping / sliced_gilbert_block_neighbor_mapping, here from the grid the forward sees
    (the I2V grid follows the image's aspect ratio, image2video.py:180-193)."""
    from . import gilbert
    l2h, h2l = gilbert.mapping_tensors(f, h, w, sliced=True)
    return l2h, h2l, gilbert.block_neighbor_mapping(f, h, w, sliced=True)


def parallelize_wan_i2v(model, group=None, attention=None):
    """Replaces `model.forward` of a Wan2.1-I2V model of wan/modules/model.py (an instance attribute, as
    WanI2V(use_usp=True) binds usp_dit_forward) with the sharded I2V forward, and sets
    `block.self_attn.jenga_sp = attention` on every block.  The blocks must carry the forwards
    install(wan_sp=True) hooks into that module.  attention: a Ulysses object with the
    hybrid_seq_parallel_attn call contract and the seq_len / dense / first_frame_blocks keywords; None
    means default_attention(group, "wan").  Returns it."""
    return _parallelize(model, group, attention, "install(wan_sp=True)", _i2v_forward_factory)


def bind_wan_i2v(model) -> None:
    """The single-GPU Wan2.1-I2V route: hooks the block classes of the model's module (wan/modules/model.py)
    and binds the one-GPU I2V forward as `model.forward`, an instance attribute that shadows the
    teacache_forward jenga_wan.py puts on the class."""
    from . import blocks
    # the classes the model's blocks are built from (wan/modules/model.py's)
    blk = model.blocks[0]
    blocks.patch_plain_wan(types.SimpleNamespace(__name__=type(blk).__module__, WanAttentionBlock=type(blk),
                                                 WanSelfAttention=type(blk.self_attn)))
    model.forward = types.MethodType(_i2v_forward_factory(LOCAL), model)


def _i2v_forward_factory(group):
    def forward(self, x, t, context, seq_len, clip_fea=None, y=None):
        """usp_dit_forward (xdit_context_parallel.py:66-146) with teacache_forward's step cache, on this
        rank's rows (all rows on one GPU); returns the full output on every rank.  Dense over the raster
        rows by default; with I2V_SA_DROP_RATES set, teacache_forward's Hilbert order and carved
        self-attention (jenga_wan.py:559,583-592,655) with the drop rate of sa_drop_schedule."""
        if clip_fea is None or y is None:
            raise ValueError(f"{_route(group)}{MODEL}-I2V needs clip_fea and y")
        rates = I2V_SA_DROP_RATES
        if rates:
            if getattr(self, "num_steps", None) is None:
                raise RuntimeError(f"{MODEL}-I2V carving follows the sampling step: the model needs the TeaCache "
                                   "step counter (cnt, num_steps) that jenga_wan.py sets")
            block_kw = dict(sa_drop_rate=sa_drop_schedule(self.cnt, self.num_steps, rates),
                            p_remain_rates=I2V_P_REMAIN)
            return _sharded_forward(self, group, x, t, context, seq_len, clip_fea, y, lambda grid: i2v_curve(*grid),
                                    block_kw)
        # one GPU: sa_drop_rate 0 on raster rows sends the self-attention to the fused dense call
        block_kw = dict(sa_drop_rate=0.0) if group is LOCAL else {}
        return _sharded_forward(self, group, x, t, context, seq_len, clip_fea, y, lambda grid: None, block_kw)
    return forward


# ------------------------------------------------------------------------------------------------
# install(wan_sp=True): wan.distributed.xdit_context_parallel
# ------------------------------------------------------------------------------------------------
def _is_jenga_model(model) -> bool:
    """jenga_wan.py sets the curve attributes on the T2V model class before sampling (:1077-1082);
    it never does for WanI2V"""
    return getattr(model, "hilbert_order", None) is not None and getattr(model, "linear_to_hilbert", None) is not None


def install_usp(xdit_module) -> list[str]:
    """Swaps usp_dit_forward / usp_attn_forward of wan.distributed.xdit_context_parallel, which
    WanT2V(use_usp=True) binds to the model and to every self-attention module (text2video.py:88-99):

      usp_dit_forward   the sharded TeaCache forward: on its first call parallelize_wan_i2v for an I2V
                        model (WanI2V, wan/modules/model.py), else parallelize_wan for a model with the
                        Jenga curve attributes (WanT2V under jenga_wan.py; takes sa_drop_rate).  Any
                        other model runs the reference function.
      usp_attn_forward  takes either WanSelfAttention.forward signature and defers to the patched class
                        forward under jenga_sp; a module without jenga_sp runs the reference function.

    Returns what it swapped: nothing when there is nothing to swap or it is already swapped."""
    from .blocks import _swap
    orig_dit = getattr(xdit_module, "usp_dit_forward", None)
    orig_attn = getattr(xdit_module, "usp_attn_forward", None)
    if orig_attn is None:
        return []

    def usp_dit_forward(self, x, t, context, seq_len, *args, **kwargs):
        """jenga_b200: sharded TeaCache forward over the Ulysses exchange"""
        # the sharded forwards' signatures: (x, t, context, seq_len, clip_fea=None, y=None[, sa_drop_rate=0.0])
        # first call: parallelize_wan_i2v / parallelize_wan replaces this bound method by the sharded forward
        if getattr(self, "model_type", None) == "i2v":
            parallelize_wan_i2v(self)
        elif _is_jenga_model(self):
            parallelize_wan(self)
        else:
            return orig_dit(self, x, t, context, seq_len, *args, **kwargs)
        return self.forward(x, t, context, seq_len, *args, **kwargs)

    def usp_attn_forward(self, x, seq_lens, grid_sizes, freqs, *args, **kwargs):
        """jenga_b200: the patched WanSelfAttention.forward under jenga_sp"""
        # WanSelfAttention.forward(x, seq_lens, grid_sizes, freqs, sa_drop_rate, per_block_tokens,
        # p_remain_rates, freq_remap, block_neighbor_list) of model_mul.py, or (x, seq_lens, grid_sizes,
        # freqs) of model.py, under jenga_sp
        if getattr(self, "jenga_sp", None) is None:
            return orig_attn(self, x, seq_lens, grid_sizes, freqs, *args, **kwargs)
        return type(self).forward(self, x, seq_lens, grid_sizes, freqs, *args, **kwargs)

    ok = (_swap(xdit_module, "usp_dit_forward", usp_dit_forward)
          and _swap(xdit_module, "usp_attn_forward", usp_attn_forward))
    return [f"{xdit_module.__name__}.usp_dit_forward", f"{xdit_module.__name__}.usp_attn_forward"] if ok else []
