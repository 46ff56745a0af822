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
"""
from __future__ import annotations

import types

import numpy as np
import torch
import torch.distributed as dist

from .hyi2v_sp import check_degree, default_attention, shard

MODEL = "Wan2.1"
MAX_WORLD = 8        # the peer arrays of the fused exchange and of the attention epilogue


def _check_world(heads: int, world: int) -> None:
    check_degree(0, heads, world, model=MODEL)
    if world > MAX_WORLD:
        raise ValueError(f"sequence-parallel {MODEL}: {world} ranks; the Ulysses exchange is built for at "
                         f"most {MAX_WORLD} (one NVLink box)")


def shard_rows(L: int, world: int, rank: int) -> tuple[int, int]:
    """(n, real): rows per rank, n = ceil(L / world), and how many of rank `rank`'s n rows are real.
    Raises when some rank would hold no real row."""
    n = -(-L // world)
    if L - (world - 1) * n <= 0:
        raise ValueError(f"sequence-parallel {MODEL}: {L} tokens over {world} ranks leave the last rank "
                         f"without a real row ({n} rows per rank)")
    return n, max(0, min(n, L - rank * n))


def _sinusoidal_embedding_1d(model):
    """model_mul.py:16-27, the reference forward's time embedding: the function in the globals of the
    model class's own unpatchify (which jenga_wan.py never replaces)"""
    return type(model).unpatchify.__globals__["sinusoidal_embedding_1d"]


def _rel_l1_from_rank0(value: torch.Tensor, group) -> float:
    """Rank 0's rel-L1 scalar on every rank.  Each rank computes its own (the modulated inputs are
    replicated, but nothing guarantees bit-equal reductions across devices); all ranks then accumulate
    the same number and take the same branch, so no rank skips the blocks while another enters the
    exchange."""
    v = value.reshape(1).clone()
    dist.broadcast(v, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    return v.cpu().item()


def parallelize_wan(model, group=None, attention=None):
    """Replaces `model.forward` (an instance attribute, as WanT2V(use_usp=True) binds usp_dit_forward)
    with the sharded TeaCache forward and sets `block.self_attn.jenga_sp = attention` on every block.
    attention: a Ulysses object with the hybrid_seq_parallel_attn call contract and the seq_len /
    dense / first_frame_blocks keywords; None means default_attention(group, "wan").  Returns it."""
    if not dist.is_initialized():
        raise RuntimeError(f"sequence-parallel {MODEL} needs an initialised process group")
    P = dist.get_world_size(group)
    _check_world(int(model.num_heads), P)
    for block in model.blocks:
        sa = block.self_attn
        # an unpatched self-attention ignores jenga_sp: every rank would attend over its own rows alone
        if not getattr(type(sa).forward, "__jenga_b200__", False):
            raise RuntimeError(f"{type(sa).__module__}.{type(sa).__name__}.forward is not the fused "
                               "jenga_b200 forward: install() (fused_blocks=True) must run before the Wan "
                               "model module is imported")
        inst = sa.__dict__.get("forward")
        if inst is not None and not getattr(getattr(inst, "__func__", inst), "__jenga_b200__", False):
            raise RuntimeError(f"{type(sa).__name__} has an instance forward ({getattr(inst, '__name__', inst)}) "
                               "that is not the jenga_b200 one: it would run instead of the sharded "
                               "self-attention (install(wan_sp=True) swaps usp_attn_forward)")
    sp = attention if attention is not None else default_attention(group, variant="wan")
    for block in model.blocks:
        block.self_attn.jenga_sp = sp
    model.forward = types.MethodType(_forward_factory(group), model)
    return sp


def _forward_factory(group):
    def forward(self, x, t, context, seq_len, clip_fea=None, y=None, sa_drop_rate=0.0):
        """jenga_wan.py:503-664 (teacache_forward) on this rank's Hilbert rows; returns the full output
        on every rank"""
        P, r = dist.get_world_size(group), dist.get_rank(group)
        for name in ("hilbert_order", "linear_to_hilbert"):
            if getattr(self, name, None) is None:
                raise RuntimeError(f"sequence-parallel {MODEL}: model.{name} is not set (jenga_wan.py sets "
                                   "the Jenga curve attributes before sampling)")
        if self.model_type == 'i2v':
            assert clip_fea is not None and y is not None
        if len(x) != 1:
            raise ValueError(f"sequence-parallel {MODEL} runs batch 1, got {len(x)} videos")
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
        # the reference pads to the sp_size-rounded seq_len and the Hilbert gather drops those rows
        # again (:554-559): gathering from the unpadded rows gives the same rows
        order = self.hilbert_order
        L = len(order)
        if L != int(seq_lens[0]):
            raise ValueError(f"sequence-parallel {MODEL}: hilbert_order has {L} entries for a latent of "
                             f"{int(seq_lens[0])} tokens (curve and grid out of step)")
        n, real = shard_rows(L, P, r)
        rows = shard(order.to(torch.long), 0, P, r)          # pad entries point at row 0 (any valid row)
        x = x[:, rows.to(x.device)]
        if real < n:
            x[:, real:] = 0
        freq_remap = rows.to(device)
        # time embeddings (:561-566)
        with torch.autocast("cuda", dtype=torch.float32, enabled=device.type == "cuda"):
            e = self.time_embedding(_sinusoidal_embedding_1d(self)(self.freq_dim, t).float())
            e0 = self.time_projection(e).unflatten(1, (6, self.dim))
            assert e.dtype == torch.float32 and e0.dtype == torch.float32
        # context (:568-579)
        context_lens = None
        context = self.text_embedding(torch.stack([
            torch.cat([u, u.new_zeros(self.text_len - u.size(0), u.size(1))]) for u in context]))
        if clip_fea is not None:
            context_clip = self.img_emb(clip_fea)
            context = torch.concat([context_clip, context], dim=1)
        kwargs = dict(e=e0, seq_lens=seq_lens, grid_sizes=grid_sizes, freqs=self.freqs, context=context,
                      context_lens=context_lens, sa_drop_rate=sa_drop_rate, freq_remap=freq_remap,
                      block_neighbor_list=self.block_neighbor_list, p_remain_rates=self.p_remain_rates)
        if self.enable_teacache:
            # :595-626, with rank 0's rel-L1 value on every rank
            modulated_inp = e0 if self.use_ref_steps else e
            even = self.cnt % 2 == 0
            self.is_even = even
            sfx = "even" if even else "odd"
            prev = getattr(self, "previous_e0_" + sfx)
            if self.cnt < self.ret_steps or self.cnt >= self.cutoff_steps or self.stage_start:
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
            # :628-648; each rank keeps the residual of its own rows
            if not should_calc:
                x += getattr(self, "previous_residual_" + sfx)
                self.use_cache = True
            else:
                ori_x = x.clone()
                for block in self.blocks:
                    x = block(x, **kwargs)
                setattr(self, "previous_residual_" + sfx, x - ori_x)
                self.use_cache = False
        else:
            for block in self.blocks:
                x = block(x, **kwargs)
        # head on the rank's rows (row-local, as usp_dit_forward runs it before its gather), then the
        # [1, n, out] rows of every rank in rank order
        x = self.head(x, e)
        parts = [torch.empty_like(x) for _ in range(P)]
        dist.all_gather(parts, x.contiguous(), group=group)
        x = torch.cat(parts, dim=1)[:, :L]
        x = x[:, self.linear_to_hilbert]                                      # :655
        x = self.unpatchify(x, grid_sizes)
        self.cnt += 1
        if self.cnt >= self.num_steps:
            self.cnt = 0
        return [u.float() for u in x]
    return forward


# ------------------------------------------------------------------------------------------------
# install(wan_sp=True): wan.distributed.xdit_context_parallel
# ------------------------------------------------------------------------------------------------
def _is_jenga_model(model) -> bool:
    """jenga_wan.py sets the curve attributes on the T2V model class before sampling (:1077-1082);
    it never does for WanI2V"""
    return getattr(model, "hilbert_order", None) is not None and getattr(model, "linear_to_hilbert", None) is not None


def install_usp(xdit_module) -> bool:
    """Swaps usp_dit_forward / usp_attn_forward of wan.distributed.xdit_context_parallel, which
    WanT2V(use_usp=True) binds to the model and to every self-attention module (text2video.py:88-99):

      usp_dit_forward   the sharded TeaCache forward; takes sa_drop_rate and calls parallelize_wan on
                        its first call.  A model without the Jenga curve attributes (WanI2V) runs the
                        reference function.
      usp_attn_forward  takes WanSelfAttention.forward's Jenga signature and defers to the patched class
                        forward under jenga_sp; a module without jenga_sp runs the reference function.

    Returns False when there is nothing to swap or it is already swapped."""
    orig_dit = getattr(xdit_module, "usp_dit_forward", None)
    orig_attn = getattr(xdit_module, "usp_attn_forward", None)
    if orig_dit is None or orig_attn is None or getattr(orig_dit, "__jenga_b200__", False):
        return False

    def usp_dit_forward(self, x, t, context, seq_len, *args, **kwargs):
        # the sharded forward's signature: (x, t, context, seq_len, clip_fea=None, y=None, sa_drop_rate=0.0)
        if not _is_jenga_model(self):
            return orig_dit(self, x, t, context, seq_len, *args, **kwargs)
        # first call: parallelize_wan replaces this bound method by the sharded forward
        parallelize_wan(self)
        return self.forward(x, t, context, seq_len, *args, **kwargs)

    def usp_attn_forward(self, x, seq_lens, grid_sizes, freqs, *args, **kwargs):
        # WanSelfAttention.forward(x, seq_lens, grid_sizes, freqs, sa_drop_rate, per_block_tokens,
        # p_remain_rates, freq_remap, block_neighbor_list) under jenga_sp
        if getattr(self, "jenga_sp", None) is None:
            return orig_attn(self, x, seq_lens, grid_sizes, freqs, *args, **kwargs)
        return type(self).forward(self, x, seq_lens, grid_sizes, freqs, *args, **kwargs)

    for fn, orig in ((usp_dit_forward, orig_dit), (usp_attn_forward, orig_attn)):
        fn.__jenga_b200__ = True
        fn.__wrapped__ = orig
    usp_dit_forward.__doc__ = "jenga_b200: Hilbert-sharded TeaCache forward over the Ulysses exchange"
    usp_attn_forward.__doc__ = "jenga_b200: the patched WanSelfAttention.forward under jenga_sp"
    xdit_module.usp_dit_forward = usp_dit_forward
    xdit_module.usp_attn_forward = usp_attn_forward
    return True


def uninstall_usp(xdit_module) -> None:
    """Puts the reference's usp_dit_forward / usp_attn_forward back"""
    for name in ("usp_dit_forward", "usp_attn_forward"):
        fn = getattr(xdit_module, name, None)
        if getattr(fn, "__jenga_b200__", False):
            setattr(xdit_module, name, fn.__wrapped__)
