"""Sequence-parallel HunyuanVideo-I2V transformer forward on the carved path.

The reference's I2V sequence parallelism (hyvideo_i2v/inference.py:110-173, parallelize_transformer)
chunks the latent by height or width BEFORE the Hilbert reorder and runs xfuser's dense attention,
so neither the curve order nor the 128-token blocks that AttenCarve selects from exist under it.
`parallelize_i2v` replaces the transformer's forward with a restatement of jenga_hyi2v.py:53-221
(`ra_forward`) sharded the way jenga_hyvideo_multigpu.py:104-331 shards HunyuanVideo T2V:

  embed (replicated) -> Hilbert gather of img, freqs_cos, freqs_sin over the FULL sequence
  -> first-frame masks (jenga_hyi2v.py:122-130) -> rank r keeps the contiguous Hilbert slice
  [r*L/P, (r+1)*L/P) of the image rows, of both RoPE tables and of the first-frame mask; the text
  rows are replicated -> double / single blocks, whose fused I2V forwards (blocks.py) route the
  attention through `block.jenga_sp`, a Ulysses object -> all-gather of the image rows in rank
  order -> inverse Hilbert scatter, final_layer, unpatchify (replicated).

The result is the single-GPU Jenga I2V forward's: same selection rule, same token replace, same
step skipping.  Only the Linears run on a rank's rows instead of all rows.
"""
from __future__ import annotations

import functools
import types

import torch
import torch.distributed as dist

from . import sharding
from .sharding import check_fused_blocks, default_attention, gather_rows, shard, world

MODEL = "HunyuanVideo-I2V"
# jenga_hyi2v.py:32 — the denoising steps that run the block loop; every other step adds the
# residual of the last computed step
STEP_CALC = (0, 1, 2, 3, 5, 7, 10, 13, 16, 19, 22, 25, 28, 31, 34, 37, 40, 42, 44, 45, 46, 47, 48, 49)
# check_degree(img_tokens, heads, world): whole head groups and whole image slices per rank
check_degree = functools.partial(sharding.check_degree, model=MODEL)


def get_cu_seqlens(text_mask: torch.Tensor, img_len: int, device) -> torch.Tensor:
    """hyvideo_i2v/modules/attenion.py:34-57 on `device`, without a host round trip: the 2B+1 entries
    [0, valid_0 + img_len, max_len, max_len + valid_1 + img_len, 2 max_len, ...] with
    max_len = text + img_len.  Under SP img_len is the rank's image length (what my_parallel_attention
    expects: it rebuilds the global table from entry [1], which limits every sample)."""
    max_len = text_mask.shape[1] + img_len
    s = text_mask.sum(dim=1).to(device=device, dtype=torch.int32) + img_len
    ends = torch.arange(1, len(s) + 1, dtype=torch.int32, device=device) * max_len
    return torch.cat([torch.zeros(1, dtype=torch.int32, device=device),
                      torch.stack([ends - max_len + s, ends], dim=1).reshape(-1)])


def _step_calc(transformer):
    """jenga_hyi2v.py's own `step_calc` when its ra_forward has been bound to the class, else STEP_CALC"""
    ra = getattr(type(transformer), "ra_forward", None)
    sc = getattr(ra, "__globals__", {}).get("step_calc") if ra is not None else None
    return tuple(sc) if sc is not None else STEP_CALC


def parallelize_i2v(transformer, group=None, attention=None):
    """Replaces `transformer.forward` (an instance attribute, as parallelize_transformer sets it) with
    the sharded I2V forward and sets `block.jenga_sp = attention` on every double and single block.
    attention: a Ulysses object with the hybrid_seq_parallel_attn call contract; None means
    default_attention(group, "hyvideo_i2v").  Returns the attention object."""
    if not dist.is_initialized():
        raise RuntimeError(f"sequence-parallel {MODEL} needs an initialised process group")
    check_degree(0, int(transformer.heads_num), dist.get_world_size(group))
    blocks = list(transformer.double_blocks) + list(transformer.single_blocks)
    check_fused_blocks(blocks, "I2V", "install() (fused_blocks=True)", instance_forward=False)
    sp = attention if attention is not None else default_attention(group, "hyvideo_i2v")
    for block in blocks:
        # deliberately not `hybrid_seq_parallel_attn`: a block with that attribute keeps running the
        # reference's own (dense) SP forward
        block.jenga_sp = sp
    transformer.forward = types.MethodType(_forward_factory(group), transformer)
    return sp


def _forward_factory(group):
    def forward(self, x: torch.Tensor, t: torch.Tensor, text_states: torch.Tensor = None,
                text_mask: torch.Tensor = None, text_states_2: torch.Tensor | None = None,
                freqs_cos: torch.Tensor | None = None, freqs_sin: torch.Tensor | None = None,
                guidance: torch.Tensor = None, return_dict: bool = True, token_per_block=128):
        """jenga_hyi2v.py:53-221 (ra_forward) on this rank's Hilbert slice; returns the full output
        on every rank"""
        P, r = world(group)
        for name in ("hilbert_order", "linear_to_hilbert", "curve_sel", "sa_drop_rate", "p_remain_rates"):
            if getattr(self, name, None) is None:
                raise RuntimeError(f"sequence-parallel HunyuanVideo-I2V: transformer.{name} is not set "
                                   "(jenga_hyi2v.py sets the Jenga attributes before sampling)")
        out = {}
        img, txt = x, text_states
        _, _, ot, oh, ow = x.shape
        tt, th, tw = ot // self.patch_size[0], oh // self.patch_size[1], ow // self.patch_size[2]
        vec = self.time_in(t)                                                      # :76-102
        if self.i2v_condition_type == "token_replace":
            token_replace_vec = self.time_in(torch.zeros_like(t))
            frist_frame_token_num = th * tw
        else:
            token_replace_vec = frist_frame_token_num = None
        vec_2 = self.vector_in(text_states_2)
        vec = vec + vec_2
        if self.i2v_condition_type == "token_replace":
            token_replace_vec = token_replace_vec + vec_2
        if self.guidance_embed:
            if guidance is None:
                raise ValueError("Didn't get guidance strength for guidance distilled model.")
            vec = vec + self.guidance_in(guidance)
        img = self.img_in(img)                                                     # :105-113
        if self.text_projection == "linear":
            txt = self.txt_in(txt)
        elif self.text_projection == "single_refiner":
            txt = self.txt_in(txt, t, text_mask if self.use_attention_mask else None)
        else:
            raise NotImplementedError(f"Unsupported text_projection: {self.text_projection}")
        T, L = txt.shape[1], img.shape[1]
        check_degree(L, int(self.heads_num), P)
        # Hilbert order over the full sequence (:119-121), then this rank's slice
        order = self.hilbert_order
        img = img[:, order]
        freqs_cos, freqs_sin = freqs_cos[order], freqs_sin[order]
        # one first-frame mask, shared by every sample (as on the single-GPU path)
        first_frame_mask = torch.zeros_like(img[0, :, 0]).bool()                   # :124-126
        first_frame_mask[:th * tw] = 1
        first_frame_mask = first_frame_mask[order]
        n = L // P
        img = shard(img, 1, P, r)
        freqs_cos, freqs_sin = shard(freqs_cos, 0, P, r), shard(freqs_sin, 0, P, r)
        first_frame_mask = shard(first_frame_mask, 0, P, r)                         # double blocks: device
        # single blocks: the CPU mask over the rank's image rows and all text rows (:129-130); the
        # token-replace kernels copy it to the device once per forward (dense._row_mask)
        full_first_frame_mask = torch.zeros(n + T).bool()
        full_first_frame_mask[:n] = first_frame_mask.cpu()
        cu_seqlens_q = get_cu_seqlens(text_mask, n, img.device)                   # :133-136, local
        cu_seqlens_kv = cu_seqlens_q
        max_seqlen_q = max_seqlen_kv = n + T
        freqs_cis = (freqs_cos, freqs_sin)
        # step skipping (:139-145): the decision depends on the step counter alone, so every rank takes
        # the same one without an all_reduce; each rank keeps the residual of its own slice
        if self.cnt in _step_calc(self) or self.start_stage:
            self.start_stage = False
            should_calc = True
        else:
            should_calc = False
        if not should_calc:
            img += self.previous_residual
        else:
            ori_img = img.clone()
            for block in self.double_blocks:
                img, txt = block(img, txt, vec, cu_seqlens_q, cu_seqlens_kv, max_seqlen_q, max_seqlen_kv,
                                 freqs_cis, self.sa_drop_rate, first_frame_mask, self.i2v_condition_type,
                                 token_replace_vec, frist_frame_token_num, self.text_amp, self.curve_sel,
                                 self.p_remain_rates)
            x = torch.cat((img, txt), 1)
            for block in self.single_blocks:
                x = block(x, vec, T, cu_seqlens_q, cu_seqlens_kv, max_seqlen_q, max_seqlen_kv,
                          (freqs_cos, freqs_sin), self.sa_drop_rate, full_first_frame_mask,
                          self.i2v_condition_type, token_replace_vec, frist_frame_token_num, self.text_amp,
                          self.curve_sel, self.p_remain_rates)
            img = x[:, :n, ...]
            self.previous_residual = img - ori_img
        self.cnt += 1
        if self.cnt == self.num_steps:
            self.cnt = 0
        # the image rows of every rank in rank order (NCCL, once per forward), then replicated as
        # jenga_hyvideo_multigpu.py:193-198 does (P*n = L rows: nothing is cut)
        img = gather_rows(img, L, P, group)
        img = img[:, self.linear_to_hilbert]                                       # :213-217
        img = self.final_layer(img, vec)
        img = self.unpatchify(img, tt, th, tw)
        if return_dict:
            out["x"] = img
            return out
        return img
    return forward


def install_parallelize_transformer(inference_module) -> list[str]:
    """Swaps hyvideo_i2v.inference.parallelize_transformer for one that calls parallelize_i2v.
    Inference.from_pretrained calls it with ulysses_degree > 1, after its xfuser / NCCL process-group
    initialisation (hyvideo_i2v/inference.py:226-250, :568-569); the sharded forward reads the Jenga
    attributes jenga_hyi2v.py sets later (hilbert_order, curve_sels, sa_drop_rates, p_remain_rates)
    when it runs.  Returns what it swapped: nothing when there is nothing to swap or it is already swapped."""
    from .blocks import _swap

    def parallelize_transformer(pipe):
        """jenga_b200: Hilbert-sharded I2V forward over the Ulysses exchange"""
        parallelize_i2v(pipe.transformer)

    swapped = _swap(inference_module, "parallelize_transformer", parallelize_transformer)
    return [f"{inference_module.__name__}.parallelize_transformer"] if swapped else []
