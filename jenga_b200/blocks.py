"""Fused attention section of the reference's DiT blocks, applied to the UNMODIFIED block classes.

`install()` pre-seeds the operator modules (install.py); that alone leaves RMSNorm, RoPE, three
`torch.cat`s and the block pooling in eager PyTorch in front of the operator.  This module goes
one step further without touching a reference file: an import hook patches, right after the
reference module is executed,

  MMDoubleStreamBlock.forward / MMSingleStreamBlock.forward
      (hyvideo/modules/models_mul_block_gc_ha_multigpu.py:161-316, :392-500)
  MMDoubleStreamBlock.forward / MMSingleStreamBlock.forward of HunyuanVideo-I2V
      (hyvideo_i2v/modules/models_mul.py:136-319, :393-505)
  WanSelfAttention.forward            (wan/modules/model_mul.py:134-180)
  WanT2VCrossAttention.forward        (wan/modules/model_mul.py:183-205)
  WanAttentionBlock.forward           (wan/modules/model_mul.py:303-346)

with versions whose attention section is `jenga_hy_prologue` / `jenga_wan_prologue` (RMSNorm +
RoPE + img||txt concatenation + block pooling in one pass over the QKV projection output)
followed by select_blocks + the carved-attention launch.  Everything around the attention
section (modulation, linear layers, gates, MLP) is executed by the block's own sub-modules and
the reference module's own helper functions (`modulate`, `apply_gate`), so those numerics are the
reference's by construction.  Whenever a call is not the carved configuration (sa_drop_rate == 0,
no RMS qk-norm, unusual dtype, batch > 1 for Wan, sequence parallel for I2V, …) the ORIGINAL forward
runs.

The I2V blocks differ from the HunyuanVideo ones in three ways the fused forwards follow: the
token-replace modulation (rows of the first frame take the `tr_` shift / scale / gate; the
reference does it with boolean-mask index_put, modulate_layers.py:51-56,84-95, here it is a per-row
parameter select inside the ln_modulate / gate_residual kernels), a ragged S = L + 400 that the
operator zero-pads to whole blocks, and the operator's default text_blocks=4.

The Wan block forward runs its elementwise chains as the wan_* dense kernels (fp32 residual stream,
one pass per chain, bf16 handed to the Linears as autocast would cast it) and leaves the Linears, the
attention modules and the FFN to the block's own sub-modules.  Its T2V cross-attention runs the
norm-only prologue and the dense class of the attention kernel, without flash_attention's segment
table and host syncs.  Its I2V cross-attention (WanI2VCrossAttention, model_mul.py:223-249) runs the
module's own Linears around the norm-only prologue and ONE jenga_wan_i2v_cross_attn launch that
attends the 257 image and the text keys and adds the two results as the reference does; the block
calls it directly, and WanI2VCrossAttention.forward itself is left as it is.

A second hook routes `x[:, long_index]` / `x[long_index]` on contiguous CUDA activations — the
token reorder of jenga_hyvideo.py:116-118,226 and jenga_wan.py:559,655 — to `jenga_gather_rows`.
"""
from __future__ import annotations

import importlib.abc
import importlib.machinery
import sys

import torch

from . import dense as DN
from . import hyvideo as HY
from . import wan as WAN

_HY_MODULES = ("hyvideo.modules.models_mul_block_gc_ha_multigpu",)
_I2V_MODULES = ("hyvideo_i2v.modules.models_mul",)
_WAN_MODULES = ("wan.modules.model_mul",)
STATS = {"hy_double": 0, "hy_single": 0, "i2v_double": 0, "i2v_single": 0, "wan_self": 0, "fallback": 0,
         "gather": 0, "ln_modulate": 0, "gate_residual": 0, "gelu_cat": 0, "wan_block": 0, "wan_cross": 0,
         "wan_i2v_cross": 0}
# the CLIP image tokens at the head of the Wan2.1-I2V context (model_mul.py:230-231)
_WAN_I2V_IMG_TOKENS = 257
# the HunyuanVideo-I2V operator's text_blocks default (hyvideo_i2v/…/attention_block_triton_diffres.py:409);
# models_mul.py never passes text_blocks, so it holds whatever the text length
_I2V_TEXT_BLOCKS = 4


# ------------------------------------------------------------------------------------------------
# eligibility helpers
# ------------------------------------------------------------------------------------------------
def _rms_params(norm):
    """(weight, eps) if `norm` is the reference RMSNorm with an affine weight
    (hyvideo/modules/norm_layers.py:6-59), else None."""
    if type(norm).__name__ != "RMSNorm" or not hasattr(norm, "weight") or not hasattr(norm, "eps"):
        return None
    return norm.weight, float(norm.eps)


def _carved_call(x, sa_drop_rate, curve_sel):
    return (x.is_cuda and x.dtype in (torch.bfloat16, torch.float16) and sa_drop_rate != 0.0
            and curve_sel is not None and not isinstance(curve_sel, int))


def _ln_mod(mod, norm, x, shift, scale, tr=None):
    """modulate(norm(x), shift, scale) — one fused pass when it is the autocast-bf16 chain.
    tr=(tr_shift, tr_scale, first_frame_mask): the I2V token-replace form (modulate_layers.py:51-56)."""
    if DN.ln_modulate_supported(x, norm, shift, scale, tr=tr):
        STATS["ln_modulate"] += 1
        return DN.ln_modulate(x, shift, scale, eps=norm.eps, tr=tr)
    if tr is None:
        return mod.modulate(norm(x), shift=shift, scale=scale)
    return mod.modulate(norm(x), shift=shift, scale=scale, condition_type="token_replace", tr_shift=tr[0],
                        tr_scale=tr[1], first_frame_mask=tr[2])


def _gate_res(mod, x, y, gate, tr=None):
    """x + apply_gate(y, gate) — one fused pass for bf16 batch-1 tensors.
    tr=(tr_gate, first_frame_mask): the I2V token-replace form (modulate_layers.py:84-95)."""
    if DN.gate_residual_supported(x, y, gate, tr=tr):
        STATS["gate_residual"] += 1
        return DN.gate_residual(x, y, gate, tr=tr)
    if tr is None:
        return x + mod.apply_gate(y, gate=gate)
    return x + mod.apply_gate(y, gate=gate, condition_type="token_replace", tr_gate=tr[0], first_frame_mask=tr[1])


def _attention_section(self, mod, img_qkv, txt_qkv, norms, freqs_cis, cu_seqlens_q, cu_seqlens_kv,
                       sa_drop_rate, txt_amp, curve_sel, p_remain_rates, txt_block_num, per_block_token,
                       text_blocks_default, out=None, pad_ragged=False):
    """prologue -> (SP exchange | select + carved attention).  Returns attn [B, L+T, H*D]
    (written into `out`, a [B, L+T, H, D] view, when given and not under SP).
    pad_ragged: S = L+T need not be a multiple of 128 (the I2V operator zero-pads it)."""
    (wq_i, eps), (wk_i, _), (wq_t, _), (wk_t, _) = norms
    heads = self.heads_num
    L = img_qkv.shape[1]
    _, _, block_neighbor_list = mod.random.choice(curve_sel)                       # :232 / :438
    top_k = int((1 - sa_drop_rate) * (L // per_block_token))                       # models_mul…:242
    sp = getattr(self, "hybrid_seq_parallel_attn", None)
    want_pool = not sp
    S = L + (0 if txt_qkv is None else txt_qkv.shape[1])
    if want_pool and S % HY.BLOCK and not pad_ragged:
        return None
    q, k, v, pools = HY.attention_prologue(img_qkv, txt_qkv, heads, wq_i, wk_i, wq_t, wk_t, eps, freqs_cis,
                                           want_pool=want_pool)
    if sp:
        top_k = mod.get_sequence_parallel_world_size() * top_k                      # :249-251
        return mod.my_parallel_attention(sp, q, k, v, img_q_len=L, img_kv_len=L, cu_seqlens_q=cu_seqlens_q,
                                         cu_seqlens_kv=cu_seqlens_kv, top_k=top_k, text_amp=txt_amp,
                                         block_neighbor_list=block_neighbor_list,
                                         p_remain_rates=p_remain_rates)
    return HY.carved_attention_from_pools(q, k, v, pools, top_k=top_k, text_blocks=txt_block_num,
                                          text_amp=txt_amp, block_neighbor_list=block_neighbor_list,
                                          p_remain_rates=p_remain_rates, cu_seqlens_q=cu_seqlens_q, out=out,
                                          pad_ragged=pad_ragged)


# ------------------------------------------------------------------------------------------------
# HunyuanVideo blocks
# ------------------------------------------------------------------------------------------------
def _make_double_forward(orig, mod, text_blocks_default):
    def forward(self, img, txt, vec, cu_seqlens_q=None, cu_seqlens_kv=None, max_seqlen_q=None,
                max_seqlen_kv=None, freqs_cis=None, sa_drop_rate=0.0, txt_amp=1.0, curve_sel=None,
                p_remain_rates=0.5, txt_block_num=text_blocks_default, per_block_token=128):
        norms = [_rms_params(n) for n in (self.img_attn_q_norm, self.img_attn_k_norm,
                                          self.txt_attn_q_norm, self.txt_attn_k_norm)]
        if (not _carved_call(img, sa_drop_rate, curve_sel) or None in norms or per_block_token != HY.BLOCK
                or cu_seqlens_q is None or img.shape[-1] // self.heads_num != 128):
            STATS["fallback"] += 1
            return orig(self, img, txt, vec, cu_seqlens_q, cu_seqlens_kv, max_seqlen_q, max_seqlen_kv,
                        freqs_cis, sa_drop_rate, txt_amp, curve_sel, p_remain_rates, txt_block_num,
                        per_block_token)
        i_shift1, i_scale1, i_gate1, i_shift2, i_scale2, i_gate2 = self.img_mod(vec).chunk(6, dim=-1)
        t_shift1, t_scale1, t_gate1, t_shift2, t_scale2, t_gate2 = self.txt_mod(vec).chunk(6, dim=-1)
        img_qkv = self.img_attn_qkv(_ln_mod(mod, self.img_norm1, img, i_shift1, i_scale1))
        txt_qkv = self.txt_attn_qkv(_ln_mod(mod, self.txt_norm1, txt, t_shift1, t_scale1))
        assert cu_seqlens_q.shape[0] == 2 * img.shape[0] + 1                         # :244-246
        attn = _attention_section(self, mod, img_qkv, txt_qkv, norms, freqs_cis, cu_seqlens_q, cu_seqlens_kv,
                                  sa_drop_rate, txt_amp, curve_sel, p_remain_rates, txt_block_num,
                                  per_block_token, text_blocks_default)
        if attn is None:
            STATS["fallback"] += 1
            return orig(self, img, txt, vec, cu_seqlens_q, cu_seqlens_kv, max_seqlen_q, max_seqlen_kv,
                        freqs_cis, sa_drop_rate, txt_amp, curve_sel, p_remain_rates, txt_block_num,
                        per_block_token)
        STATS["hy_double"] += 1
        L = img.shape[1]
        img_attn, txt_attn = attn[:, :L], attn[:, L:]
        img = _gate_res(mod, img, self.img_attn_proj(img_attn), i_gate1)
        img = _gate_res(mod, img, self.img_mlp(_ln_mod(mod, self.img_norm2, img, i_shift2, i_scale2)), i_gate2)
        txt = _gate_res(mod, txt, self.txt_attn_proj(txt_attn), t_gate1)
        txt = _gate_res(mod, txt, self.txt_mlp(_ln_mod(mod, self.txt_norm2, txt, t_shift2, t_scale2)), t_gate2)
        return img, txt
    forward.__jenga_b200__ = True
    forward.__wrapped__ = orig
    return forward


def _make_single_forward(orig, mod, text_blocks_default):
    def forward(self, x, vec, txt_len, cu_seqlens_q=None, cu_seqlens_kv=None, max_seqlen_q=None,
                max_seqlen_kv=None, freqs_cis=None, sa_drop_rate=0.0, txt_amp=1.0, curve_sel=None,
                p_remain_rates=0.5, txt_block_num=text_blocks_default, per_block_token=128):
        norms = [_rms_params(n) for n in (self.q_norm, self.k_norm)]
        if (not _carved_call(x, sa_drop_rate, curve_sel) or None in norms or per_block_token != HY.BLOCK
                or cu_seqlens_q is None or freqs_cis is None or self.hidden_size // self.heads_num != 128):
            STATS["fallback"] += 1
            return orig(self, x, vec, txt_len, cu_seqlens_q, cu_seqlens_kv, max_seqlen_q, max_seqlen_kv,
                        freqs_cis, sa_drop_rate, txt_amp, curve_sel, p_remain_rates, txt_block_num,
                        per_block_token)
        shift, scale, gate = self.modulation(vec).chunk(3, dim=-1)
        lin1 = self.linear1(_ln_mod(mod, self.pre_norm, x, shift, scale))
        C3 = 3 * self.hidden_size
        L = x.shape[1] - txt_len
        # strided views into linear1's output: no split / rearrange / cat copies (:413-441)
        img_qkv, txt_qkv = lin1[:, :L, :C3], lin1[:, L:, :C3]
        mlp = lin1[:, :, C3:]
        assert cu_seqlens_q.shape[0] == 2 * x.shape[0] + 1                           # :444-446
        # `torch.cat((attn, self.mlp_act(mlp)), 2)` (:499) without the concatenation copy: the attention
        # kernel writes its rows into the first `hidden` columns of linear2's input buffer and the
        # GELU kernel writes the rest
        act = self.mlp_act
        fuse_cat = (isinstance(act, torch.nn.GELU) and getattr(act, "approximate", "none") == "tanh"
                    and lin1.dtype == torch.bfloat16 and x.shape[0] == 1
                    and not getattr(self, "hybrid_seq_parallel_attn", None))
        cat = attn_view = None
        if fuse_cat:
            cat = torch.empty((x.shape[0], x.shape[1], C3 // 3 + mlp.shape[-1]), dtype=lin1.dtype, device=lin1.device)
            attn_view = cat[:, :, :C3 // 3].unflatten(2, (self.heads_num, -1))
        attn = _attention_section(self, mod, img_qkv, txt_qkv, [norms[0], norms[1], norms[0], norms[1]],
                                  freqs_cis, cu_seqlens_q, cu_seqlens_kv, sa_drop_rate, txt_amp, curve_sel,
                                  p_remain_rates, txt_block_num, per_block_token, text_blocks_default, out=attn_view)
        if attn is None:
            STATS["fallback"] += 1
            return orig(self, x, vec, txt_len, cu_seqlens_q, cu_seqlens_kv, max_seqlen_q, max_seqlen_kv,
                        freqs_cis, sa_drop_rate, txt_amp, curve_sel, p_remain_rates, txt_block_num,
                        per_block_token)
        STATS["hy_single"] += 1
        if fuse_cat:
            STATS["gelu_cat"] += 1
            DN.gelu_tanh_into(mlp, cat[:, :, C3 // 3:])
            out = self.linear2(cat)
        else:
            out = self.linear2(torch.cat((attn, act(mlp)), 2))
        return _gate_res(mod, x, out, gate)
    forward.__jenga_b200__ = True
    forward.__wrapped__ = orig
    return forward


# ------------------------------------------------------------------------------------------------
# HunyuanVideo-I2V blocks
# ------------------------------------------------------------------------------------------------
def _i2v_eligible(self, x, sa_drop_rate, curve_sel, norms, per_block_token, cu_seqlens_q, S, tr, mask):
    """the carved configuration the fused I2V forwards take; anything else runs the original"""
    return (_carved_call(x, sa_drop_rate, curve_sel) and None not in norms and per_block_token == HY.BLOCK
            and cu_seqlens_q is not None and x.shape[-1] // self.heads_num == 128
            # sequence parallel: the reference runs the dense parallel_attention (:264-274, :483-493)
            and not getattr(self, "hybrid_seq_parallel_attn", None)
            # the prefix form (frist_frame_token_num) is only reached outside the Jenga forward
            and not (tr and mask is None)
            and (S + HY.BLOCK - 1) // HY.BLOCK > _I2V_TEXT_BLOCKS)


def _make_i2v_double_forward(orig, mod):
    def forward(self, img, txt, vec, cu_seqlens_q=None, cu_seqlens_kv=None, max_seqlen_q=None,
                max_seqlen_kv=None, freqs_cis=None, sa_drop_rate=0.0, first_frame_mask=None,
                condition_type=None, token_replace_vec=None, frist_frame_token_num=None, txt_amp=0.0,
                curve_sel=None, p_remain_rates=0.5, per_block_token=128):
        args = (img, txt, vec, cu_seqlens_q, cu_seqlens_kv, max_seqlen_q, max_seqlen_kv, freqs_cis, sa_drop_rate,
                first_frame_mask, condition_type, token_replace_vec, frist_frame_token_num, txt_amp, curve_sel,
                p_remain_rates, per_block_token)
        tr = condition_type == "token_replace"
        norms = [_rms_params(n) for n in (self.img_attn_q_norm, self.img_attn_k_norm,
                                          self.txt_attn_q_norm, self.txt_attn_k_norm)]
        L = img.shape[1]
        if not _i2v_eligible(self, img, sa_drop_rate, curve_sel, norms, per_block_token, cu_seqlens_q,
                             L + txt.shape[1], tr, first_frame_mask):
            STATS["fallback"] += 1
            return orig(self, *args)
        if tr:                                                                         # :156-179
            img_mods, tr_mods = self.img_mod(vec, condition_type=condition_type, token_replace_vec=token_replace_vec)
            i_shift1, i_scale1, i_gate1, i_shift2, i_scale2, i_gate2 = img_mods.chunk(6, dim=-1)
            r_shift1, r_scale1, r_gate1, r_shift2, r_scale2, r_gate2 = tr_mods.chunk(6, dim=-1)
            tr_mod1 = (r_shift1, r_scale1, first_frame_mask)
            tr_mod2 = (r_shift2, r_scale2, first_frame_mask)
            tr_gate1, tr_gate2 = (r_gate1, first_frame_mask), (r_gate2, first_frame_mask)
        else:
            i_shift1, i_scale1, i_gate1, i_shift2, i_scale2, i_gate2 = self.img_mod(vec).chunk(6, dim=-1)
            tr_mod1 = tr_mod2 = tr_gate1 = tr_gate2 = None
        t_shift1, t_scale1, t_gate1, t_shift2, t_scale2, t_gate2 = self.txt_mod(vec).chunk(6, dim=-1)
        img_qkv = self.img_attn_qkv(_ln_mod(mod, self.img_norm1, img, i_shift1, i_scale1, tr=tr_mod1))
        txt_qkv = self.txt_attn_qkv(_ln_mod(mod, self.txt_norm1, txt, t_shift1, t_scale1))
        assert cu_seqlens_q.shape[0] == 2 * img.shape[0] + 1                         # :235-237
        attn = _attention_section(self, mod, img_qkv, txt_qkv, norms, freqs_cis, cu_seqlens_q, cu_seqlens_kv,
                                  sa_drop_rate, txt_amp, curve_sel, p_remain_rates, _I2V_TEXT_BLOCKS,
                                  per_block_token, _I2V_TEXT_BLOCKS, pad_ragged=True)
        STATS["i2v_double"] += 1
        img_attn, txt_attn = attn[:, :L], attn[:, L:]
        img = _gate_res(mod, img, self.img_attn_proj(img_attn), i_gate1, tr=tr_gate1)   # :281-306
        img = _gate_res(mod, img, self.img_mlp(_ln_mod(mod, self.img_norm2, img, i_shift2, i_scale2, tr=tr_mod2)),
                        i_gate2, tr=tr_gate2)
        txt = _gate_res(mod, txt, self.txt_attn_proj(txt_attn), t_gate1)                 # :309-317
        txt = _gate_res(mod, txt, self.txt_mlp(_ln_mod(mod, self.txt_norm2, txt, t_shift2, t_scale2)), t_gate2)
        return img, txt
    forward.__jenga_b200__ = True
    forward.__wrapped__ = orig
    return forward


def _make_i2v_single_forward(orig, mod):
    def forward(self, x, vec, txt_len, cu_seqlens_q=None, cu_seqlens_kv=None, max_seqlen_q=None,
                max_seqlen_kv=None, freqs_cis=None, sa_drop_rate=0.0, first_frame_mask=None,
                condition_type=None, token_replace_vec=None, frist_frame_token_num=None, txt_amp=0.0,
                curve_sel=None, p_remain_rates=0.5, per_block_token=128):
        args = (x, vec, txt_len, cu_seqlens_q, cu_seqlens_kv, max_seqlen_q, max_seqlen_kv, freqs_cis, sa_drop_rate,
                first_frame_mask, condition_type, token_replace_vec, frist_frame_token_num, txt_amp, curve_sel,
                p_remain_rates, per_block_token)
        tr = condition_type == "token_replace"
        norms = [_rms_params(n) for n in (self.q_norm, self.k_norm)]
        if (not _i2v_eligible(self, x, sa_drop_rate, curve_sel, norms, per_block_token, cu_seqlens_q, x.shape[1],
                              tr, first_frame_mask)
                or freqs_cis is None or not 0 < txt_len < x.shape[1]):
            STATS["fallback"] += 1
            return orig(self, *args)
        if tr:                                                                         # :413-424
            mods, tr_mods = self.modulation(vec, condition_type=condition_type, token_replace_vec=token_replace_vec)
            shift, scale, gate = mods.chunk(3, dim=-1)
            r_shift, r_scale, r_gate = tr_mods.chunk(3, dim=-1)
            # full_first_frame_mask (jenga_hyi2v.py:129-130): a CPU bool over L+T rows
            tr_mod, tr_gate = (r_shift, r_scale, first_frame_mask), (r_gate, first_frame_mask)
        else:
            shift, scale, gate = self.modulation(vec).chunk(3, dim=-1)
            tr_mod = tr_gate = None
        lin1 = self.linear1(_ln_mod(mod, self.pre_norm, x, shift, scale, tr=tr_mod))
        C3 = 3 * self.hidden_size
        L = x.shape[1] - txt_len
        # strided views into linear1's output: no split / rearrange / cat copies (:431-451)
        img_qkv, txt_qkv = lin1[:, :L, :C3], lin1[:, L:, :C3]
        mlp = lin1[:, :, C3:]
        assert cu_seqlens_q.shape[0] == 2 * x.shape[0] + 1                           # :464-466
        # `torch.cat((attn, self.mlp_act(mlp)), 2)` (:497) without the concatenation copy, as in the
        # HunyuanVideo single-stream forward above
        act = self.mlp_act
        fuse_cat = (isinstance(act, torch.nn.GELU) and getattr(act, "approximate", "none") == "tanh"
                    and lin1.dtype == torch.bfloat16 and x.shape[0] == 1)
        cat = attn_view = None
        if fuse_cat:
            cat = torch.empty((x.shape[0], x.shape[1], C3 // 3 + mlp.shape[-1]), dtype=lin1.dtype, device=lin1.device)
            attn_view = cat[:, :, :C3 // 3].unflatten(2, (self.heads_num, -1))
        attn = _attention_section(self, mod, img_qkv, txt_qkv, [norms[0], norms[1], norms[0], norms[1]],
                                  freqs_cis, cu_seqlens_q, cu_seqlens_kv, sa_drop_rate, txt_amp, curve_sel,
                                  p_remain_rates, _I2V_TEXT_BLOCKS, per_block_token, _I2V_TEXT_BLOCKS,
                                  out=attn_view, pad_ragged=True)
        STATS["i2v_single"] += 1
        if fuse_cat:
            STATS["gelu_cat"] += 1
            DN.gelu_tanh_into(mlp, cat[:, :, C3 // 3:])
            out = self.linear2(cat)
        else:
            out = self.linear2(torch.cat((attn, act(mlp)), 2))
        return _gate_res(mod, x, out, gate, tr=tr_gate)                              # :499-505
    forward.__jenga_b200__ = True
    forward.__wrapped__ = orig
    return forward


# ------------------------------------------------------------------------------------------------
# Wan self-attention
# ------------------------------------------------------------------------------------------------
def _make_wan_forward(orig, mod):
    def forward(self, x, seq_lens, grid_sizes, freqs, sa_drop_rate=0.0, per_block_tokens=128,
                p_remain_rates=0.8, freq_remap=None, block_neighbor_list=None):
        b, s = x.shape[:2]
        wq = getattr(self.norm_q, "weight", None)
        wk = getattr(self.norm_k, "weight", None)
        if (sa_drop_rate <= 0.25 or not x.is_cuda or b != 1 or self.head_dim != 128 or per_block_tokens != 128
                or wq is None or wk is None or type(self.norm_q).__name__ != "WanRMSNorm"):
            STATS["fallback"] += 1
            return orig(self, x, seq_lens, grid_sizes, freqs, sa_drop_rate, per_block_tokens, p_remain_rates,
                        freq_remap, block_neighbor_list)
        q_lin, k_lin = self.q(x), self.k(x)
        if q_lin.dtype not in (torch.bfloat16, torch.float32):
            STATS["fallback"] += 1
            return orig(self, x, seq_lens, grid_sizes, freqs, sa_drop_rate, per_block_tokens, p_remain_rates,
                        freq_remap, block_neighbor_list)
        v = self.v(x).view(b, s, self.num_heads, self.head_dim)
        grid = [int(g) for g in grid_sizes[0].tolist()]
        out = WAN.self_attention(q_lin, k_lin, v, wq, wk, self.num_heads, grid, freqs, sa_drop_rate,
                                 p_remain_rates=p_remain_rates, freq_remap=freq_remap,
                                 block_neighbor_list=block_neighbor_list, eps=float(self.norm_q.eps))
        STATS["wan_self"] += 1
        out = out.flatten(2)
        if not torch.is_autocast_enabled():
            # the reference returns the query dtype, fp32 (rope_apply -> .float(), model_mul.py:71;
            # operator :530-532); under autocast the following Linear casts back to bf16 anyway
            out = out.float()
        return self.o(out)
    forward.__jenga_b200__ = True
    forward.__wrapped__ = orig
    return forward


def _make_wan_cross_forward(orig, mod):
    def forward(self, x, context, context_lens):
        wq = getattr(self.norm_q, "weight", None)
        wk = getattr(self.norm_k, "weight", None)
        # context_lens: the reference's varlen form (wan/modules/attention.py:69-80); teacache_forward
        # passes None (jenga_wan.py:569)
        if (context_lens is not None or not x.is_cuda or x.dim() != 3 or x.shape[0] != 1 or context.dim() != 3
                or context.shape[0] != 1 or self.head_dim != 128 or wq is None or wk is None
                or type(self.norm_q).__name__ != "WanRMSNorm" or type(self.norm_k).__name__ != "WanRMSNorm"
                or not DN._autocast_bf16()):
            STATS["fallback"] += 1
            return orig(self, x, context, context_lens)
        q_lin, k_lin, v = self.q(x), self.k(context), self.v(context)
        if (q_lin.dtype not in (torch.bfloat16, torch.float32) or k_lin.dtype not in (torch.bfloat16, torch.float32)
                or v.dtype != torch.bfloat16):
            STATS["fallback"] += 1
            return orig(self, x, context, context_lens)
        out = WAN.cross_attention(q_lin, k_lin, v.view(1, -1, self.num_heads, self.head_dim), wq, wk,
                                  self.num_heads, eps=float(self.norm_q.eps))
        STATS["wan_cross"] += 1
        return self.o(out.flatten(2))
    forward.__jenga_b200__ = True
    forward.__wrapped__ = orig
    return forward


def _wan_i2v_cross_shape_ok(ca, x, context, context_lens):
    """the I2V cross-attention configuration the fused kernel takes, device and autocast aside: one
    sample, every context row valid (teacache_forward passes context_lens=None, jenga_wan.py:569),
    head_dim 128, WanRMSNorm q / k / k_img norms with weights and one eps, and text rows after the
    image rows"""
    norms = [getattr(ca, n, None) for n in ("norm_q", "norm_k", "norm_k_img")]
    return (context_lens is None and isinstance(x, torch.Tensor) and isinstance(context, torch.Tensor)
            and x.dim() == 3 and x.shape[0] == 1 and context.dim() == 3 and context.shape[0] == 1
            and context.shape[1] > _WAN_I2V_IMG_TOKENS and getattr(ca, "head_dim", None) == 128
            and all(type(n).__name__ == "WanRMSNorm" and getattr(n, "weight", None) is not None for n in norms)
            and len({float(n.eps) for n in norms}) == 1)


def wan_i2v_cross_eligible(ca, x, context, context_lens):
    """True when the fused block runs WanI2VCrossAttention `ca` as i2v_cross_attention: the shape rules
    above, CUDA tensors and bf16 autocast"""
    return _wan_i2v_cross_shape_ok(ca, x, context, context_lens) and x.is_cuda and DN._autocast_bf16()


def _wan_i2v_cross(ca, x, context, context_lens):
    """WanI2VCrossAttention.forward (model_mul.py:223-249) with its attention part as one
    jenga_wan_i2v_cross_attn launch; the module's own q / k / v / k_img / v_img / o Linears run around
    it.  Anything else runs the module's own forward."""
    if wan_i2v_cross_eligible(ca, x, context, context_lens):
        ctx_img, ctx = context[:, :_WAN_I2V_IMG_TOKENS], context[:, _WAN_I2V_IMG_TOKENS:]   # :230-231
        q_lin, k_lin, v = ca.q(x), ca.k(ctx), ca.v(ctx)
        kimg_lin, vimg = ca.k_img(ctx_img), ca.v_img(ctx_img)
        lin_ok = all(t.dtype in (torch.bfloat16, torch.float32) for t in (q_lin, k_lin, kimg_lin))
        if lin_ok and v.dtype == vimg.dtype == torch.bfloat16:
            n = ca.num_heads
            out = WAN.i2v_cross_attention(q_lin, k_lin, v.view(1, -1, n, 128), kimg_lin, vimg.view(1, -1, n, 128),
                                          ca.norm_q.weight, ca.norm_k.weight, ca.norm_k_img.weight, n,
                                          eps=float(ca.norm_q.eps))
            STATS["wan_i2v_cross"] += 1
            return ca.o(out.flatten(2))
    STATS["fallback"] += 1
    return ca(x, context, context_lens)


def _make_wan_block_forward(orig, mod):
    def forward(self, x, e, seq_lens, grid_sizes, freqs, context, context_lens, sa_drop_rate=0.0, freq_remap=None,
                block_neighbor_list=None, p_remain_rates=0.0):
        args = (x, e, seq_lens, grid_sizes, freqs, context, context_lens, sa_drop_rate, freq_remap,
                block_neighbor_list, p_remain_rates)
        i2v = type(self.cross_attn).__name__ == "WanI2VCrossAttention"
        ok = (isinstance(e, torch.Tensor) and e.dtype == torch.float32 and x.is_cuda and x.dim() == 3
              and (i2v or type(self.cross_attn).__name__ == "WanT2VCrossAttention")
              and self.modulation.dtype == torch.float32)
        if ok:
            with torch.autocast("cuda", dtype=torch.float32):                      # :326-327
                e6 = self.modulation + e
            ok = (DN.wan_ln_modulate_supported(x, self.norm1, e6)
                  and DN.wan_residual_ln_supported(x, self.norm3, e6, affine=True)
                  and DN.wan_residual_ln_supported(x, self.norm2, e6, affine=False)
                  and DN.wan_gate_residual_supported(x, e6))
        if not ok:
            # no autocast, batch > 1, cross_attn_norm=False (norm3 is Identity), …
            STATS["fallback"] += 1
            return orig(self, *args)
        e = e6.chunk(6, dim=1)
        # self-attention on the bf16 its q / k / v Linears would cast the fp32 modulate output to
        y = self.self_attn(DN.wan_ln_modulate(x, e[0], e[1], eps=self.norm1.eps), seq_lens, grid_sizes, freqs,
                           sa_drop_rate=sa_drop_rate, freq_remap=freq_remap, block_neighbor_list=block_neighbor_list,
                           p_remain_rates=p_remain_rates)                          # :331-333
        x, h = DN.wan_residual_ln(x, y, e[2], eps=self.norm3.eps, weight=self.norm3.weight,
                                  bias=self.norm3.bias)                            # :334-335, :339
        # WanI2VCrossAttention.forward itself stays unpatched: the block routes it here
        cross = _wan_i2v_cross(self.cross_attn, h, context, context_lens) if i2v else \
            self.cross_attn(h, context, context_lens)
        x, h = DN.wan_residual_ln(x, cross, None, eps=self.norm2.eps, shift=e[3], scale=e[4])   # :339-340
        STATS["wan_block"] += 1
        return DN.wan_gate_residual(x, self.ffn(h), e[5])                          # :340-342
    forward.__jenga_b200__ = True
    forward.__wrapped__ = orig
    return forward


def patch_module(mod) -> list[str]:
    """Patches the block classes of an already imported reference module; returns what it did."""
    done = []
    name = mod.__name__
    # hyvideo_i2v/modules/models_mul.py has its own argument order, the token_replace modulation and
    # a ragged S with four text blocks: its own pair of forwards
    i2v = name.startswith("hyvideo_i2v.")
    if ((name.startswith("hyvideo.") or i2v) and hasattr(mod, "MMDoubleStreamBlock")
            and not getattr(mod.MMDoubleStreamBlock.forward, "__jenga_b200__", False)):
        if i2v:
            mod.MMDoubleStreamBlock.forward = _make_i2v_double_forward(mod.MMDoubleStreamBlock.forward, mod)
            mod.MMSingleStreamBlock.forward = _make_i2v_single_forward(mod.MMSingleStreamBlock.forward, mod)
        else:
            mod.MMDoubleStreamBlock.forward = _make_double_forward(mod.MMDoubleStreamBlock.forward, mod, 2)
            mod.MMSingleStreamBlock.forward = _make_single_forward(mod.MMSingleStreamBlock.forward, mod, 2)
        done += [f"{name}.MMDoubleStreamBlock.forward", f"{name}.MMSingleStreamBlock.forward"]
    if hasattr(mod, "WanSelfAttention") and not getattr(mod.WanSelfAttention.forward, "__jenga_b200__", False):
        orig = mod.WanSelfAttention.forward
        mod.WanSelfAttention.forward = _make_wan_forward(orig, mod)
        done.append(f"{name}.WanSelfAttention.forward")
    # WanI2VCrossAttention overrides forward itself and is left as it is; the fused block forward runs
    # its fused form (_wan_i2v_cross)
    for cls, make in (("WanT2VCrossAttention", _make_wan_cross_forward), ("WanAttentionBlock", _make_wan_block_forward)):
        if hasattr(mod, cls) and not getattr(getattr(mod, cls).forward, "__jenga_b200__", False):
            getattr(mod, cls).forward = make(getattr(mod, cls).forward, mod)
            done.append(f"{name}.{cls}.forward")
    return done


# ------------------------------------------------------------------------------------------------
# import hook: patch right after the reference module body has run
# ------------------------------------------------------------------------------------------------
class _PatchingLoader(importlib.abc.Loader):
    def __init__(self, inner):
        self.inner = inner

    def create_module(self, spec):
        return self.inner.create_module(spec)

    def exec_module(self, module):
        self.inner.exec_module(module)
        done = patch_module(module)
        if done:
            print(f"[jenga_b200] fused attention section installed: {', '.join(done)}", file=sys.stderr)

    def __getattr__(self, item):
        return getattr(self.inner, item)


class _PatchFinder(importlib.abc.MetaPathFinder):
    targets = _HY_MODULES + _I2V_MODULES + _WAN_MODULES

    def find_spec(self, fullname, path, target=None):
        if fullname not in self.targets:
            return None
        for finder in sys.meta_path:
            if finder is self or not hasattr(finder, "find_spec"):
                continue
            spec = finder.find_spec(fullname, path, target)
            if spec is not None and spec.loader is not None:
                spec.loader = _PatchingLoader(spec.loader)
                return spec
        return None


def install_block_hook() -> None:
    """Idempotent.  Also patches target modules that were imported before the hook existed."""
    if not any(isinstance(f, _PatchFinder) for f in sys.meta_path):
        sys.meta_path.insert(0, _PatchFinder())
    for name in _PatchFinder.targets:
        if name in sys.modules and not getattr(sys.modules[name], "__jenga_b200__", False):
            patch_module(sys.modules[name])


# ------------------------------------------------------------------------------------------------
# token reorder: x[:, index] on CUDA activations -> jenga_gather_rows
# ------------------------------------------------------------------------------------------------
class _GatherMode(torch.overrides.TorchFunctionMode):
    """Routes `x[:, idx]` (x [B,N,C]) and `x[idx]` (x [N,C]) with a 1-D int64 CUDA index of at
    least 1024 entries to the gather kernel — exactly the token reorders of jenga_hyvideo.py:116-118,
    :226 / jenga_wan.py:559,655.  Same result as ATen's index kernel (a row copy); indices are
    validated once per index tensor (range check, one host sync), like ATen's device assert."""

    def __init__(self):
        super().__init__()
        self._ok = {}

    def _valid(self, idx, n):
        key = (idx.data_ptr(), idx.numel(), idx._version, n)
        hit = self._ok.get(key)
        if hit is None:
            hit = bool(((idx >= 0) & (idx < n)).all().item())
            if len(self._ok) > 256:
                self._ok.clear()
            self._ok[key] = hit
        return hit

    def __torch_function__(self, func, types, args=(), kwargs=None):
        if func is torch.Tensor.__getitem__ and len(args) == 2:
            x, item = args
            idx = None
            if isinstance(item, tuple) and len(item) == 2 and isinstance(item[0], slice) \
                    and item[0] == slice(None) and isinstance(item[1], torch.Tensor) and x.dim() == 3:
                idx = item[1]
            elif isinstance(item, torch.Tensor) and x.dim() == 2:
                idx = item
            if (idx is not None and type(x) is torch.Tensor and x.is_cuda and idx.is_cuda and idx.dtype == torch.int64
                    and idx.dim() == 1 and idx.numel() >= 1024 and idx.is_contiguous() and x.is_contiguous()
                    and not x.requires_grad and (x.shape[-1] * x.element_size()) % 16 == 0
                    and self._valid(idx, x.shape[-2])):
                STATS["gather"] += 1
                return HY.gather_tokens(x, idx)
        return func(*args, **(kwargs or {}))


_gather_mode = None


def install_gather_hook() -> None:
    global _gather_mode
    if _gather_mode is None:
        _gather_mode = _GatherMode()
        _gather_mode.__enter__()


def remove_gather_hook() -> None:
    global _gather_mode
    if _gather_mode is not None:
        _gather_mode.__exit__(None, None, None)
        _gather_mode = None
