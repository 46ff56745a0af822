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
  WanSelfAttention.forward / WanAttentionBlock.forward of wan/modules/model.py (:127-156, :274-313),
      the plain model WanI2V loads, under install(wan_sp=True) at import, and when a single-GPU
      WanI2V is built (WanI2V.__init__ of wan/image2video.py is wrapped for that)

with versions whose attention section is `jenga_hy_prologue` / `jenga_wan_prologue` (RMSNorm +
RoPE + img||txt concatenation + block pooling in one pass over the QKV projection output)
followed by select_blocks + the carved-attention launch.  Everything around the attention
section (modulation, linear layers, gates, MLP) is executed by the block's own sub-modules and
the reference module's own helper functions (`modulate`, `apply_gate`), so those numerics are the
reference's by construction.  Whenever a call is not the carved configuration (sa_drop_rate == 0,
no RMS qk-norm, unusual dtype, Wan samples on several latent grids, the reference's own sequence
parallel for I2V, …) the ORIGINAL forward runs, with the caller's own arguments (`_patched`).  An I2V
block with `jenga_sp` set (the Hilbert-sharded forward of hyi2v_sp.py) routes its attention section
through that Ulysses object and has no such fall-back; so does a WanSelfAttention with `jenga_sp` set (the Hilbert-sharded Wan
forward of wan_sp.py), whose carved and dense calls both go through the exchange; and so does a
plain-module WanSelfAttention under `jenga_sp` (the raster-sharded I2V forward of wan_sp.py), whose
block then runs the fused I2V cross-attention on the rank's rows or raises.

The I2V blocks differ from the HunyuanVideo ones in three ways the fused forwards follow: the
token-replace modulation (rows of the first frame take the `tr_` shift / scale / gate; the
reference does it with boolean-mask index_put, modulate_layers.py:51-56,84-95, here it is a per-row
parameter select inside the ln_modulate / gate_residual kernels), a ragged S = L + 400 that the
operator zero-pads to whole blocks, and the operator's default text_blocks=4.  Both variants run one
fused body per stream kind (`_double_stream`, `_single_stream`); each keeps a thin entry point with
its reference signature that hands the body these differences.

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

import functools
import importlib.abc
import sys
from typing import Callable, NamedTuple

import torch

from . import dense as DN
from . import hyi2v_sp, wan_sp
from . import hyvideo as HY
from . import ulysses as U
from . import wan as WAN
from .flash_attn_shim import flash_attn_func
from .sharding import world

# the opt-in routes (install(i2v_sp=True) / JENGA_I2V_SP=1, install(wan_sp=True) / JENGA_WAN_SP=1): see _HOOKS
I2V_SP = False
WAN_SP = False


def set_i2v_sp(on: bool) -> None:
    """Turns the sequence-parallel I2V route on or off for the rest of the process.  Off also puts the
    reference's parallelize_transformer back if hyvideo_i2v.inference was already swapped."""
    _set_route("I2V_SP", on)


def set_wan_sp(on: bool) -> None:
    """Turns the sequence-parallel Wan route on or off for the rest of the process.  Off also puts the
    reference's usp_dit_forward / usp_attn_forward back if wan.distributed.xdit_context_parallel was
    already swapped (a model that has bound them keeps what it bound), and wan.modules.model's forwards."""
    _set_route("WAN_SP", on)


def _set_route(switch: str, on: bool) -> None:
    globals()[switch] = bool(on)
    if not on:
        for name, hook in _HOOKS.items():
            if hook.switch == switch and hook.restore is not None and name in sys.modules:
                hook.restore(sys.modules[name])


STATS = {"hy_double": 0, "hy_single": 0, "i2v_double": 0, "i2v_single": 0, "i2v_double_sp": 0,
         "i2v_single_sp": 0, "wan_self": 0, "wan_self_sp": 0, "wan_self_dense_sp": 0, "fallback": 0,
         "gather": 0, "ln_modulate": 0, "gate_residual": 0, "gelu_cat": 0, "wan_block": 0, "wan_cross": 0,
         "wan_i2v_cross": 0, "linear_fp8": 0, "wan_i2v_self_sp": 0, "wan_i2v_cross_sp": 0, "wan_i2v_self": 0,
         "wan_i2v_self_dense": 0, "wan_i2v_self_carved_sp": 0}
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


def _carved_call(self, x, norms, sa_drop_rate, curve_sel, cu_seqlens_q, per_block_token):
    """the carved configuration the fused forwards of both HunyuanVideo variants take: a bf16 / fp16
    CUDA input, a sparse call with a curve, RMS qk-norms, 128-token blocks and head_dim 128"""
    return (x.is_cuda and x.dtype in (torch.bfloat16, torch.float16) and sa_drop_rate != 0.0
            and curve_sel is not None and not isinstance(curve_sel, int) and None not in norms
            and per_block_token == HY.BLOCK and cu_seqlens_q is not None and x.shape[-1] // self.heads_num == 128)


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
    """x + apply_gate(y, gate) — one fused pass per sample for bf16 tensors.
    tr=(tr_gate, first_frame_mask): the I2V token-replace form (modulate_layers.py:84-95)."""
    if DN.gate_residual_supported(x, y, gate, tr=tr):
        STATS["gate_residual"] += 1
        return DN.gate_residual(x, y, gate, tr=tr)
    if tr is None:
        return x + mod.apply_gate(y, gate=gate)
    return x + mod.apply_gate(y, gate=gate, condition_type="token_replace", tr_gate=tr[0], first_frame_mask=tr[1])


def _fp8_routed(layer, k: int):
    """DN.fp8_weight(layer) when the opt-in FP8 Linears (DN.LINEAR_FP8) route `layer` on inputs of k
    channels — its K, and a shape in DN.FP8_ROUTED — else None"""
    if not (DN.LINEAR_FP8 and DN.FP8_ROUTED and isinstance(layer, torch.nn.Module)):
        return None
    # the table is consulted before fp8_weight, which quantises and caches: a layer the table does not
    # route never carries an e4m3 copy
    w = getattr(layer, "weight", None)
    if (not isinstance(w, torch.Tensor) or w.dim() != 2 or w.shape[1] != k
            or (DN.fp8_weight_kind(layer), k, w.shape[0]) not in DN.FP8_ROUTED):
        return None
    return DN.fp8_weight(layer)


def _fp8_weight(layer, x):
    """_fp8_routed(layer, K) on input x — a bf16 CUDA tensor with 16-byte aligned rows — else None"""
    if not (DN.LINEAR_FP8 and DN.FP8_ROUTED and isinstance(x, torch.Tensor) and x.is_cuda
            and x.dtype == torch.bfloat16 and x.dim() >= 2 and x.stride(-1) == 1 and x.stride(-2) % 8 == 0
            and x.data_ptr() % 16 == 0):
        return None
    return _fp8_routed(layer, x.shape[-1])


def _linear(layer, x, x8=None):
    """layer(x), or with the FP8 Linears on, one jenga_linear_fp8 launch on the e4m3 rows of x.
    x8: (codes, a_scale) of x made by the caller (ln_modulate_fp8), which has checked _fp8_weight."""
    w = _fp8_weight(layer, x)
    if w is None:
        return layer(x)
    if x8 is None:
        try:
            x8 = DN.quantize_rows_fp8(x)
        except ValueError:                   # rows that are not uniformly strided
            return layer(x)
    return _linear8(layer, x8, x.shape[:-1])


def _linear8(layer, x8, lead):
    """one jenga_linear_fp8 launch of `layer` on the e4m3 rows x8 = (codes, a_scale) a producer made; the
    caller has checked _fp8_routed.  -> bf16 [*lead, N]"""
    w = DN.fp8_weight(layer)
    STATS["linear_fp8"] += 1
    return DN.linear_fp8(*x8, *w).view(*lead, w[0].shape[0])


def _mod_linear(mod, layer, norm, x, shift, scale, tr=None):
    """layer(_ln_mod(...)); with the FP8 Linears on, the modulated rows go straight to e4m3
    (ln_modulate_fp8) and are never written in bf16"""
    if (_fp8_weight(layer, x) is not None and x.shape[-1] % 16 == 0
            and DN.ln_modulate_supported(x, norm, shift, scale, tr=tr)):
        STATS["ln_modulate"] += 1
        return _linear(layer, x, DN.ln_modulate_fp8(x, shift, scale, eps=norm.eps, tr=tr))
    return _linear(layer, _ln_mod(mod, norm, x, shift, scale, tr=tr))


def _plain_mlp(mlp) -> bool:
    """the reference MLP (hyvideo/modules/mlp_layers.py:13-58) with tanh-GELU, no norm and no dropout"""
    act, norm, d1, d2 = (getattr(mlp, n, None) for n in ("act", "norm", "drop1", "drop2"))
    return (type(mlp).__name__ == "MLP" and all(hasattr(mlp, n) for n in ("fc1", "fc2"))
            and "forward" not in mlp.__dict__ and not mlp._forward_hooks and not mlp._forward_pre_hooks
            and isinstance(act, torch.nn.GELU) and act.approximate == "tanh" and isinstance(norm, torch.nn.Identity)
            and all(isinstance(d, torch.nn.Dropout) and d.p == 0.0 for d in (d1, d2)))


def _plain_ffn(ffn) -> bool:
    """Wan's FFN as WanAttentionBlock builds it (model_mul.py:282-284): exactly
    Sequential(Linear, GELU(approximate="tanh"), Linear), with no hooks and no forward override"""
    if type(ffn) is not torch.nn.Sequential or len(ffn) != 3:
        return False
    f0, act, f2 = ffn
    return (type(f0) is torch.nn.Linear and type(f2) is torch.nn.Linear and type(act) is torch.nn.GELU
            and act.approximate == "tanh"
            and all("forward" not in m.__dict__ and not m._forward_hooks and not m._forward_pre_hooks
                    for m in (ffn, f0, act, f2)))


def _wan_ffn(blk, x, cross, e):
    """(r, ffn(norm2(r) * (1 + e[4]) + e[3])) with r = x + cross, the fp32 residual (model_mul.py:339-341).
    With the FP8 Linears on, a plain FFN is opened into ffn.0 -> GELU -> ffn.2: each routed Linear takes
    the e4m3 rows of its input from the pass that makes that input (wan_residual_ln_fp8, gelu_tanh_fp8)."""
    norm = dict(eps=blk.norm2.eps, shift=e[3], scale=e[4])
    if not (DN.LINEAR_FP8 and DN.FP8_ROUTED and _plain_ffn(blk.ffn)):
        x, h = DN.wan_residual_ln(x, cross, None, **norm)
        return x, blk.ffn(h)
    f0, act, f2 = blk.ffn
    lead = x.shape[:-1]
    if _fp8_rows((f0,), x):
        x, h8 = DN.wan_residual_ln_fp8(x, cross, None, **norm)
        a = _linear8(f0, h8, lead)
    else:
        x, h = DN.wan_residual_ln(x, cross, None, **norm)
        a = _linear(f0, h)
    F = a.shape[-1]
    if (a.dtype == torch.bfloat16 and a.is_contiguous() and F % 16 == 0 and F <= 16384
            and _fp8_routed(f2, F) is not None):
        return x, _linear8(f2, DN.gelu_tanh_fp8(a), lead)
    return x, _linear(f2, act(a))


def _mlp(mod, mlp, norm, x, shift, scale, tr=None):
    """mlp(_ln_mod(...)); with the FP8 Linears on, a plain MLP is opened into fc1 -> act -> fc2"""
    if DN.LINEAR_FP8 and DN.FP8_ROUTED and _plain_mlp(mlp):
        return _linear(mlp.fc2, mlp.act(_mod_linear(mod, mlp.fc1, norm, x, shift, scale, tr=tr)))
    return mlp(_ln_mod(mod, norm, x, shift, scale, tr=tr))


def _modulation(layer, vec, n, tr):
    """layer(vec).chunk(n): the block's (shift, scale, gate) triples.  Also returns, per triple, the
    token-replace arguments of _ln_mod and _gate_res — (tr_shift, tr_scale, first_frame_mask) and
    (tr_gate, first_frame_mask) — or None each without token replace (I2V models_mul.py:156-179,
    :413-424).  tr: (token_replace_vec, first_frame_mask) or None."""
    if tr is None:
        return layer(vec).chunk(n, dim=-1), [None] * (n // 3 * 2)
    token_replace_vec, mask = tr
    mods, tr_mods = layer(vec, condition_type="token_replace", token_replace_vec=token_replace_vec)
    r = tr_mods.chunk(n, dim=-1)
    args = []
    for i in range(0, n, 3):
        args += [(r[i], r[i + 1], mask), (r[i + 2], mask)]
    return mods.chunk(n, dim=-1), args


def _attention_section(self, mod, img_qkv, txt_qkv, norms, *, freqs_cis, cu_seqlens_q, cu_seqlens_kv,
                       sa_drop_rate, txt_amp, curve_sel, p_remain_rates, text_blocks, pad_ragged, out=None):
    """prologue -> (SP exchange | select + carved attention).  Returns attn [B, L+T, H*D]
    (written into `out`, a [B, L+T, H, D] view, when given and not under SP).
    pad_ragged: S = L+T need not be a multiple of 128 (the I2V operator zero-pads it).
    Under `jenga_sp` (the sharded I2V forward, hyi2v_sp.py) L is the rank's image slice."""
    (wq_i, eps), (wk_i, _), (wq_t, _), (wk_t, _) = norms
    L = img_qkv.shape[1]
    _, _, block_neighbor_list = mod.random.choice(curve_sel)                       # :232 / :438
    jsp = getattr(self, "jenga_sp", None)
    if jsp is not None:
        if (txt_qkv.shape[1] + HY.BLOCK - 1) // HY.BLOCK != text_blocks:
            # the Ulysses objects hand the operator ceil(T/128) text blocks; the I2V operator always
            # takes four (text_blocks=4), so the two agree only for 385 <= T <= 512 text tokens
            raise ValueError(f"sequence-parallel HunyuanVideo-I2V needs {text_blocks} text blocks "
                             f"({(text_blocks - 1) * HY.BLOCK + 1}..{text_blocks * HY.BLOCK} text tokens), "
                             f"got {txt_qkv.shape[1]} text tokens")
        # top_k is the single-GPU rule over the GLOBAL image length, not the T2V SP quirk
        # P*int((1-drop)*(L_loc//128)) (SURVEY a-7, App. A-12): the sharded I2V forward computes
        # what one GPU computes
        top_k = HY.select_block_num(sa_drop_rate, L * world(jsp.group)[0])
        q, k, v, _ = HY.attention_prologue(img_qkv, txt_qkv, self.heads_num, wq_i, wk_i, wq_t, wk_t, eps, freqs_cis,
                                           want_pool=False)
        # the I2V reference module has no my_parallel_attention: the restatement of attenion.py:159-195
        return U.my_parallel_attention(jsp, q, k, v, img_q_len=L, img_kv_len=L, cu_seqlens_q=cu_seqlens_q,
                                       cu_seqlens_kv=cu_seqlens_kv, top_k=top_k, text_amp=txt_amp,
                                       block_neighbor_list=block_neighbor_list, p_remain_rates=p_remain_rates)
    sp = getattr(self, "hybrid_seq_parallel_attn", None)
    top_k = HY.select_block_num(sa_drop_rate, L, mod.get_sequence_parallel_world_size() if sp else 1)  # :242, :249-251
    q, k, v, pools = HY.attention_prologue(img_qkv, txt_qkv, self.heads_num, wq_i, wk_i, wq_t, wk_t, eps, freqs_cis,
                                           want_pool=not sp)
    if sp:
        return mod.my_parallel_attention(sp, q, k, v, img_q_len=L, img_kv_len=L, cu_seqlens_q=cu_seqlens_q,
                                         cu_seqlens_kv=cu_seqlens_kv, top_k=top_k, text_amp=txt_amp,
                                         block_neighbor_list=block_neighbor_list,
                                         p_remain_rates=p_remain_rates)
    return HY.carved_attention_from_pools(q, k, v, pools, top_k=top_k, text_blocks=text_blocks,
                                          text_amp=txt_amp, block_neighbor_list=block_neighbor_list,
                                          p_remain_rates=p_remain_rates, cu_seqlens_q=cu_seqlens_q, out=out,
                                          pad_ragged=pad_ragged)


# ------------------------------------------------------------------------------------------------
# HunyuanVideo and HunyuanVideo-I2V blocks: one body per stream kind
# ------------------------------------------------------------------------------------------------
# The bodies return None when the call is not the carved configuration; _patched then runs the
# original forward.  The variants hand them what differs:
#   stat          the STATS key of the fused forward
#   tr            (token_replace_vec, first_frame_mask) for I2V token replace, else None
#   text_blocks   the operator's text_blocks: txt_block_num for HunyuanVideo, always 4 for I2V
#   pad_ragged    the I2V operator zero-pads S = L + T to whole blocks
#   ok            the variant's own eligibility rules
def _double_stream(mod, self, img, txt, vec, cu_seqlens_q, cu_seqlens_kv, freqs_cis, sa_drop_rate, txt_amp, curve_sel,
                   p_remain_rates, per_block_token, *, stat, tr, text_blocks, pad_ragged, ok):
    norms = [_rms_params(n) for n in (self.img_attn_q_norm, self.img_attn_k_norm,
                                      self.txt_attn_q_norm, self.txt_attn_k_norm)]
    if not (ok and _carved_call(self, img, norms, sa_drop_rate, curve_sel, cu_seqlens_q, per_block_token)):
        return None
    (i_shift1, i_scale1, i_gate1, i_shift2, i_scale2, i_gate2), (tr_mod1, tr_gate1, tr_mod2, tr_gate2) = \
        _modulation(self.img_mod, vec, 6, tr)
    t_shift1, t_scale1, t_gate1, t_shift2, t_scale2, t_gate2 = self.txt_mod(vec).chunk(6, dim=-1)
    img_qkv = _mod_linear(mod, self.img_attn_qkv, self.img_norm1, img, i_shift1, i_scale1, tr=tr_mod1)
    txt_qkv = self.txt_attn_qkv(_ln_mod(mod, self.txt_norm1, txt, t_shift1, t_scale1))
    assert cu_seqlens_q.shape[0] == 2 * img.shape[0] + 1                         # :244-246
    attn = _attention_section(self, mod, img_qkv, txt_qkv, norms, freqs_cis=freqs_cis, cu_seqlens_q=cu_seqlens_q,
                              cu_seqlens_kv=cu_seqlens_kv, sa_drop_rate=sa_drop_rate, txt_amp=txt_amp,
                              curve_sel=curve_sel, p_remain_rates=p_remain_rates, text_blocks=text_blocks,
                              pad_ragged=pad_ragged)
    STATS[stat] += 1
    L = img.shape[1]
    img_attn, txt_attn = attn[:, :L], attn[:, L:]
    img = _gate_res(mod, img, _linear(self.img_attn_proj, img_attn), i_gate1, tr=tr_gate1)   # :297-305
    img = _gate_res(mod, img, _mlp(mod, self.img_mlp, self.img_norm2, img, i_shift2, i_scale2, tr=tr_mod2),
                    i_gate2, tr=tr_gate2)
    txt = _gate_res(mod, txt, self.txt_attn_proj(txt_attn), t_gate1)                 # :307-315
    txt = _gate_res(mod, txt, self.txt_mlp(_ln_mod(mod, self.txt_norm2, txt, t_shift2, t_scale2)), t_gate2)
    return img, txt


def _single_stream(mod, self, x, vec, txt_len, cu_seqlens_q, cu_seqlens_kv, freqs_cis, sa_drop_rate, txt_amp,
                   curve_sel, p_remain_rates, per_block_token, *, stat, tr, text_blocks, pad_ragged, ok):
    norms = [_rms_params(n) for n in (self.q_norm, self.k_norm)]
    if not (ok and freqs_cis is not None
            and _carved_call(self, x, norms, sa_drop_rate, curve_sel, cu_seqlens_q, per_block_token)):
        return None
    (shift, scale, gate), (tr_mod, tr_gate) = _modulation(self.modulation, vec, 3, tr)
    lin1 = _mod_linear(mod, self.linear1, self.pre_norm, x, shift, scale, tr=tr_mod)
    C3 = 3 * self.hidden_size
    L = x.shape[1] - txt_len
    # strided views into linear1's output: no split / rearrange / cat copies (:413-441)
    img_qkv, txt_qkv = lin1[:, :L, :C3], lin1[:, L:, :C3]
    mlp = lin1[:, :, C3:]
    assert cu_seqlens_q.shape[0] == 2 * x.shape[0] + 1                           # :444-446
    # `torch.cat((attn, self.mlp_act(mlp)), 2)` (:499) without the concatenation copy: the attention
    # kernel writes its rows into the first `hidden` columns of linear2's input buffer and the
    # GELU kernel writes the rest.  At B > 1 sample b's attention rows start b*S*(C + mlp) elements in
    # (the kernel's o_stride_b); the GELU rows stay uniformly strided
    act = self.mlp_act
    fuse_cat = (isinstance(act, torch.nn.GELU) and getattr(act, "approximate", "none") == "tanh"
                and lin1.dtype == torch.bfloat16
                and not getattr(self, "hybrid_seq_parallel_attn", None) and getattr(self, "jenga_sp", None) is None)
    cat = attn_view = None
    if fuse_cat:
        cat = torch.empty((x.shape[0], x.shape[1], C3 // 3 + mlp.shape[-1]), dtype=lin1.dtype, device=lin1.device)
        attn_view = cat[:, :, :C3 // 3].unflatten(2, (self.heads_num, -1))
    attn = _attention_section(self, mod, img_qkv, txt_qkv, norms * 2, freqs_cis=freqs_cis, cu_seqlens_q=cu_seqlens_q,
                              cu_seqlens_kv=cu_seqlens_kv, sa_drop_rate=sa_drop_rate, txt_amp=txt_amp,
                              curve_sel=curve_sel, p_remain_rates=p_remain_rates, text_blocks=text_blocks,
                              pad_ragged=pad_ragged, out=attn_view)
    STATS[stat] += 1
    if fuse_cat:
        STATS["gelu_cat"] += 1
        DN.gelu_tanh_into(mlp, cat[:, :, C3 // 3:])
        out = _linear(self.linear2, cat)
    else:
        out = _linear(self.linear2, torch.cat((attn, act(mlp)), 2))
    return _gate_res(mod, x, out, gate, tr=tr_gate)                              # :500


def _hy_ok(self, S):
    # the HunyuanVideo operator needs whole blocks; under sequence parallel the exchange takes any S
    return bool(getattr(self, "hybrid_seq_parallel_attn", None)) or S % HY.BLOCK == 0


def _hy_double(mod, self, img, txt, vec, cu_seqlens_q=None, cu_seqlens_kv=None, max_seqlen_q=None,
               max_seqlen_kv=None, freqs_cis=None, sa_drop_rate=0.0, txt_amp=1.0, curve_sel=None,
               p_remain_rates=0.5, txt_block_num=2, per_block_token=128):
    return _double_stream(mod, self, img, txt, vec, cu_seqlens_q, cu_seqlens_kv, freqs_cis, sa_drop_rate, txt_amp,
                          curve_sel, p_remain_rates, per_block_token, stat="hy_double", tr=None,
                          text_blocks=txt_block_num, pad_ragged=False,
                          ok=_hy_ok(self, img.shape[1] + txt.shape[1]))


def _hy_single(mod, self, x, vec, txt_len, cu_seqlens_q=None, cu_seqlens_kv=None, max_seqlen_q=None,
               max_seqlen_kv=None, freqs_cis=None, sa_drop_rate=0.0, txt_amp=1.0, curve_sel=None,
               p_remain_rates=0.5, txt_block_num=2, per_block_token=128):
    return _single_stream(mod, self, x, vec, txt_len, cu_seqlens_q, cu_seqlens_kv, freqs_cis, sa_drop_rate, txt_amp,
                          curve_sel, p_remain_rates, per_block_token, stat="hy_single", tr=None,
                          text_blocks=txt_block_num, pad_ragged=False, ok=_hy_ok(self, x.shape[1]))


def _i2v_ok(self, L, T, condition_type, first_frame_mask):
    # the reference's sequence parallel (hybrid_seq_parallel_attn) runs the dense parallel_attention
    # (:264-274, :483-493): the original forward; `jenga_sp` is the sharded I2V forward of hyi2v_sp.py,
    # whose L is the rank's slice of the global image length; the prefix form of token replace
    # (frist_frame_token_num) is only reached outside the Jenga forward; with text_blocks=4 the
    # operator needs at least one image block
    if getattr(self, "hybrid_seq_parallel_attn", None):
        return False
    jsp = getattr(self, "jenga_sp", None)
    S = L * (world(jsp.group)[0] if jsp is not None else 1) + T
    return (not (condition_type == "token_replace" and first_frame_mask is None)
            and (S + HY.BLOCK - 1) // HY.BLOCK > _I2V_TEXT_BLOCKS)


def _i2v_stat(self, stat):
    return stat + "_sp" if getattr(self, "jenga_sp", None) is not None else stat


def _i2v_sharded_result(self, out):
    """the sharded I2V forward has no fall-back: the original forward would attend over the rank's
    rows alone"""
    if out is None and getattr(self, "jenga_sp", None) is not None and \
            not getattr(self, "hybrid_seq_parallel_attn", None):
        raise RuntimeError(f"{type(self).__name__} under jenga_sp: the call is not the carved configuration "
                           "(sa_drop_rate 0, no curve, no RMS qk-norm, head_dim != 128, or a dtype / device "
                           "the fused forward does not take); the sharded I2V forward has no fall-back")
    return out


def _i2v_tr(condition_type, token_replace_vec, first_frame_mask):
    return (token_replace_vec, first_frame_mask) if condition_type == "token_replace" else None


def _i2v_double(mod, self, img, txt, vec, cu_seqlens_q=None, cu_seqlens_kv=None, max_seqlen_q=None,
                max_seqlen_kv=None, freqs_cis=None, sa_drop_rate=0.0, first_frame_mask=None,
                condition_type=None, token_replace_vec=None, frist_frame_token_num=None, txt_amp=0.0,
                curve_sel=None, p_remain_rates=0.5, per_block_token=128):
    return _i2v_sharded_result(self, _double_stream(
        mod, self, img, txt, vec, cu_seqlens_q, cu_seqlens_kv, freqs_cis, sa_drop_rate, txt_amp, curve_sel,
        p_remain_rates, per_block_token, stat=_i2v_stat(self, "i2v_double"),
        tr=_i2v_tr(condition_type, token_replace_vec, first_frame_mask), text_blocks=_I2V_TEXT_BLOCKS,
        pad_ragged=True, ok=_i2v_ok(self, img.shape[1], txt.shape[1], condition_type, first_frame_mask)))


def _i2v_single(mod, self, x, vec, txt_len, cu_seqlens_q=None, cu_seqlens_kv=None, max_seqlen_q=None,
                max_seqlen_kv=None, freqs_cis=None, sa_drop_rate=0.0, first_frame_mask=None,
                condition_type=None, token_replace_vec=None, frist_frame_token_num=None, txt_amp=0.0,
                curve_sel=None, p_remain_rates=0.5, per_block_token=128):
    # first_frame_mask here is full_first_frame_mask (jenga_hyi2v.py:129-130): a CPU bool over L+T rows
    return _i2v_sharded_result(self, _single_stream(
        mod, self, x, vec, txt_len, cu_seqlens_q, cu_seqlens_kv, freqs_cis, sa_drop_rate, txt_amp, curve_sel,
        p_remain_rates, per_block_token, stat=_i2v_stat(self, "i2v_single"),
        tr=_i2v_tr(condition_type, token_replace_vec, first_frame_mask), text_blocks=_I2V_TEXT_BLOCKS,
        pad_ragged=True, ok=(_i2v_ok(self, x.shape[1] - txt_len, txt_len, condition_type, first_frame_mask)
                             and 0 < txt_len < x.shape[1])))


# ------------------------------------------------------------------------------------------------
# Wan blocks
# ------------------------------------------------------------------------------------------------
def _wan_rms(norm) -> bool:
    """the q / k norm the fused Wan prologues take: WanRMSNorm (model_mul.py:74-90) with a weight"""
    return type(norm).__name__ == "WanRMSNorm" and getattr(norm, "weight", None) is not None


def _wan_self_ok(self, x, per_block_tokens=128) -> bool:
    """the WanSelfAttention call _wan_self_fused takes, the Linears' output dtypes and the grid aside:
    any batch (every sample on one latent grid, _one_grid)"""
    return (x.is_cuda and self.head_dim == 128 and per_block_tokens == 128
            and _wan_rms(self.norm_q) and _wan_rms(self.norm_k))


def _one_grid(grid_sizes) -> bool:
    """every sample of the call on one latent grid: the fused self-attention reads grid_sizes[0] for all of
    them, as teacache_forward gathers every sample with the one curve (jenga_wan.py:559)"""
    return (isinstance(grid_sizes, torch.Tensor) and grid_sizes.dim() == 2 and grid_sizes.shape[0] >= 1
            and bool((grid_sizes == grid_sizes[:1]).all()))


def _check_one_grid(grid_sizes, what: str) -> None:
    """_one_grid, or the ValueError of a route without a fall-back"""
    if not _one_grid(grid_sizes):
        rows = grid_sizes.tolist() if isinstance(grid_sizes, torch.Tensor) else grid_sizes
        raise ValueError(f"{what}: the samples of one call must share one latent grid (one curve and one RoPE "
                         f"grid for all); got grid_sizes {rows}")


def _wan_self_fused(self, jsp, x, grid_sizes, freqs, sa_drop_rate, per_block_tokens, p_remain_rates, freq_remap,
                    block_neighbor_list, stats, x8=None, fallback=False):
    """WanSelfAttention.forward with the fused norm + RoPE prologue: the body of every fused Wan
    self-attention route (_wan_self, _wan_i2v_self).
    jsp set: x is a rank's n rows of a sharded Wan forward (wan_sp.py); the prologue runs on them, then
    the Ulysses exchange and the operator over the first L (the global token count) exchanged rows.
    jsp None: x is all L rows on one GPU; a carved call runs WAN.self_attention, a dense one the flash_attn
    shim's launch.  top_k and first_frame_blocks follow the single-GPU rule over L (model_mul.py:161-164);
    sa_drop_rate <= 0.25 (:153, the warm-up steps) is a dense call.  freq_remap: the RoPE row of each row
    (None: raster, one GPU only).  stats: the STATS keys of a carved and of a dense call.  x8: see _wan_qkv.
    x may hold several samples [B, n, C] on one latent grid (grid_sizes rows all equal): the prologue and
    the attention take the batch, and freq_remap is shared by every sample.
    A call it does not take raises, except with `fallback` (the one-GPU carved route of model_mul.py), where
    samples on different grids and a q Linear dtype the prologue does not take return None for the
    original forward, and v goes to the operator as the v Linear returns it (the operator casts it)."""
    b, n = x.shape[:2]
    if not _wan_self_ok(self, x, per_block_tokens) or (jsp is not None and freq_remap is None):
        raise RuntimeError(f"{type(self).__name__}: the call is not one the fused Wan self-attention takes (a "
                           "CUDA input, head_dim 128, 128-token blocks, WanRMSNorm q / k norms with "
                           "weights and, under jenga_sp, a freq_remap); this route has no fall-back")
    if fallback and not _one_grid(grid_sizes):
        return None
    _check_one_grid(grid_sizes, type(self).__name__)
    q_lin, k_lin, v = _wan_qkv(self, x, x8)
    if fallback:
        if q_lin.dtype not in (torch.bfloat16, torch.float32):
            return None
        v = v.view(b, n, self.num_heads, self.head_dim)
    elif q_lin.dtype not in (torch.bfloat16, torch.float32) or k_lin.dtype != q_lin.dtype:
        raise RuntimeError(f"{type(self).__name__}: q / k Linears return {q_lin.dtype}, the prologue takes bf16 "
                           "or fp32")
    else:
        # the bf16 v both single-GPU routes attend: flash_attention's half() and the operator's cast
        v = v.view(b, n, self.num_heads, self.head_dim).to(torch.bfloat16).contiguous()
    grid = [int(g) for g in grid_sizes[0].tolist()]
    L = grid[0] * grid[1] * grid[2]
    eps = float(self.norm_q.eps)
    wq, wk = self.norm_q.weight, self.norm_k.weight
    dense = sa_drop_rate <= 0.25
    if jsp is None and not dense:
        out = WAN.self_attention(q_lin, k_lin, v, wq, wk, self.num_heads, grid, freqs, sa_drop_rate,
                                 p_remain_rates=p_remain_rates, freq_remap=freq_remap,
                                 block_neighbor_list=block_neighbor_list, eps=eps)
    else:
        q = WAN.norm_rope(q_lin, wq, self.num_heads, grid, freqs, freq_remap, eps)
        k = WAN.norm_rope(k_lin, wk, self.num_heads, grid, freqs, freq_remap, eps)
        if jsp is None:
            out = flash_attn_func(q, k, v)
        else:
            top_k, ff = (0, 0) if dense else WAN.block_counts(L, sa_drop_rate)
            out = jsp(None, q, k, v, top_k=top_k, block_neighbor_list=None if dense else block_neighbor_list,
                      p_remain_rates=p_remain_rates, first_frame_blocks=ff, dense=dense, seq_len=L)
    STATS[stats[dense]] += 1
    out = out.flatten(2)
    if not torch.is_autocast_enabled():
        # the reference returns the query dtype, fp32 (rope_apply -> .float(), model_mul.py:71;
        # operator :530-532); under autocast the following Linear casts back to bf16 anyway
        out = out.float()
    return _linear(self.o, out)


def _wan_qkv(self, x, x8):
    """self.q(x), self.k(x), self.v(x); or, with x8 = (codes, a_scale) — the block's wan_ln_modulate_fp8
    rows, passed as `jenga_x8` with x their [1, n, C] e4m3 view — three FP8 GEMMs on the one input"""
    if x8 is None:
        return self.q(x), self.k(x), self.v(x)
    return tuple(_linear8(lin, x8, x.shape[:-1]) for lin in (self.q, self.k, self.v))


def _wan_self(self, x, seq_lens, grid_sizes, freqs, sa_drop_rate=0.0, per_block_tokens=128, p_remain_rates=0.8,
              freq_remap=None, block_neighbor_list=None, *, jenga_x8=None):
    """WanSelfAttention.forward of model_mul.py (:134-180).  Under `jenga_sp` (the Hilbert-sharded Wan
    forward of wan_sp.py) every call runs _wan_self_fused through the exchange, or raises; on one GPU the
    carved call does, and any other call runs the original forward.
    jenga_x8: the block's e4m3 q / k / v input (_wan_qkv), passed only when _wan_self_takes says so."""
    if not _wan_self_takes(self, x, sa_drop_rate, per_block_tokens):
        return None
    jsp = getattr(self, "jenga_sp", None)
    stats = ("wan_self_sp", "wan_self_dense_sp") if jsp is not None else ("wan_self", None)
    return _wan_self_fused(self, jsp, x, grid_sizes, freqs, sa_drop_rate, per_block_tokens, p_remain_rates,
                           freq_remap, block_neighbor_list, stats, x8=jenga_x8, fallback=jsp is None)


def _wan_self_takes(self, x, sa_drop_rate=0.0, per_block_tokens=128, **_):
    """True when _wan_self runs _wan_self_fused rather than the original forward: under jenga_sp, or for
    the carved call (sa_drop_rate > 0.25) on one GPU"""
    return getattr(self, "jenga_sp", None) is not None or (
        sa_drop_rate > 0.25 and _wan_self_ok(self, x, per_block_tokens))


def _wan_i2v_self(self, x, seq_lens, grid_sizes, freqs, sa_drop_rate=None, freq_remap=None, block_neighbor_list=None,
                  p_remain_rates=0.8, *, jenga_x8=None):
    """WanSelfAttention.forward of wan/modules/model.py (:127-156).  Called in that module's signature
    (sa_drop_rate None):
      under `jenga_sp` (the raster-sharded I2V forward, wan_sp.parallelize_wan_i2v) x holds rank r's n
      rows [r*n, min((r+1)*n, L)): the fused prologue runs on them with that raster slice as the RoPE index
      (pad rows index row 0), then the dense class over the first L exchanged rows, so the pad keys are
      excluded as flash_attention(k_lens=seq_lens) excludes them on one GPU;
      without jenga_sp: the original forward.
    With the Jenga arguments of model_mul.py (the I2V forwards of wan_sp.py): _wan_self_fused, on one GPU
    or under jenga_sp.  A call it does not take runs the original forward on raster rows (freq_remap None)
    and raises on curve-ordered rows, whose RoPE positions the original forward does not know.
    jenga_x8: the block's e4m3 q / k / v input (_wan_qkv), passed only when _wan_i2v_self_takes says so."""
    if not _wan_i2v_self_takes(self, x, sa_drop_rate, freq_remap):
        if sa_drop_rate is None:
            return None
        STATS["fallback"] += 1
        return type(self).forward.__wrapped__(self, x, seq_lens, grid_sizes, freqs)
    jsp = getattr(self, "jenga_sp", None)
    if jsp is None:
        stats = ("wan_i2v_self", "wan_i2v_self_dense")
    elif sa_drop_rate is not None:
        stats = ("wan_i2v_self_carved_sp", "wan_i2v_self_sp")
    else:
        _, r = world(jsp.group)
        n = x.shape[1]
        L = int(torch.prod(grid_sizes[0]))
        rows = torch.arange(r * n, (r + 1) * n, device=x.device)
        freq_remap = torch.where(rows < L, rows, torch.zeros_like(rows))
        sa_drop_rate, p_remain_rates, stats = 0.0, 0.0, (None, "wan_i2v_self_sp")
    return _wan_self_fused(self, jsp, x, grid_sizes, freqs, sa_drop_rate, 128, p_remain_rates, freq_remap,
                           block_neighbor_list, stats, x8=jenga_x8)


def _wan_i2v_self_takes(self, x, sa_drop_rate=None, freq_remap=None, **_):
    """True when _wan_i2v_self runs _wan_self_fused (or raises) rather than the original forward: under
    jenga_sp, or with the Jenga arguments on curve-ordered rows or for a call _wan_self_fused takes"""
    return getattr(self, "jenga_sp", None) is not None or (
        sa_drop_rate is not None and (freq_remap is not None or _wan_self_ok(self, x)))


def _wan_cross_takes(self, x, context, context_lens):
    """True when _wan_cross runs the fused T2V cross-attention (the Linears' output dtypes aside): x
    [B, L, C] and context [B, Lc, C] of one batch, each sample attending its own context rows"""
    # context_lens: the reference's varlen form (wan/modules/attention.py:69-80); teacache_forward
    # passes None (jenga_wan.py:569)
    return (context_lens is None and x.is_cuda and x.dim() == 3 and context.dim() == 3
            and context.shape[0] == x.shape[0] and DN.distinct_samples(x, context) and self.head_dim == 128
            and _wan_rms(self.norm_q) and _wan_rms(self.norm_k) and DN._autocast_bf16())


def _wan_cross(self, x, context, context_lens, *, jenga_x8=None):
    """jenga_x8: the block's wan_residual_ln_fp8 rows of x (x their e4m3 view) for the q Linear, passed only
    when _wan_cross_takes says so"""
    if not _wan_cross_takes(self, x, context, context_lens):
        return None
    q_lin = self.q(x) if jenga_x8 is None else _linear8(self.q, jenga_x8, x.shape[:-1])
    k_lin, v = self.k(context), self.v(context)
    if (q_lin.dtype not in (torch.bfloat16, torch.float32) or k_lin.dtype not in (torch.bfloat16, torch.float32)
            or v.dtype != torch.bfloat16):
        if jenga_x8 is not None:
            raise RuntimeError(f"{type(self).__name__}: k / v Linears return {k_lin.dtype} / {v.dtype} under bf16 "
                               "autocast; the e4m3 q input has no fall-back")
        return None
    out = WAN.cross_attention(q_lin, k_lin, v.view(x.shape[0], -1, self.num_heads, self.head_dim),
                              self.norm_q.weight, self.norm_k.weight, self.num_heads, eps=float(self.norm_q.eps))
    STATS["wan_cross"] += 1
    return _linear(self.o, out.flatten(2))


def _wan_i2v_cross_shape_ok(ca, x, context, context_lens):
    """the I2V cross-attention configuration the fused kernel takes, device and autocast aside: a context
    of x's batch, each sample attending its own context rows, every one valid (teacache_forward passes
    context_lens=None, jenga_wan.py:569), head_dim 128, WanRMSNorm q / k / k_img norms with weights and one
    eps, and text rows after the image rows"""
    norms = [getattr(ca, n, None) for n in ("norm_q", "norm_k", "norm_k_img")]
    return (context_lens is None and isinstance(x, torch.Tensor) and isinstance(context, torch.Tensor)
            and x.dim() == 3 and context.dim() == 3 and context.shape[0] == x.shape[0]
            and DN.distinct_samples(x, context)
            and context.shape[1] > _WAN_I2V_IMG_TOKENS and getattr(ca, "head_dim", None) == 128
            and all(_wan_rms(n) for n in norms)
            and len({float(n.eps) for n in norms}) == 1)


def wan_i2v_cross_eligible(ca, x, context, context_lens):
    """True when the fused block runs WanI2VCrossAttention `ca` as i2v_cross_attention: the shape rules
    above, CUDA tensors and bf16 autocast"""
    return _wan_i2v_cross_shape_ok(ca, x, context, context_lens) and x.is_cuda and DN._autocast_bf16()


def _wan_i2v_cross(ca, x, context, context_lens, stat="wan_i2v_cross", x8=None):
    """WanI2VCrossAttention.forward (model_mul.py:223-249) with its attention part as one
    jenga_wan_i2v_cross_attn launch; the module's own q / k / v / k_img / v_img / o Linears run around
    it (q and o through _linear: the k / v / k_img / v_img Linears over the context rows are never
    FP8).  Anything else runs the module's own forward.  x8: the block's wan_residual_ln_fp8 rows of x
    (x their e4m3 view) for q, passed only when wan_i2v_cross_eligible."""
    if wan_i2v_cross_eligible(ca, x, context, context_lens):
        ctx_img, ctx = context[:, :_WAN_I2V_IMG_TOKENS], context[:, _WAN_I2V_IMG_TOKENS:]   # :230-231
        q_lin = ca.q(x) if x8 is None else _linear8(ca.q, x8, x.shape[:-1])
        k_lin, v = ca.k(ctx), ca.v(ctx)
        kimg_lin, vimg = ca.k_img(ctx_img), ca.v_img(ctx_img)
        lin_ok = all(t.dtype in (torch.bfloat16, torch.float32) for t in (q_lin, k_lin, kimg_lin))
        if lin_ok and v.dtype == vimg.dtype == torch.bfloat16:
            b, n = x.shape[0], ca.num_heads
            out = WAN.i2v_cross_attention(q_lin, k_lin, v.view(b, -1, n, 128), kimg_lin, vimg.view(b, -1, n, 128),
                                          ca.norm_q.weight, ca.norm_k.weight, ca.norm_k_img.weight, n,
                                          eps=float(ca.norm_q.eps))
            STATS[stat] += 1
            return _linear(ca.o, out.flatten(2))
        if x8 is not None:
            raise RuntimeError(f"{type(ca).__name__}: context Linears return {k_lin.dtype} / {v.dtype} under bf16 "
                               "autocast; the e4m3 q input has no fall-back")
    STATS["fallback"] += 1
    return ca(x, context, context_lens)


def _wan_block(plain, self, x, e, seq_lens, grid_sizes, freqs, context, context_lens, sa_drop_rate=0.0,
               freq_remap=None, block_neighbor_list=None, p_remain_rates=0.0):
    """WanAttentionBlock.forward of model_mul.py (:303-346), or, `plain`, of wan/modules/model.py (:274-313),
    whose own signature (sa_drop_rate None) hands the self-attention (x, seq_lens, grid_sizes, freqs) and
    whose I2V forwards in wan_sp.py pass the Jenga arguments of model_mul.py.  A call the fused body does
    not take runs the original forward, except on a plain block:
      under `self_attn.jenga_sp` (parallelize_wan_i2v) x is a rank's rows and there is no fall-back: the
      checks run before the exchange, so every rank raises alike;
      with the Jenga arguments, the original forward runs on raster rows, in model.py's own signature, and
      the block raises on curve-ordered rows (freq_remap set), whose RoPE positions it does not know.
    x may hold several samples [B, L, C] with `e` [B, 6, C] (or [1, 6, C], shared) and a context of the same
    batch; all of them on one latent grid.  Samples on different grids run the original forward, or raise
    ValueError where there is none (the sharded rows, the curve-ordered rows)."""
    attn_kw = {} if plain and sa_drop_rate is None else dict(
        sa_drop_rate=sa_drop_rate, freq_remap=freq_remap, block_neighbor_list=block_neighbor_list,
        p_remain_rates=p_remain_rates)
    sharded = plain and getattr(self.self_attn, "jenga_sp", None) is not None
    if sharded or (plain and freq_remap is not None):
        _check_one_grid(grid_sizes, type(self).__name__)
    if sharded and not (type(self.cross_attn).__name__ == "WanI2VCrossAttention"
                        and _wan_i2v_cross_shape_ok(self.cross_attn, x, context, context_lens)):
        raise RuntimeError(f"{type(self).__name__} under jenga_sp: the cross-attention is not one the fused I2V "
                           "kernel takes (a WanI2VCrossAttention with WanRMSNorm q / k / k_img norms, head_dim "
                           f"128, a context of x's batch, context_lens None and more than {_WAN_I2V_IMG_TOKENS} "
                           "context rows); the sharded I2V forward has no fall-back")
    out = _wan_block_body(self, x, e, seq_lens, grid_sizes, freqs, context, context_lens, attn_kw, sharded)
    if out is None and sharded:
        raise RuntimeError(f"{type(self).__name__} under jenga_sp: the call is not one the fused block takes (a "
                           "CUDA input under bf16 autocast, fp32 modulation, cross_attn_norm=True); the sharded "
                           "I2V forward has no fall-back")
    if out is not None or not (plain and attn_kw):
        return out                      # None: the original forward with the caller's arguments (_patched)
    if freq_remap is not None:
        raise RuntimeError(f"{type(self).__name__}: the call is not one the fused block takes (a CUDA input "
                           "under bf16 autocast, fp32 modulation, cross_attn_norm=True); the original forward "
                           "cannot take the curve-ordered rows of the carved I2V forward")
    STATS["fallback"] += 1
    return type(self).forward.__wrapped__(self, x, e, seq_lens, grid_sizes, freqs, context, context_lens)


def _wan_block_body(self, x, e, seq_lens, grid_sizes, freqs, context, context_lens, attn_kw, sharded):
    """The fused block forward, or None for a call it does not take.  attn_kw: the Jenga self-attention
    arguments of model_mul.py (empty for wan/modules/model.py called in its own signature).
    sharded: the I2V rows of parallelize_wan_i2v; the cross-attention must then be the fused one."""
    i2v = type(self.cross_attn).__name__ == "WanI2VCrossAttention"
    ok = (isinstance(e, torch.Tensor) and e.dtype == torch.float32 and x.is_cuda and x.dim() == 3
          and _one_grid(grid_sizes) and (i2v or type(self.cross_attn).__name__ == "WanT2VCrossAttention")
          and self.modulation.dtype == torch.float32
          and (not sharded or wan_i2v_cross_eligible(self.cross_attn, x, context, context_lens)))
    if ok:
        with torch.autocast("cuda", dtype=torch.float32):                      # :326-327
            e6 = self.modulation + e
        ok = (DN.wan_ln_modulate_supported(x, self.norm1, e6)
              and DN.wan_residual_ln_supported(x, self.norm3, e6, affine=True)
              and DN.wan_residual_ln_supported(x, self.norm2, e6, affine=False)
              and DN.wan_gate_residual_supported(x, e6))
    if not ok:
        return None                     # no autocast, several grids, cross_attn_norm=False (norm3 is Identity), …
    e = e6.chunk(6, dim=1)
    # self-attention on the bf16 its q / k / v Linears would cast the fp32 modulate output to; with the
    # FP8 Linears routing q / k / v, on the e4m3 rows of that bf16 instead (:331-333)
    sa, ca = self.self_attn, self.cross_attn
    if _fp8_rows((sa.q, sa.k, sa.v), x) and _fused_forward(sa, x, **attn_kw):
        x8 = DN.wan_ln_modulate_fp8(x, e[0], e[1], eps=self.norm1.eps)
        y = sa(x8[0].view(x.shape), seq_lens, grid_sizes, freqs, jenga_x8=x8, **attn_kw)
    else:
        y = sa(DN.wan_ln_modulate(x, e[0], e[1], eps=self.norm1.eps), seq_lens, grid_sizes, freqs, **attn_kw)
    # gate 1 + norm3 (:334-335, :339), e4m3 when the cross-attention's q is routed
    x8 = None
    if _fp8_rows((ca.q,), x) and (wan_i2v_cross_eligible(ca, x, context, context_lens) if i2v else
                                  _fused_forward(ca, x, context, context_lens)):
        x, x8 = DN.wan_residual_ln_fp8(x, y, e[2], eps=self.norm3.eps, weight=self.norm3.weight, bias=self.norm3.bias)
        h = x8[0].view(x.shape)
    else:
        x, h = DN.wan_residual_ln(x, y, e[2], eps=self.norm3.eps, weight=self.norm3.weight, bias=self.norm3.bias)
    # WanI2VCrossAttention.forward itself stays unpatched: the block routes it here
    if i2v:
        cross = _wan_i2v_cross(ca, h, context, context_lens,
                               stat="wan_i2v_cross_sp" if sharded else "wan_i2v_cross", x8=x8)
    else:
        cross = ca(h, context, context_lens) if x8 is None else ca(h, context, context_lens, jenga_x8=x8)
    STATS["wan_block"] += 1
    x, y = _wan_ffn(self, x, cross, e)                                         # :339-342
    return DN.wan_gate_residual(x, y, e[5])


def _fp8_rows(layers, x) -> bool:
    """True when the FP8 Linears route every one of `layers` on the rows of the Wan residual stream x
    (C % 16 == 0): the block then makes their one e4m3 input with a wan_*_fp8 producer"""
    return x.shape[-1] % 16 == 0 and all(_fp8_routed(lin, x.shape[-1]) is not None for lin in layers)


def _fused_forward(module, *args, **kwargs) -> bool:
    """True when `module`'s forward is one jenga_b200 patched in (not an instance override) and the
    predicate _patched stored on it takes the call, called as takes(module, *args, **kwargs).  Only such a
    forward is handed e4m3 rows (`jenga_x8`); one with no predicate never is."""
    fwd = type(module).forward
    if "forward" in module.__dict__ or not getattr(fwd, "__jenga_b200__", False):
        return False
    takes = getattr(fwd, "__jenga_takes__", None)
    return takes is not None and takes(module, *args, **kwargs)


# ------------------------------------------------------------------------------------------------
# patching
# ------------------------------------------------------------------------------------------------
def _swap(owner, attr: str, replacement) -> bool:
    """Sets owner.attr = replacement, marked as jenga_b200's (`__jenga_b200__`) with the original as its
    `__wrapped__`.  False, and nothing changes, when owner has no such attribute or it is swapped already."""
    orig = getattr(owner, attr, None)
    if orig is None or getattr(orig, "__jenga_b200__", False):
        return False
    replacement.__jenga_b200__ = True
    replacement.__wrapped__ = orig
    setattr(owner, attr, replacement)
    return True


def _unswap(owner, *attrs: str) -> None:
    """Puts back the originals that _swap replaced, where owner.attr is swapped"""
    for attr in attrs:
        fn = getattr(owner, attr, None)
        if getattr(fn, "__jenga_b200__", False):
            setattr(owner, attr, fn.__wrapped__)


def _patched(orig, fused, takes=None):
    """The patched forward: `fused` takes the reference arguments and returns None for a call it does
    not take; that call then runs `orig` with exactly the caller's arguments.  takes(module, *args,
    **kwargs): True when `fused` runs its fused body on the call, the Linears' output dtypes aside; it is
    stored on the forward for _fused_forward."""
    def forward(self, *args, **kwargs):
        out = fused(self, *args, **kwargs)
        if out is None:
            STATS["fallback"] += 1
            out = orig(self, *args, **kwargs)
        return out
    forward.__jenga_takes__ = takes
    return forward


def _patch_classes(mod, fused) -> list[str]:
    """fused: class name -> (fused body, its predicate or None), see _patched"""
    done = []
    for cls, (body, takes) in fused.items():
        owner = getattr(mod, cls, None)
        if owner is not None and _swap(owner, "forward", _patched(owner.forward, body, takes)):
            done.append(f"{mod.__name__}.{cls}.forward")
    return done


def _patch_hy(double, single):
    """the patch of a HunyuanVideo block module: both stream kinds, with the module's own helpers"""
    return lambda mod: _patch_classes(mod, dict(MMDoubleStreamBlock=(functools.partial(double, mod), None),
                                                MMSingleStreamBlock=(functools.partial(single, mod), None)))


def patch_plain_wan(mod) -> list[str]:
    """Patches WanSelfAttention / WanAttentionBlock of wan/modules/model.py: the block hands its
    self-attention (x, seq_lens, grid_sizes, freqs), or the Jenga arguments the I2V forwards of wan_sp.py
    pass, and runs the fused I2V cross-attention; WanT2VCrossAttention and WanI2VCrossAttention stay as
    they are"""
    # model.py's own signature has no Jenga arguments: sa_drop_rate None stands for it
    block = functools.partial(_wan_block, True, sa_drop_rate=None, p_remain_rates=0.8)
    return _patch_classes(mod, dict(WanSelfAttention=(_wan_i2v_self, _wan_i2v_self_takes),
                                    WanAttentionBlock=(block, None)))


def _unpatch_plain_wan(mod) -> None:
    for cls in ("WanSelfAttention", "WanAttentionBlock"):
        _unswap(getattr(mod, cls, None), "forward")


def _wrap_wan_i2v_init(mod) -> list[str]:
    """WanI2V.__init__ of wan/image2video.py, followed, for a pipeline built with use_usp=False, by
    wan_sp.bind_wan_i2v on its WanModel: the single-GPU I2V forward.  With use_usp=True the pipeline keeps
    what it bound (usp_dit_forward; install(wan_sp=True) decides what that is)."""
    cls = getattr(mod, "WanI2V", None)
    if cls is None:
        return []
    orig = cls.__init__

    @functools.wraps(orig)
    def __init__(self, *args, **kwargs):
        orig(self, *args, **kwargs)
        # a dit_fsdp model is an FSDP wrapper, whose forward gathers the parameters: left as it is
        if not getattr(self, "use_usp", False) and type(self.model).__name__ == "WanModel":
            wan_sp.bind_wan_i2v(self.model)

    return [f"{mod.__name__}.WanI2V.__init__"] if _swap(cls, "__init__", __init__) else []


class _Hook(NamedTuple):
    patch: Callable[..., list[str]]             # module -> what it patched
    label: str                                  # the route the stderr line names
    switch: str | None = None                   # the global (I2V_SP, WAN_SP) of an opt-in route; None: always on
    restore: Callable[..., None] | None = None  # module -> None: undoes `patch` when the switch is turned off


_FUSED = "fused attention section"
# every module the import hook patches right after it is executed
_HOOKS = {
    "hyvideo.modules.models_mul_block_gc_ha_multigpu": _Hook(_patch_hy(_hy_double, _hy_single), _FUSED),
    # hyvideo_i2v/modules/models_mul.py has its own argument order, the token_replace modulation and a
    # ragged S with four text blocks: its own pair of entry points
    "hyvideo_i2v.modules.models_mul": _Hook(_patch_hy(_i2v_double, _i2v_single), _FUSED),
    # WanI2VCrossAttention overrides forward itself and is left as it is; the fused block forward runs
    # its fused form (_wan_i2v_cross)
    "wan.modules.model_mul": _Hook(lambda mod: _patch_classes(mod, dict(
        WanSelfAttention=(_wan_self, _wan_self_takes), WanT2VCrossAttention=(_wan_cross, _wan_cross_takes),
        WanAttentionBlock=(functools.partial(_wan_block, False), None))), _FUSED),
    # WanI2V(use_usp=False) gets the single-GPU I2V forward of wan_sp.py, and the plain model's blocks the
    # fused forwards, when the pipeline is built (wan.modules.model itself, which only WanI2V imports,
    # stays untouched at import without the Wan switch).  Not undone by set_wan_sp(False).
    "wan.image2video": _Hook(_wrap_wan_i2v_init, "single-GPU Wan I2V route"),
    # parallelize_transformer is swapped for the Hilbert-sharded forward of hyi2v_sp.py
    "hyvideo_i2v.inference": _Hook(hyi2v_sp.install_parallelize_transformer, "sequence-parallel I2V route",
                                   "I2V_SP", lambda mod: _unswap(mod, "parallelize_transformer")),
    # usp_dit_forward / usp_attn_forward are swapped for the Hilbert-sharded TeaCache forward of wan_sp.py
    "wan.distributed.xdit_context_parallel": _Hook(
        wan_sp.install_usp, "sequence-parallel Wan route", "WAN_SP",
        lambda mod: _unswap(mod, "usp_dit_forward", "usp_attn_forward")),
    # wan/modules/model.py, the plain Wan model WanI2V loads (image2video.py:21), gets the fused
    # WanAttentionBlock.forward and a WanSelfAttention.forward for its signatures
    "wan.modules.model": _Hook(patch_plain_wan, _FUSED, "WAN_SP", _unpatch_plain_wan),
}


def _active_hook(name: str) -> _Hook | None:
    """the hook of module `name` when there is one and its route is on"""
    hook = _HOOKS.get(name)
    return hook if hook is not None and (hook.switch is None or globals()[hook.switch]) else None


def patch_module(mod) -> list[str]:
    """Patches an already imported reference module by its hook; returns what it did."""
    hook = _active_hook(mod.__name__)
    return hook.patch(mod) if hook is not None else []


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
            print(f"[jenga_b200] {_HOOKS[module.__name__].label} installed: {', '.join(done)}", file=sys.stderr)

    def __getattr__(self, item):
        return getattr(self.inner, item)


class _PatchFinder(importlib.abc.MetaPathFinder):
    targets = tuple(_HOOKS)

    def find_spec(self, fullname, path, target=None):
        if _active_hook(fullname) is None:
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
