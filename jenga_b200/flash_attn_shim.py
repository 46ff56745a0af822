"""FlashAttention call sites of the hot path, served by the dense mode of the sm_90a kernel.

Shadows exactly what the reference imports (SURVEY §8b):
  flash_attn.flash_attn_func                       attention_block_triton_diffres.py:15,377
  flash_attn.flash_attn_interface.flash_attn_varlen_func   hyvideo/modules/attenion.py:11,109-117;
                                                           wan/modules/attention.py:113-125
  flash_attn.flash_attn_interface._flash_attn_forward      attenion.py:221-246, xdit_ring_atten.py:302-327
                                                           (out + softmax_lse)
  flash_attn.__version__                                   attenion.py:220
Forward only, no dropout, non-causal; anything else raises instead of silently doing something
different.  Every DiT call has head_dim 128 and launches the kernel on the caller's tensors.
install() replaces flash_attn for the whole process, so calls outside the DiT arrive here too: the
Wan2.1-I2V CLIP image encoder (wan/modules/clip.py:85, ViT-H/14, 16 heads of 80 channels, 257
tokens, fp16) calls flash_attn_varlen_func in every layer, once per video.  Head dims below 128
(multiples of 8, shared by q, k and v) are served by zero-padding the channels to 128
(`_pad_head_dim`) and slicing the output: zero channels add nothing to Q.K^T and give zero output
columns.  The default softmax scale stays the caller's D ** -0.5.  The C-ABI stays at head_dim 128.

The opt-in switches of the operator apply here too, read at call time: `attention.QK_INT8`
(JENGA_QK_INT8=1; bf16 / fp16) runs Q.K^T in int8 with K smoothing, and `attention.PV_FP8`
(JENGA_PV_FP8=1; bf16 only, like the operator) runs P.V in e4m3.  Each launched segment is quantised
on its own.  _flash_attn_forward's softmax_lse stays the LSE of the unsmoothed scores: the kernel
adds back the per-row shift that K smoothing takes off.
"""
from __future__ import annotations

import torch

from . import attention as A
from .attention import BLOCK, _launch, _require_cuda

__version__ = "2.8.3+jenga_b200"
HEAD_DIM = 128   # the only head dim the kernel is built for


def _check(q, k, v, dropout_p, causal, window_size, alibi_slopes):
    _require_cuda(q, k, v)
    if dropout_p not in (0, 0.0):
        raise NotImplementedError("dropout is not built (inference path)")
    if causal:
        raise NotImplementedError("causal attention is not on the Jenga hot path")
    if window_size not in ((-1, -1), None) or alibi_slopes is not None:
        raise NotImplementedError("window / alibi are not built")
    D = q.shape[-1]
    if k.shape[-1] != D or v.shape[-1] != D:
        raise NotImplementedError(f"q, k and v must share one head_dim (got {D}, {k.shape[-1]}, {v.shape[-1]})")
    if D % 8 or not 8 <= D <= HEAD_DIM:
        raise NotImplementedError(f"head_dim {D} is not built (only multiples of 8 up to {HEAD_DIM})")


def _pad_head_dim(q, k, v):
    """q, k, v with their channels zero-padded to HEAD_DIM (one copy each).  The quantisers of the
    opt-in switches see the padded tensors: a zero channel quantises to zero, and its K mean is zero."""
    return tuple(torch.nn.functional.pad(t, (0, HEAD_DIM - t.shape[-1])) for t in (q, k, v))


def _dense(q, k, v, softmax_scale, out=None, lse=None):
    """q [B,Sq,H,D], k/v [B,Sk,H,D] -> [B,Sq,H,D]"""
    B, Sq, H, D = q.shape
    scale = D ** -0.5 if softmax_scale is None else float(softmax_scale)
    if D != HEAD_DIM:
        assert out is None, "flash_attn_varlen_func pads before it hands _dense its segments"
        return _dense(*_pad_head_dim(q, k, v), scale, lse=lse)[..., :D].contiguous()
    Sk = k.shape[1]
    if out is None:
        out = torch.empty((B, Sq, H, D), dtype=q.dtype, device=q.device)
    v8, qk8 = A.quantize_operands(q, k, v, A.PV_FP8, A.QK_INT8, lse_shift=lse is not None)
    _launch(q, k, v, None, 0, (Sq + BLOCK - 1) // BLOCK, scale, 0.0, 1 << 30, Sk, Sq, Sk, out, None,
            q.dtype, lse_out=lse, v_fp8=v8, qk_int8=qk8)
    return out


def flash_attn_func(q, k, v, dropout_p=0.0, softmax_scale=None, causal=False, window_size=(-1, -1),
                    softcap=0.0, alibi_slopes=None, deterministic=False, return_attn_probs=False):
    _check(q, k, v, dropout_p, causal, window_size, alibi_slopes)
    if softcap not in (0, 0.0) or return_attn_probs:
        raise NotImplementedError("softcap / return_attn_probs are not built")
    return _dense(q, k, v, softmax_scale)


def flash_attn_varlen_func(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k,
                           dropout_p=0.0, softmax_scale=None, causal=False, window_size=(-1, -1),
                           softcap=0.0, alibi_slopes=None, deterministic=False,
                           return_attn_probs=False, block_table=None):
    """q,k,v [(total tokens), H, D]; one dense launch per (q segment, k segment) pair.
    The segment table is read on the host (one small D2H copy) — this is the reference's
    sa_drop_rate == 0 fallback (models_mul…:254-258), not the carved path.  Head dims below 128
    (the CLIP encoder, wan/modules/clip.py:85) are padded once for all segments."""
    _check(q, k, v, dropout_p, causal, window_size, alibi_slopes)
    if block_table is not None or softcap not in (0, 0.0) or return_attn_probs:
        raise NotImplementedError
    cq = cu_seqlens_q.tolist()
    ck = cu_seqlens_k.tolist()
    if len(cq) != len(ck):
        raise ValueError("cu_seqlens_q / cu_seqlens_k length mismatch")
    D = q.shape[-1]
    if D != HEAD_DIM:
        softmax_scale = D ** -0.5 if softmax_scale is None else softmax_scale
        q, k, v = _pad_head_dim(q, k, v)
    out = torch.zeros_like(q)
    for i in range(len(cq) - 1):
        q0, q1, k0, k1 = cq[i], cq[i + 1], ck[i], ck[i + 1]
        if q1 <= q0:
            continue
        if k1 <= k0:
            continue  # no keys: FlashAttention returns zeros for the segment
        _dense(q[q0:q1].unsqueeze(0), k[k0:k1].unsqueeze(0), v[k0:k1].unsqueeze(0), softmax_scale,
               out=out[q0:q1].unsqueeze(0))
    return out if D == HEAD_DIM else out[..., :D].contiguous()


def _flash_attn_forward(q, k, v, dropout_p=0.0, softmax_scale=None, causal=False, window_size=(-1, -1),
                        softcap=0.0, alibi_slopes=None, return_softmax=False, window_size_left=-1,
                        window_size_right=-1, **kw):
    """flash_attn.flash_attn_interface._flash_attn_forward as hyvideo/modules/attenion.py:221-246 and
    xdit_ring_atten.py:302-327 call it (both the >=2.7 `window_size_left/right` and the older
    `window_size` keyword forms): returns (out, softmax_lse, S_dmask, rng_state) with
    softmax_lse fp32 [B, H, Sq] (natural log) written by the dense class of the attention kernel."""
    ws = window_size if window_size is not None else (-1, -1)
    if (window_size_left, window_size_right) != (-1, -1):
        ws = (window_size_left, window_size_right)
    _check(q, k, v, dropout_p, causal, ws, alibi_slopes)
    if softcap not in (0, 0.0) or return_softmax:
        raise NotImplementedError("softcap / return_softmax are not built")
    B, Sq, H, D = q.shape
    lse = torch.empty((B, H, Sq), dtype=torch.float32, device=q.device)
    out = _dense(q, k, v, softmax_scale, lse=lse)
    return out, lse, None, None
