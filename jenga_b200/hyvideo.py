"""HunyuanVideo-side glue of the hot path: the fused attention prologue and the block-level
call sequence of MMDoubleStreamBlock / MMSingleStreamBlock
(hyvideo/modules/models_mul_block_gc_ha_multigpu.py:161-316, :392-500), token gather/scatter
(jenga_hyvideo.py:116-118, :226) and select_block_num (:229,:242).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import check, lib
from .attention import (BLOCK, _dtype_code, _require_cuda, _stream_ptr, _launch, neighbour_bits,
                        select_blocks)


def select_block_num(sa_drop_rate: float, img_tokens: int, world_size: int = 1) -> int:
    """models_mul…:242 `int((1-sa_drop_rate) * img_block_num)` (x world_size under SP, :249-251)."""
    return world_size * int((1 - sa_drop_rate) * (img_tokens // BLOCK))


def gather_tokens(x: torch.Tensor, index: torch.Tensor) -> torch.Tensor:
    """x[:, index] for x [B, N, C] (jenga_hyvideo.py:116 img[:, hilbert_order], :226 inverse;
    also freqs_cos[hilbert_order] with B folded).  index: int64 device tensor."""
    _require_cuda(x, index)
    squeeze = x.dim() == 2
    if squeeze:
        x = x.unsqueeze(0)
    B, N, Cc = x.shape
    if not x.is_contiguous():
        x = x.contiguous()
    if index.dtype != torch.int64 or not index.is_contiguous():
        raise ValueError("index must be a contiguous int64 tensor")
    row_bytes = Cc * x.element_size()
    out = torch.empty((B, index.numel(), Cc), dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.jenga_gather_rows(x.data_ptr(), out.data_ptr(), index.data_ptr(), index.numel(), N,
                                    row_bytes, B, N * row_bytes, index.numel() * row_bytes,
                                    _stream_ptr(x.device)), "gather_rows")
    return out[0] if squeeze else out


def attention_prologue(img_qkv: torch.Tensor, txt_qkv: torch.Tensor | None, heads: int,
                       w_img_q=None, w_img_k=None, w_txt_q=None, w_txt_k=None, eps: float = 1e-6,
                       freqs_cis=None, rope_index: torch.Tensor | None = None, want_pool: bool = True):
    """Fused RMSNorm(q,k) + RoPE(img q,k) + img||txt cat + block pooling.
    img_qkv [B, L, 3*H*D], txt_qkv [B, T, 3*H*D] (the outputs of img_attn_qkv / txt_attn_qkv or
    the split of linear1, models_mul…:200,221,409-417).  Returns q, k, v [B, L+T, H, D] and
    (q_pool, k_pool) [B, H, ceil((L+T)/128), D] or None."""
    _require_cuda(img_qkv)
    B, L, C3 = img_qkv.shape
    D = C3 // (3 * heads)
    if D * 3 * heads != C3:
        raise ValueError("last dim must be 3*heads*head_dim")
    T = 0 if txt_qkv is None else txt_qkv.shape[1]
    S = L + T
    dev, dt = img_qkv.device, img_qkv.dtype
    q = torch.empty((B, S, heads, D), dtype=dt, device=dev)
    k = torch.empty_like(q)
    v = torch.empty_like(q)
    nb = (S + BLOCK - 1) // BLOCK
    qp = torch.empty((B, heads, nb, D), dtype=dt, device=dev) if want_pool else None
    kp = torch.empty_like(qp) if want_pool else None
    a = _lib.JengaHyPrologueArgs()
    a.img_qkv = img_qkv.data_ptr()
    a.txt_qkv = txt_qkv.data_ptr() if txt_qkv is not None else None
    a.dtype = _dtype_code(img_qkv)
    a.batch, a.heads, a.head_dim = B, heads, D
    a.img_tokens, a.txt_tokens = L, T
    if img_qkv.stride(2) != 1 or (txt_qkv is not None and txt_qkv.stride(2) != 1):
        raise ValueError("channel dim must be contiguous")
    a.img_stride_b, a.img_stride_s, a.img_stride_w, a.img_stride_h = img_qkv.stride(0), img_qkv.stride(1), heads * D, D
    if txt_qkv is not None:
        a.txt_stride_b, a.txt_stride_s, a.txt_stride_w, a.txt_stride_h = txt_qkv.stride(0), txt_qkv.stride(1), heads * D, D
    ws = []
    for w in (w_img_q, w_img_k, w_txt_q, w_txt_k):
        ws.append(None if w is None else w.to(device=dev, dtype=dt).contiguous())
    a.w_img_q, a.w_img_k, a.w_txt_q, a.w_txt_k = [None if w is None else w.data_ptr() for w in ws]
    a.eps = eps
    cos = sin = None
    if freqs_cis is not None:
        cos, sin = freqs_cis
        cos = cos.to(device=dev, dtype=torch.float32).contiguous()
        sin = sin.to(device=dev, dtype=torch.float32).contiguous()
        a.rope_cos, a.rope_sin = cos.data_ptr(), sin.data_ptr()
    else:
        a.rope_cos = a.rope_sin = None
    if rope_index is not None:
        # the reference builds hilbert_order from a Python list (CPU int64, sometimes int32): coerce,
        # and make sure every gathered row exists in the tables
        if freqs_cis is None:
            raise ValueError("rope_index given without freqs_cis")
        rope_index = rope_index.to(device=dev, dtype=torch.int64).contiguous()
        if rope_index.numel() < L:
            raise ValueError(f"rope_index has {rope_index.numel()} entries for {L} image tokens")
        if cos.shape[0] < L and rope_index.numel() > 0:
            # table shorter than the token count: indices must stay inside it (one host sync, rare path)
            if int(rope_index[:L].max().item()) >= cos.shape[0] or int(rope_index[:L].min().item()) < 0:
                raise ValueError("rope_index points outside the cos/sin tables")
    elif freqs_cis is not None and cos.shape[0] < L:
        raise ValueError(f"cos/sin tables have {cos.shape[0]} rows for {L} image tokens")
    a.rope_index = rope_index.data_ptr() if rope_index is not None else None
    a.q, a.k, a.v = q.data_ptr(), k.data_ptr(), v.data_ptr()
    a.q_pool = qp.data_ptr() if qp is not None else None
    a.k_pool = kp.data_ptr() if kp is not None else None
    with torch.cuda.device(dev):
        check(lib.jenga_hy_prologue(C.byref(a), _stream_ptr(dev)), "hy_prologue")
    return q, k, v, ((qp, kp) if want_pool else None)


def carved_attention_from_pools(q, k, v, pools, *, top_k: int, text_blocks: int = 2, text_amp: float = 0.0,
                                block_neighbor_list=None, p_remain_rates: float = 0.5,
                                cu_seqlens_q=None, shape_xfuse: bool = False, out: torch.Tensor | None = None,
                                pad_ragged: bool = False):
    """block_sparse_attention (…triton_diffres.py:399) when the prologue already produced the
    pooled block means: select_blocks + one carved-attention launch (2 launches per layer).
    pad_ragged: S need not be a multiple of 128 — the HunyuanVideo-I2V operator
    (hyvideo_i2v/…/attention_block_triton_diffres.py:320-335,385) zero-pads S to nb*128 blocks, the
    dense (text) query blocks attend all nb*128 keys and the output is trimmed to S.  The
    HunyuanVideo operator refuses ragged S (its :216 reshape fails), and so does this function
    without pad_ragged."""
    B, S, H, D = q.shape
    if S % BLOCK and not pad_ragged:
        raise ValueError("hyvideo variant needs S % 128 == 0")
    nb = (S + BLOCK - 1) // BLOCK
    n_img = nb - text_blocks
    qp, kp = pools
    nbr = neighbour_bits(block_neighbor_list, q.device) if block_neighbor_list is not None else None
    # pooled tensors cover all nb blocks; only the first n_img rows / columns are ranked
    bits = select_blocks(qp[:, :, :n_img].contiguous() if qp.shape[2] != n_img else qp, kp, n_img=n_img, nb=nb,
                         top_k=top_k, p_threshold=p_remain_rates, text_blocks=text_blocks, nbr_bits=nbr)
    # sample 0's valid length, cu_seqlens_q[1], limits every sample's rows, as in the operator
    # (attention_block_triton_diffres.py:328-329): exact for --num-videos, whose samples share one prompt
    seq = cu_seqlens_q[1:2].to(device=q.device, dtype=torch.int32) if cu_seqlens_q is not None else None
    if out is None:
        out = torch.empty_like(q)
    elif tuple(out.shape) != (B, S, H, D) or out.dtype != q.dtype or out.stride(3) != 1 or out.stride(2) != D:
        # e.g. the first H*D columns of the single-stream block's concatenation buffer
        raise ValueError("out must be a [B,S,H,D] view with contiguous heads")
    from . import attention as _A
    v8 = _A.quantize_v_fp8(v) if (_A.PV_FP8 and q.dtype == torch.bfloat16) else None   # opt-in FP8 P.V variant
    qk8 = _A.quantize_qk_int8(q, k) if _A.QK_INT8 else None                              # opt-in INT8 Q.K^T variant
    # kv_limit_dense = nb*128: the padded keys are zeros that the dense rows' softmax still counts
    # (== S when S % 128 == 0)
    _launch(q, k, v, bits, n_img, text_blocks, D ** -0.5, text_amp, n_img, S, S, nb * BLOCK, out, seq, q.dtype,
            v_fp8=v8, qk_int8=qk8)
    if shape_xfuse:
        return out
    return out.reshape(B, S, H * D) if out.is_contiguous() else out.flatten(2)
