"""Wan2.1-side glue of the hot path (wan/modules/model_mul.py:134-180 WanSelfAttention.forward,
:183-205 WanT2VCrossAttention.forward, :223-249 WanI2VCrossAttention.forward): fused WanRMSNorm + RoPE
prologue, the block-count rules, the operator call, the dense text cross-attention and the I2V
image + text cross-attention."""
from __future__ import annotations

import ctypes as C
import math

import torch

from . import _lib
from ._lib import check, lib
from .attention import BLOCK, _launch, _require_cuda, _stream_ptr, block_sparse_attention_variant


def rope_freqs(head_dim: int = 128, max_len: int = 1024, theta: float = 10000.0) -> torch.Tensor:
    """The complex128 table WanModel builds (model_mul.py:502-507 with rope_params :29-37)."""
    def params(dim):
        f = torch.outer(torch.arange(max_len), 1.0 / torch.pow(theta, torch.arange(0, dim, 2).to(torch.float64).div(dim)))
        return torch.polar(torch.ones_like(f), f)
    d = head_dim
    return torch.cat([params(d - 4 * (d // 6)), params(2 * (d // 6)), params(2 * (d // 6))], dim=1)


def block_counts(seq_len: int, sa_drop_rate: float, per_block_tokens: int = 128):
    """model_mul.py:161-164: (selected_top_k, first_frame_blocks)."""
    num_blocks = math.ceil(seq_len / per_block_tokens)
    return math.ceil(int(num_blocks * (1 - sa_drop_rate))), math.ceil(num_blocks // 21)


_FREQ_CACHE: dict = {}


def _device_freqs(freqs: torch.Tensor, dev) -> torch.Tensor:
    """The complex128 table as doubles [rows, 64, 2] on `dev`.  WanModel keeps `self.freqs` on the CPU
    (model_mul.py:502-507) and the reference moves it every forward; here the device copy is made once
    per table (keyed by the tensor object, dropped with it)."""
    import weakref
    key = (id(freqs), str(dev))
    hit = _FREQ_CACHE.get(key)
    if hit is not None and hit[0]() is freqs and hit[2] == freqs._version:
        return hit[1]
    fr = torch.view_as_real(freqs.to(torch.complex128)).to(dev).contiguous()
    _FREQ_CACHE[key] = (weakref.ref(freqs, lambda _r, k=key: _FREQ_CACHE.pop(k, None)), fr, freqs._version)
    return fr


def norm_rope(x: torch.Tensor, weight: torch.Tensor | None, heads: int, grid_size, freqs: torch.Tensor | None,
              freq_remap: torch.Tensor | None = None, eps: float = 1e-6) -> torch.Tensor:
    """rope_apply(norm(x).view(b, s, n, d), grid_sizes, freqs, freq_remap) as the carved
    attention consumes it: [B, L, H, 128] bf16.  x: [B, L, H*128] bf16 or fp32.
    freqs=None: the norm alone, `bf16(norm(x))` with no rotation (grid_size and freq_remap unused)."""
    _require_cuda(x)
    B, L, Cc = x.shape
    if Cc != heads * 128 or x.stride(2) != 1:
        raise ValueError("x must be [B, L, heads*128] with contiguous channels")
    dev = x.device
    out = torch.empty((B, L, heads, 128), dtype=torch.bfloat16, device=dev)
    a = _lib.JengaWanPrologueArgs()
    a.x = x.data_ptr()
    code = {torch.bfloat16: _lib.JENGA_BF16, torch.float32: _lib.JENGA_F32}
    if x.dtype not in code:
        raise ValueError("x must be bf16 or fp32")
    a.x_dtype = code[x.dtype]
    if weight is not None:
        weight = weight.to(dev).contiguous()
        if weight.dtype not in code:
            raise ValueError("weight must be bf16 or fp32")
        a.w, a.w_dtype = weight.data_ptr(), code[weight.dtype]
    else:
        a.w, a.w_dtype = None, _lib.JENGA_F32
    a.batch, a.heads, a.head_dim, a.tokens = B, heads, 128, L
    a.stride_b, a.stride_s, a.eps = x.stride(0), x.stride(1), eps
    if freqs is None:
        a.freqs, a.freq_rows = None, 0
        a.grid_f = a.grid_h = a.grid_w = 0
        freq_remap = None
    else:
        fr = _device_freqs(freqs, dev)
        a.freqs, a.freq_rows = fr.data_ptr(), fr.shape[0]
        a.grid_f, a.grid_h, a.grid_w = (int(v) for v in grid_size)
    if freq_remap is not None:
        freq_remap = freq_remap.to(device=dev, dtype=torch.int64).contiguous()
        a.freq_remap = freq_remap.data_ptr()
    else:
        a.freq_remap = None
    a.out = out.data_ptr()
    with torch.cuda.device(dev):
        check(lib.jenga_wan_prologue(C.byref(a), _stream_ptr(dev)), "wan_prologue")
    return out


def self_attention(q_lin, k_lin, v, norm_q_w, norm_k_w, heads, grid_size, freqs, sa_drop_rate, *,
                   p_remain_rates=0.8, freq_remap=None, block_neighbor_list=None, eps=1e-6):
    """WanSelfAttention.forward's attention part for sa_drop_rate > 0.25 (model_mul.py:160-176):
    q_lin/k_lin [B, L, C] are self.q(x)/self.k(x), v is self.v(x).view(b, s, n, d)."""
    q = norm_rope(q_lin, norm_q_w, heads, grid_size, freqs, freq_remap, eps)
    k = norm_rope(k_lin, norm_k_w, heads, grid_size, freqs, freq_remap, eps)
    top_k, ff = block_counts(q.shape[1], sa_drop_rate)
    return block_sparse_attention_variant("wan", q, k, v, top_k, text_blocks=0,
                                          block_neighbor_list=block_neighbor_list,
                                          p_remain_rates=p_remain_rates, first_frame_blocks=ff,
                                          shape_xfuse=True)


def cross_attention(q_lin, k_lin, v, norm_q_w, norm_k_w, heads, eps=1e-6):
    """WanT2VCrossAttention.forward's attention part (model_mul.py:195-200) with every context row valid
    (context_lens=None): q_lin [B, L, C] = self.q(x), k_lin [B, Lc, C] = self.k(context),
    v [B, Lc, H, 128] = self.v(context) bf16, sample b attending its own Lc context rows.
    Returns [B, L, H, 128] bf16.

    q and k go through the norm-only prologue, `bf16(bf16(norm(x)) * w)` — what flash_attention's
    half() makes of norm_q(self.q(x)) (wan/modules/attention.py:59-83) — and the dense class of the
    attention kernel runs over all Lc keys with softmax_scale D^-1/2.  flash_attention returns the
    result as fp32 (`x.type(out_dtype)`, :130), which self.o casts straight back to bf16 under
    autocast: the bf16 result here is what self.o sees.  No segment table, no host sync."""
    q = norm_rope(q_lin, norm_q_w, heads, None, None, eps=eps)
    k = norm_rope(k_lin, norm_k_w, heads, None, None, eps=eps)
    if k.shape[0] != q.shape[0]:
        raise ValueError("q_lin and k_lin must hold one batch")
    if v.dtype != torch.bfloat16 or v.shape != k.shape or v.stride(3) != 1:
        raise ValueError("v must be bf16 [B, Lc, heads, 128] with contiguous channels")
    _, L, _, D = q.shape
    Lc = k.shape[1]
    out = torch.empty_like(q)
    _launch(q, k, v, None, 0, (L + BLOCK - 1) // BLOCK, D ** -0.5, 0.0, 1 << 30, Lc, L, Lc, out, None, torch.bfloat16)
    return out


def i2v_cross_attn(q, k_img, v_img, k_txt, v_txt, sm_scale=None, out=None):
    """One launch of jenga_wan_i2v_cross_attn: out = bf16(f32(A_img) + f32(A_txt)), each A the bf16 result
    of a dense softmax(q k^T sm_scale) v over its own keys.  All [B, S, H, 128] bf16 with contiguous
    channels; sm_scale defaults to 128^-1/2.  Returns `out` (allocated like q when None)."""
    _require_cuda(q, k_img, v_img, k_txt, v_txt)
    ts = (q, k_img, v_img, k_txt, v_txt) + (() if out is None else (out,))
    if any(t.dim() != 4 or t.dtype != torch.bfloat16 or t.stride(3) != 1 for t in ts):
        raise ValueError("q, k_img, v_img, k_txt, v_txt and out must be bf16 [B, S, H, 128] with contiguous channels")
    B, L, H, D = q.shape
    if (k_img.shape != v_img.shape or k_txt.shape != v_txt.shape or k_img.shape[::2] != (B, H)
            or k_txt.shape[::2] != (B, H) or k_img.shape[3] != D or k_txt.shape[3] != D):
        raise ValueError("k_img / v_img and k_txt / v_txt must be [B, S, H, D] with q's B, H and D")
    if out is None:
        out = torch.empty_like(q)
    elif out.shape != q.shape:
        raise ValueError("out must have q's shape")
    a = _lib.JengaWanCrossArgs()
    a.q, a.k_img, a.v_img, a.k_txt, a.v_txt, a.out = (t.data_ptr() for t in (q, k_img, v_img, k_txt, v_txt, out))
    a.dtype, a.batch, a.heads, a.head_dim = _lib.JENGA_BF16, B, H, D
    a.q_rows, a.img_rows, a.txt_rows = L, k_img.shape[1], k_txt.shape[1]
    for name, t in (("q", q), ("ki", k_img), ("vi", v_img), ("kt", k_txt), ("vt", v_txt), ("o", out)):
        setattr(a, f"{name}_stride_b", t.stride(0))
        setattr(a, f"{name}_stride_s", t.stride(1))
        setattr(a, f"{name}_stride_h", t.stride(2))
    a.sm_scale = D ** -0.5 if sm_scale is None else float(sm_scale)
    a.err_flag = None
    with torch.cuda.device(q.device):
        check(lib.jenga_wan_i2v_cross_attn(C.byref(a), _stream_ptr(q.device)), "wan_i2v_cross_attn")
    return out


def i2v_cross_attention(q_lin, k_lin, v, kimg_lin, vimg, wq, wk, wk_img, heads, eps=1e-6):
    """WanI2VCrossAttention.forward's attention part (model_mul.py:230-247) with every context row valid:
    q_lin [B, L, C] = self.q(x); k_lin [B, Lt, C] = self.k(context[:, 257:]) and v [B, Lt, H, 128] =
    self.v(…) bf16; kimg_lin [B, Li, C] = self.k_img(context[:, :257]) and vimg [B, Li, H, 128] =
    self.v_img(…) bf16; sample b attends its own context rows.  Returns [B, L, H, 128] bf16: what self.o
    receives.

    q, k and k_img go through the norm-only prologue, as in cross_attention; one launch then computes
    both attentions and their sum, `x + img_x` in fp32 (:247) of the two fp32-typed flash_attention
    results, rounded to bf16 as self.o's autocast cast does."""
    q = norm_rope(q_lin, wq, heads, None, None, eps=eps)
    k = norm_rope(k_lin, wk, heads, None, None, eps=eps)
    ki = norm_rope(kimg_lin, wk_img, heads, None, None, eps=eps)
    if v.dtype != torch.bfloat16 or v.shape != k.shape or vimg.dtype != torch.bfloat16 or vimg.shape != ki.shape:
        raise ValueError("v / vimg must be bf16 [B, Lt / Li, heads, 128] like the projected keys")
    return i2v_cross_attn(q, ki, vimg, k, v)
