"""Host-side mirror of the reference's AttenCarve operator for the H100 path.

`block_sparse_attention` keeps the reference signature
(hyvideo/modules/attention_block_triton_diffres.py:399-424, hyvideo_i2v twin :398-423,
wan twin :535-562) and argument meaning; all arithmetic runs in libjenga_b200.so.
torch is used for device memory and the current stream only.
"""
from __future__ import annotations

import ctypes as C
import weakref

import torch

from . import _lib
from ._lib import JengaAttnArgs, JengaError, check, lib

BLOCK = 128


def _stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _dtype_code(t: torch.Tensor) -> int:
    if t.dtype == torch.bfloat16:
        return _lib.JENGA_BF16
    if t.dtype == torch.float16:
        return _lib.JENGA_F16
    raise ValueError(f"unsupported dtype {t.dtype}: the carved attention runs in bf16 or fp16")


def _require_cuda(*ts: torch.Tensor) -> None:
    for t in ts:
        if not t.is_cuda:
            raise JengaError("jenga_b200 has no CPU path: tensors must live on a CUDA device")


def mask_onehot_to_bits(onehot: torch.Tensor) -> torch.Tensor:
    """[..., nq, nb] bool one-hot block mask (the tensor the reference builder returns,
    …triton_diffres.py:252-295) -> [..., nq, ceil(nb/32)] int32 bit rows."""
    _require_cuda(onehot)
    oh = onehot.contiguous()
    if oh.dtype != torch.bool and oh.dtype != torch.uint8:
        raise ValueError("one-hot mask must be bool or uint8")
    nb = oh.shape[-1]
    words = (nb + 31) // 32
    rows = oh.numel() // nb
    bits = torch.empty(*oh.shape[:-1], words, dtype=torch.int32, device=oh.device)
    with torch.cuda.device(oh.device):
        check(lib.jenga_mask_onehot_to_bits(oh.data_ptr(), bits.data_ptr(), rows, nb, words,
                                            _stream_ptr(oh.device)), "mask_onehot_to_bits")
    return bits


def carved_attention_fwd(
    q: torch.Tensor, k: torch.Tensor, v: torch.Tensor,  # [B, S, H, D], D contiguous
    mask_bits: torch.Tensor | None,  # [B, H, nq_sparse, words] int32
    nq_sparse: int, nq_dense: int,
    sm_scale: float, text_amp: float = 0.0, text_block_start: int = 1 << 30,
    kv_limit_sparse: int | None = None, q_limit_sparse: int | None = None,
    kv_limit_dense: int | None = None, out: torch.Tensor | None = None,
    err_flag: torch.Tensor | None = None,
) -> torch.Tensor:
    """One launch of the sm_90a carved-attention kernel (C-ABI jenga_carved_attn_fwd).
    Sparse q-blocks [0, nq_sparse) follow the reference Triton kernel (:38-136); dense
    q-blocks [nq_sparse, nq_sparse+nq_dense) follow its flash_attn_func text rows (:371-380).
    Returns `out` [B, Sq, H, D]."""
    _require_cuda(q, k, v)
    if q.dim() != 4 or k.dim() != 4 or v.dim() != 4:
        raise ValueError("q, k, v must be [B, S, H, D]")
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    if k.shape != (B, Sk, H, D) or v.shape != (B, Sk, H, D):
        raise ValueError("k / v shape mismatch")
    if not (q.dtype == k.dtype == v.dtype):
        raise ValueError("q, k, v must share a dtype")
    for t in (q, k, v):
        if t.stride(3) != 1:
            raise ValueError("head_dim must be contiguous")
    if out is None:
        out = torch.empty((B, Sq, H, D), dtype=q.dtype, device=q.device)
    a = JengaAttnArgs()
    a.q, a.k, a.v, a.out = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr()
    a.dtype = _dtype_code(q)
    a.batch, a.heads, a.head_dim = B, H, D
    a.q_rows, a.kv_rows = Sq, Sk
    a.q_stride_b, a.q_stride_s, a.q_stride_h = q.stride(0), q.stride(1), q.stride(2)
    a.k_stride_b, a.k_stride_s, a.k_stride_h = k.stride(0), k.stride(1), k.stride(2)
    a.v_stride_b, a.v_stride_s, a.v_stride_h = v.stride(0), v.stride(1), v.stride(2)
    a.o_stride_b, a.o_stride_s, a.o_stride_h = out.stride(0), out.stride(1), out.stride(2)
    a.nq_sparse, a.nq_dense = nq_sparse, nq_dense
    if nq_sparse > 0:
        if mask_bits is None:
            raise ValueError("mask_bits required for sparse query blocks")
        _require_cuda(mask_bits)
        if mask_bits.dtype != torch.int32 or not mask_bits.is_contiguous():
            raise ValueError("mask_bits must be contiguous int32")
        if tuple(mask_bits.shape[:3]) != (B, H, nq_sparse):
            raise ValueError(f"mask_bits shape {tuple(mask_bits.shape)} != ({B},{H},{nq_sparse},W)")
        a.mask_bits = mask_bits.data_ptr()
        a.mask_words = mask_bits.shape[3]
    else:
        a.mask_bits, a.mask_words = None, 0
    a.sm_scale, a.text_amp, a.text_block_start = sm_scale, text_amp, min(text_block_start, 1 << 30)
    a.kv_limit_sparse = Sk if kv_limit_sparse is None else kv_limit_sparse
    a.q_limit_sparse = Sq if q_limit_sparse is None else q_limit_sparse
    a.kv_limit_dense = Sk if kv_limit_dense is None else kv_limit_dense
    a.seqlen_dev = None
    a.out_dtype = _lib.JENGA_F32 if out.dtype == torch.float32 else a.dtype
    a.err_flag = err_flag.data_ptr() if err_flag is not None else None
    with torch.cuda.device(q.device):
        check(lib.jenga_carved_attn_fwd(C.byref(a), _stream_ptr(q.device)), "carved_attn_fwd")
    return out


# --------------------------------------------------------------------------------------------
# block pooling + selection (a-8)
# --------------------------------------------------------------------------------------------
def block_pool(x: torch.Tensor, n_blocks: int, cast_out: torch.Tensor | None = None) -> torch.Tensor:
    """Mean over each 128-row block of x [B,S,H,D] -> pooled [B,H,n_blocks,D]
    (ref …triton_diffres.py:216-217).  fp32 input is rounded to bf16 first (wan/…:456-463);
    `cast_out` [B,S,H,D] bf16 then receives the rounded copy."""
    _require_cuda(x)
    B, S, H, D = x.shape
    if x.stride(3) != 1:
        raise ValueError("head_dim must be contiguous")
    in_code = _lib.JENGA_F32 if x.dtype == torch.float32 else _dtype_code(x)
    out_dtype = torch.bfloat16 if x.dtype == torch.float32 else x.dtype
    pooled = torch.empty((B, H, n_blocks, D), dtype=out_dtype, device=x.device)
    if cast_out is not None:
        if cast_out.shape != x.shape or cast_out.dtype != torch.bfloat16 or not cast_out.is_contiguous():
            raise ValueError("cast_out must be a contiguous bf16 tensor shaped like x")
    with torch.cuda.device(x.device):
        check(lib.jenga_block_pool(x.data_ptr(), pooled.data_ptr(),
                                   cast_out.data_ptr() if cast_out is not None else None,
                                   in_code, _dtype_code(pooled), B, H, D, S, x.stride(0), x.stride(1),
                                   x.stride(2), n_blocks, _stream_ptr(x.device)), "block_pool")
    return pooled


def quantize_v_fp8(v: torch.Tensor):
    """Per-head e4m3 quantisation of V [B,S,H,128] for the opt-in FP8 P.V variant (C-ABI
    jenga_quantize_v_fp8).  Returns (v8 uint8 [B,S,H,128] contiguous, amax f32 [B*H])."""
    _require_cuda(v)
    B, S, H, D = v.shape
    if D != 128 or v.stride(3) != 1:
        raise ValueError("v must be [B,S,H,128] with contiguous channels")
    v8 = torch.empty((B, S, H, D), dtype=torch.uint8, device=v.device)
    amax = torch.empty(B * H, dtype=torch.float32, device=v.device)
    with torch.cuda.device(v.device):
        check(lib.jenga_quantize_v_fp8(v.data_ptr(), _dtype_code(v), B, S, H, v.stride(0), v.stride(1), v.stride(2),
                                       v8.data_ptr(), amax.data_ptr(), _stream_ptr(v.device)), "quantize_v_fp8")
    return v8, amax


# Opt-in (never the default): route every operator call of this process through the FP8 P.V variant
# — `jenga_b200.attention.PV_FP8 = True` or JENGA_PV_FP8=1 in the environment.  Lower precision in the
# second product only (tests/test_fp8_gpu.py has its tolerance row); selection and Q.K^T are unchanged.
import os as _os
PV_FP8: bool = _os.environ.get("JENGA_PV_FP8", "0") == "1"

_NBR_CACHE: dict = {}
# tests set this to a list to record every selection result (bit rows, nb) of calls made deep
# inside a block forward; None (the default) costs nothing
MASK_CAPTURE: list | None = None


def neighbour_bits(block_neighbor_list: torch.Tensor, device) -> torch.Tensor:
    """Packs (and caches per tensor/device) the bool adjacency matrix the reference passes as
    `block_neighbor_list` (gilbert.py:597/:679 output) into bit rows on `device`."""
    key = (block_neighbor_list.data_ptr(), tuple(block_neighbor_list.shape),
           block_neighbor_list._version, str(device))
    hit = _NBR_CACHE.get(key)
    # the entry remembers WHICH tensor it was packed from: a freed adjacency whose address is
    # reused by another curve's matrix of the same shape must not hit
    if hit is not None and hit[0]() is block_neighbor_list:
        return hit[1]
    m = block_neighbor_list.to(device=device, dtype=torch.bool)
    bits = mask_onehot_to_bits(m)
    if len(_NBR_CACHE) > 64:
        _NBR_CACHE.clear()
    _NBR_CACHE[key] = (weakref.ref(block_neighbor_list), bits)
    return bits


def select_blocks(q_pool: torch.Tensor, k_pool: torch.Tensor, *, n_img: int, nb: int, top_k: int,
                  p_threshold: float, text_blocks: int, first_frame_blocks: int = 0,
                  nbr_bits: torch.Tensor | None = None, return_counts: bool = False,
                  use_workspace: bool = True):
    """Pooled scores -> per-(head, query block) bit rows of attended key blocks
    (ref …triton_diffres.py:227-293; wan first-frame rule :400-406)."""
    _require_cuda(q_pool, k_pool)
    B, H, nq, D = q_pool.shape
    if not q_pool.is_contiguous() or not k_pool.is_contiguous():
        raise ValueError("pooled tensors must be contiguous")
    words = (nb + 31) // 32
    bits = torch.empty((B, H, nq, words), dtype=torch.int32, device=q_pool.device)
    counts = torch.empty((B, H, nq), dtype=torch.int32, device=q_pool.device) if return_counts else None
    a = _lib.JengaSelectArgs()
    a.q_pool, a.k_pool, a.dtype = q_pool.data_ptr(), k_pool.data_ptr(), _dtype_code(q_pool)
    a.batch_heads, a.head_dim, a.nq = B * H, D, nq
    a.nk_pool, a.n_img, a.nb, a.mask_words = k_pool.shape[2], n_img, nb, words
    a.top_k, a.p_threshold = int(top_k), float(p_threshold)
    a.text_blocks, a.first_frame_blocks = int(text_blocks), int(first_frame_blocks)
    if nbr_bits is not None:
        a.nbr_bits, a.nbr_rows, a.nbr_words = nbr_bits.data_ptr(), nbr_bits.shape[0], nbr_bits.shape[1]
    else:
        a.nbr_bits, a.nbr_rows, a.nbr_words = None, 0, 0
    a.out_bits = bits.data_ptr()
    a.out_counts = counts.data_ptr() if counts is not None else None
    ws = None
    if use_workspace and n_img <= 1024:
        nbytes = lib.jenga_select_blocks_workspace_bytes(B * H, nq, n_img)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=q_pool.device)
        a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
    else:
        a.workspace, a.workspace_bytes = None, 0
    with torch.cuda.device(q_pool.device):
        check(lib.jenga_select_blocks(C.byref(a), _stream_ptr(q_pool.device)), "select_blocks")
    if MASK_CAPTURE is not None:
        MASK_CAPTURE.append((bits, nb))
    return (bits, counts) if return_counts else bits


def bits_to_onehot(bits: torch.Tensor, nb: int) -> torch.Tensor:
    """Test/debug helper: expands packed bit rows back to the reference's bool one-hot."""
    shifts = torch.arange(32, device=bits.device, dtype=torch.int32)
    oh = ((bits.unsqueeze(-1) >> shifts) & 1).bool().flatten(-2)
    return oh[..., :nb]


# --------------------------------------------------------------------------------------------
# the operator (a-11)
# --------------------------------------------------------------------------------------------
_VARIANT_DEFAULTS = {
    # variant: (text_blocks, p_remain_rates)   ref: hyvideo/…:399-424, hyvideo_i2v/…:398-423, wan/…:535-562
    "hyvideo": (2, 0.5),
    "hyvideo_i2v": (4, 0.5),
    "wan": (0, 0.9),
}


def block_sparse_attention_variant(
    variant: str, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, top_k: int,
    block_size_M: int = 128, block_size_N: int = 128, cu_seqlens_q=None, cu_seqlens_kv=None,
    max_seqlen_q=None, max_seqlen_kv=None, text_blocks=None, text_amp: float = 0.0,
    block_neighbor_list=None, shape_xfuse: bool = False, p_remain_rates=None,
    first_frame_blocks: int = 0, return_mask_bits: bool = False, out: torch.Tensor | None = None,
    sp_out: dict | None = None, pv_fp8: bool = False,
):
    """AttenCarve operator, [B,S,H,D] in -> [B,S,H*D] (or [B,S,H,D] when shape_xfuse).
    Same arguments, defaults and quirks as the reference function of the same name; see the
    variant table above for the file each one mirrors.  Three launches on the current stream
    (2x block_pool, select_blocks) + one carved-attention launch; no host synchronisation."""
    if variant not in _VARIANT_DEFAULTS:
        raise ValueError(f"unknown variant {variant!r}")
    d_text, d_p = _VARIANT_DEFAULTS[variant]
    text_blocks = d_text if text_blocks is None else int(text_blocks)
    p_remain_rates = d_p if p_remain_rates is None else float(p_remain_rates)
    if block_size_M != BLOCK or block_size_N != BLOCK:
        raise ValueError("only 128x128 blocks are built (the only size the reference launches)")
    _require_cuda(query, key, value)
    B, S, H, D = query.shape
    assert D in (16, 32, 64, 128), "ref :155 — head_dim must be one of {16,32,64,128}"
    out_dtype = query.dtype
    use_cu = variant != "wan" and cu_seqlens_q is not None and cu_seqlens_kv is not None
    seqlen_dev = None
    if use_cu:
        # ref :328-329 — only element [1] is read, on the device
        seqlen_dev = cu_seqlens_q[1:2].to(device=query.device, dtype=torch.int32)
    if variant == "hyvideo" and S % BLOCK != 0:
        # ref :216 reshape fails on ragged S (the padded copies of :331-335 are never used)
        raise ValueError(f"hyvideo variant needs S % 128 == 0, got {S}")
    nb = (S + BLOCK - 1) // BLOCK
    normal_blocks = nb - text_blocks
    if normal_blocks < 0:
        raise ValueError("more text blocks than blocks")
    # ---- dtype handling: wan casts everything to bf16 first (:456-463)
    q, k, v = query, key, value
    q_pool = k_pool = None
    if variant == "wan":
        def to_bf16_with_pool(x, want_pool, n_pool):
            if x.dtype == torch.bfloat16:
                return x, (block_pool(x, n_pool) if want_pool and n_pool > 0 else None)
            # the cast must cover EVERY row (wan/…:456-463 casts the whole padded tensor), so the
            # kernel runs over all nb blocks; only the first n_pool pooled rows are ranked
            xf = x if x.dtype == torch.float32 else x.float()
            xc = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
            pooled = block_pool(xf, nb, cast_out=xc)
            if not (want_pool and n_pool > 0):
                return xc, None
            return xc, (pooled if n_pool == nb else pooled[:, :, :n_pool].contiguous())
        q, q_pool = to_bf16_with_pool(q, True, normal_blocks)
        k, k_pool = to_bf16_with_pool(k, True, normal_blocks)
        v, _ = to_bf16_with_pool(v, False, 0) if v.dtype != torch.bfloat16 else (v, None)
    elif not (q.dtype == k.dtype == v.dtype):
        raise ValueError("q, k, v must share a dtype")
    mask_bits = None
    if normal_blocks > 0:
        if q_pool is None:
            q_pool = block_pool(q, normal_blocks)
        if k_pool is None:
            k_pool = block_pool(k, normal_blocks)
        nbr = neighbour_bits(block_neighbor_list, q.device) if block_neighbor_list is not None else None
        mask_bits = select_blocks(q_pool, k_pool, n_img=normal_blocks, nb=nb, top_k=top_k,
                                  p_threshold=p_remain_rates, text_blocks=text_blocks,
                                  first_frame_blocks=first_frame_blocks if variant == "wan" else 0,
                                  nbr_bits=nbr)
    want_dtype = out_dtype if variant == "wan" else q.dtype
    if sp_out is not None:
        # fused Ulysses epilogue: rows are stored into the owners' peer-mapped buffers
        _launch(q, k, v, mask_bits, normal_blocks, text_blocks, D ** -0.5, text_amp, normal_blocks,
                S, S, nb * BLOCK, None, seqlen_dev, q.dtype, sp_out=sp_out)
        return mask_bits if return_mask_bits else None
    if out is None:
        out = torch.empty((B, S, H, D), dtype=want_dtype, device=q.device)
    elif out.shape != (B, S, H, D) or out.dtype != want_dtype or out.stride(3) != 1:
        raise ValueError("out must be [B,S,H,D] in the result dtype with contiguous head_dim")
    a_out_dtype = out.dtype
    limit = S  # no cu_seqlens: seqlens = [context_size] (:336 / wan :452)
    # pv_fp8 (opt-in, SURVEY §8 f-3): V is quantised per head to e4m3 and P.V runs on the FP8 tensor
    # path; NOT the reference's arithmetic — its own tolerance row, never enabled implicitly
    v8 = quantize_v_fp8(v) if (pv_fp8 or PV_FP8) and sp_out is None and q.dtype == torch.bfloat16 else None
    o = _launch(q, k, v, mask_bits, normal_blocks, text_blocks, D ** -0.5, text_amp, normal_blocks,
                limit, limit, nb * BLOCK, out, seqlen_dev, a_out_dtype, v_fp8=v8)
    if not shape_xfuse:
        o = o.reshape(B, S, H * D)
    return (o, mask_bits) if return_mask_bits else o


def _launch(q, k, v, mask_bits, nq_sparse, nq_dense, sm_scale, text_amp, text_block_start,
            kv_limit_sparse, q_limit_sparse, kv_limit_dense, out, seqlen_dev, out_dtype, sp_out=None, lse_out=None,
            v_fp8=None):
    B, Sq, H, D = q.shape
    a = JengaAttnArgs()
    a.q, a.k, a.v = q.data_ptr(), k.data_ptr(), v.data_ptr()
    a.out = out.data_ptr() if out is not None else None
    a.dtype = _dtype_code(q)
    a.out_dtype = _lib.JENGA_F32 if out_dtype == torch.float32 else a.dtype
    a.batch, a.heads, a.head_dim = B, H, D
    a.q_rows, a.kv_rows = Sq, k.shape[1]
    a.q_stride_b, a.q_stride_s, a.q_stride_h = q.stride(0), q.stride(1), q.stride(2)
    a.k_stride_b, a.k_stride_s, a.k_stride_h = k.stride(0), k.stride(1), k.stride(2)
    a.v_stride_b, a.v_stride_s, a.v_stride_h = v.stride(0), v.stride(1), v.stride(2)
    if out is not None:
        a.o_stride_b, a.o_stride_s, a.o_stride_h = out.stride(0), out.stride(1), out.stride(2)
    if sp_out is not None:
        a.sp_world, a.sp_rank = sp_out["world"], sp_out["rank"]
        a.sp_heads_total, a.sp_rows = sp_out["heads_total"], sp_out["rows"]
        a.out_peers_host = C.addressof(sp_out["peers"])
        if "head_base" in sp_out:
            a.sp_head_base, a.sp_head_base_valid = int(sp_out["head_base"]), 1
    a.lse_out = lse_out.data_ptr() if lse_out is not None else None
    if v_fp8 is not None:
        a.v_fp8, a.v_fp8_amax = v_fp8[0].data_ptr(), v_fp8[1].data_ptr()
    a.nq_sparse, a.nq_dense = nq_sparse, nq_dense
    a.mask_bits = mask_bits.data_ptr() if mask_bits is not None else None
    a.mask_words = mask_bits.shape[-1] if mask_bits is not None else 0
    a.sm_scale, a.text_amp, a.text_block_start = sm_scale, float(text_amp), text_block_start
    a.kv_limit_sparse, a.q_limit_sparse, a.kv_limit_dense = kv_limit_sparse, q_limit_sparse, kv_limit_dense
    a.seqlen_dev = seqlen_dev.data_ptr() if seqlen_dev is not None else None
    a.err_flag = None
    with torch.cuda.device(q.device):
        check(lib.jenga_carved_attn_fwd(C.byref(a), _stream_ptr(q.device)), "carved_attn_fwd")
    return out


def block_sparse_attention(query, key, value, top_k, block_size_M=128, block_size_N=128,
                           cu_seqlens_q=None, cu_seqlens_kv=None, max_seqlen_q=None,
                           max_seqlen_kv=None, text_blocks=2, text_amp=0.0,
                           block_neighbor_list=None, shape_xfuse=False, p_remain_rates=0.5):
    """Drop-in for hyvideo/modules/attention_block_triton_diffres.py:399 block_sparse_attention."""
    return block_sparse_attention_variant(
        "hyvideo", query, key, value, top_k, block_size_M, block_size_N, cu_seqlens_q,
        cu_seqlens_kv, max_seqlen_q, max_seqlen_kv, text_blocks, text_amp, block_neighbor_list,
        shape_xfuse, p_remain_rates)
