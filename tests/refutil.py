"""Shared helpers of the reference-backed GPU parity tests (and bench.py's gpu_reference leg).

fp64 ground truth of the operator's MATH (no intermediate rounding) on a sample of query blocks,
error statistics relative to it, and the call sequence of the unmodified reference operator
(oracle/ref_loader.py).  Test infrastructure only.
"""
from __future__ import annotations

import math

import torch

BLOCK = 128
LN2 = math.log(2.0)


def pad_rows(x: torch.Tensor, rows: int) -> torch.Tensor:
    """[1,S,H,D] -> [1,rows,H,D] zero padded (what the I2V / Wan variants do, wan/…:448-451)."""
    if x.shape[1] == rows:
        return x
    return torch.nn.functional.pad(x, [0, 0, 0, 0, 0, rows - x.shape[1]])


@torch.no_grad()
def fp64_truth(q, k, v, onehot, qblocks, *, n_img_blocks, seqlen, text_amp=0.0, sm_scale=None,
               text_block_start=None, kv_limit=None, q_limit=None, kv_limit_dense=None, return_lse=False):
    """Exact softmax attention in fp64 for the query blocks `qblocks` of every batch and head.

    q: [B,Sq,H,D], k,v: [B,Sk,H,D] tensors on one device (any float dtype; values are taken as
    they are; Sq and Sk are independent, keys past Sk are zeros),
    onehot: [B,H,n_img_blocks,nb] bool — the block mask of the image rows, nb*128 >= Sk.
    Image rows (block < n_img_blocks): keys = mask-selected blocks, key columns >= kv_limit
    (default seqlen) hidden, key blocks >= text_block_start (default n_img_blocks) biased by
    text_amp in log2 units (…triton_diffres.py:96-118); when q_limit is given, rows >= q_limit
    are zeros (:59-61, :136).  Text rows: dense over ALL nb*128 keys incl. padding, no bias
    (:371-380), or over the keys below kv_limit_dense when it is given.
    Returns {qb: [H,128,D] float64} for B == 1 and {qb: [B,H,128,D]} otherwise; with
    return_lse=True also {qb: [H,128] or [B,H,128]}, the natural-log logsumexp of s * sm_scale of
    the text rows (flash_attn's softmax_lse)."""
    B, Sq, H, D = q.shape
    nb = onehot.shape[-1]
    Sp = nb * BLOCK
    sm_scale = D ** -0.5 if sm_scale is None else sm_scale
    kv_limit = seqlen if kv_limit is None else kv_limit
    text_block_start = n_img_blocks if text_block_start is None else text_block_start
    Sqp = (max(qblocks) + 1) * BLOCK
    kd = pad_rows(k, Sp).transpose(1, 2).double()                # [B,H,Sp,D]
    vd = pad_rows(v, Sp).transpose(1, 2).double()
    qd = pad_rows(q[:, :Sqp], Sqp).transpose(1, 2)
    cols = torch.arange(Sp, device=q.device)
    rows = torch.arange(BLOCK, device=q.device)
    out, lse = {}, {}
    for qb in qblocks:
        Q = qd[:, :, qb * BLOCK:(qb + 1) * BLOCK].double()      # [B,H,128,D]
        s = torch.matmul(Q, kd.transpose(-1, -2)) * sm_scale     # [B,H,128,Sp]
        if qb < n_img_blocks:
            live = onehot[:, :, qb].repeat_interleave(BLOCK, dim=-1)             # [B,H,Sp]
            if text_amp != 0.0:
                s[..., text_block_start * BLOCK:] += text_amp * LN2
            dead = (~live)[:, :, None, :] | (cols >= kv_limit)
            s = s.masked_fill(dead, float("-inf"))
        elif kv_limit_dense is not None:
            s = s.masked_fill(cols >= kv_limit_dense, float("-inf"))
        p = torch.softmax(s, dim=-1)
        o = torch.matmul(p, vd)
        if qb < n_img_blocks and q_limit is not None:
            o[:, :, qb * BLOCK + rows >= q_limit] = 0.0
        if return_lse and qb >= n_img_blocks:
            lse[qb] = torch.logsumexp(s, dim=-1)[0] if B == 1 else torch.logsumexp(s, dim=-1)
        out[qb] = o[0] if B == 1 else o
        del s, p
    return (out, lse) if return_lse else out


def error_stats(got, truth: dict, *, seqlen_rows=None):
    """got: [B,S,H*D] or [B,S,H,D]; truth from fp64_truth.  Returns (max|e|/rms, mean|e|/rms, rms)
    over the sampled blocks (rows >= seqlen_rows of a block are skipped: both implementations
    leave them zero / undefined)."""
    any_t = next(iter(truth.values()))
    H, D = any_t.shape[-3], any_t.shape[-1]
    g = got.reshape(got.shape[0], got.shape[1], H, D)
    num_max, num_sum, cnt, sq = 0.0, 0.0, 0, 0.0
    for qb, t in truth.items():
        r0 = qb * BLOCK
        r1 = min(r0 + BLOCK, g.shape[1])
        if seqlen_rows is not None:
            r1 = min(r1, seqlen_rows)
        if r1 <= r0:
            continue
        x = g[:, r0:r1].transpose(1, 2).double()
        if t.dim() == 3:
            x = x[0]
        tt = t[..., : r1 - r0, :]
        e = (x - tt).abs()
        num_max = max(num_max, e.max().item())
        num_sum += e.sum().item()
        cnt += e.numel()
        sq += tt.pow(2).sum().item()
    rms = math.sqrt(sq / max(cnt, 1)) + 1e-30
    return num_max / rms, num_sum / max(cnt, 1) / rms, rms


def pair_stats(a, b):
    """max|a-b|/rms(b), mean|a-b|/rms(b) over two same-shaped tensors."""
    a, b = a.double(), b.double()
    rms = b.pow(2).mean().sqrt().item() + 1e-30
    d = (a - b).abs()
    return d.max().item() / rms, d.mean().item() / rms


def reference_call(op, variant, q, k, v, *, top_k, cu, text_blocks, text_amp, nbr, p_remain,
                   first_frame=0, shape_xfuse=False):
    """The unmodified reference operator under the pipelines' autocast
    (pipeline_hunyuan_video_prores.py:663-665, jenga_wan.py:135)."""
    kw = dict(cu_seqlens_q=cu, cu_seqlens_kv=cu, text_blocks=text_blocks, text_amp=text_amp,
              block_neighbor_list=nbr, shape_xfuse=shape_xfuse, p_remain_rates=p_remain)
    if variant == "wan":
        kw["first_frame_blocks"] = first_frame
    with torch.autocast("cuda", dtype=torch.bfloat16):
        return op.block_sparse_attention(q, k, v, top_k, **kw)


def reference_mask(op, variant, q, k, *, top_k, text_blocks, nbr, p_remain, first_frame=0):
    """The reference builder's one-hot mask for the same inputs, called the way
    block_sparse_attention_combined calls it (…triton_diffres.py:345-356, wan :476-487)."""
    B, S, H, D = q.shape
    nb = (S + BLOCK - 1) // BLOCK
    qh = pad_rows(q, nb * BLOCK).transpose(1, 2)
    kh = pad_rows(k, nb * BLOCK).transpose(1, 2)
    if variant == "wan":
        qh, kh = qh.to(torch.bfloat16), kh.to(torch.bfloat16)
    n_img = nb - text_blocks
    kw = dict(text_start_block=n_img, num_blocks=nb, prob_threshold=p_remain, text_blocks=text_blocks,
              block_neighbor_list=nbr)
    if variant == "wan":
        kw["first_frame_blocks"] = first_frame
    with torch.autocast("cuda", dtype=torch.bfloat16):
        return op._build_block_index_with_importance_optimized(qh[:, :, :n_img * BLOCK], kh, top_k, BLOCK, BLOCK, **kw)


def mask_agreement(got: torch.Tensor, ref: torch.Tensor, n_img: int):
    """(fraction of identical rows, mean Jaccard, fraction of equal counts, text columns exact)."""
    same_rows = (got == ref).all(-1).float().mean().item()
    inter = (got & ref).sum(-1).float()
    union = (got | ref).sum(-1).float().clamp_min(1)
    jac = (inter / union).mean().item()
    counts = (got.sum(-1) == ref.sum(-1)).float().mean().item()
    text_ok = bool((got[..., n_img:] == ref[..., n_img:]).all().item())
    return same_rows, jac, counts, text_ok
