"""Restatements of the carved-attention kernel (jenga_b200/csrc/carved_attn.cu over the consumer loop of
carved_attn_common.cuh) that the full-size tests check every row against.  Plain torch; every helper
runs on whichever device its tensors live on.

Two legs:

- flat_case / flat_expected: inputs whose output is known exactly.  Q = 0 makes every score 0 in
  every class (sparse Q~ = round16(0 * qk_scale) = 0, dense raw S = 0, INT8 codes 0), so every key
  of a live tile gets p = 1, and a text key (block >= text_block_start) p = 2^a for an integer
  text_amp a.  V holds integers in [-8, 8], so the kernel's partial sums are exact as long as they
  fit in fp32's 24-bit significand (`flat_exact_bits` certifies that), and its output is
  round16(fp32(num) * fp32(1 / l)) with num and l formed exactly here.
- fp64_rows / elem_bound: realistic inputs against fp64, with a per-element bound derived from the
  kernel's rounding points.

The dense launches outside the carved path (the FlashAttention shims, the Wan T2V cross-attention and
the two-segment Wan I2V kernel, jenga_b200/csrc/wan_cross_attn.cu) reuse both legs: dense_expected
and segments_expected state a dense-only launch and a varlen call, i2v_expected / i2v_bound the I2V
sum, and fp8_case / fp8_expected the FP8 P.V epilogue on V values whose e4m3 codes are exact.
"""
from __future__ import annotations

import math
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from select_ref import MMA_REL  # noqa: E402

BLOCK = 128
D = 128
LOG2E_LITERAL = 1.44269504          # the launcher's constant (carved_attn.cu: qk_scale)
FLAT_AMPS = (0, 3, -2, 9)           # 9 > 8 fires the lazy rescale at the first text tile
V_MAX = 8


def qk_scale32(sm_scale: float) -> float:
    """The kernel's qk_scale: fp32(sm_scale * 1.44269504), formed in double on the host."""
    return float(torch.tensor(sm_scale * LOG2E_LITERAL, dtype=torch.float32))


def f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


def unpack(bits: torch.Tensor, nb: int) -> torch.Tensor:
    """[..., words] int32 -> [..., nb] bool; bits past nb are dropped, as the kernel drops them."""
    sh = torch.arange(32, device=bits.device, dtype=torch.int32)
    return ((bits.unsqueeze(-1) >> sh) & 1).bool().flatten(-2)[..., :nb]


# ------------------------------------------------------------------------------------------------
# Leg A: exact by construction
# ------------------------------------------------------------------------------------------------
def flat_case(B: int, S: int, H: int, *, seed: int, device, dtype=torch.bfloat16):
    """q = 0, k ~ N(0, 1), v integers in [-V_MAX, V_MAX] drawn per (b, s, h, d); [B, S, H, D]."""
    g = torch.Generator(device=device).manual_seed(seed)
    q = torch.zeros(B, S, H, D, dtype=dtype, device=device)
    k = torch.randn(B, S, H, D, generator=g, device=device).to(dtype)
    v = torch.randint(-V_MAX, V_MAX + 1, (B, S, H, D), generator=g, device=device).to(dtype)
    return q, k, v


def flat_num_l(v: torch.Tensor, live: torch.Tensor | None, *, nq_sparse: int, nq_dense: int, text_amp: int = 0,
               text_block_start: int = 1 << 30, kv_limit_sparse: int | None = None, kv_limit_dense: int | None = None):
    """(num [B, H, nq, D], l [B, H, nq], n_tiles [B, H, nq]) in fp64 for every query block of a flat case;
    every row of a block has the same value.  live: [B, H, nq_sparse, nb] bool (bits past nb already
    dropped).  A key counts when its block is live and its column is below the class's key limit;
    keys past v's rows (the zero-filled padding of the last block) count with v = 0."""
    B, S, H, _ = v.shape
    nb = (S + BLOCK - 1) // BLOCK
    Sp = nb * BLOCK
    vd = torch.zeros(B, Sp, H, D, dtype=torch.float64, device=v.device)
    vd[:, :S] = v.double()
    cols = torch.arange(Sp, device=v.device)

    def block_sums(limit):
        keep = (cols < limit).double()
        vs = (vd * keep[None, :, None, None]).view(B, nb, BLOCK, H, D).sum(2)      # [B, nb, H, D]
        cnt = keep.view(nb, BLOCK).sum(1)                                         # [nb]
        return vs.permute(0, 2, 1, 3), cnt                                        # [B, H, nb, D]

    nums, ls, tiles = [], [], []
    if nq_dense:
        vs, cnt = block_sums(Sp if kv_limit_dense is None else kv_limit_dense)
        n = vs.sum(2, keepdim=True).expand(B, H, nq_dense, D)
        nums.append(n)
        ls.append(cnt.sum().expand(B, H, nq_dense))
        tiles.append(torch.full((B, H, nq_dense), nb, device=v.device))
    if nq_sparse:
        vs, cnt = block_sums(S if kv_limit_sparse is None else kv_limit_sparse)
        w = torch.ones(nb, dtype=torch.float64, device=v.device)
        w[min(text_block_start, nb):] = 2.0 ** text_amp
        lw = live.double() * w                                                    # [B, H, nq, nb]
        nums.append(lw @ vs)
        ls.append(lw @ cnt)
        tiles.append(live.sum(-1))
    # the kernel numbers a head's dense blocks after its sparse ones in q rows
    return (torch.cat(nums[::-1], 2), torch.cat(ls[::-1], 2), torch.cat(tiles[::-1], 2))


def flat_expected(v: torch.Tensor, live: torch.Tensor | None, *, nq_sparse: int, nq_dense: int, q_rows: int,
                  text_amp: int = 0, text_block_start: int = 1 << 30, kv_limit_sparse: int | None = None,
                  q_limit_sparse: int | None = None, kv_limit_dense: int | None = None,
                  out_dtype: torch.dtype | None = None) -> torch.Tensor:
    """The kernel's output [B, q_rows, H, D] for a flat case, exactly: round16(fp32(num) * fp32(1 / l))
    (the epilogue's `o * inv_l` with the IEEE reciprocal), widened to fp32 when out_dtype is fp32;
    zeros for rows past q_limit_sparse and for blocks with no live tile."""
    B, S, H, _ = v.shape
    dt = v.dtype
    num, l, tiles = flat_num_l(v, live, nq_sparse=nq_sparse, nq_dense=nq_dense, text_amp=text_amp,
                               text_block_start=text_block_start, kv_limit_sparse=kv_limit_sparse,
                               kv_limit_dense=kv_limit_dense)
    assert bool((l[tiles > 0] > 0).all()), "a block with live tiles but no live key divides by zero"
    num32, l32 = num.float(), l.float()
    assert torch.equal(num32.double(), num) and torch.equal(l32.double(), l), "sums past 24 bits"
    inv = torch.where(tiles > 0, 1.0 / l32, torch.zeros_like(l32))
    o = (num32 * inv[..., None]).to(dt)                                           # [B, H, nq, D]
    out = o.repeat_interleave(BLOCK, dim=2)[:, :, :q_rows].transpose(1, 2)        # [B, q_rows, H, D]
    ql = S if q_limit_sparse is None else q_limit_sparse
    rows = torch.arange(q_rows, device=v.device)
    dead = (rows >= ql) & (rows < nq_sparse * BLOCK)
    out = out.masked_fill(dead[None, :, None, None], 0)
    if out_dtype == torch.float32:
        out = out.float()
    return out.contiguous()


def flat_exact_bits(n_img_keys: int, n_text_keys: int, text_amp: int, v_max: int = V_MAX) -> float:
    """Significand bits the largest partial sum of a flat row can need.  Every p is a power of two;
    after any rescale by a power of two the sums keep the ratio of their magnitude to their
    granularity, which is at most v_max * sum(p) / min(p) over the live keys (a partial sum of O is
    at most v_max * sum(p); of l, sum(p) <= v_max * sum(p))."""
    w_text = 2.0 ** text_amp
    total = n_img_keys + n_text_keys * w_text
    gran = min([1.0] * (n_img_keys > 0) + [w_text] * (n_text_keys > 0))
    return math.log2(v_max * total / gran)


def flat_certified(nb: int, text_blocks: int, text_amp: int, v_max: int = V_MAX) -> bool:
    """True when every partial sum of every row of a flat case with nb key blocks fits fp32 exactly:
    the worst case has every key block live (sparse rows; dense rows are the a = 0 case)."""
    n_text = text_blocks * BLOCK
    return max(flat_exact_bits((nb - text_blocks) * BLOCK, n_text, text_amp, v_max),
               flat_exact_bits(nb * BLOCK, 0, 0, v_max)) <= 24


# ------------------------------------------------------------------------------------------------
# Leg B: fp64 rows and the per-element bound
# ------------------------------------------------------------------------------------------------
@torch.no_grad()
def fp64_rows(q, k, v, live, *, b: int, h: int, qblocks, nq_sparse: int, sm_scale: float, text_amp: float = 0.0,
              text_block_start: int = 1 << 30, kv_limit: int | None = None, q_limit: int | None = None,
              kv_limit_dense: int | None = None, chunk: int = 4, small_p: bool = False):
    """fp64 evaluation of every row of query blocks `qblocks` of (sample b, head h), masked densely,
    in the kernel's class rules (refutil.fp64_truth states them):

    - sparse blocks (< nq_sparse): scores in log2 units from Q~ = round16(fp32(q * qk_scale)) exactly
      as the kernel rounds it, fp32(text_amp) added on key blocks >= text_block_start, keys of dead
      blocks and columns >= kv_limit (default Sk) hidden, rows >= q_limit (default Sq) zero;
    - dense blocks: raw q . k * sm_scale over every key below kv_limit_dense (default nb * 128,
      the zero-filled padding included).

    q, k, v: [B, S, H, D] in the kernel's input dtype; live: [B, H, nq_sparse, nb] bool.
    Returns a dict over the rows (block order, 128 rows per block, rows past Sq dropped):
    o [R, D] O*, a [R, D] sum p|v| / sum p, mag [R] the largest sum_d |q~_d k_jd| over the row's live
    keys (in the units of the row's scores before the exponent factor), c [R] that factor (1, or
    qk_scale for dense rows), lse [R] natural-log LSE (dense rows; NaN elsewhere), tiles [R] live key
    tiles, zero [R] rows the kernel writes as zeros, and with small_p tiny [R, D] = sum over keys with
    p / max p < 2^-14 of |v| / sum p (what fp16 P loses to its subnormals)."""
    B, S, H, _ = q.shape
    Sk = k.shape[1]
    nb = (Sk + BLOCK - 1) // BLOCK
    Sp = nb * BLOCK
    dev = q.device
    kvl = Sk if kv_limit is None else kv_limit
    ql = S if q_limit is None else q_limit
    kvd = Sp if kv_limit_dense is None else kv_limit_dense
    qks = qk_scale32(sm_scale)
    amp2 = f32(text_amp)
    kd = torch.zeros(Sp, D, dtype=torch.float64, device=dev)
    vd = torch.zeros(Sp, D, dtype=torch.float64, device=dev)
    kd[:Sk], vd[:Sk] = k[b, :, h].double(), v[b, :, h].double()
    kabs, vabs = kd.abs(), vd.abs()
    cols = torch.arange(Sp, device=dev)
    bias = torch.zeros(Sp, dtype=torch.float64, device=dev)
    bias[min(text_block_start, nb) * BLOCK:] = amp2
    res = {key: [] for key in ("o", "a", "mag", "c", "lse", "tiles", "zero", "tiny")}
    qblocks = list(qblocks)
    assert qblocks == sorted(qblocks)
    groups = []
    for cls in (True, False):   # a chunk holds one class
        blocks = [m for m in qblocks if (m < nq_sparse) == cls]
        groups += [blocks[i:i + chunk] for i in range(0, len(blocks), chunk)]
    for group in groups:
        sparse = [m < nq_sparse for m in group]
        r_idx = torch.cat([torch.arange(m * BLOCK, min((m + 1) * BLOCK, S), device=dev) for m in group])
        blk = torch.cat([torch.full((min((m + 1) * BLOCK, S) - m * BLOCK,), j, device=dev)
                         for j, m in enumerate(group)])
        qr = q[b, r_idx, h]
        if sparse[0]:
            qt = (qr.float() * qks).to(q.dtype).double()
            s = qt @ kd.T + bias                                                  # log2 units
            lv = live[b, h, torch.tensor(group, device=dev)].repeat_interleave(BLOCK, -1)   # [g, Sp]
            ok = lv[blk] & (cols < kvl)[None]
            c = 1.0
        else:
            qt = qr.double()
            s = (qt @ kd.T) * (sm_scale * (1.0 / math.log(2.0)))                 # log2 units
            ok = (cols < kvd)[None].expand(len(r_idx), Sp)
            c = qks
        mag = torch.where(ok, qt.abs() @ kabs.T, torch.zeros((), dtype=torch.float64, device=dev)).amax(-1)
        s = s.masked_fill(~ok, float("-inf"))
        mx = s.amax(-1, keepdim=True)
        alive = torch.isfinite(mx)
        p = torch.exp2(s - torch.where(alive, mx, torch.zeros_like(mx)))
        l = p.sum(-1, keepdim=True)
        lsafe = torch.where(alive, l, torch.ones_like(l))
        o = (p @ vd) / lsafe
        a = (p @ vabs) / lsafe
        if small_p:
            res["tiny"].append(((p < 2.0 ** -14) & ok).double() @ vabs / lsafe)
        del s
        tiles = (live[b, h, torch.tensor(group, device=dev)].sum(-1)[blk] if sparse[0]
                 else torch.full((len(r_idx),), nb, device=dev))
        zero = ~alive[:, 0] | (tiles == 0)
        if sparse[0]:
            zero |= r_idx >= ql
        o = o.masked_fill(zero[:, None], 0.0)
        lse = ((mx[:, 0] + torch.log2(l[:, 0])) * math.log(2.0) if not sparse[0]
               else torch.full((len(r_idx),), float("nan"), dtype=torch.float64, device=dev))
        for key, val in (("o", o), ("a", a), ("mag", mag), ("lse", lse), ("tiles", tiles), ("zero", zero)):
            res[key].append(val)
        res["c"].append(torch.full((len(r_idx),), c, dtype=torch.float64, device=dev))
    out = {key: torch.cat(val) for key, val in res.items() if val}
    return out


U32 = 2.0 ** -24
EX2_REL = 2.0 ** -21                 # ex2.approx.ftz.f32: documented max error 2 ulp, with margin


def elem_bound(ref: dict, dtype: torch.dtype):
    """(E [R, D], E_lse [R]) bounds on |O - O*| per element and on |lse - lse*| per dense row, for the
    kernel's arithmetic on ref = fp64_rows(...).  Rounding points of the consumer loop
    (carved_attn_common.cuh, Consumer::softmax / run, and the epilogue of carved_attn.cu), with the
    unit roundoffs u16 = 2^-8 (bf16: 8 significant bits) or 2^-11 (fp16), u32 = 2^-24, n = tiles of the row, A = sum p|v| / sum p:

    1. scores: the wgmma's fp32 accumulation of the exact 16-bit products is within
       MMA_REL = 2^-20 of sum_d |q~_d k_jd| (select_ref); the exponent factor c (1 for sparse rows,
       qk_scale = fp32(sm_scale * 1.44269504) for dense ones, off log2(e) * sm_scale by < 2^-23
       relative) scales that; fmaf(s, c, amp - m) rounds once, and its result is >= -126 - 8 for any p
       that is not flushed: each p carries a relative error
         delta <= ln2 * (c * mag * (MMA_REL + 2^-23) + 2^-24 * 160) + EX2_REL      (ex2.approx.ftz)
       and p < 2^-126 flushes to zero: at most keys * 8 * 2^-126 / l < 2^-100 absolute (l >= 1).
       Shared by numerator and l, a relative error delta on every p moves O by <= delta (A + |O|) / (1 - delta).
    2. P is rounded to 16 bits for P.V, but l sums the unrounded p (softmax(), ~l. 293-303):
       <= u16 * A; with fp16 a p below 2^-14 of the row maximum may land on a subnormal or zero,
       an absolute 2^-25 each: 2^-25 * tiny.  The lazy rescale keeps p <= 2^8, inside both formats.
    3. O accumulates in fp32 on the tensor cores, 8 k-steps of 16 keys per tile, each step within
       2^-23 of a partial sum <= sum P|v|, and each rescale O *= alpha rounds once:
       <= 9 n 2^-23 (1 + u16) A.
    4. l is a sequential fp32 sum per thread (32 columns per tile, each rescale one product), then two
       shuffled adds: relative <= (33 n + 2) u32, which moves O by that times |O|.
    5. epilogue: fp32(1 / l), fp32(o * inv_l), then round16: <= (u16 + 2 u32) |O_kernel|, plus half
       an fp16 subnormal (2^-25) absolute, eta (2^-100 for bf16: the flushed p of item 1).

    E = (1 + 2^-10) * (E_1-4 + (u16 + 2 u32) (|O*| + E_1-4)) + eta.  The LSE, (m + log2f(l)) * ln2 in
    fp32: l's relative error delta + (33 n + 2) u32 over ln2 in log2 units, log2f within 2 ulp, the add
    and the product with ln2 one rounding each."""
    u16 = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
    o, a = ref["o"], ref["a"]
    n = ref["tiles"].double()[:, None]
    delta = (math.log(2.0) * (ref["c"] * ref["mag"] * (MMA_REL + 2.0 ** -23) + U32 * 160) + EX2_REL)[:, None]
    delta = delta * 1.01                                                            # e^x - 1 <= 1.01 x here
    e_p = delta * (a + o.abs()) / (1 - delta)
    e_round_p = u16 * (1 + delta) * a
    if dtype == torch.float16:
        e_round_p = e_round_p + 2.0 ** -25 * ref["tiny"]
    e_acc = 9 * n * 2.0 ** -23 * (1 + u16) * (1 + delta) * a
    g_l = (33 * n + 2) * U32
    e_l = g_l / (1 - g_l) * (o.abs() + e_p + e_round_p + e_acc)
    e0 = e_p + e_round_p + e_acc + e_l
    eta = 2.0 ** -25 if dtype == torch.float16 else 2.0 ** -100
    E = (1 + 2.0 ** -10) * (e0 + (u16 + 2 * U32) * (o.abs() + e0)) + eta
    E = E.masked_fill(ref["zero"][:, None], 0.0)
    lse = ref["lse"]
    rel_l = delta[:, 0] + (33 * n[:, 0] + 2) * U32
    # log2 l <= log2(keys * 2^8) < 32
    e_lse = (1 + 2.0 ** -10) * (rel_l / (1 - rel_l) + math.log(2.0) * 2.0 ** -22 * 32
                                + 3 * U32 * (lse.abs() + 32 * math.log(2.0)))
    return E, e_lse


# ------------------------------------------------------------------------------------------------
# Dense launches: varlen segments, the Wan I2V cross-attention, FP8 P.V
# ------------------------------------------------------------------------------------------------
LSE_RTOL = 2.0 ** -20                # Leg A LSE ln(keys): one fp32 log2f and one product with ln 2


def dense_expected(v: torch.Tensor, q_rows: int, *, kv_limit: int | None = None,
                   out_dtype: torch.dtype | None = None) -> torch.Tensor:
    """Leg A output [B, q_rows, H, D] of one dense-only launch (nq_sparse = 0) over v's Sk keys with the
    column limit kv_limit (default Sk, what the shims and cross-attentions pass): every query block
    walks all ceil(Sk / 128) key tiles, and only the limit keeps the zero-filled keys of the last one
    out of l."""
    Sk = v.shape[1]
    return flat_expected(v, None, nq_sparse=0, nq_dense=(q_rows + BLOCK - 1) // BLOCK, q_rows=q_rows,
                         kv_limit_dense=Sk if kv_limit is None else kv_limit, out_dtype=out_dtype)


def segments_expected(v: torch.Tensor, cu_q, cu_k, q_total: int, one=dense_expected) -> torch.Tensor:
    """Expected output [q_total, H, D] of flash_attn_varlen_func on packed v [(total keys), H, D]:
    segment i's rows cu_q[i]:cu_q[i+1] hold one(v[cu_k[i]:cu_k[i+1]][None], rows)[0], the expectation
    of one dense launch over that segment's keys alone; segments with no keys (and rows no segment
    covers) are zeros."""
    out = torch.zeros(q_total, *v.shape[1:], dtype=v.dtype, device=v.device)
    for i in range(len(cu_q) - 1):
        q0, q1, k0, k1 = int(cu_q[i]), int(cu_q[i + 1]), int(cu_k[i]), int(cu_k[i + 1])
        if q1 > q0 and k1 > k0:
            out[q0:q1] = one(v[k0:k1][None], q1 - q0)[0]
    return out


def i2v_expected(v_img: torch.Tensor, v_txt: torch.Tensor, q_rows: int) -> torch.Tensor:
    """Leg A output of wan.i2v_cross_attn: round16(f32(A_img) + f32(A_txt)), each A the dense expectation
    of its own segment's keys (each segment's column limit is its own row count)."""
    a_img = dense_expected(v_img, q_rows).float()
    a_txt = dense_expected(v_txt, q_rows).float()
    return (a_img + a_txt).to(v_img.dtype)


def i2v_bound(ref_img: dict, ref_txt: dict):
    """(O* [R, D], E [R, D]) for wan.i2v_cross_attn on the rows of fp64_rows over the image keys (ref_img)
    and over the text keys (ref_txt), both dense with kv_limit_dense = the segment's row count.

    The kernel runs each segment through the dense consumer loop and rounds each result to bf16 as the
    dense epilogue does, so |A_seg - O*_seg| <= E_seg = elem_bound(ref_seg) (round16 included).  Then
    s = f32(A_img) + f32(A_txt) is one fp32 add (relative u32) and out = round16(s) one more rounding
    (relative u16).  With S* = O*_img + O*_txt, |A_img + A_txt - S*| <= E_img + E_txt and
    |A_img + A_txt| <= |S*| + E_img + E_txt, so
      |out - S*| <= E_img + E_txt + (u16 + 2 u32) (|S*| + E_img + E_txt),
    the second term covering (1 + u32)(1 + u16) - 1 < u16 + 2 u32 of the two roundings."""
    E_i, _ = elem_bound(ref_img, torch.bfloat16)
    E_t, _ = elem_bound(ref_txt, torch.bfloat16)
    o = ref_img["o"] + ref_txt["o"]
    return o, E_i + E_t + (2.0 ** -8 + 2 * U32) * (o.abs() + E_i + E_t)


E4M3_MAX = 448.0
FP8_CERT_BITS = 12                   # the FP8 wgmma's accumulator is narrower than fp32 (linear_fp8.cu)


def fp8_case(B: int, S: int, H: int, *, seed: int, device, amax=None, nnz: int = 16):
    """q = 0, k ~ N(0, 1), and a sparse v for the FP8 P.V leg: in every (sample, head, channel) nnz keys
    drawn at random hold +-2^e, e in 0..log2(amax[b]), the rest 0, and one key of every (sample, head)
    holds +-amax[b] (default 8 in every sample), so the head's amax is amax[b] and fp8.cu's
    e4m3(v * 448 / amax) is exact.  [B, S, H, D] bf16."""
    amax = [V_MAX] * B if amax is None else list(amax)
    g = torch.Generator(device=device).manual_seed(seed)
    q = torch.zeros(B, S, H, D, dtype=torch.bfloat16, device=device)
    k = torch.randn(B, S, H, D, generator=g, device=device).to(torch.bfloat16)
    v = torch.zeros(B, S, H, D, dtype=torch.float32, device=device)
    for b in range(B):
        e_max = int(math.log2(amax[b]))
        assert 2 ** e_max == amax[b]
        idx = torch.randint(0, S, (nnz, H, D), generator=g, device=device)
        mag = 2.0 ** torch.randint(0, e_max + 1, (nnz, H, D), generator=g, device=device)
        sign = torch.randint(0, 2, (nnz, H, D), generator=g, device=device) * 2 - 1
        v[b].scatter_(0, idx, mag * sign)
        at = torch.randint(0, S, (H,), generator=g, device=device)
        v[b, at, torch.arange(H, device=device), 0] = float(amax[b])
    return q, k, v.to(torch.bfloat16)


def fp8_codes(v: torch.Tensor):
    """(codes [B, S, H, D] fp32, amax [B, H] fp32) of fp8.cu: amax = max |v| of the (sample, head),
    codes the e4m3 values of satfinite(v * fp32(448 / amax)) (scale 1 where amax is 0)."""
    from test_producers_cpu import e4m3_satfinite
    amax = v.float().abs().amax(dim=(1, 3))                                     # [B, H]
    inv = torch.where(amax > 0, torch.tensor(E4M3_MAX, device=v.device) / amax, torch.ones_like(amax))
    codes = e4m3_satfinite(v.float() * inv[:, None, :, None]).view(torch.float8_e4m3fn).float()
    return codes, amax


def fp8_cert_ratio(codes: torch.Tensor, kv_limit: int | None = None) -> float:
    """Largest |partial sum| of a flat FP8 row over its granularity: with every p = 1 (exact in e4m3) a
    partial sum of channel d is at most sum |code| over the keys, and every code is a multiple of the
    lowest power of two among the channel's codes (the codes here are integers)."""
    c = codes[:, :kv_limit].double()
    ci = c.abs().long()
    low = torch.where(ci > 0, ci & -ci, torch.full_like(ci, 1 << 40)).amin(1).double().clamp_max(2.0 ** 40)
    tot = c.abs().sum(1)
    return float(torch.where(tot > 0, tot / low, torch.zeros_like(tot)).max())


def fp8_certified(codes: torch.Tensor, kv_limit: int | None = None) -> bool:
    """True when every partial sum stays within 2^12 units of its granularity: deliberately
    conservative, since Hopper's FP8 wgmma accumulates in fewer bits than fp32."""
    return fp8_cert_ratio(codes, kv_limit) <= 2.0 ** FP8_CERT_BITS


def fp8_expected(v: torch.Tensor, q_rows: int, *, kv_limit: int | None = None) -> torch.Tensor:
    """Leg A output [B, q_rows, H, D] of one dense-only FP8 P.V launch on v quantised by fp8.cu (one
    amax per (sample, head) of this launch's v), q = 0: num8 = sum of the codes below the column limit
    (exact when fp8_certified), l the number of those keys, and the epilogue of carved_attn.cu
    restated in its order:
      inv_l = fp32(1 / l);  inv_l = fp32(inv_l * fp32(amax * fp32(1 / 448)));  out = round16(fp32(num8) * inv_l)."""
    B, Sk, H, _ = v.shape
    kvl = Sk if kv_limit is None else kv_limit
    codes, amax = fp8_codes(v)
    assert fp8_certified(codes, kvl), "FP8 partial sums past the certificate"
    num8 = codes[:, :kvl].double().sum(1)                                       # [B, H, D]
    n32 = num8.float()
    assert torch.equal(n32.double(), num8)
    l = min(kvl, (Sk + BLOCK - 1) // BLOCK * BLOCK)                             # keys that score p = 1
    inv_l = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(l), dtype=torch.float32)
    unscale = amax * torch.tensor(1.0 / E4M3_MAX, dtype=torch.float32).item()  # fp32(amax * fp32(1/448))
    inv = (inv_l.to(v.device) * unscale).float()                                # [B, H]
    o = (n32 * inv[..., None]).to(v.dtype)                                      # [B, H, D]
    return o[:, None].expand(B, q_rows, H, D).contiguous()
