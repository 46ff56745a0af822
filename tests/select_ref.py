"""Exact restatements of block pooling and pooled scoring, and a certified selection oracle.

Shared by tests/test_select_oracle_cpu.py and tests/test_select_edges_gpu.py.  Every function is
plain torch and runs on the device of its inputs.

Why exact restatements are possible:
- A product of two bf16 (or two fp16) values is exact in fp32, so the fused kernel's `fmaf` chain
  over d ascending (and the SIMT GEMM's) equals a sequential fp32 `acc = acc + q[d]*k[d]`, as long
  as no product underflows fp32's normal range (true for any data the tests build).
- block_pool adds the 128 rows of a block in row order in fp32, multiplies by 1/128 (exact) and
  rounds once.
- The tensor-core GEMM's summation order is unknown, but its fp32 result lies within
  2^-20 * sum|q*k| of the exact dot product (MMA_REL below), which certifies the set of scores it
  may round to.
- Selection from given scores: equal scores give bit-equal fp32 probabilities, so only the cut
  position (fp32 cumulative sum against p) and near-equal probabilities are uncertain; both are
  bounded and reported as ambiguous rows.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

BLOCK = 128
# fp32 accumulation bound over <= 128 terms in any order, relative to sum|terms| (gamma_127 < 2^-17)
ACC_REL = 2.0 ** -16
# mma.sync m16n8k16 with fp32 accumulation over D = 128: products are exact, and each of the 8
# k-steps ends in one (at worst truncating) normalisation, an error below 2^-23 of a partial sum
# that is at most sum|q*k|: 8 * 2^-23 = 2^-20.  (On an H100 every observed score lies within 2^-22.)
MMA_REL = 2.0 ** -20
# fp32 cumulative probability vs fp64, n_img <= 2100: probabilities within ~3 ulp after expf and the
# division, a normaliser summed as <= 66-term lane partials and a 5-level butterfly, the cumulative
# sum as <= 66-term lane chunks and a 5-level scan: < 150 * 2^-24 < 2^-16
CUT_BAND = 2.0 ** -16
TIE_REL = 2.0 ** -21   # fp64 probabilities this close may round (or expf) to equal / swapped fp32
TIE_ABS = 4 * 2.0 ** -149  # the same in the fp32 subnormal range: a few subnormal ulps
ZERO_PROB = 2.0 ** -160    # below this an fp32 probability is certainly +0


def _fmt(dt):
    """(fraction bits, smallest normal exponent) of a 16-bit float type."""
    if dt == torch.bfloat16:
        return 7, -126
    if dt == torch.float16:
        return 10, -14
    raise ValueError(dt)


def ulp(x: torch.Tensor, dt) -> torch.Tensor:
    """ulp (fp64) of dtype `dt` in the binade of |x| (subnormal spacing below the normal range)."""
    frac, emin = _fmt(dt)
    x = x.double().abs()
    _, e = torch.frexp(x)
    e = torch.where(x == 0, torch.full_like(e, emin), e - 1)
    return torch.exp2((torch.clamp(e, min=emin) - frac).double())


def round_fp64(y: torch.Tensor, dt) -> torch.Tensor:
    """Round-to-nearest-even of fp64 `y` to dtype `dt`, computed in fp64 with one rounding
    (a cast through fp32 would round twice).  Returns fp64 values representable in `dt`."""
    y = y.double()
    u = ulp(y, dt)
    return torch.round(y / u) * u  # y / u is exact (power of two); torch.round is half-to-even


# ------------------------------------------------------------------------------------------------
# pooling
# ------------------------------------------------------------------------------------------------
def _rows_of_blocks(x, n_blocks, r):
    """Row r of every block, [B, n_blocks, H, D], with rows >= S given as None mask."""
    S = x.shape[1]
    idx = torch.arange(n_blocks, device=x.device) * BLOCK + r
    valid = idx < S
    rows = x.index_select(1, idx.clamp(max=S - 1))
    return rows, valid.view(1, -1, 1, 1)


def pool_exact(x: torch.Tensor, n_blocks: int, out_dtype=None) -> torch.Tensor:
    """block_pool restated: x [B,S,H,D] (bf16, fp16, or fp32 which is first rounded to bf16
    element by element) -> [B,H,n_blocks,D] in the pooled dtype.  fp32 sum of the block's rows in
    row order (rows >= S are not added), then `* (1/128)` and one rounding."""
    if out_dtype is None:
        out_dtype = torch.bfloat16 if x.dtype == torch.float32 else x.dtype
    B, S, H, D = x.shape
    acc = torch.zeros(B, n_blocks, H, D, dtype=torch.float32, device=x.device)
    for r in range(BLOCK):
        rows, valid = _rows_of_blocks(x, n_blocks, r)
        if x.dtype == torch.float32:
            rows = rows.to(torch.bfloat16)
        acc = torch.where(valid, acc + rows.float(), acc)
    out = (acc * (1.0 / BLOCK)).to(out_dtype)
    return out.permute(0, 2, 1, 3).contiguous()


def pool_fp64(x: torch.Tensor, n_blocks: int):
    """fp64 block means (zero padding) and the fp64 sum of |x| per pooled element, both
    [B,H,n_blocks,D].  fp32 input is rounded to bf16 first, as block_pool does."""
    B, S, H, D = x.shape
    s = torch.zeros(B, n_blocks, H, D, dtype=torch.float64, device=x.device)
    a = torch.zeros_like(s)
    for r in range(BLOCK):
        rows, valid = _rows_of_blocks(x, n_blocks, r)
        if x.dtype == torch.float32:
            rows = rows.to(torch.bfloat16)
        rows = torch.where(valid, rows.double(), torch.zeros((), dtype=torch.float64, device=x.device))
        s += rows
        a += rows.abs()
    return (s / BLOCK).permute(0, 2, 1, 3), (a / BLOCK).permute(0, 2, 1, 3)


def assert_pool_certified(got: torch.Tensor, mean64: torch.Tensor, abs_mean64: torch.Tensor, what=""):
    """Every pooled element within half an ulp (of its binade) of the fp64 mean plus the fp32
    accumulation bound, in any summation order."""
    dt = got.dtype
    bound = ACC_REL * abs_mean64
    u = torch.maximum(ulp(mean64.abs() + bound, dt), ulp(got.double(), dt))
    err = (got.double() - mean64).abs()
    bad = err > 0.5 * u + bound
    assert not bad.any(), (what, int(bad.sum()), float((err - 0.5 * u - bound).max()))


# ------------------------------------------------------------------------------------------------
# pooled scores
# ------------------------------------------------------------------------------------------------
def _flat(qp, kp, n_img):
    D = qp.shape[-1]
    return qp.reshape(-1, qp.shape[-2], D), kp.reshape(-1, kp.shape[-2], D)[:, :n_img], D


def _scale(D, device):
    return torch.tensor(1.0 / math.sqrt(D), dtype=torch.float32, device=device)


def scores_exact(qp: torch.Tensor, kp: torch.Tensor, n_img: int) -> torch.Tensor:
    """Fused / SIMT score arithmetic: [BH, nq, n_img] fp32 holding dtype values.
    acc = acc + q[d]*k[d] in fp32 over d ascending, then round(round(acc) * float32(D^-1/2))."""
    dt = qp.dtype
    q, k, D = _flat(qp, kp, n_img)
    q, k = q.float(), k.float()
    acc = torch.zeros(q.shape[0], q.shape[1], k.shape[1], dtype=torch.float32, device=q.device)
    for d in range(D):
        prod = q[:, :, d, None] * k[:, None, :, d]  # exact
        acc = acc + prod
    s = acc.to(dt).float() * _scale(D, q.device)
    return s.to(dt).float()


def scores_certified(qp: torch.Tensor, kp: torch.Tensor, n_img: int, rel: float = MMA_REL):
    """Certified scores of any fp32 accumulation order: (exact fp64 dot products, lowest allowed
    score, highest allowed score, ambiguous map).  The first rounding may land on any dtype value
    that rounds from [exact - b, exact + b] with b = rel * sum|q*k|; the allowed final scores
    are that range pushed through the second rounding (fp32 product with D^-1/2, then dtype)."""
    dt = qp.dtype
    q, k, D = _flat(qp, kp, n_img)
    q64, k64 = q.double(), k.double()
    exact = q64 @ k64.transpose(1, 2)
    band = rel * (q64.abs() @ k64.abs().transpose(1, 2))
    lo1 = round_fp64(exact - band, dt)
    hi1 = round_fp64(exact + band, dt)
    c = _scale(D, q.device)
    lo = (lo1.float() * c).to(dt).float()
    hi = (hi1.float() * c).to(dt).float()
    return exact, lo, hi, lo != hi


# ------------------------------------------------------------------------------------------------
# selection
# ------------------------------------------------------------------------------------------------
def pack_bits(onehot: torch.Tensor, words: int) -> torch.Tensor:
    """[R, n] bool -> [R, words] int32 bit rows (bit c of word w is column 32w + c)."""
    R, n = onehot.shape
    full = torch.zeros(R, words * 32, dtype=torch.int64, device=onehot.device)
    full[:, :min(n, words * 32)] = onehot[:, :words * 32].long()
    v = (full.view(R, words, 32) << torch.arange(32, device=onehot.device)).sum(-1)
    return torch.where(v >= 2 ** 31, v - 2 ** 32, v).to(torch.int32)


def unpack_bits(bits: torch.Tensor, n: int) -> torch.Tensor:
    """[R, words] int32 -> [R, n] bool."""
    sh = torch.arange(32, device=bits.device, dtype=torch.int32)
    return ((bits.unsqueeze(-1) >> sh) & 1).bool().flatten(-2)[..., :n]


@dataclass
class Selection:
    order: torch.Tensor      # [R, n_img] block indices in rank order
    probs: torch.Tensor      # [R, n_img] fp64 softmax (by block index)
    csum: torch.Tensor       # [R, n_img] fp64 cumulative sum in rank order
    count_lo: torch.Tensor   # [R] smallest allowed count
    count_hi: torch.Tensor   # [R] largest allowed count
    group_lo: torch.Tensor   # [R, n_img+1] for a cut at n: first rank of the near-tie group it splits
    group_hi: torch.Tensor   # [R, n_img+1] ... and one past its last rank (== n when not split)
    union: torch.Tensor      # [R, words*32] bool: neighbour / first-frame / text columns
    n_img: int
    nb: int
    words: int

    @property
    def count(self):
        """The count where it is certain (count_lo == count_hi)."""
        return self.count_lo

    def ranked_onehot(self, n: torch.Tensor) -> torch.Tensor:
        R = self.order.shape[0]
        rank = torch.arange(self.n_img, device=self.order.device).expand(R, -1)
        keep = rank < n.view(-1, 1)
        sel = torch.zeros(R, self.n_img, dtype=torch.bool, device=self.order.device)
        return sel.scatter(1, self.order, keep)

    def bits_for(self, n: torch.Tensor) -> torch.Tensor:
        """Packed rows [R, words] from the first n[r] ranked blocks plus the unions."""
        R = self.order.shape[0]
        oh = self.union.clone()
        oh[:, :self.n_img] |= self.ranked_onehot(n.to(self.order.device).long())
        return pack_bits(oh, self.words)

    def tie_split(self, n: torch.Tensor) -> torch.Tensor:
        """[R] bool: the cut after n ranked blocks splits a group of near-equal probabilities."""
        n = n.to(self.order.device).long().view(-1, 1)
        return (self.group_lo.gather(1, n) != n).view(-1) | (self.group_hi.gather(1, n) != n).view(-1)

    def check(self, bits: torch.Tensor, counts: torch.Tensor, what: str = ""):
        """Asserts the kernel's packed rows [R, words] and counts [R] against the oracle; returns
        (fraction of count-ambiguous rows, fraction of tie-ambiguous rows)."""
        dev = self.order.device
        bits = bits.reshape(-1, self.words).to(dev)
        n = counts.reshape(-1).to(dev).long()
        bad = (n < self.count_lo) | (n > self.count_hi)
        assert not bad.any(), (what, "count outside the certified set", int(bad.sum()),
                               _first(bad, n, self.count_lo, self.count_hi))
        split = self.tie_split(n)
        want = self.bits_for(n)
        row_bad = (bits != want).any(-1) & ~split
        assert not row_bad.any(), (what, "bit row != bits_for(count)", int(row_bad.sum()),
                                   _first(row_bad, bits, want))
        if split.any():
            ng = n.view(-1, 1)
            lo = self.bits_for(self.group_lo.gather(1, ng).view(-1))
            hi = self.bits_for(self.group_hi.gather(1, ng).view(-1))
            sub = ((lo & ~bits) != 0).any(-1) | ((bits & ~hi) != 0).any(-1)
            sub &= split
            assert not sub.any(), (what, "near-tie row outside its group", int(sub.sum()))
        count_amb = self.count_lo != self.count_hi
        return count_amb.float().mean().item(), split.float().mean().item()


def _first(mask, *ts):
    i = int(mask.nonzero()[0, 0])
    return i, [t[i].tolist() for t in ts]


def select_oracle(scores: torch.Tensor, n_img: int, nb: int, top_k: int, p: float, text_blocks: int,
                  ff: int, nbr_bits: torch.Tensor | None = None, nbr_rows: int | None = None,
                  nbr_words: int | None = None, nq: int | None = None, cut_band: float = CUT_BAND) -> Selection:
    """Selection oracle working from the kernel's own scores [..., nq, n_img] (fp32 holding dtype
    values).  Rank order: score descending, then index ascending, except that blocks whose fp32
    probability is certainly zero tie and go in index order.  fp64 softmax and cumulative sum;
    allowed counts #(C <= p - d) + 1 .. #(C <= p + d) + 1 (d = CUT_BAND), then max(., top_k) and at most
    n_img (`cut_band` = 0 where the fp32 cumulative sum is exact, e.g. dyadic probabilities).  Unions: neighbour bits masked to [0, n_img) (rows < nbr_rows, words < nbr_words),
    first-frame columns [0, min(ff, nb)) on rows m < ff, text columns [n_img, min(n_img + text, nb)),
    nothing at or past nb."""
    nq = scores.shape[-2] if nq is None else nq
    s = scores.reshape(-1, n_img).double()
    R, dev = s.shape[0], s.device
    words = (nb + 31) // 32
    probs = torch.softmax(s, dim=-1)
    key = torch.where(probs < ZERO_PROB, torch.full_like(s, -math.inf), s)
    _, order = torch.sort(key, dim=-1, descending=True, stable=True)
    sp = probs.gather(1, order)
    csum = torch.cumsum(sp, dim=-1)
    lo = (csum <= p - cut_band).sum(-1) + 1
    hi = (csum <= p + cut_band).sum(-1) + 1
    lo = lo.clamp(min=top_k).clamp(max=n_img)
    hi = hi.clamp(min=top_k).clamp(max=n_img)
    # near-equal neighbours in rank order: distinct scores whose fp32 probabilities may tie or swap
    ss = s.gather(1, order)
    a, b = sp[:, :-1], sp[:, 1:]
    both_zero = (a < ZERO_PROB) & (b < ZERO_PROB)
    eq = ss[:, :-1] == ss[:, 1:]
    near = ~eq & ~both_zero & ((a - b).abs() <= TIE_REL * torch.maximum(a, b) + TIE_ABS)
    # a run of equal scores next to a near-equal one joins its group: the kernel orders all of
    # them by index once their fp32 probabilities coincide
    run = torch.cat([torch.zeros(R, 1, dtype=torch.long, device=dev), (~eq).long().cumsum(1)], 1)
    touched = torch.zeros(R, n_img, dtype=torch.bool, device=dev)
    touched[:, :-1] |= near
    touched[:, 1:] |= near
    run_touched = torch.zeros(R, n_img, dtype=torch.long, device=dev).scatter_reduce(
        1, run, touched.long(), reduce="amax")
    link = near | (eq & run_touched.gather(1, run[:, :-1]).bool())
    # link[i]: ranks i and i+1 in one group.  For a cut at n: group of ranks n-1 and n.
    pos = torch.arange(n_img, device=dev).expand(R, -1)
    starts = torch.where(torch.cat([torch.ones(R, 1, dtype=torch.bool, device=dev), ~link], 1), pos,
                         torch.zeros_like(pos))
    gstart = torch.cummax(starts, 1).values                       # first rank of the group of rank i
    ends = torch.where(torch.cat([~link, torch.ones(R, 1, dtype=torch.bool, device=dev)], 1), pos + 1,
                       torch.full_like(pos, n_img + 1))
    gend = torch.flip(torch.cummin(torch.flip(ends, [1]), 1).values, [1])  # one past the group's last rank
    split = torch.zeros(R, n_img + 1, dtype=torch.bool, device=dev)
    split[:, 1:n_img] = link
    n_all = torch.arange(n_img + 1, device=dev).expand(R, -1)
    g_lo = torch.where(split, gstart[:, :n_img].gather(1, (n_all - 1).clamp(min=0)), n_all)
    g_hi = torch.where(split, gend.gather(1, n_all.clamp(max=n_img - 1)), n_all)
    # unions
    cols = torch.arange(words * 32, device=dev)
    m = torch.arange(R, device=dev) % nq
    union = torch.zeros(R, words * 32, dtype=torch.bool, device=dev)
    if nbr_bits is not None:
        nbr_rows = nbr_bits.shape[0] if nbr_rows is None else nbr_rows
        nbr_words = nbr_bits.shape[1] if nbr_words is None else nbr_words
        nb_oh = unpack_bits(nbr_bits.reshape(-1)[:nbr_rows * nbr_words].view(nbr_rows, nbr_words).to(dev),
                            nbr_words * 32)
        rows = torch.zeros(nq, words * 32, dtype=torch.bool, device=dev)
        r_n, c_n = min(nq, nbr_rows), min(words * 32, nbr_words * 32, n_img)
        rows[:r_n, :c_n] = nb_oh[:r_n, :c_n]
        union |= rows[m]
    if ff > 0:
        union |= (m < ff).view(-1, 1) & (cols < min(ff, nb)).view(1, -1)
    if text_blocks > 0:
        union |= ((cols >= n_img) & (cols < min(n_img + text_blocks, nb))).view(1, -1)
    return Selection(order=order, probs=probs, csum=csum, count_lo=lo, count_hi=hi, group_lo=g_lo,
                     group_hi=g_hi, union=union, n_img=n_img, nb=nb, words=words)
