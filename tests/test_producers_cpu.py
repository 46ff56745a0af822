"""Exact restatements of the attention producers (HunyuanVideo and Wan prologues, the INT8 Q/K and FP8 V
quantisers) and the error bounds the GPU tests (tests/test_producers_gpu.py) hold them to, checked here
without a GPU.

The restatements repeat each kernel's own arithmetic in torch, so that most GPU checks are bit identity:
  - e4m3 "satfinite, round to nearest even": clamp(+-448) then ATen's cast;
  - the INT8 code: torch.round, which rounds half to even like rintf;
  - mean(x^2) of a HunyuanVideo head row in the kernel's order: per lane a sequential fp32 sum over its 8
    channels, then the xor tree over lane offsets 8, 4, 2, 1; of a Wan token row: per lane its pairs
    (2l, 2l+1) + 64 j in order, then a 5-level tree.  Squares of 16-bit values are exact in fp32, so the
    kernel's fmaf(x, x, s) is s + x*x rounded once, and the restatement is exact;
  - the pooled block means of the bulk prologue: its work split over CTAs (whole blocks in contiguous
    chunks, the left-over blocks cut into P parts), even / odd token groups summed apart, then the P
    parts in part order.

Where a GPU check compares with fp64 instead, the bound comes from the depth of the fp32 summation
(Higham's gamma_n = n u / (1 - n u), u = 2^-24): tested here on random fp32 cases.
"""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))

U32 = 2.0 ** -24
E4M3_MAX = 448.0


def gamma(n: int) -> float:
    """Higham's gamma_n for fp32: |fl(sum) - sum| <= gamma_(depth) * sum |x| for a summation of that depth."""
    return n * U32 / (1 - n * U32)


# ------------------------------------------------------------------ e4m3 and int8 rounding
def e4m3_satfinite(x: torch.Tensor) -> torch.Tensor:
    """cvt.rn.satfinite.e4m3: round to nearest even, out-of-range values to +-448.  Returns the bytes."""
    return x.float().clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8)


def int8_code(y: torch.Tensor, sc: torch.Tensor) -> torch.Tensor:
    """clamp(rintf(y / sc), +-127), code 0 where sc == 0.  sc must be a tensor: a CUDA division by a
    Python scalar is a multiplication by its reciprocal, not an IEEE division."""
    return torch.where(sc > 0, torch.round(y / sc).clamp(-127, 127), torch.zeros_like(y))


# ------------------------------------------------------------------ sums of squares in kernel order
def hy_sumsq(x: torch.Tensor) -> torch.Tensor:
    """sum(x^2) over the last dim (128) as the HunyuanVideo prologue forms it: lane l holds channels
    8l..8l+7 and sums their squares in order, then ss += shfl_xor(ss, 8, 4, 2, 1).  x fp32."""
    s = x.reshape(*x.shape[:-1], 16, 8)
    acc = torch.zeros(s.shape[:-1], dtype=torch.float32, device=x.device)
    for i in range(8):
        acc = acc + s[..., i] * s[..., i]
    for half in (8, 4, 2, 1):
        acc = acc[..., :half] + acc[..., half:2 * half]
    return acc[..., 0]


def wan_sumsq(x: torch.Tensor) -> torch.Tensor:
    """sum(x^2) over the last dim (C = 64 j) as the Wan prologue forms it: lane l takes the pairs
    (64 j + 2 l, 64 j + 2 l + 1) for j in order, then a 5-level xor tree.  x bf16 (exact squares, so fp32
    adds are the kernel's fmaf) or fp32, where fmaf is emulated in fp64: one rounding to fp32 after an
    fp64 sum, which differs from fmaf only when the fp64 sum lands on an fp32 tie."""
    C = x.shape[-1]
    fp32_in = x.dtype == torch.float32
    v = x.float().reshape(*x.shape[:-1], C // 64, 32, 2)
    acc = torch.zeros(v.shape[:-3] + (32,), dtype=torch.float32, device=x.device)
    for j in range(C // 64):
        for t in range(2):
            a = v[..., j, :, t]
            acc = (acc.double() + a.double() * a.double()).float() if fp32_in else acc + a * a
    for half in (16, 8, 4, 2, 1):
        acc = acc[..., :half] + acc[..., half:2 * half]
    return acc[..., 0]


# ------------------------------------------------------------------ HunyuanVideo prologue rows
def hy_rows(x16: torch.Tensor, w16, cs, eps: float, kernel_order: bool) -> torch.Tensor:
    """The classic kernel's chain for head rows x16 [..., 128] (bf16 / fp16):
    n = r16(x * rsqrt(mean(x^2) + eps)), y = r16(n * w), r = r16(y cos - y_odd sin | y_odd cos + y sin)
    with separate fp32 products and sum, interleaved pairs.  cs = (cos, sin) broadcastable to x (None: no
    RoPE).  kernel_order: mean(x^2) in the kernel's order (exact), else torch's reduction."""
    dt = x16.dtype
    x = x16.float()
    ss = hy_sumsq(x) * (1.0 / 128) if kernel_order else x.pow(2).mean(-1)
    r = torch.rsqrt(ss + eps)
    n = (x * r[..., None]).to(dt).float()
    if w16 is not None:
        n = (n * w16.float()).to(dt).float()
    if cs is None:
        return n.to(dt)
    c, s = cs
    y0, y1 = n[..., 0::2], n[..., 1::2]
    a0 = y0 * c[..., 0::2] + (-y1) * s[..., 0::2]
    a1 = y1 * c[..., 1::2] + y0 * s[..., 1::2]
    return torch.stack([a0, a1], -1).flatten(-2).to(dt)


# ------------------------------------------------------------------ pooled block means
def bulk_split(nbk: int, ctas: int):
    """prologue_bulk.cu's host split of nbk blocks over `ctas` CTAs: (whole blocks per CTA, left-over
    blocks, parts per left-over block)."""
    n_full, R = divmod(nbk, ctas)
    P = 1
    if R:
        while P < 8 and R * P * 2 <= ctas:
            P *= 2
    return n_full, R, P


def pool_slots(B: int, S: int, ctas: int | None):
    """Accumulator of every token in the bulk kernel (ctas given) or the classic kernel (None):
    slot [B * nb, 128] int64 = 2 * part + group, and split [B * nb] bool (block cut into P > 1 parts).
    A CTA's two token groups take the tokens of its items alternately, counting across items."""
    nb = (S + 127) // 128
    nbk = nb * B
    slot = np.zeros((nbk, 128), dtype=np.int64)
    split = np.zeros(nbk, dtype=bool)
    if ctas is None:
        return torch.from_numpy(slot), torch.from_numpy(split), 1
    n_full, R, P = bulk_split(nbk, ctas)
    for c in range(ctas if n_full > 0 else R * P):
        items = [(c * n_full + i, 0, 128) for i in range(n_full)]
        if c < R * P:
            items.append((n_full * ctas + c // P, c % P, 128 // P))
            split[n_full * ctas + c // P] = P > 1
        nbase = 0
        for g, part, per in items:
            tok0 = (g % nb) * 128 + part * per
            nt = max(0, min(per, S - tok0))
            t = np.arange(nt)
            slot[g, part * per + t] = 2 * part + (nbase + t) % 2
            nbase += nt
    return torch.from_numpy(slot), torch.from_numpy(split), P


def pooled_means(y: torch.Tensor, slot: torch.Tensor, split: torch.Tensor, P: int) -> torch.Tensor:
    """Block means of y [B, S, H, 128] (the kernel's own q or k) in the kernel's fp32 order, rounded to
    y's dtype: per slot a sequential sum in token order, then group 0 + group 1, and for a split block
    the parts added in part order.  Missing tail tokens count as zeros.  Returns [B, H, nb, 128]."""
    B, S, H, D = y.shape
    nb = (S + 127) // 128
    yp = torch.zeros(B, nb * 128, H * D, dtype=torch.float32, device=y.device)
    yp[:, :S] = y.reshape(B, S, H * D).float()
    yp = yp.view(B * nb, 128, H * D)
    slot, split = slot.to(y.device), split.to(y.device)
    acc = torch.zeros(B * nb, 16, H * D, dtype=torch.float32, device=y.device)
    rows = torch.arange(B * nb, device=y.device)
    for t in range(128):
        acc[rows, slot[:, t]] = acc[rows, slot[:, t]] + yp[:, t]
    parts = acc[:, 0::2] + acc[:, 1::2]
    total = parts[:, 0].clone()
    for p in range(1, P):
        total = torch.where(split[:, None], total + parts[:, p], total)
    return (total * (1.0 / 128)).to(y.dtype).view(B, nb, H, D).permute(0, 2, 1, 3)


def order_sensitive_rows(B: int, n: int, tok0: int, H: int, g, device) -> torch.Tensor:
    """Pre-norm head rows [B, n, H, 128] (token tok0 + i of the sequence) whose normalised block sums round
    differently in every fp32 order: at block positions p = 0, 3 (mod 4) a constant row of sign + for
    p mod 64 < 32 and - after (normalised to +-1, cancelling over each 64 tokens), elsewhere a spike in
    channel 0 and values near 2^-20 (normalised near 2^-16.5), which partial sums of size 8..16 round."""
    p = (torch.arange(n, device=device) + tok0) % 128
    big = ((p % 4 == 0) | (p % 4 == 3))[None, :, None, None]
    sign = torch.where(p % 64 < 32, 1.0, -1.0)[None, :, None, None]
    tiny = torch.randn(B, n, H, 128, generator=g, device=device) * 2.0 ** -20
    tiny[..., 0] = 1.0
    return torch.where(big, sign.expand(B, n, H, 128), tiny)


def pool_depth(P: int, split: bool, classic: bool) -> int:
    """Additions a token's value goes through on its way into the kernel's fp32 block sum."""
    if classic:
        return 127
    per = 128 // P if split else 128
    return (per + 1) // 2 + (P - 1 if split else 0)


def pool_bound(abs_sum: torch.Tensor, depth: int) -> torch.Tensor:
    """The fp32 block mean is within gamma_depth * sum|y| / 128 of the exact mean (the 16-bit output then
    within that plus half an ulp: within_rounding)."""
    return gamma(depth) * abs_sum / 128


def ulp16(v: torch.Tensor, dtype) -> torch.Tensor:
    """ulp of a bf16 / fp16 value of magnitude |v| (subnormal spacing below the normal range)."""
    mant, emin = (7, -126) if dtype == torch.bfloat16 else (10, -14)
    e = torch.floor(torch.log2(v.abs().double().clamp_min(2.0 ** emin))).clamp_min(emin)
    return torch.exp2(e - mant)


def within_rounding(got: torch.Tensor, exact: torch.Tensor, err: torch.Tensor) -> torch.Tensor:
    """got (16-bit) is a round-to-nearest of some value within err of exact (fp64)."""
    return (got.double() - exact).abs() <= err + ulp16(exact.abs() + err, got.dtype) / 2


# ------------------------------------------------------------------ INT8 quantiser mean and shift
def colsum_mean(x: torch.Tensor) -> torch.Tensor:
    """qk_int8.cu's column mean of x [B, S, H, 128] in its fp32 order: per 128-row block, lane r0 sums
    rows r0 + 16 i (i = 0..7), then the 16 lanes in order; the blocks in order; / S.  [B*H, 128]."""
    B, S, H, D = x.shape
    nblk = (S + 127) // 128
    xp = torch.zeros(B, nblk * 128, H, D, dtype=torch.float32, device=x.device)
    xp[:, :S] = x.float()
    xp = xp.view(B, nblk, 8, 16, H, D)
    acc = xp[:, :, 0]
    for i in range(1, 8):
        acc = acc + xp[:, :, i]
    blk = acc[:, :, 0]
    for r in range(1, 16):
        blk = blk + acc[:, :, r]
    s = blk[:, 0]
    for b in range(1, nblk):
        s = s + blk[:, b]
    s = s.reshape(B * H, D)
    return s / torch.full_like(s, float(S))


def mean_depth(S: int) -> int:
    return 8 + 16 + (S + 127) // 128


def mean_bound(abs_colsum: torch.Tensor, mean64: torch.Tensor, S: int) -> torch.Tensor:
    """|kernel mean - exact mean|: the block-then-blocks fp32 sum, then one rounded division."""
    return gamma(mean_depth(S)) * abs_colsum / S * (1 + U32) + U32 * mean64.abs()


def shift_bound(sc: torch.Tensor, abs_dot: torch.Tensor, shift64: torch.Tensor) -> torch.Tensor:
    """|kernel shift - sc * sum(code * kmean)|: an 8-term fma chain + 4-level tree, then * sc."""
    return sc * gamma(12) * abs_dot * (1 + U32) + U32 * shift64.abs()


# ====================================================================== tests
def _e4m3_table():
    codes = torch.arange(256, dtype=torch.uint8)
    vals = codes.view(torch.float8_e4m3fn).float()
    return codes, vals


def test_e4m3_satfinite_against_exhaustive_enumeration():
    codes, vals = _e4m3_table()
    finite = ~torch.isnan(vals)
    # every e4m3 value maps to its own code (+0 and -0 apart)
    assert torch.equal(e4m3_satfinite(vals[finite]), codes[finite])
    assert e4m3_satfinite(torch.tensor([-0.0])).item() == 0x80
    pos = codes[(vals > 0) & finite]
    pos_v = pos.view(torch.float8_e4m3fn).float()
    order = torch.argsort(pos_v)
    pos, pos_v = pos[order], pos_v[order]
    assert pos_v[-1].item() == E4M3_MAX and pos_v[0].item() == 2.0 ** -9     # smallest subnormal
    lo = torch.cat([torch.zeros(1), pos_v[:-1]])
    lo_c = torch.cat([torch.zeros(1, dtype=torch.uint8), pos[:-1]])
    mid = (lo + pos_v) / 2                                                      # exact in fp32
    even = torch.where(lo_c % 2 == 0, lo_c, pos)                                # ties go to the even code
    for sign, bit in ((1.0, 0), (-1.0, 0x80)):
        assert torch.equal(e4m3_satfinite(sign * mid), even | bit)
        below = torch.nextafter(mid, torch.zeros_like(mid))
        above = torch.nextafter(mid, torch.full_like(mid, 1e9))
        assert torch.equal(e4m3_satfinite(sign * below), lo_c | bit)
        assert torch.equal(e4m3_satfinite(sign * above), pos | bit)
    # at and past the top: 448 < x (even past the 480 "next value" and infinity) saturates
    big = torch.tensor([torch.nextafter(torch.tensor(448.0), torch.tensor(1e9)).item(), 464.0, 479.0, 480.0,
                        1e6, float("inf")])
    assert (e4m3_satfinite(big) == 0x7E).all() and (e4m3_satfinite(-big) == 0xFE).all()
    # subnormals: multiples of 2^-9 below 2^-6, and half the smallest one rounds to zero (even)
    sub = torch.arange(1, 8) * 2.0 ** -9
    assert torch.equal(e4m3_satfinite(sub), torch.arange(1, 8, dtype=torch.uint8))
    assert e4m3_satfinite(torch.tensor([2.0 ** -10])).item() == 0
    assert e4m3_satfinite(torch.tensor([3 * 2.0 ** -10])).item() == 2


def test_int8_round_is_half_to_even_like_rintf():
    k = torch.arange(-140, 140, dtype=torch.float32)
    half = k + 0.5
    got = torch.round(half)
    assert torch.equal(got, torch.from_numpy(np.rint(half.numpy())))
    assert (got % 2 == 0).all()
    sc = torch.ones_like(half)
    codes = int8_code(half, sc)
    assert codes.max().item() == 127 and codes.min().item() == -127
    assert int8_code(torch.tensor([126.5, -126.5, 125.5]), torch.ones(3)).tolist() == [126.0, -126.0, 126.0]
    assert int8_code(torch.tensor([3.0, -2.0]), torch.zeros(2)).tolist() == [0.0, 0.0]


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_hy_sumsq_equals_the_lane_loop(dt):
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(37, 128, generator=g) * torch.exp2(torch.randint(-6, 7, (37, 128), generator=g).float())).to(dt)
    got = hy_sumsq(x.float())
    for row in range(x.shape[0]):
        xv = x[row].float().numpy()
        lanes = []
        for lane in range(16):
            s = np.float32(0)
            for i in range(8):
                v = np.float32(xv[8 * lane + i])
                s = np.float32(s + v * v)
            lanes.append(s)
        for o in (8, 4, 2, 1):
            lanes = [np.float32(lanes[i] + lanes[i ^ o]) for i in range(16)]
        assert len({float(v) for v in lanes}) == 1                       # every lane ends with the same value
        assert got[row].item() == float(lanes[0])


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32])
def test_wan_sumsq_equals_the_lane_loop(dt):
    g = torch.Generator().manual_seed(4)
    C = 5 * 128
    x = (torch.randn(9, C, generator=g) * 3).to(dt).float()
    got = wan_sumsq(x)
    for row in range(x.shape[0]):
        xv = x[row].double().numpy()
        lanes = []
        for lane in range(32):
            s = 0.0
            for c in range(2 * lane, C, 64):
                for t in range(2):
                    s = float(np.float32(s + xv[c + t] * xv[c + t]))    # fmaf: exact product, one rounding
            lanes.append(np.float32(s))
        for o in (16, 8, 4, 2, 1):
            lanes = [np.float32(lanes[i] + lanes[i ^ o]) for i in range(32)]
        assert got[row].item() == float(lanes[0])


def test_hy_rows_restatement_on_a_hand_case():
    """One row through the chain by hand: constant row -> 1 after the norm, weight 2 -> 2, a quarter turn."""
    x = torch.full((1, 128), 3.0).bfloat16()
    w = torch.full((128,), 2.0).bfloat16()
    c, s = torch.zeros(1, 128), torch.ones(1, 128)
    out = hy_rows(x, w, (c, s), 1e-6, kernel_order=True).float()
    assert torch.equal(out[0, 0::2], torch.full((64,), -2.0)) and torch.equal(out[0, 1::2], torch.full((64,), 2.0))
    assert torch.equal(hy_rows(x, None, None, 1e-6, True).float(), torch.ones(1, 128))


def test_bulk_split_and_slots():
    # HunyuanVideo 720p on 132 SMs, and the grids the GPU tests force for P = 2, 4, 8
    assert bulk_split(902, 132) == (6, 110, 1)
    assert bulk_split(902, 170)[2] == 2 and bulk_split(902, 110)[2] == 4 and bulk_split(902, 100)[2] == 8
    S = 3 * 128 + 45                                              # ragged last block
    slot, split, P = pool_slots(2, S, 3)                          # 8 blocks on 3 CTAs: 2 each + 2 left over
    assert P == 1 and not split.any()
    slot, split, P = pool_slots(1, S, 8)                          # 4 blocks left over, P = 2
    assert P == 2 and split.all()
    # parts of 64 tokens: the first part's groups 0/1 alternate from the CTA's first token
    assert slot[0, :4].tolist() == [0, 1, 0, 1] and slot[0, 64:68].tolist() == [2, 3, 2, 3]
    # a CTA that took an odd number of tokens before an item starts that item on group 1
    slot, split, P = pool_slots(2, S, 1)                          # one CTA walks both samples
    assert P == 1 and slot[4, 0].item() == 1 and slot[3, 44].item() == 0   # 3*128+45 tokens precede block 4


def _sensitive_pooled_rows(B, S, H, g):
    """Post-norm rows whose block sums depend on the fp32 order (see order_sensitive_rows)."""
    p = torch.arange(S) % 128
    big = ((p % 4 == 0) | (p % 4 == 3))[None, :, None, None]
    sign = torch.where(p % 64 < 32, 1.0, -1.0)[None, :, None, None]
    tiny = torch.randn(B, S, H, 128, generator=g) * 2.0 ** -16
    return torch.where(big, sign.expand(B, S, H, 128), tiny).bfloat16()


@pytest.mark.parametrize("classic,ctas", [(True, None), (False, 3), (False, 30), (False, 40), (False, 64)])
def test_pooled_means_within_the_summation_bound(classic, ctas):
    """The restated kernel-order block means are within the derived bound of the fp64 means, on random
    bf16 values spread over 2^-12 .. 2^12 and on order-sensitive rows; on the latter the fp32 order
    really shows (not the correctly rounded mean) and a reversed part order gives other bits."""
    g = torch.Generator().manual_seed(11)
    B, S, H = 2, 3 * 128 + 45, 2
    slot, split, P = pool_slots(B, S, ctas)
    assert P == {None: 1, 3: 1, 30: 2, 40: 4, 64: 8}[ctas]
    nb = (S + 127) // 128
    spread = (torch.randn(B, S, H, 128, generator=g) *
              torch.exp2(torch.randint(-12, 13, (B, S, H, 128), generator=g).float())).bfloat16()
    for y in (spread, _sensitive_pooled_rows(B, S, H, g)):
        got = pooled_means(y, slot, split, P)
        yp = torch.zeros(B, nb * 128, H, 128, dtype=torch.float64)
        yp[:, :S] = y.double()
        exact = yp.view(B, nb, 128, H, 128).mean(2).permute(0, 2, 1, 3)
        abs_sum = yp.abs().view(B, nb, 128, H, 128).sum(2).permute(0, 2, 1, 3)
        sp = split.view(B, nb)[:, None, :, None]
        E = torch.where(sp, pool_bound(abs_sum, pool_depth(P, True, classic)),
                        pool_bound(abs_sum, pool_depth(P, False, classic)))
        assert within_rounding(got, exact, E).all()
    assert not torch.equal(got.double(), exact.to(torch.bfloat16).double())
    if P >= 4:
        perm = torch.flip(torch.arange(P), [0])
        slot2 = torch.where(split[:, None], 2 * perm[slot // 2] + slot % 2, slot)
        assert not torch.equal(pooled_means(y, slot2, split, P), got)


def test_int8_mean_and_shift_bounds():
    g = torch.Generator().manual_seed(12)
    B, S, H = 2, 5 * 128 + 77, 3
    x = (torch.randn(B, S, H, 128, generator=g) * 40 + 9).bfloat16()
    got = colsum_mean(x)
    x64 = x.double()
    exact = x64.sum(1).reshape(B * H, 128) / S
    abs_cs = x64.abs().sum(1).reshape(B * H, 128)
    assert ((got.double() - exact).abs() <= mean_bound(abs_cs, exact, S)).all()
    assert not torch.equal(got.double(), exact.float().double())     # the fp32 order shows
    # shift: lane l's 8 channels 8l..8l+7 in an fma chain, a 4-level tree, then * sc
    code = torch.randint(-127, 128, (50, 128), generator=g).float()
    km = torch.randn(128, generator=g) * 7
    sc = torch.rand(50, generator=g) * 0.1 + 1e-3
    ck, kk = code.view(50, 16, 8).double(), km.view(16, 8).double()
    lanes = torch.zeros(50, 16)
    for i in range(8):
        lanes = (lanes.double() + ck[..., i] * kk[:, i]).float()
    for half in (8, 4, 2, 1):
        lanes = lanes[:, :half] + lanes[:, half:2 * half]
    shift = lanes[:, 0] * sc
    prod = code.double() * km.double()
    exact = sc.double() * prod.sum(-1)
    assert ((shift.double() - exact).abs() <= shift_bound(sc.double(), prod.abs().sum(-1), exact)).all()
