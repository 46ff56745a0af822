"""The kernels that produce every operand of carved attention, against exact restatements at the shapes
that ship (tests/test_producers_cpu.py holds the restatements and checks them without a GPU):

  HunyuanVideo prologue (bulk and classic)  q, k: <= 1 ulp and >= 99.5 % bit-identical to the reference
                                            chain (torch's mean(x^2)); bit-identical with mean(x^2) in the
                                            kernel's order; v exact; pooled means bit-identical to the
                                            kernel's fp32 order over its own rows, and within the summation
                                            bound of their fp64 means
  Wan prologue                              pairwise bound (err <= 2^-5 |pair|), >= 99.5 % bit-identical;
                                            the norm-only form bit-identical in the kernel's order
  INT8 Q / K quantiser                      codes and scales bit-identical from the kernel's own mean; the
                                            mean and the LSE shift within their fp32 bounds of fp64
  FP8 V quantiser                           amax exact, codes bit-identical

Every case prints its max ulp and bit-identical fraction.  The inputs are generated on the GPU and the
restatements run there in fp32, chunked over tokens; fp64 is used for the means, pools and shifts only.
"""
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
from test_producers_cpu import (e4m3_satfinite, hy_rows, int8_code, mean_bound,  # noqa: E402
                                order_sensitive_rows, pool_bound, pool_depth, pool_slots, pooled_means,
                                shift_bound, ulp16, wan_sumsq, within_rounding)
from test_prologue_bulk_gpu import _run  # noqa: E402

DEV = "cuda"
EPS = 1e-6
CHUNK = 16384


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _same(a, b):
    return a.view(torch.int16) == b.view(torch.int16)


# ====================================================================== HunyuanVideo prologue
# id: B, L, T, H, dtype, weights, rope ("hilbert" grid | "perm" | None), mode, ctas (0: one per SM),
#     extra channels per token (the single-stream linear1 split), order-sensitive q/k rows
HY = {
    "hy720p-bulk": (1, 115200, 256, 24, torch.bfloat16, True, (32, 45, 80), "bulk", 0, 0, False),
    "hy720p-classic": (1, 115200, 256, 24, torch.bfloat16, True, (32, 45, 80), "classic", 0, 0, False),
    "hy_i2v-bulk": (1, 115200, 400, 24, torch.bfloat16, True, (32, 45, 80), "bulk", 0, 0, False),
    "turbo_s0-B3": (3, 63360, 256, 24, torch.bfloat16, True, (32, 33, 60), "bulk", 0, 0, False),
    "hy_i2v-B2-P2": (2, 115200, 400, 24, torch.bfloat16, True, (32, 45, 80), "bulk", 110, 0, False),
    "hy720p-P2-sensitive": (1, 115200, 256, 24, torch.bfloat16, True, (32, 45, 80), "bulk", 170, 0, True),
    "hy720p-P4-sensitive": (1, 115200, 256, 24, torch.bfloat16, True, (32, 45, 80), "bulk", 110, 0, True),
    "hy720p-P8-sensitive": (1, 115200, 256, 24, torch.bfloat16, True, (32, 45, 80), "bulk", 100, 0, True),
    # split left-over blocks = the image/text block, a whole text block and the ragged last one
    "straddle-P8-sensitive": (2, 300 * 128 + 45, 256, 24, torch.bfloat16, True, "perm", "bulk", 200, 0, True),
    "straddle-classic-sensitive": (2, 300 * 128 + 45, 256, 24, torch.bfloat16, True, "perm", "classic", 0, 0, True),
    "ulysses-h3": (1, 115200, 256, 3, torch.bfloat16, True, (32, 45, 80), "bulk", 0, 0, False),
    "ulysses-h5": (1, 115200, 256, 5, torch.bfloat16, True, (32, 45, 80), "bulk", 0, 0, False),
    "ulysses-h6": (1, 115200, 256, 6, torch.bfloat16, True, (32, 45, 80), "bulk", 0, 0, False),
    "ulysses-h12": (1, 115200, 256, 12, torch.bfloat16, True, (32, 45, 80), "bulk", 0, 0, False),
    "fp16-noweights-notext": (1, 63360, 0, 24, torch.float16, False, (32, 33, 60), "bulk", 0, 0, False),
    "fp16-noweights-notext-classic": (1, 63360, 0, 24, torch.float16, False, (32, 33, 60), "classic", 0, 0, False),
    "linear1-split": (1, 63360, 256, 24, torch.bfloat16, True, (32, 33, 60), "bulk", 0, 4 * 3072, False),
    "h26-fallback": (1, 63360, 256, 26, torch.bfloat16, True, (32, 33, 60), "bulk", 0, 0, False),
    "h40-fallback": (1, 20000, 256, 40, torch.bfloat16, True, "perm", "bulk", 0, 0, False),
}


def _hy_inputs(B, L, T, H, dt, has_w, rope, extra, sensitive, g):
    width = 3 * H * 128 + extra

    def rows(n, tok0):
        x = torch.randn(B, n, width, generator=g, device=DEV, dtype=dt) * 1.5
        if sensitive:
            x[..., :2 * H * 128] = order_sensitive_rows(B, n, tok0, 2 * H, g, DEV).view(B, n, -1).to(dt)
        return x[..., :3 * H * 128]

    img = rows(L, 0)
    txt = rows(T, L) if T else None
    ws = [(1 + 0.2 * torch.randn(128, generator=g, device=DEV)).to(dt) for _ in range(4)] if has_w else [None] * 4
    fc = index = None
    if rope is not None:
        # one angle per channel pair, as in HunyuanVideo's tables; order-sensitive rows cancel across
        # tokens only if every token turns by the same angles
        ang = torch.rand(1 if sensitive else L, 64, generator=g, device=DEV).expand(L, 64) * 6.2832
        ang = ang.repeat_interleave(2, dim=1)
        fc = (torch.cos(ang), torch.sin(ang))
        if rope == "perm":
            index = torch.randperm(L, generator=g, device=DEV)
        else:
            from jenga_b200 import gilbert
            index = gilbert.mapping_tensors(*rope)[1].to(DEV)
    return img, txt, ws, fc, index


def _hy_row_stats(img, txt, ws, fc, index, H, q, k, v):
    """q and k against the reference chain: (max ulp of the rows without RoPE, max ulp and max err / |pair|
    of the rotated rows, bit-identical fraction); mismatches against the kernel order; v exact."""
    B, L = img.shape[:2]
    ulp_plain = ulp_rot = pair_rot = 0.0
    same, total, bad2, v_ok = 0, 0, 0, True
    for src, t0, w_q, w_k, rot in ((img, 0, ws[0], ws[1], fc is not None), (txt, L, ws[2], ws[3], False)):
        if src is None:
            continue
        for b in range(B):
            for s0 in range(0, src.shape[1], CHUNK):
                s1 = min(src.shape[1], s0 + CHUNK)
                x = src[b, s0:s1].view(s1 - s0, 3, H, 128)
                cs = None
                if rot:
                    rows = index[s0:s1] if index is not None else slice(s0, s1)
                    cs = (fc[0][rows][:, None], fc[1][rows][:, None])
                for which, out, w in ((0, q, w_q), (1, k, w_k)):
                    got = out[b, t0 + s0:t0 + s1]
                    ref1 = hy_rows(x[:, which], w, cs, EPS, kernel_order=False)
                    ref2 = hy_rows(x[:, which], w, cs, EPS, kernel_order=True)
                    err = (got.double() - ref1.double()).abs()
                    ulps = (err / ulp16(ref1, ref1.dtype)).max().item()
                    if rot:
                        pair = ref1.double().view(*ref1.shape[:-1], 64, 2).norm(dim=-1, keepdim=True)
                        ratio = (err.view(pair.shape[:-1] + (2,)) / pair.clamp_min(1e-30)).max().item()
                        ulp_rot, pair_rot = max(ulp_rot, ulps), max(pair_rot, ratio)
                    else:
                        ulp_plain = max(ulp_plain, ulps)
                    same += int(_same(got, ref1).sum())
                    total += got.numel()
                    bad2 += int((~_same(got, ref2)).sum())
                v_ok &= bool(_same(v[b, t0 + s0:t0 + s1], x[:, 2]).all())
    return ulp_plain, ulp_rot, pair_rot, same / total, bad2, v_ok


def _hy_pool_stats(y, pool, classic, ctas):
    """(mismatches vs the kernel-order restatement, elements outside the fp64 bound, P)."""
    B, S, H, _ = y.shape
    slot, split, P = pool_slots(B, S, None if classic else min(ctas or _sms(), 256))
    bad_exact = int((~_same(pool, pooled_means(y, slot, split, P))).sum())
    nb = (S + 127) // 128
    yp = torch.zeros(B, nb * 128, H, 128, dtype=torch.float64, device=DEV)
    yp[:, :S] = y.double()
    exact = yp.view(B, nb, 128, H, 128).mean(2).permute(0, 2, 1, 3)
    abs_sum = yp.abs_().view(B, nb, 128, H, 128).sum(2).permute(0, 2, 1, 3)
    sp = split.to(DEV).view(B, 1, nb, 1)
    E = torch.where(sp, pool_bound(abs_sum, pool_depth(P, True, classic)),
                    pool_bound(abs_sum, pool_depth(P, False, classic)))
    return bad_exact, int((~within_rounding(pool, exact, E)).sum()), P


@pytest.mark.parametrize("case", list(HY))
def test_hy_prologue_against_restatements(case):
    """Against the reference chain (mean(x^2) by torch's reduction) >= 99.5 % of the elements are
    bit-identical (measured on an H100: 99.9997 %, fp16 99.997 %), but the old "<= 1 ulp" holds only
    where nothing amplifies the one-ulp step of the normalised value n that another summation order of
    mean(x^2) can cause:
      - the weight: n w moves by ulp(n) |w|, up to 2 ulp of the product (measured: 2 ulp on a text row
        at 3 heads), so weighted rows without RoPE are held to 2 ulp, unweighted ones to 1;
      - the rotation: the step of the pair can land in a component much smaller than the pair (measured
        up to ~13000 ulp of the component), so rotated elements get the pairwise bound of the Wan test,
        err <= 2^-5 |pair| (measured <= 1.4e-2 |pair|).
    With mean(x^2) in the kernel's order q and k are bit-identical everywhere (torch.rsqrt and the
    kernel's rsqrtf round alike on the H100), and the pooled means are bit-identical to the kernel's fp32
    order over its own rows."""
    from jenga_b200.hyvideo import attention_prologue
    B, L, T, H, dt, has_w, rope, mode, ctas, extra, sensitive = HY[case]
    g = torch.Generator(device=DEV).manual_seed(2024 + L + H + B)
    img, txt, ws, fc, index = _hy_inputs(B, L, T, H, dt, has_w, rope, extra, sensitive, g)
    call = lambda i, t: attention_prologue(i, t, H, *ws, EPS, fc, rope_index=index)  # noqa: E731
    q, k, v, (qp, kp) = _run(mode, ctas, lambda: call(img, txt))
    classic = mode == "classic" or H > 24                        # more than 24 heads: the bulk form declines
    ulp_plain, ulp_rot, pair_rot, frac, bad2, v_ok = _hy_row_stats(img, txt, ws, fc, index, H, q, k, v)
    pools = [_hy_pool_stats(y, p, classic, ctas) for y, p in ((q, qp), (k, kp))]
    print(f"\n[hy prologue {case}] q,k vs reference chain: {frac:.5%} bit-identical, max {ulp_plain:.0f} ulp "
          f"without RoPE, rotated max {ulp_rot:.0f} ulp / {pair_rot:.2e} |pair|; vs kernel order: {bad2} differ; "
          f"pools (kernel order / fp64 bound) q {pools[0][:2]} k {pools[1][:2]}, P={pools[0][2]}")
    assert v_ok
    assert ulp_plain <= (2.0 if has_w else 1.0) and pair_rot <= 2.0 ** -5 and frac >= 0.995
    assert bad2 == 0
    for bad_exact, bad_bound, _ in pools:
        assert bad_exact == 0 and bad_bound == 0
    if B > 1:   # distinct samples: each equals its own batch-1 call and that call's pooled restatement
        for b in range(B):
            one = _run(mode, ctas, lambda: call(img[b:b + 1], txt[b:b + 1] if txt is not None else None))
            for got, want in zip(one[:3], (q, k, v)):
                assert torch.equal(got.view(torch.int16), want[b:b + 1].view(torch.int16)), b
            for y, p in zip(one[:2], one[3]):
                assert _hy_pool_stats(y, p, classic, ctas)[:2] == (0, 0), b
        assert not torch.equal(q[0].view(torch.int16), q[1].view(torch.int16))


# ====================================================================== Wan prologue
def _wan_rows(x, w, H, grid, fr, remap, kernel_order):
    """The Wan prologue restated for x [B, L, C]: r = rsqrt(mean(x^2) + eps) (torch's reduction, or the
    kernel's order with an IEEE division by C), n = x r (rounded to bf16 for bf16 x), n w (rounded for bf16
    x and w), the complex rotation in fp64 for tokens on the grid, then fp32 -> bf16.  [B, L, H, 128]."""
    B, L, Cc = x.shape
    out = torch.empty(B, L, H, 128, dtype=torch.bfloat16, device=DEV)
    n_grid = grid[0] * grid[1] * grid[2] if fr is not None else 0
    for b in range(B):
        for s0 in range(0, L, CHUNK):
            s1 = min(L, s0 + CHUNK)
            xs = x[b, s0:s1]
            xf = xs.float()
            if kernel_order:
                ss = wan_sumsq(xs)
                r = torch.rsqrt(ss / torch.full_like(ss, float(Cc)) + EPS)
            else:
                r = torch.rsqrt(xf.pow(2).mean(-1) + EPS)
            y = xf * r[:, None]
            if x.dtype == torch.bfloat16:
                y = y.bfloat16().float()
            if w is not None:
                y = y * w.float()
                if x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16:
                    y = y.bfloat16().float()
            y = y.view(-1, H, 128)
            o = y.bfloat16()
            e = min(s1, n_grid)
            if e > s0:
                tok = torch.arange(s0, e, device=DEV)
                pos = remap[tok] if remap is not None else tok
                fi, rem = pos // (grid[1] * grid[2]), pos % (grid[1] * grid[2])
                hi, wi = rem // grid[2], rem % grid[2]
                j = torch.arange(64, device=DEV)
                row = torch.where(j < 22, fi[:, None], torch.where(j < 43, hi[:, None], wi[:, None]))
                f = fr[row, j]                                           # [n, 64, 2]
                a = y[:e - s0].double().view(-1, H, 64, 2)
                re, im = f[:, None, :, 0], f[:, None, :, 1]
                o0 = a[..., 0] * re - a[..., 1] * im
                o1 = a[..., 0] * im + a[..., 1] * re
                o[:e - s0] = torch.stack([o0, o1], -1).float().bfloat16().view(-1, H, 128)
            out[b, s0:s1] = o
    return out


# id: B, grid, heads, x dtype, w dtype (None: no weight), tokens past the grid, strided x, rotate
F32, BF16 = torch.float32, torch.bfloat16
WAN = {
    "wan14b-720p": (1, (21, 45, 80), 40, BF16, BF16, 0, False, True),
    "wan1.3b-480p-bf16-bf16": (1, (21, 30, 52), 12, BF16, BF16, 0, False, True),
    "wan1.3b-480p-bf16-f32": (1, (21, 30, 52), 12, BF16, F32, 0, False, True),
    "wan1.3b-480p-f32-bf16": (1, (21, 30, 52), 12, F32, BF16, 0, False, True),
    "wan1.3b-480p-f32-f32": (1, (21, 30, 52), 12, F32, F32, 0, False, True),
    "wan1.3b-480p-no-weight": (1, (21, 30, 52), 12, BF16, None, 0, False, True),
    "wan1.3b-B3-strided-padded": (3, (21, 30, 52), 12, BF16, BF16, 72, True, True),
    "wan1.3b-B2-f32-strided-padded": (2, (21, 30, 52), 12, F32, BF16, 40, True, True),
    "cross-512-text-rows": (2, (512, 1, 1), 40, BF16, BF16, 0, False, False),
    "cross-257-clip-rows": (2, (257, 1, 1), 40, BF16, F32, 0, True, False),
    "cross-512-f32": (1, (512, 1, 1), 40, F32, F32, 0, False, False),
}


@pytest.mark.parametrize("case", list(WAN))
def test_wan_prologue_against_restatements(case):
    from jenga_b200 import gilbert, wan
    B, grid, H, xd, wd, pad, strided, rotate = WAN[case]
    Cc = H * 128
    L = grid[0] * grid[1] * grid[2] + pad
    g = torch.Generator(device=DEV).manual_seed(77 + L + H)
    if strided:   # batch and token strides both larger than the row
        x = (torch.randn(B, L + 5, Cc + 64, generator=g, device=DEV) * 1.3).to(xd)[:, :L, :Cc]
    else:
        x = (torch.randn(B, L, Cc, generator=g, device=DEV) * 1.3).to(xd)
    w = (1 + 0.2 * torch.randn(Cc, generator=g, device=DEV)).to(wd) if wd is not None else None
    freqs = wan.rope_freqs(128) if rotate else None
    remap = gilbert.mapping_tensors(*grid, sliced=True)[1].to(DEV) if rotate else None
    got = wan.norm_rope(x, w, H, grid, freqs, remap, eps=EPS)
    fr = torch.view_as_real(freqs).to(DEV) if rotate else None
    ref1 = _wan_rows(x, w, H, grid, fr, remap, kernel_order=False)
    ref2 = _wan_rows(x, w, H, grid, fr, remap, kernel_order=True)
    frac1 = _same(got, ref1).float().mean().item()
    frac2 = _same(got, ref2).float().mean().item()
    pair = ref1.float().view(B, L, H, 64, 2).norm(dim=-1, keepdim=True)
    err = (got.float() - ref1.float()).view(B, L, H, 64, 2).abs()
    ratio = (err / pair.clamp_min(1e-30)).max().item()
    worst = ((got.double() - ref1.double()).abs() / ulp16(ref1, ref1.dtype)).max().item()
    print(f"\n[wan prologue {case}] vs torch chain: {frac1:.5%} bit-identical, max {worst:.0f} ulp, "
          f"max err/|pair| {ratio:.2e}; vs kernel order: {frac2:.5%} bit-identical")
    assert frac1 >= 0.995
    assert (err <= 2.0 ** -5 * pair).all()
    if not rotate:   # no fp64 rotation (where nvcc may contract into an FMA): the kernel order is exact
        assert frac2 == 1.0
    if B > 1:
        assert not torch.equal(got[0].view(torch.int16), got[1].view(torch.int16))


# ====================================================================== INT8 Q / K quantiser
# id: B, S, H, dtype, layout ("contig" | "packed": a view of [B, S, 3, H, 128]), special inputs
INT8 = {
    "hy720p": (1, 115456, 24, BF16, "contig", None),
    "wan14b": (1, 75600, 40, BF16, "contig", None),                     # S % 128 = 80
    "hy_i2v-B2-packed": (2, 115600, 24, BF16, "packed", None),          # S % 128 = 16: a whole padding group
    "B3-packed-fp16": (3, 1000, 5, torch.float16, "packed", None),      # S % 128 = 104
    "short": (2, 37, 3, BF16, "contig", None),
    "zero-and-constant-groups": (2, 1024, 3, BF16, "contig", "flat"),
    "fp16-large": (2, 3000, 4, torch.float16, "packed", "large"),
}


def _int8_inputs(B, S, H, dt, layout, special, g):
    n = 3 if layout == "packed" else 2
    base = torch.randn(B, S, n, H, 128, generator=g, device=DEV)
    base[:, :, 1] += torch.randn(H, 128, generator=g, device=DEV) * 3         # a channel bias on K
    if special == "large":
        base = (base * 2e4).clamp(-65000, 65000)
    if special == "flat":
        base[:, 64:128, 0] = 0                          # Q: a 64-row group of zeros (sc == 0)
        base[0, :, 1, 1] = 0.75                         # K: a head of one value, equal to its mean
    x = base.to(dt)
    return x[:, :, 0], x[:, :, 1]


def _int8_restated(x, G, mean):
    B, S, H, D = x.shape
    Sp = (S + 127) // 128 * 128
    xf = torch.zeros(B, Sp, H, D, dtype=torch.float32, device=DEV)
    xf[:, :S] = x.float()
    if mean is not None:
        xf = xf - mean.view(B, 1, H, D)
    yg = xf.permute(0, 2, 1, 3).reshape(B * H, Sp // G, G * D)
    amax = yg.abs().amax(-1)
    sc = amax / torch.full_like(amax, 127.0)
    codes = int8_code(yg, sc[..., None]).to(torch.int8).view(B, H, Sp, D).permute(0, 2, 1, 3)
    return codes, sc


def _int8_check(tag, x, G, smooth, q8, scale, mean):
    B, S, H, D = x.shape
    msg = f"[int8 {tag} G={G} smooth={smooth}]"
    if smooth:
        x64 = x.double()
        exact = x64.sum(1).reshape(B * H, D) / S
        mbad = int(((mean.double() - exact).abs() > mean_bound(x64.abs().sum(1).reshape(B * H, D), exact, S)).sum())
        m_err = ((mean.double() - exact).abs() / exact.abs().clamp_min(1e-30)).max().item()
        msg += f" mean: max rel err {m_err:.1e}, {mbad} outside the bound;"
    codes, sc = _int8_restated(x, G, mean)
    cbad = int((q8 != codes).sum())
    sbad = int((scale != sc).sum())
    print(f"\n{msg} codes {cbad} differ, scales {sbad} differ, {int((sc == 0).sum())} groups with sc == 0")
    if smooth:
        assert mbad == 0
    assert cbad == 0 and sbad == 0
    return sc


@pytest.mark.parametrize("case", list(INT8))
def test_int8_quantiser_against_restatement(case):
    from jenga_b200.attention import quantize_int8, quantize_qk_int8
    B, S, H, dt, layout, special = INT8[case]
    g = torch.Generator(device=DEV).manual_seed(300 + S + H)
    q, k = _int8_inputs(B, S, H, dt, layout, special, g)
    q8, qs, qm = quantize_int8(q, 64, False)
    _int8_check(case + " Q", q, 64, False, q8, qs, None)
    k8, ks, km = quantize_int8(k, 128, True)
    _int8_check(case + " K", k, 128, True, k8, ks, km)
    k8b, ksb, kmb = quantize_int8(k, 64, True)                      # group 64 on a smoothed input
    assert torch.equal(kmb, km)
    _int8_check(case + " K", k, 64, True, k8b, ksb, kmb)
    if special == "flat":
        assert (qs[:, 1] == 0).all() and (q8[:, 64:128] == 0).all()
        assert (ks[1] == 0).all() and (k8[0, :, 1] == 0).all()      # sc == 0: code 0, scale 0
    # the LSE shift: Q' . mean(K) per row, against fp64 sc * sum(code * kmean)
    q8s, qss, k8s, kss, shift = quantize_qk_int8(q, k, lse_shift=True)
    assert torch.equal(q8s, q8) and torch.equal(qss, qs) and torch.equal(k8s, k8) and torch.equal(kss, ks)
    Sp = q8.shape[1]
    codes = q8.double().permute(0, 2, 1, 3).reshape(B * H, Sp, 128)
    dot = torch.bmm(codes, km.double()[..., None])[..., 0]
    adot = torch.bmm(codes.abs(), km.double().abs()[..., None])[..., 0]
    sc_row = qs.double().repeat_interleave(64, -1)
    exact = sc_row * dot
    bad = int(((shift.double() - exact).abs() > shift_bound(sc_row, adot, exact)).sum())
    rel = ((shift.double() - exact).abs() / exact.abs().clamp_min(1e-30)).max().item()
    print(f"[int8 {case} shift] max rel err {rel:.1e}, {bad} outside the bound")
    assert bad == 0


# ====================================================================== FP8 V quantiser
# id: B, S, H, dtype, layout ("contig" | "packed" | "headmajor": a view of [B, H, S, 128])
FP8 = {
    "hy720p": (1, 115456, 24, BF16, "contig"),
    "wan14b-packed": (1, 75600, 40, BF16, "packed"),
    "span-B2-packed": (2, 4096, 8, BF16, "packed"),
    "span-B3-headmajor-fp16": (3, 3000, 6, torch.float16, "headmajor"),
}


def _fp8_input(B, S, H, dt, layout, g):
    """Heads scaled 1e-3 .. 1e3 with elements spread over 2^-18 .. 1 of the head (the small ones land in
    e4m3 subnormals), head 1 all zeros."""
    shape = {"contig": (B, S, H, 128), "packed": (B, S, 3, H, 128), "headmajor": (B, H, S, 128)}[layout]
    view = {"contig": lambda t: t, "packed": lambda t: t[:, :, 2], "headmajor": lambda t: t.permute(0, 2, 1, 3)}[layout]
    x = torch.randn(shape, generator=g, device=DEV) * torch.exp2(-18 * torch.rand(shape, generator=g, device=DEV))
    v = view(x)
    v.mul_(torch.logspace(-3, 3, H, device=DEV).view(1, 1, H, 1))
    v[:, :, 1] = 0
    return view(x.to(dt))


def _fp8_restated(v):
    B, S, H, D = v.shape
    amax = v.float().abs().amax(dim=(1, 3)).reshape(B * H)
    inv = torch.where(amax > 0, torch.full_like(amax, 448.0) / amax, torch.ones_like(amax))
    return e4m3_satfinite(v.float() * inv.view(B, 1, H, 1)), amax


@pytest.mark.parametrize("case", list(FP8))
def test_fp8_v_quantiser_against_restatement(case):
    from jenga_b200 import _lib
    from jenga_b200.attention import _dtype_code, _stream_ptr
    B, S, H, dt, layout = FP8[case]
    g = torch.Generator(device=DEV).manual_seed(500 + S + H)
    v = _fp8_input(B, S, H, dt, layout, g)
    assert not v.is_contiguous() or layout == "contig"
    n = B * S * H * 128
    out = torch.full((n + 4096,), 0x7F, dtype=torch.uint8, device=DEV)        # NaN canaries after the output
    amax = torch.full((B * H + 16,), float("nan"), device=DEV)
    _lib.check(_lib.lib.jenga_quantize_v_fp8(v.data_ptr(), _dtype_code(v), B, S, H, v.stride(0), v.stride(1),
                                             v.stride(2), out.data_ptr(), amax.data_ptr(), _stream_ptr(v.device)),
               "quantize_v_fp8")
    want, want_amax = _fp8_restated(v)
    got = out[:n].view(B, S, H, 128)
    bad = int((got != want).sum())
    sub = int((((want & 0x78) == 0) & ((want & 0x07) != 0)).sum())
    print(f"\n[fp8 v {case}] {bad} codes differ; {sub} subnormal codes, amax of {B * H} heads "
          f"{'exact' if torch.equal(amax[:B * H], want_amax) else 'DIFFERENT'}")
    assert torch.equal(amax[:B * H], want_amax)
    assert (want_amax.view(B, H)[:, 1] == 0).all() and (got[:, :, 1] == 0).all()
    assert sub > 0
    assert bad == 0
    assert (out[n:] == 0x7F).all() and torch.isnan(amax[B * H:]).all()
    # the wrapper returns the same bytes in a contiguous [B, S, H, 128] tensor
    from jenga_b200.attention import quantize_v_fp8
    v8, a2 = quantize_v_fp8(v)
    assert v8.is_contiguous() and v8.shape == (B, S, H, 128) and torch.equal(v8, got) and torch.equal(a2, want_amax)
