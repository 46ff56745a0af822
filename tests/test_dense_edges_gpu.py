"""Edge cases of the fused LayerNorm / modulate / gate / GELU kernels (csrc/dense_fused.cu) against
plain fp64 references, at the row counts, channel widths, layouts and values where such kernels go
wrong.

References.  Each keeps exactly the rounding points of the definition (dense_fused.cu's header,
dense.py's docstrings) and computes everything else in fp64:
* HunyuanVideo ln_modulate[_tr]: n = (x - mu) / sqrt(var + eps), mu and the biased var in fp64;
  t1 = bf16(fp32(1 + scale)); v = n * t1 + shift; the output is bf16(v).  Token-replace rows take
  tr_scale / tr_shift.
* Wan wan_ln_modulate / wan_residual_ln: r = fp32(x + fp32(y * gate)) (or fp32(x + y)), checked bit
  for bit against the torch fp32 ops, then the LayerNorm of x or r in fp64.  With a bf16 x and no
  residual n is rounded to bf16 first (WanLayerNorm's `.type_as(x)`).  The epilogue is
  n * fp32(1 + scale) + shift, or w * n + b in the affine form.
* gate_residual[_tr] and wan_gate_residual: the torch expressions are exact references (bf16 ops for
  HunyuanVideo, fp32 ops for Wan): bit equality.
* ln_modulate[_tr]_fp8: bit-identical to quantize_rows_fp8(ln_modulate(...)).
* gelu_tanh: fp64 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))), and bit identity with ATen's
  F.gelu(approximate="tanh"), which the kernel restates operation by operation.

Error bound of the LayerNorm forms.  The kernel reduces a row in fp32: each thread adds at most
8 * kVec <= 48 elements in sequence, then come 5 shuffle levels and the sum of 4 warp partials, so no
element passes through more than 56 < 64 roundings and
    |d mu| <= 64 * 2^-24 * mean|x| = 2^-18 * mean|x|.
The variance is reduced the same way from the exact differences x - mu' (its relative error is at most
2^-18 plus the second-order d mu^2 / var); rsqrtf adds about 2^-22, and n = rstd * (x - mu') two more
roundings.  Hence, per element,
    dn = 2^-17 |n| + 2^-18 mean_row|x| / sqrt(var + eps),
and the fp32 epilogue (one mul and one add, or one fma) adds at most 2^-22 (|n t1| + |shift|):
    E = |t1| dn + 2^-22 (|n t1| + |shift|)        (affine: |w| dn + 2^-22 (|w n| + |b|)).
Every element must satisfy |got - v| <= 2^-8 (|v| + E) + E, where 2^-8 (|v| + E) is the final bf16
rounding.  With a bf16 x and no residual, n is rounded to bf16: v uses bf16(n) and, where n +- dn
straddles a bf16 rounding point, E includes the distance between the two candidates times |t1|.
A bound that ignored the reduction order (C * 2^-24 per term) would let a one-pass variance,
E[x^2] - mu^2, pass at the fp32 offset-300 rows; this one does not.  On the Gaussian and outlier
inputs at least 99.9 % of the outputs must also be bit-identical to bf16(v).

Grid coverage.  The LayerNorm kernels launch min(ceil(rows / 2), 132 * 32) CTAs of two rows, so rows
above 8448 run the loop body (the prefetch of the next row pair and the parity-indexed reductions)
more than once; gate_residual and gelu_tanh launch 132 * 16 = 2112 CTAs of one row, wan_gate_residual
min(rows, 2112).  kVec = ceil(C / 1024) takes every value from 1 to 6 over CHANNELS, with partly filled
last vector slots.  Every LayerNorm case above 8448 rows is launched twice and must repeat bit for bit.

GELU is checked on all 65 536 bf16 inputs.  Inputs are read from rows inside wider NaN-filled buffers,
and outputs written with a row stride wider than the row must leave the padding, and the row after the
last one, as they were.
"""
import math
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

EPS = float(torch.tensor(1e-6, dtype=torch.float32))   # the fp32 eps the kernels receive
CHUNK = 8192                                            # rows per fp64 reference chunk
LN_ROWS = [1, 2, 3, 8447, 8448, 8449, 16897]
CTA_ROWS = [2111, 2112, 2113, 4225]
CHANNELS = [8, 16, 1016, 1024, 1032, 3072, 4088, 4096, 5120, 6136, 6144]
VALUES = ["gauss", "offset", "outliers", "zero_rows", "constant_rows", "tiny"]
PADS = [0, 8, 64]               # 0: contiguous rows; else rows 8 elements into a buffer C + pad wide
IDENTICAL = ("gauss", "outliers")


def _cases(shift, rows=LN_ROWS):
    """one case per channel width; rows, values and layouts rotate so each appears, `shift` varying
    the combinations from one test to the next"""
    return [(rows[(i + shift) % len(rows)], C, VALUES[(i + shift) % len(VALUES)], PADS[(i + shift) % len(PADS)])
            for i, C in enumerate(CHANNELS)]


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _zero_rows(rows):
    """Wan zero-pads the sequence: the tail, plus every fifth row mixed among live ones"""
    r = torch.arange(rows, device="cuda")
    return (r % 5 == 3) | (r >= rows - max(1, rows // 4))


def _values(kind, rows, C, dtype, g):
    """[rows, C] input of one value case, in `dtype`"""
    f32 = dtype == torch.float32
    x = torch.randn(rows, C, generator=g, device="cuda")
    if kind == "gauss":
        x = 1.7 * x + 0.3
    elif kind == "offset":                  # mean >> std
        x = x + (300.0 if f32 else 16.0)
    elif kind == "outliers":                # "massive activations": 4 channels at +-2e4
        ch = torch.randperm(C, generator=g, device="cuda")[:4]
        x[:, ch] = torch.tensor([2e4, -2e4, 2e4, -2e4], device="cuda")[: ch.numel()]
    elif kind == "zero_rows":
        x = 1.7 * x + 0.3
        x[_zero_rows(rows)] = 0
    elif kind == "constant_rows":           # every even row one non-zero value
        c = 3 * torch.randn(rows, 1, generator=g, device="cuda") + (300.0 if f32 else 0.5)
        x = torch.where(torch.arange(rows, device="cuda")[:, None] % 2 == 0, c.expand(rows, C), x)
    elif kind == "tiny":                    # var ~ eps
        x = 1e-3 * x + 2e-4
    return x.to(dtype)


def _place(t, pad, fill=float("nan")):
    """t [rows, C] as rows 8 elements into a buffer C + pad wide (pad 0: t itself); the rest is NaN so
    that a read past a row shows"""
    if pad == 0:
        return t
    wide = torch.full((t.shape[0], t.shape[1] + pad), fill, dtype=t.dtype, device=t.device)
    wide[:, 8:8 + t.shape[1]] = t
    return wide[:, 8:8 + t.shape[1]]


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else
                               torch.int32 if t.element_size() == 4 else torch.uint8)


class _Tally:
    """hard-bound violations and bit-identity with bf16(v), accumulated over reference chunks"""

    def __init__(self, what):
        self.what, self.bad, self.same, self.n, self.worst = what, 0, 0, 0, 0.0

    def add(self, got, v, E):
        d = (got.double() - v).abs()
        lim = 2.0 ** -8 * (v.abs() + E) + E
        bad = ~(d <= lim)                                   # NaN fails
        self.bad += int(bad.sum())
        self.worst = max(self.worst, float((d / lim.clamp_min(1e-300)).max()))
        self.same += int((_bits(got) == _bits(v.to(torch.bfloat16))).sum())
        self.n += got.numel()

    def check(self, identical):
        frac = self.same / max(self.n, 1)
        print(f"\n[{self.what}] beyond bound {self.bad} (worst {self.worst:.3f} of the bound), identical {frac:.5f}")
        assert self.bad == 0, (self.what, self.bad, self.worst)
        if identical:
            assert frac >= 0.999, (self.what, frac)


def _ln64(src):
    """fp64 LayerNorm of fp32 / bf16 rows -> (n, dn)"""
    xd = src.double()
    mu = xd.mean(-1, keepdim=True)
    den = ((xd - mu).square().mean(-1, keepdim=True) + EPS).sqrt()
    n = (xd - mu) / den
    dn = 2.0 ** -17 * n.abs() + 2.0 ** -18 * xd.abs().mean(-1, keepdim=True) / den
    return n, dn


def _hy_ref(x, scale, shift):
    """x [r, C] bf16; scale / shift bf16 [C] or per row [r, C] -> (v, E)"""
    n, dn = _ln64(x)
    t1 = (scale.float() + 1).bfloat16().double()          # bf16(fp32(1 + scale)): part of the definition
    sh = shift.double()
    return n * t1 + sh, t1.abs() * dn + 2.0 ** -22 * ((n * t1).abs() + sh.abs())


def _wan_ref(src, va, vb, affine, bf16_n):
    """src [r, C] (x or r); va / vb fp32 [C]: scale / shift, or weight / bias -> (v, E)"""
    n, dn = _ln64(src)
    a, b = va.double(), vb.double()
    if affine:
        return a * n + b, a.abs() * dn + 2.0 ** -22 * ((a * n).abs() + b.abs())
    t1 = (va + 1).double()                                 # fp32(1 + scale)
    if bf16_n:                                             # WanLayerNorm(x).type_as(x) of a bf16 x
        lo, hi = (n - dn).bfloat16().double(), (n + dn).bfloat16().double()
        nb = n.bfloat16().double()
        return nb * t1 + b, (hi - lo) * t1.abs() + 2.0 ** -22 * ((nb * t1).abs() + b.abs())
    return n * t1 + b, t1.abs() * dn + 2.0 ** -22 * ((n * t1).abs() + b.abs())


def _chunks(rows):
    for r0 in range(0, rows, CHUNK):
        yield slice(r0, min(rows, r0 + CHUNK))


def _repeat_ok(fn, first, rows):
    """every LayerNorm case above one grid pass is launched twice: bit for bit the same"""
    if rows > 8448:
        again = fn()
        pairs = zip(first, again) if isinstance(first, tuple) else [(first, again)]
        for a, b in pairs:
            assert torch.equal(_bits(a), _bits(b)), "second launch differs"


def _zero_rows_exact(kind, out, vb, rows):
    """(iv): a zero row normalises to 0, so it must come out as bf16(shift) (bf16(b) when affine)"""
    if kind != "zero_rows":
        return
    z = _zero_rows(rows)
    want = vb.reshape(1, -1).to(torch.bfloat16).expand(int(z.sum()), -1)
    assert torch.equal(_bits(out[z]), _bits(want))


# ------------------------------------------------------------------------------------------------
# HunyuanVideo ln_modulate (+ the FP8 form on the same rows)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,C,value,pad", _cases(0))
def test_ln_modulate_against_fp64(rows, C, value, pad):
    from jenga_b200 import dense as DN
    g = _gen(rows * 7 + C)
    x = _place(_values(value, rows, C, torch.bfloat16, g), pad)
    scale, shift = ((0.3 * torch.randn(C, generator=g, device="cuda")).bfloat16() for _ in range(2))
    run = lambda: DN.ln_modulate(x, shift, scale, eps=EPS)   # noqa: E731
    out = run()
    tally = _Tally(f"ln_modulate {rows}x{C} {value} pad={pad}")
    for s in _chunks(rows):
        tally.add(out[s], *_hy_ref(x[s], scale, shift))
    tally.check(value in IDENTICAL)
    _zero_rows_exact(value, out, shift, rows)
    _repeat_ok(run, out, rows)
    if C % 16 == 0:
        want = DN.quantize_rows_fp8(out)
        got = DN.ln_modulate_fp8(x, shift, scale, eps=EPS)
        assert torch.equal(got[1], want[1]) and torch.equal(_bits(got[0]), _bits(want[0]))


def _tr_mask(kind, rows, g):
    r = torch.arange(rows, device="cuda")
    return {"all": r >= 0, "none": r < 0, "alternating": r % 2 == 0,
            "scattered": torch.rand(rows, generator=g, device="cuda") < 0.3}[kind]


@pytest.mark.parametrize("mask_kind", ["all", "none", "alternating", "scattered"])
@pytest.mark.parametrize("rows,C,value", [(8449, 4096, "outliers"), (16897, 1032, "gauss")])
def test_ln_modulate_tr_against_fp64(rows, C, value, mask_kind):
    """odd rows above one grid pass: the last CTA has a dead half; a CPU mask gives the same rows"""
    from jenga_b200 import dense as DN
    g = _gen(rows + C)
    x = _values(value, rows, C, torch.bfloat16, g)
    scale, shift, tr_scale, tr_shift = ((0.3 * torch.randn(C, generator=g, device="cuda")).bfloat16()
                                        for _ in range(4))
    mask = _tr_mask(mask_kind, rows, g)
    tr = (tr_shift, tr_scale, mask)
    run = lambda: DN.ln_modulate(x, shift, scale, eps=EPS, tr=tr)   # noqa: E731
    out = run()
    tally = _Tally(f"ln_modulate_tr {rows}x{C} {value} {mask_kind}")
    for s in _chunks(rows):
        m = mask[s, None]
        tally.add(out[s], *_hy_ref(x[s], torch.where(m, tr_scale, scale), torch.where(m, tr_shift, shift)))
    tally.check(True)
    _repeat_ok(run, out, rows)
    assert torch.equal(_bits(DN.ln_modulate(x, shift, scale, eps=EPS, tr=(tr_shift, tr_scale, mask.cpu()))),
                       _bits(out))
    if C % 16 == 0:
        want = DN.quantize_rows_fp8(out)
        got = DN.ln_modulate_fp8(x, shift, scale, eps=EPS, tr=(tr_shift, tr_scale, mask.cpu()))
        assert torch.equal(got[1], want[1]) and torch.equal(_bits(got[0]), _bits(want[0]))


# ------------------------------------------------------------------------------------------------
# Wan: wan_ln_modulate, wan_residual_ln, wan_gate_residual
# ------------------------------------------------------------------------------------------------
def _wan_vecs(C, g, n):
    return [0.3 * torch.randn(C, generator=g, device="cuda") for _ in range(n)]


@pytest.mark.parametrize("x_dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("rows,C,value,pad", _cases(2))
def test_wan_ln_modulate_against_fp64(rows, C, value, pad, x_dtype):
    from jenga_b200 import dense as DN
    g = _gen(rows * 3 + C + (x_dtype == torch.float32))
    x = _place(_values(value, rows, C, x_dtype, g), pad)
    scale, shift = _wan_vecs(C, g, 2)
    run = lambda: DN.wan_ln_modulate(x, shift, scale, eps=EPS)   # noqa: E731
    out = run()
    tally = _Tally(f"wan_ln_modulate {rows}x{C} {value} pad={pad} x={str(x_dtype)[6:]}")
    for s in _chunks(rows):
        tally.add(out[s], *_wan_ref(x[s], scale, shift, False, x_dtype == torch.bfloat16))
    tally.check(value in IDENTICAL)
    _zero_rows_exact(value, out, shift, rows)
    _repeat_ok(run, out, rows)


def _residual_case(rows, C, value, pad, x_dtype, gated, g):
    x = _values(value, rows, C, x_dtype, g)
    y = (0.5 * torch.randn(rows, C, generator=g, device="cuda")).bfloat16()
    if value == "zero_rows":
        y[_zero_rows(rows)] = 0
    gate = 0.3 * torch.randn(C, generator=g, device="cuda") if gated else None
    return _place(x, pad), _place(y, pad), gate


@pytest.mark.parametrize("x_dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("rows,C,value,pad", _cases(4))
def test_wan_residual_ln_against_fp64(rows, C, value, pad, x_dtype):
    """the form rotates with the case: affine + gate (gate 1 + norm3), modulate without a gate (cross
    residual + norm2), modulate with a gate"""
    from jenga_b200 import dense as DN
    form = ["affine", "modulate", "modulate_gated"][(CHANNELS.index(C) + (x_dtype == torch.float32)) % 3]
    affine = form == "affine"
    g = _gen(rows * 5 + C + (x_dtype == torch.float32))
    x, y, gate = _residual_case(rows, C, value, pad, x_dtype, form != "modulate", g)
    va, vb = _wan_vecs(C, g, 2)
    if affine:
        va = va + 1.0
        kw = dict(weight=va, bias=vb)
    else:
        kw = dict(scale=va, shift=vb)
    run = lambda: DN.wan_residual_ln(x, y, gate, eps=EPS, **kw)   # noqa: E731
    res, out = run()
    tally = _Tally(f"wan_residual_ln {form} {rows}x{C} {value} pad={pad} x={str(x_dtype)[6:]}")
    for s in _chunks(rows):
        r = x[s] + (y[s] * gate if gate is not None else y[s].float())   # torch fp32 ops
        assert r.dtype == torch.float32 and torch.equal(_bits(res[s]), _bits(r))
        tally.add(out[s], *_wan_ref(r, va, vb, affine, False))
    tally.check(value in IDENTICAL)
    _zero_rows_exact(value, out, vb, rows)
    _repeat_ok(run, (res, out), rows)


@pytest.mark.parametrize("x_dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("rows,C,value,pad", _cases(1, CTA_ROWS))
def test_wan_gate_residual_is_bit_exact(rows, C, value, pad, x_dtype):
    from jenga_b200 import dense as DN
    g = _gen(rows * 11 + C)
    x, y, gate = _residual_case(rows, C, value, pad, x_dtype, True, g)
    out = DN.wan_gate_residual(x, y, gate)
    assert torch.equal(_bits(out), _bits(x + y * gate))


# ------------------------------------------------------------------------------------------------
# gate_residual[_tr]
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,C,value,pad", _cases(3, CTA_ROWS))
def test_gate_residual_is_bit_exact(rows, C, value, pad):
    from jenga_b200 import dense as DN
    g = _gen(rows * 13 + C)
    x = _place(_values(value, rows, C, torch.bfloat16, g), pad)
    y = _place(torch.randn(rows, C, generator=g, device="cuda").bfloat16(), 64 - pad)
    gate, tr_gate = (torch.randn(C, generator=g, device="cuda").bfloat16() for _ in range(2))
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        want, want_tr = x + y * gate, x + y * tr_gate
    assert torch.equal(_bits(DN.gate_residual(x, y, gate)), _bits(want))
    mask = _tr_mask("scattered", rows, g)
    got = DN.gate_residual(x, y, gate, tr=(tr_gate, mask))
    assert torch.equal(_bits(got), _bits(torch.where(mask[:, None], want_tr, want)))


# ------------------------------------------------------------------------------------------------
# gelu_tanh
# ------------------------------------------------------------------------------------------------
def _ulp_bf16(v):
    """spacing of bf16 at |v| (the subnormal spacing below the normal range)"""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def _gelu64(x):
    xd = x.double()
    return 0.5 * xd * (1 + torch.tanh(math.sqrt(2 / math.pi) * (xd + 0.044715 * xd ** 3)))


def _gelu_check(x, got):
    """-> (elements off the fp64 bound, elements not bit-identical to ATen)"""
    g = _gelu64(x)
    gd = got.double()
    nan_ok = torch.equal(torch.isnan(gd), torch.isnan(g))
    inf = torch.isinf(g)
    inf_ok = torch.equal(gd[inf], g[inf])
    fin = torch.isfinite(x.double()) & ~torch.isnan(g)
    off = ~((gd - g).abs() <= _ulp_bf16(g) + 2.0 ** -21 * x.double().abs())
    aten = F.gelu(x, approximate="tanh")
    nan_a = torch.isnan(aten.float())
    differ = (_bits(got) != _bits(aten)) & ~(nan_a & torch.isnan(got.float()))
    assert nan_ok and inf_ok
    return int((off & fin).sum()), int(differ.sum())


def test_gelu_tanh_every_bf16_pattern():
    """all 65 536 inputs: branch points |u| = 0.6 and 9.0109, large negative x (where 1 + tanh cancels),
    subnormals, +-0, +-inf and NaN; written into a strided destination whose padding stays untouched"""
    from jenga_b200 import dense as DN
    pat = (torch.arange(65536, dtype=torch.int32) - 32768).to(torch.int16)
    x = pat.view(torch.bfloat16).reshape(1, 64, 1024).cuda()
    buf = torch.full((1, 64, 1024 + 64), 0x7FA5, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    out = DN.gelu_tanh_into(x, buf[:, :, 32:32 + 1024])
    off, differ = _gelu_check(x, out)
    print(f"\n[gelu_tanh, every bf16] beyond the fp64 bound {off}, not bit-identical to ATen {differ}")
    assert off == 0 and differ == 0
    pad = torch.cat([buf[:, :, :32], buf[:, :, 32 + 1024:]], dim=-1)
    assert bool((_bits(pad) == 0x7FA5).all())


@pytest.mark.parametrize("rows,C,value,pad", _cases(5, CTA_ROWS))
def test_gelu_tanh_rows_and_widths(rows, C, value, pad):
    from jenga_b200 import dense as DN
    g = _gen(rows * 17 + C)
    x = _place((2.5 * _values(value, rows, C, torch.float32, g)).bfloat16(), pad)
    out_pad = PADS[(PADS.index(pad) + 1) % len(PADS)]
    out = DN.gelu_tanh_into(x, _place(torch.empty(rows, C, dtype=torch.bfloat16, device="cuda"), out_pad))
    off, differ = _gelu_check(x, out)
    assert off == 0 and differ == 0, (off, differ)


# ------------------------------------------------------------------------------------------------
# what lies past the end of a row (and past the last row) stays untouched
# ------------------------------------------------------------------------------------------------
def _sentinel_buf(rows, stride, dtype):
    """[rows + 1, stride] filled with a sentinel bit pattern"""
    itype, word = {torch.bfloat16: (torch.int16, 0x7FA5), torch.float32: (torch.int32, 0x7FA5A5A5),
                   torch.uint8: (torch.uint8, 0x5A)}[dtype]
    return torch.full((rows + 1, stride), word, dtype=itype, device="cuda").view(dtype), word


def _untouched(buf, rows, C, word):
    b = _bits(buf)
    return bool((b[:, C:] == word).all()) and bool((b[rows] == word).all())


@pytest.mark.parametrize("entry", ["ln_modulate", "ln_modulate_tr", "ln_modulate_fp8", "ln_modulate_tr_fp8",
                                   "gate_residual", "gate_residual_tr", "gelu_tanh", "wan_ln_modulate",
                                   "wan_residual_ln", "wan_gate_residual"])
def test_out_stride_wider_than_the_row(entry):
    """through the C ABI with out_stride = C + 48: the output rows equal the contiguous result, and the
    padding after each row and the row after the last one keep their sentinel"""
    from jenga_b200 import _lib, dense as DN
    from jenga_b200.attention import _stream_ptr
    lib = _lib.lib
    ln = entry.startswith(("ln_", "wan_ln", "wan_res"))
    rows, C = (8449 if ln else 2113), 1040
    S = C + 48
    g = _gen(len(entry))
    x = _values("gauss", rows, C, torch.bfloat16, g)
    xf = _values("gauss", rows, C, torch.float32, g)
    y = torch.randn(rows, C, generator=g, device="cuda").bfloat16()
    v1, v2, v3, v4 = ((0.3 * torch.randn(C, generator=g, device="cuda")).bfloat16() for _ in range(4))
    f1, f2, f3 = _wan_vecs(C, g, 3)
    mask = _tr_mask("scattered", rows, g)
    st = _stream_ptr(x.device)
    P = lambda t: t.data_ptr()   # noqa: E731
    checks = []                  # (buffer, reference, sentinel word)
    if entry.startswith("ln_modulate"):
        tr = entry.startswith("ln_modulate_tr")
        want = DN.ln_modulate(x, v2, v1, eps=EPS, tr=(v4, v3, mask) if tr else None)
        if entry.endswith("fp8"):
            q, s = DN.quantize_rows_fp8(want)
            out8, w8 = _sentinel_buf(rows, S, torch.uint8)
            a_scale, ws = _sentinel_buf(rows, 1, torch.float32)
            if tr:
                rc = lib.jenga_ln_modulate_tr_fp8(P(x), C, P(v1), P(v2), P(v3), P(v4), P(mask), P(out8), S,
                                                  P(a_scale), rows, C, EPS, st)
            else:
                rc = lib.jenga_ln_modulate_fp8(P(x), C, P(v1), P(v2), P(out8), S, P(a_scale), rows, C, EPS, st)
            checks += [(out8, q.view(torch.uint8), w8), (a_scale, s[:, None], ws)]
        else:
            out, w = _sentinel_buf(rows, S, torch.bfloat16)
            if tr:
                rc = lib.jenga_ln_modulate_tr(P(x), C, P(v1), P(v2), P(v3), P(v4), P(mask), P(out), S, rows, C, EPS, st)
            else:
                rc = lib.jenga_ln_modulate(P(x), C, P(v1), P(v2), P(out), S, rows, C, EPS, st)
            checks += [(out, want, w)]
    elif entry.startswith("gate_residual"):
        tr = entry == "gate_residual_tr"
        want = DN.gate_residual(x, y, v1, tr=(v2, mask) if tr else None)
        out, w = _sentinel_buf(rows, S, torch.bfloat16)
        if tr:
            rc = lib.jenga_gate_residual_tr(P(x), C, P(y), C, P(v1), P(v2), P(mask), P(out), S, rows, C, st)
        else:
            rc = lib.jenga_gate_residual(P(x), C, P(y), C, P(v1), P(out), S, rows, C, st)
        checks += [(out, want, w)]
    elif entry == "gelu_tanh":
        want = F.gelu(x, approximate="tanh")
        out, w = _sentinel_buf(rows, S, torch.bfloat16)
        rc = lib.jenga_gelu_tanh(P(x), C, P(out), S, rows, C, st)
        checks += [(out, want, w)]
    elif entry == "wan_ln_modulate":
        want = DN.wan_ln_modulate(xf, f2, f1, eps=EPS)
        out, w = _sentinel_buf(rows, S, torch.bfloat16)
        rc = lib.jenga_wan_ln_modulate(P(xf), _lib.JENGA_F32, C, P(f1), P(f2), P(out), S, rows, C, EPS, st)
        checks += [(out, want, w)]
    elif entry == "wan_residual_ln":
        want_r, want = DN.wan_residual_ln(xf, y, f3, eps=EPS, shift=f2, scale=f1)
        out, w = _sentinel_buf(rows, S, torch.bfloat16)
        res, wr = _sentinel_buf(rows, S, torch.float32)
        rc = lib.jenga_wan_residual_ln(P(xf), _lib.JENGA_F32, C, P(y), C, P(f3), P(res), S, P(f1), P(f2), 0,
                                       P(out), S, rows, C, EPS, st)
        checks += [(out, want, w), (res, want_r, wr)]
    else:
        want = DN.wan_gate_residual(xf, y, f3)
        out, w = _sentinel_buf(rows, S, torch.float32)
        rc = lib.jenga_wan_gate_residual(P(xf), _lib.JENGA_F32, C, P(y), C, P(f3), P(out), S, rows, C, st)
        checks += [(out, want, w)]
    assert rc == 0, lib.jenga_last_error()
    torch.cuda.synchronize()
    for buf, ref, word in checks:
        n = ref.shape[1]
        assert torch.equal(_bits(buf[:rows, :n]), _bits(ref)), entry
        assert _untouched(buf, rows, n, word), entry


# ------------------------------------------------------------------------------------------------
# production sizes, once each (fp64 references in chunks of CHUNK rows)
# ------------------------------------------------------------------------------------------------
HY_ROWS, HY_C = 115456, 3072          # HunyuanVideo 720p, image + text
WAN_ROWS, WAN_C = 75600, 5120         # Wan 14B


@pytest.mark.parametrize("entry", ["ln_modulate", "ln_modulate_tr", "ln_modulate_fp8"])
def test_full_size_hunyuan_ln_modulate(entry):
    from jenga_b200 import dense as DN
    g = _gen(5)
    value = "outliers" if entry == "ln_modulate_tr" else "gauss"
    x = _values(value, HY_ROWS, HY_C, torch.bfloat16, g)
    scale, shift, tr_scale, tr_shift = ((0.3 * torch.randn(HY_C, generator=g, device="cuda")).bfloat16()
                                        for _ in range(4))
    mask = _tr_mask("scattered", HY_ROWS, g)
    tr = (tr_shift, tr_scale, mask) if entry == "ln_modulate_tr" else None
    run = lambda: DN.ln_modulate(x, shift, scale, eps=EPS, tr=tr)   # noqa: E731
    out = run()
    if entry == "ln_modulate_fp8":
        want = DN.quantize_rows_fp8(out)
        del out
        got = DN.ln_modulate_fp8(x, shift, scale, eps=EPS)
        assert torch.equal(got[1], want[1]) and torch.equal(_bits(got[0]), _bits(want[0]))
        return
    tally = _Tally(f"{entry} {HY_ROWS}x{HY_C} {value}")
    for s in _chunks(HY_ROWS):
        if tr is None:
            tally.add(out[s], *_hy_ref(x[s], scale, shift))
        else:
            m = mask[s, None]
            tally.add(out[s], *_hy_ref(x[s], torch.where(m, tr_scale, scale), torch.where(m, tr_shift, shift)))
    tally.check(True)
    _repeat_ok(run, out, HY_ROWS)


def _row_fingerprint(t):
    """one int64 per row, a weighted sum of the element bit patterns (chunked: no full-size temporary)"""
    w = torch.arange(1, t.shape[1] + 1, device=t.device, dtype=torch.int64)
    return torch.cat([(_bits(t[s]).long() * w).sum(-1) for s in _chunks(t.shape[0])])


@pytest.mark.parametrize("form,value", [("affine", "zero_rows"), ("modulate", "offset")])
def test_full_size_wan_residual_ln(form, value):
    """fp32 x, bf16 y, gated residual: x, y, res and out take 4.6 GB, the least this shape needs; the
    repeat launch is compared through row fingerprints so that no second copy is held"""
    from jenga_b200 import dense as DN
    g = _gen(6)
    x, y, gate = _residual_case(WAN_ROWS, WAN_C, value, 0, torch.float32, True, g)
    va, vb = _wan_vecs(WAN_C, g, 2)
    affine = form == "affine"
    if affine:
        va = va + 1.0
    kw = dict(weight=va, bias=vb) if affine else dict(scale=va, shift=vb)
    res, out = DN.wan_residual_ln(x, y, gate, eps=EPS, **kw)
    tally = _Tally(f"wan_residual_ln {form} {WAN_ROWS}x{WAN_C} {value}")
    for s in _chunks(WAN_ROWS):
        r = x[s] + y[s] * gate
        assert torch.equal(_bits(res[s]), _bits(r))
        tally.add(out[s], *_wan_ref(r, va, vb, affine, False))
    tally.check(False)
    _zero_rows_exact(value, out, vb, WAN_ROWS)
    first = _row_fingerprint(res), _row_fingerprint(out)
    del res, out
    res, out = DN.wan_residual_ln(x, y, gate, eps=EPS, **kw)
    assert torch.equal(_row_fingerprint(res), first[0]) and torch.equal(_row_fingerprint(out), first[1])


@pytest.mark.parametrize("entry", ["gelu_tanh", "gate_residual"])
def test_full_size_hunyuan_row_kernels(entry):
    from jenga_b200 import dense as DN
    g = _gen(7)
    x = (2.5 * torch.randn(HY_ROWS, HY_C, generator=g, device="cuda")).bfloat16()
    if entry == "gelu_tanh":
        out = DN.gelu_tanh_into(x, torch.empty_like(x))
        for s in _chunks(HY_ROWS):
            assert torch.equal(_bits(out[s]), _bits(F.gelu(x[s], approximate="tanh")))
        return
    y = torch.randn(HY_ROWS, HY_C, generator=g, device="cuda").bfloat16()
    gate = torch.randn(HY_C, generator=g, device="cuda").bfloat16()
    out = DN.gate_residual(x, y, gate)
    for s in _chunks(HY_ROWS):
        assert torch.equal(_bits(out[s]), _bits(x[s] + y[s] * gate))
