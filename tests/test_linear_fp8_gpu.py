"""Opt-in FP8 Linears (csrc/linear_fp8.cu, dense.linear_fp8, blocks._linear) on the GPU.

1. jenga_quantize_rows_fp8 is bit-identical to the torch restatement of test_linear_fp8_cpu.py, and
   jenga_ln_modulate_fp8 / _tr_fp8 to quantize_rows_fp8(ln_modulate(...)).
2. The GEMM against an fp64 product of the dequantised operands: within one bf16 ulp of the exact
   value plus 2^-14 of sum |a w|.  The second term is the accumulation inside one 128-channel slice:
   Hopper's FP8 wgmma aligns the products of an instruction to a narrower accumulator than fp32 (with
   2^-20 instead, 1 % of the outputs of a random 384 x 3072 x 9216 case fail, by up to 16x, on an H100).
   An accumulator that is not promoted to fp32 every 128 channels drifts by far more than this at
   K = 15 360 when every product carries the same sign (the constant-offset case).
3. A --use-fp8 Linear (e4m3 weight + fp8_scale) through blocks._linear against a restatement of the
   reference's fp8_linear_forward (hyvideo/modules/fp8_optimization.py): its own tolerance row,
   LINEAR_FP8_REF_TOL, which only the FP8 activations account for.
4. The unmodified HunyuanVideo and I2V blocks.  With the switch off, and with it on under the shipped
   routing table (dense.FP8_ROUTED), the output is bit-identical to the block body as it was before the
   FP8 path existed (each Linear called on the module).  With every shape routed: LINEAR_FP8_BLOCK_TOL
   of the output RMS against off, and the number of FP8 GEMM launches per block kind.
"""
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))

pytestmark = pytest.mark.gpu

from test_linear_fp8_cpu import quantize_rows_ref  # noqa: E402

# mean, max of |ours - reference fp8 forward| / output RMS; an H100 showed 2.1e-2 / 0.13 on these Gaussian
# activations, the e4m3 rounding of each activation (3 mantissa bits)
LINEAR_FP8_REF_TOL = (3e-2, 0.2)
# mean, max of |on - off| / output RMS, per block output; an H100 showed at most 2.6e-3 / 6.1e-2
LINEAR_FP8_BLOCK_TOL = (2.5e-2, 0.25)
SHAPES = [(3072, 9216), (3072, 3072), (3072, 12288), (12288, 3072), (3072, 21504), (15360, 3072)]   # (K, N)


class _Everything(frozenset):
    """a routing table that contains every shape"""
    def __contains__(self, item):
        return True


ALL_ROUTED = _Everything({None})


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda")


def _bits(t):
    return t.view(torch.uint8)


# ------------------------------------------------------------------ 1. quantisation parity
@pytest.mark.parametrize("M,K,strided", [(1, 16, False), (127, 3072, False), (300, 15360, True), (64, 12288, False)])
def test_quantize_rows_matches_the_restatement(M, K, strided):
    from jenga_b200 import dense as DN
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(M + K)
    base = torch.randn(M, K + (64 if strided else 0), generator=g, device=dev) * 3
    base[0, :] *= 1e-30 if M > 2 else 1.0       # a row of tiny values
    if M > 3:
        base[1] = 0                             # a zero row: scale 1, codes 0
        base[2, 5] = 1e4                        # one large value sets the row scale
    x = base.bfloat16()[:, :K]
    codes, scale = DN.quantize_rows_fp8(x)
    rc, rs = quantize_rows_ref(x.cpu())
    assert torch.equal(scale.cpu(), rs)
    assert torch.equal(_bits(codes).cpu(), _bits(rc))


@pytest.mark.parametrize("tr", [False, True])
@pytest.mark.parametrize("L,C", [(1, 3072), (257, 3072), (130, 512)])
def test_ln_modulate_fp8_is_quantize_of_ln_modulate(L, C, tr):
    from jenga_b200 import dense as DN
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(L * 7 + C)
    x = (torch.randn(1, L, C, generator=g, device=dev) * 2 + 0.3).bfloat16()
    sh, sc = ((torch.randn(1, C, generator=g, device=dev) * 0.4).bfloat16() for _ in range(2))
    trm = None
    if tr:
        ts, tsc = ((torch.randn(1, C, generator=g, device=dev) * 0.4).bfloat16() for _ in range(2))
        trm = (ts, tsc, torch.rand(L, generator=g, device=dev) < 0.4)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        want = DN.quantize_rows_fp8(DN.ln_modulate(x, sh, sc, eps=1e-6, tr=trm))
        got = DN.ln_modulate_fp8(x, sh, sc, eps=1e-6, tr=trm)
    assert torch.equal(got[1], want[1])
    assert torch.equal(_bits(got[0]), _bits(want[0]))


# ------------------------------------------------------------------ 2. GEMM against fp64
def _gemm_case(M, K, N, seed, offset=0.0, a_stride=None, per_tensor=False, bias=None):
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(M, a_stride or K, generator=g, device=dev) * 100 + offset
    a8 = a.clamp(-448, 448).to(torch.float8_e4m3fn)[:, :K]
    w8 = (torch.randn(N, K, generator=g, device=dev) * 100 + offset).clamp(-448, 448).to(torch.float8_e4m3fn)
    a_scale = torch.rand(M, generator=g, device=dev) * 1e-2 + 1e-3
    w_scale = (torch.rand(1 if per_tensor else N, generator=g, device=dev) * 1e-2 + 1e-3)
    b = None
    if bias is not None:
        b = torch.randn(N, generator=g, device=dev).to(bias)
    return a8, a_scale, w8, w_scale, b


def _check_gemm(a8, a_scale, w8, w_scale, b, out):
    A, W = a8.double(), w8.double()
    ws = w_scale.double().expand(W.shape[0])
    exact = (A @ W.T) * a_scale.double()[:, None] * ws[None]
    mag = (A.abs() @ W.abs().T) * a_scale.double()[:, None] * ws[None]
    if b is not None:
        exact = exact + b.double()
    ulp = torch.exp2(torch.floor(torch.log2(exact.abs().clamp_min(1e-30))) - 7)
    err = (out.double() - exact).abs()
    bound = ulp + mag * 2.0 ** -14
    bad = err > bound
    assert not bad.any(), (int(bad.sum()), float((err / bound).max()))
    assert torch.equal(out.isfinite(), torch.ones_like(out, dtype=torch.bool))


@pytest.mark.parametrize("K,N", SHAPES)
def test_gemm_on_the_hunyuan_shapes(K, N):
    from jenga_b200 import dense as DN
    case = _gemm_case(384, K, N, K + N, bias=torch.bfloat16)
    _check_gemm(*case, DN.linear_fp8(*case))


@pytest.mark.parametrize("M", [1, 127, 129, 115456])
def test_gemm_ragged_and_full_m(M):
    from jenga_b200 import dense as DN
    case = _gemm_case(M, 3072, 3072, M)
    _check_gemm(*case, DN.linear_fp8(*case))


@pytest.mark.parametrize("variant", ["fp32_bias", "per_tensor", "strided_a", "ragged_kn"])
def test_gemm_variants(variant):
    from jenga_b200 import dense as DN
    if variant == "fp32_bias":
        case = _gemm_case(200, 1024, 1536, 1, bias=torch.float32)
    elif variant == "per_tensor":
        case = _gemm_case(200, 1024, 1536, 2, per_tensor=True, bias=torch.bfloat16)
    elif variant == "strided_a":
        case = _gemm_case(333, 3072, 1024, 3, a_stride=3072 + 512)
    else:                                   # K not a multiple of 128, N not a multiple of 128
        case = _gemm_case(257, 144, 200, 4, bias=torch.bfloat16)
    _check_gemm(*case, DN.linear_fp8(*case))


def test_gemm_keeps_fp32_accumulation_over_k_15360_with_a_constant_offset():
    from jenga_b200 import dense as DN
    case = _gemm_case(256, 15360, 256, 9, offset=200.0)
    _check_gemm(*case, DN.linear_fp8(*case))


# ------------------------------------------------------------------ 3. reference --use-fp8 Linear
def _ref_fp8_linear_forward(layer, x):
    """hyvideo/modules/fp8_optimization.py:fp8_linear_forward with an e4m3 weight, restated:
    F.linear(x, weight.to(bf16) * fp8_scale.to(bf16), bias)"""
    w = layer.weight.to(torch.bfloat16) * layer.fp8_scale.to(layer.weight.device).to(torch.bfloat16)
    return torch.nn.functional.linear(x, w, layer.bias)


def test_use_fp8_linear_through_the_block_helper(monkeypatch):
    from jenga_b200 import blocks, dense as DN
    monkeypatch.setattr(DN, "FP8_ROUTED", frozenset({("fp8_ref", 3072, 3072)}))
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(5)
    lin = torch.nn.Linear(3072, 3072, bias=True, device=dev, dtype=torch.bfloat16)
    with torch.no_grad():
        w = torch.randn(3072, 3072, generator=g, device=dev) * 0.02
        s = w.abs().max() / 448
        lin.weight = torch.nn.Parameter((w / s).to(torch.float8_e4m3fn), requires_grad=False)
        lin.fp8_scale = s.cpu().to(torch.bfloat16)                      # convert_fp8_linear: fp8_map[key].to(bf16)
        lin.bias.copy_(torch.randn(3072, generator=g, device=dev) * 0.1)
    x = (torch.randn(1, 1000, 3072, generator=g, device=dev)).bfloat16()
    before = blocks.STATS["linear_fp8"]
    old = DN.LINEAR_FP8
    DN.LINEAR_FP8 = True
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            got = blocks._linear(lin, x)
            want = _ref_fp8_linear_forward(lin, x)
    finally:
        DN.LINEAR_FP8 = old
    assert blocks.STATS["linear_fp8"] == before + 1
    e = (got.double() - want.double()).abs() / want.double().pow(2).mean().sqrt()
    print(f"\n[--use-fp8 Linear] mean {e.mean():.2e} max {e.max():.2e}")
    assert e.mean() <= LINEAR_FP8_REF_TOL[0] and e.max() <= LINEAR_FP8_REF_TOL[1]


# ------------------------------------------------------------------ 4. blocks
@pytest.fixture(scope="module")
def hy_modules():
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    our_hy, _ = R.load_blocks(product=True)
    from i2v_ref import load_i2v_blocks
    yield our_hy, load_i2v_blocks(product=True)
    from jenga_b200 import blocks
    blocks.remove_gather_hook()


def _rms_err(a, b):
    e = (a.double() - b.double()).abs() / b.double().pow(2).mean().sqrt()
    return e.mean().item(), e.max().item()


def _block_case(hy_modules, variant, kind):
    from test_dropin_blocks_gpu import _hy_case, _reinit
    from test_i2v_blocks_gpu import _i2v_case
    from jenga_b200 import blocks, dense as DN
    mod = hy_modules[0 if variant == "hy" else 1]
    c = _hy_case(mod) if variant == "hy" else _i2v_case(mod, 400, 300)
    cls = "MMDoubleStreamBlock" if kind == "double" else "MMSingleStreamBlock"
    blk = getattr(mod, cls)(c["C"], c["H"], mlp_width_ratio=4.0, dtype=torch.bfloat16, device="cuda")
    _reinit(blk, 11)
    S = c["L"] + c["T"]
    if variant == "hy":
        tail = dict(sa_drop_rate=0.7, txt_amp=0.431, curve_sel=c["curve_sel"], p_remain_rates=0.3)
    else:
        mask = c["ff"] if kind == "double" else c["full"]
        tail = dict(sa_drop_rate=0.7, first_frame_mask=mask, condition_type="token_replace",
                    token_replace_vec=c["tr_vec"], frist_frame_token_num=c["hw"], txt_amp=0.431,
                    curve_sel=c["curve_sel"], p_remain_rates=0.3)

    def run(on, routed=DN.FP8_ROUTED):
        old = DN.LINEAR_FP8, DN.FP8_ROUTED
        DN.LINEAR_FP8, DN.FP8_ROUTED = on, routed
        before = dict(blocks.STATS)
        try:
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                if kind == "double":
                    out = blk(c["img"], c["txt"], c["vec"], c["cu"], c["cu"], S, S, c["freqs"], **tail)
                else:
                    out = (blk(torch.cat([c["img"], c["txt"]], 1), c["vec"], c["T"], c["cu"], c["cu"], S, S,
                               c["freqs"], **tail),)
            torch.cuda.synchronize()
        finally:
            DN.LINEAR_FP8, DN.FP8_ROUTED = old
        return out, {k: blocks.STATS[k] - before[k] for k in before if blocks.STATS[k] != before[k]}
    return run


@pytest.mark.parametrize("variant", ["hy", "i2v"])
@pytest.mark.parametrize("kind", ["double", "single"])
def test_blocks_off_and_as_shipped_equal_the_module_calls(hy_modules, variant, kind, monkeypatch):
    from jenga_b200 import blocks
    run = _block_case(hy_modules, variant, kind)
    off, d_off = run(False)
    shipped, d_shipped = run(True)
    ln_mod = blocks._ln_mod
    # the block body before the FP8 path: every Linear and the MLP called on the module
    monkeypatch.setattr(blocks, "_linear", lambda layer, x, x8=None: layer(x))
    monkeypatch.setattr(blocks, "_mod_linear", lambda mod, layer, norm, x, shift, scale, tr=None:
                        layer(ln_mod(mod, norm, x, shift, scale, tr=tr)))
    monkeypatch.setattr(blocks, "_mlp", lambda mod, mlp, norm, x, shift, scale, tr=None:
                        mlp(ln_mod(mod, norm, x, shift, scale, tr=tr)))
    before, d_before = run(False)
    key = f"{variant}_{kind}"
    for d in (d_off, d_shipped):
        assert d == d_before and "linear_fp8" not in d and d.get(key) == 1 and "fallback" not in d
    assert all(torch.equal(a, b) for a, b in zip(off, before))
    assert all(torch.equal(a, b) for a, b in zip(shipped, before))


@pytest.mark.parametrize("variant", ["hy", "i2v"])
@pytest.mark.parametrize("kind", ["double", "single"])
def test_blocks_with_every_linear_routed(hy_modules, variant, kind):
    run = _block_case(hy_modules, variant, kind)
    off, _ = run(False)
    on, d_on = run(True, ALL_ROUTED)
    key = f"{variant}_{kind}"
    assert d_on["linear_fp8"] == (4 if kind == "double" else 2) and d_on.get(key) == 1 and "fallback" not in d_on
    for a, b in zip(on, off):
        mean, mx = _rms_err(a, b)
        print(f"\n[{variant} {kind}] FP8 Linears on vs off: mean {mean:.2e} max {mx:.2e} of the output RMS")
        assert mean <= LINEAR_FP8_BLOCK_TOL[0] and mx <= LINEAR_FP8_BLOCK_TOL[1]
