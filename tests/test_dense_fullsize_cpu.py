"""The dense-launch restatements of tests/attn_ref.py, checked without a GPU: varlen segments and the Wan
I2V sum against fp64 truth and the CPU oracle on small ragged cases, the FP8 P.V expectation against the
e4m3 codes and its certificate, and the per-element bounds against restatements of the mistakes the
full-size GPU file (tests/test_dense_fullsize_gpu.py) is there to catch."""
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
import attn_ref as R  # noqa: E402
import refutil  # noqa: E402
from test_attn_edges_gpu import _oracle  # noqa: E402
from test_producers_cpu import e4m3_satfinite  # noqa: E402

BLOCK = D = 128
SM = D ** -0.5


def _truth(q, k, v, kv_limit=None):
    """fp64 dense attention [B, Sq, H, D] of every row of q over k / v's keys below kv_limit (default Sk)."""
    B, Sq, H, _ = q.shape
    Sk = k.shape[1]
    nb = (Sk + BLOCK - 1) // BLOCK
    nq = (Sq + BLOCK - 1) // BLOCK
    qp = refutil.pad_rows(q, nq * BLOCK)
    t = refutil.fp64_truth(qp, k, v, torch.zeros(B, 1, 0, nb, dtype=torch.bool), list(range(nq)), n_img_blocks=0,
                           seqlen=Sk, sm_scale=SM, kv_limit_dense=Sk if kv_limit is None else kv_limit)
    rows = torch.cat([t[m] if B > 1 else t[m][None] for m in range(nq)], 2)      # [B, H, nq*128, D]
    return rows.transpose(1, 2)[:, :Sq]


def _assert_rounds_of(got, x):
    """got is round16(x) bit for bit wherever x is not within 2^-20 (relative) of a midpoint of the
    16-bit grid: there the kernel's o * (1 / l) and the division may round apart.  x's fp64 softmax
    leaves ~1e-16 where the exact value is 0."""
    x = x.masked_fill(x.abs() < 1e-12, 0.0)
    nudge = x.abs() * 2.0 ** -20
    tie = (x + nudge).to(got.dtype) != (x - nudge).to(got.dtype)
    assert torch.equal(got[~tie], x.to(got.dtype)[~tie])
    assert int(tie.sum()) <= got.numel() // 10      # every row of a flat segment repeats the same values
    return tie


# (cu_q, cu_k, H): Sk inside a block, cu_q != cu_k, an empty segment, a keyless segment
SEGMENTS = {
    "hy_pattern": ([0, 300, 376], [0, 300, 376], 2),
    "q_ne_k": ([0, 200, 329], [0, 37, 549], 2),
    "empty_and_keyless": ([0, 140, 140, 396, 400], [0, 257, 300, 300, 428], 2),
    "batch2_wan": ([0, 260, 520], [0, 37, 549], 3),
}


@pytest.mark.parametrize("name", list(SEGMENTS))
def test_segments_expected_equals_fp64_truth(name):
    """segments_expected (each segment one dense launch over its own keys, column limit Sk inside a
    block) is the round16 of fp64 attention per segment, and zeros where a segment has no keys."""
    cu_q, cu_k, H = SEGMENTS[name]
    Tq, Tk = cu_q[-1], cu_k[-1]
    _, k, v = R.flat_case(1, Tk, H, seed=len(name), device="cpu")
    got = R.segments_expected(v[0], cu_q, cu_k, Tq)
    assert got.shape == (Tq, H, D)
    for i in range(len(cu_q) - 1):
        q0, q1, k0, k1 = cu_q[i], cu_q[i + 1], cu_k[i], cu_k[i + 1]
        if q1 == q0:
            continue
        if k1 == k0:
            assert not got[q0:q1].any()
            continue
        q = torch.zeros(1, q1 - q0, H, D, dtype=torch.bfloat16)
        _assert_rounds_of(got[q0:q1][None], _truth(q, k[:, k0:k1], v[:, k0:k1]))
    assert torch.equal(R.segments_expected(v[0], cu_q, cu_k, Tq), got)


def test_dense_expected_batch2_equals_the_oracle():
    """B = 2 in one launch with a ragged key count: each sample its own flat sum, as the CPU oracle has it."""
    q, k, v = R.flat_case(2, 300, 2, seed=4, device="cpu")
    qr = torch.zeros(2, 200, 2, D, dtype=torch.bfloat16)
    got = R.dense_expected(v, 200)
    _assert_rounds_of(got, _truth(qr, k, v))
    want = _oracle(qr, k, v, None, 0, 2, seqlen=300, kv_limit_dense=300)
    tie = _assert_rounds_of(got, _truth(qr, k, v))
    assert torch.equal(got[~tie], want[~tie])


def _i2v_parts(Lq=200, Li=257, Lt=512, H=2, seed=7, real=True, sigma=1.5):
    g = torch.Generator().manual_seed(seed)
    if real:
        q = (torch.randn(1, Lq, H, D, generator=g) * sigma).bfloat16()
        ki = (torch.randn(1, Li, H, D, generator=g) * sigma).bfloat16()
        kt = (torch.randn(1, Lt, H, D, generator=g) * sigma).bfloat16()
        vi = torch.randn(1, Li, H, D, generator=g).bfloat16()
        vt = torch.randn(1, Lt, H, D, generator=g).bfloat16()
        return q, ki, vi, kt, vt
    q, ki, vi = R.flat_case(1, Li, H, seed=seed, device="cpu")
    _, kt, vt = R.flat_case(1, Lt, H, seed=seed + 1, device="cpu")
    return q[:, :1].expand(1, Lq, H, D).contiguous(), ki, vi, kt, vt


def _seg(q, k, v, kv_limit=None):
    """One dense launch over k / v as the CPU oracle computes it (P rounded as the kernel rounds it)."""
    nq = (q.shape[1] + BLOCK - 1) // BLOCK
    return _oracle(q, k, v, None, 0, nq, seqlen=k.shape[1], kv_limit_dense=k.shape[1] if kv_limit is None else kv_limit)


def _i2v_oracle(q, ki, vi, kt, vt, mistake=None):
    """out = round16(f32(A_img) + f32(A_txt)) on the CPU oracle, or one of the kernel's possible mistakes:
    'early' the segment switch one tile early (the last image tile joins the text softmax), 'txt_limit'
    the text keys limited at the image row count, 'unrounded' A_img added in fp32 before rounding,
    'pad_keys' each segment's column limit at its tile end."""
    Li = ki.shape[1]
    if mistake == "early":
        cut = (Li - 1) // BLOCK * BLOCK
        a_img = _seg(q, ki[:, :cut], vi[:, :cut])
        a_txt = _seg(q, torch.cat([ki[:, cut:], kt], 1), torch.cat([vi[:, cut:], vt], 1))
    elif mistake == "unrounded":
        nq = (q.shape[1] + BLOCK - 1) // BLOCK
        from oracle import attention_oracle as orc
        kp, vp = (refutil.pad_rows(x, (Li + BLOCK - 1) // BLOCK * BLOCK).transpose(1, 2) for x in (ki, vi))
        qp = refutil.pad_rows(q, nq * BLOCK).transpose(1, 2)
        a_img = orc.dense_attention_rows(qp.float(), kp.float(), vp.float(), SM, Li).transpose(1, 2)[:, :q.shape[1]]
        a_txt = _seg(q, kt, vt)
    else:
        lim_i = lim_t = None
        if mistake == "txt_limit":
            lim_t = Li
        if mistake == "pad_keys":
            lim_i = (Li + BLOCK - 1) // BLOCK * BLOCK
            lim_t = (kt.shape[1] + BLOCK - 1) // BLOCK * BLOCK
        a_img = _seg(q, ki, vi, lim_i)
        a_txt = _seg(q, kt, vt, lim_t)
    return (a_img.float() + a_txt.float()).bfloat16()


def test_i2v_expected_equals_the_oracle_composition():
    """Leg A of the I2V kernel: round16(f32(A_img) + f32(A_txt)) over Li = 257 and Lt = 512 equals the CPU
    oracle's composition, and each mistake of the kernel changes it."""
    q, ki, vi, kt, vt = _i2v_parts(real=False)
    got = R.i2v_expected(vi, vt, q.shape[1])
    want = _i2v_oracle(q, ki, vi, kt, vt)
    tie_i = _assert_rounds_of(R.dense_expected(vi, q.shape[1]), _truth(q, ki, vi))
    tie_t = _assert_rounds_of(R.dense_expected(vt, q.shape[1]), _truth(q, kt, vt))
    ok = ~(tie_i | tie_t)
    assert torch.equal(got[ok], want[ok])
    for mistake in ("early", "unrounded", "txt_limit", "pad_keys"):
        bad = _i2v_oracle(q, ki, vi, kt, vt, mistake)
        assert not torch.equal(got[ok], bad[ok]), mistake


@pytest.mark.parametrize("seed", [7, 8])
def test_i2v_bound_holds_for_the_oracle_and_fails_mistakes(seed):
    """Leg B of the I2V kernel: the oracle composition lies within i2v_bound; the segment switch one tile
    early, the text segment limited at the image row count and the column limit at the tile end
    exceed it.  (A_img left unrounded is more accurate, not less: Leg A catches that one.)"""
    q, ki, vi, kt, vt = _i2v_parts(seed=seed)
    nq = (q.shape[1] + BLOCK - 1) // BLOCK
    worst = {}
    for h in range(q.shape[2]):
        kw = dict(b=0, h=h, qblocks=range(nq), nq_sparse=0, sm_scale=SM, chunk=2)
        ri = R.fp64_rows(q, ki, vi, None, kv_limit_dense=ki.shape[1], **kw)
        rt = R.fp64_rows(q, kt, vt, None, kv_limit_dense=kt.shape[1], **kw)
        o, E = R.i2v_bound(ri, rt)
        assert torch.allclose(o, (_truth(q, ki, vi) + _truth(q, kt, vt))[0, :, h], rtol=0, atol=1e-12)
        for mistake in (None, "early", "txt_limit", "pad_keys"):
            out = _i2v_oracle(q, ki, vi, kt, vt, mistake)[0, :, h].double()
            worst[mistake] = max(worst.get(mistake, 0.0), ((out - o).abs() / E).max().item())
    print(worst)
    assert worst[None] <= 1.0
    for mistake in ("early", "txt_limit", "pad_keys"):
        assert worst[mistake] > 1.0, mistake


@pytest.mark.parametrize("Sk", [76, 257, 300, 37])
def test_dense_column_limit_inside_a_block(Sk):
    """A dense launch with Sk inside a block: fp64_rows with kv_limit_dense = Sk is fp64 truth, the oracle
    is within its bound, and a column limit at the tile end (the zero-filled keys counted) differs in
    Leg A and exceeds E in Leg B."""
    H, Sq = 2, 140
    g = torch.Generator().manual_seed(Sk)
    q = (torch.randn(1, Sq, H, D, generator=g) * 1.5).bfloat16()
    k = (torch.randn(1, Sk, H, D, generator=g) * 1.5).bfloat16()
    v = torch.randn(1, Sk, H, D, generator=g).bfloat16()
    Sp = (Sk + BLOCK - 1) // BLOCK * BLOCK
    ok_out, pad_out = _seg(q, k, v), _seg(q, k, v, Sp)
    nq = (Sq + BLOCK - 1) // BLOCK
    for h in range(H):
        ref = R.fp64_rows(q, k, v, None, b=0, h=h, qblocks=range(nq), nq_sparse=0, sm_scale=SM, kv_limit_dense=Sk)
        assert torch.allclose(ref["o"], _truth(q, k, v)[0, :, h], rtol=0, atol=1e-12)
        _, lse = refutil.fp64_truth(refutil.pad_rows(q, nq * BLOCK), k, v, torch.zeros(1, H, 0, Sp // BLOCK, dtype=torch.bool),
                                    list(range(nq)), n_img_blocks=0, seqlen=Sk, sm_scale=SM, kv_limit_dense=Sk,
                                    return_lse=True)
        assert torch.allclose(ref["lse"], torch.cat([lse[m][h] for m in range(nq)])[:Sq], rtol=0, atol=1e-12)
        E, _ = R.elem_bound(ref, q.dtype)
        assert ((ok_out[0, :, h].double() - ref["o"]).abs() <= E).all()
        assert ((pad_out[0, :, h].double() - ref["o"]).abs() > E).any()
    _, _, vf = R.flat_case(1, Sk, H, seed=Sk, device="cpu")
    assert not torch.equal(R.dense_expected(vf, Sq), R.dense_expected(vf, Sq, kv_limit=Sp))


# ------------------------------------------------------------------------------------------------
# FP8 P.V
# ------------------------------------------------------------------------------------------------
# the FP8 shapes of the GPU file: (segment key counts, sample amax)
FP8_GPU_CASES = {
    "hy720p_image": ([115380], (8,)),
    "hy720p_text": ([76], (8,)),
    "hy_i2v_image": ([115500], (8,)),
    "wan14b": ([75600], (8,)),
    "wan1.3b": ([32760], (8,)),
    "lse_b2": ([100], (8, 4)),
}


def test_fp8_codes_are_exact_e4m3():
    """fp8_codes matches e4m3_satfinite byte for byte, and on fp8_case's values every code is v * 448 /
    amax exactly (multiples of 56 at amax 8)."""
    _, _, v = R.fp8_case(2, 600, 3, seed=3, device="cpu", amax=(8, 2))
    codes, amax = R.fp8_codes(v)
    assert torch.equal(amax, torch.tensor([[8.0] * 3, [2.0] * 3]))
    inv = torch.tensor(448.0) / amax
    assert torch.equal(e4m3_satfinite(v.float() * inv[:, None, :, None]).view(torch.float8_e4m3fn).float(), codes)
    assert torch.equal(codes, v.float() * inv[:, None, :, None])
    assert torch.equal(codes[0] % 56, torch.zeros_like(codes[0]))
    assert set(v.float().unique().tolist()) <= {0.0, 1.0, -1.0, 2.0, -2.0, 4.0, -4.0, 8.0, -8.0}


def test_fp8_expected_restates_the_epilogue():
    """fp8_expected is round16(fp32(sum codes) * fp32(fp32(1/l) * fp32(amax * fp32(1/448)))), element by
    element in Python floats rounded to fp32 at each step, and lies within 2^-7 relative of fp64."""
    _, _, v = R.fp8_case(2, 300, 2, seed=5, device="cpu", amax=(8, 4))
    got = R.fp8_expected(v, 3)
    codes, amax = R.fp8_codes(v)
    for b in range(2):
        for h in range(2):
            for d in (0, 5, 127):
                num = R.f32(codes[b, :, h, d].double().sum().item())
                inv = R.f32(R.f32(1.0 / R.f32(300.0)) * R.f32(amax[b, h].item() * R.f32(1.0 / 448.0)))
                want = torch.tensor(R.f32(num * inv)).bfloat16()
                assert got[b, 0, h, d] == want
                exact = v[b, :, h, d].double().mean().item()
                assert abs(got[b, 0, h, d].item() - exact) <= 2.0 ** -7 * abs(exact) + 1e-30


@pytest.mark.parametrize("case", list(FP8_GPU_CASES))
def test_fp8_certificate_holds_at_the_gpu_shapes(case):
    keys, amaxes = FP8_GPU_CASES[case]
    _, _, v = R.fp8_case(len(amaxes), keys[0], 4, seed=11, device="cpu", amax=amaxes)
    codes, _ = R.fp8_codes(v)
    assert R.fp8_certified(codes)


def test_fp8_certificate_rejects_dense_rows():
    """Dense |v| = 8 over 115 380 keys: 7 * 115 380 units of 64 per partial sum, far past 2^12; a
    handful of keys more than the certified budget also fails."""
    v = torch.full((1, 115380, 1, D), 8.0).bfloat16()
    codes, _ = R.fp8_codes(v)
    assert R.fp8_cert_ratio(codes) == 7 * 115380
    assert not R.fp8_certified(codes)
    v = torch.zeros(1, 1000, 1, D)
    v[0, :585, 0, 0] = 8.0
    assert R.fp8_certified(R.fp8_codes(v.bfloat16())[0])
    v[0, :586, 0, 0] = 8.0
    assert not R.fp8_certified(R.fp8_codes(v.bfloat16())[0])
