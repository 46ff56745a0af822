"""The restatements of tests/attn_ref.py, checked without a GPU: the exact flat-case value against the CPU
oracle, the fp64 rows against refutil.fp64_truth, the 24-bit certificate at every production block
count, and the per-element bound E against the oracle and against outputs corrupted the ways a kernel
goes wrong."""
import math
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
import attn_ref as R  # noqa: E402
import refutil  # noqa: E402
from test_attn_edges_gpu import REGIMES, STAIR_TEXT_START, _oracle, _staircase  # noqa: E402

BLOCK = D = 128
SM = D ** -0.5
WORKLOADS = ["hy720p", "hy_turbo_s0", "hy_i2v", "wan14b", "wan1.3b"]


def _rand_live(B, H, nq, nb, seed, p=0.3, text_blocks=0, garbage=False):
    """[B, H, nq, words] int32 mask bits: random live blocks, every row with at least one image block,
    text blocks always on (as the selection sets them); with garbage, bits past nb set too."""
    g = torch.Generator().manual_seed(seed)
    words = (nb + 31) // 32
    oh = torch.rand(B, H, nq, words * 32, generator=g) < p
    oh[..., nb:] = garbage
    oh[..., 0] |= ~oh[..., :nb - text_blocks].any(-1)
    if text_blocks:
        oh[..., nb - text_blocks:nb] = True
    full = (oh.view(B, H, nq, words, 32).long() << torch.arange(32)).sum(-1)
    return torch.where(full >= 2 ** 31, full - 2 ** 32, full).to(torch.int32)


def _oracle_flat(q, k, v, live, nq_sparse, nq_dense, *, seqlen, text_amp, text_start):
    return _oracle(q, k, v, live, nq_sparse, nq_dense, seqlen=seqlen, kv_limit_dense=None, text_amp=float(text_amp),
                   text_start=text_start)


# (B, nb key blocks, text blocks, dtype, seqlen short of nb * 128, out fp32, garbage bits past nb)
FLAT_CASES = {
    "three_words": (1, 70, 2, torch.bfloat16, 0, False, False),
    "garbage_past_nb": (1, 70, 2, torch.bfloat16, 0, False, True),
    "limits_mid_block": (1, 70, 2, torch.bfloat16, 200, False, True),
    "batch2": (2, 40, 2, torch.bfloat16, 76, False, False),
    "fp16": (1, 36, 4, torch.float16, 300, False, False),
    "fp32_out": (1, 40, 0, torch.bfloat16, 8, True, False),
}


@pytest.mark.parametrize("case,amp", [(c, a) for c in FLAT_CASES for a in R.FLAT_AMPS
                                      if FLAT_CASES[c][2] or a == 0])
def test_flat_expected_equals_the_oracle(case, amp):
    """flat_expected (the kernel's epilogue restated on exact sums) equals the CPU oracle bit for bit:
    multi-word masks, bits past nb, a sequence limit inside a block (rows and keys), every text_amp of
    Leg A, B = 2, fp16, and the fp32-widened output."""
    B, nb, T, dtype, short, f32_out, garbage = FLAT_CASES[case]
    H, S = 2, nb * BLOCK
    ns, nd = nb - T, T
    seqlen = S - short
    q, k, v = R.flat_case(B, S, H, seed=11 + nb, device="cpu", dtype=dtype)
    bits = _rand_live(B, H, ns, nb, seed=nb, text_blocks=T, garbage=garbage)
    live = R.unpack(bits, nb)
    assert R.flat_certified(nb, T, amp)
    got = R.flat_expected(v, live, nq_sparse=ns, nq_dense=nd, q_rows=S, text_amp=amp, text_block_start=ns,
                          kv_limit_sparse=seqlen, q_limit_sparse=seqlen, kv_limit_dense=None,
                          out_dtype=torch.float32 if f32_out else None)
    want = _oracle_flat(q, k, v, live, ns, nd, seqlen=seqlen, text_amp=amp, text_start=ns)
    if f32_out:
        want = want.float()
    assert got.dtype == want.dtype
    # The kernel multiplies by the reciprocal where the oracle divides: where num / l is a midpoint of
    # the 16-bit grid (or within 2^-20 of one, where fp32 rounding decides), the division rounds to even
    # and fp32(num) * fp32(1 / l) may land on the other side.  Everywhere else the two are bit-identical.
    tie = _ties(v, live, ns, nd, S, amp, seqlen)
    assert torch.equal(got[~tie], want[~tie])
    assert int(tie.sum()) <= got.numel() // 50
    # the value is the flat sum itself: rows of one block are equal, and zero past the limit
    assert torch.equal(got[:, :BLOCK], got[:, :1].expand_as(got[:, :BLOCK]))
    if short:
        assert not got[:, seqlen:ns * BLOCK].any()


def _ties(v, live, ns, nd, S, amp, seqlen):
    """[B, S, H, D] bool: elements whose exact value num / l lies within 2^-20 (relative) of a midpoint
    between two 16-bit values (torch rounds fp64 to 16 bits through fp32)."""
    num, l, _ = R.flat_num_l(v, live, nq_sparse=ns, nq_dense=nd, text_amp=amp, text_block_start=ns,
                             kv_limit_sparse=seqlen)
    x = num / l[..., None]
    nudge = x.abs() * 2.0 ** -20
    tie = (x + nudge).to(v.dtype) != (x - nudge).to(v.dtype)
    rows = tie.repeat_interleave(BLOCK, dim=2)[:, :, :S].transpose(1, 2)
    written = (torch.arange(S) < seqlen) | (torch.arange(S) >= ns * BLOCK)
    return rows & written[None, :, None, None]


def test_flat_expected_zeros_empty_rows_and_counts_padding_keys():
    """A block with no live tile is zeros (the oracle would divide by zero there), and dense rows count
    the zero-filled keys of a ragged last block in l."""
    S, H, nb = 3 * BLOCK - 56, 1, 3
    q, k, v = R.flat_case(1, S, H, seed=3, device="cpu")
    live = torch.tensor([[[[True, False, True], [False, False, False]]]])
    got = R.flat_expected(v, live, nq_sparse=2, nq_dense=1, q_rows=S)
    assert not got[:, BLOCK:2 * BLOCK].any()
    vd = v[0, :, 0].double()
    want_dense = (vd.sum(0).float() * (1.0 / torch.tensor(3 * BLOCK, dtype=torch.float32))).to(v.dtype)
    assert torch.equal(got[0, 2 * BLOCK:, 0], want_dense.expand(S - 2 * BLOCK, D))
    want0 = (vd[:BLOCK].sum(0) + vd[2 * BLOCK:].sum(0)).float() * (1.0 / torch.tensor(S - BLOCK, dtype=torch.float32))
    assert torch.equal(got[0, 0, 0], want0.to(v.dtype))


@pytest.mark.parametrize("name", WORKLOADS)
def test_flat_certificate_holds_at_production_block_counts(name):
    import bench
    wl = bench.workload(name, 0.7)
    t, h, w = wl["grid"]
    nb = (t * h * w + wl["text_tokens"] + BLOCK - 1) // BLOCK
    amps = R.FLAT_AMPS if wl["text_blocks"] else (0,)
    for a in amps:
        assert R.flat_certified(nb, wl["text_blocks"], a), (name, a)
    bits = R.flat_exact_bits((nb - wl["text_blocks"]) * BLOCK, wl["text_blocks"] * BLOCK, max(amps))
    assert bits <= 22.0, bits
    # a construction that breaks it: |v| up to 2^10
    assert not R.flat_certified(nb, wl["text_blocks"], 0, v_max=2 ** 10)


def test_flat_certificate_edge():
    """The certificate is tight where it should be: 2^24 / 8 keys of weight 1 fit, one more does not."""
    assert R.flat_exact_bits(2 ** 21, 0, 0) == 24.0
    assert R.flat_exact_bits(2 ** 21 + 1, 0, 0) > 24.0
    assert R.flat_exact_bits(100, 128, -2) == pytest.approx(math.log2(8 * (100 + 32) * 4))


# ------------------------------------------------------------------------------------------------
# Leg B restatements
# ------------------------------------------------------------------------------------------------
def _real_case(B=1, H=2, nb=20, T=2, seed=5, dtype=torch.bfloat16, short=0, amp=0.431, sigma=1.0):
    g = torch.Generator().manual_seed(seed)
    S = nb * BLOCK - short
    q = (torch.randn(B, S, H, D, generator=g) * sigma).to(dtype)
    k = (torch.randn(B, S, H, D, generator=g) * sigma).to(dtype)
    v = torch.randn(B, S, H, D, generator=g).to(dtype)
    live = R.unpack(_rand_live(B, H, nb - T, nb, seed, text_blocks=T), nb)
    return q, k, v, live, S, nb - T, amp


def test_fp64_rows_equals_fp64_truth():
    """Sparse rows of fp64_rows are fp64_truth evaluated on the kernel's Q~ with the scores already in
    log2 units (sm_scale = ln 2); dense rows are fp64_truth on the raw q.  Limits inside a block."""
    q, k, v, live, S, ns, amp = _real_case(short=40)
    seqlen = S - 100
    nb = live.shape[-1]
    for h in range(q.shape[2]):
        ref = R.fp64_rows(q, k, v, live, b=0, h=h, qblocks=range(nb), nq_sparse=ns, sm_scale=SM, text_amp=amp,
                          text_block_start=ns, kv_limit=seqlen, q_limit=seqlen, chunk=3)
        qt = (q.float() * R.qk_scale32(SM)).to(q.dtype).double()
        t_sp = refutil.fp64_truth(qt, k, v, live, list(range(ns)), n_img_blocks=ns, seqlen=seqlen, sm_scale=math.log(2.0),
                                  text_amp=R.f32(amp), text_block_start=ns, q_limit=seqlen)
        t_dn, lse = refutil.fp64_truth(q, k, v, live, list(range(ns, nb)), n_img_blocks=ns, seqlen=seqlen, sm_scale=SM,
                                       return_lse=True)
        want = torch.cat([t_sp[m][h] for m in range(ns)] + [t_dn[m][h] for m in range(ns, nb)])[:S]
        assert ref["o"].shape == (S, D)
        assert torch.allclose(ref["o"], want, rtol=0, atol=1e-12)
        want_lse = torch.cat([lse[m][h] for m in range(ns, nb)])[:S - ns * BLOCK]
        assert torch.allclose(ref["lse"][ns * BLOCK:], want_lse, rtol=0, atol=1e-12)
        assert ref["zero"][seqlen:ns * BLOCK].all() and not ref["zero"][:seqlen].any()
        assert (ref["a"] >= ref["o"].abs() - 1e-12).all()


def _lazy_kernel(q, k, v, live, ns, nd, *, seqlen, text_amp, text_start, corrupt=None):
    """The consumer loop in fp32 (torch) with the kernel's lazy rescale (threshold 8), P rounded to the
    input dtype, l over the unrounded p, and the epilogue's o * (1 / l) -- or one of its corruptions:
    'no_o_rescale' (alpha applied to l only), 'amp_early' (text_amp from text_start - 1), 'drop_tile'
    (the last live tile of every sparse row that holds an unmasked key skipped)."""
    dt = q.dtype
    B, S, H, _ = q.shape
    nb = (k.shape[1] + BLOCK - 1) // BLOCK
    kp, vp = (refutil.pad_rows(x, nb * BLOCK).float() for x in (k, v))
    qp = refutil.pad_rows(q, (ns + nd) * BLOCK)
    qks = torch.tensor(R.qk_scale32(SM), dtype=torch.float32)
    out = torch.zeros(B, (ns + nd) * BLOCK, H, D, dtype=dt)
    amp32 = torch.tensor(R.f32(text_amp), dtype=torch.float32)
    for b in range(B):
        for h in range(H):
            for m in range(ns + nd):
                dense = m >= ns
                qm = qp[b, m * BLOCK:(m + 1) * BLOCK, h].float()
                if not dense:
                    if m * BLOCK >= seqlen:
                        continue
                    qm = (qm * qks).to(dt).float()
                    blocks = torch.nonzero(live[b, h, m]).flatten().tolist()
                    if corrupt == "drop_tile":
                        keep = [j for j in blocks if j * BLOCK < seqlen]
                        blocks = keep[:-1] + [j for j in blocks if j * BLOCK >= seqlen]
                else:
                    blocks = list(range(nb))
                mu = torch.full((BLOCK,), float("-inf"))
                l = torch.zeros(BLOCK)
                o = torch.zeros(BLOCK, D)
                start = text_start - 1 if corrupt == "amp_early" else text_start
                for j in blocks:
                    s = qm @ kp[b, j * BLOCK:(j + 1) * BLOCK, h].T
                    ct = qks if dense else torch.tensor(1.0)
                    amp = amp32 if (not dense and j >= start) else torch.tensor(0.0)
                    if not dense:
                        cols = j * BLOCK + torch.arange(BLOCK)
                        s = s.masked_fill(cols[None] >= seqlen, float("-inf"))
                    cand = torch.maximum(mu, s.max(1).values * ct + amp)
                    if bool(((cand - mu) > 8).any()):
                        alpha = torch.where(cand == float("-inf"), torch.ones(()), torch.exp2(mu - cand))
                        l = l * alpha
                        if corrupt != "no_o_rescale":
                            o = o * alpha[:, None]
                        mu = cand
                    off = amp - torch.where(mu == float("-inf"), torch.zeros(()), mu)
                    p = torch.exp2(s * ct + off[:, None])
                    l = l + p.sum(1)
                    o = o + p.to(dt).float() @ vp[b, j * BLOCK:(j + 1) * BLOCK, h]
                res = o * (1.0 / l)[:, None]
                if not dense:
                    res = res.masked_fill((m * BLOCK + torch.arange(BLOCK) >= seqlen)[:, None], 0.0)
                out[b, m * BLOCK:(m + 1) * BLOCK, h] = res.to(dt)
    return out[:, :S]


def _teeth_cases():
    """(name, q, k, v, live, ns, nd, seqlen, amp): a realistic case and the staircase regimes."""
    cases = []
    q, k, v, live, S, ns, amp = _real_case(nb=12, T=2, short=60, amp=3.0, sigma=1.5)
    live[..., ns - 1] = True                                   # the block before the text blocks
    cases.append(("random_amp3", q, k, v, live, ns, 2, S - 100, amp))
    q, k, v, live, S, ns, amp = _real_case(nb=12, T=2, seed=9, dtype=torch.float16, amp=0.431, sigma=2.0)
    live[..., ns - 1] = True
    cases.append(("random_fp16", q, k, v, live, ns, 2, S, amp))
    for regime in ("rise30", "rise8.1", "amp+12"):
        q, k, v, mask, amp = _staircase(regime, torch.bfloat16)
        cases.append((regime, q, k, v, mask, mask.shape[2], q.shape[1] // BLOCK - mask.shape[2], k.shape[1], amp))
    return cases


TEETH = {c[0]: c for c in _teeth_cases()}


def _bound(q, k, v, live, ns, nd, seqlen, amp, text_start):
    B, S, H, _ = q.shape
    nb = (k.shape[1] + BLOCK - 1) // BLOCK
    out = []
    for h in range(H):
        ref = R.fp64_rows(q, k, v, live, b=0, h=h, qblocks=range(ns + nd), nq_sparse=ns, sm_scale=SM, text_amp=amp,
                          text_block_start=text_start, kv_limit=seqlen, q_limit=seqlen,
                          small_p=q.dtype == torch.float16)
        E, _ = R.elem_bound(ref, q.dtype)
        out.append((ref["o"], E))
    return out


def _excess(got, bound):
    """max over heads of max(|got - O*| / E) (inf where E = 0 and got differs)."""
    worst = 0.0
    for h, (o, E) in enumerate(bound):
        err = (got[0, :o.shape[0], h].double() - o).abs()
        worst = max(worst, (err / E).nan_to_num(nan=0.0, posinf=float("inf")).max().item())
    return worst


@pytest.mark.parametrize("name", list(TEETH))
def test_elem_bound_holds_for_the_oracle_and_fails_corruptions(name):
    """The oracle (P rounded as the kernel rounds it) and the lazy-rescale restatement lie within E;
    each corruption exceeds E on at least one element: a live tile dropped, O not rescaled while l is
    (only where the lazy rescale fires after the first tile), text_amp one block early, two rows
    swapped, and the neighbouring head's V."""
    _, q, k, v, live, ns, nd, seqlen, amp = TEETH[name]
    text_start = STAIR_TEXT_START if name in REGIMES else ns
    bound = _bound(q, k, v, live, ns, nd, seqlen, amp, text_start)
    kw = dict(seqlen=seqlen, text_amp=amp, text_start=text_start)
    oracle = _oracle(q, k, v, live, ns, nd, seqlen=seqlen, kv_limit_dense=None, text_amp=amp, text_start=text_start)
    ratio = _excess(oracle, bound)
    assert ratio <= 1.0, ratio
    lazy = _lazy_kernel(q, k, v, live, ns, nd, **kw)
    assert _excess(lazy, bound) <= 1.0
    print(f"{name}: oracle max|err|/E = {ratio:.3f}")
    bad = {"drop_tile": _lazy_kernel(q, k, v, live, ns, nd, corrupt="drop_tile", **kw),
           "amp_early": _lazy_kernel(q, k, v, live, ns, nd, corrupt="amp_early", **kw),
           "swap_rows": oracle[:, torch.arange(oracle.shape[1]) ^ 1],
           "neighbour_head_v": _oracle(q, k, v.roll(1, dims=2), live, ns, nd, seqlen=seqlen, kv_limit_dense=None,
                                       text_amp=amp, text_start=text_start)}
    if name in ("rise30", "rise8.1", "amp+12"):
        bad["no_o_rescale"] = _lazy_kernel(q, k, v, live, ns, nd, corrupt="no_o_rescale", **kw)
    if amp == 0.0:
        del bad["amp_early"]
    for what, out in bad.items():
        assert _excess(out, bound) > 1.0, what
