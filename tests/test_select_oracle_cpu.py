"""CPU checks of tests/select_ref.py: the exact restatements agree with fp64 within their stated
bounds, the selection oracle reproduces the reference builder, and its ambiguity flags fire
where the fp32 arithmetic really is undecided (and only there)."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / "golden"))
sys.path.insert(0, str(HERE))
import synth  # noqa: E402
import select_ref as sr  # noqa: E402

from test_oracle_cpu import assert_masks_equal_modulo_ties  # noqa: E402


def _ref_scores(c):
    """The reference restatement's pooled scores (oracle.attention_oracle.build_block_onehot)."""
    from oracle import attention_oracle as orc
    q = c["q"][:, :, :c["n_img"] * 128]
    k = c["k"]
    dt, D = q.dtype, q.shape[-1]
    B, H = q.shape[:2]
    qp = orc._round_like(q.float().reshape(B, H, -1, 128, D).mean(dim=-2), dt)
    kp = orc._round_like(k.float().reshape(B, H, -1, 128, D).mean(dim=-2), dt)
    s = orc._round_like(qp @ kp.transpose(-1, -2), dt)
    s = orc._round_like(s * torch.tensor(D ** -0.5, dtype=torch.float32), dt)
    return s[..., :c["n_img"]]


def _counts_matching(sel, onehot):
    """Per row, the count n in the allowed set with bits_for(n) == onehot's packed row (-1: none)."""
    want = sr.pack_bits(onehot.reshape(-1, onehot.shape[-1]), sel.words)
    found = torch.full((want.shape[0],), -1, dtype=torch.long)
    for off in range(int((sel.count_hi - sel.count_lo).max()) + 1):
        n = (sel.count_lo + off).clamp(max=sel.count_hi)
        hit = (sel.bits_for(n) == want).all(-1) & (found < 0)
        found[hit] = n[hit]
    return found


@pytest.mark.parametrize("name", [n for n, *_ in synth.MASK_CASES])
def test_select_oracle_reproduces_reference_builder(name):
    from oracle import attention_oracle as orc
    gold = np.load(HERE / "golden" / "mask_builder.npz")
    c = synth.mask_case(name)
    n_img, nb = c["n_img"], c["n_img"] + c["n_txt"]
    low, probs = orc.build_block_onehot(c["q"][:, :, :n_img * 128], c["k"], c["top_k"], n_img, nb, c["p"],
                                        c["n_txt"], c["nbr"], c["ff"], tie_break="low", return_probs=True)
    nbr = sr.pack_bits(c["nbr"], (nb + 31) // 32) if c["nbr"] is not None else None
    sel = sr.select_oracle(_ref_scores(c), n_img, nb, c["top_k"], c["p"], c["n_txt"], c["ff"], nbr)
    found = _counts_matching(sel, low)
    split = sel.tie_split(found.clamp(min=1))
    assert ((found >= 0) | split).all(), int(((found < 0) & ~split).sum())
    # fp32 vs fp64 cut: the count is certain on almost every row
    assert (sel.count_lo == sel.count_hi).float().mean() >= 0.95
    mine = sr.unpack_bits(sel.bits_for(found.clamp(min=1)), nb).view(low.shape)
    ref = torch.from_numpy(gold[name + "/mask"])
    assert_masks_equal_modulo_ties(mine, ref, probs, n_img)


def test_select_oracle_on_random_rows_matches_fp32_builder():
    """Larger random rows with duplicated blocks (exact ties straddling the cut) and clipped
    first-frame / text unions: the fp32 builder's mask is bits_for(n) for an allowed n."""
    from oracle import attention_oracle as orc
    g = torch.Generator().manual_seed(7)
    H, n_img, n_txt, ff = 3, 200, 3, 5
    nb = n_img + n_txt
    q = (torch.randn(1, H, n_img * 128, 128, generator=g) + 0.3).bfloat16()
    k = (torch.randn(1, H, nb * 128, 128, generator=g) + 0.3).bfloat16()
    k.view(1, H, nb, 128, 128)[:, :, 1:n_img:4] = k.view(1, H, nb, 128, 128)[:, :, 0:n_img - 1:4]
    c = dict(q=q, k=k, n_img=n_img)
    for top_k, p in ((1, 0.3), (17, 0.05), (n_img, 0.9), (0, 1.5)):
        low = orc.build_block_onehot(q, k, top_k, n_img, nb, p, n_txt, None, ff)
        sel = sr.select_oracle(_ref_scores(c), n_img, nb, top_k, p, n_txt, ff)
        found = _counts_matching(sel, low)
        assert (found >= 0).all(), (top_k, p, int((found < 0).sum()))


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_pool_exact_within_fp64_bound(dt):
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(2, 3 * 128 + 37, 3, 64, generator=g) * 2 + 0.5)
    x[:, :, 1] *= 1e-3  # small-magnitude head: checked per element, not against the global max
    x = x.to(dt)
    got = sr.pool_exact(x, 4)
    mean, amean = sr.pool_fp64(x, 4)
    sr.assert_pool_certified(got, mean, amean, str(dt))
    # the bound is per element: one ulp off on the small head fails it
    bad = got.clone()
    bad[0, 1, 0, 0] = (bad[0, 1, 0, 0].float() + sr.ulp(bad[0, 1, 0, 0], dt).float()).to(dt)
    with pytest.raises(AssertionError):
        sr.assert_pool_certified(bad, mean, amean)


def test_pool_exact_fp32_input_is_rounded_to_bf16_first():
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, 300, 2, 16, generator=g) * 3
    got = sr.pool_exact(x, 3)
    assert got.dtype == torch.bfloat16
    assert torch.equal(got, sr.pool_exact(x.bfloat16(), 3))


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_scores_exact_within_certified_set(dt):
    g = torch.Generator().manual_seed(5)
    qp = (torch.randn(2, 3, 70, 128, generator=g) * 0.7).to(dt)
    kp = (torch.randn(2, 3, 90, 128, generator=g) * 0.7).to(dt)
    s = sr.scores_exact(qp, kp, 80)
    exact, lo, hi, amb = sr.scores_certified(qp, kp, 80)
    assert s.shape == (6, 70, 80)
    assert ((s >= lo) & (s <= hi)).all()
    assert amb.float().mean() < 0.75
    # the certified set is tight: the fp64 value rounded the same way is in it, and (away from
    # ambiguous elements) it is a single value
    r = (sr.round_fp64(exact, dt).float() * sr._scale(128, "cpu")).to(dt).float()
    assert torch.equal(r[~amb], s[~amb])


def test_round_fp64_is_one_rounding():
    g = torch.Generator().manual_seed(6)
    for dt, e0, e1 in ((torch.bfloat16, -140, 20), (torch.float16, -30, 14)):
        x = torch.randn(100000, generator=g) * torch.exp2(torch.randint(e0, e1, (100000,), generator=g).float())
        want = x.to(dt).double()  # fp32 -> 16-bit: a single rounding
        assert torch.equal(sr.round_fp64(x.double(), dt), want)


# ------------------------------------------------------------------ ambiguity machinery
def test_cut_exactly_at_p_is_count_ambiguous():
    s = torch.tensor([[[0.5, 0.5, -30.0, -30.0]]])  # probs ~ 0.5, 0.5, 0, 0: C = 0.5, 1.0
    sel = sr.select_oracle(s, 4, 4, 0, 0.5, 0, 0)
    assert sel.count_lo.tolist() == [1] and sel.count_hi.tolist() == [2]
    fr_count, _ = sel.check(sel.bits_for(torch.tensor([2])), torch.tensor([2]))
    assert fr_count == 1.0
    sel.check(sel.bits_for(torch.tensor([1])), torch.tensor([1]))
    with pytest.raises(AssertionError):
        sel.check(sel.bits_for(torch.tensor([3])), torch.tensor([3]))
    # away from p the count is exact
    sel = sr.select_oracle(s, 4, 4, 0, 0.3, 0, 0)
    assert sel.count_lo.tolist() == sel.count_hi.tolist() == [1]


def test_one_ulp_apart_scores_are_a_near_tie_at_the_cut():
    x = 2.0 ** -20
    nxt = x + float(sr.ulp(torch.tensor(x), torch.bfloat16))
    assert float(torch.tensor(nxt).bfloat16()) == nxt > x
    # block 3 scores one bf16 ulp above block 1: fp64 ranks 3 first, fp32 may tie them (index order)
    s = torch.tensor([[[-40.0, x, -40.0, nxt, -40.0]]])
    sel = sr.select_oracle(s, 5, 5, 1, 0.0, 0, 0)
    assert sel.count_lo.tolist() == sel.count_hi.tolist() == [1]
    assert sel.order[0, :2].tolist() == [3, 1]
    n = torch.tensor([1])
    assert sel.tie_split(n).tolist() == [True]
    for blk in (1, 3):  # either member of the near-tie group is accepted
        bits = torch.tensor([[1 << blk]], dtype=torch.int32)
        _, fr_tie = sel.check(bits, n)
        assert fr_tie == 1.0
    with pytest.raises(AssertionError):
        sel.check(torch.tensor([[1 << 0]], dtype=torch.int32), n)
    # a real gap is not a near tie
    s2 = torch.tensor([[[-40.0, 0.25, -40.0, 0.5, -40.0]]])
    sel2 = sr.select_oracle(s2, 5, 5, 1, 0.0, 0, 0)
    assert sel2.tie_split(n).tolist() == [False]
    with pytest.raises(AssertionError):
        sel2.check(torch.tensor([[1 << 1]], dtype=torch.int32), n)


def test_exact_ties_are_taken_in_index_order_and_are_not_ambiguous():
    s = torch.tensor([[[1.0, 2.0, 1.0, 2.0, 1.0, 2.0]]])
    sel = sr.select_oracle(s, 6, 6, 2, 0.0, 0, 0)
    assert sel.order[0].tolist() == [1, 3, 5, 0, 2, 4]
    assert sel.tie_split(torch.tensor([2])).tolist() == [False]
    sel.check(torch.tensor([[(1 << 1) | (1 << 3)]], dtype=torch.int32), torch.tensor([2]))
    with pytest.raises(AssertionError):
        sel.check(torch.tensor([[(1 << 1) | (1 << 5)]], dtype=torch.int32), torch.tensor([2]))


def test_zero_probabilities_tie_in_index_order_subnormals_keep_their_order():
    # probabilities e^(s - 100): block 2 ~ e^-95 (fp32 subnormal), block 4 ~ e^-96 (subnormal),
    # blocks 0, 1, 3 ~ e^-120 and below (certainly +0 in fp32)
    s = torch.tensor([[[-20.0, -30.0, 5.0, -25.0, 4.0, 100.0]]])
    sel = sr.select_oracle(s, 6, 6, 5, 0.0, 0, 0)
    assert sel.order[0].tolist() == [5, 2, 4, 0, 1, 3]
    assert sel.tie_split(torch.tensor([5])).tolist() == [False]
    assert sel.tie_split(torch.tensor([3])).tolist() == [False]


def test_unions_and_padding():
    s = torch.zeros(1, 3, 40)
    s[..., 7] = 10.0
    nbr = torch.full((2, 3), -1, dtype=torch.int32)  # garbage past n_img and past nb; 2 rows < nq
    sel = sr.select_oracle(s, 40, 70, 1, 0.0, 100, 2, nbr, nbr_rows=2, nbr_words=1)
    oh = sr.unpack_bits(sel.bits_for(torch.ones(3, dtype=torch.long)), 96)
    assert oh[:, 70:].sum() == 0  # nothing at or past nb
    assert oh[:, 40:70].all()  # text clipped to nb
    assert oh[0, :32].all() and oh[1, :32].all() and not oh[0, 32:40].any()  # one neighbour word
    assert oh[2, :40].nonzero().flatten().tolist() == [7]  # no neighbour row, m >= ff
    sel = sr.select_oracle(s, 40, 70, 1, 0.0, 0, 75)  # first frame past nb: clipped to nb, every row < ff
    oh = sr.unpack_bits(sel.bits_for(torch.ones(3, dtype=torch.long)), 96)
    assert oh[:, :70].all() and not oh[:, 70:].any()
