"""Edge cases of the sm_90a carved-attention kernel (jenga_b200/csrc/carved_attn.cu), through the C-ABI.

The parity tests in test_attn_gpu.py feed N(0,1) inputs over at most 7 key blocks.  These cases go
where this kernel can be wrong without those noticing: the lazy softmax rescale under large and
near-threshold jumps of the running max, the three-word mask walk, the sparse and dense limits
(host and device), strided layouts and per-(batch, head) indexing, the natural-log LSE of the dense
class, and the FP8 P.V path's V^T permutation and scale.

Every case is judged against a plain reference of the same operation: the CPU oracle that rounds
where the reference rounds (oracle/attention_oracle.py, compared with test_attn_gpu.assert_close),
the fp64 truth of tests/refutil.py, or an exact expected value (torch.equal) where the inputs make
the arithmetic exact.
"""
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
import refutil  # noqa: E402
from test_attn_gpu import assert_close  # noqa: E402

BLOCK = D = 128
SM = D ** -0.5
QK = SM * 1.44269504          # scores in log2 units per unit of q.k
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]


def _bits(onehot):
    from jenga_b200.attention import mask_onehot_to_bits
    return mask_onehot_to_bits(onehot.to(DEV))


def _run(q, k, v, bits, nq_sparse, nq_dense, *, kv_limit_dense, text_amp=0.0, text_start=1 << 30,
         kv_limit=None, q_limit=None, out=None):
    """One launch through jenga_carved_attn_fwd with an error flag; inputs are moved to the GPU."""
    from jenga_b200.attention import carved_attention_fwd
    err = torch.zeros(1, dtype=torch.int32, device=DEV)
    o = carved_attention_fwd(q.to(DEV), k.to(DEV), v.to(DEV), bits, nq_sparse=nq_sparse, nq_dense=nq_dense,
                             sm_scale=SM, text_amp=text_amp, text_block_start=text_start,
                             kv_limit_sparse=kv_limit, q_limit_sparse=q_limit, kv_limit_dense=kv_limit_dense,
                             out=out, err_flag=err)
    torch.cuda.synchronize()
    assert err.item() == 0
    return o


def _oracle(q, k, v, onehot, nq_sparse, nq_dense, *, seqlen, kv_limit_dense, text_amp=0.0, text_start=1 << 30):
    """[B,Sq,H,D] from the CPU oracle: sparse q blocks with seqlen as key and row limit, dense q blocks
    over the zero-padded keys below kv_limit_dense."""
    from oracle import attention_oracle as orc
    Sq = q.shape[1]
    nb = (k.shape[1] + BLOCK - 1) // BLOCK
    nq = nq_sparse + nq_dense
    kp, vp = (refutil.pad_rows(x.cpu(), nb * BLOCK).transpose(1, 2) for x in (k, v))
    qp = refutil.pad_rows(q.cpu()[:, :nq * BLOCK], nq * BLOCK).transpose(1, 2)
    parts = []
    if nq_sparse:
        parts.append(orc.carved_attention_rows(qp[:, :, :nq_sparse * BLOCK], kp, vp, onehot.cpu(), seqlen, SM,
                                               text_amp, text_start))
    if nq_dense:
        parts.append(orc.dense_attention_rows(qp[:, :, nq_sparse * BLOCK:], kp, vp, SM, kv_limit_dense))
    return torch.cat(parts, dim=2).transpose(1, 2)[:, :Sq]


def _same_bits(a, b):
    """Bit-identical, NaNs included."""
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(torch.int16 if a.element_size() == 2
                                                                                            else torch.int32),
                                                                     b.contiguous().view(torch.int16 if b.element_size() == 2
                                                                                         else torch.int32))


# ============================================================ 1. lazy rescale and dynamic range
NB_STAIR = 44
# name: (rise of the score max per key tile in log2 units, texture sigma, rows with the staircase, text_amp)
REGIMES = {
    "rise30": (30.0, 1.0, "all", 0.0),
    "rise7.9": (7.9, 0.25, "all", 0.0),
    "rise8.1": (8.1, 0.25, "all", 0.0),
    "fall30": (-30.0, 1.0, "all", 0.0),
    "split_rows30": (30.0, 1.0, "split", 0.0),
    "amp+12": (0.0, 1.0, "all", 12.0),
    "amp-12": (0.0, 1.0, "all", -12.0),
}
STAIR_TEXT_START = NB_STAIR - 4


def _staircase(regime, dtype, H=2, nq_sparse=2, nq_dense=1, seed=0):
    """q/k whose per-row score maximum over key tile j is j * delta (log2 units): channel 127 holds
    q = a and k = 2j (exact in bf16/fp16), the other channels Gaussian texture of the given sigma.
    "split" puts the staircase on the rows with row % 16 in {1,3,5,7} only: in the wgmma accumulator
    layout those are odd lanes' first row (g, not g + 8), so lanes and the two rows of one thread
    disagree on `need`.  Sparse rows of (head h, q block m) walk key tiles [0, 44 - (2h + m) % 3), so
    the rows end on every phase of a rescale cycle; the dense rows walk all 44."""
    delta, sig, rows, amp = REGIMES[regime]
    g = torch.Generator().manual_seed(seed)
    Sq, Sk = (nq_sparse + nq_dense) * BLOCK, NB_STAIR * BLOCK
    q = torch.randn(1, Sq, H, D, generator=g) * sig
    k = torch.randn(1, Sk, H, D, generator=g) * sig
    v = torch.randn(1, Sk, H, D, generator=g)
    j = torch.arange(Sk) // BLOCK
    k[0, :, :, 127] = (2 * (j if delta >= 0 else NB_STAIR - 1 - j)).float()[:, None]
    on = torch.ones(Sq, dtype=torch.bool) if rows == "all" else torch.isin(torch.arange(Sq) % 16, torch.tensor([1, 3, 5, 7]))
    q[0, :, :, 127] = torch.where(on, abs(delta) / (2 * QK), 0.0)[:, None]
    mask = torch.zeros(1, H, nq_sparse, NB_STAIR, dtype=torch.bool)
    for h in range(H):
        for m in range(nq_sparse):
            mask[0, h, m, :NB_STAIR - (h * nq_sparse + m) % 3] = True
    return q.to(dtype), k.to(dtype), v.to(dtype), mask, amp


def _stair_launch(q, k, v, mask, amp, v_fp8=None):
    from jenga_b200.attention import _launch
    Sq, Sk = q.shape[1], k.shape[1]
    out = torch.empty(q.shape, dtype=q.dtype, device=DEV)
    _launch(q.to(DEV), k.to(DEV), v.to(DEV), _bits(mask), mask.shape[2], Sq // BLOCK - mask.shape[2], SM, amp,
            STAIR_TEXT_START, Sk, Sq, Sk, out, None, q.dtype, v_fp8=v_fp8)
    torch.cuda.synchronize()
    return out


def _stair_truth(q, k, v, mask, amp):
    nq = q.shape[1] // BLOCK
    return refutil.fp64_truth(q.to(DEV), k.to(DEV), v.to(DEV), mask.to(DEV), list(range(nq)), n_img_blocks=mask.shape[2],
                              seqlen=k.shape[1], text_amp=amp, text_block_start=STAIR_TEXT_START)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("regime", list(REGIMES))
def test_lazy_rescale_regimes_match_oracle_and_fp64(regime, dtype):
    """44 live key tiles (the two-slot ring wraps 22 times) with the running max rising by 30, 7.9
    or 8.1 log2 units per tile, falling by 30 (later tiles underflow), rising on a subset of rows
    only, or jumping by text_amp = +-12 on the text key blocks: the regimes where the lazy rescale
    (rescale o and l only when the max grew by more than 8) fires partway through a row, or just
    does not.  Sparse and dense classes in one launch.
    Bounds: assert_close against the oracle (which rescales exactly on every tile); and against
    fp64 truth the kernel's error is at most 1.5x (max) / 1.25x (mean) the oracle's own, the rule of
    test_reference_gpu.py: a lazy rescale changes only the reference point P is rounded against,
    so the kernel is no further from the exact result than the per-tile rescale is."""
    q, k, v, mask, amp = _staircase(regime, dtype)
    got = _stair_launch(q, k, v, mask, amp)
    ref = _oracle(q, k, v, mask, 2, 1, seqlen=k.shape[1], kv_limit_dense=k.shape[1], text_amp=amp,
                  text_start=STAIR_TEXT_START)
    assert_close(got, ref, dtype)
    truth = _stair_truth(q, k, v, mask, amp)
    o_max, o_mean, _ = refutil.error_stats(ref.to(DEV), truth)
    p_max, p_mean, _ = refutil.error_stats(got, truth)
    print(f"\n[{regime} {dtype}] vs fp64: oracle {o_max:.2e}/{o_mean:.2e} kernel {p_max:.2e}/{p_mean:.2e}")
    assert p_max <= 1.5 * o_max + 1e-4 and p_mean <= 1.25 * o_mean + 1e-5, (o_max, o_mean, p_max, p_mean)


def test_long_chain_is_deterministic():
    """Two launches of the 44-tile rise-by-30 case are bit-identical: nothing in the kernel (ring
    order, warp-group interleaving, the rescale vote) may depend on timing."""
    q, k, v, mask, amp = _staircase("rise30", torch.bfloat16)
    a = _stair_launch(q, k, v, mask, amp)
    b = _stair_launch(q, k, v, mask, amp)
    assert _same_bits(a, b)


def test_fp8_pv_near_threshold_staircase_against_fp64():
    """FP8 P.V with the score max rising by 7.9 log2 units per tile: P reaches ~2^7.9 between rescales,
    which e4m3 (max 448) holds only because the lazy threshold is 8.  Were the threshold ever raised
    past log2(448) ~ 8.8 (at 16, P reaches 2^15.8 on every third tile and saturates), rows ending on
    such a tile lose most of their weight.  Bound: the FP8 tolerance row of test_fp8_gpu.py against
    fp64 truth (mean <= 6e-2, max <= 0.35 of the output RMS)."""
    from jenga_b200.attention import quantize_v_fp8
    q, k, v, mask, amp = _staircase("rise7.9", torch.bfloat16)
    got = _stair_launch(q, k, v, mask, amp, v_fp8=quantize_v_fp8(v.to(DEV)))
    f_max, f_mean, _ = refutil.error_stats(got, _stair_truth(q, k, v, mask, amp))
    print(f"\n[fp8 rise7.9] vs fp64: max {f_max:.2e} mean {f_mean:.2e}")
    assert f_mean <= 6e-2 and f_max <= 0.35, (f_max, f_mean)


# ============================================================ 2. mask-word walk
def _normal(shape_q, shape_k, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape_q, generator=g).to(dtype), torch.randn(*shape_k, generator=g).to(dtype),
            torch.randn(*shape_k, generator=g).to(dtype))


@pytest.mark.parametrize("dtype", DTYPES)
def test_mask_walk_across_three_words(dtype):
    """70 key blocks: three mask words, the last holding 6 valid bits.  Rows select exactly the
    blocks on both sides of each word boundary {0, 31, 32, 63, 64, 69}, a single block (first, last,
    either side of a boundary), all 70, or a random 30 %; a dense q block walks all 70 too.
    Bound: assert_close against the oracle, which walks the one-hot row in ascending order."""
    H, NB = 2, 70
    q, k, v = _normal((1, 6 * BLOCK, H, D), (1, NB * BLOCK, H, D), dtype, 11)
    g = torch.Generator().manual_seed(12)
    mask = torch.zeros(1, H, 5, NB, dtype=torch.bool)
    mask[0, :, 0, [0, 31, 32, 63, 64, 69]] = True
    mask[0, 0, 1, 69] = mask[0, 1, 1, 32] = True
    mask[0, 0, 2, 0] = mask[0, 1, 2, 31] = True
    mask[0, :, 3] = True
    mask[0, :, 4] = torch.rand(H, NB, generator=g) < 0.3
    mask[0, :, 4, 4] = True
    Sk = NB * BLOCK
    got = _run(q, k, v, _bits(mask), 5, 1, kv_limit_dense=Sk)
    assert_close(got, _oracle(q, k, v, mask, 5, 1, seqlen=Sk, kv_limit_dense=Sk), dtype)


def test_oversized_mask_words_ignore_bits_past_the_last_block():
    """A caller may pass mask rows wider than ceil(nb/32) words.  Bits at or past nb_kv = 70 (the
    rest of word 2, and words 3..4 here, filled with random garbage) must be ignored, and row
    (b, h, m) must be read at stride mask_words: the output is bit-identical to the launch with the
    clean 3-word mask, for every row of 2 batches x 3 heads x 3 q blocks."""
    B, H, NQ, NB = 2, 3, 3, 70
    q, k, v = _normal((B, NQ * BLOCK, H, D), (B, NB * BLOCK, H, D), torch.bfloat16, 21)
    g = torch.Generator().manual_seed(22)
    mask = torch.rand(B, H, NQ, NB, generator=g) < 0.4
    for m in range(NQ):
        mask[:, :, m, 33 * m] = True
    clean = _bits(mask)
    assert clean.shape[-1] == 3
    big = torch.randint(-2 ** 31, 2 ** 31 - 1, (B, H, NQ, 5), generator=g, dtype=torch.int32).to(DEV)
    big[..., :3] = clean
    big[..., 2] |= ~((1 << (NB - 64)) - 1)                 # every bit of keys 70..95
    Sk = NB * BLOCK
    want = _run(q, k, v, clean, NQ, 0, kv_limit_dense=Sk)
    got = _run(q, k, v, big, NQ, 0, kv_limit_dense=Sk)
    assert _same_bits(got, want)
    assert_close(want, _oracle(q, k, v, mask, NQ, 0, seqlen=Sk, kv_limit_dense=Sk), torch.bfloat16)


def test_all_zero_sparse_row_gives_exact_zeros():
    """A sparse q block with an empty mask row runs no tile: the kernel writes exact zeros (and
    everything else stays finite and correct).  Not a parity case: the reference would compute
    0/0 there, but selection always keeps at least one block per row."""
    H, NB = 2, 5
    q, k, v = _normal((1, 3 * BLOCK, H, D), (1, NB * BLOCK, H, D), torch.bfloat16, 31)
    mask = torch.ones(1, H, 3, NB, dtype=torch.bool)
    mask[0, 1, 1] = False
    Sk = NB * BLOCK
    got = _run(q, k, v, _bits(mask), 3, 0, kv_limit_dense=Sk)
    assert torch.isfinite(got.float()).all()
    assert (got[0, BLOCK:2 * BLOCK, 1] == 0).all()
    ref = _oracle(q, k, v, mask, 3, 0, seqlen=Sk, kv_limit_dense=Sk)
    live = torch.ones(3 * BLOCK, H, dtype=torch.bool)
    live[BLOCK:2 * BLOCK, 1] = False
    assert_close(got[0][live], ref[0][live], torch.bfloat16)


# ============================================================ 3. limits
LIMITS = {"inside_key_block": 5 * BLOCK + 37, "block_boundary": 3 * BLOCK, "inside_q_block": 2 * BLOCK + 50}


@pytest.mark.parametrize("name", list(LIMITS))
def test_sparse_limits_host_and_device(name):
    """One limit L serves as kv_limit_sparse and q_limit_sparse (HunyuanVideo's seqlen): inside a
    key block, on a block boundary (q blocks at or past it are skipped whole), inside a q block.
    Every row also walks blocks 7 and 9, which lie wholly past L, so fully masked tiles come after
    the straddling one; head 2's q block 1 walks only those two, so its every tile is masked.
    - seqlen_dev = L (with the host limits left at the full length) gives bit-identical output to
      the host limits, NaNs included, dense q block included;
    - sparse rows >= L are exact zeros;
    - the rest matches the oracle (assert_close).  The row with no key below L is 0/0 in the
      reference (its running max stays -inf) and NaN in the kernel: the NaN pattern must agree."""
    from jenga_b200.attention import _launch
    L = LIMITS[name]
    H, NQS, NB = 3, 7, 10
    Sq, Sk = (NQS + 1) * BLOCK, NB * BLOCK
    q, k, v = _normal((1, Sq, H, D), (1, Sk, H, D), torch.bfloat16, 41)
    g = torch.Generator().manual_seed(42)
    mask = torch.rand(1, H, NQS, NB, generator=g) < 0.5
    mask[..., [0, 5, 7, 9]] = True
    mask[0, 2, 1] = False
    mask[0, 2, 1, [7, 9]] = True
    bits = _bits(mask)
    qd, kd, vd = q.to(DEV), k.to(DEV), v.to(DEV)
    host = _run(q, k, v, bits, NQS, 1, kv_limit=L, q_limit=L, kv_limit_dense=Sk)
    dev_out = torch.empty_like(host)
    _launch(qd, kd, vd, bits, NQS, 1, SM, 0.0, 1 << 30, Sk, Sq, Sk, dev_out,
            torch.tensor([L], dtype=torch.int32, device=DEV), torch.bfloat16)
    torch.cuda.synchronize()
    assert _same_bits(dev_out, host)
    assert (host[0, L:NQS * BLOCK] == 0).all()
    ref = _oracle(q, k, v, mask, NQS, 1, seqlen=L, kv_limit_dense=Sk)
    got = host.cpu()
    assert torch.equal(torch.isnan(got), torch.isnan(ref))
    assert torch.isnan(got[0, BLOCK:2 * BLOCK, 2]).all()
    assert_close(torch.nan_to_num(got), torch.nan_to_num(ref), torch.bfloat16)


@pytest.mark.parametrize("kv_limit", ["at_kv_rows", "past_kv_rows"])
def test_dense_ragged_keys_and_limit_past_the_rows(kv_limit):
    """Dense class only, Sq = 300 and Sk = 9*128 + 40 (neither a multiple of 128), B = 2, H = 3.
    kv_limit_dense = Sk masks the tail of the last tile; kv_limit_dense = 10*128 > Sk attends the
    88 keys that TMA zero-fills past the tensor (score 0, value 0), as the I2V padding does.
    Bounds: assert_close against the oracle on zero-padded keys, and the fp64-truth ratio rule."""
    B, H, Sq, Sk = 2, 3, 300, 9 * BLOCK + 40
    lim = Sk if kv_limit == "at_kv_rows" else 10 * BLOCK
    q, k, v = _normal((B, Sq, H, D), (B, Sk, H, D), torch.bfloat16, 51)
    got = _run(q, k, v, None, 0, 3, kv_limit_dense=lim)
    ref = _oracle(q, k, v, None, 0, 3, seqlen=Sk, kv_limit_dense=lim)
    assert_close(got, ref, torch.bfloat16)
    empty = torch.zeros(B, H, 0, 10, dtype=torch.bool, device=DEV)
    truth = refutil.fp64_truth(q.to(DEV), k.to(DEV), v.to(DEV), empty, [0, 1, 2], n_img_blocks=0, seqlen=Sk,
                               kv_limit_dense=lim)
    o_max, o_mean, _ = refutil.error_stats(ref.to(DEV), truth)
    p_max, p_mean, _ = refutil.error_stats(got, truth)
    assert p_max <= 1.5 * o_max + 1e-4 and p_mean <= 1.25 * o_mean + 1e-5, (o_max, o_mean, p_max, p_mean)


# ============================================================ 4. layouts and indexing
LAYOUT = dict(B=3, H=5, Sq=2 * BLOCK + 72, Sk=5 * BLOCK + 20, NQS=2, NQD=1)
LAYOUT_LIMITS = dict(kv_limit=600, q_limit=200, kv_limit_dense=LAYOUT["Sk"], text_amp=0.431, text_start=4)


@pytest.fixture(scope="module")
def layout_case():
    B, H, Sq, Sk = LAYOUT["B"], LAYOUT["H"], LAYOUT["Sq"], LAYOUT["Sk"]
    q, k, v = (x.to(DEV) for x in _normal((B, Sq, H, D), (B, Sk, H, D), torch.bfloat16, 61))
    g = torch.Generator().manual_seed(62)
    mask = torch.rand(B, H, LAYOUT["NQS"], 6, generator=g) < 0.5
    mask[..., 0] = True
    bits = _bits(mask)
    base = _run(q, k, v, bits, LAYOUT["NQS"], LAYOUT["NQD"], **LAYOUT_LIMITS)
    return q, k, v, mask, bits, base


def _launch_layout(q, k, v, bits, out=None):
    return _run(q, k, v, bits, LAYOUT["NQS"], LAYOUT["NQD"], out=out, **LAYOUT_LIMITS)


def test_layout_base_matches_oracle(layout_case):
    """B = 3, H = 5, q_rows = 328 and kv_rows = 660 (neither a multiple of 128, and different),
    sparse limits inside blocks, text_amp on key blocks >= 4: assert_close against the oracle.  The
    other layout tests compare bit for bit with this launch."""
    q, k, v, mask, bits, base = layout_case
    lim = LAYOUT_LIMITS
    # the oracle has one sparse limit; q block 1 has rows past q_limit = 200, so compare the rows
    # below it with kv_limit as the oracle's seqlen, and check that the rest are zeros
    ref = _oracle(q, k, v, mask, 2, 1, seqlen=lim["kv_limit"], kv_limit_dense=lim["kv_limit_dense"],
                  text_amp=lim["text_amp"], text_start=lim["text_start"])
    rows = torch.cat([torch.arange(lim["q_limit"]), torch.arange(2 * BLOCK, LAYOUT["Sq"])])
    assert_close(base[:, rows], ref[:, rows], torch.bfloat16)
    assert (base[:, lim["q_limit"]:2 * BLOCK] == 0).all()


def test_packed_qkv_views_are_bit_identical(layout_case):
    """q/k/v as views of one packed [B, Sk, 3, H, D] tensor (row stride 3*H*D, q a row-truncated view)."""
    q, k, v, _, bits, base = layout_case
    qkv = torch.zeros(q.shape[0], k.shape[1], 3, q.shape[2], D, dtype=q.dtype, device=DEV)
    qkv[:, :q.shape[1], 0], qkv[:, :, 1], qkv[:, :, 2] = q, k, v
    assert _same_bits(_launch_layout(qkv[:, :q.shape[1], 0], qkv[:, :, 1], qkv[:, :, 2], bits), base)


def test_bhsd_transposed_views_are_bit_identical(layout_case):
    """q/k/v as [B,S,H,D] transposes of contiguous [B,H,S,D] tensors."""
    q, k, v, _, bits, base = layout_case
    qt, kt, vt = (x.transpose(1, 2).contiguous().transpose(1, 2) for x in (q, k, v))
    assert qt.stride(2) != D
    assert _same_bits(_launch_layout(qt, kt, vt, bits), base)


def test_strided_output_view_writes_only_its_elements(layout_case):
    """Output into buf[:, 4:4+Sq, 1:1+H, 32:160] of a larger [B, Sq+9, H+2, 192] buffer: the view
    receives the contiguous launch's bits and every other element (canary) is unchanged."""
    q, k, v, _, bits, base = layout_case
    B, Sq, H, _ = q.shape
    buf = torch.full((B, Sq + 9, H + 2, 192), -3.25, dtype=q.dtype, device=DEV)
    buf[..., 7] = float("nan")
    want = buf.clone()
    view = buf[:, 4:4 + Sq, 1:1 + H, 32:160]
    _launch_layout(q, k, v, bits, out=view)
    want[:, 4:4 + Sq, 1:1 + H, 32:160] = base
    assert _same_bits(buf, want)


def test_each_head_and_each_batch_alone_are_bit_identical(layout_case):
    """Per-(batch, head) indexing: launching one head (a [B,S,1,D] view) or one batch alone gives
    the same bits as that slice of the full launch, so CTA numbering and the mask-row and
    q/k/v/out offsets of every (b, h) are right."""
    q, k, v, _, bits, base = layout_case
    for h in range(q.shape[2]):
        s = slice(h, h + 1)
        got = _launch_layout(q[:, :, s], k[:, :, s], v[:, :, s], bits[:, s].contiguous())
        assert _same_bits(got, base[:, :, s].contiguous()), h
    for b in range(q.shape[0]):
        s = slice(b, b + 1)
        got = _launch_layout(q[s], k[s], v[s], bits[s].contiguous())
        assert _same_bits(got, base[s].contiguous()), b


def test_fp32_output_is_the_16bit_output_widened(layout_case):
    """out_dtype f32: the kernel rounds through the MMA dtype and widens, so out equals base.float()."""
    q, k, v, _, bits, base = layout_case
    out = torch.empty(base.shape, dtype=torch.float32, device=DEV)
    _launch_layout(q, k, v, bits, out=out)
    assert torch.equal(out, base.float())


# ============================================================ 5. LSE of the dense class
@pytest.mark.parametrize("case", ["normal", "rise7.9", "rise30"])
def test_dense_lse_matches_fp64_logsumexp(case):
    """softmax_lse of _flash_attn_forward (natural log, from the kernel's base-2 running max and sum)
    against fp64 logsumexp(s * sm_scale) over the keys below kv_limit_dense = Sk.  "normal": B = 2,
    H = 3, Sq = 300, Sk = 9*128 + 40; the staircases put the running max up to 8 log2 units stale
    (rise7.9) or move it by 30 every tile up to ~1300 log2 units (rise30).
    The dense class rounds nothing before the exponent, so the error is fp32 accumulation of l,
    ex2.approx and log2f (~1e-6 relative), plus the fp32 rounding of m (|m| * 2^-24) and of
    qk_scale: bound 2e-4 + 1e-5 * |lse|.  Measured on an H100 80GB HBM3 (400 W power limit): max
    |err| 9.7e-7 (normal), 2.5e-5 (rise7.9), 1.1e-4 (rise30), at most 1.2 % of the bound."""
    from jenga_b200 import flash_attn_shim as F
    if case == "normal":
        q, k, v = (x.to(DEV) for x in _normal((2, 300, 3, D), (2, 9 * BLOCK + 40, 3, D), torch.bfloat16, 71))
    else:
        q, k, v, _, _ = _staircase(case, torch.bfloat16, nq_sparse=0, nq_dense=2)
        q, k, v = q.to(DEV), k.to(DEV), v.to(DEV)
    _, lse, _, _ = F._flash_attn_forward(q, k, v, softmax_scale=SM)
    torch.cuda.synchronize()
    truth = torch.logsumexp(torch.einsum("bqhd,bkhd->bhqk", q.double(), k.double()) * SM, dim=-1)
    err = (lse.double() - truth).abs()
    bound = 2e-4 + 1e-5 * truth.abs()
    print(f"\n[lse {case}] max|err| {err.max().item():.2e}, max err/bound {(err / bound).max().item():.3f}")
    assert (err <= bound).all(), (err.max().item(), (err / bound).max().item())


# ============================================================ 6. exactness probes of P.V (bf16, fp16, FP8)
NEEDLE_NB = 70
NEEDLE_TILES_SPARSE = [0, 1, 2, 5, 30, 31, 32, 33, 63, 64, 69]   # walk positions 0..10: both ring slots
NEEDLE_TILES_DENSE = [3, 4, 34, 35, 62, 65, 68]                  # tiles the sparse rows never walk


def _needles(dtype, B=2, H=3):
    """One sparse and one dense q block per (b, h).  Row c of a block has query +-32 e_c and its
    needle key has +-32 e_c (dense rows use the minus sign), every other key is zero: the needle
    scores 130 log2 units above every other key of the row, so P is exactly 1 on it and underflows
    to 0 elsewhere.  Needle positions: tile from the list above, offset (37 c + 17 b + 29 h) % 128 —
    every residue mod 128 and 32, different for every (b, h).
    V[b, n, h, d] = (-1)^(bit d%14 of n) * 2^((n + d) % 5) * 2^(b*H + h - 3): unique per key,
    exact in bf16, fp16 and (after the 448 / amax scaling, amax = 16 * 2^(b*H + h - 3)) in e4m3.
    Returns q, k, v, the sparse mask and the expected output V[needle(row)]."""
    Sq, Sk = 2 * BLOCK, NEEDLE_NB * BLOCK
    q = torch.zeros(B, Sq, H, D)
    k = torch.zeros(B, Sk, H, D)
    n = torch.arange(Sk)[:, None]
    d = torch.arange(D)[None, :]
    pattern = torch.where((n >> (d % 14)) & 1 == 1, -1.0, 1.0) * torch.pow(2.0, ((n + d) % 5).float())
    scale = torch.pow(2.0, torch.arange(B * H).float() - 3).reshape(B, 1, H, 1)
    v = pattern[None, :, None, :] * scale
    want = torch.zeros(B, Sq, H, D)
    c = torch.arange(BLOCK)
    for b in range(B):
        for h in range(H):
            for blk, tiles, sgn in ((0, NEEDLE_TILES_SPARSE, 1.0), (1, NEEDLE_TILES_DENSE, -1.0)):
                tile = torch.tensor(tiles)[(c + 5 * b + 3 * h) % len(tiles)]
                key = tile * BLOCK + (37 * c + 17 * b + 29 * h) % BLOCK
                q[b, blk * BLOCK + c, h, c] = 32.0 * sgn
                k[b, key, h, c] = 32.0 * sgn
                want[b, blk * BLOCK + c, h] = v[b, key, h]
    mask = torch.zeros(B, H, 1, NEEDLE_NB, dtype=torch.bool)
    mask[..., NEEDLE_TILES_SPARSE] = True
    return q.to(dtype), k.to(dtype), v.to(dtype), mask, want.to(dtype)


@pytest.mark.parametrize("path", ["bf16", "fp16", "fp8"])
def test_needle_rows_return_their_value_row_exactly(path):
    """Each query row attends one needle key with a margin of 130 log2 units, so its output is
    exactly the needle's V row in every P.V path (torch.equal, no tolerance).  That pins the TMA
    swizzle and the key-to-column mapping, the FP8 V^T key permutation and A-fragment packing, the
    v_fp8_amax (b, h) index and the head-major CTA numbering, at every key residue mod 32 and 128,
    in both ring slots and on both sides of the mask-word boundaries 31|32 and 63|64 (B = 2, H = 3,
    one sparse and one dense q block)."""
    from jenga_b200.attention import _launch, quantize_v_fp8
    dtype = torch.float16 if path == "fp16" else torch.bfloat16
    q, k, v, mask, want = _needles(dtype)
    q, k, v = q.to(DEV), k.to(DEV), v.to(DEV)
    v8 = None
    if path == "fp8":
        v8 = quantize_v_fp8(v)
        assert torch.equal(v8[1].cpu(), 16.0 * torch.pow(2.0, torch.arange(6).float() - 3))
    out = torch.empty(q.shape, dtype=dtype, device=DEV)
    _launch(q, k, v, _bits(mask), 1, 1, SM, 0.0, 1 << 30, k.shape[1], q.shape[1], k.shape[1], out, None, dtype,
            v_fp8=v8)
    torch.cuda.synchronize()
    bad = (out.cpu() != want).any(-1)
    assert not bad.any(), (int(bad.sum()), bad.nonzero()[:8].tolist())
