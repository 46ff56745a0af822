"""Rows that wrap the K/V ring of the sm_90a carved-attention kernel at every phase, in one launch.

carved_attn.cu streams the K and V tiles of a row through a ring of kStages slots: walk position j uses
slot j % kStages and waits on phase (j / kStages) & 1 of that slot's barriers, in the producer, the
consumers and the FP8 V-transpose warps alike.  Every head here has sparse q blocks of 0..8 live tiles
(each slot at each phase of the first passes, and every last slot for a ring of up to 8 stages) and of
40..42 tiles (every parity flips many times), plus a dense q block that walks all 44 key blocks (two mask words).  The
last key block straddles a device-side seqlen.  Sparse rows run Q.K^T on Q pre-scaled by qk_scale and
dense rows on raw Q, both held in the consumers' registers.  Each path is judged against its own
reference: the CPU oracle for bf16 and f16, and fp64 truth on the dequantised operands for INT8 Q.K^T.
Needle rows, whose exact output is one V row, pin the pairing of every tile's P with its V in every
path, FP8 P.V included.  Two launches of the same inputs are bit-identical.
"""
import math
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
import refutil  # noqa: E402
from test_attn_edges_gpu import BLOCK, D, DEV, DTYPES, SM, _bits, _oracle, _same_bits  # noqa: E402
from test_attn_gpu import assert_close  # noqa: E402
from test_qk_int8_cpu import dequantize_ref  # noqa: E402

NB = 44                                   # key blocks (two mask words)
H = 3
COUNTS = list(range(9)) + [40, 41, 42]    # live tiles of the sparse q blocks of every head
NQS = len(COUNTS)
SK = NB * BLOCK
SEQLEN = SK - 70                          # inside the last key block, which every long row walks


def _case(dtype, seed=5):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(1, (NQS + 1) * BLOCK, H, D, generator=g)
    k = torch.randn(1, SK, H, D, generator=g)
    v = torch.randn(1, SK, H, D, generator=g)
    mask = torch.zeros(1, H, NQS, NB, dtype=torch.bool)
    for h in range(H):
        for m, c in zip(torch.randperm(NQS, generator=g).tolist(), COUNTS):   # other q blocks in each head
            if c >= 40:
                mask[0, h, m, NB - 1] = True
                c -= 1
            mask[0, h, m, torch.randperm(NB - 1, generator=g)[:c]] = True
    assert sorted(mask[0, 0].sum(-1).tolist()) == COUNTS
    return q.to(dtype).to(DEV), k.to(dtype).to(DEV), v.to(dtype).to(DEV), mask


def _launch(q, k, v, mask, **kw):
    from jenga_b200.attention import _launch as launch
    out = torch.zeros(q.shape, dtype=q.dtype, device=DEV)
    seq = torch.tensor([SEQLEN], dtype=torch.int32, device=DEV)
    launch(q, k, v, _bits(mask), NQS, 1, SM, 0.0, 1 << 30, SK, q.shape[1], SEQLEN, out, seq, q.dtype, **kw)
    torch.cuda.synchronize()
    return out


def _twice(q, k, v, mask, **kw):
    a = _launch(q, k, v, mask, **kw)
    b = _launch(q, k, v, mask, **kw)
    assert _same_bits(a, b), "two launches differ"
    return a


def _empty_rows(mask):
    """[NQS * BLOCK, H] bool: sparse rows whose q block has no live tile."""
    return (mask[0].sum(-1) == 0).t().repeat_interleave(BLOCK, 0)


def _fp64_errors(got, q, k, v, mask):
    """(max, mean)/RMS of got against fp64 attention of q, k, v over the rows with a live tile; the
    sparse rows without one must be exact zeros."""
    truth = refutil.fp64_truth(q, k, v, mask.to(DEV), list(range(NQS + 1)), n_img_blocks=NQS, seqlen=SEQLEN,
                               kv_limit_dense=SEQLEN)
    e_max, e_sum, cnt, sq = 0.0, 0.0, 0, 0.0
    for b, t in truth.items():
        for h in range(H):
            x = got[0, b * BLOCK:(b + 1) * BLOCK, h].double()
            if b < NQS and not mask[0, h, b].any():
                assert (x == 0).all()
                continue
            e = (x - t[h]).abs()
            e_max, e_sum, cnt, sq = max(e_max, e.max().item()), e_sum + e.sum().item(), cnt + e.numel(), sq + t[h].pow(2).sum().item()
    rms = math.sqrt(sq / cnt)
    return e_max / rms, e_sum / cnt / rms


@pytest.mark.parametrize("dtype", DTYPES)
def test_ring_phases_match_oracle(dtype):
    """Bound: assert_close against the oracle on every row with a live tile; rows without one are exact zeros."""
    q, k, v, mask = _case(dtype)
    got = _twice(q, k, v, mask)[0].cpu()
    empty = _empty_rows(mask)
    assert (got[:NQS * BLOCK][empty] == 0).all()
    live = torch.ones(q.shape[1], H, dtype=torch.bool)
    live[:NQS * BLOCK] = ~empty
    ref = _oracle(q, k, v, mask, NQS, 1, seqlen=SEQLEN, kv_limit_dense=SEQLEN)[0]
    assert_close(got[live], ref[live], dtype)


def _needles(dtype):
    """Head h: one sparse q block walking COUNTS[h] tiles and one dense q block walking all NB.  Query
    row c of each block has a single needle key (q.k = 32 * 32 in channel c, 130 log2 units above every
    other key) in live tile (c + h) % n of its walk, so the needles sit in every ring slot at every
    phase; the exact output is that key's V row.  The dense block uses the opposite sign, which keeps
    the two classes' needles apart.  V values are +-2^e * 2^(h - 3) with e in 0..4, exact in bf16, f16
    and after the per-head e4m3 scaling; the int8 codes are 127 against 0."""
    n_heads = len(COUNTS)
    g = torch.Generator().manual_seed(9)
    q = torch.zeros(1, 2 * BLOCK, n_heads, D)
    k = torch.zeros(1, SK, n_heads, D)
    n = torch.arange(SK)[:, None]
    d = torch.arange(D)[None, :]
    pattern = torch.where((n >> (d % 13)) & 1 == 1, -1.0, 1.0) * torch.pow(2.0, ((n + 3 * d) % 5).float())
    v = pattern[None, :, None, :] * torch.pow(2.0, torch.arange(n_heads).float() - 3).reshape(1, 1, n_heads, 1)
    want = torch.zeros(1, 2 * BLOCK, n_heads, D)
    mask = torch.zeros(1, n_heads, 1, NB, dtype=torch.bool)
    c = torch.arange(BLOCK)
    for h, count in enumerate(COUNTS):
        live = torch.randperm(NB, generator=g)[:count].sort().values
        mask[0, h, 0, live] = True
        for blk, tiles, sgn in ((0, live, 1.0), (1, torch.arange(NB), -1.0)):
            if len(tiles) == 0:
                continue
            key = tiles[(c + h) % len(tiles)] * BLOCK + (37 * c + 29 * h + 17 * blk) % BLOCK
            q[0, blk * BLOCK + c, h, c] = 32.0 * sgn
            k[0, key, h, c] = 32.0 * sgn
            want[0, blk * BLOCK + c, h] = v[0, key, h]
    return q.to(dtype).to(DEV), k.to(dtype).to(DEV), v.to(dtype).to(DEV), mask, want.to(dtype)


@pytest.mark.parametrize("path", ["bf16", "fp16", "fp8", "int8", "int8+fp8"])
def test_ring_phase_needles_are_exact(path):
    """Every row returns its needle's V row exactly (torch.equal) in each path: P_j meets V_j of the
    same ring slot and phase in the consumers, the producer and the FP8 transpose warps, for rows of
    0..8 and 40..44 tiles; rows of a q block without a live tile are exact zeros."""
    from jenga_b200.attention import _launch as launch, quantize_qk_int8, quantize_v_fp8
    dtype = torch.float16 if path == "fp16" else torch.bfloat16
    q, k, v, mask, want = _needles(dtype)
    kw = {}
    if "fp8" in path:
        kw["v_fp8"] = quantize_v_fp8(v)
    if "int8" in path:
        kw["qk_int8"] = quantize_qk_int8(q, k)
    outs = []
    for _ in range(2):
        out = torch.empty(q.shape, dtype=dtype, device=DEV)
        launch(q, k, v, _bits(mask), 1, 1, SM, 0.0, 1 << 30, SK, q.shape[1], SK, out, None, dtype, **kw)
        torch.cuda.synchronize()
        outs.append(out)
    assert _same_bits(outs[0], outs[1]), "two launches differ"
    bad = (outs[0].cpu() != want).any(-1)
    assert not bad.any(), (int(bad.sum()), bad.nonzero()[:8].tolist())


@pytest.mark.parametrize("dtype", DTYPES)
def test_ring_phases_qk_int8_against_dequantised_fp64(dtype):
    """INT8 Q.K^T (Q from shared memory): the bound of test_qk_int8_gpu.py's edge cases (mean <= 5e-3,
    max <= 5e-2 of the output RMS) against fp64 attention on the dequantised operands."""
    from jenga_b200.attention import quantize_qk_int8
    q, k, v, mask = _case(dtype)
    qk8 = quantize_qk_int8(q, k)
    got = _twice(q, k, v, mask, qk_int8=qk8)
    q8, qs, k8, ks = (t.cpu() for t in qk8)
    qd = dequantize_ref(q8, qs, 64)[:, :q.shape[1]].to(DEV)
    kd = dequantize_ref(k8, ks, 128)[:, :SK].to(DEV)
    f_max, f_mean = _fp64_errors(got, qd, kd, v, mask)
    print(f"\n[ring qk_int8 {dtype}] vs dequantised fp64: max {f_max:.2e} mean {f_mean:.2e}")
    assert f_mean <= 5e-3 and f_max <= 5e-2, (f_max, f_mean)
