"""Sparse rows of the sm_90a carved-attention kernel that walk 0, 1, 2 or 3 key tiles, in one launch.

Each consumer warpgroup of carved_attn.cu issues S_j = Q K_j^T together with the previous tile's
P V and takes turns with the other warpgroup on two named barriers.  A row with one live tile runs
only the prologue (S_0, softmax) and the epilogue (the last P V); two and three tiles add one and
two loop iterations, and each count ends the turn hand-over on a different step.  Every head here
has q blocks with each of the four counts next to a dense q block that walks all 8 tiles.  In the
"rise30" regime the score max grows by 30 log2 units per key block, so O is rescaled on every
tile, after the wait that retires the previous P V.  The needle cases pin the pairing of P_j with
V_j exactly, in the FP8 P.V path too.
"""
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
from test_attn_edges_gpu import BLOCK, D, DEV, DTYPES, QK, SM, _bits, _oracle, _run  # noqa: E402
from test_attn_gpu import assert_close  # noqa: E402

NB = 8          # key blocks
H = 4
NQ_SPARSE = 8   # sparse q blocks per head; block m of head h walks (h + m) % 4 tiles


def _short_rows(dtype, regime, seed=41):
    g = torch.Generator().manual_seed(seed)
    Sq, Sk = (NQ_SPARSE + 1) * BLOCK, NB * BLOCK
    q = torch.randn(1, Sq, H, D, generator=g)
    k = torch.randn(1, Sk, H, D, generator=g)
    v = torch.randn(1, Sk, H, D, generator=g)
    if regime == "rise30":   # channel 127: q = a, k = 2j on key block j (exact in bf16 / fp16)
        k[0, :, :, 127] = (2 * (torch.arange(Sk) // BLOCK)).float()[:, None]
        q[0, :, :, 127] = 30.0 / (2 * QK)
    mask = torch.zeros(1, H, NQ_SPARSE, NB, dtype=torch.bool)
    for h in range(H):
        for m in range(NQ_SPARSE):
            mask[0, h, m, torch.randperm(NB, generator=g)[:(h + m) % 4]] = True
    return q.to(dtype), k.to(dtype), v.to(dtype), mask


def _empty_rows(mask):
    """[NQ_SPARSE * BLOCK, H] bool: sparse rows whose q block has no live tile."""
    return (mask[0].sum(-1) == 0).t().repeat_interleave(BLOCK, 0)


@pytest.mark.parametrize("regime", ["normal", "rise30"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_rows_of_zero_to_three_tiles_match_oracle(dtype, regime):
    """Bound: assert_close against the oracle on every row with a live tile; rows without one are
    exact zeros."""
    q, k, v, mask = _short_rows(dtype, regime)
    assert sorted(set(mask.sum(-1).flatten().tolist())) == [0, 1, 2, 3]
    Sk = k.shape[1]
    got = _run(q, k, v, _bits(mask), NQ_SPARSE, 1, kv_limit_dense=Sk)
    empty = _empty_rows(mask)
    assert (got[0, :NQ_SPARSE * BLOCK][empty.to(DEV)] == 0).all()
    live = torch.ones(q.shape[1], H, dtype=torch.bool)
    live[:NQ_SPARSE * BLOCK] = ~empty
    ref = _oracle(q, k, v, mask, NQ_SPARSE, 1, seqlen=Sk, kv_limit_dense=Sk)
    assert_close(got[0].cpu()[live], ref[0][live], dtype)


def _needles(dtype, n_heads=8, seed=43):
    """One sparse q block per head, walking (h % 4) tiles, and one dense q block.  Query row c has a
    single needle key with q.k = 32 * 32 in channel c (130 log2 units above every other key), so its
    exact output is that key's V row; it lies in live tile (c + h) % n, in both ring slots across
    rows.  The dense rows use the opposite sign, which keeps the two classes' needles apart.  V values
    are +-2^e * 2^(h - 3) with e in 0..4, exact in bf16, fp16 and after the per-head e4m3 scaling."""
    g = torch.Generator().manual_seed(seed)
    H = n_heads
    Sq, Sk = 2 * BLOCK, NB * BLOCK
    q = torch.zeros(1, Sq, H, D)
    k = torch.zeros(1, Sk, H, D)
    n = torch.arange(Sk)[:, None]
    d = torch.arange(D)[None, :]
    pattern = torch.where((n >> (d % 13)) & 1 == 1, -1.0, 1.0) * torch.pow(2.0, ((n + 3 * d) % 5).float())
    v = pattern[None, :, None, :] * torch.pow(2.0, torch.arange(H).float() - 3).reshape(1, 1, H, 1)
    want = torch.zeros(1, Sq, H, D)
    mask = torch.zeros(1, H, 1, NB, dtype=torch.bool)
    c = torch.arange(BLOCK)
    for h in range(H):
        live = torch.randperm(NB, generator=g)[:h % 4].sort().values
        mask[0, h, 0, live] = True
        for blk, tiles, sgn in ((0, live, 1.0), (1, torch.arange(NB), -1.0)):
            if len(tiles) == 0:
                continue
            key = tiles[(c + h) % len(tiles)] * BLOCK + (37 * c + 29 * h + 17 * blk) % BLOCK
            q[0, blk * BLOCK + c, h, c] = 32.0 * sgn
            k[0, key, h, c] = 32.0 * sgn
            want[0, blk * BLOCK + c, h] = v[0, key, h]
    return q.to(dtype), k.to(dtype), v.to(dtype), mask, want.to(dtype)


@pytest.mark.parametrize("path", ["bf16", "fp16", "fp8"])
def test_needle_rows_of_zero_to_three_tiles_are_exact(path):
    """Every row returns its needle's V row exactly (torch.equal) in each P.V path, FP8 included (its
    V^T comes from the producer warps' transpose): P_j meets V_j of the same tile in the prologue,
    the loop and the epilogue.  Rows of a q block without a live tile are exact zeros."""
    from jenga_b200.attention import _launch, quantize_v_fp8
    dtype = torch.float16 if path == "fp16" else torch.bfloat16
    q, k, v, mask, want = _needles(dtype)
    assert sorted(set(mask.sum(-1).flatten().tolist())) == [0, 1, 2, 3]
    q, k, v = q.to(DEV), k.to(DEV), v.to(DEV)
    v8 = quantize_v_fp8(v) if path == "fp8" else None
    out = torch.empty(q.shape, dtype=dtype, device=DEV)
    _launch(q, k, v, _bits(mask), 1, 1, SM, 0.0, 1 << 30, k.shape[1], q.shape[1], k.shape[1], out, None, dtype,
            v_fp8=v8)
    torch.cuda.synchronize()
    bad = (out.cpu() != want).any(-1)
    assert not bad.any(), (int(bad.sum()), bad.nonzero()[:8].tolist())
