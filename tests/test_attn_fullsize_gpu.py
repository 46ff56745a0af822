"""Every row of carved attention at production shapes, through every entry point.

Workloads come from bench.workload / bench.build_inputs, and the masks are the production selection's
own (return_mask_bits=True) for the same inputs:

  hy720p        24 heads, 902 key blocks, 29 mask words, 2 text blocks
  hy_turbo_s0   text_amp 0.431 (Leg B), 497 blocks
  hy_i2v        904 blocks, device seqlen 115 500 (inside a block), 4 text blocks, 112 padded rows
  wan14b        40 heads, first-frame square, fp32 q / k cast to bf16, fp32 output
  wan1.3b       12 heads, fp32 output, 8 padded rows
  hy720p_b2     two distinct samples with their own masks (--num-videos 2)

Leg A (exact): q = 0, integer v, integer text_amp (tests/attn_ref.py).  Every element of every item of
every head must be bit-identical to flat_expected, through the plain entry point, the ordered schedule
(attention._launch), the INT8 Q.K^T entry and, on hy720p, the fused Ulysses peer-store epilogue at an
emulated world size of 8.  Outputs land in a NaN-canary buffer with a wider head stride and extra rows,
which must stay untouched.

Leg B (fp64): bench's synthetic tokens through block_sparse_attention_variant; every element of every
row of the covered heads within the per-element bound E of attn_ref.elem_bound, the mean error within
KAPPA of the mean bound, and the text rows' LSE within its bound.
"""
import math
import sys
import time
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
import attn_ref as R  # noqa: E402

DEV = torch.device("cuda", 0)
BLOCK = D = 128
SM = D ** -0.5
CANARY = {2: 0x7FA5, 4: 0x7FA5A5A5}    # NaN patterns in bf16 / fp16 and fp32 the kernel never writes
EXTRA_ROWS, HEAD_PAD = 64, 8
# mean |O - O*| <= KAPPA * mean E over the covered rows.  Measured on an H100 80GB HBM3 (700 W):
# 0.0034 (Wan-14B) to 0.0065 (Turbo stage 0) per workload over every head; max |O - O*| / E 0.040 to 0.073.
KAPPA = 0.02

# name: (bench workload, batch, dtype override)
WORKLOADS = {
    "hy720p": ("hy720p", 1, None),
    "hy_turbo_s0": ("hy_turbo_s0", 1, None),
    "hy_i2v": ("hy_i2v", 1, None),
    "wan14b": ("wan14b", 1, None),
    "wan1.3b": ("wan1.3b", 1, None),
    "hy720p_b2": ("hy720p", 2, None),
}


class Prod:
    """One production call: inputs, geometry, output and mask bits."""

    def __init__(self, name, dtype=None):
        import bench
        wl_name, B, _ = WORKLOADS[name]
        self.wl = wl = bench.workload(wl_name, 0.7)
        inps = [bench.build_inputs(wl, DEV, seed=1234 + 1000 * b) for b in range(B)]
        inp = dict(inps[0])
        for key in ("q", "k", "v"):
            inp[key] = torch.cat([i[key] for i in inps], 0)
            if dtype is not None:
                inp[key] = inp[key].to(dtype)
        self.inp = inp
        self.B, self.S, self.H = B, inp["S"], inp["heads"]
        self.T = wl["text_blocks"]
        self.nb = (self.S + BLOCK - 1) // BLOCK
        self.ns, self.nd = self.nb - self.T, self.T
        self.wan = wl["variant"] == "wan"
        self.seqlen = self.S if self.wan else int(inp["cu"][1])
        self.seqlen_dev = None if self.wan else inp["cu"][1:2].to(torch.int32)
        out, self.bits = bench.run_operator(wl, inp, return_bits=True)
        self.out = out.view(B, self.S, self.H, D)
        torch.cuda.synchronize()
        self.live = R.unpack(self.bits, self.nb)
        # what the kernel computes in: Wan casts fp32 q / k to bf16 first
        self.q16 = inp["q"].to(torch.bfloat16) if inp["q"].dtype == torch.float32 else inp["q"]
        self.k16 = inp["k"].to(torch.bfloat16) if inp["k"].dtype == torch.float32 else inp["k"]
        self.out_dtype = torch.float32 if inp["q"].dtype == torch.float32 else self.q16.dtype


def _canary_out(B, S, H, dtype):
    """(buffer, view): a [B, S, H, D] view with head stride D + 8 inside a NaN-filled buffer with
    EXTRA_ROWS more rows per sample."""
    buf = torch.empty(B, S + EXTRA_ROWS, H, D + HEAD_PAD, dtype=dtype, device=DEV)
    _ints(buf).fill_(CANARY[buf.element_size()])
    return buf, buf[:, :S, :, :D]


def _ints(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _check_exact(buf, view, want, what):
    S = view.shape[1]
    got = view
    same = _ints(got.contiguous()) == _ints(want.contiguous())
    if not bool(same.all()):
        bad = (~same).nonzero()
        b, r, h, d = bad[0].tolist()
        pytest.fail(f"{what}: {bad.shape[0]} elements differ; first (b={b}, row={r}, head={h}, d={d}): "
                    f"got {got[b, r, h, d].item()} want {want[b, r, h, d].item()}")
    c = CANARY[buf.element_size()]
    assert bool((_ints(buf[:, S:]) == c).all()), f"{what}: rows past S written"
    assert bool((_ints(buf[..., D:]) == c).all()), f"{what}: head padding written"


def _entries(p, q, k, v, bits, amp, kv_limit, q_limit, want, *, seqlen_dev, int8=True):
    """The plain entry, the ordered schedule and the INT8 Q.K^T entry on one flat case."""
    from jenga_b200.attention import _launch, carved_attention_fwd, quantize_qk_int8
    kvd = p.nb * BLOCK
    buf, view = _canary_out(p.B, p.S, p.H, p.out_dtype)
    err = torch.zeros(1, dtype=torch.int32, device=DEV)
    carved_attention_fwd(q, k, v, bits, p.ns, p.nd, SM, text_amp=float(amp), text_block_start=p.ns,
                         kv_limit_sparse=kv_limit, q_limit_sparse=q_limit, kv_limit_dense=kvd, out=view, err_flag=err)
    torch.cuda.synchronize()
    assert err.item() == 0
    _check_exact(buf, view, want, f"plain a={amp}")
    buf, view = _canary_out(p.B, p.S, p.H, p.out_dtype)
    _launch(q, k, v, bits, p.ns, p.nd, SM, float(amp), p.ns, kv_limit, q_limit, kvd, view, seqlen_dev, p.out_dtype)
    torch.cuda.synchronize()
    _check_exact(buf, view, want, f"scheduled a={amp}")
    if not int8:
        return
    qk8 = quantize_qk_int8(q, k, lse_shift=True)
    assert not bool(qk8[4].any()), "the LSE shift of q = 0 is 0"
    buf, view = _canary_out(p.B, p.S, p.H, p.out_dtype)
    lse = torch.full((p.B, p.H, p.S), float("nan"), device=DEV)
    _launch(q, k, v, bits, p.ns, p.nd, SM, float(amp), p.ns, kv_limit, q_limit, kvd, view, seqlen_dev, p.out_dtype,
            lse_out=lse if p.nd else None, qk_int8=qk8)
    torch.cuda.synchronize()
    _check_exact(buf, view, want, f"int8 a={amp}")
    if p.nd:
        # every dense score is 0: lse = ln(keys below kv_limit_dense), one fp32 log2f and product away
        text = lse[:, :, p.ns * BLOCK:]
        assert torch.allclose(text.double(), torch.full_like(text.double(), math.log(kvd)), rtol=2 ** -20, atol=0)


def _flat(p, seed=77):
    q, k, v = R.flat_case(p.B, p.S, p.H, seed=seed, device=DEV)
    return q, k, v


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_leg_a_every_item_exact(name):
    """Every element of every (sample, head, query block) item bit-identical to flat_expected through
    the plain entry, the ordered schedule and the INT8 entry, for every text_amp of Leg A: 0, 3, -2 and 9
    (9 fires the lazy rescale with alpha = 2^-9 on every sparse row at its first text tile)."""
    t0 = time.perf_counter()
    p = Prod(name)
    q, k, v = _flat(p)
    amps = R.FLAT_AMPS if p.T else (0,)
    for a in amps:
        assert R.flat_certified(p.nb, p.T, a)
        want = R.flat_expected(v, p.live, nq_sparse=p.ns, nq_dense=p.nd, q_rows=p.S, text_amp=a, text_block_start=p.ns,
                               kv_limit_sparse=p.seqlen, q_limit_sparse=p.seqlen, kv_limit_dense=p.nb * BLOCK,
                               out_dtype=p.out_dtype)
        _entries(p, q, k, v, p.bits, a, p.seqlen, p.seqlen, want, seqlen_dev=p.seqlen_dev)
    items = p.B * p.H * (p.ns + p.nd)
    print(f"\n{name}: leg A exact on {items} items ({p.B}x{p.H}x{p.ns + p.nd}) x 3 entries x {len(amps)} text_amp, "
          f"{time.perf_counter() - t0:.1f} s")


def test_leg_a_synthetic_masks_full_size():
    """hy720p with synthetic rows mixed into the production masks: every row of a head walking all 902
    tiles, rows live only in the last word, rows with the bits past nb_kv set (with no key limit, so a
    walk past nb_kv would count zero-filled keys), and empty rows (zeros)."""
    p = Prod("hy720p")
    q, k, v = _flat(p, seed=78)
    bits = p.bits.clone()
    W = bits.shape[-1]
    r = torch.arange(p.ns, device=DEV)
    kind = (r + torch.arange(p.H, device=DEV)[:, None]) % 5          # [H, ns]
    g = torch.Generator(device=DEV).manual_seed(5)
    rnd = torch.randint(-2 ** 31, 2 ** 31 - 1, bits.shape, generator=g, device=DEV, dtype=torch.int64).to(torch.int32)
    ones = torch.full_like(bits, -1)
    last_only = torch.zeros_like(bits)
    last_only[..., W - 1] = rnd[..., W - 1] | 1
    garbage = bits.clone()
    garbage[..., W - 1] |= ~((1 << (p.nb - 32 * (W - 1))) - 1)
    kind = kind[None, :, :, None]
    bits = torch.where(kind == 0, ones, torch.where(kind == 1, last_only, torch.where(
        kind == 2, torch.zeros_like(bits), torch.where(kind == 3, garbage, bits)))).contiguous()
    live = R.unpack(bits, p.nb)
    assert bool(live[0, 0, 0].all()) and not bool(live[0, 0, 2].any())
    no_limit = 1 << 40
    for a in (0, 9):
        want = R.flat_expected(v, live, nq_sparse=p.ns, nq_dense=p.nd, q_rows=p.S, text_amp=a, text_block_start=p.ns,
                               kv_limit_sparse=no_limit, q_limit_sparse=p.S, kv_limit_dense=p.nb * BLOCK)
        _entries(p, q, k, v, bits, a, no_limit, p.S, want, seqlen_dev=None)


def test_leg_a_ulysses_epilogue_world_8():
    """hy720p through the fused Ulysses peer-store epilogue at an emulated world size of 8 (every rank's
    buffers on one device): every owner's slab bit-identical to flat_expected, canaries intact."""
    from jenga_b200.attention import _launch
    from test_ulysses_emulated_gpu import World, _guards_intact, _relaid, _same
    p = Prod("hy720p")
    q, k, v = _flat(p, seed=79)
    P, T = 8, p.S - p.ns * BLOCK
    n = p.ns * BLOCK // P
    world = World(P, n, T, torch.bfloat16)
    world.restate_qkv(q, k, v)
    a = 9
    want = R.flat_expected(v, p.live, nq_sparse=p.ns, nq_dense=p.nd, q_rows=p.S, text_amp=a, text_block_start=p.ns,
                           kv_limit_sparse=p.seqlen, q_limit_sparse=p.seqlen, kv_limit_dense=p.nb * BLOCK)
    h = p.H // P
    for rank in range(P):
        qkv = world.qkv[rank]
        sp = dict(world=P, rank=rank, heads_total=p.H, rows=n, peers=world.p_out[0])
        _launch(qkv[0][None], qkv[1][None], qkv[2][None], p.bits[:, rank * h:(rank + 1) * h].contiguous(), p.ns, p.nd,
                SM, float(a), p.ns, p.S, p.S, p.nb * BLOCK, None, p.seqlen_dev, torch.bfloat16, sp_out=sp)
    torch.cuda.synchronize()
    for owner in range(P):
        assert _guards_intact(world.out_full[0][owner], world.out_rows), owner
        assert _same(world.out[0][owner], _relaid(want, owner, n, T)), owner


def test_ex2_exact_at_integer_exponents():
    """The assumption Leg A rests on: ex2.approx.ftz.f32 returns 2^n exactly at the integers -9..9.  One
    image and one text block per row, text_amp = n, small enough to read each p off the output."""
    from jenga_b200.attention import carved_attention_fwd, mask_onehot_to_bits
    S, H = 3 * BLOCK, 1
    q, k, v = R.flat_case(1, S, H, seed=3, device=DEV)
    oh = torch.tensor([[[[True, True, False], [True, False, True]]]], device=DEV)
    bits = mask_onehot_to_bits(oh)
    for a in range(-9, 10):
        want = R.flat_expected(v, oh, nq_sparse=2, nq_dense=1, q_rows=S, text_amp=a, text_block_start=1)
        got = carved_attention_fwd(q, k, v, bits, 2, 1, SM, text_amp=float(a), text_block_start=1)
        torch.cuda.synchronize()
        assert torch.equal(_ints(got), _ints(want)), a


# ------------------------------------------------------------------------------------------------
# Leg B
# ------------------------------------------------------------------------------------------------
# name: (workload, dtype, [(sample, head)]): every head; at B = 2 the second sample's (the first is
# hy720p's own inputs)
LEG_B = {
    "hy720p": ("hy720p", None, [(0, h) for h in range(24)]),
    "hy_turbo_s0": ("hy_turbo_s0", None, [(0, h) for h in range(24)]),
    "hy_turbo_s0_fp16": ("hy_turbo_s0", torch.float16, [(0, h) for h in range(24)]),
    "hy_i2v": ("hy_i2v", None, [(0, h) for h in range(24)]),
    "wan14b": ("wan14b", None, [(0, h) for h in range(40)]),
    "wan1.3b": ("wan1.3b", None, [(0, h) for h in range(12)]),
    "hy720p_b2": ("hy720p_b2", None, [(1, h) for h in range(24)]),
}


@pytest.mark.parametrize("name", list(LEG_B))
def test_leg_b_every_row_within_fp64_bound(name):
    """Every element of every row of the covered heads: |O - O*| <= E, no exceptions; mean |O - O*| <=
    KAPPA * mean E; the text rows' LSE (through _launch(lse_out=...)) within its bound."""
    from jenga_b200.attention import _launch
    wl_name, dtype, heads = LEG_B[name]
    t0 = time.perf_counter()
    p = Prod(wl_name, dtype)
    lse = None
    if p.nd:
        lse = torch.full((p.B, p.H, p.S), float("nan"), device=DEV)
        o2 = torch.empty(p.B, p.S, p.H, D, dtype=p.out_dtype, device=DEV)
        _launch(p.q16, p.k16, p.inp["v"], p.bits, p.ns, p.nd, SM, p.wl["text_amp"], p.ns, p.seqlen, p.seqlen,
                p.nb * BLOCK, o2, p.seqlen_dev, p.out_dtype, lse_out=lse)
        torch.cuda.synchronize()
        assert torch.equal(o2, p.out), "the LSE launch computes the operator's output"
    worst, err_sum, bound_sum, rows, lse_worst = 0.0, 0.0, 0.0, 0, 0.0
    for b, h in heads:
        ref = R.fp64_rows(p.q16, p.k16, p.inp["v"], p.live, b=b, h=h, qblocks=range(p.nb), nq_sparse=p.ns, sm_scale=SM,
                          text_amp=p.wl["text_amp"], text_block_start=p.ns, kv_limit=p.seqlen, q_limit=p.seqlen,
                          small_p=p.q16.dtype == torch.float16)
        E, e_lse = R.elem_bound(ref, p.q16.dtype)
        got = p.out[b, :, h].double()
        err = (got - ref["o"]).abs()
        over = err > E
        if bool(over.any()):
            r, d = over.nonzero()[0].tolist()
            pytest.fail(f"{name} b={b} h={h}: {int(over.sum())} elements over E; row {r} d {d}: got {got[r, d].item()} "
                        f"O* {ref['o'][r, d].item()} E {E[r, d].item()}")
        live_e = E > 0
        worst = max(worst, (err[live_e] / E[live_e]).max().item())
        err_sum += err.sum().item()
        bound_sum += E.sum().item()
        rows += err.shape[0]
        if lse is not None:
            t = slice(p.ns * BLOCK, p.S)
            dl = (lse[b, h, t].double() - ref["lse"][t]).abs()
            assert bool((dl <= e_lse[t]).all()), (name, b, h, (dl / e_lse[t]).max().item())
            lse_worst = max(lse_worst, (dl / e_lse[t]).max().item())
    kappa = err_sum / bound_sum
    print(f"\n{name}: rows {rows}, max|err|/E {worst:.3f}, mean|err|/mean E {kappa:.4f}, LSE max err/bound "
          f"{lse_worst:.3f}, {time.perf_counter() - t0:.1f} s")
    assert kappa <= KAPPA, kappa
