"""Wan2.1-I2V fused cross-attention on the GPU.

1. jenga_wan_i2v_cross_attn against the composition it replaces — two dense-class launches of the
   attention kernel (one over the image keys, one over the text keys, as wan.cross_attention issues
   them), an fp32 add and a bf16 cast: bit-identical.  Also against an fp32 torch restatement, and rows
   past Lq of a sentinel-filled `out` stay untouched.
2. The fused I2V cross-attention (the module's own Linears around wan.i2v_cross_attention) against
   the unmodified WanI2VCrossAttention forward of the staged reference (flash_attention through the
   flash_attn shim) on an fp32 context of 257 + 512 rows: max 3e-2 and mean 2e-3 of the output RMS, the
   bounds of the T2V test; and against the FA2-bound reference module when importable: max 5e-2.
3. A chain of two unmodified WanAttentionBlock("i2v_cross_attn") at Wan-1.3B width, at sa_drop_rate
   0.0 (all rows) and 0.75 (rows with equal masks), the fused forward against the original forward.
4. Calls the fused path does not take run the original forwards."""
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(ROOT))

import test_wan_blocks_gpu as W  # noqa: E402  (helpers: _reinit, _compare, _fa_close, …)


# ------------------------------------------------------------------------------------------------
# 1. kernel
# ------------------------------------------------------------------------------------------------
def _composed(q, ki, vi, kt, vt):
    """two dense-class launches, `x + img_x` in fp32, the bf16 cast of self.o"""
    from jenga_b200.attention import BLOCK, _launch
    L = q.shape[1]
    nq = (L + BLOCK - 1) // BLOCK
    outs = []
    for k, v in ((ki, vi), (kt, vt)):
        o = torch.empty_like(q)
        _launch(q, k, v, None, 0, nq, 128 ** -0.5, 0.0, 1 << 30, k.shape[1], L, k.shape[1], o, None, torch.bfloat16)
        outs.append(o)
    return (outs[1].float() + outs[0].float()).bfloat16(), outs


def _fp32(q, k, v):
    s = torch.einsum("bqhd,bkhd->bhqk", q.float(), k.float()) * 128 ** -0.5
    return torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v.float())


def _case(Lq, Li, Lt, H, seed, peak=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda n: torch.randn(1, n, H, 128, generator=g, device="cuda")  # noqa: E731
    return (r(Lq).mul(peak).bfloat16(), r(Li).bfloat16(), r(Li).bfloat16(), r(Lt).bfloat16(), r(Lt).bfloat16())


def _check_kernel(Lq, Li, Lt, H, seed, peak=1.0):
    from jenga_b200 import wan
    q, ki, vi, kt, vt = _case(Lq, Li, Lt, H, seed, peak)
    sentinel = torch.full((1, Lq + 130, H, 128), float("nan"), dtype=torch.bfloat16, device="cuda")
    sentinel.view(torch.int16).fill_(0x7FC1)
    big = sentinel.clone()
    got = wan.i2v_cross_attn(q, ki, vi, kt, vt, out=big[:, :Lq])
    want, (a_img, a_txt) = _composed(q, ki, vi, kt, vt)
    torch.cuda.synchronize()
    what = f"Lq={Lq} Li={Li} Lt={Lt} H={H} peak={peak}"
    assert torch.equal(big[:, Lq:].view(torch.int16), sentinel[:, Lq:].view(torch.int16)), what
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), \
        (what, (got.float() - want.float()).abs().max().item())
    # the fp32 restatement: each segment within bf16 rounding of P and of A, then the sum's rounding
    # (three roundings of 2^-9 relative each; the mean bound leaves room for a 128-element case)
    ref = _fp32(q, ki, vi) + _fp32(q, kt, vt)
    scale = _fp32(q, ki, vi).abs() + _fp32(q, kt, vt).abs()
    d = (got.float() - ref).abs()
    rms = ref.pow(2).mean().sqrt().item()
    bad = (d > 2.0 ** -6 * scale + 1e-2 * rms).sum().item()
    assert bad == 0 and d.mean().item() <= 5e-3 * rms, (what, bad, d.max().item() / rms, d.mean().item() / rms)


@pytest.mark.parametrize("H", [1, 12, 40])
@pytest.mark.parametrize("Lt", [1, 300, 512, 513])
@pytest.mark.parametrize("Li", [1, 128, 257])
@pytest.mark.parametrize("Lq", [1, 127, 129, 1037, 4032])
def test_kernel_matches_two_dense_launches_bit_for_bit(Lq, Li, Lt, H):
    _check_kernel(Lq, Li, Lt, H, seed=Lq * 7 + Li * 131 + Lt * 17 + H)


@pytest.mark.parametrize("Lq,Li,Lt,H", [(1037, 257, 513, 12), (4032, 257, 512, 40), (129, 1, 300, 1)])
def test_kernel_peaky_scores(Lq, Li, Lt, H):
    """scores x30: the lazy rescale fires inside both segments"""
    _check_kernel(Lq, Li, Lt, H, seed=99 + Lq, peak=30.0)


def test_kernel_strided_views_and_batch():
    """non-contiguous [B, S, H, D] views (a wider channel row, a batch of 2) go through the strides"""
    from jenga_b200 import wan
    g = torch.Generator(device="cuda").manual_seed(5)
    B, Lq, Li, Lt, H = 2, 300, 257, 512, 4

    def view(n):
        wide = torch.randn(B, n, H + 2, 128, generator=g, device="cuda").bfloat16()
        return wide[:, :, 1:1 + H]
    q, ki, vi, kt, vt = view(Lq), view(Li), view(Li), view(Lt), view(Lt)
    got = wan.i2v_cross_attn(q, ki, vi, kt, vt)
    for b in range(B):
        want, _ = _composed(*(t[b:b + 1].contiguous() for t in (q, ki, vi, kt, vt)))
        assert torch.equal(got[b:b + 1], want), b


# ------------------------------------------------------------------------------------------------
# reference modules
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def wan_modules():
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    ref = R.load_blocks(product=False)[1]
    ours = R.load_blocks(product=True)[1]
    assert ours.WanAttentionBlock.forward.__jenga_b200__
    assert not getattr(ours.WanI2VCrossAttention.forward, "__jenga_b200__", False)
    yield ref, ours
    from jenga_b200 import blocks
    blocks.remove_gather_hook()


def _i2v_context(dim, seed, n_img=257, n_txt=512):
    """what jenga_wan.py:577-579 hands the blocks: cat(fp32 CLIP tokens, bf16 text tokens) -> fp32"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    img = torch.randn(1, n_img, dim, generator=g, device="cuda")
    txt = torch.randn(1, n_txt, dim, generator=g, device="cuda").bfloat16()
    return torch.concat([img, txt], dim=1)


# ------------------------------------------------------------------------------------------------
# 2. the I2V cross-attention module
# ------------------------------------------------------------------------------------------------
def test_i2v_cross_attention_matches_the_original_forward(wan_modules):
    ref, ours = wan_modules
    from jenga_b200 import blocks
    dim, H, L = 1536, 12, 4032
    ca = ours.WanI2VCrossAttention(dim, H, (-1, -1), True, 1e-6).cuda()
    W._reinit(ca, 61)
    g = torch.Generator(device="cuda").manual_seed(62)
    x = torch.randn(1, L, dim, generator=g, device="cuda").bfloat16()
    ctx = _i2v_context(dim, 63)
    assert ctx.dtype == torch.float32
    before = dict(blocks.STATS)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        got = blocks._wan_i2v_cross(ca, x, ctx, None)
        orig = ca(x, ctx, None)                      # the unpatched forward
    assert blocks.STATS["wan_i2v_cross"] == before["wan_i2v_cross"] + 1
    assert blocks.STATS["fallback"] == before["fallback"]
    assert got.dtype == orig.dtype == torch.bfloat16 and got.shape == orig.shape
    W._fa_close(orig, got, "fused vs unpatched I2V forward (flash_attn shim)")
    if W._reference_bound(ref):
        rca = ref.WanI2VCrossAttention(dim, H, (-1, -1), True, 1e-6).cuda()
        rca.load_state_dict(ca.state_dict())
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            W._fa_close(rca(x, ctx, None), got, "fused vs FA2-bound reference I2V", max_bound=5e-2)
    else:
        print("\n[wan i2v cross] FA2-bound reference leg skipped: flash_attn / Triton not importable")


# ------------------------------------------------------------------------------------------------
# 3. whole blocks
# ------------------------------------------------------------------------------------------------
def _make_i2v_blocks(mod, n, dim=1536, H=12, ffn=8960, seed=70):
    blks = [mod.WanAttentionBlock("i2v_cross_attn", dim, ffn, H, (-1, -1), True, True, 1e-6).cuda() for _ in range(n)]
    for i, b in enumerate(blks):
        W._reinit(b, seed + i)
    return blks


def _run(blk, x, c, ctx, drop, leg, ours, context_lens=None):
    from jenga_b200 import attention as A, blocks
    A.MASK_CAPTURE = []
    before = dict(blocks.STATS)
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            args = (x, c["e"], c["seq_lens"], c["grid"], c["freqs"], ctx, context_lens)
            kw = dict(sa_drop_rate=drop, **c["kw"])
            if leg == "original":
                with W._Unpatched(ours):
                    out = blk(*args, **kw)
            else:
                out = blk(*args, **kw)
        torch.cuda.synchronize()
        masks = list(A.MASK_CAPTURE)
    finally:
        A.MASK_CAPTURE = None
    return out, masks, {k: blocks.STATS[k] - before[k] for k in blocks.STATS}


@pytest.mark.parametrize("drop", [0.0, 0.75])
def test_i2v_block_chain_matches_the_original_forwards(wan_modules, drop):
    """bf16 x into block 0, its fp32 output into block 1; each block's two legs get the same input.
    At sa_drop_rate 0.0 the self-attention takes the original dense branch in both legs (the patched
    WanSelfAttention counts that as its own fallback)"""
    _, ours = wan_modules
    blks = _make_i2v_blocks(ours, 2)
    c = W._block_case(ours)
    ctx = _i2v_context(1536, 71)
    x = c["x"]
    for i, blk in enumerate(blks):
        a, ma, da = _run(blk, x, c, ctx, drop, "original", ours)
        b, mb, db = _run(blk, x, c, ctx, drop, "fused", ours)
        assert db["wan_block"] == 1 and db["wan_i2v_cross"] == 1 and db["wan_cross"] == 0, db
        assert da["wan_block"] == 0 and da["wan_i2v_cross"] == 0, da
        self_fallbacks = 1 if drop <= 0.25 else 0
        assert db["fallback"] == da["fallback"] == self_fallbacks, (da, db)
        assert a.dtype == b.dtype == torch.float32 and a.shape == b.shape == c["x"].shape
        if drop > 0.25:
            assert len(ma) == len(mb) == 1
            rows = W._equal_mask_rows(ma, mb, c["L"])
        else:
            rows = torch.ones(c["L"], dtype=torch.bool, device="cuda")
        W._compare(a, b, rows, f"I2V block {i} drop {drop} (x {str(x.dtype)[6:]}), fused vs original")
        x = a


# ------------------------------------------------------------------------------------------------
# 4. fallbacks
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["context_lens", "image_rows_only"])
def test_fused_block_runs_the_original_i2v_cross_attention(wan_modules, case):
    _, ours = wan_modules
    blk = _make_i2v_blocks(ours, 1, dim=512, H=4, ffn=1024)[0]
    c = W._block_case(ours, dim=512, H=4)
    ctx = _i2v_context(512, 81, n_txt=512 if case == "context_lens" else 0)
    lens = torch.tensor([300], dtype=torch.int32, device="cuda") if case == "context_lens" else None
    b, _, db = _run(blk, c["x"], c, ctx, 0.75, "fused", ours, context_lens=lens)
    a, _, da = _run(blk, c["x"], c, ctx, 0.75, "original", ours, context_lens=lens)
    assert db["wan_block"] == 1 and db["wan_i2v_cross"] == 0 and db["fallback"] == 1, db
    assert torch.isfinite(b).all()
    W._compare(a, b, torch.ones(c["L"], dtype=torch.bool, device="cuda"), f"{case}: fused block, original cross")


@pytest.mark.parametrize("case", ["no_autocast", "batch2"])
def test_calls_the_fused_block_does_not_take_run_the_original(wan_modules, case):
    _, ours = wan_modules
    from jenga_b200 import blocks
    dim, H = 512, 4
    blk = _make_i2v_blocks(ours, 1, dim=dim, H=H, ffn=1024)[0]
    c = W._block_case(ours, dim=dim, H=H)
    x, e, ctx = c["x"], c["e"], _i2v_context(dim, 91)
    drop = 0.75
    if case == "no_autocast":
        x = x.float()
    if case == "batch2":
        x, e, ctx = x.expand(2, -1, -1), e.expand(2, -1, -1), ctx.expand(2, -1, -1)
        c["seq_lens"] = torch.tensor([c["L"], c["L"]])
        c["grid"] = c["grid"].expand(2, -1)
        drop = 0.0
    args = (x, e, c["seq_lens"], c["grid"], c["freqs"], ctx, None)
    kw = dict(sa_drop_rate=drop, **c["kw"])
    before = dict(blocks.STATS)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=case != "no_autocast"):
        got = blk(*args, **kw)
        want = type(blk).forward.__wrapped__(blk, *args, **kw)
    assert blocks.STATS["fallback"] > before["fallback"]
    assert blocks.STATS["wan_block"] == before["wan_block"]
    assert blocks.STATS["wan_i2v_cross"] == before["wan_i2v_cross"]
    assert torch.equal(got, want)
