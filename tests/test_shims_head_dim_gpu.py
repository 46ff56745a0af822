"""Head dims below 128 in the FlashAttention shims (jenga_b200/flash_attn_shim.py).

install() replaces flash_attn for the whole process, so the Wan2.1-I2V CLIP image encoder
(wan/modules/clip.py: ViT-H/14, 16 heads of 80 channels, 257 tokens, fp16) reaches the varlen shim
before the DiT runs.  The shims serve head dims 8..128 in multiples of 8 by zero-padding the channels
to the kernel's 128 and slicing the output; the default softmax scale is the caller's D ** -0.5.

1. All three entry points against fp32 SDPA (and fp32 logsumexp for softmax_lse): D in {64, 80, 96,
   112}, bf16 and fp16, B = 2, ragged Sq / Sk including the encoder's 257, explicit and default scale;
   the varlen shim with two segments and one that has no keys.
2. At D = 80 every entry point equals, bit for bit, the dense launch on hand-padded 128-channel inputs
   at scale 80 ** -0.5, sliced to 80 channels.
3. The opt-in INT8 Q.K^T / FP8 P.V switches at D = 80: bit-identical to the direct launch of the same
   variant on the padded inputs, and within the tolerance rows of tests/test_qk_int8_paths_gpu.py.
4. What is still refused, and that head_dim 128 calls never reach the padding.
5. The unmodified reference encoder (wan/modules/clip.py, staged into oracle/_ref_clip/ by
   oracle/make_ref_clip.py; reduced depth, production width) under install(), against an
   fp32 SDPA restatement of its attention and against the FA2-bound module when importable: max 2e-2
   and mean 2e-3 of the output RMS.  Measured on an H100 80GB HBM3 (700 W power limit): max 6.8e-3 /
   mean 4.2e-4 against SDPA, max 1.0e-2 / mean 4.2e-4 against FlashAttention 2.8.3.
6. The encoder's rows through MLPProj (WanModel.img_emb) into the context of a WanAttentionBlock
   ("i2v_cross_attn") under install(): the fused I2V cross-attention runs."""
import contextlib
import importlib
import importlib.util
import sys
import types
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(ROOT))

import test_qk_int8_paths_gpu as P  # noqa: E402  (_direct, _fp64, _check_row, _qkv, _flags, ROWS)
import test_wan_blocks_gpu as W  # noqa: E402
import test_wan_i2v_gpu as I  # noqa: E402
from test_attn_gpu import assert_close  # noqa: E402

DIMS = [64, 80, 96, 112]
DTYPES = [torch.bfloat16, torch.float16]
SHAPES = [(257, 257), (300, 1000)]          # (Sq, Sk): the encoder's, and ragged q against more keys


def _randn(shape, dtype, g, gain=1.0):
    return (gain * torch.randn(shape, generator=g, device="cuda")).to(dtype)


def _case(B, Sq, Sk, H, D, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return _randn((B, Sq, H, D), dtype, g), _randn((B, Sk, H, D), dtype, g), _randn((B, Sk, H, D), dtype, g)


def _sdpa(q, k, v, scale):
    """[B,S,H,D] -> fp32 [B,Sq,H,D]"""
    o = torch.nn.functional.scaled_dot_product_attention(
        q.float().transpose(1, 2), k.float().transpose(1, 2), v.float().transpose(1, 2), scale=scale)
    return o.transpose(1, 2)


def _logsumexp(q, k, scale):
    """fp32 logsumexp of the scaled scores -> [B,H,Sq]"""
    return torch.logsumexp(torch.einsum("bqhd,bkhd->bhqk", q.float(), k.float()) * scale, dim=-1)


def _assert_lse(got, truth):
    """the bound of test_attn_edges_gpu.test_dense_lse_matches_fp64_logsumexp"""
    err = (got.double() - truth.double()).abs()
    bound = 2e-4 + 1e-5 * truth.double().abs()
    assert (err <= bound).all(), (err.max().item(), (err / bound).max().item())


def _pad128(t):
    """zero channels appended by hand (a different construction from the shim's)"""
    return torch.cat([t, t.new_zeros(*t.shape[:-1], 128 - t.shape[-1])], dim=-1).contiguous()


def _dense128(q, k, v, scale, lse=None):
    """one dense-class launch over 128-channel q [B,Sq,H,128], k / v [B,Sk,H,128]"""
    from jenga_b200.attention import BLOCK, _launch
    B, Sq, H, D = q.shape
    out = torch.empty_like(q)
    _launch(q, k, v, None, 0, (Sq + BLOCK - 1) // BLOCK, scale, 0.0, 1 << 30, k.shape[1], Sq, k.shape[1], out, None,
            q.dtype, lse_out=lse)
    return out


# varlen: three q segments; the third has no keys
SEG_Q = [257, 300, 130]
SEG_K = [257, 700, 0]


def _cu(lens):
    return torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device="cuda")


def _varlen_case(D, dtype, seed, H=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    Tq, Tk = sum(SEG_Q), sum(SEG_K)
    return _randn((Tq, H, D), dtype, g), _randn((Tk, H, D), dtype, g), _randn((Tk, H, D), dtype, g)


def _segments():
    q0 = k0 = 0
    for lq, lk in zip(SEG_Q, SEG_K):
        yield q0, q0 + lq, k0, k0 + lk
        q0, k0 = q0 + lq, k0 + lk


# ------------------------------------------------------------------------------------------------
# 1. parity against fp32 SDPA
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scale", [None, 0.1])
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", DIMS)
def test_flash_attn_func_matches_sdpa(D, dtype, shape, scale):
    from jenga_b200.flash_attn_shim import flash_attn_func
    Sq, Sk = shape
    q, k, v = _case(2, Sq, Sk, 3, D, dtype, seed=D + Sq + Sk)
    out = flash_attn_func(q, k, v, softmax_scale=scale)
    assert out.shape == q.shape and out.dtype == dtype and out.is_contiguous()
    assert_close(out, _sdpa(q, k, v, D ** -0.5 if scale is None else scale), dtype)


@pytest.mark.parametrize("scale", [None, 0.1])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", DIMS)
def test_flash_attn_varlen_func_matches_sdpa(D, dtype, scale):
    """segments of 257 / 300 / 130 query rows against 257 / 700 / 0 keys: the last one is zeros"""
    from jenga_b200.flash_attn_shim import flash_attn_varlen_func
    q, k, v = _varlen_case(D, dtype, seed=3 * D)
    out = flash_attn_varlen_func(q, k, v, _cu(SEG_Q), _cu(SEG_K), max(SEG_Q), max(SEG_K), softmax_scale=scale)
    assert out.shape == q.shape and out.dtype == dtype and out.is_contiguous()
    s = D ** -0.5 if scale is None else scale
    ref = torch.zeros(q.shape, dtype=torch.float32, device="cuda")
    for q0, q1, k0, k1 in _segments():
        if k1 > k0:
            ref[q0:q1] = _sdpa(q[None, q0:q1], k[None, k0:k1], v[None, k0:k1], s)[0]
    assert_close(out, ref, dtype)
    assert not out[SEG_Q[0] + SEG_Q[1]:].any()


@pytest.mark.parametrize("scale", [None, 0.1])
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", DIMS)
def test_flash_attn_forward_matches_sdpa_and_logsumexp(D, dtype, shape, scale):
    from jenga_b200.flash_attn_shim import _flash_attn_forward
    Sq, Sk = shape
    q, k, v = _case(2, Sq, Sk, 3, D, dtype, seed=5 * D + Sq + Sk)
    out, lse, s_dmask, rng = _flash_attn_forward(q, k, v, softmax_scale=scale)
    assert s_dmask is None and rng is None
    assert out.shape == q.shape and out.dtype == dtype
    assert lse.shape == (2, 3, Sq) and lse.dtype == torch.float32
    s = D ** -0.5 if scale is None else scale
    assert_close(out, _sdpa(q, k, v, s), dtype)
    _assert_lse(lse, _logsumexp(q, k, s))


# ------------------------------------------------------------------------------------------------
# 2. exact restatement at D = 80
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_d80_equals_the_dense_launch_on_hand_padded_inputs(dtype):
    from jenga_b200 import flash_attn_shim as F
    s = 80 ** -0.5
    q, k, v = _case(2, 257, 300, 4, 80, dtype, seed=80)
    got = F.flash_attn_func(q, k, v)
    want = _dense128(_pad128(q), _pad128(k), _pad128(v), s)
    torch.cuda.synchronize()
    assert torch.equal(got, want[..., :80])
    assert not want[..., 80:].any()                          # zero channels give zero output columns

    got, lse, _, _ = F._flash_attn_forward(q, k, v)
    want_lse = torch.empty_like(lse)
    want = _dense128(_pad128(q), _pad128(k), _pad128(v), s, lse=want_lse)
    torch.cuda.synchronize()
    assert torch.equal(got, want[..., :80]) and torch.equal(lse, want_lse)

    q, k, v = _varlen_case(80, dtype, seed=81, H=4)
    got = F.flash_attn_varlen_func(q, k, v, _cu(SEG_Q), _cu(SEG_K), max(SEG_Q), max(SEG_K))
    want = torch.zeros_like(got)
    for q0, q1, k0, k1 in _segments():
        if k1 > k0:
            want[q0:q1] = _dense128(_pad128(q[None, q0:q1]), _pad128(k[None, k0:k1]), _pad128(v[None, k0:k1]), s)[0, ..., :80]
    torch.cuda.synchronize()
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------
# 3. the opt-in switches
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["int8", "int8+fp8"])
def test_d80_follows_the_switches(monkeypatch, mode):
    """q and k are bench.synth_tokens (the regime of the tolerance rows) cut to 80 channels.  The LSE
    stays within the 16-bit-problem bounds of test_qk_int8_paths_gpu.test_int8_lse_against_fp64."""
    from jenga_b200.flash_attn_shim import _flash_attn_forward, flash_attn_func, flash_attn_varlen_func
    D, s = 80, 80 ** -0.5
    q, k, v = (t[..., :D].contiguous() for t in P._qkv((2, 300, 3, 128), (2, 1000, 3, 128), torch.bfloat16, 41))
    plain = flash_attn_func(q, k, v)
    P._flags(monkeypatch, mode)
    got = flash_attn_func(q, k, v)
    out, lse, _, _ = _flash_attn_forward(q, k, v)
    segs = (((0, 150), (0, 400)), ((150, 300), (400, 1000)))    # varlen: batch 0 cut into two segments
    cu_q = torch.tensor([0, 150, 300], dtype=torch.int32, device="cuda")
    cu_k = torch.tensor([0, 400, 1000], dtype=torch.int32, device="cuda")
    got_v = flash_attn_varlen_func(q[0], k[0], v[0], cu_q, cu_k, 150, 600)
    P._flags(monkeypatch, None)
    qp, kp, vp = _pad128(q), _pad128(k), _pad128(v)
    want = P._direct(qp, kp, vp, s, mode)[..., :D]
    want_lse = torch.empty_like(lse)
    want_out = P._direct(qp, kp, vp, s, mode, lse=want_lse)[..., :D]
    want_v = torch.cat([P._direct(qp[:1, a:b], kp[:1, c:d], vp[:1, c:d], s, mode)[0, ..., :D] for (a, b), (c, d) in segs])
    torch.cuda.synchronize()
    assert torch.equal(got, want) and not torch.equal(got, plain)
    assert torch.equal(out, want_out) and torch.equal(lse, want_lse)
    assert torch.equal(got_v, want_v)
    P._check_row(got, q, k, v, s, mode)
    _, lse_16 = P._fp64(q, k, v, s)
    e = (lse.double() - lse_16).abs()
    print(f"\n[{mode} lse, D {D}] vs 16-bit fp64: mean {e.mean().item():.2e} max {e.max().item():.2e}")
    assert e.mean().item() <= 0.08 and e.max().item() <= 0.3


def test_d80_fp16_keeps_the_default_pv_under_the_fp8_switch(monkeypatch):
    from jenga_b200.flash_attn_shim import flash_attn_func
    q, k, v = _case(1, 300, 700, 2, 80, torch.float16, seed=42)
    plain = flash_attn_func(q, k, v)
    P._flags(monkeypatch, "fp8")
    assert torch.equal(flash_attn_func(q, k, v), plain)


# ------------------------------------------------------------------------------------------------
# 4. refusals, and head_dim 128 untouched
# ------------------------------------------------------------------------------------------------
def _three_calls(q, k, v):
    from jenga_b200 import flash_attn_shim as F
    S, Sk = q.shape[1], k.shape[1]
    cu_q = torch.tensor([0, S], dtype=torch.int32, device="cuda")
    cu_k = torch.tensor([0, Sk], dtype=torch.int32, device="cuda")
    return (lambda: F.flash_attn_func(q, k, v),
            lambda: F.flash_attn_varlen_func(q[0], k[0], v[0], cu_q, cu_k, S, Sk),
            lambda: F._flash_attn_forward(q, k, v))


@pytest.mark.parametrize("dq,dk,dv", [(100, 100, 100), (160, 160, 160), (80, 80, 64), (64, 80, 80), (4, 4, 4)])
def test_other_head_dims_are_refused(dq, dk, dv):
    g = torch.Generator(device="cuda").manual_seed(7)
    q = _randn((1, 130, 2, dq), torch.bfloat16, g)
    k = _randn((1, 200, 2, dk), torch.bfloat16, g)
    v = _randn((1, 200, 2, dv), torch.bfloat16, g)
    for call in _three_calls(q, k, v):
        with pytest.raises(NotImplementedError, match=str(dv if dq == dk else dk)):
            call()


def test_head_dim_128_never_reaches_the_padding(monkeypatch):
    from jenga_b200 import flash_attn_shim as F
    q, k, v = _case(1, 300, 1000, 2, 128, torch.bfloat16, seed=9)
    want = [c() for c in _three_calls(q, k, v)]

    def refuse(*a):
        raise AssertionError("head_dim 128 must not be padded")
    monkeypatch.setattr(F, "_pad_head_dim", refuse)
    got = [c() for c in _three_calls(q, k, v)]
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    assert torch.equal(got[2][0], want[2][0]) and torch.equal(got[2][1], want[2][1])


def test_varlen_pads_once_for_all_segments(monkeypatch):
    from jenga_b200 import flash_attn_shim as F
    calls = []
    orig = F._pad_head_dim

    def counted(*a):
        calls.append(a[0].shape)
        return orig(*a)
    monkeypatch.setattr(F, "_pad_head_dim", counted)
    q, k, v = _varlen_case(80, torch.bfloat16, seed=12)
    F.flash_attn_varlen_func(q, k, v, _cu(SEG_Q), _cu(SEG_K), max(SEG_Q), max(SEG_K))
    assert calls == [q.shape]


# ------------------------------------------------------------------------------------------------
# 5. the unmodified reference CLIP image encoder
# ------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _ftfy_stand_in():
    """clip.py imports its tokenizer module (wan/modules/tokenizers.py), which imports ftfy; only the
    tokenizer calls it.  Where ftfy is missing, a stand-in takes its place while clip.py is imported."""
    added = "ftfy" not in sys.modules and importlib.util.find_spec("ftfy") is None
    if added:
        sys.modules["ftfy"] = types.ModuleType("ftfy")
    try:
        yield
    finally:
        if added:
            sys.modules.pop("ftfy", None)


def _import_reference(product, names, clip_dir):
    """the unmodified reference modules `names` of wan.modules; clip_dir: where clip.py and its
    tokenizer modules are staged when the reference root does not hold them (oracle/_ref_clip/)"""
    from oracle import ref_loader as R
    with R.reference_packages(product=product), _ftfy_stand_in():
        if clip_dir is not None:
            sys.modules["wan.modules"].__path__.append(str(clip_dir / "wan" / "modules"))
        return [importlib.import_module(n) for n in names]


@pytest.fixture(scope="module")
def clip_modules():
    """(clip bound to the shim, model_mul bound to the shim, clip bound to the real flash_attn or None)"""
    from oracle import make_ref_clip
    from oracle import ref_loader as R
    root = R.ref_root()
    if root is None:
        pytest.skip("reference files not staged (oracle/_ref/)")
    clip_dir = None
    if not (root / "wan/modules/clip.py").is_file():
        clip_dir = make_ref_clip.staged()
        if clip_dir is None:
            pytest.skip("reference CLIP encoder not staged (oracle/_ref_clip/)")
    ours, model = _import_reference(True, ["wan.modules.clip", "wan.modules.model_mul"], clip_dir)
    try:
        ref, = _import_reference(False, ["wan.modules.clip"], clip_dir)
    except ImportError as e:
        print(f"\n[clip] reference module with the real flash_attn not importable: {e}")
        ref = None
    assert ours.flash_attention.__globals__["flash_attn"].__jenga_b200__
    yield ours, model, ref
    from jenga_b200 import blocks
    blocks.remove_gather_hook()


def _fa2_bound(ref):
    if ref is None:
        return False
    gl = ref.flash_attention.__globals__
    fa = gl.get("flash_attn")
    return bool(gl.get("FLASH_ATTN_2_AVAILABLE")) and fa is not None and not getattr(fa, "__jenga_b200__", False)


LAYERS = 5        # use_31_block drops the last one: 4 attention layers run


def _vit(mod):
    """VisionTransformer as clip_xlm_roberta_vit_h_14 builds it (XLMRobertaCLIP's vision arguments), at
    reduced depth, fp16 like CLIPModel(dtype=torch.float16)"""
    with torch.device("cuda"):
        m = mod.VisionTransformer(image_size=224, patch_size=14, dim=1280, mlp_ratio=4, out_dim=1024, num_heads=16,
                                  num_layers=LAYERS, pool_type="token", pre_norm=True, post_norm=False,
                                  activation="gelu")
    return m.half().eval().requires_grad_(False)


def _encoder(mod, seed=100):
    """seeded weights; the Q and K projections scaled up so that the attention is far from uniform"""
    m = _vit(mod)
    W._reinit(m, seed)
    with torch.no_grad():
        for blk in m.transformer:
            blk.attn.to_qkv.weight[:2 * 1280].mul_(2.5)
    return m


def _image(seed=101):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(1, 3, 224, 224, generator=g, device="cuda").half()


def _visual(m, x):
    """CLIPModel.visual after its preprocessing (clip.py:540-541)"""
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        return m(x, use_31_block=True)


def _sdpa_flash_attention(q, k, v, q_lens=None, k_lens=None, dropout_p=0.0, softmax_scale=None, causal=False,
                          version=None, **_):
    """fp32 SDPA in place of wan.modules.attention.flash_attention for the encoder's calls"""
    assert q_lens is None and k_lens is None and dropout_p == 0.0 and not causal
    with torch.autocast("cuda", enabled=False):
        o = _sdpa(q, k, v, q.shape[-1] ** -0.5 if softmax_scale is None else softmax_scale)
    return o.to(q.dtype)


def _close(a, b, what, max_bound=2e-2, mean_bound=2e-3):
    a, b = a.float(), b.float()
    rms = a.pow(2).mean().sqrt().item()
    d = (a - b).abs()
    mx, mean = d.max().item() / rms, d.mean().item() / rms
    print(f"\n[clip] {what}: max {mx:.3e} mean {mean:.3e} (x RMS)")
    assert mx <= max_bound and mean <= mean_bound, (what, mx, mean)


def test_reference_encoder_runs_through_the_shim(clip_modules, monkeypatch):
    from jenga_b200 import flash_attn_shim as F
    ours, _, ref = clip_modules
    m = _encoder(ours)
    x = _image()
    padded = []
    orig = F._pad_head_dim

    def counted(*a):
        padded.append(tuple(a[0].shape))
        return orig(*a)
    monkeypatch.setattr(F, "_pad_head_dim", counted)
    got = _visual(m, x)
    monkeypatch.setattr(F, "_pad_head_dim", orig)
    assert got.shape == (1, 257, 1280) and got.dtype == torch.float16 and torch.isfinite(got).all()
    assert padded == [(257, 16, 80)] * (LAYERS - 1)
    with monkeypatch.context() as mp:
        mp.setattr(ours, "flash_attention", _sdpa_flash_attention)
        want = _visual(m, x)
    _close(want, got, "shim vs fp32 SDPA restatement")
    if _fa2_bound(ref):
        rm = _vit(ref)
        rm.load_state_dict(m.state_dict())
        _close(_visual(rm, x), got, "shim vs FA2-bound reference")
    else:
        print("\n[clip] FA2-bound reference leg skipped: flash_attn not importable")


# ------------------------------------------------------------------------------------------------
# 6. encoder -> img_emb -> the I2V block
# ------------------------------------------------------------------------------------------------
def test_encoder_rows_reach_the_fused_i2v_block(clip_modules):
    """jenga_wan.py:380 (clip.visual) -> WanModel.img_emb (MLPProj(1280, dim)) -> cat(CLIP rows, text
    rows) (jenga_wan.py:577-579) -> WanAttentionBlock("i2v_cross_attn") at the Wan-1.3B width, fused
    against its original forward"""
    ours, model, _ = clip_modules
    dim = 1536
    feats = _visual(_encoder(ours, seed=110), _image(111))
    proj = model.MLPProj(1280, dim).cuda()
    W._reinit(proj, 112)
    g = torch.Generator(device="cuda").manual_seed(113)
    txt = torch.randn(1, 512, dim, generator=g, device="cuda").bfloat16()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        ctx = torch.concat([proj(feats), txt], dim=1)
    assert ctx.shape == (1, 257 + 512, dim) and ctx.dtype == torch.float32 and torch.isfinite(ctx).all()
    blk = I._make_i2v_blocks(model, 1)[0]
    c = W._block_case(model)
    a, ma, da = I._run(blk, c["x"], c, ctx, 0.75, "original", model)
    b, mb, db = I._run(blk, c["x"], c, ctx, 0.75, "fused", model)
    assert db["wan_block"] == 1 and db["wan_i2v_cross"] == 1 and db["fallback"] == 0, db
    assert da["wan_block"] == 0 and da["wan_i2v_cross"] == 0, da
    assert len(ma) == len(mb) == 1
    W._compare(a, b, W._equal_mask_rows(ma, mb, c["L"]), "encoder -> I2V block, fused vs original")
