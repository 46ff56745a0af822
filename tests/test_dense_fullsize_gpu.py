"""Every row of the dense attention launches at production shapes: the FlashAttention shims, the Wan T2V
cross-attention and the two-segment Wan I2V cross-attention kernel.

Call patterns, as the reference issues them (bench.workload geometry):

  hy720p       flash_attn_varlen_func, cu_seqlens from get_cu_seqlens: segments [115 380 | 76], 24 heads;
               at B = 2 with text_valid 180 and 256 (the second sample's padding segment is empty)
  hy_i2v       segments [115 500 | 100]
  wan14b       flash_attention(q, k, v, k_lens=seq_lens): one segment of 75 600 per sample, 40 heads
  wan1.3b      32 760, 12 heads
  k_lens       two samples of 32 760 queries over 37 and 512 of their context keys
  lse          _flash_attn_forward on the padding text rows (76, 100) and [1, 115 456, 3, 128]
  cross        attention._launch as wan.cross_attention issues it: 75 600 / 32 760 queries x 512 keys
  i2v          wan.i2v_cross_attn: 75 600 / 32 760 queries x (257 + 512) keys, 40 heads
  clip         flash_attn_varlen_func at head dim 80, fp16, 257 tokens x 16 heads

Leg A (exact, tests/attn_ref.py): q = 0, integer v.  Every element of every head bit-identical to
segments_expected / dense_expected / i2v_expected, the default path and with attention.QK_INT8 on (the
same expectation: only the column limit hides the K padding's non-zero smoothed codes), and with
attention.PV_FP8 on fp8_expected on sparse power-of-two V.  LSE = ln(Sk).  Entries that take out= write
into a NaN-canary buffer with a wider head stride and extra rows, which must stay untouched.

Leg B (fp64): bench.synth_tokens q and k, Gaussian v.  Every element of every row of every head within
the per-element bound E of attn_ref.elem_bound (i2v_bound for the I2V sum), the mean error within kappa
of the mean bound, and every LSE within its bound.

The file runs in about 85 s on an H100 80GB HBM3 (700 W power limit).
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
CANARY = {2: 0x7FA5, 4: 0x7FA5A5A5}
EXTRA_ROWS, HEAD_PAD = 64, 8
# mean |O - O*| <= kappa * mean E over a workload's rows.  Measured on an H100 80GB HBM3 (700 W): 0.0024
# to 0.0048 on the full-length self-attention rows, where E carries the terms that grow with the key
# tiles (KAPPA, the carved file's); 0.036 to 0.096 where E is essentially the two 16-bit roundings
# (P and the output): the cross-attentions' 512 / 769 keys, CLIP's 257 and rows dominated by one key.
# An unbiased round-to-nearest meets such a bound with a mean of about a quarter of each term, so
# KAPPA_ROUNDING flags a systematic bias there.
KAPPA = 0.02
KAPPA_ROUNDING = 0.15


def _wl(name):
    import bench
    return bench.workload(name, 0.7)


def _hy_cu(name, text_valid):
    """get_cu_seqlens (hyvideo/modules/attenion.py:34-57) for one sample per text_valid entry."""
    wl = _wl(name)
    n_img = math.prod(wl["grid"])
    S = n_img + wl["text_tokens"]
    cu = [0]
    for i, tv in enumerate(text_valid):
        cu += [i * S + n_img + tv, (i + 1) * S]
    return cu, cu, wl["heads"]


def _wan_cu(name, B):
    wl = _wl(name)
    L = math.prod(wl["grid"])
    cu = [i * L for i in range(B + 1)]
    return cu, cu, wl["heads"]


# name: (cu_q, cu_k, heads), the packed varlen calls of the self-attention shapes
VARLEN = {
    "hy720p": _hy_cu("hy720p", [180]),
    "hy720p_b2": _hy_cu("hy720p", [180, 256]),
    "hy_i2v": _hy_cu("hy_i2v", [300]),
    "wan14b": _wan_cu("wan14b", 1),
    "wan1.3b": _wan_cu("wan1.3b", 1),
    "wan14b_b2": _wan_cu("wan14b", 2),
    "k_lens_37_512": ([0, 32760, 65520], [0, 37, 549], 12),
}
CANARY_SEGMENTS = ("hy720p_b2", "wan14b_b2", "k_lens_37_512")


def _ints(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _canary(shape, dtype):
    """(buffer, view): a view of `shape` [..., S, H, D] with head stride D + 8 inside a NaN-filled buffer
    with EXTRA_ROWS more rows."""
    *lead, S, H, Dv = shape
    buf = torch.empty(*lead, S + EXTRA_ROWS, H, Dv + HEAD_PAD, dtype=dtype, device=DEV)
    _ints(buf).fill_(CANARY[buf.element_size()])
    return buf, buf[..., :S, :, :Dv]


def _canary_intact(buf, S, Dv, what):
    c = CANARY[buf.element_size()]
    assert bool((_ints(buf[..., S:, :, :]) == c).all()), f"{what}: rows past S written"
    assert bool((_ints(buf[..., Dv:]) == c).all()), f"{what}: head padding written"


def _same(got, want, what):
    same = _ints(got.contiguous()) == _ints(want.contiguous())
    if not bool(same.all()):
        bad = (~same).nonzero()
        idx = tuple(bad[0].tolist())
        pytest.fail(f"{what}: {bad.shape[0]} of {same.numel()} elements differ; first {idx}: got {got[idx].item()} "
                    f"want {want[idx].item()}")
    return same.numel()


@pytest.fixture
def switches():
    """Sets attention.QK_INT8 / PV_FP8 for one test and restores them."""
    from jenga_b200 import attention as A
    saved = A.QK_INT8, A.PV_FP8

    def set_(qk_int8=False, pv_fp8=False):
        A.QK_INT8, A.PV_FP8 = qk_int8, pv_fp8
    yield set_
    A.QK_INT8, A.PV_FP8 = saved


def _varlen(q, k, v, cu_q, cu_k):
    from jenga_b200.flash_attn_shim import flash_attn_varlen_func
    cq = torch.tensor(cu_q, dtype=torch.int32, device=DEV)
    ck = torch.tensor(cu_k, dtype=torch.int32, device=DEV)
    mq = max(b - a for a, b in zip(cu_q, cu_q[1:]))
    mk = max(b - a for a, b in zip(cu_k, cu_k[1:]))
    out = flash_attn_varlen_func(q, k, v, cq, ck, mq, mk, softmax_scale=None)
    torch.cuda.synchronize()
    return out


# ------------------------------------------------------------------------------------------------
# Leg A
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(VARLEN))
def test_leg_a_varlen_every_element(name, switches):
    """flash_attn_varlen_func in the reference's call pattern: every element of every head bit-identical to
    segments_expected, by default and with QK_INT8; with PV_FP8, fp8_expected per segment.  On the B = 2
    shapes every segment also through _dense(out=...) into a NaN canary."""
    from jenga_b200.flash_attn_shim import _dense
    t0 = time.perf_counter()
    cu_q, cu_k, H = VARLEN[name]
    Tq, Tk = cu_q[-1], cu_k[-1]
    q = torch.zeros(Tq, H, D, dtype=torch.bfloat16, device=DEV)
    _, k, v = R.flat_case(1, Tk, H, seed=31, device=DEV)
    k, v = k[0], v[0]
    want = R.segments_expected(v, cu_q, cu_k, Tq)
    items = 0
    for qk_int8 in (False, True):
        switches(qk_int8=qk_int8)
        items += _same(_varlen(q, k, v, cu_q, cu_k), want, f"{name} int8={qk_int8}")
    switches()
    if name in CANARY_SEGMENTS:
        buf, view = _canary((1, Tq, H, D), torch.bfloat16)
        for i in range(len(cu_q) - 1):
            q0, q1, k0, k1 = cu_q[i], cu_q[i + 1], cu_k[i], cu_k[i + 1]
            if q1 > q0 and k1 > k0:
                _dense(q[None, q0:q1], k[None, k0:k1], v[None, k0:k1], None, out=view[:, q0:q1])
            else:
                view[:, q0:q1] = 0
        torch.cuda.synchronize()
        items += _same(view[0], want, f"{name} _dense(out=)")
        _canary_intact(buf, Tq, D, name)
    del want
    _, _, v8 = R.fp8_case(1, Tk, H, seed=32, device=DEV)
    want8 = R.segments_expected(v8[0], cu_q, cu_k, Tq, one=R.fp8_expected)
    switches(pv_fp8=True)
    items += _same(_varlen(q, k, v8[0], cu_q, cu_k), want8, f"{name} fp8")
    print(f"\n{name}: leg A exact on {items} elements (default, int8, fp8{', canary' if name in CANARY_SEGMENTS else ''}), "
          f"{time.perf_counter() - t0:.1f} s")


# name: (B, Sq = Sk, heads, sample amax for the FP8 leg)
LSE_CALLS = {
    "hy720p_text_76": (1, 76, 24, (8,)),
    "hy_i2v_text_100": (1, 100, 24, (8,)),
    "text_76_b2_amax_8_4": (2, 76, 24, (8, 4)),
    "hy720p_8way_heads": (1, 115456, 3, (8,)),
}


@pytest.mark.parametrize("name", list(LSE_CALLS))
def test_leg_a_flash_attn_forward_out_and_lse(name, switches):
    """_flash_attn_forward as parallel_attention calls it: out bit-identical, LSE = ln(Sk) to log2f's
    rounding, by default and with QK_INT8; the same launch through _dense(out=, lse=) into NaN canaries
    (LSE buffer NaN-filled past B * H * Sq); with PV_FP8, fp8_expected (a distinct amax per sample at B = 2)."""
    from jenga_b200.flash_attn_shim import _dense, _flash_attn_forward
    B, S, H, amaxes = LSE_CALLS[name]
    q, k, v = R.flat_case(B, S, H, seed=41, device=DEV)
    want = R.dense_expected(v, S)
    lse_want = torch.full((B, H, S), math.log(S), dtype=torch.float64, device=DEV)
    kw = dict(dropout_p=0.0, softmax_scale=SM, causal=False, window_size_left=-1, window_size_right=-1, softcap=0.0,
              alibi_slopes=None, return_softmax=False)
    for qk_int8 in (False, True):
        switches(qk_int8=qk_int8)
        out, lse, *_ = _flash_attn_forward(q, k, v, **kw)
        torch.cuda.synchronize()
        _same(out, want, f"{name} int8={qk_int8}")
        assert lse.shape == (B, H, S) and lse.dtype == torch.float32
        assert torch.allclose(lse.double(), lse_want, rtol=R.LSE_RTOL, atol=0), (lse.min().item(), math.log(S))
    switches()
    buf, view = _canary((B, S, H, D), torch.bfloat16)
    lse_buf = torch.full((B * H * S + 4096,), float("nan"), device=DEV)
    _dense(q, k, v, SM, out=view, lse=lse_buf[:B * H * S].view(B, H, S))
    torch.cuda.synchronize()
    _same(view, want, f"{name} canary")
    _canary_intact(buf, S, D, name)
    assert torch.allclose(lse_buf[:B * H * S].double(), lse_want.flatten(), rtol=R.LSE_RTOL, atol=0)
    assert bool(lse_buf[B * H * S:].isnan().all()), "LSE stored past B * H * Sq"
    _, _, v8 = R.fp8_case(B, S, H, seed=42, device=DEV, amax=amaxes)
    switches(pv_fp8=True)
    out, lse, *_ = _flash_attn_forward(q, k, v8, **kw)
    torch.cuda.synchronize()
    _same(out, R.fp8_expected(v8, S), f"{name} fp8")
    assert torch.allclose(lse.double(), lse_want, rtol=R.LSE_RTOL, atol=0)


CROSS = {"wan14b": (75600, 40), "wan1.3b": (32760, 12)}


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("name", list(CROSS))
def test_leg_a_t2v_cross_launch(name, B):
    """attention._launch exactly as wan.cross_attention issues it (dense-only, Lc = 512 keys, column limit
    Lc) into a NaN canary: every element bit-identical to dense_expected."""
    from jenga_b200.attention import _launch
    L, H = CROSS[name]
    q = torch.zeros(B, L, H, D, dtype=torch.bfloat16, device=DEV)
    _, k, v = R.flat_case(B, 512, H, seed=51 + B, device=DEV)
    buf, view = _canary((B, L, H, D), torch.bfloat16)
    _launch(q, k, v, None, 0, (L + BLOCK - 1) // BLOCK, SM, 0.0, 1 << 30, 512, L, 512, view, None, torch.bfloat16)
    torch.cuda.synchronize()
    _same(view, R.dense_expected(v, L), f"{name} B={B}")
    _canary_intact(buf, L, D, name)


def test_leg_a_t2v_cross_attention_zero_rows():
    """wan.cross_attention itself with q_lin = 0: the norm of a zero row is zero, so the result is the
    flat expectation over the 512 normed keys."""
    from jenga_b200 import wan
    B, L, H = 2, 32760, 12
    g = torch.Generator(device=DEV).manual_seed(61)
    q_lin = torch.zeros(B, L, H * D, dtype=torch.bfloat16, device=DEV)
    k_lin = torch.randn(B, 512, H * D, generator=g, device=DEV).bfloat16()
    w = (1 + 0.1 * torch.randn(H * D, generator=g, device=DEV)).bfloat16()
    _, _, v = R.flat_case(B, 512, H, seed=62, device=DEV)
    out = wan.cross_attention(q_lin, k_lin, v, w, w, H)
    torch.cuda.synchronize()
    _same(out, R.dense_expected(v, L), "cross_attention")


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("L", [75600, 32760])
def test_leg_a_i2v_cross_attn(L, B):
    """wan.i2v_cross_attn into a NaN canary: every element bit-identical to round16(f32(A_img) + f32(A_txt))
    over Li = 257 and Lt = 512 keys, 40 heads."""
    from jenga_b200.wan import i2v_cross_attn
    H = 40
    q = torch.zeros(B, L, H, D, dtype=torch.bfloat16, device=DEV)
    _, ki, vi = R.flat_case(B, 257, H, seed=71 + B, device=DEV)
    _, kt, vt = R.flat_case(B, 512, H, seed=81 + B, device=DEV)
    buf, view = _canary((B, L, H, D), torch.bfloat16)
    i2v_cross_attn(q, ki, vi, kt, vt, out=view)
    torch.cuda.synchronize()
    n = _same(view, R.i2v_expected(vi, vt, L), f"i2v L={L} B={B}")
    _canary_intact(buf, L, D, "i2v")
    print(f"\ni2v L={L} B={B}: leg A exact on {n} elements")


def test_leg_a_clip_head_dim_80(switches):
    """The CLIP encoder's call: flash_attn_varlen_func, 257 tokens x 16 heads of 80 channels, fp16; the
    output's 80 columns bit-identical to the padded launch's expectation, by default and with QK_INT8."""
    S, H, Dc = 257, 16, 80
    q, k, v = R.flat_case(1, S, H, seed=91, device=DEV, dtype=torch.float16)
    v = v.clone()
    v[..., Dc:] = 0
    want = R.dense_expected(v, S)[0, ..., :Dc]
    for qk_int8 in (False, True):
        switches(qk_int8=qk_int8)
        got = _varlen(q[0, ..., :Dc].contiguous(), k[0, ..., :Dc].contiguous(), v[0, ..., :Dc].contiguous(), [0, S],
                      [0, S])
        assert got.shape == (S, H, Dc)
        _same(got, want, f"clip int8={qk_int8}")


# ------------------------------------------------------------------------------------------------
# Leg B
# ------------------------------------------------------------------------------------------------
class Stats:
    def __init__(self, name, kappa=KAPPA):
        self.name, self.t0, self.kappa = name, time.perf_counter(), kappa
        self.worst = self.err = self.bound = self.lse_worst = 0.0
        self.rows = 0

    def add(self, got, o, E, what, lse=None, lse_ref=None, e_lse=None):
        err = (got.double() - o).abs()
        over = err > E
        if bool(over.any()):
            r, d = over.nonzero()[0].tolist()
            pytest.fail(f"{self.name} {what}: {int(over.sum())} elements over E; row {r} d {d}: got {got[r, d].item()} "
                        f"O* {o[r, d].item()} E {E[r, d].item()}")
        live = E > 0
        self.worst = max(self.worst, (err[live] / E[live]).max().item())
        self.err += err.sum().item()
        self.bound += E.sum().item()
        self.rows += err.shape[0]
        if lse is not None:
            dl = (lse.double() - lse_ref).abs()
            assert bool((dl <= e_lse).all()), (self.name, what, (dl / e_lse).max().item())
            self.lse_worst = max(self.lse_worst, (dl / e_lse).max().item())

    def done(self):
        kappa = self.err / self.bound
        print(f"\n{self.name}: rows {self.rows}, max|err|/E {self.worst:.3f}, mean|err|/mean E {kappa:.4f}, "
              f"LSE max err/bound {self.lse_worst:.3f}, {time.perf_counter() - self.t0:.1f} s")
        assert kappa <= self.kappa, kappa


def _real(S, H, seed, gain=1.0):
    """bench's synthetic q and k ([S, H, 128] bf16), Gaussian v; q scaled by gain."""
    import bench
    q = bench.synth_tokens(S, H, DEV, seed)[0]
    k = bench.synth_tokens(S, H, DEV, seed + 1)[0]
    v = torch.randn(S, H, D, generator=torch.Generator(device=DEV).manual_seed(seed + 2), device=DEV).bfloat16()
    if gain != 1.0:
        q = (q.float() * gain).bfloat16()
    return q, k, v


def _rows(q, k, v, h, sm_scale=SM, chunk=8, small_p=False):
    """fp64_rows of every row of head h of one dense launch (q [Sq, H, D], k / v [Sk, H, D])."""
    nq = (q.shape[0] + BLOCK - 1) // BLOCK
    return R.fp64_rows(q[None], k[None], v[None], None, b=0, h=h, qblocks=range(nq), nq_sparse=0, sm_scale=sm_scale,
                       kv_limit_dense=k.shape[0], chunk=chunk, small_p=small_p)


# name: (varlen shape, q gain, kappa): every row of every head.  The peaky case scales q by 4, so the
# row maximum climbs by more than 8 log2 units across tiles and the lazy rescale fires.
LEG_B_VARLEN = {
    "hy720p": ("hy720p", 1.0, KAPPA),
    "hy_i2v": ("hy_i2v", 1.0, KAPPA),
    "wan14b": ("wan14b", 1.0, KAPPA),
    "wan1.3b": ("wan1.3b", 1.0, KAPPA),
    "wan1.3b_peaky": ("wan1.3b", 4.0, KAPPA_ROUNDING),
}


@pytest.mark.parametrize("name", list(LEG_B_VARLEN))
def test_leg_b_varlen_within_fp64_bound(name):
    """flash_attn_varlen_func on synthetic tokens: every row of every head of every segment within E; the
    short text segments also through _flash_attn_forward, whose LSE is within E_lse."""
    from jenga_b200.flash_attn_shim import _flash_attn_forward
    shape, gain, kappa = LEG_B_VARLEN[name]
    cu_q, cu_k, H = VARLEN[shape]
    st = Stats(name, kappa)
    q, k, v = _real(cu_q[-1], H, seed=101, gain=gain)
    out = _varlen(q, k, v, cu_q, cu_k)
    for i in range(len(cu_q) - 1):
        q0, q1, k0, k1 = cu_q[i], cu_q[i + 1], cu_k[i], cu_k[i + 1]
        short = q1 - q0 <= 4 * BLOCK
        lse = None
        if short:
            o2, lse, *_ = _flash_attn_forward(q[None, q0:q1], k[None, k0:k1], v[None, k0:k1], softmax_scale=SM)
            torch.cuda.synchronize()
            assert torch.equal(o2[0], out[q0:q1]), "_flash_attn_forward computes the varlen segment"
        for h in range(H):
            ref = _rows(q[q0:q1], k[k0:k1], v[k0:k1], h)
            E, e_lse = R.elem_bound(ref, torch.bfloat16)
            st.add(out[q0:q1, h], ref["o"], E, f"segment {i} head {h}",
                   *((lse[0, h], ref["lse"], e_lse) if short else ()))
    st.done()


def test_leg_b_t2v_cross_within_fp64_bound():
    """_launch as wan.cross_attention issues it, 75 600 queries x 512 keys: every row of every head."""
    from jenga_b200.attention import _launch
    L, H = CROSS["wan14b"]
    st = Stats("t2v_cross_wan14b", KAPPA_ROUNDING)
    q, _, _ = _real(L, H, seed=111)
    _, k, v = _real(512, H, seed=121)
    out = torch.empty(1, L, H, D, dtype=torch.bfloat16, device=DEV)
    _launch(q[None], k[None], v[None], None, 0, (L + BLOCK - 1) // BLOCK, SM, 0.0, 1 << 30, 512, L, 512, out, None,
            torch.bfloat16)
    torch.cuda.synchronize()
    for h in range(H):
        ref = _rows(q, k, v, h, chunk=64)
        E, _ = R.elem_bound(ref, torch.bfloat16)
        st.add(out[0, :, h], ref["o"], E, f"head {h}")
    st.done()


def test_leg_b_i2v_cross_within_fp64_bound():
    """wan.i2v_cross_attn, 75 600 queries x (257 + 512) keys: every row of every head within i2v_bound."""
    from jenga_b200.wan import i2v_cross_attn
    L, H = 75600, 40
    st = Stats("i2v_cross_75600", KAPPA_ROUNDING)
    q, _, _ = _real(L, H, seed=131)
    _, ki, vi = _real(257, H, seed=141)
    _, kt, vt = _real(512, H, seed=151)
    out = i2v_cross_attn(q[None], ki[None], vi[None], kt[None], vt[None])
    torch.cuda.synchronize()
    for h in range(H):
        o, E = R.i2v_bound(_rows(q, ki, vi, h, chunk=64), _rows(q, kt, vt, h, chunk=64))
        st.add(out[0, :, h], o, E, f"head {h}")
    st.done()


def test_leg_b_clip_within_fp64_bound():
    """The CLIP call (head dim 80, fp16, default scale 80^-1/2): every row of every head.  The reference
    rows see the zero-padded channels, which add nothing to Q.K^T."""
    S, H, Dc = 257, 16, 80
    st = Stats("clip_d80", KAPPA_ROUNDING)
    q, k, v = (t[..., :Dc].half().contiguous() for t in _real(S, H, seed=161))
    out = _varlen(q, k, v, [0, S], [0, S])
    pad = [torch.nn.functional.pad(t, (0, D - Dc)) for t in (q, k, v)]
    for h in range(H):
        ref = _rows(*pad, h, sm_scale=Dc ** -0.5, small_p=True)
        E, _ = R.elem_bound(ref, torch.float16)
        st.add(out[:, h], ref["o"][:, :Dc], E[:, :Dc], f"head {h}")
    st.done()
