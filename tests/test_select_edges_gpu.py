"""Block pooling and block selection against exact restatements and fp64 (tests/select_ref.py), on
every selection path, at tile edges, parameter edges and the shipped workloads' block counts.

Selection paths of jenga_select_blocks (csrc/select.cu):
  tc       workspace, n_img <= 1024, mask_words <= 64, head_dim 128: tensor-core pooled-score GEMM
           (mma.sync) + one warp per row (the default of every shipped workload)
  simt     the same with JENGA_SELECT_GEMM=simt: fp32 SIMT GEMM (read once per process, so this leg
           runs in a child process)
  reg      no workspace, n_img <= 1024: fused kernel, register-resident sort
  smem     fused kernel, n_img > 1024: shared-memory 64-bit bitonic sort
  r4       fused kernel with fewer than 8 rows per CTA (n_img = 2100)
  wide     two-kernel path with text columns past bit 1023 (33 mask words)
  fallback mask_words > 64: the fused kernel even though a workspace is given
The kernel's own scores feed the selection oracle: the workspace on the two-kernel paths (checked
against the certified / exact scores first), scores_exact on the fused paths (which the existing
test_simt_gemm_path_is_bit_identical_to_fused_kernel links to the SIMT GEMM bit for bit)."""
import ctypes as C
import math
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(ROOT))
import select_ref as sr  # noqa: E402

DEV = "cuda"


# ------------------------------------------------------------------------------------------------
# C-ABI call with a workspace the test owns
# ------------------------------------------------------------------------------------------------
def select_raw(qp, kp, *, n_img, nb, top_k, p, text_blocks, ff=0, nbr=None, nbr_rows=None, nbr_words=None,
               workspace=True):
    """jenga_select_blocks on pooled [B,H,nq,D] / [B,H,nk_pool,D].  Returns (bits [B*H*nq, words]
    int32, counts [B*H*nq] int32, scores [B*H, nq, n_img] fp32 or None).  The workspace is always
    large enough for the two-kernel path; whether the kernel uses it depends on the shape."""
    from jenga_b200 import _lib
    from jenga_b200._lib import check, lib
    from jenga_b200.attention import _dtype_code, _stream_ptr
    B, H, nq, D = qp.shape
    words = (nb + 31) // 32
    bits = torch.full((B * H * nq, words), 0x5a5a5a5a, dtype=torch.int32, device=qp.device)
    counts = torch.full((B * H * nq,), -7, dtype=torch.int32, device=qp.device)
    a = _lib.JengaSelectArgs()
    a.q_pool, a.k_pool, a.dtype = qp.data_ptr(), kp.data_ptr(), _dtype_code(qp)
    a.batch_heads, a.head_dim, a.nq = B * H, D, nq
    a.nk_pool, a.n_img, a.nb, a.mask_words = kp.shape[2], n_img, nb, words
    a.top_k, a.p_threshold = int(top_k), float(p)
    a.text_blocks, a.first_frame_blocks = int(text_blocks), int(ff)
    if nbr is not None:
        a.nbr_bits = nbr.data_ptr()
        a.nbr_rows = nbr.shape[0] if nbr_rows is None else nbr_rows
        a.nbr_words = nbr.shape[1] if nbr_words is None else nbr_words
    else:
        a.nbr_bits, a.nbr_rows, a.nbr_words = None, 0, 0
    a.out_bits, a.out_counts = bits.data_ptr(), counts.data_ptr()
    ws = None
    if workspace:
        nbytes = B * H * nq * n_img * 4
        ws = torch.full((B * H, nq, n_img), float("nan"), dtype=torch.float32, device=qp.device)
        a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
    else:
        a.workspace, a.workspace_bytes = None, 0
    with torch.cuda.device(qp.device):
        check(lib.jenga_select_blocks(C.byref(a), _stream_ptr(qp.device)), "select_blocks")
    torch.cuda.synchronize()
    two_kernel = workspace and n_img <= 1024 and words <= 64 and D == 128
    return bits, counts, (ws if two_kernel else None)


def check_scores_tc(qp, kp, n_img, ws, what):
    """Tensor-core GEMM: every score in the certified set; returns the ambiguous fraction."""
    _, lo, hi, amb = sr.scores_certified(qp, kp, n_img)
    bad = (ws < lo) | (ws > hi) | torch.isnan(ws)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError((what, "score outside the certified set", int(bad.sum()), i,
                              float(ws[tuple(i)]), float(lo[tuple(i)]), float(hi[tuple(i)])))
    return amb.float().mean().item()


def check_selection(qp, kp, scores, bits, counts, what, cut_band=sr.CUT_BAND, **kw):
    """bits / counts against select_oracle fed `scores`; returns (count-, tie-ambiguous fractions)."""
    nq = qp.shape[2]
    sel = sr.select_oracle(scores, kw["n_img"], kw["nb"], kw["top_k"], kw["p"], kw["text_blocks"],
                           kw.get("ff", 0), kw.get("nbr"), kw.get("nbr_rows"), kw.get("nbr_words"), nq=nq,
                           cut_band=cut_band)
    return sel.check(bits, counts, what)


# ------------------------------------------------------------------------------------------------
# a. pooling
# ------------------------------------------------------------------------------------------------
def _pool_input(kind, B, S, H, D, dt, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    scale = torch.exp2(torch.linspace(-12, 3, H, device=DEV)).view(1, 1, H, 1)  # tiny to large heads
    off = torch.linspace(-2, 2, D, device=DEV).view(1, 1, 1, D)
    if kind == "packed":      # one slice of a packed [B,S,3,H,D]
        full = torch.randn(B, S, 3, H, D, generator=g, device=DEV) * scale.unsqueeze(2) + off.unsqueeze(2)
        return full.to(dt)[:, :, 1]
    if kind == "heads":       # head-sliced view of [B,S,H+5,D]
        full = torch.randn(B, S, H + 5, D, generator=g, device=DEV) + 0.25
        full[:, :, 2:2 + H] = full[:, :, 2:2 + H] * scale + off
        return full.to(dt)[:, :, 2:2 + H]
    x = torch.randn(B, S, H, D, generator=g, device=DEV) * scale + off * scale
    return x.to(dt)


POOL_CASES = [
    # kind, B, S, H, D, dtype, n_blocks (None: ceil(S/128))
    ("dense", 2, 1000, 5, 64, torch.bfloat16, None),       # batch 2, ragged S
    ("dense", 1, 777, 40, 128, torch.float16, None),       # fp16, ragged
    ("dense", 1, 300, 24, 128, torch.bfloat16, 2),         # n_blocks < ceil(S/128)
    ("dense", 1, 129, 1, 128, torch.float16, None),        # one row in the last block
    ("dense", 2, 333, 5, 64, torch.float32, None),         # fp32 + cast_out, batch 2, ragged
    ("dense", 1, 1000, 24, 128, torch.float32, 7),         # fp32 + cast_out, n_blocks < ceil
    ("packed", 2, 515, 24, 128, torch.bfloat16, None),
    ("packed", 1, 400, 5, 64, torch.float32, None),
    ("heads", 2, 260, 5, 128, torch.float16, None),
    ("heads", 1, 640, 40, 64, torch.bfloat16, 4),
    ("dense", 1, 115456, 24, 128, torch.bfloat16, None),   # HunyuanVideo 720p
    ("dense", 1, 75600, 40, 128, torch.float32, None),     # Wan 14B, fp32 (cast_out)
]


def check_pool(x, n_blocks, what):
    from jenga_b200.attention import block_pool
    cast = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device) if x.dtype == torch.float32 else None
    if cast is not None:
        cast.fill_(float("nan"))
    got = block_pool(x, n_blocks, cast_out=cast)
    torch.cuda.synchronize()
    want = sr.pool_exact(x, n_blocks)
    assert got.dtype == want.dtype and got.shape == want.shape
    diff = got.view(torch.int16) != want.view(torch.int16)
    assert not diff.any(), (what, "pooled != pool_exact", int(diff.sum()), diff.nonzero()[0].tolist())
    mean, amean = sr.pool_fp64(x, n_blocks)
    sr.assert_pool_certified(got, mean, amean, what)
    if cast is not None:
        # the whole bf16 copy, ragged tail rows included, whatever n_blocks is
        want_c = x.to(torch.bfloat16)
        if n_blocks * 128 < x.shape[1]:
            want_c = want_c[:, :n_blocks * 128]
            cast = cast[:, :n_blocks * 128]
        assert torch.equal(cast.view(torch.int16), want_c.view(torch.int16)), what
    return got


@pytest.mark.parametrize("kind,B,S,H,D,dt,nblk", POOL_CASES)
def test_block_pool_bit_exact_and_within_fp64_bound(kind, B, S, H, D, dt, nblk):
    x = _pool_input(kind, B, S, H, D, dt, seed=S + H)
    n_blocks = nblk or (S + 127) // 128
    check_pool(x, n_blocks, (kind, B, S, H, D, str(dt), n_blocks))


# ------------------------------------------------------------------------------------------------
# b. scores
# ------------------------------------------------------------------------------------------------
def _pooled(B, H, n, D, dt, seed, bias=0.3):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(B, H, n, D, generator=g, device=DEV) * 0.5 + bias).to(dt)


SCORE_SHAPES = [(1, 1), (1, 900), (63, 65), (64, 64), (65, 63), (65, 1024), (900, 900), (1024, 1024)]


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("nq,n_img", SCORE_SHAPES)
def test_tensor_core_scores_certified(nq, n_img, dt):
    B, H = (2, 24) if nq * n_img <= 65 * 1024 else (1, 3)   # B*H = 48 at the small shapes
    qp = _pooled(B, H, nq, 128, dt, nq * 7 + n_img)
    kp = _pooled(B, H, n_img + 5, 128, dt, nq + n_img * 3)   # nk_pool > n_img
    kw = dict(n_img=n_img, nb=n_img + 2, top_k=max(1, n_img // 4), p=0.3, text_blocks=2)
    bits, counts, ws = select_raw(qp, kp, **kw)
    frac = check_scores_tc(qp, kp, n_img, ws, (nq, n_img, str(dt)))
    print(f"tensor-core scores nq={nq} n_img={n_img} {dt}: ambiguous fraction {frac:.5f}")
    assert frac < 0.01 or nq * n_img < 100   # (a 1 x 1 tile has 48 elements)
    check_selection(qp, kp, ws, bits, counts, (nq, n_img, str(dt)), **kw)


# ------------------------------------------------------------------------------------------------
# c. selection on every path
# ------------------------------------------------------------------------------------------------
def _case_inputs(kind, B, H, nq, n_img, nk, D, dt, seed):
    """Pooled q [B,H,nq,D] and k [B,H,nk,D] whose scores have the named structure."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    if kind == "rand":
        return _pooled(B, H, nq, D, dt, seed), _pooled(B, H, nk, D, dt, seed + 1)
    if kind == "dup":       # duplicated key blocks: exact ties everywhere
        q, k = _pooled(B, H, nq, D, dt, seed, 0.1), _pooled(B, H, nk, D, dt, seed + 1, 0.1)
        src = torch.randint(0, max(1, n_img // 5), (n_img,), generator=g, device=DEV)
        k[:, :, :n_img] = k[:, :, src]
        return q, k
    if kind == "equal":     # every ranked score equal: uniform probabilities
        q = _pooled(B, H, nq, D, dt, seed)
        k = _pooled(B, H, 1, D, dt, seed + 1).expand(B, H, nk, D).contiguous()
        return q, k
    q = torch.zeros(B, H, nq, D, device=DEV)
    k = torch.zeros(B, H, nk, D, device=DEV)
    if kind == "two":       # two score values, large tie groups across the cut
        q[..., 0] = 0.8 + 0.4 * torch.rand(B, H, nq, generator=g, device=DEV)
        hi = torch.rand(B, H, nk, generator=g, device=DEV) < 0.3
        k[..., 0] = torch.where(hi, 8.0, 4.0)
        return q.to(dt), k.to(dt)
    if kind == "peaky":     # scores down to ~130 below the max: zero and fp32-subnormal probabilities
        # score ~ k0 / sqrt(D) in [-100, 30]: probabilities e^(s - 30) are fp32 subnormals for
        # s in (-67, -57) and certainly +0 for s < -83; s in [-83, -65], where an fp32 probability
        # may or may not round to zero, is left out so that the cut is decided
        q[..., 0] = 1.0
        t = torch.linspace(-82.0, 30.0, nk, device=DEV)
        t = torch.where(t < -65.0, t - 18.0, t)
        perm = torch.stack([torch.randperm(nk, generator=g, device=DEV) for _ in range(B * H)])
        k[..., 0] = t[perm].view(B, H, nk) * math.sqrt(D)
        return q.to(dt), k.to(dt)
    raise KeyError(kind)


def _nbr(kind, nq, words, seed):
    if kind is None:
        return None, None, None
    g = torch.Generator(device=DEV).manual_seed(seed)
    raw = torch.randint(-2 ** 31, 2 ** 31 - 1, (nq, words), generator=g, device=DEV, dtype=torch.int64)
    raw = (raw & torch.randint(-2 ** 31, 2 ** 31 - 1, (nq, words), generator=g, device=DEV,
                               dtype=torch.int64)).to(torch.int32)   # garbage past n_img and nb too
    if kind == "full":
        return raw, nq, words
    return raw, max(1, nq - 3), max(1, words - 1)  # fewer rows than nq, fewer words (pitch) than words


# path: (n_img, nb - n_img, head_dim); text_blocks defaults to nb - n_img
PATHS = {
    "tc": (900, 2, 128), "reg": (700, 2, 64), "smem": (1025, 2, 128), "smem1500": (1500, 4, 96),
    "r4": (2100, 2, 128), "wide": (1020, 8, 128), "fallback": (300, 1801, 128),
}
_TWO_KERNEL = {"tc", "wide"}
_FUSED = {"reg", "smem", "smem1500", "r4"}

# kind, p ("mid:x": halfway between two multiples of 1/n_img near x), top_k ("n": n_img, "n+5",
# "0.6n"), first_frame_blocks ("nb+5"), text_blocks override (clipped by nb), neighbour rows, dtype,
# B, H, nq
SEL_CASES = [
    ("rand", 0.3, 1, 0, None, "full", torch.bfloat16, 1, 3, 40),
    ("rand", 0.0, 0, 3, None, "short", torch.bfloat16, 2, 2, 37),
    ("rand", 0.05, 0, 0, None, None, torch.float16, 1, 2, 33),
    ("rand", 0.9, "n+5", "nb+5", 10 ** 6, "full", torch.bfloat16, 1, 2, 20),
    ("rand", 1.5, 1, 0, None, "short", torch.float16, 2, 1, 17),
    ("dup", 0.3, 1, 3, None, None, torch.bfloat16, 1, 2, 40),
    ("dup", 0.9, "n", 0, None, "short", torch.float16, 1, 2, 9),
    ("equal", "mid:0.3", 0, 0, None, None, torch.bfloat16, 1, 2, 10),
    ("equal", "mid:0.6", 5, 0, 10 ** 6, None, torch.float16, 2, 1, 10),
    ("two", 0.5, 1, 0, None, None, torch.bfloat16, 1, 2, 12),
    ("two", 0.05, 0, 0, None, "full", torch.float16, 1, 2, 12),
    ("peaky", 0.3, "0.6n", 0, None, None, torch.bfloat16, 1, 2, 24),
    ("peaky", 0.0, "0.9n", 0, None, None, torch.bfloat16, 1, 1, 24),
]


def _resolve(path, case, idx):
    kind, p, top_k, ff, text, nbr_kind, dt, B, H, nq = case
    n_img, extra, D = PATHS[path]
    nb = n_img + extra
    text_blocks = extra if text is None else text
    if isinstance(p, str):
        p = (math.floor(float(p[4:]) * n_img) + 0.5) / n_img
    if isinstance(top_k, str):
        top_k = {"n": n_img, "n+5": n_img + 5, "0.6n": int(0.6 * n_img), "0.9n": int(0.9 * n_img)}[top_k]
    if ff == "nb+5":
        ff = nb + 5
    seed = 1000 * idx + n_img
    qp, kp = _case_inputs(kind, B, H, nq, n_img, n_img + 3, D, dt, seed)
    words = (nb + 31) // 32
    nbr, nbr_rows, nbr_words = _nbr(nbr_kind, nq, words, seed + 5)
    kw = dict(n_img=n_img, nb=nb, top_k=top_k, p=p, text_blocks=text_blocks, ff=ff, nbr=nbr,
              nbr_rows=nbr_rows, nbr_words=nbr_words)
    return qp, kp, kw, D


def run_selection_case(path, case, idx, simt=False):
    qp, kp, kw, D = _resolve(path, case, idx)
    what = (path, idx, case[0], case[1], case[2])
    bits, counts, ws = select_raw(qp, kp, workspace=path not in _FUSED, **kw)
    assert (ws is not None) == (path in _TWO_KERNEL), what
    if ws is None:
        scores = sr.scores_exact(qp, kp, kw["n_img"])
    elif simt:
        scores = sr.scores_exact(qp, kp, kw["n_img"])
        assert torch.equal(ws.view(torch.int32), scores.view(torch.int32)), (what, "SIMT scores != scores_exact")
    else:
        check_scores_tc(qp, kp, kw["n_img"], ws, what)
        scores = ws
    fr = check_selection(qp, kp, scores, bits, counts, what, **kw)
    return fr


@pytest.mark.parametrize("path", [p for p in PATHS])
@pytest.mark.parametrize("idx", range(len(SEL_CASES)))
def test_selection_matches_oracle(path, idx):
    case = SEL_CASES[idx]
    fc, ft = run_selection_case(path, case, idx)
    print(f"{path} case {idx} ({case[0]}, p={case[1]}): ambiguous rows count {fc:.4f} tie {ft:.4f}")


# n_img a power of two and every score equal: probabilities are exactly 1/n_img, every fp32
# cumulative sum is exact, and it equals p exactly at rank p * n_img.  count = #(C <= p) + 1 is then
# certain, so the comparison `C <= p` itself is checked (not just its neighbourhood).
DYADIC = [("tc", 512, True), ("reg", 512, False), ("smem", 2048, False), ("r4", 4096, False)]


@pytest.mark.parametrize("path,n_img,ws", DYADIC)
@pytest.mark.parametrize("p", [0.25, 0.5])
def test_cumulative_sum_equal_to_p_is_counted(path, n_img, ws, p):
    qp, kp = _case_inputs("equal", 1, 2, 6, n_img, n_img, 128, torch.bfloat16, n_img)
    kw = dict(n_img=n_img, nb=n_img + 2, top_k=0, p=p, text_blocks=2)
    bits, counts, got_ws = select_raw(qp, kp, workspace=ws, **kw)
    assert (got_ws is not None) == ws
    scores = got_ws if ws else sr.scores_exact(qp, kp, n_img)
    assert (scores == scores[..., :1]).all()
    assert (counts == int(p * n_img) + 1).all(), counts.unique().tolist()
    check_selection(qp, kp, scores, bits, counts, (path, n_img, p), cut_band=0.0, **kw)


def _simt_leg():
    """Child-process body: JENGA_SELECT_GEMM=simt is set, so the two-kernel paths use the SIMT GEMM."""
    for path in sorted(_TWO_KERNEL):
        for idx, case in enumerate(SEL_CASES):
            run_selection_case(path, case, idx, simt=True)
    for p in (0.25, 0.5):
        qp, kp = _case_inputs("equal", 1, 2, 6, 512, 512, 128, torch.bfloat16, 512)
        kw = dict(n_img=512, nb=514, top_k=0, p=p, text_blocks=2)
        bits, counts, ws = select_raw(qp, kp, **kw)
        assert (counts == int(p * 512) + 1).all(), counts.unique().tolist()
        check_selection(qp, kp, ws, bits, counts, ("simt dyadic", p), cut_band=0.0, **kw)
    for nq, n_img in SCORE_SHAPES:
        for dt in (torch.bfloat16, torch.float16):
            qp = _pooled(1, 3, nq, 128, dt, nq * 7 + n_img)
            kp = _pooled(1, 3, n_img + 5, 128, dt, nq + n_img * 3)
            kw = dict(n_img=n_img, nb=n_img + 2, top_k=1, p=0.3, text_blocks=2)
            bits, counts, ws = select_raw(qp, kp, **kw)
            assert torch.equal(ws.view(torch.int32), sr.scores_exact(qp, kp, n_img).view(torch.int32)), (nq, n_img)
            check_selection(qp, kp, ws, bits, counts, (nq, n_img), **kw)
    print("SIMT_OK")


def test_simt_gemm_path_matches_scores_exact_and_oracle():
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_select_edges_gpu as t; t._simt_leg()\n" % (str(ROOT), str(HERE)))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, JENGA_SELECT_GEMM="simt"),
                       capture_output=True, text=True, timeout=900)
    assert "SIMT_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


# ------------------------------------------------------------------------------------------------
# d. the shipped operator at production shapes
# ------------------------------------------------------------------------------------------------
def _staged(wl, inp, q, k):
    from jenga_b200.attention import block_sparse_attention_variant, neighbour_bits
    S = q.shape[1]
    nb = (S + 127) // 128
    tb = wl["text_blocks"]
    n_img = nb - tb
    ff = wl["first_frame"] if wl["variant"] == "wan" else 0
    pools = []
    for x in (q, k):
        if x.dtype == torch.float32:   # the Wan cast path pools every block, then ranks n_img of them
            pooled = check_pool(x, nb, (wl["name"], "fp32 pool"))[:, :, :n_img].contiguous()
        else:
            pooled = check_pool(x, n_img, (wl["name"], "pool"))
        pools.append(pooled)
    qp, kp = pools
    nbr = neighbour_bits(inp["nbr"], q.device)
    kw = dict(n_img=n_img, nb=nb, top_k=inp["top_k"], p=wl["p_remain"], text_blocks=tb, ff=ff, nbr=nbr)
    bits, counts, ws = select_raw(qp, kp, **kw)
    f_sc = check_scores_tc(qp, kp, n_img, ws, wl["name"])
    fc, ft = check_selection(qp, kp, ws, bits, counts, wl["name"], **kw)
    print(f"{wl['name']} q/k {q.dtype}: ambiguous scores {f_sc:.5f}, rows count {fc:.5f} tie {ft:.5f}")
    _, op_bits = block_sparse_attention_variant(
        wl["variant"], q, k, inp["v"], inp["top_k"], cu_seqlens_q=inp["cu"], cu_seqlens_kv=inp["cu"],
        text_blocks=tb, text_amp=wl["text_amp"], block_neighbor_list=inp["nbr"], p_remain_rates=wl["p_remain"],
        first_frame_blocks=wl["first_frame"], return_mask_bits=True)
    torch.cuda.synchronize()
    assert torch.equal(op_bits.reshape(bits.shape), bits), wl["name"]
    return f_sc, fc, ft


@pytest.mark.parametrize("name", ["hy720p", "hy_i2v", "wan14b", "wan1.3b"])
def test_shipped_workloads_staged_and_operator(name):
    import bench
    wl = bench.workload(name, 0.7)
    inp = bench.build_inputs(wl, torch.device(DEV, 0))
    legs = [(inp["q"], inp["k"])]
    if wl["variant"] == "wan":   # build_inputs gives fp32 q/k (the cast path); bf16 is the other leg
        legs.append((inp["q"].bfloat16(), inp["k"].bfloat16()))
    for q, k in legs:
        f_sc, fc, ft = _staged(wl, inp, q, k)
        # scores: these dot products cancel heavily (sum|q*k| is many times |q.k|), so the mma bound
        # leaves ~1.2 % of them between two values; rows: the fp32 cut is undecided where a flat
        # row's cumulative sum passes within 2^-16 of p (a few % of the I2V / Wan rows)
        assert f_sc < 0.02 and fc < 0.05 and ft < 0.01, (name, q.dtype, f_sc, fc, ft)


@pytest.mark.parametrize("mode", ["classic", "bulk"])
def test_hunyuan_prologue_pools_within_one_ulp_of_fp64(mode):
    from test_prologue_bulk_gpu import _run
    from jenga_b200.hyvideo import attention_prologue
    H, L, T = 24, 115200, 256
    g = torch.Generator(device=DEV).manual_seed(31)
    img = (torch.randn((1, L, 3 * H * 128), generator=g, device=DEV) * 1.5).bfloat16()
    txt = (torch.randn((1, T, 3 * H * 128), generator=g, device=DEV) * 0.7).bfloat16()
    ws = [(1 + 0.2 * torch.randn(128, generator=g, device=DEV)).bfloat16() for _ in range(4)]
    ang = torch.rand((L, 128), generator=g, device=DEV) * 6.28
    fc = (torch.cos(ang), torch.sin(ang))
    q, k, _, (qp, kp) = _run(mode, 0, lambda: attention_prologue(img, txt, H, *ws, 1e-6, fc))
    nb = (L + T + 127) // 128
    for x, pooled, what in ((q, qp, "q_pool"), (k, kp, "k_pool")):
        mean, amean = sr.pool_fp64(x, nb)
        sr.assert_pool_certified(pooled, mean, amean, (mode, what))
