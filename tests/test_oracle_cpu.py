"""CPU suite: pins the oracle against fixtures produced by the unmodified reference
(tests/golden/make_golden.py), and checks the C-ABI surface.  No GPU needed."""
import ctypes
import hashlib
import json
import re
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(HERE / "golden"))
import synth  # noqa: E402

from oracle import attention_oracle as orc  # noqa: E402


def sha16(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


# ------------------------------------------------------------------ attention oracle vs Triton
@pytest.mark.parametrize("name", ["hy", "wan", "amp0"])
def test_attention_oracle_matches_reference_triton(name):
    gold = np.load(HERE / "golden" / "attention_fp16.npz")
    c = synth.attention_case(name)
    assert sha16(c["mask"].numpy()) == bytes(gold[name + "/mask_sha"]).decode()
    ref = torch.from_numpy(gold[name + "/o"]).float()
    got = orc.carved_attention_rows(c["q"][:, :, :c["n_img"] * 128], c["k"], c["v"], c["mask"],
                                    c["seqlen"], 128 ** -0.5, c["amp"], c["n_img"]).float()
    rms = ref.pow(2).mean().sqrt()
    d = (got - ref).abs()
    # same algorithm, same roundings; only fp32 summation order inside the dot products differs
    assert d.max() <= 2e-3 * rms + 2.0 ** -10 * ref.abs().max(), (d.max() / rms).item()
    assert d.mean() <= 1e-4 * rms
    assert (got[:, :, c["seqlen"]:] == 0).all()


# ------------------------------------------------------------------ whole-operator oracle vs reference
@pytest.mark.parametrize("name", [n for n, *_ in synth.OPERATOR_CASES])
def test_operator_oracle_matches_reference_block_sparse_attention(name):
    """oracle.block_sparse_attention against the output of the reference's own
    block_sparse_attention (glue + mask builder + Triton kernel + text rows; fixture made by
    tests/golden/make_golden.py operator): layout ([B,S,H*D] vs shape_xfuse), cu_seqlens handling,
    I2V padding/trim and the selection all have to agree for the values to agree."""
    gold = np.load(HERE / "golden" / "operator_fp16.npz")
    c = synth.operator_case(name)
    ref = torch.from_numpy(gold[name + "/o"])
    got = orc.block_sparse_attention(
        c["q"], c["k"], c["v"], c["top_k"], cu_seqlens_q=c["cu"], cu_seqlens_kv=c["cu"],
        text_blocks=c["text_blocks"], text_amp=c["amp"], block_neighbor_list=c["nbr"],
        shape_xfuse=c["xfuse"], p_remain_rates=c["p"],
        variant="i2v" if c["variant"] == "hyvideo_i2v" else "hyvideo")
    assert got.shape == ref.shape and got.dtype == ref.dtype
    ref, got = ref.float(), got.float()
    rms = ref.pow(2).mean().sqrt()
    d = (got - ref).abs()
    assert d.max() <= 5e-3 * rms + 2.0 ** -10 * ref.abs().max(), (d.max() / rms).item()
    assert d.mean() <= 2e-4 * rms, (d.mean() / rms).item()


# ------------------------------------------------------------------ fp64 truth of the GPU tests vs oracle
@pytest.mark.parametrize("seqlen", [128 + 50, 3 * 128 + 70])
def test_fp64_truth_matches_oracle_on_float64_inputs(seqlen):
    """tests/refutil.fp64_truth is the exact reference the kernel edge tests judge against.  On
    float64 inputs the oracle rounds nothing below fp32, so the two must agree to fp32 accuracy
    (~1e-6 of the output RMS; bound 1e-5): batch > 1, Sq != Sk, a ragged last key block, the
    sparse limits inside a key block and inside a query block, text_amp on key blocks that start
    elsewhere than the image query blocks, dense rows with and without a key limit, and the
    natural-log LSE of the dense rows (against an independent numpy logaddexp)."""
    sys.path.insert(0, str(HERE))
    import refutil
    g = torch.Generator().manual_seed(5)
    B, H, D, n_img, n_txt = 2, 3, 128, 2, 1
    Sq, Sk = (n_img + n_txt) * 128, 4 * 128 + 40
    nb = (Sk + 127) // 128
    q, k, v = (torch.randn(B, S, H, D, generator=g, dtype=torch.float64) for S in (Sq, Sk, Sk))
    mask = torch.rand(B, H, n_img, nb, generator=g) < 0.5
    mask[..., 0] = True
    amp, text_start = 0.7, 3
    kp, vp = (refutil.pad_rows(x, nb * 128).transpose(1, 2) for x in (k, v))
    qh = q.transpose(1, 2)
    img = orc.carved_attention_rows(qh[:, :, :n_img * 128], kp, vp, mask, seqlen, D ** -0.5, amp, text_start)
    for kv_dense in (None, Sk):
        txt = orc.dense_attention_rows(qh[:, :, n_img * 128:], kp, vp, D ** -0.5, kv_dense)
        want = torch.cat([img, txt], dim=2)                                    # [B,H,Sq,D]
        got, lse = refutil.fp64_truth(q, k, v, mask, list(range(n_img + n_txt)), n_img_blocks=n_img, seqlen=seqlen,
                                      text_amp=amp, text_block_start=text_start, q_limit=seqlen,
                                      kv_limit_dense=kv_dense, return_lse=True)
        got = torch.cat([got[i] for i in range(n_img + n_txt)], dim=2)
        rms = want.pow(2).mean().sqrt().item()
        assert (got - want).abs().max().item() <= 1e-5 * rms, (got - want).abs().max().item() / rms
        assert (got[:, :, seqlen:n_img * 128] == 0).all()
        s = (qh[:, :, n_img * 128:] @ kp.transpose(-1, -2)).numpy() * D ** -0.5
        if kv_dense is not None:
            s[..., kv_dense:] = -np.inf
        assert np.allclose(lse[n_img].numpy(), np.logaddexp.reduce(s, axis=-1), rtol=0, atol=1e-10)


# ------------------------------------------------------------------ mask-builder oracle vs torch
def assert_masks_equal_modulo_ties(got, ref, probs, n_img):
    """Selection parity contract (SURVEY §8c-v): identical masks, except that inside ONE group
    of exactly tied probabilities the reference's unstable sort may pick different members."""
    assert got.shape == ref.shape
    diff = got != ref
    assert not diff[..., n_img:].any()  # text / condition columns are exact
    rows = diff.any(-1).nonzero()
    for b, h, m in rows.tolist():
        cols = diff[b, h, m, :n_img].nonzero().flatten()
        pv = probs[b, h, m, cols]
        assert (pv == pv[0]).all(), ("non-tie mismatch", b, h, m, cols.tolist(), pv.tolist())
        # the tie group straddles the cut: same number taken by both, up to blocks that the
        # neighbour / first-frame union already covered
        assert abs(int(got[b, h, m].sum()) - int(ref[b, h, m].sum())) <= len(cols)
    return len(rows)


@pytest.mark.parametrize("name", [n for n, *_ in synth.MASK_CASES])
def test_mask_oracle_matches_reference_builder(name):
    gold = np.load(HERE / "golden" / "mask_builder.npz")
    c = synth.mask_case(name)
    nb = c["n_img"] + c["n_txt"]
    ref = torch.from_numpy(gold[name + "/mask"])
    for tb in ("low", "high"):
        got, probs = orc.build_block_onehot(c["q"][:, :, :c["n_img"] * 128], c["k"], c["top_k"],
                                            c["n_img"], nb, c["p"], c["n_txt"], c["nbr"], c["ff"],
                                            tie_break=tb, return_probs=True)
        n_rows = assert_masks_equal_modulo_ties(got, ref, probs, c["n_img"])
        assert n_rows <= 0.1 * ref.shape[1] * ref.shape[2]


# ------------------------------------------------------------------ C-ABI surface
def test_cabi_exports_every_declared_symbol_at_abi_3():
    from jenga_b200 import build
    lib_path = build.build()
    lib = ctypes.CDLL(str(lib_path))
    header = (ROOT / "include" / "jenga_b200.h").read_text()
    names = set(re.findall(r"\b(jenga_[a-z0-9_]+)\s*\(", header))
    assert len(names) >= 6
    for n in sorted(names):
        assert hasattr(lib, n), f"{n} declared in include/jenga_b200.h but not exported"
    lib.jenga_abi_version.restype = ctypes.c_int
    assert lib.jenga_abi_version() == 3


def test_attention_call_fails_loudly_without_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from jenga_b200.attention import carved_attention_fwd
    from jenga_b200._lib import JengaError
    q = torch.zeros(1, 128, 1, 128, dtype=torch.bfloat16)
    with pytest.raises(JengaError):
        carved_attention_fwd(q, q, q, None, 0, 1, 0.1)


# ------------------------------------------------------------------ gilbert (product C++) vs reference
def _ours(t, h, w, sliced):
    from jenga_b200._lib import lib
    n = t * h * w
    a = np.zeros(n, dtype=np.int64)
    b = np.zeros(n, dtype=np.int64)
    assert lib.jenga_gilbert_mapping_host(t, h, w, sliced, a.ctypes.data, b.ctypes.data) == 0
    nb = (n + 127) // 128
    nbr = np.zeros((nb, nb), dtype=np.uint8)
    assert lib.jenga_gilbert_block_neighbors_host(t, h, w, 128, sliced, nbr.ctypes.data) == 0
    return a, b, nbr.astype(np.bool_)


def test_gilbert_tables_bit_exact_vs_reference():
    cases = json.loads((HERE / "golden" / "gilbert.json").read_text())
    small = np.load(HERE / "golden" / "gilbert_small.npz")
    for name, c in cases.items():
        a, b, nbr = _ours(c["t"], c["h"], c["w"], c["sliced"])
        assert sha16(a) == c["l2h_sha"], name
        assert sha16(b) == c["h2l_sha"], name
        assert sha16(nbr) == c["nbr_sha"], name
        assert int(nbr.sum()) == c["nbr_popcount"] and int(nbr.sum(1).max()) == c["nbr_row_max"]
        assert a[:8].tolist() == c["l2h_head"]
        if name + "/l2h" in small:
            assert (small[name + "/l2h"] == a).all() and (small[name + "/h2l"] == b).all()
            assert (small[name + "/nbr"] == nbr).all()
        # permutation property
        assert (b[a] == np.arange(a.size)).all()


# ------------------------------------------------------------------ gilbert oracle (C restatement)
def _oracle_lib():
    import subprocess
    subprocess.run(["make", "-C", str(ROOT / "oracle"), "-s"], check=True)
    lib = ctypes.CDLL(str(ROOT / "oracle" / "_build" / "libgilbert_oracle.so"))
    lib.oracle_gilbert_xyz2d.restype = ctypes.c_long
    lib.oracle_gilbert_xyz2d.argtypes = [ctypes.c_long] * 6
    return lib


def _oracle_tables(lib, t, h, w, sliced):
    n = t * h * w
    a = np.zeros(n, dtype=np.int64)
    b = np.zeros(n, dtype=np.int64)
    assert lib.oracle_gilbert_mapping(t, h, w, sliced, a.ctypes.data_as(ctypes.c_void_p),
                                      b.ctypes.data_as(ctypes.c_void_p)) == 0
    nb = (n + 127) // 128
    nbr = np.zeros((nb, nb), dtype=np.uint8)
    assert lib.oracle_gilbert_block_neighbors(t, h, w, 128, sliced, nbr.ctypes.data_as(ctypes.c_void_p)) == 0
    return a, b, nbr.astype(np.bool_)


def test_gilbert_oracle_pinned_by_reference_goldens_and_agrees_with_product():
    lib = _oracle_lib()
    cases = json.loads((HERE / "golden" / "gilbert.json").read_text())
    for name, c in cases.items():
        a, b, nbr = _oracle_tables(lib, c["t"], c["h"], c["w"], c["sliced"])
        assert (sha16(a), sha16(b), sha16(nbr)) == (c["l2h_sha"], c["h2l_sha"], c["nbr_sha"]), name
    # product (curve walker) vs oracle (per-voxel queries) on shapes the fixtures do not hold:
    # odd sizes, degenerate axes, each axis being the longest
    for t, h, w, sliced in [(1, 1, 1, 0), (1, 1, 7, 0), (2, 3, 5, 0), (9, 4, 3, 0), (3, 10, 4, 0),
                            (5, 5, 5, 0), (6, 7, 15, 0), (1, 9, 14, 1), (4, 5, 3, 1), (3, 16, 16, 1)]:
        pa, pb, pn = _ours(t, h, w, sliced)
        oa, ob, on = _oracle_tables(lib, t, h, w, sliced)
        assert (pa == oa).all() and (pb == ob).all() and (pn == on).all(), (t, h, w, sliced)
        # scalar entry point
        from jenga_b200._lib import lib as plib
        if not sliced:
            for (x, y, z) in [(0, 0, 0), (w - 1, h - 1, t - 1), (w // 2, h // 2, t // 2)]:
                assert plib.jenga_gilbert_xyz2d(x, y, z, w, h, t) == lib.oracle_gilbert_xyz2d(x, y, z, w, h, t)


def test_gilbert_product_equals_oracle_on_random_grids():
    """Property test (hypothesis): for arbitrary small grids — odd sizes, unit axes, every axis
    order — the O(N) curve walker of the product and the per-voxel C restatement (pinned to the
    reference above) produce identical tables; the tables are inverse permutations; the curve is
    local (almost every step is a unit lattice step; the generalized curve has a few diagonal /
    longer steps on odd sizes, which the reference has too); the block adjacency is symmetric with
    a full diagonal."""
    from hypothesis import given, settings, strategies as st
    lib = _oracle_lib()

    @settings(max_examples=60, deadline=None, derandomize=True)
    @given(st.integers(1, 9), st.integers(1, 12), st.integers(1, 12), st.integers(0, 1))
    def check(t, h, w, sliced):
        pa, pb, pn = _ours(t, h, w, sliced)
        oa, ob, on = _oracle_tables(lib, t, h, w, sliced)
        assert (pa == oa).all() and (pb == ob).all() and (pn == on).all(), (t, h, w, sliced)
        n = t * h * w
        assert sorted(pa.tolist()) == list(range(n))
        assert (pb[pa] == np.arange(n)).all()
        assert (pn == pn.T).all() and pn.diagonal().all()
        if not sliced and n > 1:
            z, rem = np.divmod(pb, h * w)
            y, x = np.divmod(rem, w)
            step = np.abs(np.diff(x)) + np.abs(np.diff(y)) + np.abs(np.diff(z))
            assert step.min() >= 1 and (step == 1).mean() >= 0.9

    check()


def test_gilbert_python_wrappers_mirror_reference_api():
    from jenga_b200 import gilbert as g
    l2h, h2l = g.gilbert_mapping(4, 6, 8)
    assert isinstance(l2h, list) and l2h[:8] == [0, 1, 26, 25, 166, 165, 190, 191]
    assert h2l[:4] == [0, 1, 9, 8]
    nbr = g.gilbert_block_neighbor_mapping(4, 6, 8)
    assert nbr.dtype == torch.bool and tuple(nbr.shape) == (2, 2)
    sl, _ = g.sliced_gilbert_mapping(3, 5, 4)
    assert sorted(sl) == list(range(60))
    with pytest.raises(ValueError):
        g.gilbert_mapping(2, 2, 2, transpose_order=[2, 1, 1])         # gilbert.py:294-295
    with pytest.raises(NotImplementedError):
        g.block_wise_mapping(2, 2, 2)                                 # plotting/experiment helper


def test_transposed_curves_match_reference_goldens():
    """transpose_gilbert_mapping and every transpose_order argument (gilbert.py:274-330,:436-438,
    :484-486,:704) — bit-exact against tables produced by the unmodified reference."""
    import hashlib
    import json
    from jenga_b200 import gilbert as g
    gold = json.loads((HERE / "golden" / "gilbert_transpose.json").read_text())
    assert len(gold) >= 6

    def sha(a):
        return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]
    for key, c in gold.items():
        (t, h, w), order = c["dims"], c["order"]
        l2h, h2l = g.transpose_gilbert_mapping(c["dims"], order)
        assert l2h == c["l2h"] and h2l == c["h2l"], key
        assert sha(np.asarray(g.gilbert_mapping(t, h, w, order)[0], dtype=np.int64)) == c["gilbert_mapping_l2h_sha"]
        assert sha(np.asarray(g.sliced_gilbert_mapping(t, h, w, order)[0], dtype=np.int64)) == c["sliced_mapping_l2h_sha"]
        assert sha(g.gilbert_block_neighbor_mapping(t, h, w, 16, order).numpy()) == c["nbr16_sha"], key
        assert sha(g.sliced_gilbert_block_neighbor_mapping(t, h, w, 16, order).numpy()) == c["sliced_nbr16_sha"], key


def test_block_neighbour_csr_equals_dense_matrix():
    """f-4: CSR form of the adjacency (row_ptr, ascending col_idx) == the dense matrix, whose SHA is
    pinned against the reference in gilbert.json."""
    from jenga_b200 import gilbert as g
    for (t, h, w, sliced) in ((4, 6, 8, False), (8, 11, 13, True), (32, 22, 40, False)):
        dense = g.block_neighbor_mapping(t, h, w, 128, sliced)
        rp, ci = g.block_neighbor_csr(t, h, w, 128, sliced)
        assert rp.dtype == torch.int32 and ci.dtype == torch.int32
        assert int(rp[-1]) == int(dense.sum()) == ci.numel()
        rows = torch.repeat_interleave(torch.arange(dense.shape[0]), (rp[1:] - rp[:-1]).long())
        back = torch.zeros_like(dense)
        back[rows, ci.long()] = True
        assert torch.equal(back, dense)
        assert all(ci[rp[i]:rp[i + 1]].tolist() == sorted(ci[rp[i]:rp[i + 1]].tolist()) for i in range(dense.shape[0]))


def test_install_hook_preseeds_reference_module_names():
    """The drop-in hook: after install() the names the reference binds at import time resolve to
    jenga_b200 (no GPU needed to check the wiring)."""
    import importlib
    saved = {k: sys.modules.get(k) for k in list(sys.modules)
             if k.split(".")[0] in ("flash_attn", "gilbert", "hyvideo", "hyvideo_i2v", "wan")}
    try:
        from jenga_b200 import install
        names = install.install()
        assert "hyvideo.modules.attention_block_triton_diffres" in names
        m = importlib.import_module("hyvideo.modules.attention_block_triton_diffres")
        assert m.__jenga_b200__ and callable(m.block_sparse_attention)
        import inspect
        sig = inspect.signature(m.block_sparse_attention)
        # reference signature (hyvideo/modules/attention_block_triton_diffres.py:399-415)
        assert list(sig.parameters)[:15] == [
            "query", "key", "value", "top_k", "block_size_M", "block_size_N", "cu_seqlens_q",
            "cu_seqlens_kv", "max_seqlen_q", "max_seqlen_kv", "text_blocks", "text_amp",
            "block_neighbor_list", "shape_xfuse", "p_remain_rates"]
        assert sig.parameters["text_blocks"].default == 2 and sig.parameters["p_remain_rates"].default == 0.5
        w = importlib.import_module("wan.modules.attention_block_triton_diffres")
        ws = inspect.signature(w.block_sparse_attention)
        assert ws.parameters["text_blocks"].default == 0 and ws.parameters["p_remain_rates"].default == 0.9
        assert "first_frame_blocks" in ws.parameters
        i2v = importlib.import_module("hyvideo_i2v.modules.attention_block_triton_diffres")
        assert inspect.signature(i2v.block_sparse_attention).parameters["text_blocks"].default == 4
        fa = importlib.import_module("flash_attn.flash_attn_interface")
        assert callable(fa.flash_attn_varlen_func)
        import flash_attn
        assert flash_attn.__version__.startswith("2.")
        g = importlib.import_module("gilbert")
        assert g.gilbert_mapping(2, 2, 2) == ([0, 7, 1, 6, 3, 4, 2, 5], [0, 2, 6, 4, 5, 7, 3, 1])  # = reference
        # every name the four reference scripts import from gilbert (jenga_hyvideo.py:24,
        # jenga_hyi2v.py:26, jenga_hyvideo_multigpu.py:22, jenga_wan.py:34)
        for name in ("transpose_gilbert_mapping", "gilbert_mapping", "gilbert_block_neighbor_mapping",
                     "sliced_gilbert_block_neighbor_mapping", "sliced_gilbert_mapping"):
            assert callable(getattr(g, name)), name
        x = importlib.import_module("hyvideo.modules.xdit_ring_atten")
        assert hasattr(x, "xFuserLongContextAttention")
    finally:
        for k in list(sys.modules):
            if k.split(".")[0] in ("flash_attn", "gilbert", "hyvideo", "hyvideo_i2v", "wan"):
                del sys.modules[k]
        for k, v in saved.items():
            if v is not None:
                sys.modules[k] = v


def test_step_skip_schedule_matches_reference_lists():
    """jenga_hyvideo.py:28 + stage switch: 23 computed steps of 50, drop rate switches after
    step 25, 60 blocks per computed step -> 1380 hot-path calls per video."""
    from jenga_b200 import dit_loop
    s = dit_loop.schedule()
    computed = [i for i, c, _ in s if c]
    assert computed == list(dit_loop.NON_SKIP_STEPS) and len(computed) == 23
    assert {d for i, c, d in s if i <= 25} == {0.7} and {d for i, c, d in s if i > 25} == {0.8}
    assert len(computed) * (dit_loop.DOUBLE_BLOCKS + dit_loop.SINGLE_BLOCKS) == 1380


def test_install_launcher_runs_a_script_with_the_hook(tmp_path):
    """`python -m jenga_b200.install script.py args…` — the launcher form of the drop-in hook."""
    import subprocess
    script = tmp_path / "fake_jenga_script.py"
    script.write_text(
        "import sys\n"
        "from gilbert import transpose_gilbert_mapping, gilbert_mapping, gilbert_block_neighbor_mapping\n"
        "from gilbert import gilbert_mapping, sliced_gilbert_block_neighbor_mapping, sliced_gilbert_mapping, "
        "gilbert_block_neighbor_mapping\n"
        "import flash_attn\n"
        "from hyvideo.modules.attention_block_triton_diffres import block_sparse_attention\n"
        "l2h, h2l = gilbert_mapping(4, 6, 8)\n"
        "print('HOOK', l2h[:4], flash_attn.__version__, block_sparse_attention.__doc__, sys.argv[1:])\n")
    r = subprocess.run([sys.executable, "-m", "jenga_b200.install", str(script), "--video-size", "720"],
                       capture_output=True, text=True, cwd=str(ROOT), timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "HOOK [0, 1, 26, 25]" in r.stdout and "jenga_b200 drop-in (hyvideo variant)" in r.stdout
    assert "['--video-size', '720']" in r.stdout


def test_host_block_count_rules_match_reference_arithmetic():
    """a-7 (SURVEY §8a): the top_k / first-frame rules are plain host arithmetic with float
    truncation quirks — models_mul…:242,249-251 and wan/modules/model_mul.py:161-164."""
    from jenga_b200 import wan
    from jenga_b200.hyvideo import select_block_num
    assert select_block_num(0.7, 115200) == 270
    assert select_block_num(0.75, 115200) == 225
    assert select_block_num(0.8, 115200) == 179        # int(0.2 * 900) = 179: 0.19999999999999996 * 900
    assert select_block_num(0.85, 115200) == 135
    assert select_block_num(0.75, 63360) == 123        # Turbo stage 0, single GPU
    assert select_block_num(0.75, 7920, world_size=8) == 120   # SP: 8 * int(0.25 * 61)
    assert select_block_num(0.85, 14400, world_size=8) == 128  # SP: 8 * int(0.15 * 112)
    assert wan.block_counts(32760, 0.5) == (128, 12)   # Wan-1.3B: 256 blocks
    assert wan.block_counts(75600, 0.7) == (177, 28)   # Wan-14B: 591 blocks
    assert wan.block_counts(75600, 0.8) == (118, 28)
