"""f-3 (opt-in): INT8 Q.K^T variant of the carved attention (jenga_quantize_int8 +
jenga_carved_attn_fwd_qk_int8).  NOT the reference's arithmetic: Q and K are quantised to int8 with
per-block scales (K smoothed by its per-head mean), so the variant has its own tolerance row against
fp64 truth, derived in tests/test_qk_int8_cpu.py from a CPU model of the quantisation:
  qk_int8            mean |e| <= 2e-2 * RMS, max <= 0.15 * RMS   (about twice the modelled 1e-2 / 0.08)
  qk_int8 + pv_fp8   the FP8 P.V row, 6e-2 / 0.35
The block selection is unchanged (same mask bits as the default path)."""
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
import refutil  # noqa: E402
from test_qk_int8_cpu import KBIAS, TOL_MAX, TOL_MEAN, dequantize_ref, quantize_ref  # noqa: E402

DEV = "cuda"
SM = 128 ** -0.5


# ------------------------------------------------------------------ 1. the quantiser
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_quantiser_matches_the_torch_restatement(dtype):
    from jenga_b200.attention import quantize_int8
    g = torch.Generator().manual_seed(7)
    S, H = 1000, 3                                              # ragged: 24 pad rows
    x = (torch.randn(1, S, H, 128, generator=g) + 2.0 * KBIAS.float() / 8).to(dtype)
    # Q: no smoothing -> bit-identical codes and scales (absmax / 127 is exact)
    q8, qs, qm = quantize_int8(x.to(DEV), 64, False)
    rc, rs, _ = quantize_ref(x, 64, False)
    assert qm is None and q8.shape == (1, 1024, H, 128) and qs.shape == (H, 16)
    assert torch.equal(q8.cpu(), rc) and torch.equal(qs.cpu(), rs)
    # K: smoothed; the fp32 summation order of the mean may differ
    k8, ks, km = quantize_int8(x.to(DEV), 128, True)
    rc, rs, rm = quantize_ref(x, 128, True)
    assert ks.shape == (H, 8)
    assert torch.allclose(km.cpu(), rm, rtol=1e-5, atol=1e-6)
    assert ((ks.cpu() - rs).abs() <= 1e-5 * rs.abs()).all()
    diff = (k8.cpu().int() - rc.int()).abs()
    assert diff.max().item() <= 1 and (diff == 0).float().mean().item() >= 0.999
    # pad rows hold quant(0 - mean) of the kernel's own mean and scale
    km, ks = km.cpu(), ks.cpu()
    pad = torch.round(-km / ks[:, -1:]).clamp(-127, 127).to(torch.int8)        # [H, 128]
    assert torch.equal(k8.cpu()[0, S:], pad[None].expand(1024 - S, H, 128))


def test_quantiser_strided_input_gives_the_bytes_of_a_contiguous_copy():
    from jenga_b200.attention import quantize_int8
    g = torch.Generator(device=DEV).manual_seed(8)
    qkv = torch.randn(2, 777, 3, 4, 128, generator=g, device=DEV).bfloat16()   # packed QKV
    for which in (0, 1):
        view = qkv[:, :, which]
        for group, smooth in ((64, False), (128, True)):
            a = quantize_int8(view, group, smooth)
            b = quantize_int8(view.contiguous(), group, smooth)
            for x, y in zip(a, b):
                assert (x is None and y is None) or torch.equal(x, y)


# ------------------------------------------------------------------ 2-4. the operator vs fp64 truth
def _operator_errors(case, *, k_fn=None, q_fn=None, heads=2, seed=99):
    import bench
    from jenga_b200.attention import bits_to_onehot, block_sparse_attention_variant
    wl = bench.workload(case, 0.7)
    inp = bench.build_inputs(wl, torch.device(DEV, 0), heads=heads, seed=seed)
    q, k, v = inp["q"], inp["k"], inp["v"]
    if k_fn is not None:
        k = k_fn(k)
    if q_fn is not None:
        q = q_fn(q)
    kw = dict(cu_seqlens_q=inp["cu"], cu_seqlens_kv=inp["cu"], text_blocks=wl["text_blocks"], text_amp=wl["text_amp"],
              block_neighbor_list=inp["nbr"], p_remain_rates=wl["p_remain"], first_frame_blocks=wl["first_frame"],
              return_mask_bits=True)
    run = lambda **o: block_sparse_attention_variant(wl["variant"], q, k, v, inp["top_k"], **kw, **o)  # noqa: E731
    ref, bits = run()
    got, bits_i8 = run(qk_int8=True)
    got8, bits_i8f = run(qk_int8=True, pv_fp8=True)
    torch.cuda.synchronize()
    assert torch.equal(bits, bits_i8) and torch.equal(bits, bits_i8f)            # selection is untouched
    S = inp["S"]
    nb = (S + 127) // 128
    n_img = nb - wl["text_blocks"]
    seqlen = int(inp["cu"][1].item()) if inp["cu"] is not None else S
    blocks = sorted({0, n_img // 2, n_img - 1} | set(range(n_img, nb)))
    truth = refutil.fp64_truth(q, k, v, bits_to_onehot(bits, nb), blocks, n_img_blocks=n_img, seqlen=seqlen,
                               text_amp=wl["text_amp"])
    img = {b: t for b, t in truth.items() if b < n_img}
    txt = {b: t for b, t in truth.items() if b >= n_img}
    out = {}
    for name, o in (("bf16", ref), ("int8", got), ("int8+fp8", got8)):
        out[name] = [refutil.error_stats(o, img, seqlen_rows=seqlen)[:2]]
        if txt:
            out[name].append(refutil.error_stats(o, txt)[:2])
    return out


def _check_rows(errs, tag, really_ran=True):
    print(f"\n[qk_int8 {tag}] (max, mean)/RMS img, text: " +
          "; ".join(f"{k} " + ", ".join(f"{a:.2e}/{b:.2e}" for a, b in v) for k, v in errs.items()))
    for (b_max, b_mean), (f_max, f_mean), (g_max, g_mean) in zip(errs["bf16"], errs["int8"], errs["int8+fp8"]):
        assert f_mean <= TOL_MEAN and f_max <= TOL_MAX
        assert g_mean <= 6e-2 and g_max <= 0.35
        if really_ran:
            assert f_mean >= 2 * b_mean                                          # the int8 path really ran


@pytest.mark.parametrize("case", ["tiny", "hy_turbo_s0", "hy_i2v", "wan1.3b"])
def test_qk_int8_operator_against_fp64_truth(case):
    _check_rows(_operator_errors(case), case)


def test_smoothing_absorbs_a_common_channel_bias_of_k():
    """K carries a common channel bias three times the modelled one: the smoothed path stays in its row
    (unsmoothed, the CPU model leaves it)."""
    bias = (3.0 * KBIAS).to(DEV)
    _check_rows(_operator_errors("tiny", k_fn=lambda k: (k.double() + bias).bfloat16()), "K bias x3")


def test_per_block_scales_are_indexed_per_key_block_and_per_q_row_group():
    """Key blocks scaled by 2^-3 .. 2^3 and 64-row Q groups by 2^-1 .. 2^2 (on operands shrunk by 1/16 so
    the scores stay in range): a wrong scale index or granularity misweighs whole blocks."""
    def k_fn(k):
        f = torch.pow(2.0, (torch.arange(k.shape[1], device=DEV) // 128 % 7).float() - 3) / 8
        return (k.float() * f[None, :, None, None]).bfloat16()

    def q_fn(q):
        f = torch.pow(2.0, torch.tensor([2.0, -1.0, 1.0, 0.0], device=DEV))[torch.arange(q.shape[1], device=DEV) // 64 % 4] / 8
        return (q.float() * f[None, :, None, None]).bfloat16()
    # small scores shrink the int8 error but not the bf16 rounding of P: no 2x comparison here
    _check_rows(_operator_errors("tiny", k_fn=k_fn, q_fn=q_fn), "per-block scales", really_ran=False)


# ------------------------------------------------------------------ 5. needle rows
@pytest.mark.parametrize("path", ["bf16", "fp16", "fp8"])
def test_needle_rows_return_their_value_row_exactly(path):
    """Each query row has one key 130 log2 units above all others (also after quantisation: codes 127
    against 0), in live tiles of both ring slots: the output is that key's V row, torch.equal.  Pins the
    IGMMA descriptors, the int8 swizzle and the CTA numbering of the Q / K maps."""
    from test_attn_short_rows_gpu import _needles
    from test_attn_edges_gpu import _bits
    from jenga_b200.attention import _launch, quantize_qk_int8, quantize_v_fp8
    dtype = torch.float16 if path == "fp16" else torch.bfloat16
    q, k, v, mask, want = _needles(dtype)
    q, k, v = q.to(DEV), k.to(DEV), v.to(DEV)
    v8 = quantize_v_fp8(v) if path == "fp8" else None
    out = torch.empty(q.shape, dtype=dtype, device=DEV)
    _launch(q, k, v, _bits(mask), 1, 1, SM, 0.0, 1 << 30, k.shape[1], q.shape[1], k.shape[1], out, None, dtype,
            v_fp8=v8, qk_int8=quantize_qk_int8(q, k))
    torch.cuda.synchronize()
    bad = (out.cpu() != want).any(-1)
    assert not bad.any(), (int(bad.sum()), bad.nonzero()[:8].tolist())


# ------------------------------------------------------------------ 6. edge cases in the new mode
# The edge cases below are about the kernel's walk (tiles, mask words, limits), so they compare with fp64
# attention on the DEQUANTISED operands: what is left is the fp32 / 16-bit P rounding of the kernel, and
# the bound is the one of the default path's parity tests, not the quantisation row.
DQ_MEAN, DQ_MAX = 5e-3, 5e-2


def _launch_i8(q, k, v, bits, nq_sparse, nq_dense, *, seqlen_dev=None, kv_limit=None, q_limit=None):
    from jenga_b200.attention import _launch, quantize_qk_int8
    out = torch.zeros(q.shape, dtype=q.dtype, device=DEV)
    Sk = k.shape[1]
    _launch(q, k, v, bits, nq_sparse, nq_dense, SM, 0.0, 1 << 30, Sk if kv_limit is None else kv_limit,
            q.shape[1] if q_limit is None else q_limit, Sk, out, seqlen_dev, q.dtype,
            qk_int8=quantize_qk_int8(q, k))
    torch.cuda.synchronize()
    return out


def _live_row_errors(got, q, k, v, mask, nq_sparse, nq_dense, seqlen):
    """(max, mean)/RMS against fp64 attention on the dequantised int8 q / k over the (row block, head)
    pairs with a live tile; sparse pairs without one must be exact zeros."""
    import math
    from jenga_b200.attention import quantize_qk_int8
    q8, qs, k8, ks = (t.cpu() for t in quantize_qk_int8(q, k))
    qd = dequantize_ref(q8, qs, 64)[:, :q.shape[1]].to(q.device)
    kd = dequantize_ref(k8, ks, 128)[:, :k.shape[1]].to(q.device)
    truth = refutil.fp64_truth(qd, kd, v, mask.to(q.device), list(range(nq_sparse + nq_dense)), n_img_blocks=nq_sparse,
                               seqlen=seqlen, kv_limit_dense=seqlen)
    e_max, e_sum, cnt, sq = 0.0, 0.0, 0, 0.0
    for b, t in truth.items():
        for h in range(q.shape[2]):
            x = got[0, b * 128:(b + 1) * 128, h].double()
            if b < nq_sparse and not mask[0, h, b].any():
                assert (x == 0).all()
                continue
            e = (x - t[h]).abs()
            e_max, e_sum, cnt, sq = max(e_max, e.max().item()), e_sum + e.sum().item(), cnt + e.numel(), sq + t[h].pow(2).sum().item()
    rms = math.sqrt(sq / cnt)
    return e_max / rms, e_sum / cnt / rms


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_rows_of_zero_to_three_tiles(dtype):
    from test_attn_short_rows_gpu import NQ_SPARSE, _short_rows
    from test_attn_edges_gpu import _bits
    q, k, v, mask = _short_rows(dtype, "normal")
    q, k, v = q.to(DEV), k.to(DEV), v.to(DEV)
    got = _launch_i8(q, k, v, _bits(mask), NQ_SPARSE, 1)
    f_max, f_mean = _live_row_errors(got, q, k, v, mask, NQ_SPARSE, 1, k.shape[1])
    print(f"\n[qk_int8 short rows {dtype}] vs dequantised fp64: max {f_max:.2e} mean {f_mean:.2e}")
    assert f_mean <= DQ_MEAN and f_max <= DQ_MAX


def test_multi_word_masks_device_limits_and_determinism():
    """70 key blocks (three mask words), a ragged key count: fp64 parity on the dequantised operands; seqlen_dev gives the output of the
    same host limits bit for bit; two runs are bit-identical."""
    from test_attn_edges_gpu import _bits
    g = torch.Generator().manual_seed(21)
    H, nq, nb = 2, 3, 70
    Sk = nb * 128 - 40
    q = torch.randn(1, (nq + 1) * 128, H, 128, generator=g).bfloat16().to(DEV)
    k = torch.randn(1, Sk, H, 128, generator=g).bfloat16().to(DEV)
    v = torch.randn(1, Sk, H, 128, generator=g).bfloat16().to(DEV)
    mask = torch.rand(1, H, nq, nb, generator=g) < 0.3
    mask[0, :, :, nb - 1] = True                                  # the ragged last block, in word 2
    bits = _bits(mask)
    a = _launch_i8(q, k, v, bits, nq, 1)
    b = _launch_i8(q, k, v, bits, nq, 1)
    assert torch.equal(a, b)
    f_max, f_mean = _live_row_errors(a, q, k, v, mask, nq, 1, Sk)
    print(f"\n[qk_int8 multi-word] vs dequantised fp64: max {f_max:.2e} mean {f_mean:.2e}")
    assert f_mean <= DQ_MEAN and f_max <= DQ_MAX
    lim = Sk - 300
    host = _launch_i8(q, k, v, bits, nq, 1, kv_limit=lim, q_limit=lim)
    dev = _launch_i8(q, k, v, bits, nq, 1, seqlen_dev=torch.tensor([lim], dtype=torch.int32, device=DEV))
    assert torch.equal(host, dev)


# ------------------------------------------------------------------ 7. the installed HY path
def test_installed_path_follows_the_module_flag(monkeypatch):
    import bench
    from jenga_b200 import attention as A
    from jenga_b200.hyvideo import carved_attention_from_pools
    wl = bench.workload("tiny", 0.7)
    inp = bench.build_inputs(wl, torch.device(DEV, 0), heads=2, seed=5)
    q, k, v = inp["q"], inp["k"], inp["v"]
    nb = inp["S"] // 128
    pools = (A.block_pool(q, nb), A.block_pool(k, nb))
    kw = dict(top_k=inp["top_k"], text_blocks=wl["text_blocks"], text_amp=wl["text_amp"],
              block_neighbor_list=inp["nbr"], p_remain_rates=wl["p_remain"], cu_seqlens_q=inp["cu"])
    op_kw = dict(cu_seqlens_q=inp["cu"], cu_seqlens_kv=inp["cu"], text_blocks=wl["text_blocks"],
                 text_amp=wl["text_amp"], block_neighbor_list=inp["nbr"], p_remain_rates=wl["p_remain"])
    assert A.QK_INT8 is False
    default = carved_attention_from_pools(q, k, v, pools, **kw)
    assert torch.equal(default, A.block_sparse_attention_variant("hyvideo", q, k, v, inp["top_k"], **op_kw))
    monkeypatch.setattr(A, "QK_INT8", True)
    installed = carved_attention_from_pools(q, k, v, pools, **kw)
    monkeypatch.setattr(A, "QK_INT8", False)
    op = A.block_sparse_attention_variant("hyvideo", q, k, v, inp["top_k"], qk_int8=True, **op_kw)
    torch.cuda.synchronize()
    assert torch.equal(installed, op)
    assert not torch.equal(installed, default)
