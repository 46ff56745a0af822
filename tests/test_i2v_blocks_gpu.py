"""HunyuanVideo-I2V fused block path on the GPU.

* Kernels: the token-replace forms of ln_modulate / gate_residual select each row's parameters and
  change nothing else — every row is bit-identical to the plain kernel run with that row's
  parameters — and they reproduce the reference's own masked `modulate` / `apply_gate`
  (hyvideo_i2v/modules/modulate_layers.py:51-56,84-95) under autocast: the gate bit-exact,
  modulate within the bound test_dense_fused_gpu.py applies to ln_modulate.
* Prologue at ragged S = L + 400: the pooled rows of the last, partial block are the zero-padded
  means of the I2V mask builder (attention_block_triton_diffres.py:216-217,324-327), within the bound
  test_prologue_gpu.py applies to pools.
* Drop-in: the unmodified hyvideo_i2v/modules/models_mul.py blocks, A = reference operator (Triton +
  FA2), B = through install(), same weights, the tolerance of test_dropin_blocks_gpu.py."""
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(ROOT))

from test_dense_fused_gpu import _ulp_stats  # noqa: E402
from test_dropin_blocks_gpu import (_capture_reference_masks, _compare, _reinit,  # noqa: E402
                                    _rows_with_equal_masks, _structured_tokens)


def _ref_modulate_layers():
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    return R.import_by_path("_jenga_ref_i2v_modulate_layers", "hyvideo_i2v/modules/modulate_layers.py")


def _mask(kind, rows, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "all":
        return torch.ones(rows, dtype=torch.bool, device="cuda")
    if kind == "none":
        return torch.zeros(rows, dtype=torch.bool, device="cuda")
    return torch.rand(rows, generator=g, device="cuda") < 0.3             # scattered


def _vec(C, g, s=0.3):
    return (s * torch.randn(1, C, generator=g, device="cuda")).bfloat16()


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["all", "none", "scattered"])
@pytest.mark.parametrize("L,C,strided", [(2048 + 37, 3072, False), (515, 3072, True), (1001, 1536, False)])
def test_ln_modulate_tr_rows_equal_the_plain_kernel(kind, L, C, strided):
    from jenga_b200 import dense as DN
    g = torch.Generator(device="cuda").manual_seed(L + C)
    x = (torch.randn(1, L, C, generator=g, device="cuda") * 1.7 + 0.3).bfloat16()
    if strided:
        wide = torch.zeros(1, L, C + 64, dtype=torch.bfloat16, device="cuda")
        wide[:, :, 32:32 + C] = x
        x = wide[:, :, 32:32 + C]
    shift, scale, tr_shift, tr_scale = (_vec(C, g) for _ in range(4))
    mask = _mask(kind, L, L)
    plain = DN.ln_modulate(x, shift, scale)
    tr_only = DN.ln_modulate(x, tr_shift, tr_scale)
    got = DN.ln_modulate(x, shift, scale, tr=(tr_shift, tr_scale, mask))
    assert torch.equal(got, torch.where(mask[None, :, None], tr_only, plain))
    # a CPU mask gives the same rows; its device copy is made once and reused
    cpu = mask.cpu()
    assert torch.equal(DN.ln_modulate(x, shift, scale, tr=(tr_shift, tr_scale, cpu)), got)
    assert DN._row_mask(cpu, x.device) is DN._row_mask(cpu, x.device)


@pytest.mark.parametrize("kind", ["all", "none", "scattered"])
@pytest.mark.parametrize("L,C,strided", [(3001, 3072, False), (515, 3072, True)])
def test_gate_residual_tr_rows_equal_the_plain_kernel(kind, L, C, strided):
    from jenga_b200 import dense as DN
    g = torch.Generator(device="cuda").manual_seed(L + 7)
    x = torch.randn(1, L, C, generator=g, device="cuda").bfloat16()
    y = torch.randn(1, L, C + 128, generator=g, device="cuda").bfloat16()
    y = y[:, :, 64:64 + C] if strided else y[:, :, :C].contiguous()
    gate, tr_gate = _vec(C, g, 1.0), _vec(C, g, 1.0)
    mask = _mask(kind, L, L + 1)
    want = torch.where(mask[None, :, None], DN.gate_residual(x, y, tr_gate), DN.gate_residual(x, y, gate))
    assert torch.equal(DN.gate_residual(x, y, gate, tr=(tr_gate, mask)), want)
    assert torch.equal(DN.gate_residual(x, y, gate, tr=(tr_gate, mask.cpu())), want)


@pytest.mark.parametrize("kind", ["all", "none", "scattered"])
def test_token_replace_chains_match_the_reference_functions(kind):
    """modulate_layers.py's own `modulate` / `apply_gate` with condition_type="token_replace" and a
    first_frame_mask (they write into their input: given a clone) under autocast"""
    ML = _ref_modulate_layers()
    from jenga_b200 import dense as DN
    L, C = 2048 + 37, 3072
    g = torch.Generator(device="cuda").manual_seed(9)
    x = (torch.randn(1, L, C, generator=g, device="cuda") * 1.7 + 0.3).bfloat16()
    y = torch.randn(1, L, C, generator=g, device="cuda").bfloat16()
    shift, scale, tr_shift, tr_scale = (_vec(C, g) for _ in range(4))
    gate, tr_gate = _vec(C, g, 1.0), _vec(C, g, 1.0)
    mask = _mask(kind, L, 10)
    norm = torch.nn.LayerNorm(C, elementwise_affine=False, eps=1e-6).cuda()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        mid = ML.modulate(norm(x).clone(), shift=shift, scale=scale, condition_type="token_replace",
                          tr_shift=tr_shift, tr_scale=tr_scale, first_frame_mask=mask)
        assert mid.dtype == torch.float32
        ref = mid.to(torch.bfloat16)                        # the cast the following Linear applies
        tr = (tr_shift, tr_scale, mask)
        assert DN.ln_modulate_supported(x, norm, shift, scale, tr=tr)
        got = DN.ln_modulate(x, shift, scale, eps=norm.eps, tr=tr)
        gref = x + ML.apply_gate(y.clone(), gate=gate, condition_type="token_replace", tr_gate=tr_gate,
                                 first_frame_mask=mask)
        assert DN.gate_residual_supported(x, y, gate, tr=(tr_gate, mask))
        ggot = DN.gate_residual(x, y, gate, tr=(tr_gate, mask))
    mx, same = _ulp_stats(got, ref)
    d = (got.float() - ref.float()).abs()
    bad = (d > 2.0 ** -7 * ref.float().abs() + 4e-6).sum().item()
    print(f"\n[ln_modulate_tr {kind}] max ulp distance {mx}, identical {same:.5f}, beyond 1 ulp / 4e-6: {bad}")
    assert bad == 0 and same >= 0.999
    assert torch.equal(ggot, gref)


# ------------------------------------------------------------------------------------------------
# prologue at ragged S
# ------------------------------------------------------------------------------------------------
def test_prologue_pools_the_partial_last_block_like_the_i2v_builder():
    from jenga_b200.hyvideo import attention_prologue
    L, T, H, D = 2048 + 64, 400, 4, 128                  # S = 2512: the last block holds 80 rows
    g = torch.Generator(device="cuda").manual_seed(21)
    img = torch.randn(1, L, 3 * H * D, generator=g, device="cuda").bfloat16()
    txt = torch.randn(1, T, 3 * H * D, generator=g, device="cuda").bfloat16()
    w = [(1.0 + 0.2 * torch.randn(D, generator=g, device="cuda")).bfloat16() for _ in range(4)]
    ang = torch.rand(L, 64, generator=g, device="cuda") * 6.2831853
    freqs = (torch.cos(ang).repeat_interleave(2, 1).contiguous(), torch.sin(ang).repeat_interleave(2, 1).contiguous())
    q, k, _, (qp, kp) = attention_prologue(img, txt, H, *w, 1e-6, freqs)
    S = L + T
    nb = (S + 127) // 128
    assert S % 128 and qp.shape[2] == nb
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for x, pool in ((q, qp), (k, kp)):
            # attention_block_triton_diffres.py:314-327 (transpose, zero pad), :216-217 (block means)
            xp = torch.nn.functional.pad(x.transpose(1, 2), [0, 0, 0, nb * 128 - S, 0, 0, 0, 0])
            ref = xp.reshape(1, H, nb, 128, D).mean(dim=-2)
            bound = 2.0 ** -8 * ref.float().abs().max() + 1e-6
            assert (pool.float() - ref.float()).abs().max() <= bound
            assert (pool[:, :, -1].float() - ref[:, :, -1].float()).abs().max() <= bound


# ------------------------------------------------------------------------------------------------
# drop-in: the unmodified I2V blocks, reference operator vs install()
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def i2v_modules():
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    from i2v_ref import load_i2v_blocks
    ref = load_i2v_blocks(product=False)
    ours = load_i2v_blocks(product=True)
    assert not getattr(ref.MMDoubleStreamBlock.forward, "__jenga_b200__", False)
    assert ours.MMDoubleStreamBlock.forward.__jenga_b200__
    assert "_triton_block_sparse_attention_onehot" in ref.block_sparse_attention.__globals__
    yield ref, ours
    from jenga_b200 import blocks
    blocks.remove_gather_hook()


def _i2v_case(mod, T, valid):
    from jenga_b200 import gilbert
    t, h, w = 8, 16, 16
    L, C, H = t * h * w, 512, 4
    l2h, h2l = gilbert.mapping_tensors(t, h, w)
    nbr = gilbert.block_neighbor_mapping(t, h, w)
    h2l = h2l.cuda()
    curve_sel = [[l2h.cuda(), h2l, nbr]]
    img = _structured_tokens(L, C, 1)
    txt = _structured_tokens(-(-T // 128) * 128, C, 2, gain=0.5)[:, :T].contiguous()   # T = 400: ragged
    gen = torch.Generator(device="cuda").manual_seed(3)
    vec = torch.randn(1, C, generator=gen, device="cuda").bfloat16()
    tr_vec = torch.randn(1, C, generator=gen, device="cuda").bfloat16()
    text_mask = torch.zeros(1, T, dtype=torch.int64, device="cuda")
    text_mask[:, :valid] = 1
    cu = mod.get_cu_seqlens(text_mask, L)
    ang = torch.rand(L, 64, generator=torch.Generator(device="cuda").manual_seed(4), device="cuda") * 6.2831853
    freqs = (torch.cos(ang).repeat_interleave(2, dim=1).contiguous(), torch.sin(ang).repeat_interleave(2, dim=1).contiguous())
    # jenga_hyi2v.py:124-130: the first frame in Hilbert order (device, over L), and the CPU mask over L+T
    ff = torch.zeros(L, dtype=torch.bool, device="cuda")
    ff[:h * w] = True
    ff = ff[h2l]
    full = torch.zeros(L + T).bool()
    full[:L] = ff.cpu()
    return dict(L=L, T=T, C=C, H=H, curve_sel=curve_sel, img=img, txt=txt, vec=vec, tr_vec=tr_vec, cu=cu,
                freqs=freqs, ff=ff, full=full, hw=h * w)


def _run_blocks(ref_mod, ours_mod, kind, c, condition_type, qk_int8=False):
    from jenga_b200 import attention as A, blocks
    cls = "MMDoubleStreamBlock" if kind == "double" else "MMSingleStreamBlock"
    mk = lambda m: getattr(m, cls)(c["C"], c["H"], mlp_width_ratio=4.0, dtype=torch.bfloat16, device="cuda")  # noqa: E731
    ref_blk, our_blk = mk(ref_mod), mk(ours_mod)
    _reinit(ref_blk, 11)
    our_blk.load_state_dict(ref_blk.state_dict())
    S = c["L"] + c["T"]
    tr = condition_type == "token_replace"
    mask = (c["ff"] if kind == "double" else c["full"]) if tr else None
    tail = (0.7, mask, condition_type, c["tr_vec"] if tr else None, c["hw"] if tr else None, 0.431, c["curve_sel"], 0.3)
    rec, undo = _capture_reference_masks(ref_mod.block_sparse_attention)
    before = dict(blocks.STATS)
    A.MASK_CAPTURE = []
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            if kind == "double":
                head = (c["img"], c["txt"], c["vec"], c["cu"], c["cu"], S, S, c["freqs"])
                ra = ref_blk(*head, *tail)
                oa = our_blk(*head, *tail)
                if qk_int8:
                    A.QK_INT8 = True
                    o8 = our_blk(*head, *tail)
            else:
                x = torch.cat([c["img"], c["txt"]], 1)
                head = (x, c["vec"], c["T"], c["cu"], c["cu"], S, S, c["freqs"])
                ra = (ref_blk(*head, *tail),)
                oa = (our_blk(*head, *tail),)
                if qk_int8:
                    A.QK_INT8 = True
                    o8 = (our_blk(*head, *tail),)
        torch.cuda.synchronize()
        bits, nb = A.MASK_CAPTURE[0]
    finally:
        A.QK_INT8 = False
        A.MASK_CAPTURE = None
        undo()
    key = "i2v_double" if kind == "double" else "i2v_single"
    assert blocks.STATS[key] == before[key] + (2 if qk_int8 else 1), "the fused I2V forward did not run"
    assert blocks.STATS["fallback"] == before["fallback"]
    assert len(rec) == 1 and nb == (S + 127) // 128
    n_img = nb - 4                                       # the I2V operator's text_blocks=4, whatever T is
    same_blocks = _rows_with_equal_masks(rec[0], bits, nb)
    # image rows past n_img*128 (T=256: the last two image blocks) are dense rows: no mask to compare
    row_ok = torch.cat([same_blocks.repeat_interleave(128),
                        torch.ones(max(0, c["L"] - n_img * 128), dtype=torch.bool, device="cuda")])[:c["L"]]
    split = lambda o: (o[0][:, :c["L"]], o[1] if kind == "double" else o[0][:, c["L"]:])  # noqa: E731
    return split(ra), split(oa), (split(o8) if qk_int8 else None), row_ok


@pytest.mark.parametrize("kind", ["double", "single"])
@pytest.mark.parametrize("condition_type,T,valid", [("token_replace", 400, 300), (None, 400, 300),
                                                    ("token_replace", 256, 180)])
def test_unmodified_i2v_blocks_through_install_hook(i2v_modules, kind, condition_type, T, valid):
    ref_mod, ours_mod = i2v_modules
    c = _i2v_case(ref_mod, T, valid)
    (ai, at), (bi, bt), _, row_ok = _run_blocks(ref_mod, ours_mod, kind, c, condition_type)
    what = f"I2V {kind} {condition_type} T={T}"
    _compare(ai, bi, row_ok, f"{what} image rows")
    _compare(at, bt, torch.ones(T, dtype=torch.bool, device="cuda"), f"{what} text rows")


def test_i2v_double_block_under_qk_int8(i2v_modules):
    """JENGA_QK_INT8 reaches the I2V forwards through carved_attention_from_pools: the block output
    changes, and stays within that flag's tolerance row (mean 2e-2, max 0.15 of the RMS) of A"""
    import test_qk_int8_cpu as Q
    ref_mod, ours_mod = i2v_modules
    c = _i2v_case(ref_mod, 400, 300)
    (ai, _), (bi, _), (ci, _), row_ok = _run_blocks(ref_mod, ours_mod, "double", c, "token_replace", qk_int8=True)
    assert not torch.equal(bi, ci)
    a, q8 = ai.float()[0][row_ok], ci.float()[0][row_ok]
    rms = a.pow(2).mean().sqrt()
    d = (q8 - a).abs()
    print(f"\n[I2V double qk_int8] max {(d.max() / rms).item():.3e} mean {(d.mean() / rms).item():.3e} (x RMS)")
    assert d.mean() <= Q.TOL_MEAN * rms and d.max() <= Q.TOL_MAX * rms


class _SentinelCalled(Exception):
    pass


@pytest.mark.parametrize("kind", ["double", "single"])
def test_sequence_parallel_runs_the_original_forward(i2v_modules, kind):
    """with hybrid_seq_parallel_attn set the reference calls the dense parallel_attention
    (models_mul.py:264-274, :483-493): the fused forward hands the call to the original one"""
    from jenga_b200 import blocks
    _, ours_mod = i2v_modules
    c = _i2v_case(ours_mod, 400, 300)
    calls = []

    def sentinel(*a, **k):
        calls.append(1)
        raise _SentinelCalled

    cls = "MMDoubleStreamBlock" if kind == "double" else "MMSingleStreamBlock"
    blk = getattr(ours_mod, cls)(c["C"], c["H"], mlp_width_ratio=4.0, dtype=torch.bfloat16, device="cuda")
    blk.hybrid_seq_parallel_attn = sentinel
    S = c["L"] + c["T"]
    before = dict(blocks.STATS)
    mask = c["ff"] if kind == "double" else c["full"]
    tail = (0.7, mask, "token_replace", c["tr_vec"], c["hw"], 0.431, c["curve_sel"], 0.3)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16), pytest.raises(_SentinelCalled):
        if kind == "double":
            blk(c["img"], c["txt"], c["vec"], c["cu"], c["cu"], S, S, c["freqs"], *tail)
        else:
            blk(torch.cat([c["img"], c["txt"]], 1), c["vec"], c["T"], c["cu"], c["cu"], S, S, c["freqs"], *tail)
    assert calls == [1]
    assert blocks.STATS["fallback"] == before["fallback"] + 1
    assert blocks.STATS["i2v_double"] == before["i2v_double"] and blocks.STATS["i2v_single"] == before["i2v_single"]
