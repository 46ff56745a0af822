"""Several samples per call (`--num-videos N`) on the fused HunyuanVideo and HunyuanVideo-I2V block path.

The unmodified block classes are loaded as test_dropin_blocks_gpu.py / test_i2v_blocks_gpu.py load them
(random weights, bf16 autocast, C = 512, 4 heads of 128, sa_drop_rate 0.7, one curve).  Each sample of a
batch is built from its own seed; the text mask gives every sample 180 valid text rows, as one prompt
does for --num-videos.

* Kernels: ln_modulate[_tr][_fp8] / gate_residual[_tr] / quantize_rows_fp8 on [B, L, C] with [B, C] (or
  shared [1, C]) vectors are bit-identical, sample by sample, to the B = 1 call on that sample.
* Attention section: prologue + selection + carved attention on B stacked samples' qkv equals, with
  torch.equal, the section run on each sample alone; in the single-stream form this includes the rows
  written into the concatenation buffer of linear2 and the GELU columns beside them.
* Blocks at B = 2: the fused forward of each sample matches the fused forward of that sample alone,
  with the FP8 Linears off and with them forced on for every shape.  Not bit for bit: cuBLAS may pick
  another algorithm for the [2, C] modulation rows (img_mod(vec)) and the 2·L image rows than for one
  sample, so the tolerance is the drop-in tests' (test_dropin_blocks_gpu._compare) on rows whose
  selection is the same.  blocks.STATS moves as for one B = 1 call: one fused forward, no fallback, the
  same ln_modulate / gate_residual / gelu_cat / linear_fp8 counts.
* Against the original forward (forward.__wrapped__, on the jenga_b200 operator as the drop-in tests
  bind it) at B = 2, within the same tolerance."""
import inspect
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))

from test_dropin_blocks_gpu import _compare, _reinit, _structured_tokens, modules  # noqa: E402,F401
from test_hy_block_routing_gpu import C, _inputs  # noqa: E402
from test_i2v_blocks_gpu import i2v_modules  # noqa: E402,F401
from test_linear_fp8_gpu import ALL_ROUTED  # noqa: E402

VALID = 180          # valid text rows of every sample (_inputs' text mask)


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------
def _vecs(B, C, g, shared, n, s=0.3):
    return [(s * torch.randn(1 if shared else B, C, generator=g, device="cuda")).bfloat16() for _ in range(n)]


def _row(v, b):
    return v[b:b + 1] if v.shape[0] > 1 else v


def _rows_x(B, L, C, g, strided):
    """x [B, L, C]; strided: a view whose batch stride does not continue its row pitch"""
    x = (torch.randn(B, L + 3, C + 64, generator=g, device="cuda") * 1.7 + 0.3).bfloat16()
    return x[:, 1:L + 1, 32:32 + C] if strided else x[:, :L, :C].contiguous()


def _same8(a, b):
    return torch.equal(a[0].view(torch.uint8), b[0].view(torch.uint8)) and torch.equal(a[1], b[1])


CASES = [(2, 2048 + 37, 3072, False), (3, 515, 6144, True), (4, 1001, 1536, False), (2, 4225, 6144, False)]


@pytest.mark.parametrize("shared", [False, True], ids=["per_sample", "shared"])
@pytest.mark.parametrize("B,L,C,strided", CASES)
def test_ln_modulate_samples_equal_the_batch_one_calls(B, L, C, strided, shared):
    from jenga_b200 import dense as DN
    g = torch.Generator(device="cuda").manual_seed(B * L + C)
    x = _rows_x(B, L, C, g, strided)
    shift, scale, tr_shift, tr_scale = _vecs(B, C, g, shared, 4)
    mask = torch.rand(L, generator=g, device="cuda") < 0.3
    got = DN.ln_modulate(x, shift, scale)
    got_tr = DN.ln_modulate(x, shift, scale, tr=(tr_shift, tr_scale, mask.cpu()))
    got8 = DN.ln_modulate_fp8(x, shift, scale) if C % 16 == 0 else None
    got8_tr = DN.ln_modulate_fp8(x, shift, scale, tr=(tr_shift, tr_scale, mask)) if C % 16 == 0 else None
    assert got.shape == x.shape and (got8 is None or got8[0].shape == (B * L, C))
    for b in range(B):
        one = [x[b:b + 1]] + [_row(v, b) for v in (shift, scale, tr_shift, tr_scale)]
        assert torch.equal(got[b:b + 1], DN.ln_modulate(*one[:3])), b
        assert torch.equal(got_tr[b:b + 1], DN.ln_modulate(*one[:3], tr=(one[3], one[4], mask))), b
        if got8 is not None:
            rows = slice(b * L, (b + 1) * L)
            assert _same8((got8[0][rows], got8[1][rows]), DN.ln_modulate_fp8(*one[:3])), b
            assert _same8((got8_tr[0][rows], got8_tr[1][rows]),
                          DN.ln_modulate_fp8(*one[:3], tr=(one[3], one[4], mask))), b


@pytest.mark.parametrize("shared", [False, True], ids=["per_sample", "shared"])
@pytest.mark.parametrize("B,L,C,strided", CASES)
def test_gate_residual_samples_equal_the_batch_one_calls(B, L, C, strided, shared):
    from jenga_b200 import dense as DN
    g = torch.Generator(device="cuda").manual_seed(B * L + C + 1)
    x = _rows_x(B, L, C, g, False)
    y = _rows_x(B, L, C, g, strided)
    gate, tr_gate = _vecs(B, C, g, shared, 2, 1.0)
    mask = torch.rand(L, generator=g, device="cuda") < 0.3
    got = DN.gate_residual(x, y, gate)
    got_tr = DN.gate_residual(x, y, gate, tr=(tr_gate, mask))
    for b in range(B):
        assert torch.equal(got[b:b + 1], DN.gate_residual(x[b:b + 1], y[b:b + 1], _row(gate, b))), b
        assert torch.equal(got_tr[b:b + 1], DN.gate_residual(x[b:b + 1], y[b:b + 1], _row(gate, b),
                                                             tr=(_row(tr_gate, b), mask.cpu()))), b


def test_quantize_rows_takes_a_batch_whose_rows_are_not_uniformly_strided():
    """attn[:, :L] of the double-stream block, the input of img_attn_proj under the FP8 Linears"""
    from jenga_b200 import dense as DN
    g = torch.Generator(device="cuda").manual_seed(5)
    attn = torch.randn(3, 2048 + 256, 3072, generator=g, device="cuda").bfloat16()
    got = DN.quantize_rows_fp8(attn[:, :2048])
    for b in range(3):
        assert _same8((got[0][b * 2048:(b + 1) * 2048], got[1][b * 2048:(b + 1) * 2048]),
                      DN.quantize_rows_fp8(attn[b:b + 1, :2048])), b


def test_mismatched_vectors_raise_before_any_launch():
    from jenga_b200 import dense as DN
    x = torch.zeros(2, 64, 512, dtype=torch.bfloat16, device="cuda")
    ok, bad = torch.zeros(2, 512, dtype=torch.bfloat16, device="cuda"), torch.zeros(3, 512, dtype=torch.bfloat16,
                                                                                     device="cuda")
    mask = torch.zeros(64, dtype=torch.bool, device="cuda")
    for call in (lambda: DN.ln_modulate(x, bad, ok), lambda: DN.ln_modulate_fp8(x, ok, ok, tr=(ok, bad, mask)),
                 lambda: DN.gate_residual(x, x, bad), lambda: DN.gate_residual(x, x, ok, tr=(bad, mask)),
                 lambda: DN.ln_modulate(x, ok, ok, tr=(ok, ok, torch.zeros(128, dtype=torch.bool)))):
        with pytest.raises(ValueError):
            call()


# ------------------------------------------------------------------------------------------------
# call arguments with one sample per seed
# ------------------------------------------------------------------------------------------------
def _mod(modules, i2v_modules, variant):
    return i2v_modules[1] if variant == "i2v" else modules[2]


def _block(mod, kind):
    cls = getattr(mod, "MMDoubleStreamBlock" if kind == "double" else "MMSingleStreamBlock")
    blk = cls(C, 4, mlp_width_ratio=4.0, dtype=torch.bfloat16, device="cuda")
    _reinit(blk, 11)
    return blk


def _batch_args(mod, kind, variant, seeds):
    """parameter name -> value of the eligible call of test_hy_block_routing_gpu.py, with one sample per
    seed: its own image and text rows, vec and token_replace_vec; the curve, RoPE tables and first-frame
    mask are shared, and every sample has VALID text rows"""
    a = _inputs(mod, kind, variant == "i2v")
    L = a["freqs_cis"][0].shape[0]
    T = a["txt"].shape[1] if kind == "double" else a["txt_len"]
    imgs, txts, vecs, trs = [], [], [], []
    for s in seeds:
        imgs.append(_structured_tokens(L, C, 100 * s + 1))
        txts.append(_structured_tokens(-(-T // 128) * 128, C, 100 * s + 2, gain=0.5)[:, :T])
        g = torch.Generator(device="cuda").manual_seed(100 * s + 3)
        vecs.append(torch.randn(1, C, generator=g, device="cuda").bfloat16())
        trs.append(torch.randn(1, C, generator=g, device="cuda").bfloat16())
    img, txt = torch.cat(imgs), torch.cat(txts)
    a.update(dict(img=img, txt=txt) if kind == "double" else dict(x=torch.cat([img, txt], 1)))
    a["vec"] = torch.cat(vecs)
    if variant == "i2v":
        a["token_replace_vec"] = torch.cat(trs)
    text_mask = torch.zeros(len(seeds), T, dtype=torch.int64, device="cuda")
    text_mask[:, :VALID] = 1
    a["cu_seqlens_q"] = a["cu_seqlens_kv"] = mod.get_cu_seqlens(text_mask, L)
    return a, L, T


def _run(blk, a, original=False):
    """(outputs as a tuple, STATS moves, selection bit rows of every select_blocks call)"""
    from jenga_b200 import attention as A, blocks
    names = list(inspect.signature(type(blk).forward.__wrapped__).parameters)[1:]
    fn = type(blk).forward.__wrapped__ if original else type(blk).forward
    before = dict(blocks.STATS)
    A.MASK_CAPTURE = []
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            out = fn(blk, *(a[n] for n in names))
        torch.cuda.synchronize()
        bits = [b for b, _ in A.MASK_CAPTURE]
    finally:
        A.MASK_CAPTURE = None
    moved = {k: blocks.STATS[k] - before[k] for k in blocks.STATS if blocks.STATS[k] != before[k]}
    return (out if isinstance(out, tuple) else (out,)), moved, bits


def _split(outs, bits):
    """a batch's outputs and its one selection -> one (outputs, selection) per sample"""
    assert len(bits) == 1
    return [(tuple(o[b:b + 1] for o in outs), bits[0][b:b + 1]) for b in range(outs[0].shape[0])]


def _check_samples(kind, got, got_bits, want, L, what):
    """sample b of `got` / `got_bits` (a batch) against want[b] = (outputs, selection bits) of sample b:
    the drop-in tolerance on image rows whose selection is the same in every head, and on every text
    row"""
    for b, ((g, gb), (w, wb)) in enumerate(zip(_split(got, got_bits), want, strict=True)):
        same = (gb[0] == wb[0]).all(-1).all(0)                        # [n_img blocks]
        row_ok = torch.cat([same.repeat_interleave(128),
                            torch.ones(max(0, L - same.numel() * 128), dtype=torch.bool, device="cuda")])[:L]
        if kind == "double":
            (gi, gt), (wi, wt) = g, w
        else:
            gi, gt, wi, wt = g[0][:, :L], g[0][:, L:], w[0][:, :L], w[0][:, L:]
        _compare(wi, gi, row_ok, f"{what} sample {b} image rows")
        _compare(wt, gt, torch.ones(gt.shape[1], dtype=torch.bool, device="cuda"), f"{what} sample {b} text rows")


# ------------------------------------------------------------------------------------------------
# attention section
# ------------------------------------------------------------------------------------------------
def _section(blk, mod, variant, kind, img_qkv, txt_qkv, a, out=None):
    from jenga_b200 import blocks
    if kind == "double":
        norms = [blocks._rms_params(n) for n in (blk.img_attn_q_norm, blk.img_attn_k_norm, blk.txt_attn_q_norm,
                                                 blk.txt_attn_k_norm)]
    else:
        norms = [blocks._rms_params(n) for n in (blk.q_norm, blk.k_norm)] * 2
    return blocks._attention_section(
        blk, mod, img_qkv, txt_qkv, norms, freqs_cis=a["freqs_cis"], cu_seqlens_q=a["cu_seqlens_q"],
        cu_seqlens_kv=a["cu_seqlens_kv"], sa_drop_rate=a["sa_drop_rate"], txt_amp=a["txt_amp"],
        curve_sel=a["curve_sel"], p_remain_rates=a["p_remain_rates"],
        text_blocks=blocks._I2V_TEXT_BLOCKS if variant == "i2v" else a["txt_block_num"],
        pad_ragged=variant == "i2v", out=out)


@pytest.mark.parametrize("B", [2, 3])
@pytest.mark.parametrize("kind", ["double", "single"])
@pytest.mark.parametrize("variant", ["hy", "i2v"])
def test_attention_section_of_each_sample_equals_the_sample_alone(modules, i2v_modules, variant, kind, B):
    from jenga_b200 import attention as A, dense as DN
    mod = _mod(modules, i2v_modules, variant)
    blk = _block(mod, kind)
    seeds = list(range(7, 7 + B))
    a, L, T = _batch_args(mod, kind, variant, seeds)
    S, C3 = L + T, 3 * C
    # qkv rows with per-block structure (well separated block scores), one seed per sample; the single
    # stream's are column slices of linear1's output [B, S, 3C + 4C], as the fused forward takes them
    qkv = torch.cat([_structured_tokens(-(-S // 128) * 128, 7 * C, 100 * s + 4, gain=2.0)[:, :S] for s in seeds])
    A.MASK_CAPTURE = []
    try:
        with torch.no_grad():
            if kind == "double":
                img_qkv, txt_qkv = qkv[:, :L, :C3].contiguous(), qkv[:, L:, :C3].contiguous()
                got = _section(blk, mod, variant, kind, img_qkv, txt_qkv, a)
                alone = [_section(blk, mod, variant, kind, img_qkv[b:b + 1], txt_qkv[b:b + 1],
                                  _batch_args(mod, kind, variant, [s])[0]) for b, s in enumerate(seeds)]
            else:
                def section(lin1, args):
                    cat = torch.empty((lin1.shape[0], S, C + 4 * C), dtype=torch.bfloat16, device="cuda")
                    view = cat[:, :, :C].unflatten(2, (4, -1))
                    _section(blk, mod, variant, kind, lin1[:, :L, :C3], lin1[:, L:, :C3], args, out=view)
                    DN.gelu_tanh_into(lin1[:, :, C3:], cat[:, :, C:])
                    return cat
                got = section(qkv, a)
                alone = [section(qkv[b:b + 1], _batch_args(mod, kind, variant, [s])[0]) for b, s in enumerate(seeds)]
            torch.cuda.synchronize()
        bits = [b for b, _ in A.MASK_CAPTURE]
    finally:
        A.MASK_CAPTURE = None
    assert len(bits) == 1 + B and bits[0].shape[0] == B
    for b in range(B):
        assert torch.equal(bits[0][b:b + 1], bits[1 + b]), f"selection of sample {b}"
        assert torch.equal(got[b:b + 1], alone[b]), f"attention of sample {b}"


# ------------------------------------------------------------------------------------------------
# blocks at B = 2
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fp8", [False, True], ids=["fp8_off", "fp8_every_shape"])
@pytest.mark.parametrize("kind", ["double", "single"])
@pytest.mark.parametrize("variant", ["hy", "i2v"])
def test_block_of_two_samples_matches_each_sample_alone(modules, i2v_modules, variant, kind, fp8, monkeypatch):
    from jenga_b200 import dense as DN
    if fp8:
        monkeypatch.setattr(DN, "LINEAR_FP8", True)
        monkeypatch.setattr(DN, "FP8_ROUTED", ALL_ROUTED)
    mod = _mod(modules, i2v_modules, variant)
    blk = _block(mod, kind)
    seeds = [21, 22]
    a, L, _ = _batch_args(mod, kind, variant, seeds)
    got, moved, got_bits = _run(blk, a)
    alone = [_run(blk, _batch_args(mod, kind, variant, [s])[0]) for s in seeds]
    key = f"{variant}_{kind}"
    # one fused forward for the whole batch, no fallback, and per call the fused chains of one B = 1 call
    for _, moved1, _ in alone:
        assert moved == moved1, (moved, moved1)
    assert moved[key] == 1 and "fallback" not in moved
    assert moved["ln_modulate"] == (4 if kind == "double" else 1)
    assert moved["gate_residual"] == (4 if kind == "double" else 1)
    assert moved.get("gelu_cat", 0) == (1 if kind == "single" else 0)
    assert moved.get("linear_fp8", 0) == ((4 if kind == "double" else 2) if fp8 else 0)
    _check_samples(kind, got, got_bits, [_split(o, bits)[0] for o, _, bits in alone], L,
                   f"{variant} {kind} {'fp8' if fp8 else 'bf16'} B=2 vs B=1")


@pytest.mark.parametrize("kind", ["double", "single"])
@pytest.mark.parametrize("variant", ["hy", "i2v"])
def test_block_of_two_samples_matches_the_original_forward(modules, i2v_modules, variant, kind):
    mod = _mod(modules, i2v_modules, variant)
    blk = _block(mod, kind)
    a, L, _ = _batch_args(mod, kind, variant, [31, 32])
    want, moved_orig, want_bits = _run(blk, a, original=True)
    got, moved, got_bits = _run(blk, a)
    key = f"{variant}_{kind}"
    assert moved[key] == 1 and "fallback" not in moved and key not in moved_orig
    _check_samples(kind, got, got_bits, _split(want, want_bits), L, f"{variant} {kind} B=2 fused vs original")
