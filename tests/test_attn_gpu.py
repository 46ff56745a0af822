"""GPU parity of the carved-attention kernel (through the C-ABI) against the CPU oracle.

Tolerance (SURVEY §8c-iv): bf16 max-abs <= 2e-2 and mean-abs <= 2e-3 relative to the output
RMS; fp16 max-abs <= 5e-3 relative to the output RMS... stated per test below.
"""
import math
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel_err(got, ref):
    got, ref = got.float().cpu(), ref.float().cpu()
    rms = ref.pow(2).mean().sqrt().item() + 1e-12
    d = (got - ref).abs()
    return d.max().item() / rms, d.mean().item() / rms


def assert_close(got, ref, dtype):
    """Stated tolerance (SURVEY §8c-iv, FA2-vs-fp32 class error), per element:
         bf16: |got-ref| <= 2e-2*RMS(ref) + 2^-7*|ref|   and mean|got-ref| <= 3e-3*RMS(ref)
         fp16: |got-ref| <= 5e-3*RMS(ref) + 2^-10*|ref|  and mean|got-ref| <= 5e-4*RMS(ref)
    The |ref| term admits a 1-2 ulp flip of the 16-bit output rounding on large elements.
    The mean bound sits ~1.5x above the noise floor two CORRECT implementations have against
    each other: P is rounded to bf16 (relative error 2^-9/sqrt(3) rms per term) relative to a
    different running max in each (the reference rescales per tile, the oracle per tile, the
    kernel lazily), which for uncorrelated V gives sqrt(2)*1.1e-3*RMS rms ~ 1.3e-3*RMS
    mean-abs, plus the 16-bit output rounding."""
    got, ref = got.float().cpu(), ref.float().cpu()
    rms = ref.pow(2).mean().sqrt().item() + 1e-12
    a, r, m = (2e-2, 2.0 ** -7, 3e-3) if dtype == torch.bfloat16 else (5e-3, 2.0 ** -10, 5e-4)
    d = (got - ref).abs()
    bad = d > (a * rms + r * ref.abs())
    assert not bad.any(), (int(bad.sum()), (d / rms).max().item())
    assert d.mean().item() <= m * rms, d.mean().item() / rms


def _random_mask(B, H, nq, nb, density, gen, always=()):
    m = torch.rand(B, H, nq, nb, generator=gen) < density
    for i in range(min(nq, nb)):
        m[:, :, i, i] = True  # self block, like the neighbour matrix guarantees
    for c in always:
        m[..., c] = True
    return m


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", ["hy_small", "wan_ragged"])
def test_carved_attention_matches_oracle(dtype, case):
    from jenga_b200.attention import carved_attention_fwd, mask_onehot_to_bits
    from oracle import attention_oracle as orc

    g = torch.Generator().manual_seed(1234)
    D = 128
    if case == "hy_small":
        B, H, n_img, n_txt, t_valid = 1, 3, 5, 2, 180
        S = (n_img + n_txt) * 128
        seqlen = n_img * 128 + t_valid
        text_amp, text_start = 0.431, n_img
        S_alloc = S
    else:
        B, H, n_img, n_txt = 2, 2, 4, 0
        S_alloc = 4 * 128 - 8  # ragged: 8 rows of zero padding supplied by TMA OOB fill
        S = 4 * 128
        seqlen = S_alloc
        text_amp, text_start = 0.0, n_img
    q = torch.randn(B, S_alloc, H, D, generator=g).to(dtype)
    k = torch.randn(B, S_alloc, H, D, generator=g).to(dtype)
    v = torch.randn(B, S_alloc, H, D, generator=g).to(dtype)
    nb = n_img + n_txt
    mask = _random_mask(B, H, n_img, nb, 0.4, g, always=range(n_img, nb))
    sm_scale = D ** -0.5

    # oracle on zero-padded [B,H,S,D]
    def pad(x):
        return torch.nn.functional.pad(x, [0, 0, 0, 0, 0, S - S_alloc]).transpose(1, 2)
    qo, ko, vo = pad(q), pad(k), pad(v)
    ref_img = orc.carved_attention_rows(qo[:, :, :n_img * 128], ko, vo, mask, seqlen, sm_scale,
                                        text_amp, text_start)
    refs = [ref_img]
    if n_txt:
        refs.append(orc.dense_attention_rows(qo[:, :, n_img * 128:], ko, vo, sm_scale))
    ref = torch.cat(refs, dim=2).transpose(1, 2)[:, :S_alloc]  # [B,S,H,D]

    dev = "cuda"
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    bits = mask_onehot_to_bits(mask.to(dev))
    out = carved_attention_fwd(
        q.to(dev), k.to(dev), v.to(dev), bits, nq_sparse=n_img, nq_dense=n_txt,
        sm_scale=sm_scale, text_amp=text_amp, text_block_start=text_start,
        kv_limit_sparse=seqlen, q_limit_sparse=seqlen, kv_limit_dense=S, err_flag=err)
    torch.cuda.synchronize()
    assert err.item() == 0
    assert_close(out, ref, dtype)
    if case == "wan_ragged":
        # rows >= seqlen do not exist in the tensor; the rest must be finite
        assert torch.isfinite(out.float()).all()


@pytest.mark.parametrize("name", ["hy", "wan", "amp0"])
def test_carved_attention_matches_reference_triton_golden(name):
    """fp16 fixtures produced by the UNMODIFIED reference Triton kernel (interpreter mode,
    tests/golden/make_golden.py) — image rows only, exactly what the kernel writes."""
    import numpy as np
    from pathlib import Path
    import sys
    sys.path.insert(0, str(Path(__file__).parent / "golden"))
    import synth
    from jenga_b200.attention import carved_attention_fwd, mask_onehot_to_bits

    gold = np.load(Path(__file__).parent / "golden" / "attention_fp16.npz")
    c = synth.attention_case(name)
    ref = torch.from_numpy(gold[name + "/o"])  # [1,H,n_img*128,D]
    n_img, n_txt = c["n_img"], c["n_txt"]
    dev = "cuda"
    q = c["q"].transpose(1, 2).contiguous().to(dev)  # [1,S,H,D]
    k = c["k"].transpose(1, 2).contiguous().to(dev)
    v = c["v"].transpose(1, 2).contiguous().to(dev)
    bits = mask_onehot_to_bits(c["mask"].to(dev))
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    out = carved_attention_fwd(q, k, v, bits, nq_sparse=n_img, nq_dense=n_txt,
                               sm_scale=128 ** -0.5, text_amp=c["amp"], text_block_start=n_img,
                               kv_limit_sparse=c["seqlen"], q_limit_sparse=c["seqlen"],
                               err_flag=err)
    torch.cuda.synchronize()
    assert err.item() == 0
    got = out[:, :n_img * 128].transpose(1, 2)
    assert_close(got, ref, torch.float16)
    # rows at or past seqlen are exact zeros in both
    if c["seqlen"] < n_img * 128:
        assert (got[:, :, c["seqlen"]:] == 0).all() and (ref[:, :, c["seqlen"]:] == 0).all()
