"""GPU parity of the fused attention prologue and the token gather (a-4, a-5, a-6)."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / "golden"))
import synth  # noqa: E402


def _ulp_diff_bf16(a, b):
    """|a-b| in units of the bf16 ulp of b (both bf16 tensors)."""
    af, bf = a.float(), b.float()
    ulp = torch.exp2(torch.floor(torch.log2(bf.abs().clamp_min(1e-30))) - 7)
    return ((af - bf).abs() / ulp)


def test_prologue_matches_reference_modules_golden():
    """Fixture = the reference's RMSNorm + apply_rotary_emb + cat chain (make_golden.py).
    Contract (SURVEY §8c-iii): <= 1 bf16 ulp everywhere; exact on >= 99.5 % of elements (the
    residue comes from the fp32 summation order of mean(x^2))."""
    from jenga_b200.hyvideo import attention_prologue
    gold = np.load(HERE / "golden" / "prologue.npz")
    c = synth.prologue_case()
    dev = "cuda"
    cos, sin = torch.from_numpy(gold["cos"]), torch.from_numpy(gold["sin"])
    index = torch.from_numpy(gold["index"]).to(dev)
    q, k, v, pools = attention_prologue(
        c["img"].to(dev), c["txt"].to(dev), c["H"], c["w_img_q"], c["w_img_k"], c["w_txt_q"],
        c["w_txt_k"], 1e-6, (cos, sin), rope_index=index)
    torch.cuda.synchronize()
    q_ref = torch.from_numpy(gold["q"]).view(torch.bfloat16)
    k_ref = torch.from_numpy(gold["k"]).view(torch.bfloat16)
    for got, ref in ((q.cpu(), q_ref), (k.cpu(), k_ref)):
        d = _ulp_diff_bf16(got, ref)
        assert d.max() <= 1.0, d.max().item()
        assert (got.view(torch.int16) == ref.view(torch.int16)).float().mean() >= 0.995
    # v: bit-exact concatenation
    H = c["H"]
    v_ref = torch.cat([c["img"].view(1, -1, 3, H, 128)[:, :, 2], c["txt"].view(1, -1, 3, H, 128)[:, :, 2]], dim=1)
    assert (v.cpu().view(torch.int16) == v_ref.contiguous().view(torch.int16)).all()
    # pooled block means of the normed/rotated q,k (zero padding for the ragged last block)
    qp, kp = pools
    S = q.shape[1]
    nb = (S + 127) // 128
    qpad = torch.nn.functional.pad(q.float().cpu(), [0, 0, 0, 0, 0, nb * 128 - S])
    qp_ref = qpad.view(1, nb, 128, H, 128).mean(2).permute(0, 2, 1, 3)
    assert (qp.float().cpu() - qp_ref).abs().max() <= 2.0 ** -8 * qp_ref.abs().max() + 1e-6


def test_gather_scatter_bit_exact():
    from jenga_b200.hyvideo import gather_tokens
    from jenga_b200 import gilbert
    t, h, w = 4, 6, 8
    l2h, h2l = gilbert.mapping_tensors(t, h, w)
    x = synth.normal((2, t * h * w, 256), 77).bfloat16()
    dev = "cuda"
    g = gather_tokens(x.to(dev), h2l.to(dev))
    assert (g.cpu().view(torch.int16) == x[:, h2l].view(torch.int16)).all()
    back = gather_tokens(g, l2h.to(dev))
    assert (back.cpu().view(torch.int16) == x.view(torch.int16)).all()
    # fp32 table rows (freqs_cos[hilbert_order], jenga_hyvideo.py:117)
    tab = synth.normal((t * h * w, 128), 78)
    gt = gather_tokens(tab.to(dev), h2l.to(dev))
    assert (gt.cpu() == tab[h2l]).all()


def test_wan_prologue_matches_reference_golden():
    """Fixture = WanRMSNorm + rope_apply from wan/modules/model_mul.py (make_golden.py), rounded
    to bf16 like the operator does.  <= 1 bf16 ulp, >= 99.5 % bit-identical."""
    import hashlib
    from jenga_b200 import wan
    gold = np.load(HERE / "golden" / "wan_prologue.npz")
    c = synth.wan_prologue_case()
    freqs = wan.rope_freqs(128)
    sha = hashlib.sha256(np.ascontiguousarray(torch.view_as_real(freqs).numpy()).tobytes()).hexdigest()[:16]
    assert sha == bytes(gold["freqs_sha"]).decode()  # same table as the reference builds
    dev = "cuda"
    for tag, x, w in (("q", c["xq"], c["wq"]), ("k", c["xk"], c["wk"])):
        got = wan.norm_rope(x.to(dev), w.to(dev), c["H"], c["grid"], freqs, c["remap"], eps=1e-6).cpu()
        ref = torch.from_numpy(gold[tag]).view(torch.bfloat16)
        d = _ulp_diff_bf16(got, ref)
        assert d.max() <= 1.0, (tag, d.max().item())
        assert (got.view(torch.int16) == ref.view(torch.int16)).float().mean() >= 0.995
    assert wan.block_counts(32760, 0.5) == (128, 12) and wan.block_counts(75600, 0.7) == (177, 28)


def _wan_norm_rope_torch(x, w, heads, grid, freqs, remap, eps):
    """WanRMSNorm + rope_apply (the chain make_golden.py runs from the reference) restated in torch, then
    the operator's bf16 cast."""
    B, L, _ = x.shape
    xf = x.float()
    y = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).type_as(x) * w
    y = y.view(B, L, heads, 128)
    f, h, wd = grid
    n = f * h * wd
    parts = freqs.to(x.device).split([22, 21, 21], dim=1)
    fr = torch.cat([parts[0][:f].view(f, 1, 1, -1).expand(f, h, wd, -1),
                    parts[1][:h].view(1, h, 1, -1).expand(f, h, wd, -1),
                    parts[2][:wd].view(1, 1, wd, -1).expand(f, h, wd, -1)], dim=-1).reshape(n, 1, -1)[remap]
    rot = torch.view_as_real(torch.view_as_complex(y[:, :n].double().reshape(B, n, heads, 64, 2)) * fr).flatten(3)
    return torch.cat([rot, y[:, n:].double()], dim=1).float().bfloat16()


@pytest.mark.parametrize("dt,heads,grid", [(torch.float32, 12, (3, 6, 8)), (torch.bfloat16, 12, (3, 6, 8)),
                                           (torch.float32, 40, (2, 5, 7)), (torch.bfloat16, 5, (4, 4, 4))])
def test_wan_prologue_matches_torch_restatement(dt, heads, grid):
    """fp32 and bf16 input (bf16 weights with bf16 input), batch 2, odd and large head counts, a remapped
    grid and 37 tokens past it that get no rotation.  >= 99.5 % bit-identical, as in the golden test.  The
    residue again comes from the fp32 summation order of mean(x^2): a rounding of the normalised pair that
    falls the other way moves it by about one bf16 ulp of its magnitude, and the rotation can carry that
    into a component much smaller than the pair.  So the error of every element is bounded relative to
    the magnitude of its complex pair, not to the element itself."""
    from jenga_b200 import wan
    dev = "cuda"
    L = grid[0] * grid[1] * grid[2] + 37
    g = torch.Generator().manual_seed(99 + heads)
    x = (torch.randn((2, L, heads * 128), generator=g) * 1.3).to(dt).to(dev)
    w = (1 + 0.2 * torch.randn(heads * 128, generator=g)).to(dt).to(dev)
    remap = torch.randperm(grid[0] * grid[1] * grid[2], generator=g).to(dev)
    freqs = wan.rope_freqs(128)
    got = wan.norm_rope(x, w, heads, grid, freqs, remap, eps=1e-6)
    ref = _wan_norm_rope_torch(x, w, heads, grid, freqs, remap, 1e-6)
    assert (got.view(torch.int16) == ref.view(torch.int16)).float().mean() >= 0.995
    pair = ref.float().view(*ref.shape[:-1], 64, 2).norm(dim=-1, keepdim=True)
    err = (got.float() - ref.float()).view(*ref.shape[:-1], 64, 2).abs()
    assert (err <= 2.0 ** -5 * pair).all(), (err / pair).max().item()
