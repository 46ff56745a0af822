"""Full-size (HunyuanVideo 720x1280x125f, S=115456, H=24: bench.py's hy720p workload) checks through
size-independent properties, plus sampled rows against an fp32 torch evaluation on the GPU."""
import math
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


@pytest.fixture(scope="module")
def hy720p():
    import bench
    from jenga_b200.attention import bits_to_onehot
    dev = torch.device("cuda", 0)
    wl = bench.workload("hy720p", 0.7)
    inp = bench.build_inputs(wl, dev)
    out, bits = bench.run_operator(wl, inp, return_bits=True)
    torch.cuda.synchronize()
    return wl, inp, out, bits


def test_mask_invariants_full_size(hy720p):
    from jenga_b200.attention import bits_to_onehot, neighbour_bits
    wl, inp, out, bits = hy720p
    nb_img, nb = inp["nb_img"], inp["nb_img"] + wl["text_blocks"]
    assert bits.shape == (1, 24, nb_img, (nb + 31) // 32)
    oh = bits_to_onehot(bits, bits.shape[-1] * 32)
    assert not oh[..., nb:].any()                       # no bits past the key blocks
    assert oh[..., nb_img:nb].all()                     # text columns always on (ref :292-293)
    counts = oh[..., :nb_img].sum(-1)
    assert int(counts.min()) >= inp["top_k"]            # top_k is a floor (ref :247-250)
    nbr = inp["nbr"].to(oh.device)
    assert (oh[0, :, :, :nb_img] | ~nbr[None]).all()    # neighbour rows are a subset (ref :280-289)
    assert int(counts.max()) <= nb_img


def test_sampled_rows_against_fp32_torch(hy720p):
    """Rows of 6 query blocks x 3 heads recomputed in fp32 from the same mask, with the
    reference's rounding points (Q pre-scale re-rounding, P in bf16, text rows dense)."""
    from jenga_b200.attention import bits_to_onehot
    wl, inp, out, bits = hy720p
    q, k, v = inp["q"], inp["k"], inp["v"]
    S, nb_img = inp["S"], inp["nb_img"]
    nb = nb_img + wl["text_blocks"]
    seqlen = inp["n_img"] + wl["text_valid"]
    oh = bits_to_onehot(bits, nb)
    qk_scale = torch.tensor((128 ** -0.5) * 1.44269504, dtype=torch.float32, device=q.device)
    o4 = out.view(1, S, 24, 128)
    worst = 0.0
    for h in (0, 11, 23):
        kh, vh = k[0, :, h].float(), v[0, :, h].float()
        for m in (0, 1, 450, 899, 900, 901):
            rows = slice(m * 128, (m + 1) * 128)
            qm = q[0, rows, h].float()
            if m < nb_img:
                live = oh[0, h, m].nonzero().flatten()
                cols = (live[:, None] * 128 + torch.arange(128, device=q.device)[None]).flatten()
                qt = (qm * qk_scale).to(torch.bfloat16).float()
                s = qt @ kh[cols].T
                s = s.masked_fill(cols[None, :] >= seqlen, float("-inf"))
                p = torch.exp2(s - s.max(-1, keepdim=True).values)
            else:  # text rows: dense, FlashAttention semantics, padded text keys attended
                cols = torch.arange(S, device=q.device)
                s = (qm @ kh.T) * (128 ** -0.5)
                p = torch.exp(s - s.max(-1, keepdim=True).values)
            ref = (p.to(torch.bfloat16).float() @ vh[cols]) / p.sum(-1, keepdim=True)
            got = o4[0, rows, h].float()
            rms = ref.pow(2).mean().sqrt()
            d = (got - ref).abs()
            assert (d <= 2e-2 * rms + 2.0 ** -7 * ref.abs()).all(), (h, m, (d / rms).max().item())
            assert d.mean() <= 3e-3 * rms  # see test_attn_gpu.assert_close for the noise floor
            worst = max(worst, (d / rms).max().item())
    print("worst max|err|/rms over sampled rows:", worst)


def test_value_linearity_is_bit_exact(hy720p):
    """O is linear in V and scaling by 2 is exact in every format on the path, so
    attention(q, k, 2v) must equal 2*attention(q, k, v) bit for bit at full size."""
    import bench
    wl, inp, out, bits = hy720p
    out2 = bench.run_operator(wl, inp, v=inp["v"] * 2)
    torch.cuda.synchronize()
    assert torch.equal(out2, out * 2)
    assert torch.isfinite(out.float()).all()


def test_gather_scatter_round_trip_full_size():
    """[1, 115200, 3072] bf16 hidden states along the 32x45x80 curve and back (a-4)."""
    from jenga_b200 import gilbert
    from jenga_b200.hyvideo import gather_tokens
    dev = torch.device("cuda", 0)
    l2h, h2l = gilbert.mapping_tensors(32, 45, 80)
    x = torch.randn(1, 115200, 3072, device=dev, dtype=torch.bfloat16)
    g = gather_tokens(x, h2l.to(dev))
    idx = torch.tensor([0, 1, 57599, 115199], device=dev)
    assert torch.equal(g[0, idx], x[0, h2l.to(dev)[idx]])
    back = gather_tokens(g, l2h.to(dev))
    assert torch.equal(back, x)


def _check_rows(q, k, v, out4, oh, n_img_blocks, seqlen, S_pad, rows_to_check, heads, text_blocks):
    """fp32 torch evaluation of selected q blocks (sparse: reference Triton semantics; dense:
    FlashAttention semantics over the zero-padded keys)."""
    dev = q.device
    qk_scale = torch.tensor((128 ** -0.5) * 1.44269504, dtype=torch.float32, device=dev)
    S = q.shape[1]
    for h in heads:
        kh = torch.zeros(S_pad, 128, device=dev)
        vh = torch.zeros(S_pad, 128, device=dev)
        kh[:S], vh[:S] = k[0, :, h].float(), v[0, :, h].float()
        for m in rows_to_check:
            r0, r1 = m * 128, min((m + 1) * 128, S)
            qm = q[0, r0:r1, h].float()
            if m < n_img_blocks:
                live = oh[0, h, m].nonzero().flatten()
                cols = (live[:, None] * 128 + torch.arange(128, device=dev)[None]).flatten()
                qt = (qm * qk_scale).to(torch.bfloat16).float()
                s = (qt @ kh[cols].T).masked_fill(cols[None, :] >= seqlen, float("-inf"))
                pr = torch.exp2(s - s.max(-1, keepdim=True).values)
            else:
                cols = torch.arange(S_pad, device=dev)
                s = (qm @ kh.T) * (128 ** -0.5)
                pr = torch.exp(s - s.max(-1, keepdim=True).values)
            ref = (pr.to(torch.bfloat16).float() @ vh[cols]) / pr.sum(-1, keepdim=True)
            valid = (torch.arange(r0, r1, device=dev) < seqlen) if m < n_img_blocks else torch.ones(r1 - r0, dtype=torch.bool, device=dev)
            ref = torch.where(valid[:, None], ref, torch.zeros_like(ref))
            got = out4[0, r0:r1, h].float()
            rms = ref.pow(2).mean().sqrt()
            d = (got - ref).abs()
            assert (d <= 2e-2 * rms + 2.0 ** -7 * ref.abs()).all(), (h, m, (d / rms).max().item())
            assert d.mean() <= 3e-3 * rms


def test_wan_1_3b_full_size_fp32_inputs():
    """Wan2.1-1.3B 832x480x81f — q,k fp32 [1,32760,12,128] (rope_apply returns
    .float()), v bf16, 8 zero-padded rows, sliced-gilbert adjacency, first-frame rule, fp32 output."""
    import bench
    from jenga_b200 import gilbert, wan
    from jenga_b200.attention import bits_to_onehot, block_sparse_attention_variant
    dev = torch.device("cuda", 0)
    t, h, w = 21, 30, 52
    S, H = t * h * w, 12
    q = bench.synth_tokens(S, H, dev, 4321).float()
    k = bench.synth_tokens(S, H, dev, 4322).float()
    v = torch.randn(1, S, H, 128, device=dev, generator=torch.Generator(device=dev).manual_seed(4323)).bfloat16()
    nbr = gilbert.sliced_gilbert_block_neighbor_mapping(t, h, w)
    top_k, ff = wan.block_counts(S, 0.5)
    assert (top_k, ff) == (128, 12)
    out, bits = block_sparse_attention_variant("wan", q, k, v, top_k, text_blocks=0, block_neighbor_list=nbr,
                                               p_remain_rates=0.9, first_frame_blocks=ff, shape_xfuse=True,
                                               return_mask_bits=True)
    torch.cuda.synchronize()
    assert out.dtype == torch.float32 and out.shape == (1, S, H, 128)
    nb = 256
    oh = bits_to_onehot(bits, nb)
    assert oh[0, :, :ff, :ff].all()                                   # first-frame square (wan/…:400-406)
    assert (oh[0] | ~nbr.to(dev)[None]).all()
    assert int(oh.sum(-1).min()) >= top_k
    # values are bf16-rounded before widening (wan/…:530-532)
    assert torch.equal(out, out.bfloat16().float())
    _check_rows(q.bfloat16(), k.bfloat16(), v, out, oh, nb, S, nb * 128, (0, 5, 128, 255), (0, 11), 0)


def test_hyvideo_i2v_full_size_ragged():
    """HunyuanVideo-I2V shape: 115200 image + 400 text tokens -> 904 blocks, text_blocks=4, the
    last block has 112 zero-padded rows that text queries DO attend (SURVEY A-3)."""
    import bench
    from jenga_b200 import gilbert
    from jenga_b200.attention import bits_to_onehot, block_sparse_attention_variant
    dev = torch.device("cuda", 0)
    n_img, T, H = 115200, 400, 4  # 4 of the 24 heads keep the test short; the shape per head is full size
    S = n_img + T
    q = bench.synth_tokens(S, H, dev, 5321)
    k = bench.synth_tokens(S, H, dev, 5322)
    v = torch.randn(1, S, H, 128, device=dev, generator=torch.Generator(device=dev).manual_seed(5323)).bfloat16()
    nbr = gilbert.gilbert_block_neighbor_mapping(32, 45, 80)
    cu = torch.tensor([0, n_img + 300, S], dtype=torch.int32, device=dev)
    top_k = int((1 - 0.75) * (n_img // 128))
    out, bits = block_sparse_attention_variant("hyvideo_i2v", q, k, v, top_k, cu_seqlens_q=cu, cu_seqlens_kv=cu,
                                               text_blocks=4, block_neighbor_list=nbr, p_remain_rates=0.3,
                                               shape_xfuse=True, return_mask_bits=True)
    torch.cuda.synchronize()
    assert out.shape == (1, S, H, 128)
    oh = bits_to_onehot(bits, 904)
    assert oh[..., 900:904].all() and bits.shape[2] == 900
    _check_rows(q, k, v, out, oh, 900, n_img + 300, 904 * 128, (0, 899, 900, 903), (0, 3), 4)
