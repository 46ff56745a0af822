#!/usr/bin/env python
"""Wan2.1 DiT block stack on one GPU: unmodified wan/modules/model_mul.py WanAttentionBlocks (T2V or
I2V cross-attention, cross_attn_norm=True, random init, fp32 parameters, bf16 autocast as jenga_wan.py
runs them) timed three ways on the same weights and inputs:

  A  the reference operator (Triton + FlashAttention-2), if both import
  B  the original WanAttentionBlock and WanT2VCrossAttention / WanI2VCrossAttention forwards on the
     jenga_b200 operator (WanSelfAttention patched): what `python -m jenga_b200.install jenga_wan.py`
     ran before the fused Wan forwards existed
  C  the fused forwards that install() patches in (jenga_b200/blocks.py)

Block 0 receives a bf16 x (patch_embedding runs under bf16 autocast) and returns the fp32 residual
stream the following blocks carry.  Default shape: Wan-14B (scripts/wan_14B_jenga_base.sh), grid
21x45x80, dim 5120, 40 heads, ffn 13824, 512 context tokens, sa_drop_rate 0.7, p_remain_rates 0.8,
4 blocks.  --model 1.3b: grid 21x30x52, dim 1536, 12 heads, ffn 8960, 0.75 / 0.9, 8 blocks.
--model i2v-14b (jenga_wan.py --task i2v-14B): the 14B shape with "i2v_cross_attn" blocks, the context
cat(fp32 [1, 257, C] CLIP tokens, bf16 [1, 512, C] text) = fp32 as jenga_wan.py:577-579 builds it,
sa_drop_rate 0.0 (the I2V path never passes one), 4 blocks; it also times the I2V cross-attention
kernel alone at L = 75 600, H = 40 against the two dense launches + fp32 add + bf16 cast it replaces.
Legs alternate after a warm-up; CUDA events time each stack.  One JSON line on stdout; nothing is
written to the tree.

    python bench_wan_blocks.py [--model 14b|1.3b|i2v-14b] [--blocks N] [--reps 3]
"""
from __future__ import annotations

import argparse
import contextlib
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

from bench_i2v_blocks import card  # noqa: E402

MODELS = {
    # grid, dim, heads, ffn, sa_drop_rate, p_remain_rates, blocks
    "14b": ((21, 45, 80), 5120, 40, 13824, 0.7, 0.8, 4),
    "1.3b": ((21, 30, 52), 1536, 12, 8960, 0.75, 0.9, 8),
    "i2v-14b": ((21, 45, 80), 5120, 40, 13824, 0.0, 0.8, 4),
}
I2V_IMG_TOKENS = 257


def modelled_bytes(L: int, C: int, i2v: bool = False) -> dict:
    """HBM bytes per block of the elementwise chains around the Linears and attentions, eager (one
    read and one write per ATen kernel, L2 ignored) and fused, from the activation shape alone"""
    lc = L * C
    # bytes per (row, channel): eager ATen chain -> fused pass
    chains = {
        # x fp32: layer_norm 4+4, * (1+e) 4+4, + e 4+4, three bf16 casts at q / k / v 3 x (4+2)
        # -> read 4, write 2
        "norm1_modulate": (42, 6),
        # y*e 2+4, x + . 4+4+4, affine layer_norm 4+4, cast at cross q 4+2 -> read 4+2, write 4+2
        "gate1_norm3": (32, 12),
        # q: .float() 2+4, pow 4+4, mean 4, * rsqrt 4+4, type_as 4+2, * w 2+4, half() 4+2,
        # fp32 output 2+4, cast at o 4+2 -> prologue read 2, write 2
        "cross_q_rmsnorm": (56, 4),
        # I2V instead of cross_q_rmsnorm: q as above up to the first half() (44), a second half() 4+2, two
        # fp32 outputs 2 x (2+4), x + img_x 4+4+4, cast at o 4+2 -> prologue read 2, write 2
        "i2v_cross": (80, 4),
        # x + y 4+2+4, layer_norm 4+4, * (1+e) 4+4, + e 4+4, cast at ffn 4+2 -> read 4+2, write 4+2
        "cross_residual_norm2": (40, 12),
        # y*e 2+4, x + . 4+4+4 -> read 4+2, write 4
        "gate2": (18, 10),
    }
    chains.pop("cross_q_rmsnorm" if i2v else "i2v_cross")
    out = {k: {"eager_gb": e * lc / 1e9, "fused_gb": f * lc / 1e9} for k, (e, f) in chains.items()}
    out["total"] = {"eager_gb": sum(e for e, _ in chains.values()) * lc / 1e9,
                    "fused_gb": sum(f for _, f in chains.values()) * lc / 1e9}
    return out


def i2v_cross_kernel(dev, L: int, H: int, Li: int, Lt: int, launches: int = 20, rounds: int = 3) -> dict:
    """jenga_wan_i2v_cross_attn alone against the composition it replaces — two dense-class launches of
    the attention kernel (as wan.cross_attention issues them), an fp32 add and the bf16 cast — on the same
    seeded bf16 inputs.  The two alternate, `launches` back-to-back calls per CUDA-event window; the best
    window of `rounds` is reported per call."""
    from jenga_b200 import wan
    from jenga_b200.attention import BLOCK, _launch
    g = torch.Generator(device=dev).manual_seed(7)
    r = lambda n: torch.randn(1, n, H, 128, generator=g, device=dev).bfloat16()  # noqa: E731
    q, ki, vi, kt, vt = r(L), r(Li), r(Li), r(Lt), r(Lt)
    nq = (L + BLOCK - 1) // BLOCK
    out = torch.empty_like(q)
    a_img, a_txt = torch.empty_like(q), torch.empty_like(q)

    def fused():
        return wan.i2v_cross_attn(q, ki, vi, kt, vt, out=out)

    def composed():
        for k, v, o in ((ki, vi, a_img), (kt, vt, a_txt)):
            _launch(q, k, v, None, 0, nq, 128 ** -0.5, 0.0, 1 << 30, k.shape[1], L, k.shape[1], o, None,
                    torch.bfloat16)
        return (a_txt.float() + a_img.float()).bfloat16()

    def window(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / launches

    got, want = fused().clone(), composed()
    torch.cuda.synchronize()
    ms = {"fused": [], "composed": []}
    for _ in range(rounds):
        ms["fused"].append(window(fused))
        ms["composed"].append(window(composed))
    flop = 4.0 * L * H * 128 * (Li + Lt)          # Q K^T and P V over both segments
    best = {k: min(v) for k, v in ms.items()}
    d = (got.float() - want.float()).abs()
    return {
        "L": L, "heads": H, "img_keys": Li, "txt_keys": Lt, "launches_per_window": launches,
        "ms_per_call": best, "ms_all": ms, "composed_over_fused": best["composed"] / best["fused"],
        "algorithmic_tflop_per_call": flop / 1e12,
        "tflops": {k: flop / (v * 1e-3) / 1e12 for k, v in best.items()},
        "bit_identical": bool(torch.equal(got, want)), "max_abs_diff": d.max().item(),
        "elements_differing": int((d > 0).sum().item()),
    }


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--model", choices=sorted(MODELS), default="14b")
    ap.add_argument("--blocks", type=int, default=None, help="blocks in the stack (default: per model)")
    ap.add_argument("--reps", type=int, default=3, help="timed stack forwards per leg")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_wan_blocks.py measures on a GPU; none is visible")
    from oracle import ref_loader
    if not ref_loader.available():
        raise SystemExit("oracle/_ref/ is not staged: run __graft_entry__.build() first")
    (f, h, w), dim, heads, ffn, drop, p_remain, n_blocks = MODELS[args.model]
    n_blocks = args.blocks or n_blocks
    i2v = args.model.startswith("i2v")
    Lc = 512
    dev = torch.device("cuda")

    # the reference module first, so that its flash_attention binds the real FlashAttention-2 before
    # install() puts the shim in sys.modules
    ref, ref_err = None, None
    try:
        import flash_attn  # noqa: F401
        import triton  # noqa: F401
        ref = ref_loader.load_blocks(product=False)[1]
    except Exception as e:  # noqa: BLE001
        ref_err = f"{type(e).__name__}: {e}"
    our = ref_loader.load_blocks(product=True)[1]
    from jenga_b200 import blocks as jb
    from jenga_b200 import gilbert

    g = torch.Generator(device=dev).manual_seed(2024)

    def init(m):
        with torch.no_grad():
            for n_, p_ in m.named_parameters():
                if p_.dim() >= 2 and "modulation" not in n_:
                    p_.copy_(torch.randn(p_.shape, generator=g, device=dev).mul_(0.02))
                elif "norm" in n_ and n_.endswith("weight"):
                    p_.fill_(1.0)
                else:
                    p_.copy_(torch.randn(p_.shape, generator=g, device=dev).mul_(0.02))

    cross_type = "i2v_cross_attn" if i2v else "t2v_cross_attn"

    def stack(mod, meta=False):
        mk = lambda: mod.WanAttentionBlock(cross_type, dim, ffn, heads, (-1, -1), True, True, 1e-6)  # noqa: E731
        if meta:
            with torch.device("meta"):
                return [mk() for _ in range(n_blocks)]
        with torch.device(dev):
            return [mk() for _ in range(n_blocks)]

    ob = stack(our)
    for b_ in ob:
        init(b_)
    rb = None
    if ref is not None:
        rb = stack(ref, meta=True)
        for a_, b_ in zip(rb, ob):
            a_.load_state_dict(b_.state_dict(), assign=True)      # shared weights, no second copy

    L = f * h * w
    _, h2l = gilbert.mapping_tensors(f, h, w, sliced=True)
    nbr = gilbert.block_neighbor_mapping(f, h, w, sliced=True)
    d = dim // heads
    freqs = torch.cat([our.rope_params(1024, d - 4 * (d // 6)), our.rope_params(1024, 2 * (d // 6)),
                       our.rope_params(1024, 2 * (d // 6))], dim=1).to(dev)      # WanModel moves it, :550-551
    seq_lens = torch.tensor([L], dtype=torch.long)
    grid = torch.tensor([[f, h, w]], dtype=torch.long)
    x0 = torch.randn(1, L, dim, generator=g, device=dev).bfloat16()
    e0 = 0.1 * torch.randn(1, 6, dim, generator=g, device=dev)
    ctx = torch.randn(1, Lc, dim, generator=g, device=dev).bfloat16()
    if i2v:
        # img_emb's final LayerNorm runs in fp32 (model_mul.py:379-391); the concat promotes the text
        ctx = torch.concat([torch.randn(1, I2V_IMG_TOKENS, dim, generator=g, device=dev), ctx], dim=1)
    kw = dict(sa_drop_rate=drop, freq_remap=h2l.to(dev), block_neighbor_list=nbr, p_remain_rates=p_remain)

    def forward(blks):
        """the block loop of WanModel.forward (model_mul.py), reorders done once, outside"""
        x = x0
        for blk in blks:
            x = blk(x, e0, seq_lens, grid, freqs, ctx, None, **kw)
        return x

    class unpatched:
        """leg B: the unpatched block and cross-attention forwards for the duration of one stack"""

        def __enter__(self):
            self.saved = {c: getattr(our, c).forward for c in ("WanAttentionBlock", "WanT2VCrossAttention")}
            for c, fn in self.saved.items():
                setattr(getattr(our, c), "forward", fn.__wrapped__)

        def __exit__(self, *exc):
            for c, fn in self.saved.items():
                setattr(getattr(our, c), "forward", fn)

    legs = {"B": (ob, unpatched), "C": (ob, contextlib.nullcontext)}
    if rb is not None:
        legs = {"A": (rb, contextlib.nullcontext), **legs}

    def timed(leg):
        blks, mode = legs[leg]
        e_0, e_1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        with mode():
            e_0.record()
            out = forward(blks)
            e_1.record()
            torch.cuda.synchronize()
        return e_0.elapsed_time(e_1) * 1e-3, out

    times = {k: [] for k in legs}
    outs = {}
    jb.remove_gather_hook()
    info = card()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for k in legs:                                                 # Triton JIT, cuBLAS, caches
            outs[k] = timed(k)[1]
        stats0 = dict(jb.STATS)
        for _ in range(args.reps):
            for k in legs:
                s_, outs[k] = timed(k)
                times[k].append(s_)
    stats = {k: jb.STATS[k] - stats0[k] for k in jb.STATS}
    info_after = card()

    def err(a, b):
        a, b = a.float(), b.float()
        rms = a.pow(2).mean().sqrt().item()
        diff = (b - a).abs()
        return {"max_over_rms": diff.max().item() / rms, "mean_over_rms": diff.mean().item() / rms}

    sec = {k: min(v) for k, v in times.items()}
    res = {
        "bench": "wan_blocks", "model": args.model, "grid": [f, h, w], "tokens": L, "context_tokens": Lc,
        "dim": dim, "heads": heads, "ffn_dim": ffn, "blocks": n_blocks, "sa_drop_rate": drop,
        "p_remain_rates": p_remain, "reps": args.reps,
        "seconds_per_stack": sec, "seconds_all": times,
        "B_over_C": sec["B"] / sec["C"],
        "A_over_C": (sec["A"] / sec["C"]) if "A" in sec else None,
        "output_dtype": str(outs["C"].dtype),
        "stats_per_timed_window": stats,
        "C_vs_B": err(outs["B"], outs["C"]),
        "C_vs_A": err(outs["A"], outs["C"]) if "A" in outs else None,
        "B_vs_A": err(outs["A"], outs["B"]) if "A" in outs else None,
        "modelled_bytes_per_block": modelled_bytes(L, dim, i2v=i2v),
        "reference_leg": "ran" if ref is not None else f"unavailable ({ref_err})",
        "card": info, "card_after": info_after,
    }
    if i2v:
        res["context_tokens"] = I2V_IMG_TOKENS + Lc
        res["i2v_cross_kernel"] = i2v_cross_kernel(dev, L, heads, I2V_IMG_TOKENS, Lc)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
