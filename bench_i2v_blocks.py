#!/usr/bin/env python
"""HunyuanVideo-I2V DiT block stack on one GPU: the unmodified hyvideo_i2v/modules/models_mul.py
blocks (MMDoubleStreamBlock / MMSingleStreamBlock, random init at the HunyuanVideo width) timed
three ways on the same weights and inputs:

  A  the reference operator (Triton + FlashAttention-2), if both import
  B  the original I2V forwards bound to the jenga_b200 operator: what `python -m jenga_b200.install
     jenga_hyi2v.py` ran before the fused I2V forwards existed (forward.__wrapped__)
  C  the fused I2V forwards that install() patches in (jenga_b200/blocks.py)

The call sequence is that of jenga_hyi2v.py:118-206 with the hyi2v_jenga_base.sh settings: grid
32x45x80 (L = 115200), 400 text tokens of which 300 are valid, token_replace with the first frame
scattered by the Hilbert order (a device mask for the double blocks, a CPU mask built anew on every
forward for the single blocks), sa_drop_rate 0.75, p_remain_rates 0.3, text_amp 0, bf16 autocast.
Legs alternate after a warm-up; CUDA events time each stack.  One JSON line on stdout; nothing is
written to the tree.

    python bench_i2v_blocks.py [--blocks 4,8] [--reps 3]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def card():
    """name, power limit and SM clock of the current device, read now"""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10)
        name, pl, sm, smax = [s.strip() for s in r.stdout.strip().split(",")]
        return {"name": name, "power_limit_w": pl, "sm_mhz": sm, "sm_max_mhz": smax}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(), "nvidia_smi": f"unavailable: {e}"}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--blocks", default="4,8", help="double,single blocks in the stack")
    ap.add_argument("--reps", type=int, default=3, help="timed stack forwards per leg")
    ap.add_argument("--grid", default="32,45,80", help="latent t,h,w")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_i2v_blocks.py measures on a GPU; none is visible")
    from oracle import ref_loader
    if not ref_loader.available():
        raise SystemExit("oracle/_ref/ is not staged: run __graft_entry__.build() first")
    n_double, n_single = (int(v) for v in args.blocks.split(","))
    t, h, w = (int(v) for v in args.grid.split(","))
    hidden, heads, T, valid = 3072, 24, 400, 300
    drop, p_remain, txt_amp = 0.75, 0.3, 0.0
    dev = torch.device("cuda")

    from i2v_ref import load_i2v_blocks
    our = load_i2v_blocks(product=True)
    ref, ref_err = None, None
    try:
        import flash_attn  # noqa: F401
        import triton  # noqa: F401
        ref = load_i2v_blocks(product=False)
    except Exception as e:  # noqa: BLE001
        ref_err = f"{type(e).__name__}: {e}"
    from jenga_b200 import blocks as jb
    from jenga_b200 import gilbert

    g = torch.Generator(device=dev).manual_seed(2024)

    def init(m):
        with torch.no_grad():
            for n_, p_ in m.named_parameters():
                if p_.dim() >= 2:
                    p_.copy_(torch.randn(p_.shape, generator=g, device=dev).mul_(0.02))
                elif "norm" in n_:
                    p_.fill_(1.0)
                else:
                    p_.copy_(torch.randn(p_.shape, generator=g, device=dev).mul_(0.02))

    def stack(mod, meta=False):
        kw = dict(mlp_width_ratio=4.0, dtype=torch.bfloat16)
        if meta:
            with torch.device("meta"):
                return ([mod.MMDoubleStreamBlock(hidden, heads, **kw) for _ in range(n_double)],
                        [mod.MMSingleStreamBlock(hidden, heads, **kw) for _ in range(n_single)])
        return ([mod.MMDoubleStreamBlock(hidden, heads, device=dev, **kw) for _ in range(n_double)],
                [mod.MMSingleStreamBlock(hidden, heads, device=dev, **kw) for _ in range(n_single)])

    od, osg = stack(our)
    for b_ in od + osg:
        init(b_)
    rd = rs = None
    if ref is not None:
        rd, rs = stack(ref, meta=True)
        for a_, b_ in zip(rd + rs, od + osg):
            a_.load_state_dict(b_.state_dict(), assign=True)     # shared weights, no second copy

    L = t * h * w
    l2h, h2l = gilbert.mapping_tensors(t, h, w)
    l2h, h2l = l2h.to(dev), h2l.to(dev)
    nbr = gilbert.block_neighbor_mapping(t, h, w).to(dev)
    curve_sel = [[l2h, h2l, nbr]]
    img0 = torch.randn(1, L, hidden, generator=g, device=dev).bfloat16()
    txt0 = torch.randn(1, T, hidden, generator=g, device=dev).bfloat16()
    vec = torch.randn(1, hidden, generator=g, device=dev).bfloat16()
    tr_vec = torch.randn(1, hidden, generator=g, device=dev).bfloat16()
    ang = torch.rand(L, 64, generator=g, device=dev) * 6.2831853
    cos = torch.cos(ang).repeat_interleave(2, dim=1).contiguous()[h2l]
    sin = torch.sin(ang).repeat_interleave(2, dim=1).contiguous()[h2l]
    text_mask = torch.zeros(1, T, dtype=torch.int64, device=dev)
    text_mask[:, :valid] = 1
    cu = our.get_cu_seqlens(text_mask, L)
    ff0 = torch.zeros(L, dtype=torch.bool, device=dev)
    ff0[:h * w] = True
    ff = ff0[h2l]                                                      # jenga_hyi2v.py:124-126
    img_h = img0[:, h2l]
    S = L + T

    def forward(dbl, sgl, call):
        """the block loop of jenga_hyi2v.py:149-206 (reorders done once, outside)"""
        full = torch.zeros(L + T).bool()                               # :129-130, anew per forward
        full[:L] = ff.cpu()
        img, txt = img_h, txt0
        for blk in dbl:
            img, txt = call(blk, img, txt, vec, cu, cu, S, S, (cos, sin), drop, ff, "token_replace", tr_vec, h * w,
                            txt_amp, curve_sel, p_remain)
        x = torch.cat((img, txt), 1)
        for blk in sgl:
            x = call(blk, x, vec, T, cu, cu, S, S, (cos, sin), drop, full, "token_replace", tr_vec, h * w, txt_amp,
                     curve_sel, p_remain)
        return x

    fused = lambda blk, *a: blk(*a)                                    # noqa: E731
    original = lambda blk, *a: type(blk).forward.__wrapped__(blk, *a)   # noqa: E731
    legs = {"B": (od, osg, original), "C": (od, osg, fused)}
    if ref is not None:
        legs = {"A": (rd, rs, fused), **legs}

    def timed(leg):
        d_, s_, call = legs[leg]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = forward(d_, s_, call)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3, out

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
        d = (b - a).abs()
        return {"max_over_rms": d.max().item() / rms, "mean_over_rms": d.mean().item() / rms}

    sec = {k: min(v) for k, v in times.items()}
    res = {
        "bench": "i2v_blocks", "grid": [t, h, w], "img_tokens": L, "txt_tokens": T, "txt_valid": valid,
        "hidden": hidden, "heads": heads, "blocks": {"double": n_double, "single": n_single},
        "sa_drop_rate": drop, "p_remain_rates": p_remain, "condition_type": "token_replace", "reps": args.reps,
        "seconds_per_stack": sec, "seconds_all": times,
        "B_over_C": sec["B"] / sec["C"],
        "A_over_C": (sec["A"] / sec["C"]) if "A" in sec else None,
        "stats_per_timed_window": stats,
        "C_vs_B": err(outs["B"], outs["C"]),
        "C_vs_A": err(outs["A"], outs["C"]) if "A" in outs else None,
        "B_vs_A": err(outs["A"], outs["B"]) if "A" in outs else None,
        "reference_leg": "ran" if ref is not None else f"unavailable ({ref_err})",
        "card": info, "card_after": info_after,
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
