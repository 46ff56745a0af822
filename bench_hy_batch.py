#!/usr/bin/env python
"""Several videos per DiT call (`--num-videos N`) on one GPU: the fused HunyuanVideo and
HunyuanVideo-I2V block forwards against the original forwards, at N = 1, 2 and 4.

Two stacks of unmodified reference blocks (random init at the HunyuanVideo width, 3072 channels, 24
heads), one after the other:

  hy   the 4 double + 8 single hyvideo/modules/models_mul_block_gc_ha_multigpu.py blocks of
       `bench.py --dit-blocks 4,8`, with its hy720p call: grid 32x45x80 (L = 115200), 256 text tokens of
       which 180 are valid, sa_drop_rate 0.7, p_remain_rates 0.3, text_amp 0
  i2v  the same stack of hyvideo_i2v/modules/models_mul.py blocks with the call of
       bench_i2v_blocks.py: 400 text tokens of which 300 are valid, token_replace with the first frame
       scattered by the Hilbert order, sa_drop_rate 0.75, p_remain_rates 0.3, text_amp 0

Each sample of a batch has its own image rows, text rows, vec and token_replace_vec; all share one
text mask, as the samples of --num-videos share one prompt.  Two legs on the same weights and inputs:

  fused     the forwards install() patches in (jenga_b200/blocks.py)
  original  forward.__wrapped__: the reference forward on the jenga_b200 operator, what a batch > 1
            call ran before the fused forwards took it

After one untimed call of each leg (whose outputs give the distance between the legs), the legs
alternate for --reps rounds; the best round counts.  Per leg: seconds per stack, seconds per video
(stack / N, and that scaled to the DiT loop of one video: 60 blocks x computed steps), and
torch.cuda.max_memory_allocated over the leg's calls (reset at the start of each call, so it is the
peak of one stack forward on top of weights and inputs).  Then the cost of the one-launch-per-sample
LayerNorm + modulate and gate + residual chains (split_cost).  The card's name, power limit and SM
clock are read before and after.  One JSON line on stdout; nothing is written to the tree.

    python bench_hy_batch.py [--models hy,i2v] [--videos 1,2,4] [--reps 3] [--grid 32,45,80]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

HIDDEN, HEADS = 3072, 24
# text tokens, valid, sa_drop_rate, p_remain_rates, text_amp, computed steps per video (bench.py's
# hy720p and hy_i2v720p workloads)
MODELS = {"hy": (256, 180, 0.7, 0.3, 0.0, 23), "i2v": (400, 300, 0.75, 0.3, 0.0, 24)}


def load(model):
    if model == "hy":
        from oracle import ref_loader
        return ref_loader.load_blocks(product=True)[0]
    from i2v_ref import load_i2v_blocks
    return load_i2v_blocks(product=True)


def rms_distance(ref, out):
    a, b = ref.float(), out.float()
    rms = a.pow(2).mean().sqrt().item()
    d = (b - a).abs()
    return {"max_over_rms": d.max().item() / rms, "mean_over_rms": d.mean().item() / rms}


def bench_model(model, n_double, n_single, grid, videos, reps, dev):
    from jenga_b200 import blocks as jb
    from jenga_b200 import gilbert
    T, valid, drop, p_remain, txt_amp, steps = MODELS[model]
    i2v = model == "i2v"
    mod = load(model)
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

    kw = dict(mlp_width_ratio=4.0, dtype=torch.bfloat16, device=dev)
    dbl = [mod.MMDoubleStreamBlock(HIDDEN, HEADS, **kw) for _ in range(n_double)]
    sgl = [mod.MMSingleStreamBlock(HIDDEN, HEADS, **kw) for _ in range(n_single)]
    for b_ in dbl + sgl:
        init(b_)

    t, h, w = grid
    L, S = t * h * w, t * h * w + T
    l2h, h2l = gilbert.mapping_tensors(t, h, w)
    l2h, h2l = l2h.to(dev), h2l.to(dev)
    curve_sel = [[l2h, h2l, gilbert.block_neighbor_mapping(t, h, w).to(dev)]]
    ang = torch.rand(L, 64, generator=g, device=dev) * 6.2831853
    cos = torch.cos(ang).repeat_interleave(2, dim=1).contiguous()[h2l]
    sin = torch.sin(ang).repeat_interleave(2, dim=1).contiguous()[h2l]
    ff0 = torch.zeros(L, dtype=torch.bool, device=dev)
    ff0[:h * w] = True
    ff = ff0[h2l]                                                      # jenga_hyi2v.py:124-126

    def inputs(n):
        """n samples, each from its own draws, image rows in Hilbert order"""
        img = torch.cat([torch.randn(1, L, HIDDEN, generator=g, device=dev).bfloat16()[:, h2l] for _ in range(n)])
        txt = torch.cat([torch.randn(1, T, HIDDEN, generator=g, device=dev).bfloat16() for _ in range(n)])
        vec = torch.randn(n, HIDDEN, generator=g, device=dev).bfloat16()
        tr_vec = torch.randn(n, HIDDEN, generator=g, device=dev).bfloat16()
        text_mask = torch.zeros(n, T, dtype=torch.int64, device=dev)
        text_mask[:, :valid] = 1
        return img, txt, vec, tr_vec, mod.get_cu_seqlens(text_mask, L)

    def forward(call, img, txt, vec, tr_vec, cu):
        """the block loops of jenga_hyvideo.py:132-178 / jenga_hyi2v.py:149-206 (reorders done once)"""
        if i2v:
            full = torch.zeros(S).bool()                               # jenga_hyi2v.py:129-130, per forward
            full[:L] = ff.cpu()
        for blk in dbl:
            if i2v:
                img, txt = call(blk, img, txt, vec, cu, cu, S, S, (cos, sin), drop, ff, "token_replace", tr_vec,
                                h * w, txt_amp, curve_sel, p_remain)
            else:
                img, txt = call(blk, img, txt, vec, cu, cu, S, S, (cos, sin), drop, txt_amp, curve_sel, p_remain)
        x = torch.cat((img, txt), 1)
        for blk in sgl:
            if i2v:
                x = call(blk, x, vec, T, cu, cu, S, S, (cos, sin), drop, full, "token_replace", tr_vec, h * w,
                         txt_amp, curve_sel, p_remain)
            else:
                x = call(blk, x, vec, T, cu, cu, S, S, (cos, sin), drop, txt_amp, curve_sel, p_remain)
        return x

    legs = {"fused": lambda blk, *a: blk(*a),
            "original": lambda blk, *a: type(blk).forward.__wrapped__(blk, *a)}

    def timed(leg, inp):
        """(seconds, peak bytes, output) of one stack forward, or (None, None, None) out of memory"""
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        try:
            e0.record()
            out = forward(legs[leg], *inp)
            e1.record()
            torch.cuda.synchronize()
        except torch.cuda.OutOfMemoryError:
            torch.cuda.empty_cache()
            return None, None, None
        return e0.elapsed_time(e1) * 1e-3, torch.cuda.max_memory_allocated(dev), out

    nblk = n_double + n_single
    res = {"img_tokens": L, "txt_tokens": T, "txt_valid": valid, "sa_drop_rate": drop, "p_remain_rates": p_remain,
           "text_amp": txt_amp, "blocks": {"double": n_double, "single": n_single},
           "condition_type": "token_replace" if i2v else None, "computed_steps": steps, "by_videos": {}}
    jb.remove_gather_hook()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for n in videos:
            inp = inputs(n)
            base = torch.cuda.memory_allocated(dev)
            before = dict(jb.STATS)
            _, _, out_f = timed("fused", inp)
            fused_stats = {k: jb.STATS[k] - before[k] for k in jb.STATS if jb.STATS[k] != before[k]}
            _, _, out_o = timed("original", inp)
            dist = rms_distance(out_o, out_f) if out_f is not None and out_o is not None else None
            del out_f, out_o
            sec = {k: [] for k in legs}
            peak = {k: [] for k in legs}
            for _ in range(reps):
                for leg in legs:
                    s_, p_, o_ = timed(leg, inp)
                    del o_
                    if s_ is not None:
                        sec[leg].append(s_)
                        peak[leg].append(p_)
            row = {"weights_and_inputs_bytes": base, "fused_vs_original": dist, "fused_stats_per_stack": fused_stats}
            for leg in legs:
                best = min(sec[leg]) if sec[leg] else None
                row[leg] = {"seconds_per_stack": best, "seconds_all": sec[leg],
                            "stack_seconds_per_video": best / n if best else None,
                            "dit_loop_seconds_per_video": best / n * 60 / nblk * steps if best else None,
                            "max_memory_allocated_bytes": max(peak[leg]) if peak[leg] else "out of memory"}
            f, o = row["fused"]["seconds_per_stack"], row["original"]["seconds_per_stack"]
            row["original_over_fused"] = o / f if f and o else None
            res["by_videos"][str(n)] = row
            del inp
            torch.cuda.empty_cache()
    del dbl, sgl
    torch.cuda.empty_cache()
    return res


def split_cost(videos, tokens, dev, iters=20, rounds=3):
    """What launching the LayerNorm + modulate and gate + residual chains once per sample costs: x
    [N, tokens, 3072] with [N, C] vectors (N launches each) against the same rows as one sample with one
    vector (one launch each, the same bytes).  Milliseconds per call, best of `rounds` alternating
    windows of `iters` calls."""
    from jenga_b200 import dense as DN
    g = torch.Generator(device=dev).manual_seed(7)
    res = {}
    for n in videos:
        if n == 1:
            continue
        x = torch.randn(n, tokens, HIDDEN, generator=g, device=dev).bfloat16()
        y = torch.randn(n, tokens, HIDDEN, generator=g, device=dev).bfloat16()
        v = torch.randn(n, HIDDEN, generator=g, device=dev).bfloat16()
        x1, y1, v1 = x.view(1, n * tokens, HIDDEN), y.view(1, n * tokens, HIDDEN), v[:1]
        calls = {"ln_modulate_per_sample": lambda: DN.ln_modulate(x, v, v),
                 "ln_modulate_one_launch": lambda: DN.ln_modulate(x1, v1, v1),
                 "gate_residual_per_sample": lambda: DN.gate_residual(x, y, v),
                 "gate_residual_one_launch": lambda: DN.gate_residual(x1, y1, v1)}
        ms = {k: [] for k in calls}
        for fn in calls.values():
            fn()
        for _ in range(rounds):
            for k, fn in calls.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(iters):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                ms[k].append(e0.elapsed_time(e1) / iters)
        res[str(n)] = {k: min(t) for k, t in ms.items()}
        del x, y, x1, y1
        torch.cuda.empty_cache()
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--models", default="hy,i2v", help="stacks to time, in order: hy, i2v")
    ap.add_argument("--videos", default="1,2,4", help="samples per DiT call")
    ap.add_argument("--blocks", default="4,8", help="double,single blocks in each stack")
    ap.add_argument("--reps", type=int, default=3, help="timed rounds; the best counts")
    ap.add_argument("--grid", default="32,45,80", help="latent t,h,w")
    args = ap.parse_args(argv)
    models = [m for m in args.models.split(",") if m]
    if any(m not in MODELS for m in models):
        raise SystemExit(f"--models takes {', '.join(MODELS)}")
    videos = [int(v) for v in args.videos.split(",")]
    n_double, n_single = (int(v) for v in args.blocks.split(","))
    grid = tuple(int(v) for v in args.grid.split(","))
    if not torch.cuda.is_available():
        raise SystemExit("bench_hy_batch.py measures on a GPU; none is visible")
    from oracle import ref_loader
    if not ref_loader.available():
        raise SystemExit("oracle/_ref/ is not staged: run __graft_entry__.build() first")
    from bench_i2v_blocks import card
    dev = torch.device("cuda")
    info = card()
    out = {"bench": "hy_batch", "grid": list(grid), "hidden": HIDDEN, "heads": HEADS, "reps": args.reps,
           "models": {m: bench_model(m, n_double, n_single, grid, videos, args.reps, dev) for m in models}}
    with torch.no_grad():
        out["per_sample_launch_cost_ms"] = split_cost(videos, grid[0] * grid[1] * grid[2] + MODELS["hy"][0], dev)
    out.update(card=info, card_after=card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
