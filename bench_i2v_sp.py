#!/usr/bin/env python
"""Sequence-parallel HunyuanVideo-I2V block stack: the unmodified hyvideo_i2v/modules/models_mul.py
blocks (random init at the HunyuanVideo width, 4 double + 8 single as in bench_i2v_blocks.py) on one
GPU against the same stack sharded over the N ranks of `torchrun --nproc-per-node N`.

  single  every rank runs the whole stack on its own GPU (the fused I2V forwards, L image rows)
  sp      every rank runs its Hilbert slice of L/N image rows with `block.jenga_sp` set, the route of
          jenga_b200/hyi2v_sp.py: the attention runs over the Ulysses exchange (peer stores, or the
          NCCL all-to-all where symmetric memory is unavailable)

Same inputs and settings as bench_i2v_blocks.py (grid 32x45x80, 400 text tokens of which 300 are
valid, token_replace, sa_drop_rate 0.75, p_remain_rates 0.3, bf16 autocast).  Reports seconds per
stack (the slowest rank, CUDA events), the SM clock at the start and end of each leg, and the distance
of the gathered sp image rows from the single-GPU rows in units of their RMS.  The sp leg's timed
region is the block stack plus the all-gather of the image rows that the sharded forward adds once
per forward; the Hilbert gather, the slicing of the inputs, the inverse scatter and the final layer
are outside both legs.  Rank 0 prints one JSON line; nothing is written to the tree.

    torchrun --nproc-per-node N bench_i2v_sp.py [--blocks 4,8] [--reps 3]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from pathlib import Path

import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--blocks", default="4,8", help="double,single blocks in the stack")
    ap.add_argument("--reps", type=int, default=3, help="timed stack forwards per leg")
    ap.add_argument("--grid", default="32,45,80", help="latent t,h,w")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_i2v_sp.py measures on GPUs; none is visible")
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl")
    P, r = dist.get_world_size(), dist.get_rank()
    from oracle import ref_loader
    if not ref_loader.available():
        raise SystemExit("oracle/_ref/ is not staged: run __graft_entry__.build() first")
    from bench_i2v_blocks import card
    from i2v_ref import load_i2v_blocks
    from jenga_b200 import blocks as jb
    from jenga_b200 import gilbert
    from jenga_b200.sharding import check_degree, default_attention, shard

    n_double, n_single = (int(v) for v in args.blocks.split(","))
    t, h, w = (int(v) for v in args.grid.split(","))
    hidden, heads, T, valid = 3072, 24, 400, 300
    drop, p_remain, txt_amp = 0.75, 0.3, 0.0
    L = t * h * w
    check_degree(L, heads, P, "HunyuanVideo-I2V")
    n = L // P
    dev = torch.device("cuda", local)
    mod = load_i2v_blocks(product=True)
    jb.remove_gather_hook()
    g = torch.Generator(device=dev).manual_seed(2024)            # the same weights and inputs on every rank

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
    dbl = [mod.MMDoubleStreamBlock(hidden, heads, **kw) for _ in range(n_double)]
    sgl = [mod.MMSingleStreamBlock(hidden, heads, **kw) for _ in range(n_single)]
    for b_ in dbl + sgl:
        init(b_)
    l2h, h2l = gilbert.mapping_tensors(t, h, w)
    l2h, h2l = l2h.to(dev), h2l.to(dev)
    curve_sel = [[l2h, h2l, gilbert.block_neighbor_mapping(t, h, w).to(dev)]]
    img0 = torch.randn(1, L, hidden, generator=g, device=dev).bfloat16()
    txt0 = torch.randn(1, T, hidden, generator=g, device=dev).bfloat16()
    vec = torch.randn(1, hidden, generator=g, device=dev).bfloat16()
    tr_vec = torch.randn(1, hidden, generator=g, device=dev).bfloat16()
    ang = torch.rand(L, 64, generator=g, device=dev) * 6.2831853
    cos = torch.cos(ang).repeat_interleave(2, dim=1).contiguous()[h2l]
    sin = torch.sin(ang).repeat_interleave(2, dim=1).contiguous()[h2l]
    ff0 = torch.zeros(L, dtype=torch.bool, device=dev)
    ff0[:h * w] = True
    ff = ff0[h2l]
    img_h = img0[:, h2l]
    shards = dict(img=shard(img_h, 1, P, r), cos=shard(cos, 0, P, r), sin=shard(sin, 0, P, r), ff=shard(ff, 0, P, r))

    def forward(rows, img, cos_, sin_, ff_):
        """jenga_hyi2v.py:149-206 on `rows` image rows (L on one GPU, L/N on a rank)"""
        cu = torch.tensor([0, rows + valid, rows + T], dtype=torch.int32, device=dev)
        full = torch.zeros(rows + T).bool()
        full[:rows] = ff_.cpu()
        S = rows + T
        txt = txt0
        for blk in dbl:
            img, txt = blk(img, txt, vec, cu, cu, S, S, (cos_, sin_), drop, ff_, "token_replace", tr_vec, h * w,
                           txt_amp, curve_sel, p_remain)
        x = torch.cat((img, txt), 1)
        for blk in sgl:
            x = blk(x, vec, T, cu, cu, S, S, (cos_, sin_), drop, full, "token_replace", tr_vec, h * w, txt_amp,
                    curve_sel, p_remain)
        return x[:, :rows]

    def set_sp(sp):
        for b_ in dbl + sgl:
            if sp is None:
                b_.__dict__.pop("jenga_sp", None)
            else:
                b_.jenga_sp = sp

    def sp_forward():
        out = forward(n, shards["img"], shards["cos"], shards["sin"], shards["ff"])
        parts = [torch.empty_like(out) for _ in range(P)]
        dist.all_gather(parts, out.contiguous())                      # as hyi2v_sp's forward does
        return torch.cat(parts, 1)

    legs = {"single": lambda: forward(L, img_h, cos, sin, ff), "sp": sp_forward}
    sp = default_attention(None, "hyvideo_i2v")

    def timed(leg):
        set_sp(sp if leg == "sp" else None)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dist.barrier()
        torch.cuda.synchronize()
        e0.record()
        out = legs[leg]()
        e1.record()
        torch.cuda.synchronize()
        s = torch.tensor([e0.elapsed_time(e1) * 1e-3], device=dev)
        dist.all_reduce(s, op=dist.ReduceOp.MAX)
        return s.item(), out

    times = {k: [] for k in legs}
    clocks = {k: [] for k in legs}
    outs = {}
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for k in legs:                                                 # warm-up: cuBLAS, buffers, caches
            outs[k] = timed(k)[1]
        stats0 = dict(jb.STATS)
        for _ in range(args.reps):
            for k in legs:
                c0 = card().get("sm_mhz")
                s_, outs[k] = timed(k)
                times[k].append(s_)
                clocks[k].append([c0, card().get("sm_mhz")])
    stats = {k: jb.STATS[k] - stats0[k] for k in jb.STATS if jb.STATS[k] != stats0[k]}
    a, b = outs["single"].float(), outs["sp"].float()
    rms = a.pow(2).mean().sqrt().item()
    d = (b - a).abs()
    if r == 0:
        sec = {k: min(v) for k, v in times.items()}
        print(json.dumps({
            "bench": "i2v_sp", "world": P, "grid": [t, h, w], "img_tokens": L, "txt_tokens": T, "txt_valid": valid,
            "hidden": hidden, "heads": heads, "blocks": {"double": n_double, "single": n_single},
            "sa_drop_rate": drop, "p_remain_rates": p_remain, "condition_type": "token_replace", "reps": args.reps,
            "exchange": type(sp).__name__,
            "timed": "block stack; sp leg also the image-row all-gather",
            "seconds_per_stack": sec, "seconds_all": times,
            "speedup": sec["single"] / sec["sp"], "sm_mhz_start_end": clocks,
            "sp_vs_single": {"max_over_rms": d.max().item() / rms, "mean_over_rms": d.mean().item() / rms},
            "stats_per_timed_window_rank0": stats, "card": card()}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
