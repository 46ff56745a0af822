#!/usr/bin/env python
"""Carved against dense self-attention for the Wan2.1-I2V block stack: the unmodified wan/modules/model.py
I2V WanAttentionBlocks (random init at Wan-I2V-14B, 4 blocks) with the fused forwards of the single-GPU
I2V route, on one GPU and sharded over the N ranks of `torchrun --nproc-per-node N`.

  single_dense   L raster rows, sa_drop_rate 0: the fused prologue and the dense class (the default route)
  single_carved  L Hilbert rows of the sliced Gilbert curve, sa_drop_rate --sa-drop-rate: the Wan operator
                 with top_k and first_frame_blocks of the single-GPU rule (JENGA_WAN_I2V_SA_DROP)
  sp_dense       rank r's raster rows [r*n, min((r+1)*n, L)), n = ceil(L/N), the dense class over the
                 Ulysses exchange (parallelize_wan_i2v's default route) + the row all-gather
  sp_carved      rank r's Hilbert rows, the carved operator over the exchange + the row all-gather

Inputs of Wan-I2V-14B 720p: grid 21x45x80 (75 600 tokens), 257 CLIP + 512 text context rows in fp32, bf16
autocast.  The legs alternate; each reports seconds per stack (the slowest rank, CUDA events, best of
--reps), the SM clock at the start and end of each timed stack and its live (query block, key block)
tiles per stack over all heads (dense: heads x nb^2 per block).  Also the card's name and power limit,
read in the same run, and the distance of each sp leg's rows from its single leg's in units of RMS.
Rank 0 prints one JSON line; nothing is written to the tree.

    torchrun --nproc-per-node N bench_wan_i2v_carve.py [--sa-drop-rate 0.7] [--blocks 4] [--reps 3]
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
    ap.add_argument("--sa-drop-rate", type=float, default=0.7, help="drop rate of the carved legs (> 0.25)")
    ap.add_argument("--blocks", type=int, default=4, help="blocks in the stack")
    ap.add_argument("--reps", type=int, default=3, help="timed stack forwards per leg")
    ap.add_argument("--grid", default="21,45,80", help="latent f,h,w (after patching)")
    args = ap.parse_args(argv)
    if not 0.25 < args.sa_drop_rate < 1:
        raise SystemExit("--sa-drop-rate must be in (0.25, 1): at <= 0.25 the carved leg runs the dense class")
    if not torch.cuda.is_available():
        raise SystemExit("bench_wan_i2v_carve.py measures on GPUs; none is visible")
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl")
    P, r = dist.get_world_size(), dist.get_rank()
    from bench_i2v_blocks import card
    from jenga_b200 import attention as A
    from jenga_b200 import blocks as jb
    from jenga_b200.sharding import check_world, default_attention, shard, shard_rows
    from jenga_b200.wan_sp import i2v_curve
    from test_wan_i2v_sp_cpu import load_plain_wan
    mod = load_plain_wan(wan_sp=False)
    if mod is None:
        raise SystemExit("oracle/_ref/ and oracle/_ref_wan_model/ are not staged: run __graft_entry__.build() first")
    jb.patch_plain_wan(mod)                                  # what a single-GPU WanI2V does when it is built

    f, h, w = (int(v) for v in args.grid.split(","))
    dim, heads, ffn, n_img, n_txt = 5120, 40, 13824, 257, 512
    L = f * h * w
    nb = (L + 127) // 128
    check_world(heads, P, "Wan2.1")
    n, _ = shard_rows(L, P, r, "Wan2.1")
    dev = torch.device("cuda", local)
    g = torch.Generator(device=dev).manual_seed(2024)            # the same weights and inputs on every rank

    def init(m):
        with torch.no_grad():
            for n_, p_ in m.named_parameters():
                if "norm" in n_ and n_.endswith("weight"):
                    p_.fill_(1.0)
                else:
                    p_.copy_(torch.randn(p_.shape, generator=g, device=dev).mul_(0.02))

    with torch.device(dev):
        blks = [mod.WanAttentionBlock("i2v_cross_attn", dim, ffn, heads, (-1, -1), True, True, 1e-6)
                for _ in range(args.blocks)]
    for b_ in blks:
        init(b_)
    d = dim // heads
    freqs = torch.cat([mod.rope_params(1024, d - 4 * (d // 6)), mod.rope_params(1024, 2 * (d // 6)),
                       mod.rope_params(1024, 2 * (d // 6))], dim=1).to(dev)
    seq_lens = torch.tensor([L], dtype=torch.long)
    grid = torch.tensor([[f, h, w]], dtype=torch.long)
    x0 = torch.randn(1, L, dim, generator=g, device=dev).bfloat16()     # raster rows
    e0 = 0.1 * torch.randn(1, 6, dim, generator=g, device=dev)
    ctx = torch.randn(1, n_img + n_txt, dim, generator=g, device=dev)   # fp32, as cat(CLIP, text) arrives
    l2h, h2l, nbr = i2v_curve(f, h, w)
    xh = x0[:, h2l.to(dev)].contiguous()                                # Hilbert rows
    carve = dict(sa_drop_rate=args.sa_drop_rate, block_neighbor_list=nbr, p_remain_rates=0.8)
    sp = default_attention(None, "wan")
    # leg -> (rows, block keyword arguments, sharded)
    legs = {
        "single_dense": (x0, dict(sa_drop_rate=0.0), False),
        "single_carved": (xh, dict(carve, freq_remap=h2l.to(dev)), False),
        "sp_dense": (shard(x0, 1, P, r), {}, True),
        "sp_carved": (shard(xh, 1, P, r), dict(carve, freq_remap=shard(h2l, 0, P, r).to(dev)), True),
    }

    def forward(leg):
        x, kw, sharded = legs[leg]
        for b_ in blks:
            if sharded:
                b_.self_attn.jenga_sp = sp
            else:
                b_.self_attn.__dict__.pop("jenga_sp", None)
        for b_ in blks:
            x = b_(x, e0, seq_lens, grid, freqs, ctx, None, **kw)
        if not sharded:
            return x
        parts = [torch.empty_like(x) for _ in range(P)]
        dist.all_gather(parts, x.contiguous())                       # as the sharded forward does (of the head)
        return torch.cat(parts, 1)[:, :L]

    def timed(leg):
        e_0, e_1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dist.barrier()
        torch.cuda.synchronize()
        e_0.record()
        out = forward(leg)
        e_1.record()
        torch.cuda.synchronize()
        s = torch.tensor([e_0.elapsed_time(e_1) * 1e-3], device=dev)
        dist.all_reduce(s, op=dist.ReduceOp.MAX)
        return s.item(), out

    times = {k: [] for k in legs}
    clocks = {k: [] for k in legs}
    tiles = {}
    outs = {}
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for k in legs:                                                  # warm-up, and the live tiles
            A.MASK_CAPTURE = []
            outs[k] = timed(k)[1]
            live = sum(int(A.bits_to_onehot(bits, m).sum()) for bits, m in A.MASK_CAPTURE)
            A.MASK_CAPTURE = None
            t_ = torch.tensor([live], device=dev, dtype=torch.float64)
            dist.all_reduce(t_)                                         # the ranks' head groups
            tiles[k] = int(t_.item()) if "carved" in k else args.blocks * heads * nb * nb
        stats0 = dict(jb.STATS)
        for _ in range(args.reps):
            for k in legs:
                c0 = card().get("sm_mhz")
                s_, outs[k] = timed(k)
                times[k].append(s_)
                clocks[k].append([c0, card().get("sm_mhz")])
    stats = {k: jb.STATS[k] - stats0[k] for k in jb.STATS if jb.STATS[k] != stats0[k]}

    def dist_rms(a, b):
        a, b = a.float(), b.float()
        rms = a.pow(2).mean().sqrt().item()
        dd = (b - a).abs()
        return {"max_over_rms": dd.max().item() / rms, "mean_over_rms": dd.mean().item() / rms}

    if r == 0:
        sec = {k: min(v) for k, v in times.items()}
        print(json.dumps({
            "bench": "wan_i2v_carve", "world": P, "grid": [f, h, w], "tokens": L, "rows_per_rank": n,
            "dim": dim, "heads": heads, "blocks": args.blocks, "context_tokens": [n_img, n_txt],
            "sa_drop_rate": args.sa_drop_rate, "reps": args.reps, "exchange": type(sp).__name__,
            "timed": "block stack; sp legs also the row all-gather",
            "seconds_per_stack": sec, "seconds_all": times,
            "carved_over_dense": {"single": sec["single_carved"] / sec["single_dense"],
                                  "sp": sec["sp_carved"] / sec["sp_dense"]},
            "live_tiles_per_stack": tiles, "sm_mhz_start_end": clocks,
            "sp_vs_single": {"dense": dist_rms(outs["single_dense"], outs["sp_dense"]),
                             "carved": dist_rms(outs["single_carved"], outs["sp_carved"])},
            "stats_per_timed_window_rank0": stats, "card": card()}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
