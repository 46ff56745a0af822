#!/usr/bin/env python
"""Sequence-parallel Wan2.1-I2V block stack: the unmodified wan/modules/model.py I2V WanAttentionBlocks
(random init at Wan-I2V-14B, 4 blocks) on one GPU against the same stack sharded over the N ranks of
`torchrun --nproc-per-node N`.

  single  every rank runs the whole stack on its own GPU: the block forward install(wan_sp=True) hooks
          into wan/modules/model.py without `jenga_sp` (the wan_* dense kernels, the fused I2V
          cross-attention, the original self-attention through the flash_attn shim), L rows
  sp      every rank runs its raster rows [r*n, min((r+1)*n, L)), n = ceil(L/N), zero-padded to n, with
          `block.self_attn.jenga_sp` set, the route of jenga_b200/wan_sp.py's parallelize_wan_i2v: the
          self-attention runs the dense class over the Ulysses exchange (peer stores, or the NCCL
          all-to-all where symmetric memory is unavailable), the cross-attention the fused I2V kernel

Inputs of Wan-I2V-14B 720p: grid 21x45x80 (75 600 tokens), 257 CLIP + 512 text context rows in fp32,
bf16 autocast.  Reports seconds per stack (the slowest rank, CUDA events, best of --reps), the SM clock
at the start and end of each timed stack, and the distance of the gathered sp rows from the single-GPU
rows in units of their RMS.  The sp leg's timed region is the block stack plus the all-gather of the
rows that the sharded forward adds once per forward (here of the stack's output rows; the forward
gathers the head's 64 output channels instead).  Rank 0 prints one JSON line; nothing is written to
the tree.

    torchrun --nproc-per-node N bench_wan_i2v_sp.py [--blocks 4] [--reps 3]
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
    ap.add_argument("--blocks", type=int, default=4, help="blocks in the stack")
    ap.add_argument("--reps", type=int, default=3, help="timed stack forwards per leg")
    ap.add_argument("--grid", default="21,45,80", help="latent f,h,w (after patching)")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_wan_i2v_sp.py measures on GPUs; none is visible")
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl")
    P, r = dist.get_world_size(), dist.get_rank()
    from bench_i2v_blocks import card
    from jenga_b200 import blocks as jb
    from jenga_b200.hyi2v_sp import default_attention, shard
    from jenga_b200.wan_sp import _check_world, shard_rows
    from test_wan_i2v_sp_cpu import load_plain_wan
    mod = load_plain_wan(wan_sp=True)
    if mod is None:
        raise SystemExit("oracle/_ref/ and oracle/_ref_wan_model/ are not staged: run __graft_entry__.build() first")

    f, h, w = (int(v) for v in args.grid.split(","))
    dim, heads, ffn, n_img, n_txt = 5120, 40, 13824, 257, 512
    L = f * h * w
    _check_world(heads, P)
    n, _ = shard_rows(L, P, r)
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
    x_r = shard(x0, 1, P, r)

    def forward(x):
        for b_ in blks:
            x = b_(x, e0, seq_lens, grid, freqs, ctx, None)
        return x

    def sp_forward():
        out = forward(x_r)
        parts = [torch.empty_like(out) for _ in range(P)]
        dist.all_gather(parts, out.contiguous())                     # as the sharded forward does (of the head)
        return torch.cat(parts, 1)[:, :L]

    sp = default_attention(variant="wan")

    def set_sp(on):
        for b_ in blks:
            if on:
                b_.self_attn.jenga_sp = sp
            else:
                b_.self_attn.__dict__.pop("jenga_sp", None)

    legs = ("single", "sp")

    def timed(leg):
        set_sp(leg == "sp")
        e_0, e_1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dist.barrier()
        torch.cuda.synchronize()
        e_0.record()
        out = sp_forward() if leg == "sp" else forward(x0)
        e_1.record()
        torch.cuda.synchronize()
        s = torch.tensor([e_0.elapsed_time(e_1) * 1e-3], device=dev)
        dist.all_reduce(s, op=dist.ReduceOp.MAX)
        return s.item(), out

    times = {k: [] for k in legs}
    clocks = {k: [] for k in legs}
    outs = {}
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for k in legs:                                                  # warm-up: cuBLAS, buffers, caches
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
    dd = (b - a).abs()
    if r == 0:
        sec = {k: min(v) for k, v in times.items()}
        print(json.dumps({
            "bench": "wan_i2v_sp", "world": P, "grid": [f, h, w], "tokens": L, "rows_per_rank": n,
            "pad_rows": P * n - L, "dim": dim, "heads": heads, "blocks": args.blocks,
            "context_tokens": [n_img, n_txt], "reps": args.reps, "exchange": type(sp).__name__,
            "timed": "block stack; sp leg also the row all-gather",
            "seconds_per_stack": sec, "seconds_all": times, "sp_over_single": sec["sp"] / sec["single"],
            "sm_mhz_start_end": clocks,
            "sp_vs_single": {"max_over_rms": dd.max().item() / rms, "mean_over_rms": dd.mean().item() / rms},
            "stats_per_timed_window_rank0": stats, "card": card()}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
