#!/usr/bin/env python
"""Sequence-parallel Wan2.1 T2V block stack: the unmodified wan/modules/model_mul.py WanAttentionBlocks
(random init at Wan-14B, 4 blocks as in bench_wan_blocks.py) on one GPU against the same stack sharded
over the N ranks of `torchrun --nproc-per-node N`.

  single  every rank runs the whole stack on its own GPU (the fused Wan block forward, L rows)
  sp      every rank runs its Hilbert rows [r*n, min((r+1)*n, L)), n = ceil(L/N), zero-padded to n, with
          `block.self_attn.jenga_sp` set, the route of jenga_b200/wan_sp.py: the self-attention runs over
          the Ulysses exchange (peer stores, or the NCCL all-to-all where symmetric memory is unavailable)

Same inputs as bench_wan_blocks.py --model 14b (grid 21x45x80, 512 context tokens, p_remain_rates 0.8,
bf16 autocast); --model 1.3b takes Wan2.1-1.3B's blocks (dim 1536, 12 heads, FFN 8960) at its 480p grid
21x30x52, where 8 ranks need the ragged head split (JENGA_ULYSSES_RAGGED=1: 2,2,2,2,1,1,1,1 heads), in two legs each: the carved leg at sa_drop_rate 0.7 and the dense leg at 0.2 (the
warm-up steps, model_mul.py:153).  Reports seconds per stack (the slowest rank, CUDA events), the SM
clock at the start and end of each leg, and the distance of the gathered sp rows from the single-GPU
rows in units of their RMS.  The sp leg's timed region is the block stack plus the all-gather of the
rows that the sharded forward adds once per forward (here of the stack's output rows; the forward
gathers the head's 64 output channels instead); the Hilbert gather, the slicing of the inputs and the
inverse scatter are outside both legs.  Rank 0 prints one JSON line; nothing is written to the tree.

    torchrun --nproc-per-node N bench_wan_sp.py [--model 14b|1.3b] [--blocks 4] [--reps 3]
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

MODELS = {"14b": (5120, 40, 13824, "21,45,80"), "1.3b": (1536, 12, 8960, "21,30,52")}   # dim, heads, FFN, grid


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--blocks", type=int, default=4, help="blocks in the stack")
    ap.add_argument("--reps", type=int, default=3, help="timed stack forwards per leg")
    ap.add_argument("--model", choices=sorted(MODELS), default="14b", help="Wan2.1 block shapes")
    ap.add_argument("--grid", default=None, help="latent f,h,w (after patching); default: the model's")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_wan_sp.py measures on GPUs; none is visible")
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl")
    P, r = dist.get_world_size(), dist.get_rank()
    from oracle import ref_loader
    if not ref_loader.available():
        raise SystemExit("oracle/_ref/ is not staged: run __graft_entry__.build() first")
    from bench_i2v_blocks import card
    from jenga_b200 import blocks as jb
    from jenga_b200 import gilbert
    from jenga_b200.hyi2v_sp import default_attention, shard
    from jenga_b200.wan_sp import _check_world, shard_rows

    dim, heads, ffn, grid_default = MODELS[args.model]
    f, h, w = (int(v) for v in (args.grid or grid_default).split(","))
    p_remain, Lc = 0.8, 512
    drops = {"carved": 0.7, "dense": 0.2}
    L = f * h * w
    _check_world(heads, P)
    n, real = shard_rows(L, P, r)
    dev = torch.device("cuda", local)
    mod = ref_loader.load_blocks(product=True)[1]
    jb.remove_gather_hook()
    g = torch.Generator(device=dev).manual_seed(2024)            # the same weights and inputs on every rank

    def init(m):
        with torch.no_grad():
            for n_, p_ in m.named_parameters():
                if p_.dim() >= 2 and "modulation" not in n_:
                    p_.copy_(torch.randn(p_.shape, generator=g, device=dev).mul_(0.02))
                elif "norm" in n_ and n_.endswith("weight"):
                    p_.fill_(1.0)
                else:
                    p_.copy_(torch.randn(p_.shape, generator=g, device=dev).mul_(0.02))

    with torch.device(dev):
        blks = [mod.WanAttentionBlock("t2v_cross_attn", dim, ffn, heads, (-1, -1), True, True, 1e-6)
                for _ in range(args.blocks)]
    for b_ in blks:
        init(b_)
    _, h2l = gilbert.mapping_tensors(f, h, w, sliced=True)
    nbr = gilbert.block_neighbor_mapping(f, h, w, sliced=True)
    d = dim // heads
    freqs = torch.cat([mod.rope_params(1024, d - 4 * (d // 6)), mod.rope_params(1024, 2 * (d // 6)),
                       mod.rope_params(1024, 2 * (d // 6))], dim=1).to(dev)
    seq_lens = torch.tensor([L], dtype=torch.long)
    grid = torch.tensor([[f, h, w]], dtype=torch.long)
    x0 = torch.randn(1, L, dim, generator=g, device=dev).bfloat16()     # Hilbert-ordered rows
    e0 = 0.1 * torch.randn(1, 6, dim, generator=g, device=dev)
    ctx = torch.randn(1, Lc, dim, generator=g, device=dev).bfloat16()
    remap = h2l.to(dev)
    x_r, remap_r = shard(x0, 1, P, r), shard(remap, 0, P, r)

    def forward(x, rm, drop):
        for b_ in blks:
            x = b_(x, e0, seq_lens, grid, freqs, ctx, None, sa_drop_rate=drop, freq_remap=rm,
                   block_neighbor_list=nbr, p_remain_rates=p_remain)
        return x

    def sp_forward(drop):
        out = forward(x_r, remap_r, drop)
        parts = [torch.empty_like(out) for _ in range(P)]
        dist.all_gather(parts, out.contiguous())                     # as wan_sp's forward does (of the head)
        return torch.cat(parts, 1)[:, :L]

    sp = default_attention(variant="wan")

    def set_sp(on):
        for b_ in blks:
            if on:
                b_.self_attn.jenga_sp = sp
            else:
                b_.self_attn.__dict__.pop("jenga_sp", None)

    legs = {f"{kind}_{route}": (kind, route) for kind in drops for route in ("single", "sp")}

    def timed(leg):
        kind, route = legs[leg]
        set_sp(route == "sp")
        e_0, e_1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dist.barrier()
        torch.cuda.synchronize()
        e_0.record()
        out = sp_forward(drops[kind]) if route == "sp" else forward(x0, remap, drops[kind])
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
    dist_rms = {}
    for kind in drops:
        a, b = outs[f"{kind}_single"].float(), outs[f"{kind}_sp"].float()
        rms = a.pow(2).mean().sqrt().item()
        dd = (b - a).abs()
        dist_rms[kind] = {"max_over_rms": dd.max().item() / rms, "mean_over_rms": dd.mean().item() / rms}
    if r == 0:
        sec = {k: min(v) for k, v in times.items()}
        print(json.dumps({
            "bench": "wan_sp", "world": P, "grid": [f, h, w], "tokens": L, "rows_per_rank": n,
            "pad_rows": P * n - L, "dim": dim, "heads": heads, "blocks": args.blocks, "context_tokens": Lc,
            "sa_drop_rate": drops, "p_remain_rates": p_remain, "reps": args.reps, "exchange": type(sp).__name__,
            "timed": "block stack; sp legs also the row all-gather",
            "seconds_per_stack": sec, "seconds_all": times,
            "speedup": {kind: sec[f"{kind}_single"] / sec[f"{kind}_sp"] for kind in drops},
            "sm_mhz_start_end": clocks, "sp_vs_single": dist_rms,
            "stats_per_timed_window_rank0": stats, "card": card()}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
