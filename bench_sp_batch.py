#!/usr/bin/env python
"""Several videos per DiT call on the sequence-parallel HunyuanVideo and HunyuanVideo-I2V paths: the
fused Ulysses exchange against the NCCL form, at N = 1, 2 and 4 samples per call.  Run under torchrun:

    torchrun --nproc-per-node P bench_sp_batch.py [--models hy,i2v] [--videos 1,2,4] [--reps 3]

The stacks and calls of bench_hy_batch.py (4 double + 8 single unmodified reference blocks at the
HunyuanVideo width, random init, the 720p grid 32x45x80), sharded over the P ranks as the multi-GPU
scripts shard them: rank r holds the contiguous 1/P slice of the Hilbert-ordered image rows, of the RoPE
tables and of the first-frame mask, and every text row.  The blocks route their attention through
`hybrid_seq_parallel_attn` (HunyuanVideo, jenga_hyvideo_multigpu.py) or `jenga_sp` (HunyuanVideo-I2V,
the sharded forward of hyi2v_sp.py).  Two legs on the same weights and inputs:

  fused  UlyssesFusedAttention: peer stores over NVLink (symmetric memory), the exchange fused into the
         kernels
  nccl   UlyssesCarvedAttention: all-to-all and all-gather collectives around the operator

After one untimed call of each leg, the legs alternate for --reps rounds; the best round counts.  Per leg:
seconds per stack (the slowest rank), seconds per video, torch.cuda.max_memory_allocated of one stack
forward (the largest over ranks), the bytes of the leg's symmetric buffers for N (allocated outside the
caching allocator, so not in that peak) and their sum.  The symmetric buffers of every N a run has used
stay allocated for the rest of the run.  The card's name, power limit and SM clock are read before and
after.  Rank 0 prints one JSON line; nothing is written to the tree.
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

from bench_hy_batch import HEADS, HIDDEN, MODELS, load  # noqa: E402


def _symm_bytes(sp, batch):
    """bytes of the symmetric buffers a UlyssesFusedAttention holds for `batch` samples per call (0 for the
    NCCL form); the buffers of other batch sizes it has run stay allocated too"""
    total = 0
    for key, (qkv, _, _, outs) in getattr(sp, "_bufs", {}).items():
        if key[-1] == batch:
            total += qkv.numel() * qkv.element_size() + sum(o.numel() * o.element_size() for o, _, _ in outs)
    return total


def bench_model(model, n_double, n_single, grid, videos, reps, dev, P, r):
    from jenga_b200 import blocks as jb
    from jenga_b200 import gilbert
    from jenga_b200.ulysses import UlyssesCarvedAttention, UlyssesFusedAttention
    T, valid, drop, p_remain, txt_amp, steps = MODELS[model]
    i2v = model == "i2v"
    variant = "hyvideo_i2v" if i2v else "hyvideo"
    mod = load(model)
    g = torch.Generator(device=dev).manual_seed(2024)        # the same draws on every rank

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
    L = t * h * w
    if L % P:
        raise SystemExit(f"{L} image tokens do not split over {P} ranks")
    n = L // P
    S = n + T                                                          # the rows a rank holds
    sl = slice(r * n, (r + 1) * n)
    l2h, h2l = gilbert.mapping_tensors(t, h, w)
    l2h, h2l = l2h.to(dev), h2l.to(dev)
    curve_sel = [[l2h, h2l, gilbert.block_neighbor_mapping(t, h, w).to(dev)]]
    ang = torch.rand(L, 64, generator=g, device=dev) * 6.2831853
    cos = torch.cos(ang).repeat_interleave(2, dim=1).contiguous()[h2l][sl].contiguous()
    sin = torch.sin(ang).repeat_interleave(2, dim=1).contiguous()[h2l][sl].contiguous()
    ff0 = torch.zeros(L, dtype=torch.bool, device=dev)
    ff0[:h * w] = True
    ff = ff0[h2l][sl].contiguous()                                     # jenga_hyi2v.py:124-126, this rank's slice

    def inputs(N):
        """N samples, each from its own draws, image rows in Hilbert order; this rank's slice"""
        img = torch.cat([torch.randn(1, L, HIDDEN, generator=g, device=dev).bfloat16()[:, h2l][:, sl]
                         for _ in range(N)]).contiguous()
        txt = torch.cat([torch.randn(1, T, HIDDEN, generator=g, device=dev).bfloat16() for _ in range(N)])
        vec = torch.randn(N, HIDDEN, generator=g, device=dev).bfloat16()
        tr_vec = torch.randn(N, HIDDEN, generator=g, device=dev).bfloat16()
        text_mask = torch.zeros(N, T, dtype=torch.int64, device=dev)
        text_mask[:, :valid] = 1
        return img, txt, vec, tr_vec, mod.get_cu_seqlens(text_mask, n)

    def forward(img, txt, vec, tr_vec, cu):
        """the block loops of jenga_hyvideo_multigpu.py / hyi2v_sp.py on this rank's rows"""
        if i2v:
            full = torch.zeros(S).bool()                               # the single blocks' CPU mask
            full[:n] = ff.cpu()
        for blk in dbl:
            if i2v:
                img, txt = blk(img, txt, vec, cu, cu, S, S, (cos, sin), drop, ff, "token_replace", tr_vec, h * w,
                               txt_amp, curve_sel, p_remain)
            else:
                img, txt = blk(img, txt, vec, cu, cu, S, S, (cos, sin), drop, txt_amp, curve_sel, p_remain)
        x = torch.cat((img, txt), 1)
        for blk in sgl:
            if i2v:
                x = blk(x, vec, T, cu, cu, S, S, (cos, sin), drop, full, "token_replace", tr_vec, h * w, txt_amp,
                        curve_sel, p_remain)
            else:
                x = blk(x, vec, T, cu, cu, S, S, (cos, sin), drop, txt_amp, curve_sel, p_remain)
        return x

    legs = {"fused": UlyssesFusedAttention(variant=variant), "nccl": UlyssesCarvedAttention(variant=variant)}

    def use(leg):
        for blk in dbl + sgl:
            setattr(blk, "jenga_sp" if i2v else "hybrid_seq_parallel_attn", legs[leg])

    def timed(leg, inp):
        """(seconds of the slowest rank, largest peak bytes over ranks) of one stack forward; None when
        some rank ran out of memory"""
        use(leg)
        torch.cuda.synchronize()
        dist.barrier()
        torch.cuda.reset_peak_memory_stats(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        oom = 0
        try:
            e0.record()
            out = forward(*inp)
            e1.record()
            torch.cuda.synchronize()
            del out
        except torch.cuda.OutOfMemoryError:
            oom = 1
            torch.cuda.empty_cache()
        v = torch.tensor([oom, 0.0 if oom else e0.elapsed_time(e1) * 1e-3,
                          float(torch.cuda.max_memory_allocated(dev))], dtype=torch.float64, device=dev)
        dist.all_reduce(v, op=dist.ReduceOp.MAX)
        return (None, None) if v[0].item() else (v[1].item(), int(v[2].item()))

    nblk = n_double + n_single
    res = {"img_tokens": L, "img_tokens_per_rank": n, "txt_tokens": T, "txt_valid": valid, "sa_drop_rate": drop,
           "p_remain_rates": p_remain, "text_amp": txt_amp, "blocks": {"double": n_double, "single": n_single},
           "computed_steps": steps, "by_videos": {}}
    jb.remove_gather_hook()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for N in videos:
            inp = inputs(N)
            before = dict(jb.STATS)
            for leg in legs:
                timed(leg, inp)                                        # untimed: buffers, rendezvous, autotuning
            stats = {k: jb.STATS[k] - before[k] for k in jb.STATS if jb.STATS[k] != before[k]}
            sec = {k: [] for k in legs}
            peak = {k: [] for k in legs}
            for _ in range(reps):
                for leg in legs:
                    s_, p_ = timed(leg, inp)
                    if s_ is not None:
                        sec[leg].append(s_)
                        peak[leg].append(p_)
            row = {"stats_first_call_both_legs": stats}
            for leg, sp in legs.items():
                best = min(sec[leg]) if sec[leg] else None
                symm = _symm_bytes(sp, N)
                row[leg] = {"seconds_per_stack": best, "seconds_all": sec[leg],
                            "stack_seconds_per_video": best / N if best else None,
                            "dit_loop_seconds_per_video": best / N * 60 / nblk * steps if best else None,
                            "max_memory_allocated_bytes": max(peak[leg]) if peak[leg] else "out of memory",
                            "symmetric_buffer_bytes": symm,
                            "peak_with_symmetric_bytes": max(peak[leg]) + symm if peak[leg] else None}
            f, c = row["fused"]["seconds_per_stack"], row["nccl"]["seconds_per_stack"]
            row["nccl_over_fused"] = c / f if f and c else None
            res["by_videos"][str(N)] = row
            del inp
            torch.cuda.empty_cache()
    for blk in dbl + sgl:
        for a in ("jenga_sp", "hybrid_seq_parallel_attn"):
            blk.__dict__.pop(a, None)
    del dbl, sgl, legs
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
    if "RANK" not in os.environ:
        raise SystemExit("bench_sp_batch.py runs under torchrun (--nproc-per-node P)")
    if not torch.cuda.is_available():
        raise SystemExit("bench_sp_batch.py measures on GPUs; none is visible")
    from oracle import ref_loader
    if not ref_loader.available():
        raise SystemExit("oracle/_ref/ is not staged: run __graft_entry__.build() first")
    from bench_i2v_blocks import card
    r = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(r)
    dev = torch.device("cuda", r)
    dist.init_process_group("nccl", device_id=dev)
    try:
        P, rank = dist.get_world_size(), dist.get_rank()
        info = card()
        out = {"bench": "sp_batch", "world": P, "grid": list(grid), "hidden": HIDDEN, "heads": HEADS,
               "reps": args.reps,
               "models": {m: bench_model(m, n_double, n_single, grid, videos, args.reps, dev, P, rank) for m in models}}
        out.update(card=info, card_after=card())
        if rank == 0:
            print(json.dumps(out))
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
