#!/usr/bin/env python
"""Several videos per DiT call on one GPU: the fused Wan2.1 / Wan2.1-I2V block forwards against the
original forwards, at N = 1, 2 and 4.

Three stacks of unmodified wan/modules/model_mul.py WanAttentionBlocks (random init), the shapes of
bench_wan_blocks.py:

  14b      4 T2V blocks at Wan-14B (5120 channels, 40 heads), grid 21x45x80 (L = 75 600), 512 context
           rows, sa_drop_rate 0.7, p_remain_rates 0.8
  i2v-14b  4 I2V blocks at Wan-I2V-14B, 257 fp32 CLIP + 512 text context rows, dense (sa_drop_rate 0)
  1.3b     8 T2V blocks at Wan-1.3B (1536 channels, 12 heads), grid 21x30x52 (L = 32 760), sa_drop_rate
           0.75, p_remain_rates 0.9

Each sample of a batch has its own x, its own modulation e (its own timestep) and its own context.  Two
legs on the same weights and inputs:

  fused     the forwards install() patches in (jenga_b200/blocks.py)
  original  forward.__wrapped__ of WanAttentionBlock, WanSelfAttention and the cross-attention: what a
            batch above 1 ran before the fused block took it

After one untimed call of each leg (whose outputs give the distance between the legs, on sample 0), the legs
alternate for --reps rounds; the best round counts.  Per leg: seconds per stack, seconds per video, and
torch.cuda.max_memory_allocated of one stack forward.  Then the cost of launching the Wan chains once
per sample (split_cost).  The card's name, power limit and SM clock are read before and after.  One JSON
line on stdout; nothing is written to the tree.

With --sp, under `torchrun --nproc-per-node P`, the 14b and i2v-14b stacks run the route of the sharded
forwards (jenga_b200/wan_sp.py) instead: `block.self_attn.jenga_sp` is the default Ulysses exchange,
rank r takes the same Hilbert rows [r*n, min((r+1)*n, L)) of every sample (pad rows zeroed) with
freq_remap that slice, and the legs are

  sharded   the Hilbert gather of the rank's rows, the stack on them over the exchange, and the
            all-gather of its output rows
  one_gpu   the Hilbert gather of all L rows and the fused stack on them on one GPU, without jenga_sp

(the I2V stack is model_mul.py's I2V block, dense, under jenga_sp).  Rank 0 prints the JSON line.

    python bench_wan_batch.py [--models 14b,i2v-14b,1.3b] [--videos 1,2,4] [--reps 3]
    torchrun --nproc-per-node 1 bench_wan_batch.py --sp [--models 14b,i2v-14b]
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

from bench_wan_blocks import I2V_IMG_TOKENS, MODELS  # noqa: E402

LC = 512
PATCHED = ("WanAttentionBlock", "WanSelfAttention", "WanT2VCrossAttention")


def rms_distance(ref, out):
    a, b = ref.float(), out.float()
    rms = a.pow(2).mean().sqrt().item()
    d = (b - a).abs()
    return {"max_over_rms": d.max().item() / rms, "mean_over_rms": d.mean().item() / rms}


class _Original:
    """the unpatched forwards of PATCHED for the duration of one stack"""

    def __init__(self, mod):
        self.mod = mod

    def __enter__(self):
        self.saved = {c: getattr(self.mod, c).forward for c in PATCHED}
        for c, fn in self.saved.items():
            setattr(getattr(self.mod, c), "forward", fn.__wrapped__)

    def __exit__(self, *exc):
        for c, fn in self.saved.items():
            setattr(getattr(self.mod, c), "forward", fn)


def bench_model(model, videos, reps, dev, sp=None):
    """sp: None, or (Ulysses object, group, world size, rank) for the sharded legs"""
    import contextlib

    from oracle import ref_loader
    from jenga_b200 import blocks as jb
    from jenga_b200 import gilbert
    (f, h, w), dim, heads, ffn, drop, p_remain, n_blocks = MODELS[model]
    i2v = model.startswith("i2v")
    mod = ref_loader.load_blocks(product=True)[1]
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
    with torch.device(dev):
        blks = [mod.WanAttentionBlock(cross_type, dim, ffn, heads, (-1, -1), True, True, 1e-6) for _ in range(n_blocks)]
    for b_ in blks:
        init(b_)
    L = f * h * w
    _, h2l = gilbert.mapping_tensors(f, h, w, sliced=True)
    nbr = gilbert.block_neighbor_mapping(f, h, w, sliced=True)
    d = dim // heads
    freqs = torch.cat([mod.rope_params(1024, d - 4 * (d // 6)), mod.rope_params(1024, 2 * (d // 6)),
                       mod.rope_params(1024, 2 * (d // 6))], dim=1).to(dev)
    kw = dict(sa_drop_rate=drop, freq_remap=h2l.to(dev), block_neighbor_list=nbr, p_remain_rates=p_remain)

    def inputs(n):
        """n samples, each with its own x, e and context"""
        x = torch.randn(n, L, dim, generator=g, device=dev).bfloat16()
        e = 0.1 * torch.randn(n, 6, dim, generator=g, device=dev)
        ctx = torch.randn(n, LC, dim, generator=g, device=dev).bfloat16()
        if i2v:
            # img_emb's final LayerNorm runs in fp32 (model_mul.py:379-391); the concat promotes the text
            ctx = torch.concat([torch.randn(n, I2V_IMG_TOKENS, dim, generator=g, device=dev), ctx], dim=1)
        return x, e, torch.tensor([L] * n, dtype=torch.long), torch.tensor([[f, h, w]] * n, dtype=torch.long), ctx

    def forward(x, e, seq_lens, grid, ctx):
        for blk in blks:
            x = blk(x, e, seq_lens, grid, freqs, ctx, None, **kw)
        return x

    legs = {"fused": contextlib.nullcontext, "original": lambda: _Original(mod)}
    if sp is not None:
        from jenga_b200.sharding import gather_rows, shard, shard_rows
        attn, group, P, r = sp
        n, real = shard_rows(L, P, r, model="Wan2.1")
        rows = shard(h2l.to(dev), 0, P, r)
        one_gpu_kw = kw

        class _Sharded:
            def __enter__(self):
                for blk in blks:
                    blk.self_attn.jenga_sp = attn

            def __exit__(self, *exc):
                for blk in blks:
                    del blk.self_attn.jenga_sp

        h2l_dev = h2l.to(dev)

        def forward(x, e, seq_lens, grid, ctx):                                    # noqa: F811
            # x is raster-ordered here: one GPU gathers every row in the Hilbert order, rank r its rows
            if getattr(blks[0].self_attn, "jenga_sp", None) is None:
                out = x[:, h2l_dev]
                for blk in blks:
                    out = blk(out, e, seq_lens, grid, freqs, ctx, None, **one_gpu_kw)
                return out
            xr = x[:, rows]
            if real < n:
                xr[:, real:] = 0
            skw = dict(one_gpu_kw, freq_remap=rows)
            for blk in blks:
                xr = blk(xr, e, seq_lens, grid, freqs, ctx, None, **skw)
            return gather_rows(xr, L, P, group)

        legs = {"sharded": _Sharded, "one_gpu": contextlib.nullcontext}

    def timed(leg, inp):
        """(seconds, peak bytes, output) of one stack forward, or (None, None, None) out of memory"""
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        try:
            with legs[leg]():
                e0.record()
                out = forward(*inp)
                e1.record()
                torch.cuda.synchronize()
        except torch.cuda.OutOfMemoryError:
            torch.cuda.empty_cache()
            return None, None, None
        return e0.elapsed_time(e1) * 1e-3, torch.cuda.max_memory_allocated(dev), out

    res = {"grid": [f, h, w], "tokens": L, "dim": dim, "heads": heads, "ffn": ffn, "blocks": n_blocks,
           "context_rows": LC + (I2V_IMG_TOKENS if i2v else 0), "sa_drop_rate": drop, "p_remain_rates": p_remain,
           "by_videos": {}}
    jb.remove_gather_hook()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for n in videos:
            inp = inputs(n)
            base = torch.cuda.memory_allocated(dev)
            before = dict(jb.STATS)
            (a, b) = list(legs)
            _, _, out_f = timed(a, inp)
            fused_stats = {k: jb.STATS[k] - before[k] for k in jb.STATS if jb.STATS[k] != before[k]}
            # the distance is taken on sample 0, so that the second leg runs with one sample kept beside it
            out_f = out_f[:1].clone() if out_f is not None else None
            before = dict(jb.STATS)
            _, _, out_o = timed(b, inp)
            original_stats = {k: jb.STATS[k] - before[k] for k in jb.STATS if jb.STATS[k] != before[k]}
            dist = rms_distance(out_o[:1], out_f) if out_f is not None and out_o is not None else None
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
            row = {"weights_and_inputs_bytes": base, f"{a}_vs_{b}": dist, f"{a}_stats_per_stack": fused_stats,
                   f"{b}_stats_per_stack": original_stats}
            for leg in legs:
                best = min(sec[leg]) if sec[leg] else None
                row[leg] = {"seconds_per_stack": best, "seconds_all": sec[leg],
                            "stack_seconds_per_video": best / n if best else None,
                            "max_memory_allocated_bytes": max(peak[leg]) if peak[leg] else "out of memory"}
            (a, b) = list(legs)
            f_, o_ = row[a]["seconds_per_stack"], row[b]["seconds_per_stack"]
            row[f"{b}_over_{a}"] = o_ / f_ if f_ and o_ else None
            res["by_videos"][str(n)] = row
            del inp
            torch.cuda.empty_cache()
    del blks
    torch.cuda.empty_cache()
    return res


def split_cost(videos, tokens, dim, dev, iters=10, rounds=3):
    """What launching the Wan chains once per sample costs: the block's five chain calls
    (ln_modulate, residual_ln affine and modulate, gate_residual) on x [N, tokens, dim] fp32 with
    per-sample [N, 1, dim] vectors (N launches each) against the same rows as one sample with one vector
    (one launch each, the same bytes).  Milliseconds per block's chains, best of `rounds` alternating
    windows of `iters` calls."""
    from jenga_b200 import dense as DN
    g = torch.Generator(device=dev).manual_seed(7)
    res = {}
    w3 = torch.ones(dim, device=dev)
    for n in videos:
        if n == 1:
            continue
        x = torch.randn(n, tokens, dim, generator=g, device=dev)
        y = torch.randn(n, tokens, dim, generator=g, device=dev).bfloat16()
        e = torch.randn(n, 6, dim, generator=g, device=dev).chunk(6, dim=1)
        x1, y1, e1 = x.view(1, n * tokens, dim), y.view(1, n * tokens, dim), [v[:1] for v in e]

        def chains(x, y, e):
            DN.wan_ln_modulate(x, e[0], e[1])
            DN.wan_residual_ln(x, y, e[2], weight=w3, bias=w3)
            DN.wan_residual_ln(x, y, None, shift=e[3], scale=e[4])
            DN.wan_gate_residual(x, y, e[5])

        calls = {"per_sample": lambda: chains(x, y, e), "one_launch": lambda: chains(x1, y1, e1)}
        ms = {k: [] for k in calls}
        for fn in calls.values():
            fn()
        for _ in range(rounds):
            for k, fn in calls.items():
                e0, e_1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(iters):
                    fn()
                e_1.record()
                torch.cuda.synchronize()
                ms[k].append(e0.elapsed_time(e_1) / iters)
        res[str(n)] = {k: min(t) for k, t in ms.items()}
        del x, y, x1, y1
        torch.cuda.empty_cache()
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--models", default="14b,i2v-14b,1.3b", help="stacks to time, in order")
    ap.add_argument("--videos", default="1,2,4", help="samples per DiT call")
    ap.add_argument("--reps", type=int, default=3, help="timed rounds; the best counts")
    ap.add_argument("--sp", action="store_true", help="the sharded route under torchrun (14b, i2v-14b)")
    args = ap.parse_args(argv)
    if args.sp and args.models == ap.get_default("models"):
        args.models = "14b,i2v-14b"
    models = [m for m in args.models.split(",") if m]
    if any(m not in MODELS for m in models):
        raise SystemExit(f"--models takes {', '.join(MODELS)}")
    videos = [int(v) for v in args.videos.split(",")]
    if not torch.cuda.is_available():
        raise SystemExit("bench_wan_batch.py measures on a GPU; none is visible")
    from oracle import ref_loader
    if not ref_loader.available():
        raise SystemExit("oracle/_ref/ is not staged: run __graft_entry__.build() first")
    from bench_i2v_blocks import card
    sp, rank = None, 0
    if args.sp:
        import os

        import torch.distributed as dist

        from jenga_b200.sharding import default_attention
        rank = int(os.environ.get("RANK", "0"))
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
        sp = (default_attention(None, "wan"), None, dist.get_world_size(), rank)
    dev = torch.device("cuda", torch.cuda.current_device())
    info = card()
    out = {"bench": "wan_batch_sp" if sp else "wan_batch", "reps": args.reps, "models": {}}
    if sp:
        out.update(world=sp[2], exchange=type(sp[0]).__name__)
    for m in models:
        out["models"][m] = bench_model(m, videos, args.reps, dev, sp)
    if sp is None:
        (f, h, w), dim = MODELS["14b"][0], MODELS["14b"][1]
        with torch.no_grad():
            out["per_sample_launch_cost_ms"] = {"model": "14b", "by_videos": split_cost(videos, f * h * w, dim, dev)}
    out.update(card=info, card_after=card())
    if rank == 0:
        print(json.dumps(out))
    if sp:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
