"""Opt-in FP8 Linears (JENGA_LINEAR_FP8): per-shape GEMM timing and the HunyuanVideo block stack, off vs on.

Per image-row Linear of the HunyuanVideo 720p blocks (M = 115 200 rows in the double stream, 115 456
in the single stream), timed alternately, best of --windows windows of --iters calls each:
  bf16 checkpoints    torch's bf16 F.linear (cuBLAS) against jenga_quantize_rows_fp8 + jenga_linear_fp8
                      (per-channel weight scales), and the FP8 GEMM alone
  --use-fp8 weights   the reference's fp8_linear_forward (hyvideo/modules/fp8_optimization.py, restated:
                      weight.sum() != 0 with its host sync, bf16 dequantisation of the whole weight,
                      F.linear) against quantisation + FP8 GEMM with the per-tensor scale
These decide dense.FP8_ROUTED.  Then the 4 double + 8 single block stack (unmodified reference classes
through install(), random-init bf16 weights) with the switch off and on with EVERY image-row Linear
routed (what routing them would cost), alternately, the SM clock after each leg, and the difference of
the two outputs.  Prints one JSON line with the card name, power limit and SM clock read in the same run.

--model wan-14b / wan-1.3b: the Linears of one Wan2.1 WanAttentionBlock (wan/modules/model_mul.py), fp32
nn.Linear weights as the Wan pipelines keep them, M = 75 600 (14B, 21x45x80) or 32 760 (1.3B, 21x30x52)
rows.  Each site is timed as the chain the switch replaces, producer included:
  self_qkv   wan_ln_modulate + q, k, v module calls   | wan_ln_modulate_fp8 + three FP8 GEMMs
  self_o     o module call on the attention output    | quantize_rows_fp8 + FP8 GEMM      (also cross_o)
  cross_q    wan_residual_ln (norm3) + q module call  | wan_residual_ln_fp8 + FP8 GEMM
  ffn.0      wan_residual_ln (norm2) + module call    | wan_residual_ln_fp8 + FP8 GEMM
  ffn.2      gelu_tanh + module call                  | gelu_tanh_fp8 + FP8 GEMM
The module calls run under bf16 autocast, which re-casts the fp32 weight on every call.  Also per site:
the module calls alone, the FP8 GEMMs alone, and torch._scaled_mm with row-wise scales on the same e4m3
operands (a yardstick of what the card reaches, never on a hot path).  A (K, N) shape is "faster" when the
sum of its sites' FP8 chains beats the sum of their bf16 chains; those are the ("fp32", K, N) entries of
dense.FP8_ROUTED.  Then the block stack of bench_wan_blocks.py (4 Wan-14B or 8 Wan-1.3B T2V blocks) with
the switch off and on with every Wan shape routed, alternately: times, peak memory, the output distance
and the SM clock around each leg.
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

SHAPES = {   # name: (M, K, N)
    "img_attn_qkv": (115200, 3072, 9216), "img_attn_proj": (115200, 3072, 3072),
    "img_mlp.fc1": (115200, 3072, 12288), "img_mlp.fc2": (115200, 12288, 3072),
    "linear1": (115456, 3072, 21504), "linear2": (115456, 15360, 3072),
}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def sm_clock():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        return int(r.stdout.split()[0])
    except Exception:  # noqa: BLE001
        return None


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / iters


def gemm_leg(windows, iters):
    from jenga_b200 import dense as DN
    out = {}
    g = torch.Generator(device="cuda").manual_seed(7)
    for name, (M, K, N) in SHAPES.items():
        x = torch.randn(M, K, generator=g, device="cuda").bfloat16()
        w = (torch.randn(N, K, generator=g, device="cuda") * 0.02).bfloat16()
        b = (torch.randn(N, generator=g, device="cuda") * 0.1).bfloat16()
        w8, ws = DN.quantize_rows_fp8(w)
        bf16 = lambda: torch.nn.functional.linear(x, w, b)                          # noqa: E731
        fp8 = lambda: DN.linear_fp8(*DN.quantize_rows_fp8(x), w8, ws, b)            # noqa: E731
        gemm = lambda x8=DN.quantize_rows_fp8(x): DN.linear_fp8(*x8, w8, ws, b)     # noqa: E731
        # a --use-fp8 layer: e4m3 weight, per-tensor bf16 fp8_scale on the host (convert_fp8_linear)
        s_ref = (w.float().abs().max() / 448).to(torch.bfloat16)
        w_ref = (w.float() / s_ref.float()).to(torch.float8_e4m3fn)
        s_cpu, s_dev = s_ref.cpu(), s_ref.float().reshape(1)

        def ref_fp8():
            # weight.sum() != 0 (summed as bytes here: e4m3 has no CUDA sum), a device-to-host sync
            assert bool(w_ref.view(torch.uint8).sum() != 0)
            return torch.nn.functional.linear(x, w_ref.to(torch.bfloat16) * s_cpu.to("cuda"), b)

        ours_ref = lambda: DN.linear_fp8(*DN.quantize_rows_fp8(x), w_ref, s_dev, b)   # noqa: E731
        legs = {"bf16": bf16, "fp8_quantise_gemm": fp8, "fp8_gemm_only": gemm,
                "use_fp8_reference": ref_fp8, "use_fp8_ours": ours_ref}
        for f in legs.values():
            f()
        t = {k: [] for k in legs}
        for _ in range(windows):
            for k, f in legs.items():
                t[k].append(timed(f, iters))
        ref = bf16().float()
        err = (fp8().float() - ref).abs() / ref.pow(2).mean().sqrt()
        flop = 2.0 * M * K * N
        best = {k: min(v) for k, v in t.items()}
        out[name] = {"M": M, "K": K, "N": N, "seconds_best": best,
                     "tflops": {k: flop / v / 1e12 for k, v in best.items()},
                     "speedup_quantise_gemm": best["bf16"] / best["fp8_quantise_gemm"],
                     "speedup_use_fp8": best["use_fp8_reference"] / best["use_fp8_ours"],
                     "fp8_vs_bf16_mean_max_over_rms": [err.mean().item(), err.max().item()]}
        del x, w, w8, w_ref
        torch.cuda.empty_cache()
    return out


def stack_leg(n_double, n_single, rounds):
    import bench
    from oracle import ref_loader
    from jenga_b200 import blocks as jb, dense as DN, gilbert
    if not ref_loader.available():
        return {"unavailable": "oracle/_ref/ not staged"}
    our_hy, _ = ref_loader.load_blocks(product=True)
    wl = bench.workload("hy720p", 0.7)
    inp = bench.build_inputs(wl, torch.device("cuda"))
    hidden, heads = 3072, 24
    t, h, w = wl["grid"]
    L, T = inp["n_img"], wl["text_tokens"]
    g = torch.Generator(device="cuda").manual_seed(2024)
    dbl = [our_hy.MMDoubleStreamBlock(hidden, heads, mlp_width_ratio=4.0, dtype=torch.bfloat16, device="cuda")
           for _ in range(n_double)]
    sgl = [our_hy.MMSingleStreamBlock(hidden, heads, mlp_width_ratio=4.0, dtype=torch.bfloat16, device="cuda")
           for _ in range(n_single)]
    with torch.no_grad():
        for m in dbl + sgl:
            for n_, p_ in m.named_parameters():
                if p_.dim() >= 2:
                    p_.copy_(torch.randn(p_.shape, generator=g, device="cuda").mul_(0.02))
                elif "norm" in n_:
                    p_.fill_(1.0)
                else:
                    p_.zero_()
    l2h, h2l = (m_.cuda() for m_ in gilbert.mapping_tensors(t, h, w))
    curve_sel = [[l2h, h2l, inp["nbr"]]]
    img0 = torch.randn(1, L, hidden, generator=g, device="cuda").bfloat16()
    txt0 = torch.randn(1, T, hidden, generator=g, device="cuda").bfloat16()
    vec = torch.randn(1, hidden, generator=g, device="cuda").bfloat16()
    ang = torch.rand(L, 64, generator=g, device="cuda") * 6.2831853
    cos = torch.cos(ang).repeat_interleave(2, dim=1).contiguous()[h2l]
    sin = torch.sin(ang).repeat_interleave(2, dim=1).contiguous()[h2l]
    cu = inp["cu"]

    every = frozenset(("bf16", k_, n_) for _, k_, n_ in SHAPES.values())

    def forward(on):
        DN.LINEAR_FP8, DN.FP8_ROUTED = on, every if on else frozenset()
        img, txt = img0[:, h2l], txt0
        for blk in dbl:
            img, txt = blk(img, txt, vec, cu, cu, L + T, L + T, (cos, sin), wl["drop"], wl["text_amp"], curve_sel,
                           wl["p_remain"])
        x = torch.cat((img, txt), 1)
        for blk in sgl:
            x = blk(x, vec, T, cu, cu, L + T, L + T, (cos, sin), wl["drop"], wl["text_amp"], curve_sel, wl["p_remain"])
        return x[:, :L][:, l2h]

    res = {"off": [], "on": []}
    clocks = {"off": [], "on": []}
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            out_off, out_on = forward(False), forward(True)       # warm-up, weight quantisation
            s0 = dict(jb.STATS)
            forward(True)
            per_on = {k: jb.STATS[k] - s0[k] for k in s0 if jb.STATS[k] != s0[k]}
            for r in range(rounds):
                for leg in (("off", "on") if r % 2 == 0 else ("on", "off")):
                    res[leg].append(timed(lambda: forward(leg == "on"), 1))
                    clocks[leg].append(sm_clock())
    finally:
        DN.LINEAR_FP8, DN.FP8_ROUTED = False, frozenset()
    rms = out_off.float().pow(2).mean().sqrt()
    d = (out_on.float() - out_off.float()).abs() / rms
    return {"blocks": {"double": n_double, "single": n_single}, "seconds": res, "sm_clock_after_leg_mhz": clocks,
            "best": {k: min(v) for k, v in res.items()}, "speedup": min(res["off"]) / min(res["on"]),
            "on_vs_off_mean_max_over_rms": [d.mean().item(), d.max().item()], "stats_per_forward_on": per_on}


# Wan2.1 block shapes: grid, dim, heads, ffn, sa_drop_rate, p_remain_rates, blocks (bench_wan_blocks.MODELS)
WAN = {"wan-14b": "14b", "wan-1.3b": "1.3b"}


def wan_sites(C, F):
    """site: (K, N, producer, GEMMs per call) of one WanAttentionBlock's routable Linears"""
    return {"self_qkv": (C, C, "ln_modulate", 3), "self_o": (C, C, "quantize", 1),
            "cross_q": (C, C, "residual_norm3", 1), "cross_o": (C, C, "quantize", 1),
            "ffn.0": (C, F, "residual_norm2", 1), "ffn.2": (F, C, "gelu", 1)}


def wan_routed(model):
    """every ("fp32", K, N) shape of the Wan model's routable Linears"""
    from bench_wan_blocks import MODELS
    _, C, _, F, *_ = MODELS[WAN[model]]
    return frozenset(("fp32", k_, n_) for k_, n_, _, _ in wan_sites(C, F).values())


def scaled_mm(x8, a_scale, w8, w_scale, b):
    # row-wise _scaled_mm takes a bf16 bias only
    return torch._scaled_mm(x8, w8.t(), scale_a=a_scale[:, None], scale_b=w_scale[None, :],
                            bias=b.to(torch.bfloat16), out_dtype=torch.bfloat16)


def wan_gemm_leg(model, windows, iters):
    from bench_wan_blocks import MODELS
    from jenga_b200 import dense as DN
    (f, h, w_), C, _, F, *_ = MODELS[WAN[model]]
    M = f * h * w_
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(11)
    e = 0.1 * torch.randn(6, C, generator=g, device=dev)
    xr = torch.randn(1, M, C, generator=g, device=dev)                    # fp32 residual stream
    y = torch.randn(1, M, C, generator=g, device=dev).bfloat16()          # attention / cross output
    nw, nb = torch.ones(C, device=dev), torch.zeros(C, device=dev)        # norm3 (affine)
    out, sites = {}, {}
    for site, (K, N, prod, n) in wan_sites(C, F).items():
        lin = torch.nn.Linear(K, N, device=dev)                           # fp32, as the Wan pipelines keep it
        lin.requires_grad_(False)
        with torch.no_grad():
            lin.weight.normal_(0.0, 0.02, generator=g)
            lin.bias.normal_(0.0, 0.02, generator=g)
        w8, ws, b = DN.fp8_weight(lin)
        a_in = torch.randn(1, M, K, generator=g, device=dev).bfloat16() if prod == "gelu" else None
        if prod == "ln_modulate":
            p16 = lambda: DN.wan_ln_modulate(xr, e[0], e[1])                                    # noqa: E731
            p8 = lambda: DN.wan_ln_modulate_fp8(xr, e[0], e[1])                                 # noqa: E731
        elif prod == "quantize":
            p16 = lambda: y                                                                     # noqa: E731
            p8 = lambda: DN.quantize_rows_fp8(y)                                                # noqa: E731
        elif prod == "residual_norm3":
            p16 = lambda: DN.wan_residual_ln(xr, y, e[2], weight=nw, bias=nb)[1]                # noqa: E731
            p8 = lambda: DN.wan_residual_ln_fp8(xr, y, e[2], weight=nw, bias=nb)[1]             # noqa: E731
        elif prod == "residual_norm2":
            p16 = lambda: DN.wan_residual_ln(xr, y, None, shift=e[3], scale=e[4])[1]            # noqa: E731
            p8 = lambda: DN.wan_residual_ln_fp8(xr, y, None, shift=e[3], scale=e[4])[1]         # noqa: E731
        else:
            p16 = lambda: DN.gelu_tanh_into(a_in, torch.empty_like(a_in))                       # noqa: E731
            p8 = lambda: DN.gelu_tanh_fp8(a_in)                                                 # noqa: E731
        h16, h8 = p16(), p8()

        def bf16_chain():
            hh = p16()
            return [lin(hh) for _ in range(n)]

        def fp8_chain():
            hh = p8()
            return [DN.linear_fp8(*hh, w8, ws, b) for _ in range(n)]

        legs = {"bf16_chain": bf16_chain, "fp8_chain": fp8_chain,
                "bf16_module_only": lambda: [lin(h16) for _ in range(n)],
                "fp8_gemm_only": lambda: [DN.linear_fp8(*h8, w8, ws, b) for _ in range(n)]}
        try:
            scaled_mm(*h8, w8, ws, b)
            legs["scaled_mm_yardstick"] = lambda: [scaled_mm(*h8, w8, ws, b) for _ in range(n)]
            mm_err = None
        except Exception as ex:  # noqa: BLE001
            mm_err = f"{type(ex).__name__}: {ex}"[:200]
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            for fn in legs.values():
                fn()
            t = {k: [] for k in legs}
            for _ in range(windows):
                for k, fn in legs.items():
                    t[k].append(timed(fn, iters))
            ref = lin(h16).float()
            got = DN.linear_fp8(*h8, w8, ws, b).float()
        err = (got - ref).abs() / ref.pow(2).mean().sqrt()
        flop = 2.0 * M * K * N * n
        best = {k: min(v) for k, v in t.items()}
        sites[site] = {"M": M, "K": K, "N": N, "gemms": n, "seconds_best": best,
                       "tflops": {k: flop / v / 1e12 for k, v in best.items() if "only" in k or "scaled" in k},
                       "speedup_chain": best["bf16_chain"] / best["fp8_chain"],
                       "scaled_mm_error": mm_err,
                       "fp8_vs_bf16_mean_max_over_rms": [err.mean().item(), err.max().item()]}
        del lin, w8, a_in, h16, h8, ref, got
        torch.cuda.empty_cache()
    shapes = {}
    for site, r in sites.items():
        s_ = shapes.setdefault(f"{r['K']}x{r['N']}", {"sites": [], "bf16_chain": 0.0, "fp8_chain": 0.0})
        s_["sites"].append(site)
        s_["bf16_chain"] += r["seconds_best"]["bf16_chain"]
        s_["fp8_chain"] += r["seconds_best"]["fp8_chain"]
    for s_ in shapes.values():
        s_["faster"] = s_["fp8_chain"] < s_["bf16_chain"]
    out["sites"], out["shapes"] = sites, shapes
    return out


def wan_stack_leg(model, rounds):
    from oracle import ref_loader
    from bench_wan_blocks import MODELS
    from jenga_b200 import blocks as jb, dense as DN, gilbert
    if not ref_loader.available():
        return {"unavailable": "oracle/_ref/ not staged"}
    our = ref_loader.load_blocks(product=True)[1]
    (f, h, w_), dim, heads, ffn, drop, p_remain, n_blocks = MODELS[WAN[model]]
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(2024)
    with torch.device(dev):
        blks = [our.WanAttentionBlock("t2v_cross_attn", dim, ffn, heads, (-1, -1), True, True, 1e-6)
                for _ in range(n_blocks)]
    with torch.no_grad():
        for m in blks:
            m.requires_grad_(False)
            for n_, p_ in m.named_parameters():
                if "norm" in n_ and n_.endswith("weight"):
                    p_.fill_(1.0)
                else:
                    p_.copy_(torch.randn(p_.shape, generator=g, device=dev).mul_(0.02))
    L = f * h * w_
    _, h2l = gilbert.mapping_tensors(f, h, w_, sliced=True)
    nbr = gilbert.block_neighbor_mapping(f, h, w_, sliced=True)
    d = dim // heads
    freqs = torch.cat([our.rope_params(1024, d - 4 * (d // 6)), our.rope_params(1024, 2 * (d // 6)),
                       our.rope_params(1024, 2 * (d // 6))], dim=1).to(dev)
    seq_lens = torch.tensor([L], dtype=torch.long)
    grid = torch.tensor([[f, h, w_]], dtype=torch.long)
    x0 = torch.randn(1, L, dim, generator=g, device=dev).bfloat16()
    e0 = 0.1 * torch.randn(1, 6, dim, generator=g, device=dev)
    ctx = torch.randn(1, 512, dim, generator=g, device=dev).bfloat16()
    kw = dict(sa_drop_rate=drop, freq_remap=h2l.to(dev), block_neighbor_list=nbr, p_remain_rates=p_remain)
    every = wan_routed(model)
    saved = DN.LINEAR_FP8, DN.FP8_ROUTED
    jb.remove_gather_hook()

    def forward(on):
        DN.LINEAR_FP8, DN.FP8_ROUTED = on, every if on else frozenset()
        x = x0
        for blk in blks:
            x = blk(x, e0, seq_lens, grid, freqs, ctx, None, **kw)
        return x

    res, clocks, peak = {"off": [], "on": []}, {"off": [], "on": []}, {}
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            for leg in ("off", "on"):                 # warm-up; the first "on" quantises and caches the weights
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                out_ = forward(leg == "on")
                torch.cuda.synchronize()
                peak[leg] = {"peak_gb": torch.cuda.max_memory_allocated() / 1e9,
                             "above_start_gb": (torch.cuda.max_memory_allocated() - base) / 1e9}
                if leg == "off":
                    out_off = out_
                else:
                    out_on = out_
            peak["e4m3_weight_cache_gb"] = sum(
                m.__dict__["_jenga_fp8"][1].numel() for b_ in blks for m in b_.modules()
                if "_jenga_fp8" in m.__dict__) / 1e9
            s0 = dict(jb.STATS)
            forward(True)
            per_on = {k: jb.STATS[k] - s0[k] for k in s0 if jb.STATS[k] != s0[k]}
            for r in range(rounds):
                for leg in (("off", "on") if r % 2 == 0 else ("on", "off")):
                    c0 = sm_clock()
                    res[leg].append(timed(lambda: forward(leg == "on"), 1))
                    clocks[leg].append([c0, sm_clock()])
    finally:
        DN.LINEAR_FP8, DN.FP8_ROUTED = saved
    rms = out_off.float().pow(2).mean().sqrt()
    dd = (out_on.float() - out_off.float()).abs() / rms
    return {"blocks": n_blocks, "tokens": L, "routed": sorted(every), "seconds": res,
            "sm_clock_before_after_leg_mhz": clocks, "memory": peak,
            "best": {k: min(v) for k, v in res.items()}, "speedup": min(res["off"]) / min(res["on"]),
            "on_vs_off_mean_max_over_rms": [dd.mean().item(), dd.max().item()], "stats_per_forward_on": per_on}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--model", choices=["hy", *WAN], default="hy")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--blocks", default="4,8")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--skip-stack", action="store_true")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_linear_fp8.py measures on a GPU; none is visible")
    line = {"card_start": card()}
    if a.model == "hy":
        line["gemm"] = gemm_leg(a.windows, a.iters)
        if not a.skip_stack:
            nd, ns = (int(v) for v in a.blocks.split(","))
            line["stack"] = stack_leg(nd, ns, a.rounds)
    else:
        line["model"] = a.model
        line["gemm"] = wan_gemm_leg(a.model, a.windows, a.iters)
        if not a.skip_stack:
            line["stack"] = wan_stack_leg(a.model, a.rounds)
    line["card_end"] = card()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
