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


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--blocks", default="4,8")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--skip-stack", action="store_true")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_linear_fp8.py measures on a GPU; none is visible")
    line = {"card_start": card()}
    line["gemm"] = gemm_leg(a.windows, a.iters)
    if not a.skip_stack:
        nd, ns = (int(v) for v in a.blocks.split(","))
        line["stack"] = stack_leg(nd, ns, a.rounds)
    line["card_end"] = card()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
