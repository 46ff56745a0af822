#!/usr/bin/env python
"""bench_attn_l2.py — how much of the carved-attention kernel's time is K/V traffic from HBM.

Times `jenga_b200.attention._launch` at a bench.py workload (default hy720p) on two masks:

  real    the operator's own selection mask;
  shared  within each head, every sparse row gets the mask of one fixed row of that head.  The rows
          keep about the same number of live tiles, but each head's K/V working set shrinks to the
          tiles of one row, which fits in L2 whatever order the CTAs run in.

The legs alternate for --rounds rounds, each leg --iters launches timed with CUDA events after a
warm-up.  The gap between the two is the time the kernel spends waiting for K/V tiles that L2 did not
hold.  Prints one JSON line: ms per launch, SM cycles per tile (kernel time x median SM clock x SMs /
tiles), the K/V tile bytes per second, and the card's name, power limit and median SM clock.

    python bench_attn_l2.py [--workload hy720p] [--rounds 3] [--iters 10]

On an H100 80GB HBM3 (700 W limit, median SM clock 1470-1485 MHz) at hy720p, three runs: real
90.4-91.5 ms, shared 84.2-85.0 ms per launch (2.84-2.88 k against 2.69-2.73 k SM cycles per tile).
The shared mask is 6.5-6.9 % faster there.  Power-capped at about 1 GHz the gap is larger, and the
ordered schedule of jenga_carved_attn_fwd_sched runs the real mask faster than the shared one (whose
rows are not ordered).
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent


def gpu_info(index: int) -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits",
                        "-i", str(index)], capture_output=True, text=True, timeout=10)
    name, power = (s.strip() for s in r.stdout.strip().split(",")) if r.returncode == 0 else ("unknown", "unknown")
    return {"name": name, "power_limit_w": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="hy720p")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    sys.path.insert(0, str(ROOT))
    import torch
    import bench
    from jenga_b200 import attention as A

    if not torch.cuda.is_available():
        raise SystemExit("bench_attn_l2.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    wl = bench.workload(args.workload, 0.7)
    inp = bench.build_inputs(wl, dev)
    _, bits = bench.run_operator(wl, inp, return_bits=True)
    torch.cuda.synchronize()
    S, nb_img, H = inp["S"], inp["nb_img"], inp["heads"]
    nb = (S + 127) // 128
    fixed = bits.shape[2] // 2
    shared = bits[:, :, fixed:fixed + 1].expand_as(bits).contiguous()

    def tiles(m):
        _, pop = bench.algorithmic_flops(wl, inp, m)
        return pop + H * wl["text_blocks"] * nb

    aq, ak = (x if x.dtype == torch.bfloat16 else x.bfloat16() for x in (inp["q"], inp["k"]))
    out = torch.empty_like(aq)
    seq = inp["cu"][1:2].contiguous() if inp["cu"] is not None else None

    def launch(m):
        A._launch(aq, ak, inp["v"], m, nb_img, wl["text_blocks"], 128 ** -0.5, wl["text_amp"],
                  nb_img, S, S, nb * 128, out, seq, torch.bfloat16)

    def timed(m):
        for _ in range(2):
            launch(m)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            launch(m)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.iters

    legs = {"real": bits, "shared": shared}
    ms = {k: [] for k in legs}
    with bench.ClockSampler(0) as clk:
        for _ in range(args.rounds):
            for k, m in legs.items():
                ms[k].append(timed(m))
    clocks = clk.summary()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    tile_bytes = 2 * 128 * 128 * 2   # one K and one V tile, bf16
    res = {"workload": wl["name"], "gpu": gpu_info(0), "sms": sms,
           "sm_mhz_median": clocks.get("sm_mhz"), "clock_reasons": clocks.get("reasons"), "legs": {}}
    for k, m in legs.items():
        n = tiles(m)
        med = statistics.median(ms[k])
        leg = {"ms_per_launch": ms[k], "ms_median": med, "tiles": n,
               "tile_bytes_per_s": n * tile_bytes / (med * 1e-3)}
        if clocks.get("sm_mhz"):
            leg["cycles_per_tile"] = med * 1e-3 * clocks["sm_mhz"] * 1e6 * sms / n
        res["legs"][k] = leg
    res["shared_vs_real"] = res["legs"]["shared"]["ms_median"] / res["legs"]["real"]["ms_median"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
