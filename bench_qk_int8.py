#!/usr/bin/env python
"""bench_qk_int8.py — the opt-in INT8 Q.K^T variant of the carved attention against the default path.

For each workload (default: hy720p, hy_turbo_s0, wan14b; all heads) the four modes default, qk_int8,
pv_fp8 and qk_int8+pv_fp8 run in alternation, `--rounds` times each:
  kernel_ms    the attention launch alone, CUDA events, with the mask bits and the quantised operands
               computed beforehand (median of `--iters` launches)
  operator_ms  the whole operator call (pooling, selection, the quantisation passes, the launch)
  cycles/tile  kernel time x the median SM clock sampled during the run x 132 SMs / live tiles
and, once per mode, the error of its output against the default path's (max and mean |diff| / RMS).
Prints one JSON line per workload, with the card name, power limit and SM clock read in the same run.

    python bench_qk_int8.py [--workloads hy720p,hy_turbo_s0,wan14b] [--rounds 3] [--iters 5]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import bench  # noqa: E402
from bench import algorithmic_flops, build_inputs, workload  # noqa: E402

MODES = {"default": (False, False), "qk_int8": (True, False), "pv_fp8": (False, True), "qk_int8+pv_fp8": (True, True)}
SMS = 132


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=10)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def events_ms(fn, iters):
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def run_workload(name, rounds, iters):
    from jenga_b200 import attention as A
    from refutil import pair_stats
    wl = workload(name, 0.7)
    dev = torch.device("cuda", 0)
    inp = build_inputs(wl, dev)
    S, H = inp["S"], inp["heads"]
    nb = (S + 127) // 128
    n_img = nb - wl["text_blocks"]
    kw = dict(cu_seqlens_q=inp["cu"], cu_seqlens_kv=inp["cu"], text_blocks=wl["text_blocks"], text_amp=wl["text_amp"],
              block_neighbor_list=inp["nbr"], p_remain_rates=wl["p_remain"], first_frame_blocks=wl["first_frame"])
    ref, bits = A.block_sparse_attention_variant(wl["variant"], inp["q"], inp["k"], inp["v"], inp["top_k"],
                                                 return_mask_bits=True, **kw)
    _, tiles = algorithmic_flops(wl, inp, bits)
    tiles += H * wl["text_blocks"] * nb                                   # the dense rows' tiles
    # operands of the attention launch, as the operator makes them
    q = inp["q"].bfloat16() if inp["q"].dtype == torch.float32 else inp["q"]
    k = inp["k"].bfloat16() if inp["k"].dtype == torch.float32 else inp["k"]
    v = inp["v"]
    qk8 = A.quantize_qk_int8(q, k)
    v8 = A.quantize_v_fp8(v)
    seq = inp["cu"][1:2].to(torch.int32) if inp["cu"] is not None else None
    out = torch.empty(q.shape, dtype=q.dtype, device=dev)

    def kernel(mode):
        i8, f8 = MODES[mode]
        return lambda: A._launch(q, k, v, bits, n_img, wl["text_blocks"], 128 ** -0.5, wl["text_amp"], n_img, S, S,
                                 nb * 128, out, seq, q.dtype, v_fp8=v8 if f8 else None, qk_int8=qk8 if i8 else None)

    def operator(mode):
        i8, f8 = MODES[mode]
        return lambda: A.block_sparse_attention_variant(wl["variant"], inp["q"], inp["k"], inp["v"], inp["top_k"],
                                                        qk_int8=i8, pv_fp8=f8, **kw)

    res = {m: {"kernel_ms": [], "operator_ms": []} for m in MODES}
    for m in MODES:                                                       # warm up every shape
        kernel(m)()
        operator(m)()
    torch.cuda.synchronize()
    with bench.ClockSampler(0) as clk:
        for _ in range(rounds):
            for m in MODES:
                res[m]["kernel_ms"].append(events_ms(kernel(m), iters))
                res[m]["operator_ms"].append(events_ms(operator(m), iters))
    clock = clk.summary()
    for m in MODES:
        o = operator(m)()
        torch.cuda.synchronize()
        e_max, e_mean = pair_stats(o, ref)
        k_med = statistics.median(res[m]["kernel_ms"])
        res[m].update(err_vs_default_max=e_max, err_vs_default_mean=e_mean,
                      cycles_per_tile=(k_med * 1e-3 * clock["sm_mhz"] * 1e6 * SMS / tiles) if clock["sm_mhz"] else None)
    return {"workload": name, "shape": wl["name"], "live_tiles": tiles, "mask_popcount": tiles - H * wl["text_blocks"] * nb,
            "clock": clock, "card": card(), "modes": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="hy720p,hy_turbo_s0,wan14b")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_qk_int8.py measures on a CUDA device; none found")
    for name in args.workloads.split(","):
        print(json.dumps(run_workload(name, args.rounds, args.iters)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
