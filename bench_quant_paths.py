#!/usr/bin/env python
"""bench_quant_paths.py — the opt-in INT8 Q.K^T (JENGA_QK_INT8) and FP8 P.V (JENGA_PV_FP8) switches on the
FlashAttention shim path, where Wan's dense self-attention lands, against the default kernel.

Cases:
  wan_i2v_dense   flash_attn_varlen_func as Wan2.1-I2V-14B's WanSelfAttention dense branch calls it
                  (sa_drop_rate 0): one segment of L = 75 600 tokens (21x45x80), 40 heads, bf16
  wan_1.3b_dense  the same at Wan-1.3B: L = 32 760 (21x30x52), 12 heads
For each, the modes default, int8 and int8+fp8 run in alternation; each window times `--iters` calls
with CUDA events and the best of `--windows` windows is reported as ms per call, with TFLOP/s from
4 L^2 D H operations, and the output's mean / max |difference| from the default mode over its RMS.
  wan_i2v_stack   `bench_wan_blocks.py --model i2v-14b` (4 fused I2V blocks) run once without and once
                  with JENGA_QK_INT8=1, in subprocesses: seconds per stack of the fused leg.
The card's name, power limit and SM clock are read (nvidia-smi queries only) at the start and the end.
One JSON line on stdout; nothing is written to the tree.

    python bench_quant_paths.py [--iters 5] [--windows 3] [--no-stack]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

from bench_i2v_blocks import card  # noqa: E402

CASES = {"wan_i2v_dense": (75600, 40), "wan_1.3b_dense": (32760, 12)}
MODES = {"default": (False, False), "int8": (True, False), "int8+fp8": (True, True)}


def dense_case(L, H, iters, windows):
    from jenga_b200 import attention as A
    from jenga_b200.flash_attn_shim import flash_attn_varlen_func
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(11)
    # Wan's flash_attention hands the shim [L, H, 128] bf16 rows of q, k, v and cu_seqlens [0, L]
    q, k, v = (torch.randn(L, H, 128, generator=g, device=dev).bfloat16() for _ in range(3))
    cu = torch.tensor([0, L], dtype=torch.int32, device=dev)

    def call(mode):
        A.QK_INT8, A.PV_FP8 = MODES[mode]
        try:
            return flash_attn_varlen_func(q, k, v, cu, cu, L, L)
        finally:
            A.QK_INT8, A.PV_FP8 = False, False

    outs = {m: call(m) for m in MODES}                 # warm-up of every mode, and its output
    torch.cuda.synchronize()
    best = {m: float("inf") for m in MODES}
    for _ in range(windows):
        for m in MODES:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                call(m)
            e1.record()
            torch.cuda.synchronize()
            best[m] = min(best[m], e0.elapsed_time(e1) / iters)
    flops = 4.0 * L * L * 128 * H
    ref = outs["default"].float()
    rms = ref.pow(2).mean().sqrt().item()
    res = {"tokens": L, "heads": H, "flop_per_call": flops}
    for m in MODES:
        d = (outs[m].float() - ref).abs()
        res[m] = {"ms_per_call": best[m], "tflops": flops / (best[m] * 1e-3) / 1e12,
                  "mean_diff_over_rms": d.mean().item() / rms, "max_diff_over_rms": d.max().item() / rms}
    res["int8_speedup"] = best["default"] / best["int8"]
    res["int8+fp8_speedup"] = best["default"] / best["int8+fp8"]
    return res


def stack_case():
    res = {}
    for name, env_val in (("default", None), ("int8", "1")):
        env = dict(os.environ)
        env.pop("JENGA_QK_INT8", None)
        env.pop("JENGA_PV_FP8", None)
        if env_val:
            env["JENGA_QK_INT8"] = env_val
        r = subprocess.run([sys.executable, str(ROOT / "bench_wan_blocks.py"), "--model", "i2v-14b", "--reps", "3"],
                           capture_output=True, text=True, env=env, timeout=3000)
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
        if r.returncode != 0 or not lines:
            raise SystemExit(f"bench_wan_blocks.py ({name}) failed:\n{r.stdout[-2000:]}\n{r.stderr[-3000:]}")
        out = json.loads(lines[-1])
        res[name] = {"seconds_per_stack_fused": out["seconds_per_stack"]["C"], "blocks": out["blocks"],
                     "card": out["card"]}
    res["int8_speedup"] = res["default"]["seconds_per_stack_fused"] / res["int8"]["seconds_per_stack_fused"]
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=5, help="calls per timed window")
    ap.add_argument("--windows", type=int, default=3, help="timed windows per mode (best is reported)")
    ap.add_argument("--no-stack", action="store_true", help="skip the bench_wan_blocks.py i2v-14b stack")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_quant_paths.py measures on a GPU; none is visible")
    res = {"bench": "quant_paths", "card_start": card()}
    for name, (L, H) in CASES.items():
        res[name] = dense_case(L, H, args.iters, args.windows)
        torch.cuda.empty_cache()
    res["wan_i2v_stack"] = "not run (--no-stack)" if args.no_stack else stack_case()
    res["card_end"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
