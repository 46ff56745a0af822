"""Hot-path schedule of one HunyuanVideo Jenga-Base generation (a-13): which of the 50 denoising
steps run the 60-block loop, with which sa-drop rate, and a harness that executes exactly that
many hot-path calls on synthetic activations to measure DiT-loop seconds per video for the
part of the loop this repository implements (prologue + selection + carved attention; the
dense layers of the DiT are out of scope).

Reference: jenga_hyvideo.py:28 (non_skip_steps), :128-179 (skip / residual reuse);
pipeline_hunyuan_video_prores.py:697-698,763-767 (stage switch -> sa_drop_rates[stage], forced
compute at the stage start); scripts/hyvideo_jenga_base.sh (step-rate-list 0.5 1.0).
"""
from __future__ import annotations

import torch

NON_SKIP_STEPS = (0, 1, 2, 3, 4, 7, 10, 13, 16, 19, 22, 25, 26, 29, 32, 35, 38, 41, 43, 45, 46, 47, 49)
DOUBLE_BLOCKS, SINGLE_BLOCKS = 20, 40


def schedule(num_steps: int = 50, step_rates=(0.5, 1.0), sa_drop_rates=(0.7, 0.8)):
    """[(step, computed?, sa_drop_rate)] — stage s covers steps < step_rates[s]*num_steps; the first
    step of a new stage is always computed (start_stage)."""
    out = []
    bounds = [int(r * num_steps) for r in step_rates]
    stage = 0
    start_stage = True
    for i in range(num_steps):
        while stage + 1 < len(bounds) and i > bounds[stage]:
            stage += 1
            start_stage = True
        compute = (i in NON_SKIP_STEPS) or start_stage
        start_stage = False if compute else start_stage
        out.append((i, compute, sa_drop_rates[min(stage, len(sa_drop_rates) - 1)]))
    return out


def run_hot_path_loop(img_qkv, txt_qkv, heads, norm_w, freqs_cis, nbr, cu_seqlens, *, p_remain=0.3,
                      sa_drop_rates=(0.7, 0.8), num_steps=50, max_computed_steps=None):
    """Executes the hot path for every computed (step, block) of the schedule on the given
    fused-QKV activations and returns (seconds, calls).  CUDA-event timed, no host sync inside."""
    from .hyvideo import attention_prologue, carved_attention_from_pools, select_block_num
    L = img_qkv.shape[1]
    sched = [s for s in schedule(num_steps, sa_drop_rates=sa_drop_rates) if s[1]]
    if max_computed_steps is not None:
        sched = sched[:max_computed_steps]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    calls = 0
    e0.record()
    for _, _, drop in sched:
        top_k = select_block_num(drop, L)
        for _blk in range(DOUBLE_BLOCKS + SINGLE_BLOCKS):
            q, k, v, pools = attention_prologue(img_qkv, txt_qkv, heads, *norm_w, eps=1e-6, freqs_cis=freqs_cis)
            carved_attention_from_pools(q, k, v, pools, top_k=top_k, text_blocks=2, text_amp=0.0,
                                        block_neighbor_list=nbr, p_remain_rates=p_remain,
                                        cu_seqlens_q=cu_seqlens)
            calls += 1
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3, calls
