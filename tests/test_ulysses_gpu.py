"""2-GPU NCCL run of the Ulysses wrapper; skipped on boxes with one GPU.  The SP result must equal
the single-GPU operator bit for bit.  This is the only test whose peer stores cross NVLink; the
fused exchange at world sizes 1-8, ragged per-rank slices, head sub-groups and HostPipelinedUlysses
are covered on one GPU by tests/test_ulysses_emulated_gpu.py."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent

WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["JENGA_ROOT"]); sys.path.insert(0, os.path.join(os.environ["JENGA_ROOT"], "tests", "golden"))
import synth
from jenga_b200.ulysses import UlyssesCarvedAttention, UlyssesFusedAttention, my_parallel_attention
from jenga_b200.attention import block_sparse_attention
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank); dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
H, nbi, T = 4, 8, 256
n_img = nbi * 128; nb = nbi + 2
q = synth.peaky(H, nb, 128, 2.0, 801).transpose(1, 2).contiguous().bfloat16().to(dev)
k = synth.peaky(H, nb, 128, 2.0, 802).transpose(1, 2).contiguous().bfloat16().to(dev)
v = synth.normal((1, nb * 128, H, 128), 803).bfloat16().to(dev)
nbr = synth.band_neighbours(nbi)
n_loc = n_img // world; sl = slice(rank * n_loc, (rank + 1) * n_loc)
ql = torch.cat([q[:, sl], q[:, n_img:]], 1); kl = torch.cat([k[:, sl], k[:, n_img:]], 1); vl = torch.cat([v[:, sl], v[:, n_img:]], 1)
cu = torch.tensor([0, n_loc + 180, n_loc + T], dtype=torch.int32, device=dev)
out = my_parallel_attention(UlyssesCarvedAttention(), ql, kl, vl, n_loc, n_loc, cu, cu, top_k=2, text_amp=0.3,
                            block_neighbor_list=nbr, p_remain_rates=0.3)
cuf = torch.tensor([0, n_img + 180, n_img + T], dtype=torch.int32, device=dev)
full = block_sparse_attention(q, k, v, 2, cu_seqlens_q=cuf, cu_seqlens_kv=cuf, text_amp=0.3,
                              block_neighbor_list=nbr, p_remain_rates=0.3, text_blocks=2)
torch.cuda.synchronize()
ok = torch.equal(out[:, :n_loc], full[:, sl]) and torch.equal(out[:, n_loc:], full[:, n_img:])
fz = UlyssesFusedAttention(groups=2)   # head sub-group pipelining (auto would pick 1 at this toy size)
for _ in range(3):  # three times: the result buffer is double-buffered across calls
    out2 = my_parallel_attention(fz, ql, kl, vl, n_loc, n_loc, cu, cu, top_k=2, text_amp=0.3,
                                 block_neighbor_list=nbr, p_remain_rates=0.3)
    torch.cuda.synchronize()
    ok = ok and torch.equal(out2, out)
# I2V-shaped joint tensors: 400 text tokens (ragged: 4 text blocks with 112 zero-padded rows)
from jenga_b200.attention import block_sparse_attention_variant
T2 = 400
tq = synth.normal((1, T2, H, 128), 811).bfloat16().to(dev); tk = synth.normal((1, T2, H, 128), 812).bfloat16().to(dev)
tv = synth.normal((1, T2, H, 128), 813).bfloat16().to(dev)
ql2 = torch.cat([q[:, sl], tq], 1); kl2 = torch.cat([k[:, sl], tk], 1); vl2 = torch.cat([v[:, sl], tv], 1)
cu2 = torch.tensor([0, n_loc + 300, n_loc + T2], dtype=torch.int32, device=dev)
cuf2 = torch.tensor([0, n_img + 300, n_img + T2], dtype=torch.int32, device=dev)
qf = torch.cat([q[:, :n_img], tq], 1); kf = torch.cat([k[:, :n_img], tk], 1); vf = torch.cat([v[:, :n_img], tv], 1)
full2 = block_sparse_attention_variant("hyvideo_i2v", qf, kf, vf, 2, cu_seqlens_q=cuf2, cu_seqlens_kv=cuf2, text_blocks=4,
                                       text_amp=0.0, block_neighbor_list=nbr, p_remain_rates=0.3)
for cls in (UlyssesCarvedAttention, UlyssesFusedAttention):
    o2 = my_parallel_attention(cls(variant="hyvideo_i2v"), ql2, kl2, vl2, n_loc, n_loc, cu2, cu2, top_k=2, text_amp=0.0,
                               block_neighbor_list=nbr, p_remain_rates=0.3)
    torch.cuda.synchronize()
    ok = ok and torch.equal(o2[:, :n_loc], full2[:, sl]) and torch.equal(o2[:, n_loc:], full2[:, n_img:])
t = torch.tensor([1 if ok else 0], device=dev); dist.all_reduce(t, op=dist.ReduceOp.MIN)
if rank == 0: print("ULYSSES_OK" if t.item() == 1 else "ULYSSES_MISMATCH")
dist.destroy_process_group()
'''


def test_ulysses_two_gpus_equals_single_gpu(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, JENGA_ROOT=str(ROOT))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29611", str(script)],
                       capture_output=True, text=True, env=env, timeout=600)
    assert "ULYSSES_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
