"""The ragged Ulysses head split (ulysses.RAGGED_HEADS / JENGA_ULYSSES_RAGGED=1) without a GPU.

* head_offsets: contiguous groups covering [0, H), sizes differing by at most one, larger groups first,
  r*H/P when P divides H.
* gloo ranks at (H, P) in {(3,2), (5,3), (12,8), (24,5), (40,6)}: the ragged seq_to_heads /
  heads_to_seq / gather_heads are exact inverses, and UlyssesCarvedAttention with the oracle operator
  equals the single-process operator bit for bit, with and without text rows.
* The switch: without it every refusal and message is today's; with it the Wan and HunyuanVideo-I2V
  routes accept 12 heads at P = 8, and HostPipelinedUlysses refuses a ragged split clearly.
* C-ABI validation of jenga_ulysses_scatter_ragged, before any launch.
"""
import ctypes as C
import os
import sys
from pathlib import Path

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(HERE / "golden"))

T, VALID, TOP_K = 256, 180, 2
# (H, P): image tokens (a whole number of 128-row blocks divisible by P; 768 / 8 = 96 straddles blocks)
CASES = {(3, 2): 384, (5, 3): 384, (12, 8): 768, (24, 5): 640, (40, 6): 768}


@pytest.fixture
def ragged_on(monkeypatch):
    from jenga_b200 import ulysses
    monkeypatch.setattr(ulysses, "RAGGED_HEADS", True)


@pytest.mark.parametrize("H", [1, 3, 5, 12, 24, 40, 64])
@pytest.mark.parametrize("P", [1, 2, 3, 4, 5, 6, 7, 8])
def test_head_offsets(H, P):
    from jenga_b200.ulysses import head_offsets
    off = head_offsets(H, P)
    assert len(off) == P + 1 and off[0] == 0 and off[-1] == H
    sizes = [off[r + 1] - off[r] for r in range(P)]
    assert all(s >= 0 for s in sizes) and max(sizes) - min(sizes) <= 1
    assert sizes == sorted(sizes, reverse=True)                       # larger groups first
    assert sizes == [H // P + (r < H % P) for r in range(P)]
    if H % P == 0:
        assert off == tuple(r * H // P for r in range(P + 1))


def test_wan_1p3b_at_8_ranks():
    from jenga_b200.ulysses import head_offsets
    off = head_offsets(12, 8)
    assert [off[r + 1] - off[r] for r in range(8)] == [2, 2, 2, 2, 1, 1, 1, 1]


def _inputs(H, n_img):
    import synth
    nb = n_img // 128 + T // 128
    q = synth.peaky(H, nb, 128, 2.0, 811).transpose(1, 2).contiguous().bfloat16()   # [1, S, H, D]
    k = synth.peaky(H, nb, 128, 2.0, 812).transpose(1, 2).contiguous().bfloat16()
    v = synth.normal((1, nb * 128, H, 128), 813).bfloat16()
    return q, k, v, synth.band_neighbours(n_img // 128)


def _oracle_attn(q, k, v, **kw):
    from oracle import attention_oracle as orc
    kw.pop("block_size_M", None)
    kw.pop("block_size_N", None)
    return orc.block_sparse_attention(q, k, v, variant="hyvideo", **kw)


def _worker(rank, world, H, n_img, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from jenga_b200 import ulysses as U
        U.RAGGED_HEADS = True
        q, k, v, nbr = _inputs(H, n_img)
        n = n_img // world
        off = U.head_offsets(H, world)
        b, h = off[rank], off[rank + 1] - off[rank]
        sl = slice(rank * n, (rank + 1) * n)
        # layout round trips
        y = U.seq_to_heads(q[:, sl], offsets=off)
        assert torch.equal(y, q[:, :n_img, b:b + h])
        buf = torch.empty_like(y)
        assert U.seq_to_heads(q[:, sl], out=buf, offsets=off) is buf and torch.equal(buf, y)
        assert torch.equal(U.heads_to_seq(y, offsets=off), q[:, sl])
        assert torch.equal(U.gather_heads(q[:, n_img:, b:b + h], offsets=off), q[:, n_img:])
        # the operator, with text rows (through my_parallel_attention) and without
        ql, kl, vl = (torch.cat([x[:, sl], x[:, n_img:]], 1) for x in (q, k, v))
        cu = torch.tensor([0, n + VALID, n + T], dtype=torch.int32)
        sp = U.UlyssesCarvedAttention(attn_fn=_oracle_attn)
        joint = U.my_parallel_attention(sp, ql, kl, vl, n, n, cu, cu, top_k=TOP_K, text_amp=0.3,
                                        block_neighbor_list=nbr, p_remain_rates=0.3)
        img = sp(None, q[:, sl], k[:, sl], v[:, sl], top_k=TOP_K, block_neighbor_list=nbr, p_remain_rates=0.3)
        ret[rank] = dict(joint=joint, img=img)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("H,P", list(CASES))
def test_carved_attention_equals_single_process(H, P):
    n_img = CASES[(H, P)]
    mgr = mp.Manager()
    ret = mgr.dict()
    port = 29500 + (os.getpid() + 53 * H + P) % 2000
    mp.spawn(_worker, args=(P, H, n_img, port, ret), nprocs=P, join=True)
    from jenga_b200.ulysses import head_offsets
    q, k, v, nbr = _inputs(H, n_img)
    cu = torch.tensor([0, n_img + VALID, n_img + T], dtype=torch.int32)
    off = head_offsets(H, P)
    # the single-process operator over each rank's head group, side by side: the CPU oracle's fp32 GEMMs
    # may round a one-head batch differently from a many-head one, which is not the layout's doing
    full, img = [], []
    for p in range(P):
        qs, ks, vs = (x[:, :, off[p]:off[p + 1]] for x in (q, k, v))
        full.append(_oracle_attn(qs, ks, vs, top_k=TOP_K, cu_seqlens_q=cu, cu_seqlens_kv=cu, text_amp=0.3,
                                 block_neighbor_list=nbr, p_remain_rates=0.3, text_blocks=T // 128, shape_xfuse=True))
        img.append(_oracle_attn(qs[:, :n_img], ks[:, :n_img], vs[:, :n_img], top_k=TOP_K, block_neighbor_list=nbr,
                                p_remain_rates=0.3, text_blocks=0, shape_xfuse=True))
    full = torch.cat(full, dim=2).flatten(2)
    img = torch.cat(img, dim=2)
    n = n_img // P
    for r in range(P):
        got = ret[r]
        assert got["joint"].shape == (1, n + T, H * 128)
        assert torch.equal(got["joint"][:, :n], full[:, r * n:(r + 1) * n]), r
        assert torch.equal(got["joint"][:, n:], full[:, n_img:]), r
        assert torch.equal(got["img"], img[:, r * n:(r + 1) * n]), r


def test_refusals_without_the_switch():
    from jenga_b200 import hyi2v_sp, ulysses, wan_sp
    assert not ulysses.RAGGED_HEADS or os.environ.get("JENGA_ULYSSES_RAGGED") == "1"
    if ulysses.RAGGED_HEADS:
        pytest.skip("JENGA_ULYSSES_RAGGED=1 in the environment")
    assert not ulysses.ragged(12, 8)
    with pytest.raises(ValueError, match="12 attention heads do not split over 8 ranks"):
        wan_sp._check_world(12, 8)
    with pytest.raises(ValueError, match="24 attention heads do not split over 5 ranks"):
        hyi2v_sp.check_degree(115200, 24, 5)


def test_routes_accept_ragged_degrees_under_the_switch(ragged_on):
    from jenga_b200 import hyi2v_sp, ulysses, wan_sp
    assert ulysses.ragged(12, 8) and not ulysses.ragged(12, 4)
    for P in range(1, 9):
        wan_sp._check_world(12, P)
        wan_sp._check_world(40, P)
        hyi2v_sp.check_degree(0, 24, P)
    hyi2v_sp.check_degree(115200, 24, 5)
    # what stays refused: P > 8, L % P for HunyuanVideo-I2V, a rank without a head or a real row
    with pytest.raises(ValueError, match="9 ranks; the Ulysses exchange is built for at most 8"):
        wan_sp._check_world(12, 9)
    with pytest.raises(ValueError, match="115201 image tokens do not split over 5 ranks"):
        hyi2v_sp.check_degree(115201, 24, 5)
    with pytest.raises(ValueError, match="3 attention heads over 4 ranks leave a rank without a head"):
        hyi2v_sp.check_degree(0, 3, 4)
    with pytest.raises(ValueError, match="without a real row"):
        wan_sp.shard_rows(7, 5, 0)


def test_host_pipelined_refuses_a_ragged_split(ragged_on, monkeypatch):
    from jenga_b200 import ulysses

    class _Fused:
        group = None

    monkeypatch.setattr(ulysses.dist, "get_world_size", lambda g=None: 5)
    with pytest.raises(ValueError, match="HostPipelinedUlysses needs the degree to divide the head count"):
        ulysses.HostPipelinedUlysses(128, 0, 24, fused=_Fused())


# ------------------------------------------------------------------------------------------------
# C-ABI validation: every bad argument is refused with a message before anything launches
# ------------------------------------------------------------------------------------------------
def _scatter_args(world=3, heads=5):
    from jenga_b200._lib import JengaUlyssesScatterArgs
    a = JengaUlyssesScatterArgs()
    a.x = (C.c_void_p * 3)(0x10000, 0x20000, 0x30000)     # never dereferenced on the validation paths
    a.x_stride_s = heads * 128
    a.world, a.rank, a.heads, a.head_dim, a.n_loc, a.n_text = world, 0, heads, 128, 128, 0
    peers = (C.c_uint64 * 8)(*[0x100000 * (i + 1) for i in range(8)])
    a.peer_qkv_host = C.addressof(peers)
    return a, peers


@pytest.mark.parametrize("case,needle", [
    ("null_args", "null pointer"),
    ("null_offsets", "null pointer"),
    ("null_x", "null pointer"),
    ("null_peers", "null pointer"),
    ("start", "from 0 to heads"),
    ("end", "from 0 to heads"),
    ("decreasing", "decrease"),
    ("too_large", "exceeds the 2 slots"),
    ("world9", "bad shape"),
    ("slot_range", "slot range"),
    ("peer_unaligned", "not 16-byte aligned"),
    ("joint_missing", "joint tensors missing"),
])
def test_scatter_ragged_validation(case, needle):
    from jenga_b200._lib import lib
    a, peers = _scatter_args()
    off = [0, 2, 4, 5]
    if case == "start":
        off = [1, 2, 4, 5]
    elif case == "end":
        off = [0, 2, 4, 4]
    elif case == "decreasing":
        off = [0, 2, 1, 5]
    elif case == "too_large":
        off = [0, 1, 2, 5]
    elif case == "world9":
        a.world, a.heads = 9, 12
        off = [0, 2, 4, 6, 7, 8, 9, 10, 11, 12]
    elif case == "slot_range":
        a.head_begin, a.head_count = 1, 2
    elif case == "null_x":
        a.x[1] = None
    elif case == "null_peers":
        a.peer_qkv_host = None
    elif case == "peer_unaligned":
        peers[1] = 0x100008
    elif case == "joint_missing":
        a.n_text = 256
    c_off = (C.c_int32 * len(off))(*off)
    rc = lib.jenga_ulysses_scatter_ragged(None if case == "null_args" else C.byref(a),
                                          None if case == "null_offsets" else c_off, None)
    msg = lib.jenga_last_error().decode()
    assert rc == -1 and needle in msg, (rc, msg)


def test_scatter_ragged_accepts_valid_arguments_up_to_the_launch():
    """Valid arguments pass validation: without a device the call fails at the launch (a CUDA error,
    not a fall-back); with one, nothing here is dereferenced because the test does not launch."""
    if torch.cuda.is_available():
        pytest.skip("GPU present: the launch would dereference the dummy pointers")
    from jenga_b200._lib import lib
    a, peers = _scatter_args()
    c_off = (C.c_int32 * 4)(0, 2, 4, 5)
    rc = lib.jenga_ulysses_scatter_ragged(C.byref(a), c_off, None)
    assert rc == -3, (rc, lib.jenga_last_error().decode())
