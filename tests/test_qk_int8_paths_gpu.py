"""The opt-in INT8 Q.K^T (`attention.QK_INT8`) and FP8 P.V (`attention.PV_FP8`) switches on the paths that
did not follow them before: the fused Ulysses exchange (the operator's sp_out branch, so
UlyssesFusedAttention and HostPipelinedUlysses), the FlashAttention shims, and through the
varlen shim the dense self-attention of a Wan-I2V block.  Also the LSE of the INT8 kernel, which adds
back the per-row shift Q'_i . mean(K) that K smoothing takes off every score.

Every sequence-parallel rank computes the same per-(b, h) quantisation over the same N+T rows as the
single-GPU operator (K mean, Q / K groups, the V absmax per head) and attention is per head, so the
exchanged rows must equal the single-GPU result bit for bit.  The shims must equal a direct dense
launch of the same variant bit for bit, and stay within the tolerance rows of tests/test_qk_int8_gpu.py
against fp64 truth."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(HERE / "golden"))
import synth  # noqa: E402
import test_ulysses_emulated_gpu as U  # noqa: E402
import test_wan_blocks_gpu as W  # noqa: E402
import test_wan_i2v_gpu as I  # noqa: E402
from test_qk_int8_cpu import KBIAS, TOL_MAX, TOL_MEAN, dequantize_ref  # noqa: E402
from test_wan_i2v_gpu import wan_modules  # noqa: E402,F401  (fixture)

DEV = torch.device("cuda", 0)
MODES = {"int8": dict(qk_int8=True), "fp8": dict(pv_fp8=True), "int8+fp8": dict(qk_int8=True, pv_fp8=True)}
ROWS = {"int8": (TOL_MEAN, TOL_MAX), "fp8": (6e-2, 0.35), "int8+fp8": (6e-2, 0.35)}   # (mean, max) / RMS


def _flags(monkeypatch, mode):
    from jenga_b200 import attention as A
    f = MODES.get(mode, {})
    monkeypatch.setattr(A, "QK_INT8", bool(f.get("qk_int8")))
    monkeypatch.setattr(A, "PV_FP8", bool(f.get("pv_fp8")))


def _single(variant, q, k, v, T, valid, amp, nbr, **flags):
    from jenga_b200.attention import block_sparse_attention_variant
    cu = U._cu(q.shape[1] - T, T, valid)
    return block_sparse_attention_variant(variant, q, k, v, U.TOP_K, cu_seqlens_q=cu, cu_seqlens_kv=cu,
                                          text_blocks=(T + U.BLOCK - 1) // U.BLOCK, text_amp=amp,
                                          block_neighbor_list=nbr, p_remain_rates=U.P_REMAIN, shape_xfuse=True,
                                          **flags)


# ------------------------------------------------------------------------------------------------
# 0. the entry point attention._launch uses for INT8 operands
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_ex_entry_point_equals_the_older_ones_without_lse_and_ulysses(monkeypatch, dtype):
    """_launch passes INT8 operands to jenga_carved_attn_fwd_qk_int8_ex; the same launch through
    jenga_carved_attn_fwd_sched, through _ex without a work order and through the unordered
    jenga_carved_attn_fwd_qk_int8 gives the same bits."""
    import ctypes as C
    import test_attn_schedule_gpu as S
    from jenga_b200 import attention as A
    from jenga_b200._lib import lib
    q, k, v, bits = S._inputs(dtype, 5)
    qk8 = A.quantize_qk_int8(q, k)
    ex = lib.jenga_carved_attn_fwd_qk_int8_ex
    routes = {
        "sched": lambda a, x, sched, st: lib.jenga_carved_attn_fwd_sched(a, C.byref(x._obj.base), sched, st),
        "ex, no order": lambda a, x, sched, st: ex(a, x, None, st),
        "qk_int8": lambda a, x, sched, st: lib.jenga_carved_attn_fwd_qk_int8(a, C.byref(x._obj.base), st),
    }
    kws = [dict(qk_int8=qk8)] + ([dict(qk_int8=qk8, v_fp8=A.quantize_v_fp8(v))] if dtype == torch.bfloat16 else [])
    for kw in kws:
        got = S._run(q, k, v, bits, **kw)
        for name, fn in routes.items():
            with monkeypatch.context() as m:
                m.setattr(lib, "jenga_carved_attn_fwd_qk_int8_ex", fn)
                want = S._run(q, k, v, bits, **kw)
            torch.cuda.synchronize()
            assert S._same_bits(got, want), (name, list(kw))


# ------------------------------------------------------------------------------------------------
# 1. the fused Ulysses exchange, emulated at world sizes 1-8
# ------------------------------------------------------------------------------------------------
CASES = [(P, G, "hy_amp") for P, G in U.WORLD_G] + [(2, 1, "i2v"), (8, 3, "i2v")]


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("P,G,name", CASES)
def test_emulated_ulysses_follows_the_switches(monkeypatch, P, G, name, mode):
    variant, T, valid, amp = U.VARIANTS[name]
    n_img = U._n_img(P, "ragged")
    n, h = n_img // P, U.H // P
    hg = h // G
    q, k, v = U._inputs(n_img, T, torch.bfloat16)
    nbr = synth.band_neighbours(n_img // U.BLOCK)
    plain = _single(variant, q, k, v, T, valid, amp, nbr)
    ref = _single(variant, q, k, v, T, valid, amp, nbr, **MODES[mode])
    assert not U._same(ref, plain)                      # the variant really differs
    world = U.World(P, n, T, torch.bfloat16)
    world.restate_qkv(q, k, v)
    _flags(monkeypatch, mode)
    for r in range(P):
        for g in range(G):
            U._attend(world, r, g, hg, variant, valid, amp, nbr, world.p_out[0])
    torch.cuda.synchronize()
    for p in range(P):
        assert U._guards_intact(world.out_full[0][p], world.out_rows)
        assert U._guards_intact(world.qkv_full[p], world.qkv_rows)    # the quantisers only read it
        assert U._same(world.out[0][p], U._relaid(ref, p, n, T)), p


@pytest.mark.parametrize("P,G", [(2, 3), (8, None)])
def test_production_classes_follow_the_switches(monkeypatch, P, G):
    """UlyssesFusedAttention (through my_parallel_attention) and HostPipelinedUlysses, unmodified, on
    emulated ranks with both switches on: every rank's rows are the single-GPU variant's."""
    from jenga_b200 import ulysses
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    monkeypatch.setattr(ulysses.dist, "get_world_size", lambda g=None: g.size)
    variant, T, valid, amp = U.VARIANTS["hy_amp"]
    n_img = U._n_img(P, "ragged")
    n, N, H, D = n_img // P, n_img, U.H, U.D
    nbr = synth.band_neighbours(n_img // U.BLOCK)
    x = U._inputs(n_img, T, torch.bfloat16)
    ref = _single(variant, *x, T, valid, amp, nbr, qk_int8=True, pv_fp8=True)
    _flags(monkeypatch, "int8+fp8")
    cu = torch.tensor([0, n + valid, n + T], dtype=torch.int32, device=DEV)
    kw = dict(top_k=U.TOP_K, text_amp=amp, block_neighbor_list=nbr, p_remain_rates=U.P_REMAIN)

    def local(t, r):
        return torch.cat([t[:, r * n:(r + 1) * n], t[:, N:]], dim=1)

    world = U.World(P, n, T, torch.bfloat16, n_out=2)
    got = [None] * P

    def fused_rank(r, bar):
        sp = U._emulated_fused(world, bar)(group=U._FakeGroup(P, r), variant=variant, groups=G)
        out = ulysses.my_parallel_attention(sp, *(local(t, r) for t in x), n, n, cu, cu, **kw)
        torch.cuda.synchronize()
        got[r] = out.clone()

    U._run_ranks(P, fused_rank)
    world2 = U.World(P, n, T, torch.bfloat16, n_out=2)
    host = [[local(t, r).cpu().pin_memory() for t in x] for r in range(P)]
    hout = [torch.empty((1, n + T, H, D), dtype=torch.bfloat16).pin_memory() for _ in range(P)]

    def host_rank(r, bar):
        fused = U._emulated_fused(world2, bar)(group=U._FakeGroup(P, r), variant=variant, groups=G)
        hp = ulysses.HostPipelinedUlysses(n, T, H, D, dtype=torch.bfloat16, device=DEV, fused=fused)
        hp(*host[r], hout[r], cu_seqlens_q=cu, cu_seqlens_kv=cu, **kw)
        torch.cuda.synchronize()

    U._run_ranks(P, host_rank)
    for r in range(P):
        assert U._same(got[r].view(n + T, H, D), U._relaid(ref, r, n, T)), r
        assert U._same(hout[r].to(DEV), got[r].view(1, n + T, H, D)), r
    for w in (world, world2):
        for p in range(P):
            assert U._guards_intact(w.out_full[0][p], w.out_rows) and U._guards_intact(w.out_full[1][p], w.out_rows)


# ------------------------------------------------------------------------------------------------
# 2. the real exchange on two GPUs
# ------------------------------------------------------------------------------------------------
WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["JENGA_ROOT"]); sys.path.insert(0, os.path.join(os.environ["JENGA_ROOT"], "tests", "golden"))
import synth
from jenga_b200 import attention as A
from jenga_b200.ulysses import UlyssesFusedAttention, my_parallel_attention
assert A.QK_INT8 and A.PV_FP8
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
cuf = torch.tensor([0, n_img + 180, n_img + T], dtype=torch.int32, device=dev)
full = A.block_sparse_attention_variant("hyvideo", q, k, v, 2, cu_seqlens_q=cuf, cu_seqlens_kv=cuf, text_amp=0.3,
                                        block_neighbor_list=nbr, p_remain_rates=0.3, text_blocks=2)
A.QK_INT8 = A.PV_FP8 = False
plain = A.block_sparse_attention_variant("hyvideo", q, k, v, 2, cu_seqlens_q=cuf, cu_seqlens_kv=cuf, text_amp=0.3,
                                         block_neighbor_list=nbr, p_remain_rates=0.3, text_blocks=2)
A.QK_INT8 = A.PV_FP8 = True
ok = not torch.equal(full, plain)
fz = UlyssesFusedAttention(groups=2)
for _ in range(3):
    out = my_parallel_attention(fz, ql, kl, vl, n_loc, n_loc, cu, cu, top_k=2, text_amp=0.3,
                                block_neighbor_list=nbr, p_remain_rates=0.3)
    torch.cuda.synchronize()
    ok = ok and torch.equal(out[:, :n_loc], full[:, sl]) and torch.equal(out[:, n_loc:], full[:, n_img:])
t = torch.tensor([1 if ok else 0], device=dev); dist.all_reduce(t, op=dist.ReduceOp.MIN)
if rank == 0: print("ULYSSES_QUANT_OK" if t.item() == 1 else "ULYSSES_QUANT_MISMATCH")
dist.destroy_process_group()
'''


def test_two_gpu_exchange_with_both_switches_equals_single_gpu(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, JENGA_ROOT=str(ROOT), JENGA_QK_INT8="1", JENGA_PV_FP8="1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29613", str(script)],
                       capture_output=True, text=True, env=env, timeout=600)
    assert "ULYSSES_QUANT_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


# ------------------------------------------------------------------------------------------------
# 3. the FlashAttention shims
# ------------------------------------------------------------------------------------------------
def _direct(q, k, v, scale, mode, out=None, lse=None):
    """One dense-class launch of the variant over q [1|B, Sq, H, D] against k, v: what the shims must do."""
    from jenga_b200.attention import _launch, quantize_qk_int8, quantize_v_fp8
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    out = torch.empty_like(q) if out is None else out
    f = MODES[mode]
    v8 = quantize_v_fp8(v) if f.get("pv_fp8") else None
    qk8 = quantize_qk_int8(q, k, lse_shift=lse is not None) if f.get("qk_int8") else None
    _launch(q, k, v, None, 0, (Sq + 127) // 128, scale, 0.0, 1 << 30, Sk, Sq, Sk, out, None, q.dtype, lse_out=lse,
            v_fp8=v8, qk_int8=qk8)
    return out


def _fp64(q, k, v, scale):
    """[B,Sq,H,D] -> (out fp64 [B,Sq,H,D], lse fp64 [B,H,Sq])"""
    qd, kd, vd = (t.double().transpose(1, 2) for t in (q, k, v))
    s = qd @ kd.transpose(-1, -2) * scale
    return (torch.softmax(s, -1) @ vd).transpose(1, 2), torch.logsumexp(s, -1)


def _check_row(got, q=None, k=None, v=None, scale=None, mode=None, truth=None):
    if truth is None:
        truth, _ = _fp64(q, k, v, scale)
    rms = truth.pow(2).mean().sqrt()
    e = (got.double() - truth).abs() / rms
    mean, mx = ROWS[mode]
    print(f"\n[{mode}] vs fp64: mean {e.mean().item():.2e} max {e.max().item():.2e}")
    assert e.mean().item() <= mean and e.max().item() <= mx


def _qkv(shape_q, shape_k, dtype, seed, model=True):
    """model: q and k are bench.synth_tokens (the regime the tolerance rows are modelled on), v normal;
    otherwise all three normal.  Shapes [B, S, H, 128] or [S, H, 128]."""
    import bench
    g = torch.Generator(device="cuda").manual_seed(seed)
    v = torch.randn(shape_k, generator=g, device="cuda").to(dtype)
    if not model:
        return (torch.randn(shape_q, generator=g, device="cuda").to(dtype),
                torch.randn(shape_k, generator=g, device="cuda").to(dtype), v)

    def tokens(shape, s):
        lead = shape[:-3] or (1,)
        S, H = shape[-3], shape[-2]
        x = torch.cat([bench.synth_tokens(S, H, DEV, s + 7 * i) for i in range(lead[0])])
        return x.reshape(shape).to(dtype)
    return tokens(shape_q, seed + 1), tokens(shape_k, seed + 2), v


SHIM_CASES = [(m, torch.bfloat16) for m in MODES] + [("int8", torch.float16)]


@pytest.mark.parametrize("mode,dtype", SHIM_CASES)
def test_flash_attn_func_follows_the_switches(monkeypatch, mode, dtype):
    from jenga_b200.flash_attn_shim import flash_attn_func
    q, k, v = _qkv((2, 300, 3, 128), (2, 1000, 3, 128), dtype, 31)
    plain = flash_attn_func(q, k, v, softmax_scale=0.1)
    _flags(monkeypatch, mode)
    got = flash_attn_func(q, k, v, softmax_scale=0.1)
    _flags(monkeypatch, None)
    want = _direct(q, k, v, 0.1, mode)
    torch.cuda.synchronize()
    assert torch.equal(got, want) and not torch.equal(got, plain)
    _check_row(got, q, k, v, 0.1, mode)


def test_fp8_switch_leaves_fp16_shims_on_the_default_path(monkeypatch):
    from jenga_b200.flash_attn_shim import flash_attn_func
    q, k, v = _qkv((1, 300, 2, 128), (1, 700, 2, 128), torch.float16, 32)
    plain = flash_attn_func(q, k, v)
    _flags(monkeypatch, "fp8")
    assert torch.equal(flash_attn_func(q, k, v), plain)


@pytest.mark.parametrize("mode,dtype", SHIM_CASES)
def test_flash_attn_varlen_func_quantises_each_segment(monkeypatch, mode, dtype):
    """Two ragged segments (1290 and 1280 rows): each is its own launch, quantised on its own."""
    from jenga_b200.flash_attn_shim import flash_attn_varlen_func
    S, H, cut = 2570, 2, 1290
    q, k, v = _qkv((S, H, 128), (S, H, 128), dtype, 33)
    cu = torch.tensor([0, cut, S], dtype=torch.int32, device="cuda")
    plain = flash_attn_varlen_func(q, k, v, cu, cu, S, S)
    _flags(monkeypatch, mode)
    got = flash_attn_varlen_func(q, k, v, cu, cu, S, S)
    _flags(monkeypatch, None)
    want = torch.zeros_like(q)
    for a, b in ((0, cut), (cut, S)):
        _direct(q[None, a:b], k[None, a:b], v[None, a:b], 128 ** -0.5, mode, out=want[None, a:b])
    torch.cuda.synchronize()
    assert torch.equal(got, want) and not torch.equal(got, plain)
    truth = torch.cat([_fp64(q[None, a:b], k[None, a:b], v[None, a:b], 128 ** -0.5)[0] for a, b in ((0, cut), (cut, S))], 1)
    _check_row(got[None], truth=truth, mode=mode)


@pytest.mark.parametrize("mode,dtype", SHIM_CASES)
def test_flash_attn_forward_follows_the_switches_with_its_lse(monkeypatch, mode, dtype):
    from jenga_b200.flash_attn_shim import _flash_attn_forward
    q, k, v = _qkv((1, 300, 3, 128), (1, 1000, 3, 128), dtype, 34)
    _flags(monkeypatch, mode)
    got, lse, _, _ = _flash_attn_forward(q, k, v, softmax_scale=0.1, window_size_left=-1, window_size_right=-1)
    _flags(monkeypatch, None)
    want_lse = torch.empty_like(lse)
    want = _direct(q, k, v, 0.1, mode, lse=want_lse)
    torch.cuda.synchronize()
    assert torch.equal(got, want) and torch.equal(lse, want_lse)
    _check_row(got, q, k, v, 0.1, mode)


# ------------------------------------------------------------------------------------------------
# 4. the LSE of the INT8 kernel
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("kbias", [0.0, 3.0])
def test_int8_lse_against_fp64(monkeypatch, dtype, kbias):
    """Tight against the fp64 LSE of the dequantised problem (Q' = q8 q_scale, K' = k8 k_scale + mean):
    that checks the shift arithmetic.  Loose against the fp64 LSE of the 16-bit problem.  With a large
    common channel bias of K, a missing or wrongly signed shift is several units off."""
    from jenga_b200 import attention as A
    from jenga_b200.flash_attn_shim import _flash_attn_forward
    B, Sq, Sk, H, scale = 1, 300, 1000, 2, 128 ** -0.5
    q, k, v = _qkv((B, Sq, H, 128), (B, Sk, H, 128), dtype, 35, model=False)
    k = (k.double() + kbias * KBIAS.to(k.device)).to(dtype)
    _flags(monkeypatch, "int8")
    _, lse, _, _ = _flash_attn_forward(q, k, v, softmax_scale=scale)
    _flags(monkeypatch, None)
    q8, qs, k8, ks, shift = A.quantize_qk_int8(q, k, lse_shift=True)
    mean = A.quantize_int8(k, 128, True)[2]                                     # [B*H, 128]
    qd = dequantize_ref(q8.cpu(), qs.cpu(), 64)[:, :Sq]
    kd = dequantize_ref(k8.cpu(), ks.cpu(), 128)[:, :Sk] + mean.cpu().double().reshape(B, 1, H, 128)
    _, lse_dq = _fp64(qd, kd, kd, scale)
    _, lse_16 = _fp64(q.cpu(), k.cpu(), k.cpu(), scale)
    got = lse.cpu().double()
    tight = (got - lse_dq).abs().max().item()
    loose = (got - lse_16).abs()
    unshifted = (got - scale * shift.cpu().double().reshape(B, H, -1)[..., :Sq] - lse_16).abs()
    print(f"\n[int8 lse, K bias x{kbias:g}, {dtype}] vs dequantised fp64: max {tight:.2e}; vs 16-bit fp64: "
          f"mean {loose.mean().item():.2e} max {loose.max().item():.2e}; without the shift: mean {unshifted.mean().item():.2e}")
    assert tight <= 1e-4
    assert loose.mean().item() <= 0.08 and loose.max().item() <= 0.3
    if kbias:
        assert unshifted.mean().item() >= 1.0


# ------------------------------------------------------------------------------------------------
# 5. the Wan-I2V block, whose dense self-attention reaches the varlen shim
# ------------------------------------------------------------------------------------------------
def _varlen_int8_by_hand(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, dropout_p=0.0,
                         softmax_scale=None, causal=False, window_size=(-1, -1), deterministic=False, **_):
    assert dropout_p in (0, 0.0) and not causal
    cq, ck = cu_seqlens_q.tolist(), cu_seqlens_k.tolist()
    scale = q.shape[-1] ** -0.5 if softmax_scale is None else float(softmax_scale)
    out = torch.zeros_like(q)
    for i in range(len(cq) - 1):
        q0, q1, k0, k1 = cq[i], cq[i + 1], ck[i], ck[i + 1]
        if q1 > q0 and k1 > k0:
            _direct(q[None, q0:q1], k[None, k0:k1], v[None, k0:k1], scale, "int8", out=out[None, q0:q1])
    return out


def test_wan_i2v_block_dense_self_attention_follows_the_switch(wan_modules, monkeypatch):
    _, ours = wan_modules
    blk = I._make_i2v_blocks(ours, 1)[0]
    c = W._block_case(ours)
    ctx = I._i2v_context(1536, 71)
    x = c["x"]
    before, _, d0 = I._run(blk, x, c, ctx, 0.0, "fused", ours)
    _flags(monkeypatch, "int8")
    on, _, d1 = I._run(blk, x, c, ctx, 0.0, "fused", ours)
    _flags(monkeypatch, None)
    fa = ours.flash_attention.__globals__["flash_attn"]
    with monkeypatch.context() as m:
        m.setattr(fa, "flash_attn_varlen_func", _varlen_int8_by_hand)
        hand, _, d2 = I._run(blk, x, c, ctx, 0.0, "fused", ours)
    off, _, d3 = I._run(blk, x, c, ctx, 0.0, "fused", ours)
    for d in (d0, d1, d2, d3):   # the self-attention is still the original forward's dense branch
        assert d["wan_block"] == 1 and d["wan_i2v_cross"] == 1 and d["fallback"] == 1 and d["wan_self"] == 0, d
    assert not torch.equal(on, before)
    assert torch.equal(on, hand)
    assert torch.equal(off, before)
