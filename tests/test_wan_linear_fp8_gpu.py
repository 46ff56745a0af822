"""Opt-in FP8 Linears on the Wan2.1 blocks, on the GPU.

1. Each Wan-side producer (wan_ln_modulate_fp8, both wan_residual_ln_fp8 forms, gelu_tanh_fp8) is
   bit-identical to quantize_rows_fp8 of its bf16 kernel's output, and the fp32 residual to the bf16
   kernel's, for bf16 and fp32 x, contiguous and strided rows.
2. The GEMM on every Wan (K, N), within the bound of tests/test_linear_fp8_gpu.py, at ragged M; and a
   row's output does not depend on M (a slice against the whole).
3. An fp32 nn.Linear's e4m3 weight is the quantisation of its bf16 cast, and the cache follows the weight.
4. The unmodified wan/modules/model_mul.py T2V block: with the switch off, and with it on under the
   shipped table (which routes no 1.3B shape), bit-identical to the block with every Linear called on its
   module, no FP8 launch and no e4m3 weight cached; with one shape routed, only that Linear is quantised
   and cached; with every Wan shape routed, eight FP8 GEMMs per block and WAN_FP8_BLOCK_TOL of the RMS.
5. The single-GPU Wan2.1-I2V forward over unmodified wan/modules/model.py blocks: off and as shipped
   bit-identical with no FP8 launch; every shape routed: eight FP8 GEMMs per block and WAN_FP8_I2V_TOL;
   and with every shape routed, the sharded route at P = 1 equals it bit for bit (the GEMM's rows do not
   depend on M).
"""
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))

pytestmark = pytest.mark.gpu

from test_linear_fp8_gpu import _check_gemm, _gemm_case  # noqa: E402

# mean, max of |on - off| / output RMS of one T2V block with every Wan-1.3B Linear routed; an H100 80GB
# showed 1.9e-3 / 2.4e-2 on both block inputs
WAN_FP8_BLOCK_TOL = (5e-3, 6e-2)
# the same for the two-block I2V model output (patch embedding and head included); an H100 80GB showed
# at most 1.4e-3 / 2.6e-2 over three steps
WAN_FP8_I2V_TOL = (4e-3, 7e-2)
WAN_SHAPES = [(5120, 5120), (5120, 13824), (13824, 5120), (1536, 1536), (1536, 8960), (8960, 1536)]


def _bits(t):
    return t.view(torch.uint8)


def _strided(t, pad):
    wide = torch.zeros(*t.shape[:-1], t.shape[-1] + pad, dtype=t.dtype, device=t.device)
    wide[..., 16:16 + t.shape[-1]] = t
    return wide[..., 16:16 + t.shape[-1]]


def _same_codes(got, want, what):
    assert torch.equal(got[1], want[1]), what
    assert torch.equal(_bits(got[0]), _bits(want[0])), what


# ------------------------------------------------------------------ 1. producers
@pytest.mark.parametrize("C", [1536, 5120])
@pytest.mark.parametrize("x_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("strided", [False, True])
def test_wan_ln_producers_are_quantize_of_the_bf16_kernels(C, x_dtype, strided):
    from jenga_b200 import dense as DN
    L = 1037 if C == 1536 else 333
    g = torch.Generator(device="cuda").manual_seed(C + L + strided)
    x = (torch.randn(1, L, C, generator=g, device="cuda") * 1.7 + 0.3).to(x_dtype)
    y = torch.randn(1, L, C, generator=g, device="cuda").bfloat16()
    e = (0.3 * torch.randn(6, C, generator=g, device="cuda")).unbind(0)
    w = 1.0 + 0.2 * torch.randn(C, generator=g, device="cuda")
    b = 0.1 * torch.randn(C, generator=g, device="cuda")
    if strided:
        x, y = _strided(x, 64), _strided(y, 32)
    x[0, 3] = 0                                          # a constant row
    what = f"C={C} x={x_dtype} strided={strided}"
    _same_codes(DN.wan_ln_modulate_fp8(x, e[0], e[1]), DN.quantize_rows_fp8(DN.wan_ln_modulate(x, e[0], e[1])), what)
    for kw, gate in ((dict(weight=w, bias=b), e[2]), (dict(shift=e[3], scale=e[4]), None)):
        r16, h16 = DN.wan_residual_ln(x, y, gate, **kw)
        r8, h8 = DN.wan_residual_ln_fp8(x, y, gate, **kw)
        assert r8.dtype == torch.float32 and torch.equal(r8, r16), what
        _same_codes(h8, DN.quantize_rows_fp8(h16), f"{what} {sorted(kw)}")


@pytest.mark.parametrize("C", [1536, 5120, 8960, 13824])
@pytest.mark.parametrize("strided", [False, True])
def test_gelu_tanh_fp8_is_quantize_of_gelu_tanh(C, strided):
    from jenga_b200 import dense as DN
    L = 517
    g = torch.Generator(device="cuda").manual_seed(C * 3 + strided)
    a = (torch.randn(1, L, C, generator=g, device="cuda") * 2).bfloat16()
    a[0, 7] = 0
    a[0, 9, 11] = 300.0
    if strided:
        a = _strided(a, 48)
    want = DN.quantize_rows_fp8(DN.gelu_tanh_into(a, torch.empty(a.shape, dtype=torch.bfloat16, device="cuda")))
    _same_codes(DN.gelu_tanh_fp8(a), want, f"C={C} strided={strided}")
    ref = torch.nn.GELU(approximate="tanh")(a)
    _same_codes(DN.gelu_tanh_fp8(a), DN.quantize_rows_fp8(ref), f"ATen C={C}")


# ------------------------------------------------------------------ 2. GEMM
@pytest.mark.parametrize("K,N", WAN_SHAPES)
@pytest.mark.parametrize("M", [1, 300])
def test_gemm_on_the_wan_shapes(K, N, M):
    from jenga_b200 import dense as DN
    case = _gemm_case(M, K, N, K + N + M, bias=torch.float32)
    _check_gemm(*case, DN.linear_fp8(*case))


@pytest.mark.parametrize("K,N", [(1536, 8960), (8960, 1536)])
def test_gemm_rows_do_not_depend_on_m(K, N):
    from jenga_b200 import dense as DN
    a8, a_scale, w8, w_scale, b = _gemm_case(2000, K, N, 3, bias=torch.float32)
    whole = DN.linear_fp8(a8, a_scale, w8, w_scale, b)
    for lo, hi in ((0, 1), (5, 6), (129, 1000), (1000, 2000), (1777, 1999)):
        part = DN.linear_fp8(a8[lo:hi], a_scale[lo:hi], w8, w_scale, b)
        assert torch.equal(part, whole[lo:hi]), (lo, hi)


# ------------------------------------------------------------------ 3. fp32 weights
def test_fp32_weight_is_quantised_as_its_bf16_cast_and_the_cache_follows_it():
    from jenga_b200 import dense as DN
    lin = torch.nn.Linear(1536, 8960, device="cuda")
    lin.requires_grad_(False)
    w8, ws, b = DN.fp8_weight(lin)
    r8, rs = DN.quantize_rows_fp8(lin.weight.to(torch.bfloat16))
    assert torch.equal(_bits(w8), _bits(r8)) and torch.equal(ws, rs) and b is lin.bias
    assert DN.fp8_weight(lin)[0] is w8                          # cached
    with torch.no_grad():
        lin.weight.mul_(3.0)
    w8b, wsb, _ = DN.fp8_weight(lin)
    assert w8b is not w8 and torch.equal(wsb, DN.quantize_rows_fp8(lin.weight.to(torch.bfloat16))[1])


# ------------------------------------------------------------------ 4. the T2V block
@pytest.fixture(scope="module")
def wan_mod():
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    yield R.load_blocks(product=True)[1]
    from jenga_b200 import blocks
    blocks.remove_gather_hook()


def _t2v_run(mod):
    from test_wan_blocks_gpu import _block_case, _make_blocks
    from jenga_b200 import blocks, dense as DN
    c = _block_case(mod)
    blk = _make_blocks(mod, 1)[0]
    x1 = None

    def run(on, routed):
        nonlocal x1
        old = DN.LINEAR_FP8, DN.FP8_ROUTED
        DN.LINEAR_FP8, DN.FP8_ROUTED = on, routed
        before = dict(blocks.STATS)
        try:
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                # block 0 takes a bf16 x, every later block the fp32 residual stream
                out0 = blk(c["x"], c["e"], c["seq_lens"], c["grid"], c["freqs"], c["ctx"], None, sa_drop_rate=0.75,
                           **c["kw"])
                if x1 is None:
                    x1 = out0.clone()
                out1 = blk(x1, c["e"], c["seq_lens"], c["grid"], c["freqs"], c["ctx"], None, sa_drop_rate=0.75,
                           **c["kw"])
            torch.cuda.synchronize()
        finally:
            DN.LINEAR_FP8, DN.FP8_ROUTED = old
        return (out0, out1), {k: blocks.STATS[k] - before[k] for k in before if blocks.STATS[k] != before[k]}
    run.blk = blk
    return run


def _cached(blk):
    return sorted(n for n, m in blk.named_modules() if "_jenga_fp8" in m.__dict__)


def test_t2v_block_off_and_as_shipped(wan_mod, monkeypatch):
    from jenga_b200 import blocks, dense as DN
    run = _t2v_run(wan_mod)
    off, d_off = run(False, DN.FP8_ROUTED)
    shipped, d_shipped = run(True, DN.FP8_ROUTED)
    assert not _cached(run.blk)
    # the block body before the FP8 path: every Linear called on its module
    monkeypatch.setattr(blocks, "_linear", lambda layer, x, x8=None: layer(x))
    monkeypatch.setattr(blocks, "_wan_ffn", lambda blk, x, cross, e: (
        lambda r: (r[0], blk.ffn(r[1])))(DN.wan_residual_ln(x, cross, None, eps=blk.norm2.eps, shift=e[3],
                                                              scale=e[4])))
    monkeypatch.setattr(blocks, "_fp8_rows", lambda layers, x: False)
    before, d_before = run(False, frozenset())
    for d in (d_off, d_shipped):
        assert d == d_before and "linear_fp8" not in d and d.get("wan_block") == 2 and "fallback" not in d
    assert all(torch.equal(a, b) for a, b in zip(off, before))
    assert all(torch.equal(a, b) for a, b in zip(shipped, before))


def test_t2v_block_quantises_only_the_routed_linears(wan_mod):
    run = _t2v_run(wan_mod)
    _, d = run(True, frozenset({("fp32", 8960, 1536)}))            # ffn.2 of the 1.3B block alone
    assert d["linear_fp8"] == 2 and "fallback" not in d
    assert _cached(run.blk) == ["ffn.2"]


def test_t2v_block_with_every_wan_shape_routed(wan_mod):
    import bench_linear_fp8 as B
    run = _t2v_run(wan_mod)
    off, _ = run(False, frozenset())
    on, d_on = run(True, B.wan_routed("wan-1.3b"))
    # q, k, v, o, cross q, cross o, ffn.0, ffn.2 in each of the two block calls
    assert d_on["linear_fp8"] == 16 and d_on.get("wan_block") == 2 and "fallback" not in d_on
    for i, (a, b) in enumerate(zip(on, off)):
        e = (a.double() - b.double()).abs() / b.double().pow(2).mean().sqrt()
        print(f"\n[Wan T2V block, input {i}] FP8 Linears on vs off: mean {e.mean():.2e} max {e.max():.2e} of the RMS")
        assert e.mean() <= WAN_FP8_BLOCK_TOL[0] and e.max() <= WAN_FP8_BLOCK_TOL[1]


# ------------------------------------------------------------------ 5. the I2V forward (model.py blocks)
class _Everything(frozenset):
    def __contains__(self, item):
        return True


@pytest.fixture
def plain():
    from test_wan_i2v_sp_cpu import load_plain_wan
    mod = load_plain_wan(wan_sp=False)
    if mod is None:
        pytest.skip("reference files not staged (oracle/_ref/, oracle/_ref_wan_model/)")
    return mod


def _switch(monkeypatch, on, routed):
    from jenga_b200 import dense as DN
    monkeypatch.setattr(DN, "LINEAR_FP8", on)
    monkeypatch.setattr(DN, "FP8_ROUTED", routed)


def _i2v_single(mod):
    from test_wan_i2v_sp_gpu import _model
    from jenga_b200 import wan_sp
    m = _model(mod, torch.device("cuda"))
    wan_sp.bind_wan_i2v(m)
    return m


def _steps(m):
    from test_wan_i2v_sp_gpu import _run
    from jenga_b200 import blocks
    before = dict(blocks.STATS)
    outs = _run(m, m.forward, torch.device("cuda"))                      # computed, computed, skipped
    return outs, {k: blocks.STATS[k] - before[k] for k in before if blocks.STATS[k] != before[k]}


def test_i2v_forward_off_as_shipped_and_every_shape_routed(plain, monkeypatch):
    from jenga_b200 import dense as DN
    # one model per leg (the TeaCache state advances with every call), the same seeded weights each time
    _switch(monkeypatch, False, DN.FP8_ROUTED)
    off, d_off = _steps(_i2v_single(plain))
    _switch(monkeypatch, True, DN.FP8_ROUTED)
    m = _i2v_single(plain)
    shipped, d_shipped = _steps(m)
    assert d_shipped == d_off and "linear_fp8" not in d_off and "fallback" not in d_off
    assert d_off["wan_i2v_self_dense"] == 4 and d_off["wan_i2v_cross"] == 4
    assert all(torch.equal(a, b) for a, b in zip(off, shipped))
    assert not any("_jenga_fp8" in mod.__dict__ for mod in m.modules())
    _switch(monkeypatch, True, _Everything({None}))
    m = _i2v_single(plain)
    on, d_on = _steps(m)
    # two computed steps x two blocks x (q, k, v, o, cross q, cross o, ffn.0, ffn.2)
    assert d_on["linear_fp8"] == 32 and "fallback" not in d_on
    assert {k: v for k, v in d_on.items() if k != "linear_fp8"} == d_off
    for blk in m.blocks:
        cached = sorted(n for n, mod in blk.named_modules() if "_jenga_fp8" in mod.__dict__)
        assert cached == ["cross_attn.o", "cross_attn.q", "ffn.0", "ffn.2", "self_attn.k", "self_attn.o",
                          "self_attn.q", "self_attn.v"], cached
    for i, (a, b) in enumerate(zip(on, off)):
        e = (a.double() - b.double()).abs() / b.double().pow(2).mean().sqrt()
        print(f"\n[Wan I2V forward, step {i}] FP8 Linears on vs off: mean {e.mean():.2e} max {e.max():.2e} of the RMS")
        assert e.mean() <= WAN_FP8_I2V_TOL[0] and e.max() <= WAN_FP8_I2V_TOL[1]


def test_i2v_sharded_route_at_one_rank_equals_single_gpu_with_every_shape_routed(plain, monkeypatch):
    import copy
    from jenga_b200 import ulysses, wan_sp
    from test_ulysses_emulated_gpu import _run_ranks
    from test_wan_i2v_sp_gpu import GRID, HEADS, _model, _run
    from test_wan_sp_forward_gpu import _emulated_all_gather, _emulated_broadcast, _Group
    from test_wan_sp_gpu import _World
    _switch(monkeypatch, True, _Everything({None}))
    fresh = _model(plain, torch.device("cuda"))
    single = copy.deepcopy(fresh)
    wan_sp.bind_wan_i2v(single)
    got_single, d_single = _steps(single)
    assert d_single["linear_fp8"] == 32 and "fallback" not in d_single
    dist = ulysses.dist
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    for name, fn in dict(get_world_size=lambda g=None: g.size, get_rank=lambda g=None: g.rank,
                         get_global_rank=lambda g, r: r, is_initialized=lambda: True,
                         all_gather=_emulated_all_gather, broadcast=_emulated_broadcast).items():
        monkeypatch.setattr(dist, name, fn)
    shared = {"rows": {}}
    got = {}
    L = GRID[0] * GRID[1] * GRID[2]
    from jenga_b200 import blocks
    before = dict(blocks.STATS)

    def rank(r, bar):
        shared["bar"] = bar
        wan_sp.parallelize_wan_i2v(fresh, group=_Group(1, 0, shared),
                                   attention=_World(1, L, HEADS).fused(bar, 1, 0, None))
        got[r] = _run(fresh, fresh.forward, torch.device("cuda"), 1)

    _run_ranks(1, rank)
    assert blocks.STATS["linear_fp8"] - before["linear_fp8"] == 32
    assert blocks.STATS["fallback"] == before["fallback"]
    for i in range(3):
        assert torch.equal(got[0][i], got_single[i]), i
