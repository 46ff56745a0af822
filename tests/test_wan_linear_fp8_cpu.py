"""Opt-in FP8 Linears on the Wan2.1 blocks, without a GPU: argument validation of the three Wan-side
producers (jenga_wan_ln_modulate_fp8, jenga_wan_residual_ln_fp8, jenga_gelu_tanh_fp8), the routing
kind of fp32 weights, and which Wan FFNs the block opens into ffn.0 -> GELU -> ffn.2."""
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
from jenga_b200 import _lib  # noqa: E402
from jenga_b200._lib import lib  # noqa: E402
from test_cabi_validation_cpu import E_CUDA, E_INVALID, E_UNSUPPORTED, _err  # noqa: E402

P = 0x10000
BF16, F32 = _lib.JENGA_BF16, _lib.JENGA_F32


def _ln(over):
    a = dict(x=P, x_dtype=F32, x_stride=256, scale=P, shift=P, out8=P, out_stride=256, a_scale=P, rows=10,
             channels=256)
    a.update(over)
    return lib.jenga_wan_ln_modulate_fp8(a["x"], a["x_dtype"], a["x_stride"], a["scale"], a["shift"], a["out8"],
                                         a["out_stride"], a["a_scale"], a["rows"], a["channels"], 1e-6, None)


def _res(over):
    a = dict(x=P, x_dtype=F32, x_stride=256, y=P, y_stride=256, gate=None, res=P, res_stride=256, va=P, vb=P,
             affine=1, out8=P, out_stride=256, a_scale=P, rows=10, channels=256)
    a.update(over)
    return lib.jenga_wan_residual_ln_fp8(a["x"], a["x_dtype"], a["x_stride"], a["y"], a["y_stride"], a["gate"],
                                         a["res"], a["res_stride"], a["va"], a["vb"], a["affine"], a["out8"],
                                         a["out_stride"], a["a_scale"], a["rows"], a["channels"], 1e-6, None)


def _gelu(over):
    a = dict(x=P, x_stride=256, out8=P, out_stride=256, a_scale=P, rows=10, channels=256)
    a.update(over)
    return lib.jenga_gelu_tanh_fp8(a["x"], a["x_stride"], a["out8"], a["out_stride"], a["a_scale"], a["rows"],
                                   a["channels"], None)


COMMON = [
    (dict(x=None), E_INVALID, "null"),
    (dict(a_scale=None), E_INVALID, "null"),
    (dict(out8=None), E_INVALID, "null"),
    (dict(rows=0), E_INVALID, "shape"),
    (dict(channels=72, x_stride=72, out_stride=80), E_UNSUPPORTED, "multiple of 16"),
    (dict(out_stride=264), E_INVALID, "aligned"),
    (dict(x=P + 8), E_INVALID, "aligned"),
    (dict(out8=P + 8), E_INVALID, "aligned"),
    (dict(a_scale=P + 2), E_INVALID, "aligned"),
]


@pytest.mark.parametrize("over,code,needle", COMMON + [
    (dict(scale=None), E_INVALID, "null"),
    (dict(shift=P + 4), E_INVALID, "aligned"),
    (dict(x_dtype=_lib.JENGA_F16), E_INVALID, "bf16 or f32"),
    (dict(channels=6160, x_stride=6160, out_stride=6160), E_UNSUPPORTED, "6144"),
    (dict(x_stride=252), E_INVALID, "shape"),
])
def test_wan_ln_modulate_fp8_argument_validation(over, code, needle):
    assert _ln(over) == code, _err()
    assert needle in _err().lower(), _err()


@pytest.mark.parametrize("over,code,needle", COMMON + [
    (dict(y=None), E_INVALID, "null"),
    (dict(res=None), E_INVALID, "null"),
    (dict(va=None), E_INVALID, "null"),
    (dict(y_stride=128), E_INVALID, "shape"),
    (dict(res_stride=260), E_INVALID, "shape"),
    (dict(gate=P + 4), E_INVALID, "aligned"),
    (dict(res=P + 8), E_INVALID, "aligned"),
    (dict(x_dtype=7), E_INVALID, "bf16 or f32"),
])
def test_wan_residual_ln_fp8_argument_validation(over, code, needle):
    assert _res(over) == code, _err()
    assert needle in _err().lower(), _err()


@pytest.mark.parametrize("over,code,needle", COMMON + [
    (dict(x_stride=260), E_INVALID, "shape"),
    (dict(channels=16400, x_stride=16400, out_stride=16400), E_UNSUPPORTED, "16384"),
])
def test_gelu_tanh_fp8_argument_validation(over, code, needle):
    assert _gelu(over) == code, _err()
    assert needle in _err().lower(), _err()


def test_without_a_device_the_producers_report_a_cuda_error():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert _ln({}) == E_CUDA and _err()
    assert _ln(dict(x_dtype=BF16)) == E_CUDA
    assert _res({}) == E_CUDA and _res(dict(affine=0, gate=P)) == E_CUDA
    assert _gelu(dict(channels=13824, x_stride=13824, out_stride=13824)) == E_CUDA and _err()


# ------------------------------------------------------------------ routing kinds
def test_fp32_weights_have_a_kind_of_their_own():
    from jenga_b200 import dense as DN
    kinds = {dt: DN.fp8_weight_kind(torch.nn.Linear(32, 16, dtype=dt))
             for dt in (torch.float32, torch.bfloat16)}
    assert kinds == {torch.float32: "fp32", torch.bfloat16: "bf16"}


def test_fp32_keys_never_match_a_hunyuan_layer():
    """HunyuanVideo checkpoints are bf16 (kind "bf16") or --use-fp8 (kind "fp8_ref"): a table of every Wan
    ("fp32", K, N) shape routes none of them, whatever their K and N"""
    from jenga_b200 import blocks, dense as DN
    import bench_linear_fp8 as B
    wan = B.wan_routed("wan-14b") | B.wan_routed("wan-1.3b")
    assert wan and all(k[0] == "fp32" for k in wan)
    assert {(k, n) for _, k, n in wan} == {(5120, 5120), (5120, 13824), (13824, 5120), (1536, 1536),
                                           (1536, 8960), (8960, 1536)}
    hy = {(k, n) for _, k, n in B.SHAPES.values()}
    lin = torch.nn.Linear(16, 16, dtype=torch.bfloat16)
    for k, n in hy | {(5120, 5120), (1536, 1536)}:
        assert (DN.fp8_weight_kind(lin), k, n) not in wan
    fp8_layer = torch.nn.Linear(16, 16).to(torch.float8_e4m3fn)
    assert DN.fp8_weight_kind(fp8_layer) == "fp8_ref"
    # and a CPU weight is never taken, whatever the table says
    old = DN.LINEAR_FP8, DN.FP8_ROUTED
    DN.LINEAR_FP8, DN.FP8_ROUTED = True, wan
    try:
        assert blocks._fp8_routed(torch.nn.Linear(1536, 1536), 1536) is None
    finally:
        DN.LINEAR_FP8, DN.FP8_ROUTED = old


def test_the_table_is_consulted_before_any_weight_is_quantised(monkeypatch):
    """an unrouted layer is never handed to fp8_weight, which quantises and caches an e4m3 copy"""
    from jenga_b200 import blocks, dense as DN
    seen = []
    monkeypatch.setattr(DN, "fp8_weight", lambda layer: seen.append(layer))
    monkeypatch.setattr(DN, "LINEAR_FP8", True)
    monkeypatch.setattr(DN, "FP8_ROUTED", frozenset({("fp32", 8960, 1536)}))
    for lin in (torch.nn.Linear(1536, 1536), torch.nn.Linear(1536, 8960),
                torch.nn.Linear(8960, 1536, dtype=torch.bfloat16), torch.nn.Linear(3072, 3072, dtype=torch.bfloat16)):
        assert blocks._fp8_routed(lin, lin.in_features) is None
    assert seen == []
    routed = torch.nn.Linear(8960, 1536)
    blocks._fp8_routed(routed, 8960)
    assert seen == [routed]


def test_shipped_routes_are_wan_shapes_only():
    from jenga_b200 import dense as DN
    assert all(k[0] == "fp32" for k in DN.FP8_ROUTED)


# ------------------------------------------------------------------ FFN eligibility
def _ffn(act=None):
    return torch.nn.Sequential(torch.nn.Linear(64, 256), act or torch.nn.GELU(approximate="tanh"),
                               torch.nn.Linear(256, 64))


def test_the_wan_ffn_is_opened_only_when_plain():
    from jenga_b200 import blocks
    assert blocks._plain_ffn(_ffn())
    assert not blocks._plain_ffn(_ffn(torch.nn.GELU()))                       # erf GELU
    assert not blocks._plain_ffn(_ffn(torch.nn.SiLU()))
    assert not blocks._plain_ffn(torch.nn.Sequential(*_ffn(), torch.nn.Identity()))
    assert not blocks._plain_ffn(torch.nn.Sequential(torch.nn.Linear(64, 256), torch.nn.GELU(approximate="tanh")))

    class Sub(torch.nn.Sequential):
        pass
    assert not blocks._plain_ffn(Sub(*_ffn()))
    for where in range(4):                                                    # the Sequential, then each child
        f = _ffn()
        m = f if where == 0 else f[where - 1]
        h = m.register_forward_hook(lambda *a: None)
        assert not blocks._plain_ffn(f), where
        h.remove()
        assert blocks._plain_ffn(f)
        h = m.register_forward_pre_hook(lambda *a: None)
        assert not blocks._plain_ffn(f), where
        h.remove()
    f = _ffn()
    f[0].forward = lambda x: x
    assert not blocks._plain_ffn(f)
    f = _ffn()
    f[2] = torch.nn.Bilinear(256, 256, 64)
    assert not blocks._plain_ffn(f)
