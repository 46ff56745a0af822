"""When the fused HunyuanVideo / HunyuanVideo-I2V block forwards run, and when they hand the call to
the original forward.

Each case starts from the eligible call of test_dropin_blocks_gpu.py / test_i2v_blocks_gpu.py (C = 512,
4 heads of 128, bf16 under autocast, sa_drop_rate 0.7, one curve, cu_seqlens from a text mask) and
changes one input.  The eligible call counts the variant's fused forward once and no fallback.  Every
other call counts one fallback and no fused kernel, and returns bit for bit what the original forward
returns, or raises the exception type the original raises."""
import inspect
import math
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))

from test_dropin_blocks_gpu import _reinit, _structured_tokens, modules  # noqa: E402,F401
from test_i2v_blocks_gpu import i2v_modules  # noqa: E402,F401

C = 512


def _inputs(mod, kind, i2v, t=8, T=None, heads=4):
    """parameter name -> value of the eligible call (t frames of 16 x 16 tokens, T text rows)"""
    from jenga_b200 import gilbert
    h, w = 16, 16
    L = t * h * w
    T = T or (400 if i2v else 256)
    S = L + T
    l2h, h2l = gilbert.mapping_tensors(t, h, w)
    h2l = h2l.cuda()
    img = _structured_tokens(L, C, 1)
    txt = _structured_tokens(-(-T // 128) * 128, C, 2, gain=0.5)[:, :T].contiguous()
    gen = torch.Generator(device="cuda").manual_seed(3)
    vec = torch.randn(1, C, generator=gen, device="cuda").bfloat16()
    text_mask = torch.zeros(1, T, dtype=torch.int64, device="cuda")
    text_mask[:, :180] = 1
    cu = mod.get_cu_seqlens(text_mask, L)
    ang = torch.rand(L, C // heads // 2, generator=torch.Generator(device="cuda").manual_seed(4), device="cuda")
    ang = ang * 2 * math.pi
    freqs = (torch.cos(ang).repeat_interleave(2, 1).contiguous(), torch.sin(ang).repeat_interleave(2, 1).contiguous())
    a = dict(vec=vec, cu_seqlens_q=cu, cu_seqlens_kv=cu, max_seqlen_q=S, max_seqlen_kv=S, freqs_cis=freqs,
             sa_drop_rate=0.7, txt_amp=0.431, curve_sel=[[l2h.cuda(), h2l, gilbert.block_neighbor_mapping(t, h, w)]],
             p_remain_rates=0.3, per_block_token=128)
    a.update(dict(img=img, txt=txt) if kind == "double" else dict(x=torch.cat([img, txt], 1), txt_len=T))
    if not i2v:
        a["txt_block_num"] = 2
        return a
    # jenga_hyi2v.py:124-130: the first frame in Hilbert order, a device mask over L for the double
    # block and a CPU mask over L + T for the single block
    ff = torch.zeros(L, dtype=torch.bool, device="cuda")
    ff[:h * w] = True
    ff = ff[h2l]
    if kind == "single":
        full = torch.zeros(S, dtype=torch.bool)
        full[:L] = ff.cpu()
        ff = full
    tr_vec = torch.randn(1, C, generator=gen, device="cuda").bfloat16()
    a.update(first_frame_mask=ff, condition_type="token_replace", token_replace_vec=tr_vec,
             frist_frame_token_num=h * w)
    return a


def _stream(a):
    return "img" if "img" in a else "x"


# case -> (variants, kinds, block kwargs, _inputs kwargs, argument overrides: a -> dict)
_ANY = ("hy", "i2v")
_BOTH = ("double", "single")
CASES = {
    "sa_drop_rate_0": (_ANY, _BOTH, {}, {}, lambda a: dict(sa_drop_rate=0.0)),
    "curve_sel_none": (_ANY, _BOTH, {}, {}, lambda a: dict(curve_sel=None)),
    "curve_sel_int": (_ANY, _BOTH, {}, {}, lambda a: dict(curve_sel=1)),
    "per_block_token_64": (_ANY, _BOTH, {}, {}, lambda a: dict(per_block_token=64)),
    "cu_seqlens_q_none": (_ANY, _BOTH, {}, {}, lambda a: dict(cu_seqlens_q=None)),
    "freqs_cis_none": (_ANY, ("single",), {}, {}, lambda a: dict(freqs_cis=None)),
    "head_dim_64": (_ANY, _BOTH, dict(heads=8), dict(heads=8), lambda a: {}),
    "layernorm_qk_norm": (_ANY, _BOTH, dict(qk_norm_type="layer"), {}, lambda a: {}),
    "fp32_input": (_ANY, _BOTH, {}, {}, lambda a: {_stream(a): a[_stream(a)].float()}),
    "ragged_S": (("hy",), _BOTH, {}, dict(T=200), lambda a: {}),
    "token_replace_prefix": (("i2v",), _BOTH, {}, {}, lambda a: dict(first_frame_mask=None)),
    "four_blocks": (("i2v",), _BOTH, {}, dict(t=1, T=256), lambda a: {}),
    "txt_len_0": (("i2v",), ("single",), {}, {}, lambda a: dict(txt_len=0)),
    "txt_len_all_rows": (("i2v",), ("single",), {}, {}, lambda a: dict(txt_len=a["x"].shape[1])),
}
PARAMS = [pytest.param(v, k, c, id=f"{v}-{k}-{c}") for c, (vs, ks, *_) in CASES.items() for v in vs for k in ks]


def _setup(hy_modules, i2v_mods, variant, kind, block_kw=None, input_kw=None):
    mod = i2v_mods[1] if variant == "i2v" else hy_modules[2]
    bk = {"heads": 4, **(block_kw or {})}
    heads = bk.pop("heads")
    cls = getattr(mod, "MMDoubleStreamBlock" if kind == "double" else "MMSingleStreamBlock")
    blk = cls(C, heads, mlp_width_ratio=4.0, dtype=torch.bfloat16, device="cuda", **bk)
    _reinit(blk, 11)
    a = _inputs(mod, kind, variant == "i2v", **(input_kw or {}))
    names = list(inspect.signature(type(blk).forward.__wrapped__).parameters)[1:]
    return blk, a, names


def _run(fn):
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            out = fn()
        torch.cuda.synchronize()
        return out, None
    except Exception as e:       # noqa: BLE001 — the exception type is what is compared
        return None, type(e)


@pytest.mark.parametrize("variant,kind", [(v, k) for v in _ANY for k in _BOTH])
def test_eligible_call_runs_the_fused_forward(modules, i2v_modules, variant, kind):
    from jenga_b200 import blocks
    blk, a, names = _setup(modules, i2v_modules, variant, kind)
    before = dict(blocks.STATS)
    out, exc = _run(lambda: blk(*(a[n] for n in names)))
    assert exc is None
    key = f"{'i2v' if variant == 'i2v' else 'hy'}_{kind}"
    assert blocks.STATS[key] == before[key] + 1
    assert blocks.STATS["fallback"] == before["fallback"]


@pytest.mark.parametrize("variant,kind,case", PARAMS)
def test_ineligible_call_runs_the_original_forward(modules, i2v_modules, variant, kind, case):
    from jenga_b200 import blocks
    _, _, block_kw, input_kw, over = CASES[case]
    blk, a, names = _setup(modules, i2v_modules, variant, kind, block_kw, input_kw)
    a.update(over(a))
    args = tuple(a[n] for n in names)
    want, want_exc = _run(lambda: type(blk).forward.__wrapped__(blk, *args))
    before = dict(blocks.STATS)
    got, got_exc = _run(lambda: blk(*args))
    moved = {k: blocks.STATS[k] - before[k] for k in blocks.STATS if blocks.STATS[k] != before[k]}
    # one fallback, and no fused forward or fused kernel ran before the call was handed over
    assert moved == {"fallback": 1}
    assert got_exc is want_exc
    if want_exc is None:
        want, got = (want, got) if kind == "double" else ((want,), (got,))
        assert len(got) == len(want) and all(torch.equal(g, w) for g, w in zip(got, want))
