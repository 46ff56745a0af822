"""The Wan2.1-I2V single-GPU route and its opt-in carving (jenga_b200/wan_sp.py) without a GPU.

* sa_drop_schedule equals a restatement of t2v_generate's drop-rate loop (jenga_wan.py:189-206) for
  every model call of a 40-step and a 50-step run, with one and with two rates.
* The switches (install(wan_i2v_sa_drop_rates=..., wan_i2v_p_remain=...), JENGA_WAN_I2V_SA_DROP,
  JENGA_WAN_I2V_P_REMAIN) take well-formed values and refuse malformed ones.
* i2v_curve equals the reference-pinned sliced Gilbert tables of tests/golden/gilbert.json for the
  Wan grids 21x30x52 and 21x45x80 by hash, and the reference's Python walker on a portrait grid; it is
  cached per grid.
* The binding rules, with stub `wan` modules: WanI2V(use_usp=False) gets the single-GPU I2V forward and
  the hooked wan.modules.model blocks; WanI2V(use_usp=True) keeps what it binds, with and without
  JENGA_WAN_SP; wan.modules.model_mul (T2V) is not touched.
"""
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(HERE))


def restated_schedule(steps, rates):
    """jenga_wan.py:189-206 for a run of `steps` sampling steps: the drop rate of every model call, the
    conditional and the unconditional call of each step"""
    out = []
    for idx in range(steps):
        if idx <= 25:
            cur_sa_drop_rate = rates[0]
        else:
            if len(rates) == 1:
                cur_sa_drop_rate = rates[0]
            else:
                cur_sa_drop_rate = rates[1]
        step_normed = idx / (steps - 1) * 10
        cur_sa_drop_rate = min(cur_sa_drop_rate, (step_normed) * cur_sa_drop_rate)
        out += [cur_sa_drop_rate, cur_sa_drop_rate]
    return out


@pytest.mark.parametrize("steps", [40, 50])
@pytest.mark.parametrize("rates", [(0.7,), (0.7, 0.8), (0.5, 0.3)])
def test_schedule_equals_t2v_generate(steps, rates):
    from jenga_b200.wan_sp import sa_drop_schedule
    want = restated_schedule(steps, rates)
    got = [sa_drop_schedule(cnt, 2 * steps, rates) for cnt in range(2 * steps)]
    assert got == want
    assert got[0] == 0.0 and min(got[2:]) > 0.0          # the first step is dense, the others are not zero
    assert any(d <= 0.25 for d in got) and any(d > 0.25 for d in got)


def test_schedule_refuses_a_single_step():
    from jenga_b200.wan_sp import sa_drop_schedule
    with pytest.raises(ValueError, match="at least two sampling steps"):
        sa_drop_schedule(0, 2, (0.7,))


@pytest.mark.parametrize("value,want", [("0.7", (0.7,)), (" 0.7 , 0.8 ", (0.7, 0.8)), ("0", (0.0,)), ("", ()),
                                        (None, ()), ((0.6, 0.9), (0.6, 0.9)), ([0.5], (0.5,))])
def test_sa_drop_rates_parse(value, want):
    from jenga_b200.wan_sp import parse_sa_drop_rates
    assert parse_sa_drop_rates(value) == want


@pytest.mark.parametrize("value", ["x", "0.7,", ",0.7", "0.7,0.8,0.9", "1", "1.5", "-0.1", "nan", "inf", "0.7;0.8",
                                   (), (0.1, 0.2, 0.3), ("a",)])
def test_sa_drop_rates_refuse_malformed_values(value):
    from jenga_b200.wan_sp import parse_sa_drop_rates
    with pytest.raises(ValueError, match="sa_drop_rates"):
        parse_sa_drop_rates(value)


@pytest.mark.parametrize("value,want", [(None, 0.8), ("", 0.8), ("0.5", 0.5), ("1", 1.0), (0.9, 0.9)])
def test_p_remain_parse(value, want):
    from jenga_b200.wan_sp import parse_p_remain
    assert parse_p_remain(value) == want


@pytest.mark.parametrize("value", ["0", "-1", "1.01", "x", "nan", "0.5,0.6"])
def test_p_remain_refuses_malformed_values(value):
    from jenga_b200.wan_sp import parse_p_remain
    with pytest.raises(ValueError, match="p_remain"):
        parse_p_remain(value)


def test_install_reads_the_switches(monkeypatch):
    from jenga_b200 import install, wan_sp
    monkeypatch.setattr(wan_sp, "I2V_SA_DROP_RATES", wan_sp.I2V_SA_DROP_RATES)
    monkeypatch.setattr(wan_sp, "I2V_P_REMAIN", wan_sp.I2V_P_REMAIN)
    kw = dict(flash_attn=False, gilbert=False, ulysses=False, fused_blocks=False, gather=False)
    monkeypatch.delenv("JENGA_WAN_I2V_SA_DROP", raising=False)
    monkeypatch.delenv("JENGA_WAN_I2V_P_REMAIN", raising=False)
    install.install(**kw)
    assert (wan_sp.I2V_SA_DROP_RATES, wan_sp.I2V_P_REMAIN) == ((), 0.8)
    monkeypatch.setenv("JENGA_WAN_I2V_SA_DROP", "0.7,0.8")
    with pytest.raises(ValueError, match="needs fused_blocks"):
        install.install(**kw)
    assert wan_sp.I2V_SA_DROP_RATES == ()
    monkeypatch.setenv("JENGA_WAN_I2V_P_REMAIN", "0.6")
    install.install(**dict(kw, fused_blocks=True))
    assert (wan_sp.I2V_SA_DROP_RATES, wan_sp.I2V_P_REMAIN) == ((0.7, 0.8), 0.6)
    install.install(**dict(kw, fused_blocks=True), wan_i2v_sa_drop_rates="", wan_i2v_p_remain=0.9)
    assert (wan_sp.I2V_SA_DROP_RATES, wan_sp.I2V_P_REMAIN) == ((), 0.9)
    for bad in ("0.7,x", "2"):
        monkeypatch.setenv("JENGA_WAN_I2V_SA_DROP", bad)
        with pytest.raises(ValueError, match="sa_drop_rates"):
            install.install(**dict(kw, fused_blocks=True))
    monkeypatch.setenv("JENGA_WAN_I2V_SA_DROP", "0.7")
    monkeypatch.setenv("JENGA_WAN_I2V_P_REMAIN", "0")
    with pytest.raises(ValueError, match="p_remain"):
        install.install(**dict(kw, fused_blocks=True))
    assert (wan_sp.I2V_SA_DROP_RATES, wan_sp.I2V_P_REMAIN) == ((), 0.9), "a refused value changed the setting"
    from jenga_b200 import blocks
    blocks.remove_gather_hook()


# ------------------------------------------------------------------------------------------------
# the per-grid curve
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["wan1.3B_21x30x52", "wan14B_21x45x80"])
def test_curve_equals_the_golden_tables(name):
    from jenga_b200.wan_sp import i2v_curve
    from test_oracle_cpu import sha16
    c = json.loads((HERE / "golden" / "gilbert.json").read_text())[name]
    assert c["sliced"] == 1
    l2h, h2l, nbr = i2v_curve(c["t"], c["h"], c["w"])
    assert l2h.dtype == h2l.dtype == torch.int64 and nbr.dtype == torch.bool
    assert sha16(l2h.numpy()) == c["l2h_sha"] and sha16(h2l.numpy()) == c["h2l_sha"]
    assert sha16(nbr.numpy()) == c["nbr_sha"]
    assert i2v_curve(c["t"], c["h"], c["w"]) is i2v_curve(c["t"], c["h"], c["w"]), "not cached per grid"


def test_curve_of_a_portrait_grid_matches_the_python_walker():
    """21 x 52 x 30: a 480x832 portrait image (image2video.py:180-193 with patch 2): not a SIZE_CONFIGS grid"""
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    from jenga_b200.wan_sp import i2v_curve
    g = R.gilbert()
    t, h, w = 21, 52, 30
    l2h, h2l, nbr = i2v_curve(t, h, w)
    rl2h, rh2l = g.sliced_gilbert_mapping(t, h, w)
    assert l2h.tolist() == list(rl2h) and h2l.tolist() == list(rh2l)
    assert torch.equal(nbr, torch.as_tensor(np.asarray(g.sliced_gilbert_block_neighbor_mapping(t, h, w)), dtype=torch.bool))


# ------------------------------------------------------------------------------------------------
# binding rules, stub wan modules
# ------------------------------------------------------------------------------------------------
_MODEL = '''
import torch


class WanSelfAttention(torch.nn.Module):
    def forward(self, x, seq_lens, grid_sizes, freqs):
        return "model.py self-attention"


class WanAttentionBlock(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.self_attn = WanSelfAttention()

    def forward(self, x, e, seq_lens, grid_sizes, freqs, context, context_lens):
        return "model.py block"


class WanModel(torch.nn.Module):
    model_type = "i2v"
    num_heads = 40

    def __init__(self):
        super().__init__()
        self.blocks = torch.nn.ModuleList([WanAttentionBlock()])

    def forward(self, *a, **k):
        return "model.py forward"
'''

_MODEL_MUL = '''
import torch


class WanSelfAttention(torch.nn.Module):
    def forward(self, *a, **k):
        return "model_mul self-attention"


class WanT2VCrossAttention(WanSelfAttention):
    def forward(self, *a, **k):
        return "model_mul cross-attention"


class WanAttentionBlock(torch.nn.Module):
    def forward(self, *a, **k):
        return "model_mul block"
'''

# image2video.py:99-114 in brief
_IMAGE2VIDEO = '''
import types

from .modules.model import WanModel


class WanI2V:
    def __init__(self, use_usp=False):
        self.use_usp = use_usp
        self.model = WanModel()
        if use_usp:
            from .distributed.xdit_context_parallel import usp_attn_forward, usp_dit_forward
            for block in self.model.blocks:
                block.self_attn.forward = types.MethodType(usp_attn_forward, block.self_attn)
            self.model.forward = types.MethodType(usp_dit_forward, self.model)
'''

_XDIT = '''
def usp_dit_forward(self, x, t, context, seq_len, clip_fea=None, y=None):
    return "reference usp_dit_forward"


def usp_attn_forward(self, x, seq_lens, grid_sizes, freqs, dtype=None):
    return "reference usp_attn_forward"
'''

_PROBE = '''
import json, sys
sys.path.insert(0, {root!r})
sys.path.insert(0, {stub!r})
from jenga_b200 import install
install.install(flash_attn=False, gilbert=False, ulysses=False, gather=False)
import wan.modules.model_mul as mm
import wan.modules.model as plain
import wan.distributed.xdit_context_parallel as xdit
mm_before = {{c: getattr(mm, c).forward for c in ("WanSelfAttention", "WanT2VCrossAttention", "WanAttentionBlock")}}
hooked = lambda: {{c: bool(getattr(getattr(plain, c).forward, "__jenga_b200__", False))
                   for c in ("WanSelfAttention", "WanAttentionBlock")}}
res = dict(plain_at_import=hooked())
from wan.image2video import WanI2V
res["init_wrapped"] = bool(getattr(WanI2V.__init__, "__jenga_b200__", False))
usp = WanI2V(use_usp=True)
f = usp.model.__dict__["forward"]
res["usp"] = dict(forward=f.__func__ is xdit.usp_dit_forward, jenga=bool(getattr(f.__func__, "__jenga_b200__", False)),
                  attn=usp.model.blocks[0].self_attn.__dict__["forward"].__func__ is xdit.usp_attn_forward,
                  plain=hooked())
single = WanI2V(use_usp=False)
f = single.model.__dict__.get("forward")
res["single"] = dict(forward=f.__func__.__qualname__ if f is not None else None, plain=hooked(),
                     attn_instance="forward" in single.model.blocks[0].self_attn.__dict__)
res["usp_after"] = usp.model.__dict__["forward"].__func__ is xdit.usp_dit_forward
res["mm_untouched"] = all(getattr(mm, c).forward is fn for c, fn in mm_before.items())
print(json.dumps(res))
'''


@pytest.mark.parametrize("wan_sp", ["0", "1"])
def test_wan_i2v_binding_rules(tmp_path, wan_sp):
    stub = tmp_path / "stub"
    for d in ("wan", "wan/modules", "wan/distributed"):
        (stub / d).mkdir(parents=True, exist_ok=True)
        (stub / d / "__init__.py").write_text("")
    (stub / "wan" / "modules" / "model.py").write_text(_MODEL)
    (stub / "wan" / "modules" / "model_mul.py").write_text(_MODEL_MUL)
    (stub / "wan" / "image2video.py").write_text(_IMAGE2VIDEO)
    (stub / "wan" / "distributed" / "xdit_context_parallel.py").write_text(_XDIT)
    env = {k: v for k, v in os.environ.items() if not k.startswith("JENGA_WAN")}
    env["JENGA_WAN_SP"] = wan_sp
    code = _PROBE.format(root=str(ROOT), stub=str(stub))
    r = subprocess.run([sys.executable, "-s", "-c", code], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    on = wan_sp == "1"
    assert got["init_wrapped"]
    # the module itself is hooked at import only under JENGA_WAN_SP, as before
    assert got["plain_at_import"] == dict(WanSelfAttention=on, WanAttentionBlock=on)
    # use_usp=True: what the pipeline binds (install(wan_sp=True) swaps the module functions themselves)
    assert got["usp"] == dict(forward=True, jenga=on, attn=True, plain=dict(WanSelfAttention=on, WanAttentionBlock=on))
    # use_usp=False: the single-GPU forward, and the blocks hooked
    assert got["single"] == dict(forward="_i2v_forward_factory.<locals>.forward",
                                 plain=dict(WanSelfAttention=True, WanAttentionBlock=True), attn_instance=False)
    assert got["usp_after"] and got["mm_untouched"]
