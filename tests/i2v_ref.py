"""Loads the UNMODIFIED HunyuanVideo-I2V block module hyvideo_i2v/modules/models_mul.py
(MMDoubleStreamBlock / MMSingleStreamBlock) through oracle/ref_loader.py's reference packages —
checker only, used by tests/test_i2v_blocks_*.py and bench_i2v_blocks.py."""
from __future__ import annotations

import importlib
import sys
import types


def _stub_if_missing(name: str, **attrs) -> None:
    try:
        importlib.import_module(name)
    except Exception:
        m = sys.modules.get(name)
        if m is None:
            m = types.ModuleType(name)
            m.__dict__["__oracle_stub__"] = True
            sys.modules[name] = m
        for k, v in attrs.items():
            if not hasattr(m, k):
                setattr(m, k, v)


def load_i2v_blocks(product: bool):
    """hyvideo_i2v/modules/models_mul.py bound to the reference operator (product=False) or to
    jenga_b200 through install() (product=True).  hyvideo_i2v/utils/helpers.py:11-13 imports
    `deepspeed` and tensorboard's SummaryWriter for training helpers the blocks never call: stubbed
    when absent, like the packages ref_loader.install_environment_stubs() stubs."""
    from oracle import ref_loader
    _stub_if_missing("deepspeed")
    _stub_if_missing("torch.utils.tensorboard", SummaryWriter=object)
    with ref_loader.reference_packages(product=product):
        return importlib.import_module("hyvideo_i2v.modules.models_mul")
