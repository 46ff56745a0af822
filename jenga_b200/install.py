"""Makes the UNMODIFIED reference scripts (jenga_hyvideo.py, jenga_hyvideo_multigpu.py,
jenga_hyi2v.py, jenga_wan.py) import the H100 path instead of Triton / FlashAttention / the
Python gilbert module.

The reference binds names at import time
  from .attention_block_triton_diffres import block_sparse_attention
      (hyvideo/modules/models_mul_block_gc_ha_multigpu.py:25, xdit_ring_atten.py:16,
       hyvideo_i2v/modules/models_mul.py:22, wan/modules/model_mul.py:9)
  from flash_attn import flash_attn_func / flash_attn.flash_attn_interface...
  from gilbert import gilbert_mapping, ...
so the replacement must be in sys.modules BEFORE those imports run:

    python -m jenga_b200.install jenga_hyvideo.py --video-size 720 1280 ...      # launcher form
or  import jenga_b200.install; jenga_b200.install.install()                        # in-process
"""
from __future__ import annotations

import runpy
import sys
import types


def _module(name: str, **attrs) -> types.ModuleType:
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    m.__jenga_b200__ = True
    return m


def install(flash_attn: bool = True, gilbert: bool = True, ulysses: bool = True, fused_blocks: bool = True,
            gather: bool = True, i2v_sp: bool | None = None, wan_sp: bool | None = None,
            wan_i2v_sa_drop_rates=None, wan_i2v_p_remain=None) -> list[str]:
    """Pre-seeds sys.modules; returns the names it installed.
    fused_blocks: also patch the reference block classes right after they are imported so that
    RMSNorm + RoPE + cat + pooling run as the fused prologue kernel (jenga_b200/blocks.py).
    gather: route the token reorder `x[:, hilbert_order]` to the gather kernel.
    i2v_sp: `jenga_hyi2v.py --ulysses-degree N` runs the Hilbert-sharded I2V forward over the Ulysses
    exchange (jenga_b200/hyi2v_sp.py) instead of the reference's spatial-chunk dense SP; off by
    default, None reads JENGA_I2V_SP=1.  Needs fused_blocks.
    wan_sp: `jenga_wan.py --ulysses_size N` runs the Hilbert-sharded TeaCache forward over the Ulysses
    exchange (jenga_b200/wan_sp.py) instead of the reference's usp_dit_forward / usp_attn_forward; off
    by default, None reads JENGA_WAN_SP=1.  Needs fused_blocks.
    fused_blocks also gives `WanI2V(use_usp=False)` the single-GPU I2V forward of jenga_b200/wan_sp.py
    (dense, as the original model).
    wan_i2v_sa_drop_rates: "d0[,d1]" or one or two numbers, as jenga_wan.py --sa_drop_rates: the Wan2.1-I2V
    forwards (one GPU and sharded) run the carved self-attention over the Hilbert order with T2V's drop-rate
    schedule; None reads JENGA_WAN_I2V_SA_DROP, unset or "" keeps them dense.  wan_i2v_p_remain: the
    carved steps' p_remain_rates, default 0.8; None reads JENGA_WAN_I2V_P_REMAIN.  Carving needs
    fused_blocks."""
    import os
    if i2v_sp is None:
        i2v_sp = os.environ.get("JENGA_I2V_SP", "") == "1"
    if wan_sp is None:
        wan_sp = os.environ.get("JENGA_WAN_SP", "") == "1"
    if i2v_sp and not fused_blocks:
        raise ValueError("i2v_sp routes the attention through the fused I2V block forwards: it needs fused_blocks")
    if wan_sp and not fused_blocks:
        raise ValueError("wan_sp routes the self-attention through the fused WanSelfAttention forward: it needs "
                         "fused_blocks")
    from . import wan_sp as WSP
    if wan_i2v_sa_drop_rates is None:
        wan_i2v_sa_drop_rates = os.environ.get("JENGA_WAN_I2V_SA_DROP")
    if wan_i2v_p_remain is None:
        wan_i2v_p_remain = os.environ.get("JENGA_WAN_I2V_P_REMAIN")
    if WSP.parse_sa_drop_rates(wan_i2v_sa_drop_rates) and not fused_blocks:
        raise ValueError("Wan2.1-I2V carving runs in the fused WanAttentionBlock forward: it needs fused_blocks")
    WSP.set_i2v_carving(wan_i2v_sa_drop_rates, wan_i2v_p_remain)
    from . import attention as A
    from . import flash_attn_shim as F
    from . import gilbert as G
    from .sharding import default_attention

    def variant(name, text_blocks, p):
        def block_sparse_attention(query, key, value, top_k, block_size_M=128, block_size_N=128,
                                   cu_seqlens_q=None, cu_seqlens_kv=None, max_seqlen_q=None,
                                   max_seqlen_kv=None, text_blocks=text_blocks, text_amp=0.0,
                                   block_neighbor_list=None, shape_xfuse=False, p_remain_rates=p,
                                   first_frame_blocks=0):
            return A.block_sparse_attention_variant(
                name, query, key, value, top_k, block_size_M, block_size_N, cu_seqlens_q,
                cu_seqlens_kv, max_seqlen_q, max_seqlen_kv, text_blocks, text_amp,
                block_neighbor_list, shape_xfuse, p_remain_rates, first_frame_blocks)
        block_sparse_attention.__doc__ = f"jenga_b200 drop-in ({name} variant)"
        return block_sparse_attention

    done = []
    for pkg, name, tb, p in (("hyvideo", "hyvideo", 2, 0.5), ("hyvideo_i2v", "hyvideo_i2v", 4, 0.5),
                             ("wan", "wan", 0, 0.9)):
        fn = variant(name, tb, p)
        modname = f"{pkg}.modules.attention_block_triton_diffres"
        sys.modules[modname] = _module(modname, block_sparse_attention=fn,
                                       block_sparse_attention_combined=fn)
        done.append(modname)
    if ulysses:
        class xFuserLongContextAttention:
            """Same constructor surface as the reference class (all arguments ignored: ring degree
            is 1 in every Jenga script, xdit_ring_atten.py:24-59) and the same forward contract.
            The exchange runs fused over NVLink peer memory (UlyssesFusedAttention); if symmetric
            memory cannot be set up on this box — or JENGA_ULYSSES=nccl — all ranks agree on the
            NCCL all-to-all implementation.  Both are GPU paths of this library."""
            _impl = None

            def __init__(self, *a, **k):
                pass

            def forward(self, attn, query, key, value, **kw):
                cls = type(self)
                if cls._impl is None:
                    cls._impl = default_attention(None, "hyvideo")
                return cls._impl(attn, query, key, value, **kw)

            __call__ = forward
        modname = "hyvideo.modules.xdit_ring_atten"
        sys.modules[modname] = _module(modname, xFuserLongContextAttention=xFuserLongContextAttention)
        done.append(modname)
    if flash_attn:
        iface = _module("flash_attn.flash_attn_interface", flash_attn_func=F.flash_attn_func,
                        flash_attn_varlen_func=F.flash_attn_varlen_func,
                        _flash_attn_forward=F._flash_attn_forward)
        top = _module("flash_attn", flash_attn_func=F.flash_attn_func,
                      flash_attn_varlen_func=F.flash_attn_varlen_func, flash_attn_interface=iface,
                      __version__=F.__version__)
        top.__path__ = []  # behave like a package for `import flash_attn.flash_attn_interface`
        sys.modules["flash_attn"] = top
        sys.modules["flash_attn.flash_attn_interface"] = iface
        done += ["flash_attn", "flash_attn.flash_attn_interface"]
    if gilbert:
        sys.modules["gilbert"] = G
        done.append("gilbert")
    from . import blocks
    blocks.set_i2v_sp(i2v_sp)
    blocks.set_wan_sp(wan_sp)
    if fused_blocks:
        blocks.install_block_hook()
        done.append("block-forward hook")
        if i2v_sp:
            done.append("sequence-parallel I2V route")
        if wan_sp:
            done.append("sequence-parallel Wan route")
    if gather:
        from . import blocks
        blocks.install_gather_hook()
        done.append("gather hook")
    return done


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        raise SystemExit("usage: python -m jenga_b200.install <reference_script.py> [script args...]")
    installed = install()
    print(f"[jenga_b200] installed: {', '.join(installed)}", file=sys.stderr)
    sys.argv = argv
    runpy.run_path(argv[0], run_name="__main__")


if __name__ == "__main__":
    main()
