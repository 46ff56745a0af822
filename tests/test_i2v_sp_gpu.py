"""Sequence-parallel HunyuanVideo-I2V on the fused block path, emulated on one GPU.

The ranks are emulated as tests/test_ulysses_emulated_gpu.py does: every rank's exchange buffers on
one device, UlyssesFusedAttention unmodified, one Python thread per rank with host barriers.

* Attention section: blocks._attention_section under `jenga_sp` (prologue without pooling, then the
  Ulysses exchange) at world sizes 1, 2, 3, 4, 8 and head sub-groups 1-3, production I2V shapes (24
  heads, 400 text tokens of which 300 are valid, ragged S).  On every rank's rows it equals, bit for
  bit, the single-GPU fused I2V attention section (prologue pools, select, carved attention) and the
  single-GPU operator on the full prologue output, and every selection of the two agrees.
* Blocks: one unmodified hyvideo_i2v/modules/models_mul.py double block and one single block at the
  HunyuanVideo width, token replace on, emulated at P = 2 and 4, against the single-GPU fused forward.
  Linears run on a rank's rows, so the tolerance is that of tests/test_dropin_blocks_gpu.py, on rows
  whose masks are equal.  STATS counts the i2v_*_sp forwards and no fallback.
* A block with hybrid_seq_parallel_attn set still runs the original forward, jenga_sp or not.
"""
import copy
import random
import sys
import threading
import types
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE / "golden"))
import synth  # noqa: E402
from test_dropin_blocks_gpu import _compare, _reinit, _structured_tokens  # noqa: E402
from test_ulysses_emulated_gpu import (DEV, H, WORLD_G, World, _emulated_fused, _FakeGroup,  # noqa: E402
                                       _run_ranks)

D, BLOCK = 128, 128
T, VALID = 400, 300
DROP, P_REMAIN = 0.7, 0.3


@pytest.fixture
def emulated_groups(monkeypatch):
    from jenga_b200 import ulysses
    monkeypatch.setattr(ulysses, "_group_size_rank", lambda g: (g.size, g.rank))
    monkeypatch.setattr(ulysses.dist, "get_world_size", lambda g=None: g.size)


class _Capture(list):
    """A.MASK_CAPTURE that records which emulated rank appended each selection"""
    local = threading.local()

    def append(self, item):
        super().append((getattr(self.local, "rank", None), item))


def _onehot(bits, nb):
    from jenga_b200.attention import bits_to_onehot
    return bits_to_onehot(bits, nb)


def _bits(a):
    return a.view(torch.int16)


# ------------------------------------------------------------------------------------------------
# attention section
# ------------------------------------------------------------------------------------------------
def _section_inputs(L, seed=5100):
    g = torch.Generator(device=DEV).manual_seed(seed)
    img_qkv = (_structured_tokens(L, 3 * H * D, seed) * 0.5).contiguous()
    txt_qkv = (torch.randn(1, T, 3 * H * D, generator=g, device=DEV) * 0.5).bfloat16()
    w = [(1.0 + 0.2 * torch.randn(D, generator=g, device=DEV)).bfloat16() for _ in range(4)]
    ang = torch.rand(L, D // 2, generator=g, device=DEV) * 6.2831853
    freqs = (torch.cos(ang).repeat_interleave(2, 1).contiguous(), torch.sin(ang).repeat_interleave(2, 1).contiguous())
    return img_qkv, txt_qkv, [(wi, 1e-6) for wi in w], freqs


def _cu(n):
    return torch.tensor([0, n + VALID, n + T], dtype=torch.int32, device=DEV)


@pytest.mark.parametrize("P,G", WORLD_G)
def test_attention_section_under_sp_equals_single_gpu(emulated_groups, P, G):
    from jenga_b200 import attention as A, blocks
    from jenga_b200.hyvideo import attention_prologue, select_block_num
    L = 9 * BLOCK                                     # n_loc = 1152 / P: 576, 384, 288, 144 rows straddle blocks
    S, n = L + T, L // P
    nb = (S + BLOCK - 1) // BLOCK
    assert S % BLOCK and nb - 4 == L // BLOCK
    img_qkv, txt_qkv, norms, freqs = _section_inputs(L)
    curve_sel = [[None, None, synth.band_neighbours(L // BLOCK).to(DEV)]]
    mod = types.SimpleNamespace(random=random)
    kw = dict(sa_drop_rate=DROP, txt_amp=0.0, curve_sel=curve_sel, p_remain_rates=P_REMAIN, text_blocks=4,
              pad_ragged=True)
    # single GPU: the fused I2V attention section, and the operator on the full prologue output
    A.MASK_CAPTURE = []
    try:
        fused = blocks._attention_section(types.SimpleNamespace(heads_num=H), mod, img_qkv, txt_qkv, norms,
                                          freqs_cis=freqs, cu_seqlens_q=_cu(L), cu_seqlens_kv=_cu(L), **kw)
        fused_bits = A.MASK_CAPTURE[0][0]
        q, k, v, _ = attention_prologue(img_qkv, txt_qkv, H, *(w for w, _ in norms), 1e-6, freqs, want_pool=False)
        op, op_bits = A.block_sparse_attention_variant("hyvideo_i2v", q, k, v, select_block_num(DROP, L),
                                                       cu_seqlens_q=_cu(L), cu_seqlens_kv=_cu(L), text_blocks=4,
                                                       block_neighbor_list=curve_sel[0][2], p_remain_rates=P_REMAIN,
                                                       return_mask_bits=True)
    finally:
        A.MASK_CAPTURE = None
    world = World(P, n, T, torch.bfloat16, n_out=2)
    got = {}

    def rank(r, bar):
        sp = _emulated_fused(world, bar)(group=_FakeGroup(P, r), variant="hyvideo_i2v", groups=G)
        blk = types.SimpleNamespace(heads_num=H, jenga_sp=sp)
        sl = slice(r * n, (r + 1) * n)
        out = blocks._attention_section(blk, mod, img_qkv[:, sl], txt_qkv, norms,
                                        freqs_cis=(freqs[0][sl], freqs[1][sl]), cu_seqlens_q=_cu(n),
                                        cu_seqlens_kv=_cu(n), **kw)
        torch.cuda.synchronize()
        got[r] = out.clone()

    _run_ranks(P, rank)
    # the prologue's pools and the operator's select the same key blocks for every (head, query block)
    assert torch.equal(_onehot(fused_bits, nb), _onehot(op_bits, nb))
    for r in range(P):
        sl = slice(r * n, (r + 1) * n)
        assert got[r].shape == (1, n + T, H * D)
        assert torch.equal(_bits(got[r]), _bits(torch.cat([op[:, sl], op[:, L:]], 1))), r
        assert torch.equal(_bits(got[r]), _bits(torch.cat([fused[:, sl], fused[:, L:]], 1))), r


# ------------------------------------------------------------------------------------------------
# the unmodified I2V blocks
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def i2v_module():
    from oracle import ref_loader as R
    if not R.available():
        pytest.skip("reference files not staged (oracle/_ref/)")
    from i2v_ref import load_i2v_blocks
    ours = load_i2v_blocks(product=True)
    assert ours.MMDoubleStreamBlock.forward.__jenga_b200__
    yield ours
    from jenga_b200 import blocks
    blocks.remove_gather_hook()


def _block_case(mod):
    from jenga_b200 import gilbert
    t, h, w = 8, 16, 16
    L, C = t * h * w, H * D
    l2h, h2l = gilbert.mapping_tensors(t, h, w)
    curve_sel = [[l2h.to(DEV), h2l.to(DEV), gilbert.block_neighbor_mapping(t, h, w).to(DEV)]]
    img = _structured_tokens(L, C, 1)
    txt = _structured_tokens(4 * BLOCK, C, 2, gain=0.5)[:, :T].contiguous()
    gen = torch.Generator(device=DEV).manual_seed(3)
    vec = torch.randn(1, C, generator=gen, device=DEV).bfloat16()
    tr_vec = torch.randn(1, C, generator=gen, device=DEV).bfloat16()
    ang = torch.rand(L, 64, generator=torch.Generator(device=DEV).manual_seed(4), device=DEV) * 6.2831853
    freqs = (torch.cos(ang).repeat_interleave(2, 1).contiguous(), torch.sin(ang).repeat_interleave(2, 1).contiguous())
    ff = torch.zeros(L, dtype=torch.bool, device=DEV)                   # jenga_hyi2v.py:124-130
    ff[:h * w] = True
    ff = ff[h2l.to(DEV)]
    return dict(L=L, C=C, curve_sel=curve_sel, img=img, txt=txt, vec=vec, tr_vec=tr_vec, freqs=freqs, ff=ff,
                hw=h * w)


def _call(blk, kind, c, img, n, freqs, mask):
    tail = (DROP, mask, "token_replace", c["tr_vec"], c["hw"], 0.0, c["curve_sel"], P_REMAIN)
    cu, S = _cu(n), n + T
    if kind == "double":
        return blk(img, c["txt"], c["vec"], cu, cu, S, S, freqs, *tail)
    return (blk(torch.cat([img, c["txt"]], 1), c["vec"], T, cu, cu, S, S, freqs, *tail),)


@pytest.mark.parametrize("kind", ["double", "single"])
@pytest.mark.parametrize("P", [2, 4])
def test_unmodified_i2v_block_under_sp_matches_single_gpu(emulated_groups, i2v_module, kind, P):
    from jenga_b200 import attention as A, blocks
    c = _block_case(i2v_module)
    L = c["L"]
    n, S = L // P, L + T
    nb = (S + BLOCK - 1) // BLOCK
    cls = getattr(i2v_module, "MMDoubleStreamBlock" if kind == "double" else "MMSingleStreamBlock")
    blk = cls(c["C"], H, mlp_width_ratio=4.0, dtype=torch.bfloat16, device=DEV)
    _reinit(blk, 11)
    full_mask = lambda m, rows: torch.cat([m[rows].cpu(), torch.zeros(T, dtype=torch.bool)])   # noqa: E731
    stat = "i2v_double" if kind == "double" else "i2v_single"
    cap = _Capture()
    A.MASK_CAPTURE = cap
    try:
        before = dict(blocks.STATS)
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            ref = _call(blk, kind, c, c["img"], L, c["freqs"],
                        c["ff"] if kind == "double" else full_mask(c["ff"], slice(None)))
        torch.cuda.synchronize()
        assert blocks.STATS[stat] == before[stat] + 1
        world = World(P, n, T, torch.bfloat16, n_out=2)
        ranks = [copy.deepcopy(blk) for _ in range(P)]
        got = {}

        def rank(r, bar):
            _Capture.local.rank = r
            b = ranks[r]
            b.jenga_sp = _emulated_fused(world, bar)(group=_FakeGroup(P, r), variant="hyvideo_i2v", groups=1)
            sl = slice(r * n, (r + 1) * n)
            mask = c["ff"][sl] if kind == "double" else full_mask(c["ff"], sl)
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                out = _call(b, kind, c, c["img"][:, sl].contiguous(), n, (c["freqs"][0][sl], c["freqs"][1][sl]),
                            mask)
            torch.cuda.synchronize()
            got[r] = [o.clone() for o in out]

        before = dict(blocks.STATS)
        _run_ranks(P, rank)
    finally:
        A.MASK_CAPTURE = None
    assert blocks.STATS[stat + "_sp"] == before[stat + "_sp"] + P, "the sharded I2V forward did not run"
    assert blocks.STATS["fallback"] == before["fallback"] and blocks.STATS[stat] == before[stat]
    # the selections: the single-GPU one, and the ranks' head groups in rank order
    single = [b for r, (b, _) in cap if r is None]
    per_rank = {r: b for r, (b, _) in cap if r is not None}
    assert len(single) == 1 and sorted(per_rank) == list(range(P))
    sp_bits = torch.cat([per_rank[r] for r in range(P)], dim=1)
    same = (_onehot(single[0], nb) == _onehot(sp_bits, nb)).all(-1).all(1)[0]   # per query block, all heads
    n_img = nb - 4
    row_ok = torch.cat([same.repeat_interleave(BLOCK),
                        torch.ones(max(0, L - n_img * BLOCK), dtype=torch.bool, device=DEV)])[:L]
    ref_img = ref[0][:, :L]
    ref_txt = ref[1] if kind == "double" else ref[0][:, L:]
    got_img = torch.cat([got[r][0][:, :n] for r in range(P)], 1)
    _compare(ref_img, got_img, row_ok, f"I2V {kind} P={P} image rows")
    for r in range(P):
        got_txt = got[r][1] if kind == "double" else got[r][0][:, n:]
        _compare(ref_txt, got_txt, torch.ones(T, dtype=torch.bool, device=DEV), f"I2V {kind} P={P} rank {r} text")


class _SentinelCalled(Exception):
    pass


@pytest.mark.parametrize("kind", ["double", "single"])
def test_hybrid_seq_parallel_attn_still_runs_the_original_forward(i2v_module, kind):
    """hybrid_seq_parallel_attn keeps its meaning, with or without jenga_sp next to it: the reference's
    own SP forward (models_mul.py:264-274, :483-493) runs"""
    from jenga_b200 import blocks
    from jenga_b200.ulysses import UlyssesCarvedAttention
    c = _block_case(i2v_module)
    L = c["L"]
    calls = []

    def sentinel(*a, **k):
        calls.append(1)
        raise _SentinelCalled

    cls = getattr(i2v_module, "MMDoubleStreamBlock" if kind == "double" else "MMSingleStreamBlock")
    blk = cls(512, 4, mlp_width_ratio=4.0, dtype=torch.bfloat16, device=DEV)
    c.update(img=c["img"][..., :512].contiguous(), txt=c["txt"][..., :512].contiguous(), vec=c["vec"][:, :512],
             tr_vec=c["tr_vec"][:, :512])
    blk.hybrid_seq_parallel_attn = sentinel
    for jsp in (None, UlyssesCarvedAttention(group=None, variant="hyvideo_i2v")):
        if jsp is not None:
            blk.jenga_sp = jsp
        before = dict(blocks.STATS)
        mask = c["ff"] if kind == "double" else torch.cat([c["ff"].cpu(), torch.zeros(T, dtype=torch.bool)])
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16), pytest.raises(_SentinelCalled):
            _call(blk, kind, c, c["img"], L, c["freqs"], mask)
        assert blocks.STATS["fallback"] == before["fallback"] + 1
        assert all(blocks.STATS[k] == before[k] for k in ("i2v_double", "i2v_single", "i2v_double_sp",
                                                          "i2v_single_sp"))
    assert calls == [1, 1]
