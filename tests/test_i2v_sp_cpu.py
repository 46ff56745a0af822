"""Sequence-parallel HunyuanVideo-I2V (jenga_b200/hyi2v_sp.py) without a GPU.

* The sharded forward at world sizes 2 and 4 (gloo), on a small transformer whose embedders, blocks
  and final layer are elementwise stand-ins and whose attention is the oracle operator through
  UlyssesCarvedAttention: every rank's image rows, RoPE rows, first-frame masks and cu_seqlens are
  the matching slices of the full Hilbert-ordered tensors, and the gathered, inverse-scattered output
  equals a single-process restatement of jenga_hyi2v.py's ra_forward bit for bit — on a computed step
  and on a skipped step that reuses the residual.
* The degree checks: L % P and heads % P.
* install(): hyvideo_i2v.inference.parallelize_transformer is swapped only with the switch on; without
  it the reference function stays, and with it no block gets hybrid_seq_parallel_attn.
"""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
sys.path.insert(0, str(ROOT))

GRID = (4, 8, 16)                  # t, h, w: L = 512 image tokens
# two heads per rank at P = 4: the CPU oracle matches itself bit for bit across head groups of two or
# more heads (a one-head group rounds its text rows differently)
HEADS, D = 8, 128
C = HEADS * D
T, VALID = 400, 300                # S = 912: ragged, eight 128-row blocks, four of them text
DROP, P_REMAIN, AMP = 0.5, 0.3, 0.2


def _oracle_attn(q, k, v, **kw):
    from oracle import attention_oracle as orc
    kw.pop("block_size_M", None)
    kw.pop("block_size_N", None)
    return orc.block_sparse_attention(q, k, v, variant="i2v", **kw)


def _vec(seed, n=C, s=0.5):
    g = torch.Generator().manual_seed(seed)
    return 1.0 + s * torch.randn(n, generator=g)


class _Double(torch.nn.Module):
    """Stand-in MMDoubleStreamBlock with the I2V argument order: elementwise q/k/v, RoPE-like use of
    the tables, token replace by the mask, attention through jenga_sp (Ulysses) or, without it, the
    oracle over the whole sequence.  Records what it was given."""

    def __init__(self, seed, log):
        super().__init__()
        self.w = [_vec(seed + i) for i in range(5)]
        self.log = log

    def attend(self, img_q, img_k, img_v, txt_q, txt_k, txt_v, cu, drop, amp, curve_sel, p_remain):
        from jenga_b200.hyvideo import select_block_num
        from jenga_b200.ulysses import my_parallel_attention
        n = img_q.shape[1]
        q, k, v = (torch.cat([a, b], 1).unflatten(2, (HEADS, D)).bfloat16()
                   for a, b in ((img_q, txt_q), (img_k, txt_k), (img_v, txt_v)))
        nbr = curve_sel[0][2]
        sp = getattr(self, "jenga_sp", None)
        P = dist.get_world_size(sp.group) if sp is not None else 1
        top_k = select_block_num(drop, n * P)
        if sp is not None:
            out = my_parallel_attention(sp, q, k, v, n, n, cu, cu, top_k=top_k, text_amp=amp,
                                        block_neighbor_list=nbr, p_remain_rates=p_remain)
        else:
            out = _oracle_attn(q, k, v, top_k=top_k, cu_seqlens_q=cu, cu_seqlens_kv=cu, text_amp=amp,
                               block_neighbor_list=nbr, p_remain_rates=p_remain, text_blocks=4)
        return out.float()

    def forward(self, img, txt, vec, cu_q, cu_kv, max_q, max_kv, freqs_cis, drop, ff_mask, cond, tr_vec,
                ff_num, amp, curve_sel, p_remain):
        cos, sin = freqs_cis
        self.log.append(dict(img=img.clone(), cos=cos.clone(), sin=sin.clone(), mask=ff_mask.clone(), cu=cu_q.clone(),
                             max_q=max_q))
        mod = torch.where(ff_mask[None, :, None], tr_vec[:, None], vec[:, None])
        rope = lambda x: x * cos.repeat(1, HEADS) + sin.repeat(1, HEADS)   # noqa: E731
        a = self.attend(rope(img * self.w[0] * mod), rope(img * self.w[1]), img * self.w[2],
                        txt * self.w[0], txt * self.w[1], txt * self.w[2], cu_q, drop, amp, curve_sel, p_remain)
        n = img.shape[1]
        return img + a[:, :n] * self.w[3] * mod, txt + a[:, n:] * self.w[4]

    # the stand-ins route jenga_sp themselves, as the fused forwards of blocks.py do
    forward.__jenga_b200__ = True


class _Single(_Double):
    def forward(self, x, vec, txt_len, cu_q, cu_kv, max_q, max_kv, freqs_cis, drop, full_mask, cond, tr_vec,
                ff_num, amp, curve_sel, p_remain):
        cos, sin = freqs_cis
        self.log.append(dict(img=x.clone(), cos=cos.clone(), sin=sin.clone(), mask=full_mask.clone(), cu=cu_q.clone(),
                             max_q=max_q))
        n = x.shape[1] - txt_len
        mod = torch.where(full_mask[None, :, None], tr_vec[:, None], vec[:, None])
        rope = lambda y: y * cos.repeat(1, HEADS) + sin.repeat(1, HEADS)   # noqa: E731
        img, txt = x[:, :n], x[:, n:]
        a = self.attend(rope(img * self.w[0]), rope(img * self.w[1]), img * self.w[2], txt * self.w[0],
                        txt * self.w[1], txt * self.w[2], cu_q, drop, amp, curve_sel, p_remain)
        return x + a * self.w[3] * mod

    forward.__jenga_b200__ = True


class _Elementwise(torch.nn.Module):
    def __init__(self, seed):
        super().__init__()
        self.w = _vec(seed)

    def forward(self, x, *a):
        return x * self.w


class _Final(torch.nn.Module):
    def __init__(self, seed):
        super().__init__()
        self.w = _vec(seed)

    def forward(self, x, vec):
        return x * self.w + vec[:, None]


class _Transformer(torch.nn.Module):
    """The attributes and sub-modules ra_forward reads, patch size 1, C latent channels."""
    patch_size = (1, 1, 1)
    i2v_condition_type = "token_replace"
    guidance_embed = False
    text_projection = "linear"
    heads_num = HEADS

    def __init__(self, log, n_double=2, n_single=2):
        super().__init__()
        self.img_in, self.txt_in, self.vector_in = _Elementwise(1), _Elementwise(2), _Elementwise(3)
        self.final_layer = _Final(4)
        self.double_blocks = torch.nn.ModuleList([_Double(10 + 10 * i, log) for i in range(n_double)])
        self.single_blocks = torch.nn.ModuleList([_Single(100 + 10 * i, log) for i in range(n_single)])
        from jenga_b200 import gilbert
        t, h, w = GRID
        l2h, h2l = gilbert.mapping_tensors(t, h, w)
        self.curve_sel = [[l2h, h2l, gilbert.block_neighbor_mapping(t, h, w)]]
        self.linear_to_hilbert, self.hilbert_order = l2h, h2l
        self.sa_drop_rate, self.p_remain_rates, self.text_amp = DROP, P_REMAIN, AMP
        self.cnt, self.num_steps, self.start_stage, self.previous_residual = 0, 50, True, None

    def time_in(self, t):
        return t[:, None] * _vec(5) * 1e-3

    def unpatchify(self, x, tt, th, tw):
        return x.transpose(1, 2).reshape(1, C, tt, th, tw)


def _inputs():
    g = torch.Generator().manual_seed(7)
    t, h, w = GRID
    x = torch.randn(1, C, t, h, w, generator=g)
    txt = torch.randn(1, T, C, generator=g)
    mask = torch.zeros(1, T, dtype=torch.int64)
    mask[:, :VALID] = 1
    txt2 = torch.randn(1, C, generator=g)
    ang = torch.rand(t * h * w, D // 2, generator=g) * 6.2831853
    cos, sin = torch.cos(ang).repeat_interleave(2, 1), torch.sin(ang).repeat_interleave(2, 1)
    return x, torch.tensor([900.0]), txt, mask, txt2, cos, sin


def _ra_forward_single(self, x, t, text_states, text_mask, text_states_2, freqs_cos, freqs_sin):
    """jenga_hyi2v.py:53-221 in one process (batch 1, token_replace, linear text projection)"""
    _, _, tt, th, tw = x.shape
    vec = self.time_in(t)
    tr_vec = self.time_in(torch.zeros_like(t))
    vec_2 = self.vector_in(text_states_2)
    vec, tr_vec = vec + vec_2, tr_vec + vec_2
    img, txt = self.img_in(x.flatten(2).transpose(1, 2)), self.txt_in(text_states)
    T_, L = txt.shape[1], img.shape[1]
    img = img[:, self.hilbert_order]
    freqs_cos, freqs_sin = freqs_cos[self.hilbert_order], freqs_sin[self.hilbert_order]
    ff = torch.zeros_like(img[0, :, 0]).bool()
    ff[:th * tw] = 1
    ff = ff[self.hilbert_order]
    full = torch.zeros(L + T_).bool()
    full[:L] = ff
    s = int(text_mask.sum()) + L
    cu = torch.tensor([0, s, L + T_], dtype=torch.int32)
    if self.cnt in (0, 1, 2, 3, 5, 7, 10) or self.start_stage:
        self.start_stage = False
        ori = img.clone()
        for b in self.double_blocks:
            img, txt = b(img, txt, vec, cu, cu, L + T_, L + T_, (freqs_cos, freqs_sin), self.sa_drop_rate, ff,
                         "token_replace", tr_vec, th * tw, self.text_amp, self.curve_sel, self.p_remain_rates)
        xx = torch.cat((img, txt), 1)
        for b in self.single_blocks:
            xx = b(xx, vec, T_, cu, cu, L + T_, L + T_, (freqs_cos, freqs_sin), self.sa_drop_rate, full,
                   "token_replace", tr_vec, th * tw, self.text_amp, self.curve_sel, self.p_remain_rates)
        img = xx[:, :L]
        self.previous_residual = img - ori
    else:
        img += self.previous_residual
    self.cnt += 1
    img = img[:, self.linear_to_hilbert]
    return self.unpatchify(self.final_layer(img, vec), tt, th, tw)


class _SpTransformer(_Transformer):
    """img_in takes the latent [1, C, t, h, w] as the reference's PatchEmbed does"""

    def __init__(self, log):
        super().__init__(log)
        inner = self.img_in
        self.img_in = _Embed(inner)


class _Embed(torch.nn.Module):
    def __init__(self, inner):
        super().__init__()
        self.inner = inner

    def forward(self, x):
        return self.inner(x.flatten(2).transpose(1, 2))


def _worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from jenga_b200 import hyi2v_sp
        from jenga_b200.ulysses import UlyssesCarvedAttention
        log = []
        model = _SpTransformer(log)
        sp = UlyssesCarvedAttention(attn_fn=_oracle_attn, variant="hyvideo_i2v")
        assert hyi2v_sp.parallelize_i2v(model, attention=sp) is sp
        assert all(b.jenga_sp is sp and not hasattr(b, "hybrid_seq_parallel_attn")
                   for b in list(model.double_blocks) + list(model.single_blocks))
        x, t, txt, mask, txt2, cos, sin = _inputs()
        out = model(x, t, txt, mask, txt2, cos, sin)["x"]
        model.cnt = 4                                           # not in jenga_hyi2v.py's step_calc: skipped
        log_len = len(log)
        out_skip = model(x, t, txt, mask, txt2, cos, sin, return_dict=False)
        assert len(log) == log_len, "a skipped step ran a block"
        ret[rank] = dict(out=out, out_skip=out_skip, log=log)
        if world == 2:
            # L % P: 9 image tokens over 2 ranks
            model.cnt, model.start_stage = 0, True
            with pytest.raises(ValueError, match="image tokens do not split over 2 ranks"):
                model(x[:, :, :1, :3, :3], t, txt, mask, txt2, cos, sin)
            # heads % P: 3 heads over 2 ranks
            odd = _SpTransformer([])
            odd.heads_num = 3
            with pytest.raises(ValueError, match="3 attention heads do not split over 2 ranks"):
                hyi2v_sp.parallelize_i2v(odd, attention=sp)
            assert not hasattr(odd.double_blocks[0], "jenga_sp")
            # a block whose forward is not the fused one would ignore jenga_sp
            plain = _SpTransformer([])
            plain.single_blocks.append(torch.nn.Linear(2, 2))
            with pytest.raises(RuntimeError, match="Linear.forward is not the fused jenga_b200 forward"):
                hyi2v_sp.parallelize_i2v(plain, attention=sp)
            assert not hasattr(plain.double_blocks[0], "jenga_sp")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_forward_equals_single_process(world):
    mgr = mp.Manager()
    ret = mgr.dict()
    port = 29500 + (os.getpid() + 37 * world) % 2000
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)

    log = []
    model = _Transformer(log)
    x, t, txt, mask, txt2, cos, sin = _inputs()
    with torch.no_grad():
        ref = _ra_forward_single(model, x, t, txt, mask, txt2, cos, sin)
        model.cnt = 4
        ref_skip = _ra_forward_single(model, x, t, txt, mask, txt2, cos, sin)
    L = GRID[0] * GRID[1] * GRID[2]
    n = L // world
    for r in range(world):
        got = ret[r]
        assert torch.equal(got["out"], ref), r
        assert torch.equal(got["out_skip"], ref_skip), r
        assert len(got["log"]) == len(log)
        for i, (g, e) in enumerate(zip(got["log"], log)):
            sl = slice(r * n, (r + 1) * n)
            # image rows (and, for the single blocks, the replicated text rows after them)
            want = torch.cat([e["img"][:, sl], e["img"][:, L:]], 1)
            assert torch.equal(g["img"], want), (r, i)
            assert torch.equal(g["cos"], e["cos"][sl]) and torch.equal(g["sin"], e["sin"][sl]), (r, i)
            want_mask = e["mask"][sl] if e["mask"].numel() == L else torch.cat([e["mask"][sl], e["mask"][L:]])
            assert torch.equal(g["mask"].cpu(), want_mask), (r, i)
            assert g["cu"].tolist() == [0, n + VALID, n + T], (r, i)
            assert g["max_q"] == n + T
    # the single-process first-frame mask really marks the first frame, scattered by the curve
    assert int(log[0]["mask"].sum()) == GRID[1] * GRID[2] and not bool(log[0]["mask"][:GRID[1] * GRID[2]].all())


def test_degree_errors():
    from jenga_b200.hyi2v_sp import check_degree
    check_degree(115200, 24, 8)
    for P in (1, 2, 3, 4, 6, 8):
        check_degree(115200, 24, P)
    with pytest.raises(ValueError, match="24 attention heads do not split over 5 ranks"):
        check_degree(115200, 24, 5)
    with pytest.raises(ValueError, match="115201 image tokens do not split over 2 ranks"):
        check_degree(115201, 24, 2)


# ------------------------------------------------------------------------------------------------
# install(): the switch
# ------------------------------------------------------------------------------------------------
_STUB = '''
def parallelize_transformer(pipe):
    """the reference's spatial-chunk dense SP (stand-in)"""
    for block in list(pipe.transformer.double_blocks) + list(pipe.transformer.single_blocks):
        block.hybrid_seq_parallel_attn = "dense xfuser attention"
'''

_PROBE = '''
import os, sys, types, json
import torch
import torch.distributed as dist
sys.path.insert(0, {root!r})
sys.path.insert(0, {stub!r})
from jenga_b200 import install
kw = {kw}
done = install.install(flash_attn=False, gilbert=False, ulysses=False, gather=False, **kw)
import hyvideo_i2v.inference as inf
if {then_off!r}:
    install.install(flash_attn=False, gilbert=False, ulysses=False, gather=False, i2v_sp=False)
    done = []
from jenga_b200 import blocks as jb
os.environ["MASTER_ADDR"] = "127.0.0.1"
os.environ["MASTER_PORT"] = {port!r}
dist.init_process_group("gloo", rank=0, world_size=1)
class Blk(torch.nn.Module):   # stands in for a block class the fused-forward hook has patched
    def forward(self, *a):
        raise AssertionError("not called")
    forward.__jenga_b200__ = True
tr = torch.nn.Module()
tr.heads_num = 24
tr.double_blocks = torch.nn.ModuleList([Blk()])
tr.single_blocks = torch.nn.ModuleList([Blk()])
inf.parallelize_transformer(types.SimpleNamespace(transformer=tr))
blocks = list(tr.double_blocks) + list(tr.single_blocks)
print(json.dumps(dict(
    swapped=bool(getattr(inf.parallelize_transformer, "__jenga_b200__", False)),
    route="sequence-parallel I2V route" in done,
    hybrid=[getattr(b, "hybrid_seq_parallel_attn", None) for b in blocks],
    jenga_sp=[type(getattr(b, "jenga_sp", None)).__name__ for b in blocks],
    variant=[getattr(getattr(b, "jenga_sp", None), "variant", None) for b in blocks],
    instance_forward="forward" in tr.__dict__, i2v_sp_flag=jb.I2V_SP)))
dist.destroy_process_group()
'''


def _probe(tmp_path, kw, env_switch, then_off=False):
    import json
    stub = tmp_path / "stub"
    (stub / "hyvideo_i2v").mkdir(parents=True)
    (stub / "hyvideo_i2v" / "__init__.py").write_text("")
    (stub / "hyvideo_i2v" / "inference.py").write_text(_STUB)
    env = {k: v for k, v in os.environ.items() if k != "JENGA_I2V_SP"}
    if env_switch is not None:
        env["JENGA_I2V_SP"] = env_switch
    code = _PROBE.format(root=str(ROOT), stub=str(stub), kw=repr(kw), port=str(31000 + os.getpid() % 2000),
                         then_off=then_off)
    r = subprocess.run([sys.executable, "-s", "-c", code], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("kw,env_switch", [({}, None), ({}, "0"), ({"i2v_sp": False}, "1")])
def test_without_the_switch_the_reference_route_stays(tmp_path, kw, env_switch):
    got = _probe(tmp_path, kw, env_switch)
    assert not got["swapped"] and not got["route"]
    assert got["hybrid"] == ["dense xfuser attention"] * 2
    assert got["jenga_sp"] == ["NoneType"] * 2 and not got["instance_forward"]


@pytest.mark.parametrize("kw,env_switch", [({}, "1"), ({"i2v_sp": True}, None)])
def test_with_the_switch_parallelize_transformer_runs_parallelize_i2v(tmp_path, kw, env_switch):
    got = _probe(tmp_path, kw, env_switch)
    assert got["swapped"] and got["route"]
    assert got["hybrid"] == [None, None]                 # hybrid_seq_parallel_attn is never set
    # gloo has no symmetric memory: the all-ranks agreement picks the NCCL-style exchange
    assert got["jenga_sp"] == ["UlyssesCarvedAttention"] * 2 and got["variant"] == ["hyvideo_i2v"] * 2
    assert got["instance_forward"]


def test_install_without_the_switch_turns_the_route_back_off(tmp_path):
    """install(i2v_sp=True), import, then install(i2v_sp=False): the reference function is back and
    the route stays off"""
    got = _probe(tmp_path, {"i2v_sp": True}, None, then_off=True)
    assert not got["swapped"] and got["i2v_sp_flag"] is False
    assert got["hybrid"] == ["dense xfuser attention"] * 2 and got["jenga_sp"] == ["NoneType"] * 2


@pytest.mark.parametrize("text_tokens", [256, 384, 513])
def test_sharded_attention_refuses_text_lengths_other_than_four_blocks(text_tokens):
    """the Ulysses objects pass ceil(T/128) text blocks, the I2V operator always four"""
    import random
    import types
    from jenga_b200 import blocks
    blk = types.SimpleNamespace(heads_num=HEADS, jenga_sp=object())
    img = torch.zeros(1, 256, 3 * C, dtype=torch.bfloat16)
    txt = torch.zeros(1, text_tokens, 3 * C, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match=f"needs 4 text blocks \\(385..512 text tokens\\), got {text_tokens}"):
        blocks._attention_section(blk, types.SimpleNamespace(random=random), img, txt, [(None, 1e-6)] * 4,
                                  freqs_cis=None, cu_seqlens_q=None, cu_seqlens_kv=None, sa_drop_rate=0.7,
                                  txt_amp=0.0, curve_sel=[[None, None, None]], p_remain_rates=0.3, text_blocks=4,
                                  pad_ragged=True)


def test_i2v_sp_needs_the_fused_blocks():
    from jenga_b200 import install
    with pytest.raises(ValueError, match="fused_blocks"):
        install.install(flash_attn=False, gilbert=False, ulysses=False, fused_blocks=False, gather=False,
                        i2v_sp=True)
