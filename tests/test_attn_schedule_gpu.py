"""The ordered schedule (jenga_carved_attn_fwd_sched, what attention._launch calls) changes only which
CTA runs which query block: its results must equal the unordered entry points' bit for bit."""
import pytest
import torch

from jenga_b200 import attention as A
from jenga_b200._lib import lib

pytestmark = pytest.mark.gpu

B, H, S = 2, 3, 5000            # 40 key blocks: two mask words, the last one partial
NQS, NQD = 37, 2                # sparse blocks [0, 37), dense blocks 37, 38
SEQLEN = 4500                   # device-side seqlen: sparse rows past it are zeros


def _unordered(a, x, sched, stream):
    if x is None:
        return lib.jenga_carved_attn_fwd(a, stream)
    return lib.jenga_carved_attn_fwd_qk_int8(a, x, stream)


def _inputs(dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, k, v = (torch.randn(B, S, H, 128, generator=g, device="cuda").to(dtype) for _ in range(3))
    words = 2
    bits = torch.randint(-2 ** 31, 2 ** 31 - 1, (B, H, NQS, words), generator=g, device="cuda", dtype=torch.int32)
    bits &= torch.randint(-2 ** 31, 2 ** 31 - 1, bits.shape, generator=g, device="cuda", dtype=torch.int32)
    bits[:, :, 0] = 0                                   # empty row
    for n in (1, 2, 3):                                 # rows with 1..3 live tiles
        bits[:, :, n] = 0
        bits[:, :, n, 0] = (1 << n) - 1
    bits[:, :, 4] = 0
    bits[:, :, 4, 1] = 1 << 1                           # one tile, in the second word only
    return q, k, v, bits


def _run(q, k, v, bits, lse=None, **kw):
    out = torch.zeros_like(q)
    seq = torch.tensor([SEQLEN], dtype=torch.int32, device="cuda")
    A._launch(q, k, v, bits, NQS, NQD, 128 ** -0.5, 0.431, NQS, S, S, S, out, seq, q.dtype, lse_out=lse, **kw)
    return out


def _same_bits(x, y):
    """bit for bit, NaN included (a random row whose tiles all lie past seqlen is 0/0)"""
    view = {2: torch.int16, 4: torch.int32}[x.element_size()]
    return x.dtype == y.dtype and torch.equal(x.view(view), y.view(view))


def _both(monkeypatch, fn):
    got = fn()
    torch.cuda.synchronize()
    with monkeypatch.context() as m:
        m.setattr(lib, "jenga_carved_attn_fwd_sched", _unordered)
        want = fn()
    torch.cuda.synchronize()
    return got, want


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_schedule_is_bit_identical(monkeypatch, dtype):
    q, k, v, bits = _inputs(dtype, 1)

    def fn():
        lse = torch.full((B, H, S), 7.0, device="cuda")
        return _run(q, k, v, bits, lse=lse), lse
    (o1, l1), (o0, l0) = _both(monkeypatch, fn)
    assert _same_bits(o1, o0)
    assert _same_bits(l1, l0)
    assert o1[:, SEQLEN:NQS * 128].abs().max().item() == 0          # sparse rows past seqlen
    assert o1[:, :128].abs().max().item() == 0                        # the empty row
    assert o1[:, NQS * 128:].abs().max().item() > 0                   # dense rows


def test_schedule_is_bit_identical_fp8_pv_and_qk_int8(monkeypatch):
    q, k, v, bits = _inputs(torch.bfloat16, 2)
    v8 = A.quantize_v_fp8(v)
    qk8 = A.quantize_qk_int8(q, k)
    for kw in (dict(v_fp8=v8), dict(qk_int8=qk8), dict(v_fp8=v8, qk_int8=qk8)):
        got, want = _both(monkeypatch, lambda: _run(q, k, v, bits, **kw))
        assert _same_bits(got, want), kw


def test_two_streams_each_with_its_own_workspace(monkeypatch):
    ins = [_inputs(torch.bfloat16, s) for s in (3, 4)]
    streams = [torch.cuda.Stream() for _ in ins]

    def fn():
        outs = []
        for st, x in zip(streams, ins):
            st.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(st):
                outs.append(_run(*x))
        for st in streams:
            torch.cuda.current_stream().wait_stream(st)
        return outs
    got, want = _both(monkeypatch, fn)
    for g_, w_ in zip(got, want):
        assert _same_bits(g_, w_)
