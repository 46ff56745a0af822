"""GPU parity of the bulk-async form of the HunyuanVideo prologue (csrc/prologue_bulk.cu, the default) against
the register-staged kernel (JENGA_PROLOGUE=classic): q, k, v bit-identical (same rounding chain), pooled means within the summation-order
tolerance of tests/test_prologue_gpu.py.  Grid sizes are forced with JENGA_PROLOGUE_CTAS so that small
inputs go through whole-block chunks, split left-over blocks and the ticket combine."""
import os
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / "golden"))
import synth  # noqa: E402


def _run(mode, ctas, fn):
    old = {k: os.environ.get(k) for k in ("JENGA_PROLOGUE", "JENGA_PROLOGUE_CTAS")}
    try:
        if mode:
            os.environ["JENGA_PROLOGUE"] = mode
        else:
            os.environ.pop("JENGA_PROLOGUE", None)
        if ctas:
            os.environ["JENGA_PROLOGUE_CTAS"] = str(ctas)
        else:
            os.environ.pop("JENGA_PROLOGUE_CTAS", None)
        out = fn()
        torch.cuda.synchronize()
        return out
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


CASES = [
    # B, L, T, H, dtype, weights, rope, index, ctas
    (1, 300, 77, 24, torch.bfloat16, True, True, True, 0),      # 3 blocks: only split left-over blocks (P=8)
    (1, 640, 128, 24, torch.bfloat16, True, True, True, 2),     # 6 blocks on 2 CTAs: whole-block chunks only
    (1, 700, 100, 24, torch.bfloat16, True, True, False, 3),    # 7 blocks on 3 CTAs: 2 each + 1 left-over (P=2), ragged
    (2, 333, 45, 5, torch.bfloat16, True, True, True, 4),       # odd head count, batch 2, ragged
    (1, 512, 0, 24, torch.float16, False, True, True, 3),       # fp16, no weights, no text
    (1, 384, 64, 8, torch.bfloat16, True, False, False, 0),     # no RoPE
    (1, 148 * 128 + 5 * 128 + 17, 256, 4, torch.bfloat16, True, True, True, 0),  # > 132 blocks (H100 SMs) on the real grid
]


@pytest.mark.parametrize("B,L,T,H,dt,has_w,rope,use_index,ctas", CASES)
def test_bulk_prologue_equals_classic(B, L, T, H, dt, has_w, rope, use_index, ctas):
    from jenga_b200.hyvideo import attention_prologue
    dev = "cuda"
    g = torch.Generator().manual_seed(1234 + L + H)
    img = (torch.randn((B, L, 3 * H * 128), generator=g) * 1.5).to(dt).to(dev)
    txt = (torch.randn((B, T, 3 * H * 128), generator=g) * 0.7).to(dt).to(dev) if T else None
    ws = [(1 + 0.2 * torch.randn(128, generator=g)).to(dt).to(dev) for _ in range(4)] if has_w else [None] * 4
    rows = L + 9
    ang = torch.rand((rows, 128), generator=g) * 6.28
    fc = (torch.cos(ang).to(dev), torch.sin(ang).to(dev)) if rope else None
    index = torch.randperm(rows, generator=g)[:L].to(dev) if (rope and use_index) else None
    if rope and not use_index:
        fc = (fc[0][:L].contiguous(), fc[1][:L].contiguous())

    def call():
        return attention_prologue(img, txt, H, *ws, 1e-6, fc, rope_index=index)

    q0, k0, v0, (qp0, kp0) = _run("classic", 0, call)
    q1, k1, v1, (qp1, kp1) = _run("bulk", ctas, call)
    for a, b, name in ((q0, q1, "q"), (k0, k1, "k"), (v0, v1, "v")):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), name
    for a, b, name in ((qp0, qp1, "q_pool"), (kp0, kp1, "k_pool")):
        d = (a.float() - b.float()).abs().max().item()
        assert d <= 2.0 ** -8 * a.float().abs().max().item() + 1e-6, (name, d)
        same = (a.view(torch.int16) == b.view(torch.int16)).float().mean().item()
        assert same >= 0.98, (name, same)
    # twice in a row on the same stream: the tickets of the split blocks were reset
    q2, k2, v2, (qp2, kp2) = _run("bulk", ctas, call)
    assert torch.equal(qp1.view(torch.int16), qp2.view(torch.int16)) and torch.equal(kp1.view(torch.int16), kp2.view(torch.int16))
    assert torch.equal(q1.view(torch.int16), q2.view(torch.int16))


def test_bulk_prologue_declines_unsupported_layouts():
    """More than 24 heads is outside the bulk form: the classic kernel must run and give the same answer,
    not an error.  A strided token dimension (the single-stream block's split of linear1) is inside it."""
    from jenga_b200.hyvideo import attention_prologue
    dev = "cuda"
    H = 26
    img = torch.randn((1, 256, 3 * H * 128), device=dev).bfloat16()
    q0, k0, v0, _ = _run("classic", 0, lambda: attention_prologue(img, None, H))
    q1, k1, v1, _ = _run("bulk", 0, lambda: attention_prologue(img, None, H))
    assert torch.equal(q0.view(torch.int16), q1.view(torch.int16))
    assert torch.equal(v0.view(torch.int16), v1.view(torch.int16))
    H = 24
    wide = torch.randn((1, 300, 3 * H * 128 + 512), device=dev).bfloat16()
    view = wide[:, :, :3 * H * 128]
    q0, k0, v0, (p0, _) = _run("classic", 0, lambda: attention_prologue(view, None, H))
    q1, k1, v1, (p1, _) = _run("bulk", 3, lambda: attention_prologue(view, None, H))
    assert torch.equal(q0.view(torch.int16), q1.view(torch.int16)) and torch.equal(k0.view(torch.int16), k1.view(torch.int16))
    assert torch.equal(v0.view(torch.int16), v1.view(torch.int16))
    assert (p0.float() - p1.float()).abs().max() <= 2.0 ** -8 * p0.float().abs().max() + 1e-6
