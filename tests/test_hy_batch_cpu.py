"""Several samples per call on the HunyuanVideo dense chains, CPU side: the shape rules of the
modulation vectors and the token-replace mask are checked before any device check or launch.  A
vector is [B, C] (one row per sample) or holds C values (shared by every sample); anything else is a
ValueError.  Well-shaped CPU arguments get past the shape checks and stop at the device check
(JengaError: there is no CPU path)."""
import pytest
import torch

from jenga_b200 import dense as DN
from jenga_b200._lib import JengaError

B, L, C = 3, 16, 64


def _x(b=B):
    return torch.zeros(b, L, C, dtype=torch.bfloat16)


def _v(*shape):
    return torch.zeros(*shape, dtype=torch.bfloat16)


def _calls(x, v, mask=None):
    """every HunyuanVideo chain with `v` as each of its vectors in turn, the others well-shaped"""
    ok = _v(x.shape[0], C)
    m = torch.zeros(L, dtype=torch.bool) if mask is None else mask
    return [
        lambda: DN.ln_modulate(x, v, ok),
        lambda: DN.ln_modulate(x, ok, v),
        lambda: DN.ln_modulate(x, ok, ok, tr=(v, ok, m)),
        lambda: DN.ln_modulate(x, ok, ok, tr=(ok, v, m)),
        lambda: DN.ln_modulate_fp8(x, v, ok),
        lambda: DN.ln_modulate_fp8(x, ok, ok, tr=(ok, v, m)),
        lambda: DN.gate_residual(x, x, v),
        lambda: DN.gate_residual(x, x, ok, tr=(v, m)),
    ]


@pytest.mark.parametrize("shape", [(B, C), (1, C), (C,), (B, 1, C)])
def test_per_sample_and_shared_vectors_pass_the_shape_checks(shape):
    for call in _calls(_x(), _v(*shape)):
        with pytest.raises(JengaError, match="no CPU path"):
            call()


@pytest.mark.parametrize("shape", [(B - 1, C), (B + 1, C), (B, C // 2), (1, B * C), (B * C,), (B, C + 8)])
def test_mismatched_vectors_raise_value_error(shape):
    for call in _calls(_x(), _v(*shape)):
        with pytest.raises(ValueError, match="one value per channel"):
            call()


def test_batch_one_takes_c_values_only():
    """at B = 1 the rule is the one the chains always had: C values, in any shape"""
    for call in _calls(_x(1), _v(2, C)):
        with pytest.raises(ValueError, match="one value per channel"):
            call()
    for call in _calls(_x(1), _v(1, 1, C)):
        with pytest.raises(JengaError):
            call()


@pytest.mark.parametrize("rows", [B * L, L - 1, L + 1])
def test_token_replace_mask_has_one_entry_per_row_of_a_sample(rows):
    """the first-frame mask covers one sample's rows and is shared by all samples"""
    x, ok = _x(), _v(B, C)
    m = torch.zeros(rows, dtype=torch.bool)
    for call in (lambda: DN.ln_modulate(x, ok, ok, tr=(ok, ok, m)),
                 lambda: DN.ln_modulate_fp8(x, ok, ok, tr=(ok, ok, m)),
                 lambda: DN.gate_residual(x, x, ok, tr=(ok, m))):
        with pytest.raises(ValueError, match="one entry per row"):
            call()


def test_gate_residual_needs_y_shaped_like_x():
    x, ok = _x(), _v(B, C)
    with pytest.raises(ValueError, match="shaped like x"):
        DN.gate_residual(x, x[:, 1:], ok)


def test_samples_split_a_batch_with_any_batch_stride():
    """B > 1 is launched sample by sample, so a batch stride that does not continue the row pitch
    (attn[:, :L] of the double-stream block, whose rows also hold the text) is taken; B = 1 keeps the
    single launch over uniformly strided rows"""
    full = torch.zeros(B, L + 8, 3 * C, dtype=torch.bfloat16)
    img = full[:, :L, :C]
    assert DN._samples(img) == (B, L, 3 * C, (L + 8) * 3 * C)
    assert DN._samples(full[:1, :L, :C]) == (1, L, 3 * C, 0)
    with pytest.raises(ValueError, match="uniformly strided"):
        DN._rows2d(img)


def test_predicates_take_every_batch_size_on_the_same_conditions():
    """pure shape / dtype rules: a CPU tensor is refused at any B, and the batch size alone never is"""
    x, g = _x(), _v(B, C)
    norm = torch.nn.LayerNorm(C, elementwise_affine=False)
    assert not DN.ln_modulate_supported(x, norm, g, g)
    assert not DN.gate_residual_supported(x, x, g)
    assert DN._tr_supported(x, (g, g), torch.zeros(L, dtype=torch.bool))
    assert not DN._tr_supported(x, (g, g), torch.zeros(B * L, dtype=torch.bool))
