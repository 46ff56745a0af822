"""Fused elementwise chains of the DiT blocks around the attention (SURVEY §8 f-1, first slice).

Host mirror of csrc/dense_fused.cu; each function replaces a chain of ATen kernels of
hyvideo/modules/models_mul_block_gc_ha_multigpu.py (file:line in each docstring) with one pass
that keeps the chain's rounding points under torch.autocast(bf16).  bf16 CUDA tensors only; the
callers (jenga_b200/blocks.py) fall back to the reference's own ops for anything else.

`ln_modulate` and `gate_residual` also take the token-replace form of HunyuanVideo-I2V
(hyvideo_i2v/modules/modulate_layers.py:51-56,84-95): `tr=(tr_shift, tr_scale, row_mask)` /
`tr=(tr_gate, row_mask)`, where rows whose mask entry is true take the tr_ parameters.

The HunyuanVideo chains take several samples per call (`--num-videos N`): x [B, L, C] with
modulation vectors [B, C], one row per sample, or [1, C] shared by all.  Sample b runs the same
launch as a B = 1 call, on its rows with its vector row, so its result is bit-identical to that
call; a token-replace row mask has one entry per row of a sample and is shared by all samples.

The `wan_*` functions are the chains of Wan2.1's WanAttentionBlock.forward
(wan/modules/model_mul.py:326-346), whose residual stream is fp32 and whose modulation vectors are
the fp32 rows of `e` [B, 6, C] (one row per sample, as `t` [B] makes them) or [1, 6, C] (shared by
every sample).  They take several samples the same way: sample b runs the batch-1 launch on its rows
with its vector row, so its result is bit-identical to that call."""
from __future__ import annotations

import weakref

import torch

from . import _lib
from ._lib import check, lib
from .attention import _require_cuda, _stream_ptr


def _rows2d(x: torch.Tensor):
    """[..., C] tensor whose leading dims collapse to uniformly strided rows -> (rows, row_stride)."""
    if x.stride(-1) != 1:
        raise ValueError("channel dim must be contiguous")
    C = x.shape[-1]
    rows = x.numel() // C
    if x.dim() == 1:
        return 1, C
    stride = x.stride(-2)
    # leading dims must continue the same row pitch (true for [B, L, C] slices of contiguous tensors)
    expect = stride * x.shape[-2]
    for d in range(x.dim() - 3, -1, -1):
        if x.shape[d] != 1 and x.stride(d) != expect:
            raise ValueError("rows are not uniformly strided")
        expect *= x.shape[d]
    return rows, stride


_MASK_CACHE: dict = {}


def _tr_supported(x: torch.Tensor, vecs, mask) -> bool:
    """token-replace parameters: bf16 vectors and a 1-D bool mask with one entry per row of x
    (on x's device, or on the CPU)"""
    return (all(v is not None and v.dtype == torch.bfloat16 for v in vecs) and isinstance(mask, torch.Tensor)
            and mask.dtype == torch.bool and mask.dim() == 1 and mask.numel() == x.shape[-2]
            and (mask.device == x.device or mask.device.type == "cpu"))


def _row_mask(mask: torch.Tensor, device: torch.device) -> torch.Tensor:
    """One byte per row on `device`.  A contiguous bool mask already there is used as it is; a CPU
    mask (the single-stream block's `full_first_frame_mask`, jenga_hyi2v.py:129-130, built anew on
    every forward and shared by all blocks) is copied once and cached by tensor identity and
    version, as attention.neighbour_bits caches the adjacency."""
    if mask.device == device:
        return mask if mask.dtype == torch.bool and mask.is_contiguous() else mask.to(torch.bool).contiguous()
    key = (mask.data_ptr(), mask.numel(), mask._version, str(device))
    hit = _MASK_CACHE.get(key)
    # the entry remembers WHICH tensor it was copied from: a freed mask whose address is reused by
    # the next forward's mask must not hit
    if hit is not None and hit[0]() is mask:
        return hit[1]
    dev = mask.to(device=device, dtype=torch.bool).contiguous()
    if len(_MASK_CACHE) > 8:
        _MASK_CACHE.clear()
    _MASK_CACHE[key] = (weakref.ref(mask), dev)
    return dev


def _samples(x: torch.Tensor):
    """x [..., C] -> (samples, rows per sample, row stride, sample stride), strides in elements.  A 3-D x
    with B > 1 is B samples, each launched on its own rows, so its batch stride may be any multiple of 8
    (attn[:, :L] of the double-stream block); any other x is one sample of uniformly strided rows."""
    if x.dim() == 3 and x.shape[0] > 1:
        if x.stride(-1) != 1:
            raise ValueError("channel dim must be contiguous")
        return x.shape[0], x.shape[1], x.stride(1), x.stride(0)
    rows, stride = _rows2d(x)
    return 1, rows, stride, 0


def _sample_vecs(x: torch.Tensor, vecs: dict, mask=None) -> dict:
    """The shape checks of the HunyuanVideo chains, made before any device check or launch.  Each vector
    of `vecs` (name -> tensor) holds C values, shared by every sample, or is [B, C] for x [B, L, C], one
    row per sample; a token-replace mask is 1-D with one entry per row of a sample.
    -> name -> [1, C] or [B, C] view."""
    C = x.shape[-1]
    B = x.shape[0] if x.dim() == 3 else 1
    out = {}
    for name, v in vecs.items():
        if v.numel() == C:
            out[name] = v.reshape(1, C)
        elif B > 1 and v.dim() >= 2 and v.shape[-1] == C and v.numel() == B * C:
            out[name] = v.reshape(B, C)
        else:
            raise ValueError(f"{name} must hold one value per channel ({C}), or one row of them per sample "
                             f"([{B}, {C}]); got {tuple(v.shape)}")
    if mask is not None and (mask.dim() != 1 or mask.numel() * B * C != x.numel()):
        raise ValueError("row mask must hold one entry per row")
    return out


def _vec_ptr(v: torch.Tensor, b: int) -> int:
    """address of sample b's row of a contiguous [1, C] / [B, C] vector"""
    return v.data_ptr() + (b if v.shape[0] > 1 else 0) * v.stride(0) * v.element_size()


def ln_modulate_supported(x: torch.Tensor, norm: torch.nn.Module, shift, scale, tr=None) -> bool:
    return (isinstance(norm, torch.nn.LayerNorm) and norm.weight is None and norm.bias is None
            and x.is_cuda and x.dtype == torch.bfloat16 and torch.is_autocast_enabled()
            and torch.get_autocast_dtype("cuda") == torch.bfloat16 and x.dim() == 3
            and shift is not None and scale is not None and shift.dtype == torch.bfloat16
            and scale.dtype == torch.bfloat16 and x.shape[-1] % 8 == 0 and x.shape[-1] <= 6144
            and x.stride(-1) == 1 and x.stride(-2) % 8 == 0 and (x.shape[0] == 1 or x.stride(0) % 8 == 0)
            and (tr is None or _tr_supported(x, tr[:2], tr[2])))


def ln_modulate(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, eps: float = 1e-6,
                tr=None) -> torch.Tensor:
    """`modulate(LayerNorm(x), shift=shift, scale=scale)` followed by the bf16 cast the next Linear
    applies under autocast (models_mul…:196-199,297-304,409; modulate_layers.py:31-49).
    x [B, L, C] bf16, shift/scale [B, C] or [1, C] bf16 -> [B, L, C] bf16.
    tr=(tr_shift, tr_scale, row_mask): the token-replace form (hyvideo_i2v/…/modulate_layers.py:51-56),
    row_mask a bool [L] on x's device or on the CPU."""
    return _ln_modulate(x, shift, scale, eps, tr, fp8=False)


def _ln_modulate(x, shift, scale, eps, tr, fp8):
    vecs = {"shift": shift, "scale": scale}
    if tr is not None:
        vecs.update(tr_shift=tr[0], tr_scale=tr[1])
    v = _sample_vecs(x, vecs, tr[2] if tr is not None else None)
    _require_cuda(x, *vecs.values())
    n, rows, xs, xb = _samples(x)
    C = x.shape[-1]
    v = {k: t.contiguous() for k, t in v.items()}
    m = _row_mask(tr[2], x.device) if tr is not None else None
    if fp8:
        out, a_scale = _fp8_rows(n * rows, C, x.device)
    else:
        out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    stream = _stream_ptr(x.device)
    with torch.cuda.device(x.device):
        for b in range(n):
            xp = x.data_ptr() + b * xb * x.element_size()
            op = out.data_ptr() + b * rows * C * out.element_size()
            sc, sh = _vec_ptr(v["scale"], b), _vec_ptr(v["shift"], b)
            if tr is not None:
                tsc, tsh = _vec_ptr(v["tr_scale"], b), _vec_ptr(v["tr_shift"], b)
            if fp8:
                sp = a_scale.data_ptr() + b * rows * a_scale.element_size()
                if tr is None:
                    check(lib.jenga_ln_modulate_fp8(xp, xs, sc, sh, op, C, sp, rows, C, float(eps), stream),
                          "ln_modulate_fp8")
                else:
                    check(lib.jenga_ln_modulate_tr_fp8(xp, xs, sc, sh, tsc, tsh, m.data_ptr(), op, C, sp, rows, C,
                                                       float(eps), stream), "ln_modulate_tr_fp8")
            elif tr is None:
                check(lib.jenga_ln_modulate(xp, xs, sc, sh, op, C, rows, C, float(eps), stream), "ln_modulate")
            else:
                check(lib.jenga_ln_modulate_tr(xp, xs, sc, sh, tsc, tsh, m.data_ptr(), op, C, rows, C, float(eps),
                                               stream), "ln_modulate_tr")
    return (out, a_scale) if fp8 else out


def gate_residual_supported(x, y, gate, tr=None) -> bool:
    return (x.is_cuda and x.dtype == y.dtype == torch.bfloat16 and gate is not None and gate.dtype == torch.bfloat16
            and x.shape == y.shape and x.dim() == 3 and x.shape[-1] % 8 == 0
            and x.stride(-1) == 1 and y.stride(-1) == 1 and x.stride(-2) % 8 == 0 and y.stride(-2) % 8 == 0
            and (x.shape[0] == 1 or (x.stride(0) % 8 == 0 and y.stride(0) % 8 == 0))
            and (tr is None or _tr_supported(x, tr[:1], tr[1])))


def gate_residual(x: torch.Tensor, y: torch.Tensor, gate: torch.Tensor, tr=None) -> torch.Tensor:
    """`x + apply_gate(y, gate=gate)` (models_mul…:295-315,:500; modulate_layers.py:52-68).
    x, y [B, L, C] bf16, gate [B, C] or [1, C] bf16 -> [B, L, C] bf16.
    tr=(tr_gate, row_mask): the token-replace form (hyvideo_i2v/…/modulate_layers.py:84-95)."""
    vecs = {"gate": gate}
    if tr is not None:
        vecs["tr_gate"] = tr[0]
    v = _sample_vecs(x, vecs, tr[1] if tr is not None else None)
    if y.shape != x.shape:
        raise ValueError("y must be shaped like x")
    _require_cuda(x, y, *vecs.values())
    n, rows, xs, xb = _samples(x)
    _, _, ys, yb = _samples(y)
    C = x.shape[-1]
    v = {k: t.contiguous() for k, t in v.items()}
    m = _row_mask(tr[1], x.device) if tr is not None else None
    out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    stream = _stream_ptr(x.device)
    with torch.cuda.device(x.device):
        for b in range(n):
            xp = x.data_ptr() + b * xb * x.element_size()
            yp = y.data_ptr() + b * yb * y.element_size()
            op = out.data_ptr() + b * rows * C * out.element_size()
            g = _vec_ptr(v["gate"], b)
            if tr is None:
                check(lib.jenga_gate_residual(xp, xs, yp, ys, g, op, C, rows, C, stream), "gate_residual")
            else:
                check(lib.jenga_gate_residual_tr(xp, xs, yp, ys, g, _vec_ptr(v["tr_gate"], b), m.data_ptr(), op, C,
                                                 rows, C, stream), "gate_residual_tr")
    return out


def gelu_tanh_into(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """`out[...] = nn.GELU(approximate="tanh")(x)` for strided [1, L, C] bf16 views (the MLP half of
    linear1's output into the concatenation buffer, models_mul…:413,:499)."""
    _require_cuda(x, out)
    if x.shape != out.shape or x.dtype != torch.bfloat16 or out.dtype != torch.bfloat16:
        raise ValueError("x / out must be bf16 tensors of one shape")
    rows, xs = _rows2d(x)
    _, os_ = _rows2d(out)
    with torch.cuda.device(x.device):
        check(lib.jenga_gelu_tanh(x.data_ptr(), xs, out.data_ptr(), os_, rows, x.shape[-1], _stream_ptr(x.device)),
              "gelu_tanh")
    return out


# ------------------------------------------------------------------------------------------------
# Wan2.1 (wan/modules/model_mul.py:303-346)
# ------------------------------------------------------------------------------------------------
def _autocast_bf16() -> bool:
    return torch.is_autocast_enabled() and torch.get_autocast_dtype("cuda") == torch.bfloat16


def distinct_samples(*ts: torch.Tensor) -> bool:
    """each tensor holds one sample, or a batch of samples of their own (batch stride non-zero): an
    expanded batch (stride 0) is one sample seen B times, which the fused Wan path does not take"""
    return all(t.shape[0] == 1 or t.stride(0) != 0 for t in ts)


def _wan_rows_ok(x: torch.Tensor, e: torch.Tensor) -> bool:
    """x [B, L, C] bf16 or fp32 on a GPU with 8-aligned rows and distinct, 8-aligned sample starts, e the
    fp32 modulation sum [B, 6, C] (one row per sample) or [1, 6, C] (shared by every sample)"""
    return (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype in (torch.bfloat16, torch.float32)
            and x.dim() == 3 and x.shape[-1] % 8 == 0 and x.shape[-1] <= 6144
            and x.stride(-1) == 1 and x.stride(-2) % 8 == 0
            and (x.shape[0] == 1 or (x.stride(0) % 8 == 0 and distinct_samples(x)))
            and isinstance(e, torch.Tensor) and e.is_cuda and e.dtype == torch.float32 and e.dim() == 3
            and tuple(e.shape[1:]) == (6, x.shape[-1]) and e.shape[0] in (1, x.shape[0]) and _autocast_bf16())


def _wan_layer_norm(norm, affine: bool) -> bool:
    """WanLayerNorm (model_mul.py:93-103), with fp32 weight and bias when `affine`"""
    if type(norm).__name__ != "WanLayerNorm" or not isinstance(norm, torch.nn.LayerNorm):
        return False
    if not affine:
        return norm.weight is None and norm.bias is None
    return (norm.weight is not None and norm.bias is not None and norm.weight.dtype == torch.float32
            and norm.bias.dtype == torch.float32)


def wan_ln_modulate_supported(x: torch.Tensor, norm: torch.nn.Module, e: torch.Tensor) -> bool:
    """norm1 + modulate of a Wan block: x the block input (bf16 in block 0, fp32 after)"""
    return _wan_rows_ok(x, e) and _wan_layer_norm(norm, affine=False)


def wan_residual_ln_supported(x: torch.Tensor, norm: torch.nn.Module, e: torch.Tensor, affine: bool) -> bool:
    """gate 1 + norm3 (affine) or cross residual + norm2 (not affine) of a Wan block"""
    return _wan_rows_ok(x, e) and _wan_layer_norm(norm, affine=affine)


def wan_gate_residual_supported(x: torch.Tensor, e: torch.Tensor) -> bool:
    """gate 2 of a Wan block"""
    return _wan_rows_ok(x, e)


def _wan_vecs(x: torch.Tensor, vecs: dict) -> dict:
    """_sample_vecs for the Wan chains, whose optional vectors may be None: each one holds C values,
    shared by every sample, or one row of C values per sample of x [B, L, C] (a [B, 1, C] view of
    `e6.chunk(6, dim=1)`, batch stride 6*C).  -> name -> [1, C] or [B, C] view, or None."""
    out = _sample_vecs(x, {k: v for k, v in vecs.items() if v is not None})
    return {k: out.get(k) for k in vecs}


def _wan_vec(v: torch.Tensor | None, what: str) -> torch.Tensor | None:
    """a [1, C] / [B, C] view of _wan_vecs on the GPU, fp32, with contiguous channels"""
    if v is None:
        return None
    _require_cuda(v)
    if v.dtype != torch.float32:
        raise ValueError(f"{what} must be fp32")
    return v if v.stride(-1) == 1 else v.contiguous()


def _wan_samples(x: torch.Tensor, y: torch.Tensor | None = None):
    """(samples, rows per sample, x row stride, x batch stride, y row stride, y batch stride) of the Wan
    residual stream x — [B, L, C], B samples launched one by one at 8-element aligned starts, or at B = 1
    uniformly strided rows — and of y, bf16 shaped like x (None: y strides 0)"""
    if y is not None and (y.dtype != torch.bfloat16 or y.shape != x.shape):
        raise ValueError("y must be a bf16 tensor shaped like x")
    n, rows, xs, xb = _samples(x)
    ys, yb = _samples(y)[2:] if y is not None else (0, 0)
    if n > 1 and (xb % 8 or yb % 8):
        raise ValueError("the batch stride of x and y must be a multiple of 8 elements")
    return n, rows, xs, xb, ys, yb


def _x_code(x: torch.Tensor) -> int:
    codes = {torch.bfloat16: _lib.JENGA_BF16, torch.float32: _lib.JENGA_F32}
    if x.dtype not in codes:
        raise ValueError("x must be bf16 or fp32")
    return codes[x.dtype]


def _at(t: torch.Tensor, elems: int) -> int:
    """address `elems` elements past t's start"""
    return t.data_ptr() + elems * t.element_size()


def wan_ln_modulate(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    """`norm1(x).float() * (1 + scale) + shift` (model_mul.py:331-333, WanLayerNorm :98-103) followed by
    the bf16 cast the q / k / v Linears apply under autocast.  x [B, L, C] bf16 or fp32, shift / scale
    fp32 with C values (e[0] / e[1] of a [1, 6, C] e) or one row of them per sample (of a [B, 6, C] e)
    -> [B, L, C] bf16.  Sample b runs the batch-1 launch on its rows with its vector row."""
    return _wan_ln_modulate(x, shift, scale, eps, fp8=False)


def wan_ln_modulate_fp8(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, eps: float = 1e-6):
    """`quantize_rows_fp8(wan_ln_modulate(x, shift, scale, eps))` in one pass, bit for bit; the bf16 rows
    are never written.  Returns (codes float8_e4m3fn [B*L, C], a_scale fp32 [B*L]), sample after sample."""
    return _wan_ln_modulate(x, shift, scale, eps, fp8=True)


def _fp8_rows(rows: int, C: int, device):
    return (torch.empty((rows, C), dtype=torch.float8_e4m3fn, device=device),
            torch.empty((rows,), dtype=torch.float32, device=device))


def _wan_ln_modulate(x, shift, scale, eps, fp8):
    v = _wan_vecs(x, {"scale": scale, "shift": shift})
    n, rows, xs, xb, _, _ = _wan_samples(x)
    _require_cuda(x)
    C = x.shape[-1]
    sc, sh = _wan_vec(v["scale"], "scale"), _wan_vec(v["shift"], "shift")
    if fp8:
        out, a_scale = _fp8_rows(n * rows, C, x.device)
    else:
        out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    with torch.cuda.device(x.device):
        for b in range(n):
            xp, op = _at(x, b * xb), _at(out, b * rows * C)
            if fp8:
                check(lib.jenga_wan_ln_modulate_fp8(xp, _x_code(x), xs, _vec_ptr(sc, b), _vec_ptr(sh, b), op, C,
                                                    _at(a_scale, b * rows), rows, C, float(eps),
                                                    _stream_ptr(x.device)), "wan_ln_modulate_fp8")
            else:
                check(lib.jenga_wan_ln_modulate(xp, _x_code(x), xs, _vec_ptr(sc, b), _vec_ptr(sh, b), op, C, rows,
                                                C, float(eps), _stream_ptr(x.device)), "wan_ln_modulate")
    return (out, a_scale) if fp8 else out


def wan_residual_ln(x: torch.Tensor, y: torch.Tensor, gate: torch.Tensor | None, eps: float = 1e-6, *,
                    weight: torch.Tensor | None = None, bias: torch.Tensor | None = None,
                    shift: torch.Tensor | None = None, scale: torch.Tensor | None = None):
    """r = x + y * gate (gate None: x + y), then the next LayerNorm of r as the following Linear sees it.
    weight / bias: `norm3(r)`, the affine WanLayerNorm (gate 1 + norm3, model_mul.py:334-339).
    shift / scale: `norm2(r).float() * (1 + scale) + shift` (cross residual + norm2, :339-340).
    x [B, L, C] bf16 or fp32, y bf16 like x -> (r fp32 [B, L, C], normed bf16 [B, L, C]).  gate, shift
    and scale hold C values or one row of them per sample (wan_ln_modulate); weight and bias C values."""
    return _wan_residual_ln(x, y, gate, eps, weight, bias, shift, scale, fp8=False)


def wan_residual_ln_fp8(x: torch.Tensor, y: torch.Tensor, gate: torch.Tensor | None, eps: float = 1e-6, *,
                        weight: torch.Tensor | None = None, bias: torch.Tensor | None = None,
                        shift: torch.Tensor | None = None, scale: torch.Tensor | None = None):
    """wan_residual_ln with the normed rows quantised as quantize_rows_fp8 does, in the same pass and bit
    for bit; r is the same fp32 residual.  -> (r fp32 [B, L, C], (codes float8_e4m3fn [B*L, C],
    a_scale [B*L])), sample after sample."""
    return _wan_residual_ln(x, y, gate, eps, weight, bias, shift, scale, fp8=True)


def _wan_residual_ln(x, y, gate, eps, weight, bias, shift, scale, fp8):
    affine = weight is not None
    if affine == (scale is not None) or (bias is None) != (weight is None) or (shift is None) != (scale is None):
        raise ValueError("pass either weight and bias or shift and scale")
    C = x.shape[-1]
    v = _wan_vecs(x, {"gate": gate, "scale": scale, "shift": shift})
    if affine:                                  # norm3's parameters: one row for every sample
        v.update(_wan_vecs(x[:1], {"weight": weight, "bias": bias}))
    n, rows, xs, xb, ys, yb = _wan_samples(x, y)
    _require_cuda(x, y)
    va = _wan_vec(v["weight"] if affine else v["scale"], "weight" if affine else "scale")
    vb = _wan_vec(v["bias"] if affine else v["shift"], "bias" if affine else "shift")
    g = _wan_vec(v["gate"], "gate")
    res = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    if fp8:
        out, a_scale = _fp8_rows(n * rows, C, x.device)
    else:
        out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    with torch.cuda.device(x.device):
        for b in range(n):
            xp, yp, rp, op = _at(x, b * xb), _at(y, b * yb), _at(res, b * rows * C), _at(out, b * rows * C)
            gp = _vec_ptr(g, b) if g is not None else None
            if fp8:
                check(lib.jenga_wan_residual_ln_fp8(xp, _x_code(x), xs, yp, ys, gp, rp, C, _vec_ptr(va, b),
                                                    _vec_ptr(vb, b), int(affine), op, C, _at(a_scale, b * rows),
                                                    rows, C, float(eps), _stream_ptr(x.device)),
                      "wan_residual_ln_fp8")
            else:
                check(lib.jenga_wan_residual_ln(xp, _x_code(x), xs, yp, ys, gp, rp, C, _vec_ptr(va, b),
                                                _vec_ptr(vb, b), int(affine), op, C, rows, C, float(eps),
                                                _stream_ptr(x.device)), "wan_residual_ln")
    return (res, (out, a_scale)) if fp8 else (res, out)


def wan_gate_residual(x: torch.Tensor, y: torch.Tensor, gate: torch.Tensor) -> torch.Tensor:
    """`x + y * gate` under autocast(float32) (gate 2, model_mul.py:341-342): x [B, L, C] bf16 or fp32,
    y bf16 like x, gate fp32 with C values (e[5]) or one row of them per sample -> fp32 [B, L, C]."""
    v = _wan_vecs(x, {"gate": gate})
    n, rows, xs, xb, ys, yb = _wan_samples(x, y)
    _require_cuda(x, y)
    C = x.shape[-1]
    g = _wan_vec(v["gate"], "gate")
    out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        for b in range(n):
            check(lib.jenga_wan_gate_residual(_at(x, b * xb), _x_code(x), xs, _at(y, b * yb), ys, _vec_ptr(g, b),
                                              _at(out, b * rows * C), C, rows, C, _stream_ptr(x.device)),
                  "wan_gate_residual")
    return out


# ------------------------------------------------------------------------------------------------
# Opt-in FP8 Linears (csrc/linear_fp8.cu): `jenga_b200.dense.LINEAR_FP8 = True` or JENGA_LINEAR_FP8=1.
# W8A8 e4m3 with one scale per activation row and per weight output channel (or per tensor for the
# reference's --use-fp8 checkpoints); fp32 accumulation.  Its own tolerance row (tests/test_linear_fp8_gpu.py).
# ------------------------------------------------------------------------------------------------
import os as _os

LINEAR_FP8: bool = _os.environ.get("JENGA_LINEAR_FP8", "0") == "1"
# (weight kind, K, N) of the block Linears the switch routes: only those where quantisation + FP8 GEMM
# measured faster than the call it replaces (bench_linear_fp8.py; kind "bf16" against bf16 F.linear,
# "fp8_ref" against the reference's --use-fp8 forward, "fp32" against Wan's producer + autocast module
# call, weight cast included).  On an H100 80GB at 700 W none of the six HunyuanVideo image-row shapes did,
# and of the Wan shapes only Wan-14B's ffn.2, 13 824 -> 5120, fed by gelu_tanh_fp8 (README, "Opt-in FP8
# Linears").
FP8_ROUTED: frozenset = frozenset({("fp32", 13824, 5120)})


def linear_fp8_shape_ok(k: int, n: int) -> bool:
    """the GEMM's shape rules: K % 16 == 0 and N % 8 == 0 (any M)"""
    return k > 0 and n > 0 and k % 16 == 0 and n % 8 == 0


def quantize_rows_fp8(x: torch.Tensor):
    """x [..., K] bf16 (uniformly strided rows, or [B, L, K] with any batch stride) -> (codes
    float8_e4m3fn [rows, K], scale fp32 [rows]): scale = amax(row) / 448 (1 for a zero row),
    codes = e4m3_rn_satfinite(x / scale)."""
    _require_cuda(x)
    if x.dtype != torch.bfloat16:
        raise ValueError("x must be bf16")
    n, rows, xs, xb = _samples(x)
    if n > 1 and xb % 8:
        raise ValueError("batch stride must be a multiple of 8 elements")
    K = x.shape[-1]
    out = torch.empty((n * rows, K), dtype=torch.float8_e4m3fn, device=x.device)
    scale = torch.empty((n * rows,), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        for b in range(n):
            check(lib.jenga_quantize_rows_fp8(x.data_ptr() + b * xb * x.element_size(), xs, rows, K,
                                              out.data_ptr() + b * rows * K, K,
                                              scale.data_ptr() + b * rows * scale.element_size(),
                                              _stream_ptr(x.device)), "quantize_rows_fp8")
    return out, scale


def ln_modulate_fp8(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, eps: float = 1e-6, tr=None):
    """`quantize_rows_fp8(ln_modulate(x, shift, scale, eps, tr))` in one pass, bit for bit; the bf16 rows
    are never written.  Returns (codes float8_e4m3fn [B*L, C], a_scale fp32 [B*L]), sample after sample."""
    return _ln_modulate(x, shift, scale, eps, tr, fp8=True)


def gelu_tanh_fp8(x: torch.Tensor):
    """`quantize_rows_fp8(nn.GELU(approximate="tanh")(x))` in one pass, bit for bit (gelu_tanh_into's
    arithmetic); the bf16 rows are never written.  x [..., C] bf16 with uniformly strided rows, C <= 16384
    (Wan's ffn.0 output) -> (codes float8_e4m3fn [rows, C], a_scale fp32 [rows])."""
    _require_cuda(x)
    if x.dtype != torch.bfloat16:
        raise ValueError("x must be bf16")
    rows, xs = _rows2d(x)
    C = x.shape[-1]
    out, a_scale = _fp8_rows(rows, C, x.device)
    with torch.cuda.device(x.device):
        check(lib.jenga_gelu_tanh_fp8(x.data_ptr(), xs, out.data_ptr(), C, a_scale.data_ptr(), rows, C,
                                      _stream_ptr(x.device)), "gelu_tanh_fp8")
    return out, a_scale


def linear_fp8(x8: torch.Tensor, a_scale: torch.Tensor, w8: torch.Tensor, w_scale: torch.Tensor,
               bias: torch.Tensor | None = None) -> torch.Tensor:
    """bf16( (x8 . w8^T) * a_scale[m] * w_scale[n] + bias[n] ), fp32 accumulation.
    x8 e4m3 [M, K] (rows may be strided), a_scale fp32 [M], w8 e4m3 [N, K] contiguous, w_scale fp32 [N]
    or one value (per tensor), bias bf16 / fp32 [N] or None -> bf16 [M, N]."""
    _require_cuda(x8, a_scale, w8, w_scale)
    if x8.dtype != torch.float8_e4m3fn or w8.dtype != torch.float8_e4m3fn:
        raise ValueError("x8 / w8 must be float8_e4m3fn")
    if a_scale.dtype != torch.float32 or w_scale.dtype != torch.float32:
        raise ValueError("scales must be fp32")
    if x8.dim() != 2 or w8.dim() != 2 or x8.stride(-1) != 1 or not w8.is_contiguous():
        raise ValueError("x8 must be [M, K] with contiguous rows and w8 a contiguous [N, K]")
    M, K = x8.shape
    N = w8.shape[0]
    if w8.shape[1] != K or a_scale.numel() != M or w_scale.numel() not in (1, N):
        raise ValueError("shape mismatch")
    a_scale, w_scale = a_scale.contiguous(), w_scale.contiguous()
    codes = {torch.bfloat16: _lib.JENGA_BF16, torch.float32: _lib.JENGA_F32}
    if bias is not None:
        _require_cuda(bias)
        if bias.dtype not in codes or bias.numel() != N:
            raise ValueError("bias must be bf16 or fp32 with N values")
        bias = bias.contiguous()
    out = torch.empty((M, N), dtype=torch.bfloat16, device=x8.device)
    args = _lib.JengaLinearFp8Args(
        a=x8.data_ptr(), a_stride=x8.stride(0), a_scale=a_scale.data_ptr(), w=w8.data_ptr(),
        w_scale=w_scale.data_ptr(), w_scale_stride=1 if w_scale.numel() == N and N > 1 else 0,
        bias=bias.data_ptr() if bias is not None else None,
        bias_dtype=codes[bias.dtype] if bias is not None else _lib.JENGA_BF16,
        out=out.data_ptr(), out_stride=N, m=M, n=N, k=K)
    with torch.cuda.device(x8.device):
        check(lib.jenga_linear_fp8(_lib.C.byref(args), _stream_ptr(x8.device)), "linear_fp8")
    return out


def fp8_weight_kind(layer: torch.nn.Module) -> str:
    """the FP8_ROUTED kind of a layer fp8_weight takes: "fp8_ref" for a --use-fp8 layer, "fp32" for an
    fp32 weight (Wan2.1's Linears), else "bf16"; HunyuanVideo layers are never of kind "fp32"
    """
    dt = layer.weight.dtype
    return "fp8_ref" if dt == torch.float8_e4m3fn else "fp32" if dt == torch.float32 else "bf16"


def fp8_weight(layer: torch.nn.Module):
    """(w8 e4m3 [N, K], w_scale fp32, bias) of an nn.Linear, or None when the layer is not one the FP8
    path takes.  A bf16 weight is quantised once per output channel (w_scale[n] = amax / 448) and the
    result is cached on the module, keyed on the weight's data_ptr and _version (one extra byte per
    parameter).  An fp32 weight (Wan2.1 keeps fp32 parameters) is first rounded to bf16, the operand
    autocast hands cuBLAS, then quantised and cached the same way.  A reference --use-fp8 layer (e4m3
    weight and `fp8_scale`, hyvideo/modules/fp8_optimization.py:convert_fp8_linear) is used as it is with
    the per-tensor scale float(fp8_scale.to(bf16)) that fp8_activation_dequant multiplies by."""
    w = getattr(layer, "weight", None)
    if not isinstance(w, torch.Tensor) or not w.is_cuda or w.dim() != 2 or not w.is_contiguous():
        return None
    s = getattr(layer, "fp8_scale", None)
    fp8_ref = w.dtype == torch.float8_e4m3fn and isinstance(s, torch.Tensor) and s.numel() == 1
    plain = (type(layer) is torch.nn.Linear and w.dtype in (torch.bfloat16, torch.float32)
             and "forward" not in layer.__dict__)
    if not (fp8_ref or plain) or layer._forward_hooks or layer._forward_pre_hooks:
        return None
    if not linear_fp8_shape_ok(w.shape[1], w.shape[0]):
        return None
    b = getattr(layer, "bias", None)
    if b is not None and (not b.is_cuda or b.dtype not in (torch.bfloat16, torch.float32)):
        return None
    if fp8_ref:
        key = ("ref", w.data_ptr(), w._version, s.data_ptr(), s._version)
    else:
        key = (fp8_weight_kind(layer), w.data_ptr(), w._version)
    hit = layer.__dict__.get("_jenga_fp8")
    if hit is not None and hit[0] == key:
        return hit[1], hit[2], b
    with torch.no_grad():
        if fp8_ref:
            w8 = w
            w_scale = torch.tensor([float(s.to(torch.bfloat16))], dtype=torch.float32,
                                   device=w.device)
        else:
            w8, w_scale = quantize_rows_fp8(w.to(torch.bfloat16))
    layer.__dict__["_jenga_fp8"] = (key, w8, w_scale)
    return w8, w_scale, b
