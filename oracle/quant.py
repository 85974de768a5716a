"""Oracle (test infrastructure): the int8 ``QLinear`` of the reference, restated on the CPU.

Reference: ``moshi/moshi/utils/quantize.py:13-40`` — ``QLinear.__init__`` quantises ``weight.to(float16)`` with
``bitsandbytes.functional.int8_vectorwise_quant`` (row-wise absmax: ``CB = round(127 * W / absmax_row)``,
``SCB = absmax_row``) and ``forward`` calls ``bnb.matmul(x.half(), CB, state)`` with the default threshold 0, i.e.
row-wise absmax int8 quantisation of the activations too, an int8 x int8 -> int32 product and dequantisation by
``SCA[m] * SCB[n] / 127^2``.

**Parity unpinned**: bitsandbytes (``>=0.45,<0.50``, ``moshi/pyproject.toml:9``) is not installed and not vendored, and no
reference test or fixture touches this path (SURVEY.md 8c), so this file restates the *published* algorithm; the rounding
mode of the quantiser (ties to even, like ``torch.round``) and the fp32 order of the dequantisation are this repo's
definition, and the CUDA path is checked against it bit for bit (exact integer accumulation).  Deviation from the
reference kept on purpose: activations and outputs stay bfloat16 (the reference round-trips through float16).
"""
from __future__ import annotations

import numpy as np
import torch

INV_127_SQ = np.float32(1.0) / np.float32(16129.0)


def quantize_rows(t: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """Row-wise absmax int8: ``q = round(t * (127 / absmax))`` in fp32 (ties to even), rows of zeros stay zero."""
    t = t.float()
    absmax = t.abs().amax(dim=-1)
    inv = torch.where(absmax > 0, torch.tensor(127.0, dtype=torch.float32) / absmax, torch.zeros_like(absmax))
    q = torch.round(t * inv[..., None]).clamp_(-127, 127).to(torch.int8)
    return q, absmax


def quantize_weight(w: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """``QLinear.__init__``: the weight goes through float16 before the row-wise quantiser (quantize.py:20)."""
    return quantize_rows(w.to(torch.float16).float())


# QLinear quantises its weight once, at construction (quantize.py:16-21): cache per weight tensor OBJECT so that stepping a large
# model does not re-quantise billions of weights every frame.  Keyed by id() and guarded by a weak reference (a storage address
# alone is reused by the allocator as soon as a tensor dies); clear_cache() drops everything.
_QCACHE: dict[int, tuple] = {}


def clear_cache() -> None:
    _QCACHE.clear()


def cached_quantize_weight(w: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    import weakref
    hit = _QCACHE.get(id(w))
    if hit is not None and hit[0]() is w and hit[1] == w._version:
        return hit[2]
    val = quantize_weight(w)
    key = id(w)
    _QCACHE[key] = (weakref.ref(w, lambda _r, k=key: _QCACHE.pop(k, None)), w._version, val)
    return val


def qproduct_f32(qx: torch.Tensor, sa: torch.Tensor, qw: torch.Tensor, sw: torch.Tensor) -> torch.Tensor:
    """The int8 x int8 product of quantised rows qx [M, K] (scales sa [M]) and qw [N, K] (scales sw [N]), dequantised in
    fp32: [M, N]."""
    acc = qx.double() @ qw.double().t()                       # exact integers (|acc| < 2^31)
    scale = (sa[:, None] * sw[None, :]) * torch.tensor(float(INV_127_SQ), dtype=torch.float32)
    return acc.float() * scale


def qlinear_f32(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """Dequantised product in fp32 (before the caller's bf16 rounding): [..., K] x [N, K] -> [..., N]."""
    qw, sw = cached_quantize_weight(w)
    lead = x.shape[:-1]
    qx, sa = quantize_rows(x.reshape(-1, x.shape[-1]))
    return qproduct_f32(qx, sa, qw, sw).reshape(*lead, w.shape[0])


def qlinear(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """``QLinear.forward`` with the output rounded to the activation dtype (bf16 on this path)."""
    return qlinear_f32(x, w).to(x.dtype)
