"""The fp8 (e4m3) KV cache of GPT-2 generation and beam search: the definition of what ``kv_quantize_`` and the fp8
``decode_attention_`` (csrc/ops_decode.cu) store, evaluated with torch on the CPU or the GPU. It is the CPU / non-bf16
path of ``GPT2DoubleHeads`` with ``kv_cache_dtype="fp8_e4m3"`` and the reference the GPU tests compare the kernels
against, bit for bit.

Each cached key vector and each value vector (one (layer, row, head, position) of ``k`` or ``v``, ``Dh`` elements) is
quantized on its own:

* ``amax`` is the vector's largest ``|x|``, exact from its bf16 values;
* the scale is the power of two ``2^e`` with ``e = ilogb(amax) - 7``, so ``amax · 2^-e`` lies in [128, 256), inside
  e4m3's finite range of ±448; ``e = 0`` when ``amax = 0``. A vector with a NaN or an infinity gets the scale NaN and
  zero bytes, so every later read of it is NaN rather than silently finite;
* the stored byte of ``x`` is ``q = e4m3(x · 2^-e)``, rounded to nearest even and saturated to the finite range
  (``__nv_cvt_float_to_fp8(..., __NV_SATFINITE, __NV_E4M3)``);
* the read value is ``fl32(q) · 2^e``. It is exact: it fits in fp32, and in bf16 too unless ``amax`` is below about
  2^-117.

Storage: ``k`` / ``v`` are raw bytes, uint8 [n_layer, R, H, t_max, Dh]; ``k_scale`` / ``v_scale`` fp32
[n_layer, R, H, t_max]. Every cached position is quantized, the prompt's included: unlike HuggingFace's
``QuantizedCache`` there is no window of recent positions kept in full precision. The prefill's own causal attention
runs on the unquantized keys and values, and in a decode step the new token attends to its own key and value
unquantized; every later token sees the quantized copy.

Because the scales are powers of two, scaling commutes exactly with every fp32 product and sum. So the fp8 kernel
multiplies a key's dot product by its scale once, and folds a value's scale into its softmax weight, and still gives
the bits of the bf16 kernel run on a bf16 cache that holds the dequantized values.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

KV_CACHE_DTYPES = ("fp8_e4m3",)


def check_kv_cache_dtype(who: str, kv_cache_dtype: Optional[str]) -> Optional[str]:
    """``kv_cache_dtype`` if it is None (the model's dtype) or one of ``KV_CACHE_DTYPES``; ``ValueError`` otherwise."""
    if kv_cache_dtype is not None and kv_cache_dtype not in KV_CACHE_DTYPES:
        raise ValueError(f"{who}: kv_cache_dtype must be None or one of {KV_CACHE_DTYPES}, got {kv_cache_dtype!r}")
    return kv_cache_dtype


def quantize(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(q, scale)`` of the vectors along the last dimension of ``x`` (bf16 or any float whose values are bf16):
    ``q`` uint8 of ``x``'s shape, ``scale`` fp32 of its shape without the last dimension."""
    xd = x.double()
    amax = xd.abs().amax(-1)                          # NaN propagates through amax
    finite = torch.isfinite(amax)
    _, ex = torch.frexp(torch.where(finite & (amax > 0), amax, torch.ones_like(amax)))
    e = torch.where(finite & (amax > 0), ex.long() - 1 - 7, torch.zeros_like(ex.long()))   # ilogb(amax) - 7
    y = (xd * torch.pow(2.0, -e.double())[..., None]).float()     # exact in fp64; |y| < 256 is normal or rounds to 0
    q = y.to(torch.float8_e4m3fn).view(torch.uint8)
    q = torch.where(finite[..., None], q, torch.zeros_like(q))
    scale = torch.where(finite, torch.pow(2.0, e.double()).float(), torch.full_like(amax, float("nan")).float())
    return q, scale


def dequantize(q: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """fp32 ``fl32(q) · scale`` of bytes ``q`` and the scales of their vectors (``q``'s shape without the last
    dimension)."""
    return q.view(torch.float8_e4m3fn).float() * scale[..., None]


def store_(x: torch.Tensor, q: torch.Tensor, scale: torch.Tensor) -> None:
    """Quantize ``x`` into ``q`` (uint8, ``x``'s shape) and ``scale`` in place."""
    qx, sx = quantize(x)
    q.copy_(qx)
    scale.copy_(sx)
