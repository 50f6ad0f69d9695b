"""Classifier-free guidance for GPT-2 generation (Sanchez et al. 2023, "Stay on Topic with Classifier-Free Guidance"):
the definition of ``guidance_mix_`` (csrc/ops_guidance.cu) in fp64, which the CPU / non-bf16 path of
``GPT2DoubleHeads.generate`` evaluates and the GPU tests compare the kernel against, and the argument checks of
``generate``'s guidance arguments.

With c the logits of a prompt row and u those of its negative prompt row (DESIGN.md §4a), over the first ``vocab``
columns:

    lc = c - logsumexp(c),   lu = u - logsumexp(u),   s = g * (lc - lu) + lu

with ``g`` the guidance scale rounded to fp32 once, in HuggingFace's order of operations
(``UnbatchedClassifierFreeGuidanceLogitsProcessor``). ``g == 1`` is off: ``generate`` then computes nothing of this.
``g == 0`` gives the negative prompt's log-probabilities; a negative ``g`` is allowed. The guided scores replace the
prompt row's logits before the repetition controls (``ops/repeats.py``) and the sampler (``ops/sampling.py``).
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np
import torch

FP32_MAX = float(np.finfo(np.float32).max)       # the kernel takes the scale as an fp32 value


def check_guidance_args(who: str, scale: float, batch: int, negative_prompt_ids: Optional[torch.Tensor],
                        negative_lengths, negative_token_type_ids: Optional[torch.Tensor],
                        token_type_ids: Optional[torch.Tensor], max_new_tokens: int,
                        n_positions: int) -> Optional[List[int]]:
    """``ValueError`` naming ``who`` unless ``scale`` is a finite number and the negative prompts fit: ``[batch, Tn]``
    ids, ``batch`` lengths in ``[1, Tn]`` (default Tn), token types of the ids' shape (only together with the prompt's
    ``token_type_ids``), and the longest negative prompt plus ``max_new_tokens`` within ``n_positions``. Returns the
    negative prompts' lengths (``[1] * batch`` for the default negative prompt, each row's last prompt token), or None
    when guidance is off (``scale == 1``)."""
    try:
        g = float(scale)
    except (TypeError, ValueError):
        g = float("nan")
    if not (math.isfinite(g) and abs(g) <= FP32_MAX):
        raise ValueError(f"{who}: guidance_scale must be a finite number (in fp32), got {scale!r}")
    if negative_prompt_ids is None:
        if negative_lengths is not None or negative_token_type_ids is not None:
            raise ValueError(f"{who}: negative_lengths and negative_token_type_ids need negative_prompt_ids")
        lengths = [1] * batch
    else:
        if negative_prompt_ids.dim() != 2 or negative_prompt_ids.shape[0] != batch or negative_prompt_ids.shape[1] < 1:
            raise ValueError(f"{who}: negative_prompt_ids must be [{batch}, Tn] with Tn >= 1, got "
                             f"{tuple(negative_prompt_ids.shape)}")
        Tn = negative_prompt_ids.shape[1]
        lengths = [Tn] * batch if negative_lengths is None else [int(x) for x in negative_lengths]
        if len(lengths) != batch or any(not 1 <= x <= Tn for x in lengths):
            raise ValueError(f"{who}: need {batch} negative_lengths in [1, {Tn}], got {lengths}")
        if negative_token_type_ids is not None:
            if token_type_ids is None:
                raise ValueError(f"{who}: negative_token_type_ids need the prompts' token_type_ids")
            if negative_token_type_ids.shape != negative_prompt_ids.shape:
                raise ValueError(f"{who}: negative_token_type_ids must have negative_prompt_ids' shape "
                                 f"{tuple(negative_prompt_ids.shape)}, got {tuple(negative_token_type_ids.shape)}")
    if max(lengths, default=0) + int(max_new_tokens) > n_positions:
        raise ValueError(f"{who}: the longest negative prompt ({max(lengths)}) plus max_new_tokens ({max_new_tokens}) "
                         f"exceeds n_positions = {n_positions}")
    return None if g == 1.0 else lengths


def guided_scores_reference(cond, uncond, vocab: int, scale: float) -> torch.Tensor:
    """The guided scores of ``cond`` and ``uncond`` [R, >= vocab] (fp32 values) in fp64: ``g * (lc - lu) + lu`` over
    the first ``vocab`` columns, ``lc`` / ``lu`` the rows' log-softmaxes and ``g`` the scale rounded to fp32. Returns an
    fp64 tensor [R, vocab] on ``cond``'s device."""
    c = torch.as_tensor(cond)
    x = c.detach()[:, :vocab].to(device="cpu", dtype=torch.float32).numpy().astype(np.float64)
    y = torch.as_tensor(uncond).detach()[:, :vocab].to(device="cpu", dtype=torch.float32).numpy().astype(np.float64)

    def log_softmax(z):
        m = z.max(axis=1, keepdims=True)
        return z - (m + np.log(np.exp(z - m).sum(axis=1, keepdims=True)))

    lc, lu = log_softmax(x), log_softmax(y)
    g = float(np.float32(scale))
    return torch.from_numpy(g * (lc - lu) + lu).to(c.device)
