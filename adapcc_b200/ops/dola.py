"""DoLa layer-contrast decoding for GPT-2 generation (Chuang et al. 2023, "DoLa: Decoding by Contrasting Layers Improves
Factuality in Large Language Models"; HuggingFace's ``dola_layers``): the candidate layers, the argument checks of
``generate(dola_layers=)`` and the definition of ``dola_contrast_`` (csrc/ops_dola.cu) in fp64, which the CPU /
non-bf16 path of ``GPT2DoubleHeads.generate`` evaluates and the GPU tests compare the kernel against (DESIGN.md §4a).

With N = ``n_layer``, hidden state 0 is the embedding sum, hidden state i (1 <= i < N) the residual stream entering
block i (block i - 1's output, no LayerNorm) and hidden state N the final LayerNorm's output. For each row, f are the
logits of hidden state N and q_j those of hidden state C_j through the same tied head, over the first ``vocab``
columns. With lf = log_softmax(f), lq_j = log_softmax(q_j) and M = (exp lf + exp lq_j) / 2:

    KL1_j = mean_i M_i (log M_i - lf_i),   KL2_j = mean_i M_i (log M_i - lq_j,i),   JS_j = (KL1_j + KL2_j) / 2

(a term with M_i = 0 is 0). c is C_0 for one candidate, else the first j with the largest JS_j. With
thr = fl32(max_i lf_i + fl32(ln 0.1)) (HuggingFace's relative top filter, ``relative_top = 0.1``), the scores are
lf_i - lq_c,i where lf_i >= thr and -inf elsewhere. They replace the row's logits before the repetition controls and the
sampler. The layer is chosen per row, where HuggingFace averages JS over the batch: a row's tokens then depend on its
own prompt only, and the two agree for one row.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import numpy as np
import torch

LN_TENTH = float(np.float32(math.log(0.1)))      # fl32(ln 0.1), the kernel's constant


def dola_candidate_layers(n_layer: int, spec) -> List[int]:
    """The candidate layers C of ``dola_layers`` = ``spec`` for a model of ``n_layer`` blocks with a tied head
    (HuggingFace's rule, start layer 1): ``"low"`` is ``[1]`` when ``n_layer // 2 == 1``, else every second layer from
    1 below ``n_layer // 2`` (from 1 below 20 when ``n_layer > 40``); ``"high"`` every second layer from
    ``n_layer // 2`` below ``n_layer`` (from ``n_layer - 20`` when ``n_layer > 40``); a list keeps its entries below
    ``n_layer``, in the given order. ``ValueError`` naming ``dola_layers`` for a negative or non-integer entry, an
    empty C or more than ``ops.DOLA_MAX_LAYERS`` layers."""
    from . import DOLA_MAX_LAYERS

    N = int(n_layer)
    if isinstance(spec, str):
        if spec not in ("low", "high"):
            raise ValueError(f"dola_layers must be 'low', 'high' or a list of layer indices, got {spec!r}")
        if spec == "low":
            if N > 40:
                layers = list(range(1, 20, 2))
            else:
                layers = [1] if N // 2 == 1 else list(range(1, N // 2, 2))
        else:
            layers = list(range(N - 20, N, 2)) if N > 40 else list(range(N // 2, N, 2))
    else:
        try:
            entries = list(spec)
        except TypeError:
            raise ValueError(f"dola_layers must be 'low', 'high' or a list of layer indices, got {spec!r}") from None
        for i in entries:
            if isinstance(i, (bool, np.bool_)) or not isinstance(i, (int, np.integer)) or i < 0:
                raise ValueError(f"dola_layers: every entry must be a non-negative integer, got {i!r} in {entries}")
        layers = [int(i) for i in entries if i < N]
    if not layers:
        raise ValueError(f"dola_layers: no candidate layer below n_layer = {N} in {spec!r}")
    if len(layers) > DOLA_MAX_LAYERS:
        raise ValueError(f"dola_layers: at most {DOLA_MAX_LAYERS} candidate layers, got {len(layers)} ({layers})")
    return layers


def check_dola_args(who: str, dola_layers, n_layer: int, guidance_scale: float = 1.0,
                    prompt_lookup_num_tokens: int = 0, assistant_model=None) -> Optional[List[int]]:
    """The candidate layers of ``dola_layers`` (``dola_candidate_layers``), or None when it is None (off).
    ``ValueError`` naming ``who`` and ``dola_layers`` when it is combined with ``guidance_scale != 1``,
    ``prompt_lookup_num_tokens`` or ``assistant_model``."""
    if dola_layers is None:
        return None
    if guidance_scale != 1.0 or prompt_lookup_num_tokens != 0 or assistant_model is not None:
        raise ValueError(f"{who}: dola_layers cannot be combined with guidance_scale != 1, prompt_lookup_num_tokens or "
                         f"assistant_model (got {guidance_scale}, {prompt_lookup_num_tokens}, "
                         f"{type(assistant_model).__name__})")
    try:
        return dola_candidate_layers(n_layer, dola_layers)
    except ValueError as e:
        raise ValueError(f"{who}: {e}") from None


def _log_softmax(z: np.ndarray) -> np.ndarray:
    m = z.max(axis=-1, keepdims=True)
    return z - (m + np.log(np.exp(z - m).sum(axis=-1, keepdims=True)))


def _js(lf: np.ndarray, lq: np.ndarray) -> np.ndarray:
    """JS_j [C, B] of the log-softmaxes lf [B, V] and lq [C, B, V]."""
    mid = 0.5 * (np.exp(lf)[None] + np.exp(lq))
    with np.errstate(divide="ignore", invalid="ignore"):
        lm = np.log(mid)
        t1 = np.where(mid > 0, mid * (lm - lf[None]), 0.0)
        t2 = np.where(mid > 0, mid * (lm - lq), 0.0)
    return 0.5 * (t1.mean(-1) + t2.mean(-1))


def dola_scores_reference(final, premature, vocab: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The DoLa scores in fp64: ``final`` [B, >= vocab] the final logits and ``premature`` [n_cand, B, >= vocab] the
    candidate layers' logits (fp32 values), over the first ``vocab`` columns. Returns ``(scores, chosen)``: fp64
    [B, vocab] on ``final``'s device (-inf outside the kept set) and int64 [B], the index into the candidates of each
    row's chosen layer."""
    f_t = torch.as_tensor(final)
    f = f_t.detach()[:, :vocab].to(device="cpu", dtype=torch.float32).numpy().astype(np.float64)
    q = torch.as_tensor(premature).detach()[:, :, :vocab].to(device="cpu", dtype=torch.float32).numpy()
    q = q.astype(np.float64)
    if q.ndim != 3 or q.shape[1] != f.shape[0] or q.shape[0] < 1:
        raise ValueError(f"dola_scores_reference: premature must be [n_cand, {f.shape[0]}, >= {vocab}], got "
                         f"{tuple(q.shape)}")
    lf, lq = _log_softmax(f), _log_softmax(q)                       # [B, V], [C, B, V]
    B = f.shape[0]
    if q.shape[0] == 1:
        chosen = np.zeros(B, dtype=np.int64)
    else:
        chosen = _js(lf, lq).argmax(0).astype(np.int64)              # the first maximum
    thr = np.float32(lf.max(-1) + LN_TENTH).astype(np.float64)      # fl32(max lf + fl32(ln 0.1))
    base = lq[chosen, np.arange(B)]
    scores = np.where(lf >= thr[:, None], lf - base, -np.inf)
    return torch.from_numpy(scores).to(f_t.device), torch.from_numpy(chosen)


def dola_js_reference(final, premature, vocab: int) -> torch.Tensor:
    """JS_j of every candidate and row in fp64, [n_cand, B]: the quantity the layer choice maximises."""
    f = torch.as_tensor(final).detach()[:, :vocab].to(device="cpu", dtype=torch.float32).numpy().astype(np.float64)
    q = torch.as_tensor(premature).detach()[:, :, :vocab].to(device="cpu", dtype=torch.float32).numpy()
    return torch.from_numpy(_js(_log_softmax(f), _log_softmax(q.astype(np.float64))))
