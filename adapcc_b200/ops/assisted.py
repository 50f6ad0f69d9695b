"""Assisted generation (HuggingFace's ``assistant_model``): a draft model proposes up to k tokens per row and the
target verifies them in one step. This module is the CPU / non-bf16 path of ``GPT2DoubleHeads.generate(...,
assistant_model=draft, num_assistant_tokens=k)`` and the reference the GPU tests compare ``sample_slots_``,
``lookup_accept_drawn_`` and ``assist_round_`` against. It uses prompt lookup's conventions (``ops/lookup.py``): row b
has emitted ``e_b`` tokens, its last token ``x_b`` is not cached yet, ``lens[b] = len_b + e_b - 1``.

One round of a live row, with ``r_b = min(k, max_new_tokens - e_b - 1)``:

1. *Draft.* The draft's cache holds the row's sequence before ``x_b`` (its lengths are set to the target's at the start
   of every round). It consumes ``x_b, d_1, ..., d_k`` at positions ``lens[b] + j``; ``d_{j+1}`` is the draw of
   ``ops/sampling.py`` on the draft's logits at step j, with the Philox counter ``lens[b] + j + 1``, step ``e_b + j``
   (the same temperature, top-k, top-p, filters, and ``suppress_ids`` while ``e_b + j < min_new_tokens``). Drafts past
   ``r_b`` are pads (id 0). Consuming ``d_k`` too leaves the draft's cache covering every position a round can accept.
2. *Verify.* The target runs slots ``x_b, d_1 .. d_k`` at ``lens[b] + j`` with ``1 + r_b`` real slots (a done row: 0).
3. *Target draws.* ``g_j`` is the same draw on slot j's target logits: counter ``lens[b] + j + 1``, step ``e_b + j``.
4. *Accept.* Prompt lookup's rule (``ops.lookup.accept_row``): emit ``g_0 .. g_a`` while ``d_i == g_{i-1}``.

Token ``len_b + i`` of plain ``generate`` is drawn with the counter ``len_b + i`` at step i, and every emitted token
here is drawn from the same ``(seed, position, step)``: given the same per-position logits, assisted generation
returns exactly the tokens of plain ``generate``, whatever the draft. The draft changes the speed only. This is the
default, ``assistant_verification="coupled"``.

``assistant_verification="rejection"`` (temperature > 0; Leviathan et al. 2023) replaces steps 3 and 4. ``Q_j`` is
the draft's filtered distribution at step j (``e_i / Z'`` over the ids ``ops.sampling.reference_row`` keeps, 0
elsewhere) and ``P_j`` the model's at slot j, with the same scalars; ``v_j`` is Philox word 1 and ``u'_j`` word 2 at
the counter ``lens[b] + j + 1`` (``ops.sampling.uniform``), so neither depends on the word-0 draw that gave the draft.

3'. *Decide.* Draft ``d_{j+1}`` (j < r_b) is accepted iff ``v_j Q_j(d_{j+1}) < P_j(d_{j+1})`` (strict: an id with
   P = 0 never is); ``a`` is the number of leading accepts.
4'. *Emit* ``d_1 .. d_a, t`` through ``accept_row``'s stop and length rules. For a < r_b, t is the residual draw at
   slot a: with ``rho_i = max(0, P_a(i) - Q_a(i))`` and ``rho`` of ``d_{a+1}`` set to 0, the smallest i whose
   inclusive prefix of rho exceeds ``u'_a sum(rho)``, else the largest i with ``rho_i > 0``; ``g_a`` if ``sum(rho) =
   0``. For a = r_b, t is ``g_r``, the draw of slot r.

Given the per-position logits, every emitted token is then distributed as the model's filtered distribution, and
acceptance is ``sum_i min(P_i, Q_i)``; the tokens depend on the draft. A counter reused by a later round only feeds
draws no emitted token depended on.
"""
from __future__ import annotations

from typing import Sequence, Tuple

import numpy as np
import torch

from .sampling import reference_row, uniform

VERIFICATIONS = ("coupled", "rejection")


def check_assist_args(who: str, target, assistant, k: int, max_k: int, prompt_lookup_num_tokens: int,
                      repetition_penalty: float, no_repeat_ngram_size: int) -> None:
    """``ValueError`` naming the argument unless ``assistant`` can draft for ``target``: no prompt lookup and no
    repetition control with it, ``1 <= k <= max_k``, the same ``vocab_size``, and, when the target runs the native
    kernels (bf16 on CUDA), bf16 weights on the target's device."""
    if prompt_lookup_num_tokens:
        raise ValueError(f"{who}: assistant_model cannot be combined with prompt_lookup_num_tokens > 0, got "
                         f"{prompt_lookup_num_tokens}")
    if repetition_penalty != 1.0:
        raise ValueError(f"{who}: assistant_model cannot be combined with repetition_penalty != 1, got "
                         f"{repetition_penalty}")
    if no_repeat_ngram_size > 0:
        raise ValueError(f"{who}: assistant_model cannot be combined with no_repeat_ngram_size > 0, got "
                         f"{no_repeat_ngram_size}")
    if int(k) != k or not 1 <= int(k) <= max_k:
        raise ValueError(f"{who}: num_assistant_tokens must be an integer in [1, {max_k}], got {k}")
    cfg = getattr(assistant, "cfg", None)
    if cfg is None or not hasattr(assistant, "wte"):
        raise ValueError(f"{who}: assistant_model must be a GPT2DoubleHeads, got {type(assistant).__name__}")
    if cfg.vocab_size != target.cfg.vocab_size:
        raise ValueError(f"{who}: assistant_model's vocab_size ({cfg.vocab_size}) differs from the model's "
                         f"({target.cfg.vocab_size})")
    w, d = target.wte.weight, assistant.wte.weight
    if w.is_cuda and w.dtype == torch.bfloat16 and (d.dtype != torch.bfloat16 or d.device != w.device):
        raise ValueError(f"{who}: assistant_model must have bf16 weights on {w.device} like the model, got {d.dtype} "
                         f"on {d.device}")


def check_verification(who: str, verification: str, assistant) -> None:
    """``ValueError`` naming ``assistant_verification`` unless it is one of ``VERIFICATIONS``, and unless
    ``"rejection"`` comes with an assistant."""
    if not isinstance(verification, str) or verification not in VERIFICATIONS:
        raise ValueError(f"{who}: assistant_verification must be one of {VERIFICATIONS}, got {verification!r}")
    if verification == "rejection" and assistant is None:
        raise ValueError(f"{who}: assistant_verification='rejection' needs an assistant_model")


def filtered_probs(r) -> np.ndarray:
    """The filtered distribution fp64 [vocab] of a ``reference_row`` result ``r``: ``e_i / Z'`` on the kept ids, 0
    elsewhere (one-hot at temperature 0; all 0 for a row without a finite logit)."""
    if "e" not in r:
        return r["kept"].astype(np.float64)
    return np.where(r["kept"], r["e"], 0.0) / r["Zp"]


def spec_slot(p_logits, q_logits, d: int, temperature: float, top_k: int, top_p: float, seed: int, lens: int,
              emitted: int, j: int, min_new: int = 0, suppress_ids: Sequence[int] = (), **filters) -> dict:
    """Steps 3' and 4' for one slot: the model's fp32 ``p_logits`` [vocab] at slot j and, when slot j has a draft
    ``d`` = d_{j+1}, the draft's ``q_logits`` [vocab] at step j (else None). Returns ``g`` (the slot's draw) and, with
    a draft, ``accept``, ``t`` (the residual draw) and what they were decided from: ``P``, ``Q``, ``v``, ``rho``,
    ``cum`` (its inclusive prefix sums), ``target`` (``u' sum(rho)``) and the two ``reference_row`` results ``rp`` and
    ``rq``."""
    pos, step = lens + j + 1, emitted + j
    args = (temperature, top_k, top_p, seed, pos, step, min_new, suppress_ids)
    rp = reference_row(p_logits, *args, **filters)
    out = {"g": int(rp["token"]), "rp": rp}
    if q_logits is None:
        return out
    rq = reference_row(q_logits, *args, **filters)
    P, Q = filtered_probs(rp), filtered_probs(rq)
    v = uniform(seed, pos, 1)
    rho = np.maximum(P - Q, 0.0)
    rho[d] = 0.0
    cum = np.cumsum(rho)
    target = uniform(seed, pos, 2) * cum[-1]
    live = rho > 0
    hit = np.flatnonzero(live & (cum > target))
    t = int(hit[0]) if hit.size else int(np.flatnonzero(live)[-1]) if live.any() else out["g"]
    out.update(accept=bool(v * Q[d] < P[d]), t=t, P=P, Q=Q, v=v, rho=rho, cum=cum, target=target, rq=rq)
    return out


def spec_slots(logits: torch.Tensor, qlogits: torch.Tensor, vocab: int, temperature: float, top_k: int, top_p: float,
               seeds: Sequence[int], lens: torch.Tensor, emitted: torch.Tensor, done: torch.Tensor, nq: torch.Tensor,
               ids: torch.Tensor, min_new: int = 0, suppress_ids: Sequence[int] = (),
               **filters) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """``spec_slots_`` for a batch on the host: ``logits`` [B·(k+1), >= vocab] the model's slots, ``qlogits``
    [B, k, >= vocab] the draft's logits at each draft step, ``ids`` [B·(k+1)] the round's input (the drafts in slots
    1..k). Returns int64 ``(g, acc, last)`` [B, k+1]: each real slot's draw, whether its draft is accepted, and the
    token the round emits last if it ends there (the residual draw, or g for the last real slot); -1 / 0 where
    nothing is decided."""
    B = len(seeds)
    S = logits.shape[0] // B
    rows = logits[:, :vocab].detach().float().cpu().numpy().reshape(B, S, vocab)
    qrows = qlogits[:, :, :vocab].detach().float().cpu().numpy()
    ids = ids.cpu().reshape(B, S)
    g, last = np.full((B, S), -1, dtype=np.int64), np.full((B, S), -1, dtype=np.int64)
    acc = np.zeros((B, S), dtype=np.int64)
    for b in range(B):
        n = 0 if done[b] else int(nq[b])
        for j in range(n):
            more = j + 1 < n
            r = spec_slot(rows[b, j], qrows[b, j] if more else None, int(ids[b, j + 1]) if more else 0, temperature,
                          top_k, top_p, int(seeds[b]), int(lens[b]), int(emitted[b]), j, min_new, suppress_ids,
                          **filters)
            g[b, j] = r["g"]
            acc[b, j] = int(more and r["accept"])
            last[b, j] = r["t"] if more else r["g"]
    return g, acc, last


def draw_slot(logits, temperature: float, top_k: int, top_p: float, seed: int, lens: int, emitted: int, j: int,
              min_new: int = 0, suppress_ids: Sequence[int] = (), **filters) -> int:
    """Steps 1 and 3 for one slot: the draw of fp32 ``logits`` [vocab] for the token at sequence index ``lens + j + 1``
    (the Philox counter), step ``emitted + j``. At temperature 0 this is ``ops.lookup.greedy_token``."""
    return int(reference_row(logits, temperature, top_k, top_p, seed, lens + j + 1, emitted + j, min_new, suppress_ids,
                             **filters)["token"])


def assist_round(seq: torch.Tensor, lens: torch.Tensor, emitted: torch.Tensor, done: torch.Tensor, k: int, max_new: int,
                 n_pos: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """``assist_round_`` for a batch on the host: ``seq`` [B, t_max], ``lens``, ``emitted``, ``done`` [B]. Returns
    ``(ids, pos, nq, d_in, d_pos)``: int64 [B·(k+1)] slot 0 the last token and 0 in the draft slots, int64 [B·(k+1)]
    ``lens[b] + j`` clamped to ``t_max - 1``, int32 [B] the real slots, int64 [B] the draft's first input and int64
    [k+1, B] the draft's positions ``lens[b] + j`` clamped to ``n_pos - 1``."""
    B, t_max = seq.shape
    S = int(k) + 1
    seq, lens, emitted, done = (t.cpu() for t in (seq, lens, emitted, done))
    L = lens.long().clamp(0, t_max - 1)
    live = done == 0
    x = torch.where(live, seq.long()[torch.arange(B), L], torch.zeros(B, dtype=torch.int64))
    ids = torch.zeros(B, S, dtype=torch.int64)
    ids[:, 0] = x
    pos = (L[:, None] + torch.arange(S)).clamp(max=t_max - 1)
    r = (int(max_new) - emitted.long() - 1).clamp(0, int(k))
    nq = torch.where(live, 1 + r, torch.zeros_like(r)).to(torch.int32)
    d_pos = (L[None, :] + torch.arange(S)[:, None]).clamp(max=int(n_pos) - 1)
    return ids.reshape(-1), pos.reshape(-1), nq, x.clone(), d_pos


def draw_slots(logits: torch.Tensor, vocab: int, temperature: float, top_k: int, top_p: float, seeds: Sequence[int],
               lens: torch.Tensor, emitted: torch.Tensor, done: torch.Tensor, nq: torch.Tensor, slot0: int = 0,
               draft: bool = False, min_new: int = 0, suppress_ids: Sequence[int] = (), **filters) -> np.ndarray:
    """``sample_slots_`` for a batch on the host: ``logits`` [B·kq, >= vocab]; returns int64 [B, kq] the tokens of
    slots ``slot0 .. slot0 + kq - 1`` (-1 where nothing is drawn: a done row, or a pad slot, which for ``draft`` is a
    draft ``j + 1 >= nq[b]``; draft draws take one logits row per row)."""
    B = len(seeds)
    kq = logits.shape[0] // B
    if draft and kq != 1:
        raise ValueError(f"draw_slots: draft draws take one logits row per row (draft j + 1 depends on draft j), got "
                         f"{kq}")
    rows = logits[:, :vocab].detach().float().cpu().numpy().reshape(B, kq, vocab)
    out = np.full((B, kq), -1, dtype=np.int64)
    for b in range(B):
        for x in range(kq):
            j = slot0 + x
            if done[b] or j + int(draft) >= int(nq[b]):
                continue
            out[b, x] = draw_slot(rows[b, x], temperature, top_k, top_p, int(seeds[b]), int(lens[b]),
                                  int(emitted[b]), j, min_new, suppress_ids, **filters)
    return out
