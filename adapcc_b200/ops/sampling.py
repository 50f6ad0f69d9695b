"""The sampling definition of ``sample_tokens_`` (csrc/ops_sample.cu) evaluated in fp64: the CPU / non-bf16 path of
``GPT2DoubleHeads.generate`` and the reference the GPU tests compare the kernel against.

For each row (DESIGN.md §4a):

1. while ``step < min_new`` the ids in ``suppress_ids`` are removed (set to -inf) before anything else;
2. ``temperature == 0``: the token is the arg-max over the remaining ids, the lowest index on a tie;
3. otherwise ``x_i = fl32(l_i / temperature)`` (correctly rounded);
4. top-k (0 < k < number of candidates): keep ``x_i >= tau``, tau the k-th largest value counted with multiplicity;
5. ``m`` = max of the kept values, ``e_i = exp(x_i - m)`` for kept ids, ``Z = sum e_i``;
6. top-p (p < 1): keep i iff the weight of the kept ids with a strictly larger value is ``<= p Z`` (tied values are
   kept or dropped together; the maximum always stays);
6a. the truncation filters, each over the ids kept so far (K), in HuggingFace's order, with ``Z = sum of e_i`` and
   ``p_i = e_i / Z`` recomputed over K before each, and ``H = -sum p_i log p_i = log Z - sum p_i (x_i - m)``:
   min-p (``min_p > 0``) keeps ``e_i >= min_p`` (``p_i >= min_p p_max``); typical (``typical_p < 1``) keeps
   ``d_i <= d*``, ``d_i = |-log p_i - H|`` and ``d*`` the smallest ``d_j`` whose set ``{d_i <= d_j}`` holds at least
   ``typical_p Z`` of the weight (tied deviations kept or dropped together; it may drop the maximum);
   epsilon (``epsilon_cutoff > 0``) keeps ``p_i >= epsilon_cutoff``; eta (``eta_cutoff > 0``) keeps
   ``p_i >= min(eta, sqrt(eta) exp(-H))``; epsilon and eta also keep the largest values of K (ties together), which
   matters only when no id reaches the threshold. Each scalar is rounded to fp32 first, as ``top_p`` is;
7. ``u = (w0 >> 8) 2^-24`` with ``w0`` the first word of Philox4x32-10 at counter ``(pos, 0, 0, 0)`` and key
   ``(seed mod 2^32, seed >> 32)``; the token is the smallest kept i whose prefix sum of surviving weights exceeds
   ``u Z'`` (Z' = their total), or the largest kept id if there is none;
8. a token in ``stop_ids`` ends the row: ``done`` is set and the reply gets -1 instead of the token.

Ids at -inf are never candidates; a row without a finite logit draws id 0. A row that is already done draws nothing:
its reply gets -1 and its next id is 0.
"""
from __future__ import annotations

from typing import Dict, Sequence, Tuple

import numpy as np
import torch

_M0, _M1 = 0xD2511F53, 0xCD9E8D57
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF


def philox4x32_10(counter: Sequence[int], key: Sequence[int]) -> Tuple[int, int, int, int]:
    """Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11) in integer arithmetic:
    four 32-bit counter words and two key words in, four words out."""
    c0, c1, c2, c3 = (int(c) & _MASK for c in counter)
    k0, k1 = (int(k) & _MASK for k in key)
    for _ in range(10):
        p0, p1 = _M0 * c0, _M1 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & _MASK, p1 & _MASK, ((p0 >> 32) ^ c3 ^ k1) & _MASK, p0 & _MASK
        k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
    return c0, c1, c2, c3


def uniform(seed: int, pos: int, word: int = 0) -> float:
    """``(w >> 8) * 2^-24`` (exact in fp32) for output word ``word`` of Philox4x32-10 at counter ``(pos, 0, 0, 0)``:
    word 0 is the draw of a row; rejection-sampling verification (``ops/assisted.py``) uses words 1 and 2."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return (philox4x32_10((pos, 0, 0, 0), (seed & _MASK, seed >> 32))[word] >> 8) * 2.0 ** -24


def top_filtering(logits: torch.Tensor, top_k: int = 0, top_p: float = 0.9, threshold: float = -float("inf")) -> torch.Tensor:
    """The sort-based top-k / nucleus / threshold filter of the sequential sampling loops (steps 4 and 6 of the
    definition, in the logits' own precision): logits [..., V] with the dropped entries at -inf along the last
    dimension; the input is left as it is. The nucleus step runs only for ``0 < top_p < 1``."""
    if top_k > 0:
        kth = torch.topk(logits, min(top_k, logits.shape[-1])).values[..., -1:]
        logits = logits.masked_fill(logits < kth, float("-inf"))
    if 0.0 < top_p < 1.0:
        srt, idx = torch.sort(logits, descending=True)
        drop = torch.softmax(srt, -1).cumsum(-1) > top_p
        drop = torch.cat([torch.zeros_like(drop[..., :1]), drop[..., :-1]], -1)   # keep the token that crosses top_p
        logits = logits.masked_fill(torch.zeros_like(drop).scatter(-1, idx, drop), float("-inf"))
    if threshold > -float("inf"):
        logits = logits.masked_fill(logits < threshold, float("-inf"))
    return logits


def check_filter_args(who: str, min_p: float, typical_p: float, epsilon_cutoff: float, eta_cutoff: float) -> None:
    """``ValueError`` naming the argument unless ``0 <= min_p <= 1``, ``0 < typical_p <= 1``, ``0 <= epsilon_cutoff <
    1`` and ``0 <= eta_cutoff < 1`` (each filter is off at 0, 1, 0 and 0 respectively)."""
    for name, v, ok, rng in (("min_p", min_p, lambda f: 0 <= f <= 1, "[0, 1]"),
                             ("typical_p", typical_p, lambda f: 0 < f <= 1, "(0, 1]"),
                             ("epsilon_cutoff", epsilon_cutoff, lambda f: 0 <= f < 1, "[0, 1)"),
                             ("eta_cutoff", eta_cutoff, lambda f: 0 <= f < 1, "[0, 1)")):
        try:
            f = float(v)
        except (TypeError, ValueError):
            f = float("nan")
        if not ok(f):
            raise ValueError(f"{who}: {name} must be in {rng}, got {v!r}")


def _filter(x: np.ndarray, e: np.ndarray, m: float, kept: np.ndarray, min_p: float, typical_p: float,
            epsilon_cutoff: float, eta_cutoff: float) -> Dict[str, Dict[str, object]]:
    """Step 6a on ``kept`` in place. Returns, per filter that is on, the quantity it compared (``q``, NaN outside K)
    and its threshold (``thr``); typical, epsilon and eta also give ``Z`` and ``mu`` (= sum p_i (x_i - m)) of the K
    they saw, and typical the weight ``G`` of ``{d_i <= d}`` at each distinct deviation of K in ascending order and
    ``pZ``, the weight G must reach."""
    out: Dict[str, Dict[str, object]] = {}
    mp, tp, ep, et = (float(np.float32(v)) for v in (min_p, typical_p, epsilon_cutoff, eta_cutoff))
    y = x - m
    if mp > 0:
        out["min_p"] = dict(q=np.where(kept, e, np.nan), thr=mp)
        kept &= e >= mp
    if tp < 1:
        Z = float(e[kept].sum())
        mu = float((e[kept] * y[kept]).sum()) / Z
        d = np.where(kept, np.abs(y - mu), np.nan)            # -log p_i - H = mu - (x_i - m)
        order = np.argsort(d[kept], kind="stable")
        ds = d[kept][order]
        G = np.cumsum(e[kept][order])[np.searchsorted(ds, ds, side="right") - 1]   # the weight up to each tie's end
        hit = np.flatnonzero(G >= tp * Z)
        dstar = float(ds[hit[0]] if hit.size else ds[-1])
        out["typical"] = dict(q=d, thr=dstar, G=G, pZ=tp * Z, Z=Z, mu=mu)
        kept &= d <= dstar
    for name, c in (("epsilon", ep), ("eta", et)):
        if c > 0:
            Z = float(e[kept].sum())
            p = np.where(kept, e / Z, np.nan)
            thr, mu = c, float((e[kept] * y[kept]).sum()) / Z
            if name == "eta":
                thr = min(c, np.sqrt(c) * np.exp(mu - np.log(Z)))        # exp(-H), H = log Z - mu
            out[name] = dict(q=p, thr=float(thr), Z=Z, mu=mu)
            kept &= (p >= thr) | (x == x[kept].max())
    return out


def reference_row(logits, temperature: float, top_k: int, top_p: float, seed: int, pos: int, step: int = 0,
                  min_new: int = 0, suppress_ids: Sequence[int] = (), min_p: float = 0.0, typical_p: float = 1.0,
                  epsilon_cutoff: float = 0.0, eta_cutoff: float = 0.0) -> Dict[str, object]:
    """One row of the definition (steps 1-7) in fp64. ``logits``: the row's ``vocab`` fp32 values. Returns the token
    and what it was decided from: ``kept`` (bool mask of the surviving ids), ``e`` (fp64 weights of the ids kept by
    top-k), ``Z``, ``pZ``, ``Zp`` (Z'), ``target`` (u Z'), ``cum`` (inclusive prefix sums of the surviving weights),
    ``tail`` (for each top-k survivor, the weight of the larger values: the quantity top-p compares with pZ) and
    ``filters`` (per truncation filter that is on, what it compared with which threshold: see ``_filter``)."""
    x = np.array(logits, dtype=np.float32).reshape(-1)
    if step < min_new:
        ids = np.array([i for i in suppress_ids if 0 <= i < x.size], dtype=np.int64)
        x[ids] = -np.inf
    cand = x > -np.inf
    out: Dict[str, object] = {"token": 0, "kept": cand & False}
    if not cand.any():
        return out
    if temperature == 0:
        out["token"] = int(np.argmax(np.where(cand, x, -np.inf)))
        out["kept"] = np.arange(x.size) == out["token"]
        return out
    x = (x / np.float32(temperature)).astype(np.float32)
    kept = cand.copy()
    if 0 < top_k < int(cand.sum()):
        tau = np.sort(x[cand])[::-1][top_k - 1]
        kept &= x >= tau
    xd = x.astype(np.float64)
    m = xd[kept].max()
    e = np.where(kept, np.exp(np.where(kept, xd - m, 0.0)), 0.0)
    Z = float(e.sum())
    pZ = float(np.float32(top_p)) * Z
    order = np.argsort(-xd[kept], kind="stable")
    vals = xd[kept][order]
    csum = np.cumsum(e[kept][order])
    # weight of the values strictly larger than each kept value: the sum before the first of its ties
    first = np.searchsorted(-vals, -vals, side="left")
    above = np.where(first > 0, csum[np.maximum(first - 1, 0)], 0.0)
    tail = np.full(x.size, np.nan)
    tail[np.flatnonzero(kept)[order]] = above
    if float(np.float32(top_p)) < 1.0:
        kept &= ~(tail > pZ)
    filters = _filter(xd, e, m, kept, min_p, typical_p, epsilon_cutoff, eta_cutoff)
    w = np.where(kept, e, 0.0)
    cum = np.cumsum(w)
    Zp = float(cum[-1])
    target = uniform(seed, pos) * Zp
    hit = np.flatnonzero(kept & (cum > target))
    out.update(token=int(hit[0]) if hit.size else int(np.flatnonzero(kept)[-1]), kept=kept, e=e, Z=Z, pZ=pZ, Zp=Zp,
               target=target, cum=cum, tail=tail, filters=filters)
    return out


def sample_reference(logits: torch.Tensor, vocab: int, temperature: float, top_k: int, top_p: float,
                     seeds: torch.Tensor, pos: torch.Tensor, step: int, min_new: int = 0,
                     suppress_ids: Sequence[int] = (), stop_ids: Sequence[int] = (),
                     done: torch.Tensor = None, min_p: float = 0.0, typical_p: float = 1.0,
                     epsilon_cutoff: float = 0.0,
                     eta_cutoff: float = 0.0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """``sample_tokens_`` for a batch, in fp64 on the host: ``logits`` [B, >= vocab] (fp32 values), ``seeds`` [B],
    ``pos`` [B], the scalar ``step``, ``done`` [B] (default: no row done). Returns ``(next_ids, tokens, done)``: int64
    [B] the ids fed to the next step, int64 [B] this step's reply column (-1 for stopped or finished rows), and the
    updated done flags (int32 [B])."""
    if temperature < 0 or top_k < 0 or not 0 < top_p <= 1:
        raise ValueError(f"sample_reference: need temperature >= 0, top_k >= 0 and 0 < top_p <= 1, got "
                         f"{temperature}, {top_k}, {top_p}")
    check_filter_args("sample_reference", min_p, typical_p, epsilon_cutoff, eta_cutoff)
    filters = dict(min_p=min_p, typical_p=typical_p, epsilon_cutoff=epsilon_cutoff, eta_cutoff=eta_cutoff)
    B = logits.shape[0]
    rows = logits[:, :vocab].detach().float().cpu().numpy()
    seeds, pos = seeds.cpu().tolist(), pos.cpu().tolist()
    done = torch.zeros(B, dtype=torch.int32) if done is None else done.cpu().to(torch.int32).clone()
    stop = set(int(s) for s in stop_ids)
    nxt, tok = torch.zeros(B, dtype=torch.int64), torch.full((B,), -1, dtype=torch.int64)
    for b in range(B):
        if done[b]:
            continue
        t = reference_row(rows[b], temperature, top_k, top_p, seeds[b], pos[b], step, min_new, suppress_ids,
                          **filters)["token"]
        nxt[b] = t
        if t in stop:
            done[b] = 1
        else:
            tok[b] = t
    return nxt, tok, done
