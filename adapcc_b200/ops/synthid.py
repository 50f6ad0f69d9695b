"""SynthID Text watermarking for GPT-2 generation (Dathathri et al., "Scalable watermarking for identifying large
language model outputs", Nature 2024; HuggingFace's ``SynthIDTextWatermarkingConfig`` /
``SynthIDTextWatermarkLogitsProcessor``): the definition of the sampler's tournament (``ops.sample_tokens_(...,
synthid=)``, csrc/ops_synthid.cu) and of the detector's counts (``ops.synthid_count_``), which ``synthid_flags``,
``ops.sampling.reference_row`` and ``synthid_counts_reference`` evaluate in numpy, and ``detect_synthid``.

Unlike the green-list watermark (``ops/watermark.py``) this one reproduces HuggingFace's exactly, so text marked here
can be scored by HuggingFace's tools (a trained ``BayesianDetectorModel`` included) and text HuggingFace marked with a
CPU-built table can be scored here.

- config: ``ngram_len`` n in [2, 16], ``keys`` k_0..k_{m-1} (m in [1, ``SYNTHID_MAX_DEPTH``], int64 values),
  ``context_history_size`` H >= 1, ``sampling_table_seed``, ``sampling_table_size`` S in [1, 2^24] and
  ``skip_first_ngram_calls``. ``debug_mode`` is not offered.
- table: ``torch.randint(0, 2, (S,), generator=torch.Generator("cpu").manual_seed(seed))``. It equals HuggingFace's
  ``sampling_table`` only when HuggingFace builds its processor on the CPU; it builds it on the generation device,
  whose generator draws other bits. On the device it is a bitset of ceil(S / 32) uint32 words.
- hash (uint64, wrapping): ``acc(h, x) = (h + x) * 6364136223846793005 + 1`` folded left to right. The hash of a
  context c (n - 1 ids) is ``acc(1, c)``; layer l's key for candidate v is ``acc(acc(acc(1, c), [v]), [k_l])`` and
  ``g_l(c, v) = table[signed(key) mod S]`` with Python's non-negative floor-mod.
- generation (HuggingFace's processor state, derived from the tokens): at generated step t (0-based) the context is
  ``gen[t - n + 1 .. t - 1]`` with ``gen[j] = 0`` for j < 0; the prompt does not enter. With s0 = n - 1 under
  ``skip_first_ngram_calls`` (else 0), steps t < s0 are *skipped*; a step t >= s0 is *repeated* when its context hash
  equals that of a step in max(s0, t - H) .. t - 1, or is 0 while t - s0 < H (the history starts as zeros). Other
  steps are *watermarked*.
- tournament (step 6b of ``ops/sampling.py``, after the truncation filters and before the draw), on a watermarked
  step: ``p_i = w_i / Z'`` over the survivors; for each layer l, ``mass = sum_i g_l(c, i) p_i`` and ``p_i <- p_i ((1
  + g_l) - mass)``; the draw is step 7's rule and Philox word over p' instead of w. At temperature 0 (HuggingFace's
  greedy decoding) p is the softmax over every finite id, unscaled, and the token is the arg-max of p', the lowest id
  on a tie. Over random keys the tournament leaves the distribution unchanged in expectation. A skipped or repeated
  step draws exactly the token it would draw without SynthID.
- detection, of right-padded ids [B, T] with ``lengths``, per-row ``scored_from`` and an optional ``eos_token_id``:
  position j (the n-gram ``s[j - n + 1 .. j]``) is scored when n - 1 <= j < L, j >= scored_from, j precedes the row's
  first EOS (HuggingFace's ``compute_eos_token_mask``) and its context ``s[j - n + 1 .. j - 1]`` is not repeated in
  the sense of ``compute_context_repetition_mask``, whose history runs over every context of the row, scored or not.
  The counts N (positions scored) and c_l (the sum of g_l over them) are exact integers; in fp64 on the host the mean
  score is ``sum c_l / (m N)``, the weighted mean ``sum w_l c_l / (m N)`` with w linear from 10 down to 1 normalised
  to sum to m, and ``z = (sum c_l - rho m N) / sqrt(m N rho (1 - rho))`` with rho the table's share of ones,
  ``p = erfc(z / sqrt(2)) / 2`` and ``prediction = z > z_threshold``. z treats the m N g-values as independent draws;
  table collisions (two keys that fall on one entry) make that approximate.
"""
from __future__ import annotations

import dataclasses
import functools
import math
from numbers import Integral, Real
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

SYNTHID_MAX_DEPTH = 64
SYNTHID_MAX_NGRAM = 16
SYNTHID_MAX_TABLE = 2 ** 24
MULTIPLIER = 6364136223846793005


@dataclasses.dataclass(frozen=True)
class SynthIDTextWatermarkingConfig:
    """HuggingFace's ``SynthIDTextWatermarkingConfig`` fields and defaults (see the module docstring);
    ``check_synthid_args`` validates one. ``debug_mode=True`` is refused."""
    ngram_len: int
    keys: Sequence[int]
    context_history_size: int = 1024
    sampling_table_seed: int = 0
    sampling_table_size: int = 2 ** 16
    skip_first_ngram_calls: bool = False
    debug_mode: bool = False

    @property
    def depth(self) -> int:
        """m, the number of tournament layers."""
        return len(self.keys)

    @property
    def skip(self) -> int:
        """s0: the first step that can be watermarked."""
        return int(self.ngram_len) - 1 if self.skip_first_ngram_calls else 0


def is_synthid_config(config) -> bool:
    """Whether a decoder's ``watermarking_config`` asks for SynthID: a ``SynthIDTextWatermarkingConfig`` or a dict with
    ``keys`` or ``ngram_len`` (any other dict is a green-list ``WatermarkingConfig``)."""
    return isinstance(config, SynthIDTextWatermarkingConfig) or (
        isinstance(config, dict) and ("keys" in config or "ngram_len" in config))


def _int(x) -> bool:
    return isinstance(x, Integral) and not isinstance(x, bool)


def check_synthid_args(who: str, config) -> Optional[SynthIDTextWatermarkingConfig]:
    """``config`` (a ``SynthIDTextWatermarkingConfig``, a dict with its keys or None: off) validated, as a new config
    with ``keys`` a tuple of ints; ``ValueError`` naming ``who`` and the argument for an unknown or missing key, n
    outside [2, 16], m outside [1, SYNTHID_MAX_DEPTH], a key outside int64, H < 1, S outside [1, 2^24], a seed that
    ``torch.Generator.manual_seed`` refuses or ``debug_mode``."""
    if config is None:
        return None
    if isinstance(config, SynthIDTextWatermarkingConfig):
        kw = dataclasses.asdict(config)
    elif isinstance(config, dict):
        names = {f.name for f in dataclasses.fields(SynthIDTextWatermarkingConfig)}
        unknown = sorted(str(k) for k in config if k not in names)
        if unknown:
            raise ValueError(f"{who}: watermarking_config has unknown keys {unknown}; the SynthID keys are "
                             f"{sorted(names)}")
        missing = [k for k in ("ngram_len", "keys") if k not in config]
        if missing:
            raise ValueError(f"{who}: a SynthID watermarking_config needs {missing}")
        kw = dataclasses.asdict(SynthIDTextWatermarkingConfig(**config))
    else:
        raise ValueError(f"{who}: watermarking_config must be a SynthIDTextWatermarkingConfig, a dict or None, got "
                         f"{type(config).__name__}")
    n = kw["ngram_len"]
    if not _int(n) or not 2 <= int(n) <= SYNTHID_MAX_NGRAM:
        raise ValueError(f"{who}: ngram_len must be an integer in [2, {SYNTHID_MAX_NGRAM}], got {n!r}")
    keys = kw["keys"]
    if isinstance(keys, (str, bytes)) or not hasattr(keys, "__len__") or not 1 <= len(keys) <= SYNTHID_MAX_DEPTH:
        raise ValueError(f"{who}: keys must be a sequence of 1 to {SYNTHID_MAX_DEPTH} integers, got {keys!r}")
    if any(not _int(k) or not -2 ** 63 <= int(k) < 2 ** 63 for k in keys):
        raise ValueError(f"{who}: every key must be an integer in int64, got {list(keys)!r}")
    h = kw["context_history_size"]
    if not _int(h) or int(h) < 1:
        raise ValueError(f"{who}: context_history_size must be an integer >= 1, got {h!r}")
    s = kw["sampling_table_size"]
    if not _int(s) or not 1 <= int(s) <= SYNTHID_MAX_TABLE:
        raise ValueError(f"{who}: sampling_table_size must be an integer in [1, 2^24], got {s!r}")
    seed = kw["sampling_table_seed"]
    try:
        if not _int(seed):
            raise TypeError
        torch.Generator("cpu").manual_seed(int(seed))
    except (TypeError, RuntimeError, OverflowError, ValueError):
        raise ValueError(f"{who}: sampling_table_seed must be an integer torch.Generator.manual_seed accepts, got "
                         f"{seed!r}") from None
    skip = kw["skip_first_ngram_calls"]
    if not isinstance(skip, (bool, np.bool_)):
        raise ValueError(f"{who}: skip_first_ngram_calls must be a bool, got {skip!r}")
    if kw["debug_mode"] is not False:
        raise ValueError(f"{who}: debug_mode is not offered, got {kw['debug_mode']!r}")
    return SynthIDTextWatermarkingConfig(int(n), tuple(int(k) for k in keys), int(h), int(seed), int(s), bool(skip))


@functools.lru_cache(maxsize=8)
def _table(seed: int, size: int) -> np.ndarray:
    g = torch.Generator("cpu").manual_seed(seed)
    return torch.randint(0, 2, (size,), generator=g).numpy().astype(np.uint8)


def sampling_table(cfg: SynthIDTextWatermarkingConfig) -> np.ndarray:
    """The g-value table, uint8 [S] (a cached array: do not modify)."""
    return _table(int(cfg.sampling_table_seed), int(cfg.sampling_table_size))


def table_ones(cfg: SynthIDTextWatermarkingConfig) -> float:
    """rho, the table's share of ones: the null probability of g = 1."""
    return float(sampling_table(cfg).mean())


def table_words(cfg: SynthIDTextWatermarkingConfig) -> np.ndarray:
    """The table as the device's bitset: uint32 [ceil(S / 32)], entry i in bit i & 31 of word i >> 5."""
    t = sampling_table(cfg)
    pad = np.zeros(-t.size % 32, dtype=np.uint8)
    bits = np.concatenate([t, pad]).reshape(-1, 32).astype(np.uint64)
    return (bits << np.arange(32, dtype=np.uint64)).sum(1).astype(np.uint32)


_TABLES = {}


def device_table(cfg: SynthIDTextWatermarkingConfig, device) -> torch.Tensor:
    """``table_words`` as an int32 tensor on ``device``, cached per table and device (a graph keeps its pointer)."""
    key = (int(cfg.sampling_table_seed), int(cfg.sampling_table_size), str(torch.device(device)))
    t = _TABLES.get(key)
    if t is None:
        t = _TABLES[key] = torch.from_numpy(table_words(cfg).view(np.int32)).to(device)
    return t


def _u64(x) -> np.ndarray:
    """int64 ids or uint64 hashes as uint64 (two's complement)."""
    a = np.asarray(x)
    return a if a.dtype == np.uint64 else a.astype(np.int64).astype(np.uint64)


def accumulate(h, data) -> np.ndarray:
    """``acc`` folded over the last axis of ``data`` (int64 ids) from ``h`` (broadcast), in wrapping uint64."""
    h = np.array(_u64(h), copy=True)
    d = _u64(data)
    mult, one = np.uint64(MULTIPLIER), np.uint64(1)
    with np.errstate(over="ignore"):
        for i in range(d.shape[-1]):
            h = (h + d[..., i]) * mult + one
    return h


def g_values(ctx_hash, v, cfg: SynthIDTextWatermarkingConfig) -> np.ndarray:
    """uint8 [..., m]: the g-values of candidates ``v`` after contexts with hashes ``ctx_hash`` (broadcast)."""
    hv = accumulate(ctx_hash, np.asarray(v, dtype=np.int64)[..., None])
    keys = np.asarray(cfg.keys, dtype=np.int64)
    key = accumulate(hv[..., None], keys[:, None])           # [..., m]
    idx = key.astype(np.int64) % np.int64(cfg.sampling_table_size)   # Python's floor-mod
    return sampling_table(cfg)[idx]


def context_of(gen, t: int, n: int) -> np.ndarray:
    """The n - 1 ids before generated step t: ``gen[t - n + 1 .. t - 1]``, 0 before the first generated id."""
    g = np.asarray(gen, dtype=np.int64).reshape(-1)
    return np.array([g[j] if j >= 0 else 0 for j in range(t - n + 1, t)], dtype=np.int64)


def synthid_flags(gen, cfg: SynthIDTextWatermarkingConfig) -> Tuple[str, int]:
    """What generated step t = len(gen) is, for a row whose generated ids so far are ``gen``: ``("skipped" |
    "repeated" | "watermarked", context hash)``."""
    g = np.asarray(gen.cpu() if isinstance(gen, torch.Tensor) else gen, dtype=np.int64).reshape(-1)
    t, n, s0, H = g.size, cfg.ngram_len, cfg.skip, cfg.context_history_size
    hc = int(accumulate(1, context_of(g, t, n)))
    if t < s0:
        return "skipped", hc
    if hc == 0 and t - s0 < H:
        return "repeated", hc
    for j in range(max(s0, t - H), t):
        if int(accumulate(1, context_of(g, j, n))) == hc:
            return "repeated", hc
    return "watermarked", hc


def tournament(p: np.ndarray, g: np.ndarray) -> np.ndarray:
    """The layers of step 6b in fp64: ``p`` [V] (0 off the survivors), ``g`` [V, m]. Returns p'."""
    p = np.asarray(p, dtype=np.float64).copy()
    for layer in range(g.shape[1]):
        gl = g[:, layer].astype(np.float64)
        mass = float((gl * p).sum())
        p = p * ((1.0 + gl) - mass)
    return p


def row_tournament(p: np.ndarray, hc: int, cfg: SynthIDTextWatermarkingConfig) -> np.ndarray:
    """``tournament`` over the ids with p > 0 of a row whose context hash is ``hc``."""
    out = np.zeros(p.size, dtype=np.float64)
    ids = np.flatnonzero(p > 0)
    out[ids] = tournament(p[ids], g_values(np.uint64(hc), ids, cfg))
    return out


# ---- detection -------------------------------------------------------------------------------------------------------
def synthid_mask_reference(ids, lengths: Sequence[int], scored_from: Sequence[int], cfg,
                           eos_token_id: Optional[int] = None) -> Tuple[np.ndarray, np.ndarray]:
    """The detector's inputs in HuggingFace's layout: g uint8 [B, T - n + 1, m] (every n-gram) and the mask uint8
    [B, T - n + 1] of the scored ones (see the module docstring)."""
    cfg = check_synthid_args("synthid_mask_reference", cfg)
    a = np.asarray(ids.cpu() if isinstance(ids, torch.Tensor) else ids, dtype=np.int64)
    B, T = a.shape
    n, H = cfg.ngram_len, cfg.context_history_size
    nc = T - n + 1
    ctx = np.stack([a[:, i:i + n - 1] for i in range(nc)], 1) if nc > 0 else np.zeros((B, 0, n - 1), np.int64)
    hashes = accumulate(np.ones((B, nc), dtype=np.uint64), ctx)              # [B, nc]
    g = g_values(hashes, a[:, n - 1:], cfg)                                 # [B, nc, m]
    mask = np.zeros((B, nc), dtype=np.uint8)
    for b in range(B):
        L = min(max(int(lengths[b]), 0), T)
        eos = T
        if eos_token_id is not None:
            hit = np.flatnonzero(a[b] == int(eos_token_id))
            eos = int(hit[0]) if hit.size else T
        for i in range(nc):
            h = hashes[b, i]
            rep = (h == 0 and i < H) or bool((hashes[b, max(0, i - H):i] == h).any())
            j = i + n - 1
            mask[b, i] = not rep and j < L and j >= int(scored_from[b]) and j < eos
    return g.astype(np.uint8), mask


def synthid_counts_reference(ids, lengths: Sequence[int], scored_from: Sequence[int], cfg,
                             eos_token_id: Optional[int] = None) -> np.ndarray:
    """The detector's counts: int64 [B, 1 + m], (N, c_0, ..., c_{m-1}) per row."""
    g, mask = synthid_mask_reference(ids, lengths, scored_from, cfg, eos_token_id)
    N = mask.sum(1).astype(np.int64)
    c = (g.astype(np.int64) * mask[:, :, None]).sum(1)
    return np.concatenate([N[:, None], c], 1)


@dataclasses.dataclass
class SynthIDDetectorOutput:
    """Per-row detection results."""
    num_tokens_scored: np.ndarray        # int64 [B], N
    g_counts: np.ndarray                 # int64 [B, m], c_l
    mean_score: np.ndarray               # fp64 [B], nan where nothing was scored
    weighted_mean_score: np.ndarray      # fp64 [B], nan where nothing was scored
    z_score: np.ndarray                  # fp64 [B], nan where nothing was scored
    p_value: np.ndarray                  # fp64 [B], nan where nothing was scored
    prediction: np.ndarray               # bool [B]


def synthid_scores(counts, rho: float, weights=None, z_threshold: float = 3.0) -> SynthIDDetectorOutput:
    """The statistics of the counts [B, 1 + m] in fp64 (see the module docstring)."""
    counts = np.asarray(counts, dtype=np.int64)
    N, c = counts[:, 0], counts[:, 1:]
    m = c.shape[1]
    w = np.linspace(10, 1, m) if weights is None else np.asarray(weights, dtype=np.float64).reshape(-1)
    if w.size != m:
        raise ValueError(f"synthid_scores: need {m} weights, got {w.size}")
    w = w * (m / w.sum())
    nf = N.astype(np.float64)
    tot = c.sum(1).astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = np.where(N > 0, tot / (m * nf), np.nan)
        wmean = np.where(N > 0, (c.astype(np.float64) * w).sum(1) / (m * nf), np.nan)
        z = np.where(N > 0, (tot - rho * m * nf) / np.sqrt(m * nf * rho * (1 - rho)), np.nan)
    p = np.array([0.5 * math.erfc(x / math.sqrt(2)) if math.isfinite(x) else math.nan for x in z], dtype=np.float64)
    return SynthIDDetectorOutput(N, c, mean, wmean, z, p, np.where(np.isfinite(z), z > z_threshold, False))


def _detect_args(who, input_ids, config, lengths, scored_from, eos_token_id):
    cfg = check_synthid_args(who, config)
    if cfg is None:
        raise ValueError(f"{who}: config must be a SynthIDTextWatermarkingConfig or a dict, got None")
    if not isinstance(input_ids, torch.Tensor):
        input_ids = torch.as_tensor(np.asarray(input_ids, dtype=np.int64))
    if input_ids.dim() != 2 or input_ids.dtype.is_floating_point or input_ids.dtype == torch.bool:
        raise ValueError(f"{who}: input_ids must be an integer [B, T] tensor, got {input_ids.dtype} "
                         f"{tuple(input_ids.shape)}")
    B, T = input_ids.shape
    if T < cfg.ngram_len:
        raise ValueError(f"{who}: need at least ngram_len = {cfg.ngram_len} columns, got {T}")
    lengths = [T] * B if lengths is None else [int(x) for x in lengths]
    if len(lengths) != B or any(not 0 <= x <= T for x in lengths):
        raise ValueError(f"{who}: need {B} lengths in [0, {T}], got {lengths}")
    scored_from = 0 if scored_from is None else scored_from
    starts = [scored_from] * B if isinstance(scored_from, Integral) else list(scored_from)
    if len(starts) != B or any(not _int(x) or x < 0 for x in starts):
        raise ValueError(f"{who}: scored_from must be an integer >= 0 or {B} of them, got {scored_from!r}")
    if eos_token_id is not None and (not _int(eos_token_id) or eos_token_id < 0):
        raise ValueError(f"{who}: eos_token_id must be None or an integer >= 0, got {eos_token_id!r}")
    return cfg, input_ids, lengths, [int(x) for x in starts]


def synthid_g_values(input_ids, config, lengths=None, scored_from=None,
                     eos_token_id: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """HuggingFace's detector inputs for the rows of ``input_ids`` [B, T]: g uint8 [B, T - n + 1, m] (every n-gram)
    and the combined mask uint8 [B, T - n + 1] (1: scored), on the inputs' device; with every length T, no
    ``scored_from`` and HuggingFace's EOS, the mask is its ``context_repetition_mask * eos_token_mask[:, n - 1:]``, so
    a trained ``BayesianDetectorModel`` can take both directly. Computed by ``ops.synthid_count_`` for CUDA inputs,
    by ``synthid_mask_reference`` otherwise."""
    who = "synthid_g_values"
    cfg, ids, lengths, starts = _detect_args(who, input_ids, config, lengths, scored_from, eos_token_id)
    if ids.is_cuda:
        from . import synthid_count_

        i32 = dict(dtype=torch.int32, device=ids.device)
        _, g, mask = synthid_count_(ids.to(torch.int32).contiguous(), torch.tensor(lengths, **i32),
                                    torch.tensor(starts, **i32), cfg, eos_token_id, with_g_values=True)
        return g, mask
    g, mask = synthid_mask_reference(ids, lengths, starts, cfg, eos_token_id)
    return torch.from_numpy(g), torch.from_numpy(mask)


def detect_synthid(input_ids, config, lengths=None, scored_from=None, eos_token_id: Optional[int] = None,
                   weights=None, z_threshold: float = 3.0) -> SynthIDDetectorOutput:
    """Scores the rows of ``input_ids`` [B, T] (right-padded to ``lengths``, default T) for the SynthID watermark of
    ``config``: ``scored_from`` (an int or B ints, default 0) is each row's first scored position, so a prompt can be
    passed as context; ``eos_token_id`` ends a row's scored region at its first EOS; ``weights`` (m values, default
    linear from 10 to 1) weight the layers of the weighted mean score. Counts on the device (``ops.synthid_count_``)
    for CUDA inputs, with ``synthid_counts_reference`` otherwise; the statistics in fp64 (see the module docstring)."""
    who = "detect_synthid"
    cfg, ids, lengths, starts = _detect_args(who, input_ids, config, lengths, scored_from, eos_token_id)
    if isinstance(z_threshold, bool) or not isinstance(z_threshold, Real) or not math.isfinite(z_threshold):
        raise ValueError(f"{who}: z_threshold must be a finite number, got {z_threshold!r}")
    if ids.is_cuda:
        from . import synthid_count_

        i32 = dict(dtype=torch.int32, device=ids.device)
        counts = synthid_count_(ids.to(torch.int32).contiguous(), torch.tensor(lengths, **i32),
                                torch.tensor(starts, **i32), cfg, eos_token_id)
        counts = counts.cpu().numpy().astype(np.int64)
    else:
        counts = synthid_counts_reference(ids, lengths, starts, cfg, eos_token_id)
    return synthid_scores(counts, table_ones(cfg), weights, float(z_threshold))
