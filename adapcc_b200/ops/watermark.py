"""Green-list watermarking for GPT-2 generation (Kirchenbauer et al. 2023, "A Watermark for Large Language Models";
HuggingFace's ``watermarking_config`` / ``WatermarkLogitsProcessor`` and ``WatermarkDetector``): the definition of
``watermark_`` and ``watermark_count_`` (csrc/ops_watermark.cu), which ``watermark_reference`` and
``watermark_counts_reference`` evaluate with numpy bit for bit, the CPU / non-bf16 path of the batched decoders, and
``detect_watermark``, the detector.

A ``WatermarkingConfig`` has HuggingFace's names and defaults: ``greenlist_ratio`` γ = 0.25, ``bias`` δ = 2.0,
``hashing_key`` K = 15485863, ``seeding_scheme`` ``"lefthash"`` or ``"selfhash"`` and ``context_width`` w = 1 (at
most ``MAX_CONTEXT_WIDTH``). The decoders take one, or a dict with the same keys, as ``watermarking_config``.

The green lists are not HuggingFace's: it draws each list with ``torch.randperm`` on a generator reseeded per token,
which depends on torch's generator on the device where it runs and cannot be reproduced inside a kernel. Here they
come from a keyed hash built on the project's Philox4x32-10 (``philox4`` in csrc/philox.cuh, ``ops.sampling.
philox4x32_10`` in Python integers, ``philox`` below vectorised), ``philox4(c0, c1, c2, c3; k0, k1)`` its four output
words (x, y, z, w) for that counter and key:

- threshold: θ = round(γ·2³²), which must lie in [1, 2³² − 1]; the detector uses γ_eff = θ / 2³².
- green test: for a 64-bit seed (s0, s1), id v is *green* iff ``philox4(v, 0, 0, TAG_GREEN; s0, s1).x < θ``: one
  Bernoulli(γ_eff) draw per id and seed, the null model of the z-test.
- ``lefthash``, for a row whose sequence ``s[:L]`` has L >= w: (s0, s1) = (K mod 2³², K >> 32), then for i = 1..w
  (s0, s1) <- the (x, y) words of ``philox4(s[L - i], i, 0, TAG_CTX; s0, s1)``. One seed serves the whole row. Unlike
  HuggingFace's lefthash, which reads only the last id whatever w is, this one hashes the last w ids.
- ``selfhash``, for L >= w - 1: candidate v's seed is the minimum of h(x) over x in ``s[L - w + 1:L]`` and v, with
  h(x) the 64-bit value (y << 32) | x of ``philox4(x, v, 0, TAG_SELF; K mod 2³², K >> 32)`` (HuggingFace's min-PRF);
  v is green iff the green test passes under that seed. HuggingFace tests only the 40 largest logits; here every
  id < vocab is tested. At w = 1 the green set does not depend on the sequence.
- biasing, after rules 0-4 of ``ops/repeats.py`` (HuggingFace appends its watermark after the other processors): every
  green id v < vocab gets l_v <- fl32(l_v + δ), δ rounded to fp32 once. Other ids keep their bits, -inf stays -inf,
  columns from vocab on are untouched and a row whose sequence is too short is unchanged. In beam search the bias acts
  before the log-softmax, as the other rules do.
- detection, of right-padded ids [B, T] with ``lengths`` and per-row ``scored_from`` (default 0, so a prompt can be
  passed as context without being scored): position j of a row is scored when j >= scored_from, j < L and j >= w for
  lefthash (j >= w - 1 for selfhash); it is green when ``s[j]`` passes the test with the seed computed from ``s[:j]``.
  With ``ignore_repeated_ngrams`` only the first scored occurrence of each distinct n-gram ``s[j - n + 1:j + 1]``
  counts, n = w + 1 for lefthash and w for selfhash (the window and the id, as HuggingFace counts). The counts n
  (scored) and g (green) are exact integers; in fp64 on the host z = (g − γ_eff·n) / √(n·γ_eff·(1 − γ_eff)),
  p = ½·erfc(z / √2) (the exact normal tail) and ``prediction`` = z > ``z_threshold``. A row with n = 0 has
  z = nan and prediction False.
"""
from __future__ import annotations

import dataclasses
import math
from numbers import Integral, Real
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

TAG_CTX = 0x57435458             # "WCTX": the lefthash context chain
TAG_SELF = 0x57534C46            # "WSLF": the selfhash min-PRF
TAG_GREEN = 0x5747524E           # "WGRN": the green test
SCHEMES = ("lefthash", "selfhash")
MAX_CONTEXT_WIDTH = 8

_M32 = np.uint64(0xFFFFFFFF)


@dataclasses.dataclass(frozen=True)
class WatermarkingConfig:
    """HuggingFace's ``WatermarkingConfig`` fields and defaults (see the module docstring); ``check_watermark_args``
    validates one."""
    greenlist_ratio: float = 0.25
    bias: float = 2.0
    hashing_key: int = 15485863
    seeding_scheme: str = "lefthash"
    context_width: int = 1

    @property
    def threshold(self) -> int:
        """θ = round(γ·2³²)."""
        return int(round(float(self.greenlist_ratio) * 2.0 ** 32))

    @property
    def gamma_eff(self) -> float:
        """θ / 2³², the green probability of an id."""
        return self.threshold / 2.0 ** 32

    @property
    def delta(self) -> np.float32:
        """δ rounded to fp32."""
        return np.float32(self.bias)

    @property
    def key_words(self) -> Tuple[int, int]:
        """(K mod 2³², K >> 32)."""
        return int(self.hashing_key) & 0xFFFFFFFF, int(self.hashing_key) >> 32

    @property
    def selfhash(self) -> bool:
        return self.seeding_scheme == "selfhash"

    @property
    def min_position(self) -> int:
        """The first position a row can score, and the sequence length the bias needs: w (lefthash), w - 1
        (selfhash)."""
        return int(self.context_width) - int(self.selfhash)


def check_watermark_args(who: str, config) -> Optional[WatermarkingConfig]:
    """``config`` (a ``WatermarkingConfig``, a dict with its keys or None: off) validated, as a new
    ``WatermarkingConfig``; ``ValueError`` naming ``who`` and the argument for an unknown key, γ outside (0, 1) or θ out
    of range, δ not finite in fp32, an unknown scheme, w not an integer in [1, MAX_CONTEXT_WIDTH] or K not an integer
    in [0, 2⁶⁴)."""
    if config is None:
        return None
    if isinstance(config, WatermarkingConfig):
        kw = dataclasses.asdict(config)
    elif isinstance(config, dict):
        names = {f.name for f in dataclasses.fields(WatermarkingConfig)}
        unknown = sorted(str(k) for k in config if k not in names)
        if unknown:
            raise ValueError(f"{who}: watermarking_config has unknown keys {unknown}; the keys are {sorted(names)}")
        kw = dict(config)
    else:
        raise ValueError(f"{who}: watermarking_config must be a WatermarkingConfig, a dict or None, got "
                         f"{type(config).__name__}")
    cfg = WatermarkingConfig(**kw)
    g = cfg.greenlist_ratio
    if isinstance(g, bool) or not isinstance(g, Real) or not 0 < float(g) < 1:
        raise ValueError(f"{who}: greenlist_ratio must be a number in (0, 1), got {g!r}")
    if not 1 <= cfg.threshold <= 2 ** 32 - 1:
        raise ValueError(f"{who}: greenlist_ratio {g!r} rounds to the threshold {cfg.threshold}, outside [1, 2^32 - 1]")
    b = cfg.bias
    if isinstance(b, bool) or not isinstance(b, Real):
        raise ValueError(f"{who}: bias must be a number that is finite in fp32, got {b!r}")
    with np.errstate(over="ignore"):
        if not np.isfinite(np.float32(b)):
            raise ValueError(f"{who}: bias must be a number that is finite in fp32, got {b!r}")
    if cfg.seeding_scheme not in SCHEMES:
        raise ValueError(f"{who}: seeding_scheme must be one of {SCHEMES}, got {cfg.seeding_scheme!r}")
    w = cfg.context_width
    if isinstance(w, bool) or not isinstance(w, Integral) or not 1 <= int(w) <= MAX_CONTEXT_WIDTH:
        raise ValueError(f"{who}: context_width must be an integer in [1, {MAX_CONTEXT_WIDTH}], got {w!r}")
    k = cfg.hashing_key
    if isinstance(k, bool) or not isinstance(k, Integral) or not 0 <= int(k) < 2 ** 64:
        raise ValueError(f"{who}: hashing_key must be an integer in [0, 2^64), got {k!r}")
    return WatermarkingConfig(float(g), float(b), int(k), str(cfg.seeding_scheme), int(w))


def philox(c0, c1, c2, c3, k0, k1) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """Philox4x32-10 (``ops.sampling.philox4x32_10``) vectorised over broadcast counters and keys: the four output words
    as uint64 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & _M32 for x in (c0, c1, c2, c3)]
    k0, k1 = (np.asarray(x, dtype=np.uint64) & _M32 for x in (k0, k1))
    c = np.broadcast_arrays(*c, k0, k1)
    c, k0, k1 = c[:4], c[4], c[5]
    m0, m1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    w0, w1, s32 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85), np.uint64(32)
    for _ in range(10):
        p0, p1 = m0 * c[0], m1 * c[2]
        c = [(p1 >> s32) ^ c[1] ^ k0, p1 & _M32, (p0 >> s32) ^ c[3] ^ k1, p0 & _M32]
        k0, k1 = (k0 + w0) & _M32, (k1 + w1) & _M32
    return tuple(c)


def _u32(ids) -> np.ndarray:
    return np.asarray(ids, dtype=np.int64).astype(np.uint64) & _M32


def is_green(v, s0, s1, theta: int) -> np.ndarray:
    """The green test of ids ``v`` under seeds ``(s0, s1)`` (broadcast)."""
    return philox(_u32(v), 0, 0, TAG_GREEN, s0, s1)[0] < np.uint64(theta)


def lefthash_seed(ctx, cfg: WatermarkingConfig) -> Tuple[np.ndarray, np.ndarray]:
    """The lefthash seed words after the ids ``ctx`` [..., w] (the last w ids of a sequence, oldest first)."""
    ctx = _u32(ctx)
    s0, s1 = (np.full(ctx.shape[:-1], x, dtype=np.uint64) for x in cfg.key_words)
    for i in range(1, cfg.context_width + 1):
        s0, s1 = philox(ctx[..., -i], i, 0, TAG_CTX, s0, s1)[:2]
    return s0, s1


def selfhash_green(v, win, cfg: WatermarkingConfig) -> np.ndarray:
    """The selfhash green test of ids ``v`` [...] with windows ``win`` [..., w - 1] (the ids before each)."""
    v, win = _u32(v), _u32(win)
    k0, k1 = cfg.key_words

    def h(x):
        x, y = philox(x, v, 0, TAG_SELF, k0, k1)[:2]
        return (y << np.uint64(32)) | x

    m = h(v)
    for i in range(win.shape[-1]):
        m = np.minimum(m, h(win[..., i]))
    return is_green(v, m & _M32, m >> np.uint64(32), cfg.threshold)


def green_ids(seq, vocab: int, cfg: WatermarkingConfig) -> Optional[np.ndarray]:
    """The bool [vocab] green mask of the next id after the sequence ``seq``, None when it is too short."""
    s = np.asarray(seq.cpu() if isinstance(seq, torch.Tensor) else seq, dtype=np.int64).reshape(-1)
    L, w = s.size, cfg.context_width
    if L < cfg.min_position:
        return None
    v = np.arange(vocab, dtype=np.int64)
    if cfg.selfhash:
        return selfhash_green(v, np.broadcast_to(s[L - w + 1:L], (vocab, w - 1)), cfg)
    s0, s1 = lefthash_seed(s[L - w:], cfg)
    return is_green(v, s0, s1, cfg.threshold)


def watermark_reference(logits, seqs: Sequence, vocab: int, config) -> torch.Tensor:
    """The bias for R rows: ``logits`` [R, >= vocab] (fp32 values), ``seqs`` R sequences, ``config`` a
    ``WatermarkingConfig`` (or its dict). Returns a new fp32 tensor of the logits' shape on their device."""
    cfg = check_watermark_args("watermark_reference", config)
    t = logits if isinstance(logits, torch.Tensor) else torch.as_tensor(logits)
    x = t.detach().to(device="cpu", dtype=torch.float32).numpy().copy()
    if len(seqs) != x.shape[0]:
        raise ValueError(f"watermark_reference: {x.shape[0]} rows but {len(seqs)} sequences")
    for r, s in enumerate(seqs):
        green = green_ids(s, vocab, cfg)
        if green is not None:
            row = x[r, :vocab]
            row[green] = row[green] + cfg.delta
    return torch.from_numpy(x).to(t.device if isinstance(logits, torch.Tensor) else "cpu")


def position_green(s: np.ndarray, pos: np.ndarray, cfg: WatermarkingConfig) -> np.ndarray:
    """Whether ``s[j]`` is green under the seed of ``s[:j]``, for the positions ``pos`` (each >= min_position)."""
    w = cfg.context_width
    if cfg.selfhash:
        win = s[pos[:, None] - np.arange(w - 1, 0, -1)[None, :]] if w > 1 else np.zeros((pos.size, 0), np.int64)
        return selfhash_green(s[pos], win, cfg)
    s0, s1 = lefthash_seed(s[pos[:, None] - np.arange(w, 0, -1)[None, :]], cfg)
    return is_green(s[pos], s0, s1, cfg.threshold)


def watermark_counts_reference(ids, lengths: Sequence[int], scored_from: Sequence[int], config,
                               ignore_repeated_ngrams: bool = False) -> np.ndarray:
    """Detection counts of the rows of ``ids`` [B, T]: int64 [B, 2], (n scored, g green) per row."""
    cfg = check_watermark_args("watermark_counts_reference", config)
    a = np.asarray(ids.cpu() if isinstance(ids, torch.Tensor) else ids, dtype=np.int64)
    out = np.zeros((a.shape[0], 2), dtype=np.int64)
    n_gram = cfg.context_width + 1 - int(cfg.selfhash)
    for b in range(a.shape[0]):
        L = min(max(int(lengths[b]), 0), a.shape[1])
        s = a[b, :L]
        pos = np.arange(max(int(scored_from[b]), cfg.min_position, 0), L)
        if ignore_repeated_ngrams:
            seen, keep = set(), []
            for j in pos:
                key = tuple(s[j - n_gram + 1:j + 1].tolist())
                if key not in seen:
                    seen.add(key)
                    keep.append(j)
            pos = np.asarray(keep, dtype=np.int64)
        out[b] = pos.size, int(position_green(s, pos, cfg).sum()) if pos.size else 0
    return out


@dataclasses.dataclass
class WatermarkDetectorOutput:
    """Per-row detection results, HuggingFace's ``WatermarkDetectorOutput`` fields without ``confidence``."""
    num_tokens_scored: np.ndarray        # int64 [B]
    num_green_tokens: np.ndarray         # int64 [B]
    green_fraction: np.ndarray           # fp64 [B], nan where nothing was scored
    z_score: np.ndarray                  # fp64 [B], nan where nothing was scored
    p_value: np.ndarray                  # fp64 [B], nan where nothing was scored
    prediction: np.ndarray               # bool [B]


def z_scores(n, g, gamma_eff: float, z_threshold: float = 3.0) -> WatermarkDetectorOutput:
    """The statistics of the counts ``n`` and ``g``, in fp64."""
    n, g = np.asarray(n, dtype=np.int64), np.asarray(g, dtype=np.int64)
    nf, gf = n.astype(np.float64), g.astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        frac = np.where(n > 0, gf / np.maximum(nf, 1), np.nan)
        z = np.where(n > 0, (gf - gamma_eff * nf) / np.sqrt(nf * gamma_eff * (1 - gamma_eff)), np.nan)
    p = np.array([0.5 * math.erfc(x / math.sqrt(2)) if math.isfinite(x) else math.nan for x in z.reshape(-1)],
                 dtype=np.float64).reshape(z.shape)
    return WatermarkDetectorOutput(n, g, frac, z, p, np.where(np.isnan(z), False, z > z_threshold))


def detect_watermark(input_ids, config, lengths: Optional[Sequence[int]] = None, scored_from=None,
                     ignore_repeated_ngrams: bool = False, z_threshold: float = 3.0) -> WatermarkDetectorOutput:
    """Scores the rows of ``input_ids`` [B, T] (right-padded to ``lengths``, default T) for the watermark of ``config``
    (a ``WatermarkingConfig`` or its dict): ``scored_from`` (an int or B ints, default 0) is each row's first scored
    position, so a prompt can be passed as context. Counts on the device (``ops.watermark_count_``) for CUDA inputs,
    with ``watermark_counts_reference`` otherwise; the statistics in fp64 (see the module docstring)."""
    who = "detect_watermark"
    cfg = check_watermark_args(who, config)
    if cfg is None:
        raise ValueError(f"{who}: config must be a WatermarkingConfig or a dict, got None")
    if not isinstance(input_ids, torch.Tensor):
        input_ids = torch.as_tensor(np.asarray(input_ids, dtype=np.int64))
    if input_ids.dim() != 2 or input_ids.dtype.is_floating_point or input_ids.dtype == torch.bool:
        raise ValueError(f"{who}: input_ids must be an integer [B, T] tensor, got {input_ids.dtype} "
                         f"{tuple(input_ids.shape)}")
    B, T = input_ids.shape
    lengths = [T] * B if lengths is None else [int(x) for x in lengths]
    if len(lengths) != B or any(not 0 <= x <= T for x in lengths):
        raise ValueError(f"{who}: need {B} lengths in [0, {T}], got {lengths}")
    if scored_from is None:
        scored_from = 0
    starts = [scored_from] * B if isinstance(scored_from, Integral) else list(scored_from)
    if len(starts) != B or any(isinstance(x, bool) or not isinstance(x, Integral) or x < 0 for x in starts):
        raise ValueError(f"{who}: scored_from must be an integer >= 0 or {B} of them, got {scored_from!r}")
    if not isinstance(ignore_repeated_ngrams, (bool, np.bool_)):
        raise ValueError(f"{who}: ignore_repeated_ngrams must be a bool, got {ignore_repeated_ngrams!r}")
    if isinstance(z_threshold, bool) or not isinstance(z_threshold, Real) or not math.isfinite(z_threshold):
        raise ValueError(f"{who}: z_threshold must be a finite number, got {z_threshold!r}")
    if input_ids.is_cuda:
        from . import watermark_count_

        dev = input_ids.device
        i32 = dict(dtype=torch.int32, device=dev)
        counts = watermark_count_(input_ids.to(torch.int32).contiguous(), torch.tensor(lengths, **i32),
                                  torch.tensor([int(x) for x in starts], **i32), cfg, bool(ignore_repeated_ngrams))
        counts = counts.cpu().numpy().astype(np.int64)
    else:
        counts = watermark_counts_reference(input_ids, lengths, starts, cfg, bool(ignore_repeated_ngrams))
    return z_scores(counts[:, 0], counts[:, 1], cfg.gamma_eff, float(z_threshold))
