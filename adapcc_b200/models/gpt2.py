"""GPT-2 small with the "double heads" (LM + multiple choice) of the reference's flagship workload.

The reference trains ``transformers.GPT2DoubleHeadsModel(GPT2Config())`` (12 layers, d=768, 12 heads,
ctx 1024, vocab 50257 + 5 special tokens) on PersonaChat-shaped batches
``input_ids/token_type_ids/lm_labels [B, C, T]``, ``mc_token_ids [B, C]``, ``mc_labels [B]`` with
loss = lm_coef * LM cross-entropy + mc_coef * multiple-choice cross-entropy
(/root/reference/models/gpt2/train_gpt2_ddp.py:28-31,100-107,157-195). This is the same
architecture written for H100 training:

* parameters live in bf16 (fp32 master copy inside the fused optimizer), so gradients are born in
  bf16 and the gradient all-reduce moves half the bytes with fp32 accumulation in the kernel;
* attention goes through ``scaled_dot_product_attention`` (flash kernels; the backward in its deterministic mode, so a
  step computes the same bits every run), MLP through the fused GEMMs;
* the LM head + cross-entropy is one fused pass per row chunk: bf16 logits from the GEMM, a softmax-CE
  kernel that overwrites them in place with their gradient, and the two backward GEMMs right away — fp32
  logits / probabilities (50 304 x 8192 x 4 B = 1.6 GB each in the stock path) never exist;
* no data-dependent host syncs: the whole step can be captured in one CUDA graph.

Token-type embeddings reuse ``wte`` exactly as HF GPT-2 does.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops.dropout import DropoutState, check_p, dropout, site_attn, site_embed, site_mlp, site_summary
from ..ops.guidance import check_guidance_args, guided_scores_reference
from ..ops.kvcache import check_kv_cache_dtype
from ..ops.layers import FusedLayerNorm, FusedLinear
from ..ops.repeats import check_repeat_args, check_sequence_bias_args, penalize_repeats_reference
from ..ops.sampling import check_filter_args, sample_reference, top_filtering


@dataclass
class GPT2Config:
    """GPT-2 small hyper-parameters (HF ``GPT2Config()`` + the five dialogue tokens) — the model of the reference's
    flagship workload, /root/reference/models/gpt2/train_gpt2_ddp.py:157-159."""

    vocab_size: int = 50257 + 5          # GPT2Config() + the five PersonaChat special tokens
    n_positions: int = 1024
    n_embd: int = 768
    n_layer: int = 12
    n_head: int = 12
    layer_norm_epsilon: float = 1e-5
    initializer_range: float = 0.02
    lm_chunk_rows: int = 8192            # rows of the fused LM-head/CE evaluated at a time (bf16 logits of one
                                         # chunk: 8192 x 50304 x 2 B = 0.8 GB; measured 2 % faster per step than 2048)
    # Dropout of the embedding sum, of every block's attention and MLP output, and of the multiple-choice head's
    # summary input, where HF GPT-2 applies it (whose GPT2Config() defaults are 0.1 each); masks as ops/dropout.py
    # defines them. 0: off, and the step is the one without these fields. Attention-probability dropout (HF's
    # attn_pdrop) does not exist here: see ROADMAP.md.
    embd_pdrop: float = 0.0
    resid_pdrop: float = 0.0
    summary_first_dropout: float = 0.0

    @classmethod
    def tiny(cls) -> "GPT2Config":
        return cls(vocab_size=512, n_positions=64, n_embd=64, n_layer=2, n_head=4, lm_chunk_rows=64)


class _Deterministic:
    """PyTorch's deterministic algorithms switched on (not warn-only) inside the block, the previous setting restored.
    Filling freshly allocated tensors with NaN (what the mode also does by default) is switched off inside: attention
    writes every element it allocates, so the fill would only cost time."""

    def __enter__(self):
        import torch.utils.deterministic as det

        self.prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(),
                     det.fill_uninitialized_memory)
        torch.use_deterministic_algorithms(True)
        det.fill_uninitialized_memory = False

    def __exit__(self, *exc):
        import torch.utils.deterministic as det

        torch.use_deterministic_algorithms(self.prev[0], warn_only=self.prev[1])
        det.fill_uninitialized_memory = self.prev[2]


class _CausalAttention(torch.autograd.Function):
    """Causal ``scaled_dot_product_attention`` run, forward and backward, with PyTorch's deterministic algorithms
    switched on and restored afterwards: the flash backward then sums dQ in a fixed order instead of with atomics, so
    the same inputs give the same gradient bits every run (PyTorch settles the mode when the forward runs, so both
    passes need it). At GPT-2 small's shape on an H100: 0.44 ms per layer forward + backward instead of 0.26."""

    @staticmethod
    def forward(ctx, q, k, v):
        with torch.enable_grad(), _Deterministic():
            inner = [t.detach().requires_grad_(True) for t in (q, k, v)]
            out = F.scaled_dot_product_attention(*inner, is_causal=True)
        ctx.inner, ctx.out = inner, out
        return out.detach()

    @staticmethod
    def backward(ctx, dout):
        with _Deterministic():
            grads = torch.autograd.grad(ctx.out, ctx.inner, dout)
        del ctx.inner, ctx.out
        return grads


def causal_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """Causal attention [B, H, T, Dh]; repeatable backward on CUDA (see ``_CausalAttention``)."""
    if q.is_cuda and torch.is_grad_enabled() and (q.requires_grad or k.requires_grad or v.requires_grad):
        return _CausalAttention.apply(q, k, v)
    return F.scaled_dot_product_attention(q, k, v, is_causal=True)


class KVCache:
    """Keys and values of every layer for incremental decoding (``GPT2DoubleHeads.new_cache``): ``k`` / ``v``
    [L, B, H, t_max, Dh] in the model's dtype, ``lens`` (int32 [B] on the device: tokens cached per row, what the
    kernels read), ``host_lens`` (the same numbers on the host, which issues every step and so always knows them) and
    ``work``, the split-partials workspace of the native decode-attention kernel (bf16 on CUDA; None otherwise),
    allocated once so a captured step reuses it.

    ``kv_cache_dtype="fp8_e4m3"``: ``k`` / ``v`` hold e4m3 bytes (uint8) and ``k_scale`` / ``v_scale`` (fp32
    [L, B, H, t_max]) the power-of-two scale of each vector, as ``ops/kvcache.py`` defines; every cached position is
    quantized, the prompt's included. Otherwise the scales are None."""

    def __init__(self, n_layer: int, batch: int, n_head: int, t_max: int, head_dim: int, dtype: torch.dtype, device,
                 kv_cache_dtype: Optional[str] = None):
        self.batch, self.t_max = int(batch), int(t_max)
        self.kv_cache_dtype = check_kv_cache_dtype("KVCache", kv_cache_dtype)
        fp8 = kv_cache_dtype is not None
        self.k = torch.zeros(n_layer, batch, n_head, t_max, head_dim, dtype=torch.uint8 if fp8 else dtype,
                             device=device)
        self.v = torch.zeros_like(self.k)
        self.k_scale = self.v_scale = None
        if fp8:
            self.k_scale = torch.zeros(n_layer, batch, n_head, t_max, dtype=torch.float32, device=self.k.device)
            self.v_scale = torch.zeros_like(self.k_scale)
        self.lens = torch.zeros(batch, dtype=torch.int32, device=self.k.device)
        self.host_lens: List[int] = [0] * self.batch
        self.work = None
        if self.k.is_cuda and dtype == torch.bfloat16:
            from ..ops import decode_attention_work_numel
            self.work = torch.empty(decode_attention_work_numel(batch, n_head, head_dim, t_max), dtype=torch.float32,
                                    device=self.k.device)

    @property
    def parts(self) -> List[torch.Tensor]:
        """Every per-position tensor: ``k``, ``v`` and, with an fp8 cache, ``k_scale`` and ``v_scale`` (each indexed
        [layer, row, head, position, ...])."""
        return [self.k, self.v] + ([self.k_scale, self.v_scale] if self.k_scale is not None else [])

    def scales(self, layer: int):
        """``(k_scale, v_scale)`` of layer ``layer``; (None, None) for a cache in the model's dtype."""
        if self.k_scale is None:
            return None, None
        return self.k_scale[layer], self.v_scale[layer]

    def reset(self, lengths: Sequence[int], T: int) -> None:
        """Lengths after a prefill of T (right-padded) positions."""
        lengths = [int(n) for n in lengths]
        if len(lengths) != self.batch or T > self.t_max or any(not 1 <= n <= T for n in lengths):
            raise ValueError(f"KVCache: a prefill of {T} positions (at most t_max = {self.t_max}) needs {self.batch} "
                             f"lengths in [1, {T}], got {lengths}")
        self.host_lens = lengths
        self.lens.copy_(torch.tensor(lengths, dtype=torch.int32))

    def check_room(self) -> None:
        if max(self.host_lens) >= self.t_max:
            raise ValueError(f"KVCache: full (t_max = {self.t_max}, lengths {self.host_lens}); prefill again")

    def advance(self) -> None:
        """After the last layer of a step: every row holds one more token."""
        self.lens.add_(1)
        self.advance_host()

    def advance_host(self) -> None:
        self.host_lens = [n + 1 for n in self.host_lens]


def decode_attention(qkv: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, lens: torch.Tensor,
                     work: Optional[torch.Tensor] = None, k_scale: Optional[torch.Tensor] = None,
                     v_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One layer of decode attention: ``qkv`` [B, 3·H·Dh] (q | k | v of each row's new token), caches [B, H, t_max, Dh],
    ``lens`` int32 [B]. Stores the new k / v at position ``lens[b]`` and returns softmax(q·K[0..lens[b]]ᵀ/√Dh)·V [B, H·Dh]
    with an fp32 softmax. With ``work`` (bf16 CUDA caches) this is the native kernel (``ops.decode_attention_``);
    otherwise the same computation in PyTorch, the reference the CPU tests use. With ``k_scale`` / ``v_scale`` (fp32
    [B, H, t_max]) the caches are fp8 (``ops/kvcache.py``): the new k / v are stored quantized, and the new token
    attends to them unquantized and to the dequantized cache before ``lens[b]``."""
    B, H, t_max, Dh = k_cache.shape
    if work is not None:
        from ..ops import decode_attention_
        out = torch.empty(B, H * Dh, dtype=qkv.dtype, device=qkv.device)
        return decode_attention_(qkv, k_cache, v_cache, lens, out, work, k_scale=k_scale, v_scale=v_scale)
    q, k, v = qkv.reshape(B, 3, H, Dh).unbind(1)
    pos = lens.long()
    rows = torch.arange(B, device=qkv.device)
    if k_scale is not None:
        from ..ops.kvcache import dequantize, quantize
        keys, values = dequantize(k_cache, k_scale), dequantize(v_cache, v_scale)
        keys[rows, :, pos] = k.float()
        values[rows, :, pos] = v.float()
        for x, qc, sc in ((k, k_cache, k_scale), (v, v_cache, v_scale)):
            qc[rows, :, pos], sc[rows, :, pos] = quantize(x)
    else:
        k_cache[rows, :, pos] = k
        v_cache[rows, :, pos] = v
        keys, values = k_cache.float(), v_cache.float()
    s = torch.einsum("bhd,bhtd->bht", q.float(), keys) / math.sqrt(Dh)
    s = s.masked_fill(torch.arange(t_max, device=qkv.device) > pos[:, None, None], float("-inf"))
    p = torch.softmax(s, dim=-1)
    return torch.einsum("bht,bhtd->bhd", p, values).to(qkv.dtype).reshape(B, H * Dh)


class CandidateKV:
    """What a candidate step of contrastive search attends over: ``top_k`` candidate tokens per row of ``cache``, the
    candidates of row b in rows ``b·k .. b·k + k - 1``. Candidate (b, j) attends over the row's cached positions and its
    own new key and value at ``cache.lens[b]``; the cache is only read, and every layer's new keys and values go to
    ``side`` [n_layer, 2, B·k, D] (model dtype) for the winner's commit. With ``work`` (bf16 CUDA caches) this is the
    native kernel (``ops.cand_attention_``); otherwise ``decode_attention`` in PyTorch on a k-fold copy of the rows."""

    def __init__(self, cache: "KVCache", top_k: int, side: torch.Tensor, work: Optional[torch.Tensor] = None):
        self.cache, self.top_k, self.side, self.work = cache, int(top_k), side, work

    def attend(self, qkv: torch.Tensor, layer: int) -> torch.Tensor:
        """Layer ``layer``'s attention of the candidates ``qkv`` [B·k, 3·H·Dh] -> [B·k, H·Dh]."""
        c, K = self.cache, self.top_k
        B, H, t_max, Dh = c.k[layer].shape
        if self.work is not None:
            from ..ops import cand_attention_
            out = torch.empty(B * K, H * Dh, dtype=qkv.dtype, device=qkv.device)
            return cand_attention_(qkv, c.k[layer], c.v[layer], c.lens, K, out, self.side[layer, 0],
                                   self.side[layer, 1], self.work)
        q, k, v = qkv.reshape(B * K, 3, H * Dh).unbind(1)
        self.side[layer, 0].copy_(k)
        self.side[layer, 1].copy_(v)
        return decode_attention(qkv, c.k[layer].repeat_interleave(K, 0), c.v[layer].repeat_interleave(K, 0),
                                c.lens.repeat_interleave(K))


class VerifyKV:
    """What a verify step of prompt-lookup decoding attends over: ``slots`` (k + 1) slots per row of ``cache``, slot j
    of row b in row ``b·(k+1) + j`` at position ``cache.lens[b] + j``, the first ``nq[b]`` of them real (int32 [B]).
    Real slot j attends over the row's cached positions and the new keys and values of its slots ``0..j``, which are
    stored at their positions; pad slots write nothing and give zero. The lengths do not move. With ``work`` (bf16 CUDA
    caches) this is the native kernel (``ops.verify_attention_``); otherwise masked fp32 attention in PyTorch."""

    def __init__(self, cache: "KVCache", slots: int, nq: torch.Tensor, work: Optional[torch.Tensor] = None):
        self.cache, self.slots, self.nq, self.work = cache, int(slots), nq, work

    def attend(self, qkv: torch.Tensor, layer: int) -> torch.Tensor:
        """Layer ``layer``'s attention of the slots ``qkv`` [B·(k+1), 3·H·Dh] -> [B·(k+1), H·Dh]."""
        c, S = self.cache, self.slots
        kc, vc = c.k[layer], c.v[layer]
        B, H, t_max, Dh = kc.shape
        if self.work is not None:
            from ..ops import verify_attention_
            out = torch.empty(B * S, H * Dh, dtype=qkv.dtype, device=qkv.device)
            return verify_attention_(qkv, kc, vc, c.lens, self.nq, S - 1, out, self.work)
        q, k, v = qkv.reshape(B, S, 3, H, Dh).unbind(2)
        pos = c.lens.long()[:, None] + torch.arange(S, device=qkv.device)                       # [B, S]
        real = (torch.arange(S, device=qkv.device) < self.nq.to(qkv.device).long()[:, None]) & (pos < t_max)
        rows, slot = real.nonzero(as_tuple=True)
        kc[rows, :, pos[rows, slot]] = k[rows, slot]
        vc[rows, :, pos[rows, slot]] = v[rows, slot]
        s = torch.einsum("bjhd,bhtd->bjht", q.float(), kc.float()) / math.sqrt(Dh)
        s = s.masked_fill(torch.arange(t_max, device=qkv.device) > pos[:, :, None, None], float("-inf"))
        o = torch.einsum("bjht,bhtd->bjhd", torch.softmax(s, dim=-1), vc.float()) * real[:, :, None, None]
        return o.to(qkv.dtype).reshape(B * S, H * Dh)


class _Repeats:
    """The repetition controls of a batched decoder over the first R rows of its cache (``rows``; default all of them,
    ``generate`` with guidance passes its B prompt rows): ``seq`` int32 [R, t_max] each row's sequence (its prompt,
    then its tokens), ``prompt_len`` int32 [R] the lengths after the prefill, the sequence-bias table
    (``ops.repeats.SequenceBias`` or None), the repetition penalty, the n-gram size, the frequency and presence
    penalties and the context n-gram size (the keyword arguments ``GPT2DoubleHeads._decode_setup`` returns).
    ``create`` returns None when all of them are off, so then nothing is allocated or launched."""

    def __init__(self, input_ids: torch.Tensor, cache: KVCache, vocab: int, penalty: float, ngram: int,
                 rows: Optional[int] = None, bias=None, frequency: float = 0.0, presence: float = 0.0,
                 context_ngram: int = 0):
        B, T = input_ids.shape
        self.rows = cache.batch if rows is None else int(rows)
        self.seq = torch.zeros(self.rows, cache.t_max, dtype=torch.int32, device=input_ids.device)
        self.seq[:, :T] = input_ids.repeat_interleave(self.rows // B, dim=0)
        self.prompt_len = cache.lens[:self.rows].clone()
        self.host_prompt_len = list(cache.host_lens[:self.rows])
        self.vocab, self.penalty, self.ngram, self.bias = vocab, penalty, ngram, bias
        self.counts = dict(frequency=float(frequency), presence=float(presence), context_ngram=int(context_ngram))
        if bias is not None and input_ids.is_cuda:
            bias.device_tensors(input_ids.device)       # before any capture: the graph keeps these pointers

    @classmethod
    def create(cls, input_ids: torch.Tensor, cache: KVCache, vocab: int, penalty: float, ngram: int,
               rows: Optional[int] = None, bias=None, frequency: float = 0.0, presence: float = 0.0,
               context_ngram: int = 0) -> Optional["_Repeats"]:
        on = (penalty != 1.0 or ngram > 0 or bias is not None or frequency != 0 or presence != 0
              or context_ngram > 0)
        return cls(input_ids, cache, vocab, penalty, ngram, rows, bias, frequency, presence,
                   context_ngram) if on else None

    def eager(self, logits: torch.Tensor, cache: KVCache, consumed: Optional[torch.Tensor]) -> torch.Tensor:
        """``penalize_repeats_reference`` over every row's sequence, after storing ``consumed`` [R] (the tokens the last
        decode step consumed; None before the first one) at ``lens - 1``."""
        R = self.rows
        if consumed is not None:
            dev = self.seq.device
            self.seq[torch.arange(R, device=dev), cache.lens[:R].long() - 1] = consumed.to(dev, torch.int32)
        return penalize_repeats_reference(logits, [self.seq[r, :x] for r, x in enumerate(cache.host_lens[:R])],
                                          self.vocab, self.penalty, self.ngram, self.bias,
                                          prompt_lens=self.host_prompt_len, **self.counts)

    def reorder(self, rows: torch.Tensor) -> None:
        """Row r continues row ``rows[r]`` (a beam its parent)."""
        self.seq = self.seq[rows]

    def native(self, logits: torch.Tensor, lens: torch.Tensor, step: torch.Tensor, ids: torch.Tensor,
               parent: Optional[torch.Tensor] = None, group: int = 1) -> None:
        """``ops.penalize_repeats_`` on ``logits`` in place; it also stores ``ids`` and follows ``parent``."""
        from ..ops import penalize_repeats_
        penalize_repeats_(logits, self.vocab, self.seq, self.prompt_len, lens, step, ids, parent, group,
                          self.penalty, self.ngram, self.bias, **self.counts)


def _row_seeds(seed, B: int, dev) -> torch.Tensor:
    """``generate``'s per-row seeds, int64 [B] on ``dev``: an int (row b uses ``seed + b``) or an int64 [B] tensor."""
    if isinstance(seed, torch.Tensor):
        if seed.dtype != torch.int64 or seed.numel() != B:
            raise ValueError(f"generate: a seed tensor must be int64 with {B} elements, got {seed.dtype} "
                             f"{tuple(seed.shape)}")
        return seed.reshape(B).to(dev)
    return (int(seed) + torch.arange(B, dtype=torch.int64)).to(dev)


class Block(nn.Module):
    """Pre-LN transformer block; the MLP runs as two GEMMs with the activation passes in GEMM epilogues when
    supported (ops/gemm.py), residual adds optionally fused into the following LayerNorm (``forward_deferred``)."""

    def __init__(self, cfg: GPT2Config):
        super().__init__()
        d = cfg.n_embd
        self.n_head = cfg.n_head
        # fused kernels on CUDA/bf16, stock ATen otherwise (same parameters either way)
        self.ln_1 = FusedLayerNorm(d, eps=cfg.layer_norm_epsilon)
        self.c_attn = FusedLinear(d, 3 * d)
        self.c_proj = FusedLinear(d, d)
        self.ln_2 = FusedLayerNorm(d, eps=cfg.layer_norm_epsilon)
        self.c_fc = FusedLinear(d, 4 * d)
        self.c_proj2 = FusedLinear(4 * d, d)
        # the MLP's activation passes live in our wgmma GEMM's epilogues (ops/gemm.py, csrc/gemm_wgmma.cu):
        # 2 (default): c_fc + bias + GELU forward AND dGELU + the c_fc bias gradient in the backward GEMM dY.W2 — no
        #    stand-alone GELU / GELU-backward / column-sum kernel;
        # 1: forward fusion only; 0: cuBLAS + separate activation kernels
        self.tc_mlp = int(os.environ.get("ADAPCC_TCGEN05_MLP", "2") or 0)

    def _mlp(self, h: torch.Tensor) -> torch.Tensor:
        if self.tc_mlp and h.is_cuda and h.dtype == torch.bfloat16 and torch.is_grad_enabled():
            from ..ops.gemm import linear_gelu, mlp_gelu, supported
            if supported(h, self.c_fc.weight):
                if self.tc_mlp >= 2 and self.c_fc.weight.shape[0] % 64 == 0:
                    return mlp_gelu(h, self.c_fc.weight, self.c_fc.bias, self.c_proj2.weight, self.c_proj2.bias)
                return self.c_proj2(linear_gelu(h, self.c_fc.weight, self.c_fc.bias))
        return self.c_proj2(F.gelu(self.c_fc(h), approximate="tanh"))

    def _attn(self, h: torch.Tensor, cache: Optional["KVCache"] = None, layer: int = 0) -> torch.Tensor:
        if isinstance(cache, (CandidateKV, VerifyKV)):   # contrastive search / prompt lookup: k + 1 slots per row
            return self.c_proj(cache.attend(self.c_attn(h), layer))
        if cache is not None and h.dim() == 2:       # decode: one new token per row [B, D] against the cache
            return self.c_proj(decode_attention(self.c_attn(h), cache.k[layer], cache.v[layer], cache.lens, cache.work,
                                                *cache.scales(layer)))
        B, T, D = h.shape
        # split along the feature dim (views; measured 6 % faster fwd+bwd than the packed permute:
        # the backward writes dq/dk/dv straight into one [B, T, 3D] buffer layout-wise)
        qkv = self.c_attn(h)
        q, k, v = (t.view(B, T, self.n_head, D // self.n_head).transpose(1, 2) for t in qkv.split(D, dim=-1))
        if cache is not None and cache.k_scale is not None:     # prefill of an fp8 cache: quantize every position
            ks, vs = cache.scales(layer)
            if cache.work is not None:
                from ..ops import kv_quantize_
                kv_quantize_(qkv.detach(), cache.k[layer], cache.v[layer], ks, vs)
            else:
                from ..ops.kvcache import store_
                store_(k.detach(), cache.k[layer, :, :, :T], ks[:, :, :T])
                store_(v.detach(), cache.v[layer, :, :, :T], vs[:, :, :T])
        elif cache is not None:                       # prefill: keep this layer's keys and values
            cache.k[layer, :, :, :T].copy_(k.detach())
            cache.v[layer, :, :, :T].copy_(v.detach())
        a = causal_attention(q, k, v)
        return self.c_proj(a.transpose(1, 2).reshape(B, T, D))

    def forward_deferred(self, x: torch.Tensor, delta: Optional[torch.Tensor], cache: Optional["KVCache"] = None,
                         layer: int = 0, drop=None):
        """Same block with every residual add fused into the LayerNorm that follows it: takes the
        residual stream ``x`` and the previous block's not-yet-added MLP output ``delta``, returns
        (stream, this block's not-yet-added MLP output). ``drop = (p, state)``: residual dropout, applied to each
        branch inside the add-LayerNorm that adds it (``delta`` is block ``layer - 1``'s MLP output)."""
        if delta is None:
            h = self.ln_1(x)
        else:
            x, h = self.ln_1.forward_add(x, delta, drop and (*drop, site_mlp(layer - 1)))
        x, h = self.ln_2.forward_add(x, self._attn(h, cache, layer), drop and (*drop, site_attn(layer)))
        return x, self._mlp(h)

    def forward(self, x: torch.Tensor, cache: Optional["KVCache"] = None, layer: int = 0, drop=None) -> torch.Tensor:
        if drop is None:
            x = x + self._attn(self.ln_1(x), cache, layer)
            return x + self._mlp(self.ln_2(x))
        x = x + dropout(self._attn(self.ln_1(x), cache, layer), *drop, site_attn(layer))
        return x + dropout(self._mlp(self.ln_2(x)), *drop, site_mlp(layer))


def use_sink(p) -> bool:
    from ..ops.layers import _sink
    return p.is_cuda and _sink(p) is not None


class _ChunkedLMLoss(torch.autograd.Function):
    """sum over rows of CE(h @ W^T, labels), ``chunk`` rows at a time. The backward of every chunk
    is produced inside the forward pass (fused softmax-CE kernel overwrites the bf16 logits with
    their gradient), so logits never outlive a chunk and are touched twice instead of ~8 times."""

    @staticmethod
    def forward(ctx, h, weight, labels, chunk, vocab, scale=None):
        """-> (scaled, total): ``total`` is the sum of row losses (no gradient flows through it), ``scaled`` is
        ``scale * total``, or ``total`` itself without a scale.

        ``scale`` (1-element fp32 device tensor or None): the gradients produced here already contain it — the caller
        promises that ``scaled`` enters the total
        loss with coefficient exactly 1 (GPT2DoubleHeads.forward does). That is what allows the weight gradient to be
        written straight into the engine's flat gradient buffer during the forward pass (``weight`` carries a grad sink,
        ops/layers.py::_sink): no 77 MB ``grad_w * g`` and no 77 MB accumulate kernel in the backward."""
        n = h.shape[0]
        use_kernel = h.is_cuda and h.dtype == torch.bfloat16 and weight.shape[0] % 8 == 0
        grad_h = torch.empty_like(h)
        grad_w = None
        total = torch.zeros((), dtype=torch.float32, device=h.device)
        direct = False
        if use_kernel:
            from ..ops import fused_ce_
            from ..ops.layers import _sink
            direct = (scale is not None and _sink(weight) is not None and weight.grad.dtype == h.dtype
                      and ctx.needs_input_grad[1])
        for s in range(0, n, chunk):
            hs = h[s:s + chunk]
            ls = labels[s:s + chunk]
            logits = hs @ weight.t()
            if use_kernel:
                total += fused_ce_(logits, ls, vocab, grad_scale=scale).sum()
                g = logits                                         # now d loss / d logits (bf16)
            else:                                                  # CPU / fp32 reference path
                lf = logits.float()
                lf[:, vocab:] = float("-inf")
                valid = (ls >= 0)
                lse = torch.logsumexp(lf, dim=-1)
                tgt = lf.gather(1, ls.clamp(min=0).unsqueeze(1)).squeeze(1)
                total += ((lse - tgt) * valid).sum()
                p = torch.softmax(lf, dim=-1)
                p.scatter_add_(1, ls.clamp(min=0).unsqueeze(1), -torch.ones_like(p[:, :1]))
                g = p * valid.unsqueeze(1)
                if scale is not None:
                    g = g * scale
                g = g.to(h.dtype)
            torch.mm(g, weight, out=grad_h[s:s + chunk])
            # dW accumulates across chunks inside the GEMM (fp32 accumulator, beta = 1 epilogue) — an
            # fp32 side buffer cost ~1 GB of extra HBM traffic per chunk at vocab 50304
            if direct:
                if s == 0:
                    torch.mm(g.t(), hs, out=weight.grad)           # the flat-buffer view (zeroed at step start)
                else:
                    weight.grad.addmm_(g.t(), hs)
            elif grad_w is None:
                grad_w = g.t() @ hs
            else:
                grad_w.addmm_(g.t(), hs)
        scaled = total * scale.reshape(()) if scale is not None else total.clone()
        ctx.direct, ctx.weight = direct, weight
        if direct:
            ctx.save_for_backward(grad_h)
        else:
            if grad_w is None:
                grad_w = torch.zeros_like(weight)
            ctx.save_for_backward(grad_h, grad_w)
        ctx.mark_non_differentiable(total)
        return scaled, total

    @staticmethod
    def backward(ctx, g, _):
        if ctx.direct:                       # unit upstream gradient by contract; dW is already in weight.grad
            return ctx.saved_tensors[0], None, None, None, None, None
        grad_h, grad_w = ctx.saved_tensors
        gw = grad_w * g.to(grad_w.dtype)
        if use_sink(ctx.weight):
            # the table's gradient is owned by a sink (its LAST writer, the fused embedding backward, reports it):
            # autograd must not see a gradient for it, or the engine would count the parameter twice
            ctx.weight.grad.add_(gw)
            gw = None
        return grad_h * g.to(grad_h.dtype), gw, None, None, None, None


class GPT2DoubleHeads(nn.Module):
    """GPT-2 with a tied LM head and a multiple-choice head on a chosen token (HF ``GPT2DoubleHeadsModel``):
    ``forward`` returns the training losses (LM on labelled positions + MC over candidates); fused embedding,
    chunked LM-head + CE, optional scored-rows-only LM head."""

    def __init__(self, cfg: Optional[GPT2Config] = None):
        super().__init__()
        self.cfg = cfg = cfg or GPT2Config()
        # rows padded to a multiple of 64 so the LM-head GEMM and the fused CE kernel see aligned rows;
        # ids >= vocab_size are never produced and their logits are masked out
        self.padded_vocab = (cfg.vocab_size + 63) // 64 * 64
        self.wte = nn.Embedding(self.padded_vocab, cfg.n_embd)
        self.wpe = nn.Embedding(cfg.n_positions, cfg.n_embd)
        self.h = nn.ModuleList([Block(cfg) for _ in range(cfg.n_layer)])
        self.ln_f = FusedLayerNorm(cfg.n_embd, eps=cfg.layer_norm_epsilon)
        self.mc_head = nn.Linear(cfg.n_embd, 1)           # SequenceSummary(summary_type="cls_index")
        # > 0: evaluate the LM head only on (at most) this many rows whose label is not -100. Rows with
        # an ignored label contribute neither loss nor gradient, so the result is identical; PersonaChat
        # batches score only the last candidate's reply, i.e. ~1/8 of the rows at the bench shape.
        self.lm_row_capacity = 0
        # residual adds fused into the following LayerNorm (fwd) / its input gradient (bwd)
        # (default on since the fused MLP GEMMs)
        self.fuse_add_ln = os.environ.get("ADAPCC_FUSE_ADD_LN", "1") == "1"
        # wte[ids] + wpe[pos] + wte[token types] as one kernel, sort-free fp32-accumulating backward
        # (csrc/ops_embed.cu); the flat engine gives both tables a gradient sink (parallel/engine.py)
        self.fused_embed = os.environ.get("ADAPCC_FUSED_EMBED", "1") != "0"
        if self.fused_embed:
            self.wte.weight._adapcc_embed_table = True
            self.wpe.weight._adapcc_embed_table = True
        self._pos_cache = {}
        for name, p in (("embd_pdrop", cfg.embd_pdrop), ("resid_pdrop", cfg.resid_pdrop),
                        ("summary_first_dropout", cfg.summary_first_dropout)):
            check_p(f"GPT2Config.{name}", p)
        # The arguments of every dropout mask (ops/dropout.py), on the model's device so that a captured step reads
        # the current values. Plain attributes that _apply moves with the module, NOT buffers: state_dict() keeps its
        # keys (the engine checkpoints them), and DistributedDataParallel, which broadcasts rank 0's buffers at
        # construction and before every forward, neither overwrites the per-rank seeds nor gains a collective per step.
        self.dropout_seed = torch.zeros(1, dtype=torch.int64)
        self.dropout_step = torch.zeros(1, dtype=torch.int32)
        self.apply(self._init)
        for blk in self.h:                                  # GPT-2 residual-projection scaling
            for lin in (blk.c_proj, blk.c_proj2):
                nn.init.normal_(lin.weight, std=cfg.initializer_range / math.sqrt(2 * cfg.n_layer))

    def _init(self, m):
        if isinstance(m, (nn.Linear, nn.Embedding)):
            nn.init.normal_(m.weight, std=self.cfg.initializer_range)
            if isinstance(m, nn.Linear) and m.bias is not None:
                nn.init.zeros_(m.bias)

    def _apply(self, fn, *args, **kwargs):
        """``.to`` / ``.cuda`` / ``.bfloat16`` ...: the dropout state follows the parameters' device (a conversion of
        the floating-point dtype leaves the two integer tensors as they are, as it would leave integer buffers)."""
        super()._apply(fn, *args, **kwargs)
        self.dropout_seed, self.dropout_step = fn(self.dropout_seed), fn(self.dropout_step)
        return self

    def num_parameters(self) -> int:
        return sum(p.numel() for p in self.parameters())

    @property
    def has_dropout(self) -> bool:
        """Whether any dropout probability of the configuration is non-zero."""
        cfg = self.cfg
        return cfg.embd_pdrop > 0 or cfg.resid_pdrop > 0 or cfg.summary_first_dropout > 0

    def set_dropout(self, seed: int, step: int = 0) -> None:
        """The seed of the dropout masks and the number of training forwards already run (in place: a captured step
        keeps reading the same tensors). Two models with equal parameters, seed and step train alike bit for bit.
        The state is per process: data-parallel ranks that should draw different masks get different seeds, and
        DistributedDataParallel does not synchronise it."""
        fresh = DropoutState.create(seed, step)
        self.dropout_seed.copy_(fresh.seed)
        self.dropout_step.copy_(fresh.step)

    def dropout_state(self) -> DropoutState:
        """The model's seed and step buffers as the ``DropoutState`` the ops take (views, not copies)."""
        return DropoutState(self.dropout_seed, self.dropout_step)

    def _begin_dropout(self) -> Optional[DropoutState]:
        """The state of an active training forward, its step counter advanced; None when nothing drops.

        The counter advances HERE, before the first mask of the step is drawn, and nowhere else: the backward
        recomputes its masks from the counter, so it must read the value the forward read, and the next forward the
        next one. Advancing at the end of the forward would hand the backward the next step's masks."""
        if not (self.training and self.has_dropout):
            return None
        state = self.dropout_state()
        state.advance()
        return state

    def hidden(self, input_ids: torch.Tensor, token_type_ids: Optional[torch.Tensor], cache: Optional["KVCache"] = None,
               lengths: Optional[Sequence[int]] = None, drop: Optional[DropoutState] = None) -> torch.Tensor:
        """Final-LayerNorm hidden states [N, T, D]. With ``cache`` this is also the prefill of incremental decoding:
        every layer's keys and values of positions 0..T-1 go into the cache and its lengths become ``lengths`` (the real
        length of each right-padded row; default T for all). Causal attention makes the padding invisible to the real
        tokens, and ``decode_step`` overwrites the padded slots. ``drop``: the state of an active training forward
        (``forward`` passes it; never together with a cache, so no decoding path drops whatever the mode)."""
        N, T = input_ids.shape
        if cache is not None:
            if drop is not None:
                raise ValueError("hidden: dropout and a KV cache exclude each other")
            cache.reset(lengths if lengths is not None else [T] * N, T)
        cfg = self.cfg
        embd = (cfg.embd_pdrop, drop, site_embed()) if drop is not None and cfg.embd_pdrop > 0 else None
        resid = (cfg.resid_pdrop, drop) if drop is not None and cfg.resid_pdrop > 0 else None
        return self._blocks(self._embed(input_ids, token_type_ids, drop=embd), cache, resid)

    def _embed(self, ids: torch.Tensor, tt: Optional[torch.Tensor], pos: Optional[torch.Tensor] = None,
               drop=None) -> torch.Tensor:
        """wte[ids] + wpe[pos] (+ wte[tt]), added in that order: [*ids.shape, D]; ``pos`` defaults to 0..T-1 in every
        row of ids [N, T]. One ``fused_embedding_sum`` for bf16 CUDA tables if ``fused_embed``. ``drop = (p, state,
        site)``: dropout of the sum."""
        if (self.fused_embed and ids.is_cuda and self.wte.weight.dtype == torch.bfloat16
                and self.wpe.weight.dtype == torch.bfloat16):
            from ..ops import fused_embedding_sum
            if pos is None:                  # cached: a captured training step reads the same positions every replay
                N, T = ids.shape
                pos = self._pos_cache.get((N, T, ids.device))
                if pos is None:
                    pos = self._pos_cache[(N, T, ids.device)] = torch.arange(T, device=ids.device).repeat(N)
            lookups = [(0, ids), (1, pos)] + ([(0, tt)] if tt is not None else [])
            return fused_embedding_sum([self.wte.weight, self.wpe.weight], lookups, drop).view(*ids.shape, -1)
        # the default positions broadcast over the rows, so wpe's gradient is summed over them before the lookup
        x = self.wte(ids) + self.wpe(torch.arange(ids.shape[-1], device=ids.device) if pos is None else pos)
        if tt is not None:
            x = x + self.wte(tt)
        return x if drop is None else dropout(x, *drop)

    def lm_logits(self, h: torch.Tensor, head: Optional[torch.Tensor] = None) -> torch.Tensor:
        """fp32 logits [..., vocab_size] of ``h`` [..., D] through the tied head; ``head``: a kept fp32 ``wte.weight``."""
        if head is None:
            head = self.wte.weight.float()
        return (h.float() @ head.t())[..., :self.cfg.vocab_size]

    def _blocks(self, x: torch.Tensor, cache: Optional["KVCache"], drop=None) -> torch.Tensor:
        """``drop = (p, state)``: residual dropout; the final add-LayerNorm carries the last block's MLP site."""
        if self.fuse_add_ln:
            delta = None
            for i, blk in enumerate(self.h):
                x, delta = blk.forward_deferred(x, delta, cache, i, drop)
            return self.ln_f.forward_add(x, delta, drop and (*drop, site_mlp(len(self.h) - 1)))[1]
        for i, blk in enumerate(self.h):
            x = blk(x, cache, i, drop)
        return self.ln_f(x)

    def new_cache(self, batch: int, t_max: Optional[int] = None, kv_cache_dtype: Optional[str] = None) -> "KVCache":
        """An empty KV cache for ``batch`` rows of up to ``t_max`` (default ``n_positions``) tokens, on the model's
        device and in its dtype, or in fp8 with ``kv_cache_dtype="fp8_e4m3"`` (``ops/kvcache.py``)."""
        cfg = self.cfg
        t_max = cfg.n_positions if t_max is None else int(t_max)
        if not 1 <= t_max <= cfg.n_positions:
            raise ValueError(f"new_cache: t_max must be in [1, {cfg.n_positions}], got {t_max}")
        w = self.wte.weight
        return KVCache(cfg.n_layer, batch, cfg.n_head, t_max, cfg.n_embd // cfg.n_head, w.dtype, w.device,
                       kv_cache_dtype)

    @torch.no_grad()
    def decode_step(self, input_ids: torch.Tensor, token_type_ids: Optional[torch.Tensor], cache: "KVCache") -> torch.Tensor:
        """One step of incremental decoding: ``input_ids`` [B] (and ``token_type_ids`` [B]) are the next token of each
        row, at position ``cache.lens[b]``; returns their final-LayerNorm hidden state [B, D] and advances the cache by
        one. The same modules and fused-add LayerNorm structure as ``hidden``; attention runs over the cache through
        ``decode_attention``. No host sync, so a step can be captured in a CUDA graph (``DecodeGraph``). Raises
        ``ValueError`` before launching anything if a row's cache is full."""
        B = input_ids.shape[0]
        if input_ids.dim() != 1 or B != cache.batch:
            raise ValueError(f"decode_step: input_ids must be [{cache.batch}], got {tuple(input_ids.shape)}")
        cache.check_room()
        h = self._blocks(self._embed(input_ids, token_type_ids, cache.lens.long()), cache)
        cache.advance()
        return h

    def _decode_setup(self, who: str, input_ids: torch.Tensor, lengths: Optional[Sequence[int]],
                      token_type_ids: Optional[torch.Tensor], reply_type, max_new_tokens: int, min_new_tokens: int,
                      repetition_penalty: float, no_repeat_ngram_size: int, num_beams: int = 1,
                      rows_name: str = "beam rows (batch x num_beams)", sequence_bias=None, bad_words_ids=None,
                      stop_ids: Sequence[int] = (), kv_cache_dtype: Optional[str] = None,
                      frequency_penalty: float = 0.0, presence_penalty: float = 0.0,
                      context_no_repeat_ngram_size: int = 0):
        """The checks and prompt quantities the batched decoders share, before anything is launched:
        ``(B, T, lengths, n, t_max, last, tt_new, native, controls)``. ``last`` [B] is each prompt's last position,
        ``tt_new`` [B] the token type of new tokens (None without token types), ``native`` says whether the bf16 CUDA
        kernels run; they take at most ``LM_HEAD_MAX_ROWS`` rows, ``num_beams`` per prompt (called ``rows_name`` in
        the error when more than one). ``controls`` are the keyword arguments of ``_Repeats.create`` after the
        decoder's own: the repetition penalty and n-gram size, ``bias`` the table of ``sequence_bias`` and
        ``bad_words_ids`` (``ops.repeats.check_sequence_bias_args``; None when both are off), and the frequency,
        presence and context n-gram settings. ``kv_cache_dtype`` must be None or one of
        ``ops.kvcache.KV_CACHE_DTYPES``. Errors name ``who``."""
        from ..ops import LM_HEAD_MAX_ROWS

        if input_ids.dim() != 2 or input_ids.shape[0] < 1 or input_ids.shape[1] < 1:
            raise ValueError(f"{who}: input_ids must be [B, T], got {tuple(input_ids.shape)}")
        B, T = input_ids.shape
        dev = input_ids.device
        lengths = [T] * B if lengths is None else [int(x) for x in lengths]
        if len(lengths) != B or any(not 1 <= x <= T for x in lengths):
            raise ValueError(f"{who}: need {B} lengths in [1, {T}], got {lengths}")
        n = int(max_new_tokens)
        if n < 1 or int(min_new_tokens) < 0:
            raise ValueError(f"{who}: need max_new_tokens >= 1 and min_new_tokens >= 0, got {max_new_tokens}, "
                             f"{min_new_tokens}")
        check_repeat_args(who, repetition_penalty, no_repeat_ngram_size, frequency_penalty, presence_penalty,
                          context_no_repeat_ngram_size)
        check_kv_cache_dtype(who, kv_cache_dtype)
        bias = check_sequence_bias_args(who, sequence_bias, bad_words_ids, self.cfg.vocab_size, stop_ids)
        t_max = max(lengths) + n
        if t_max > self.cfg.n_positions:
            raise ValueError(f"{who}: the longest prompt ({max(lengths)}) plus max_new_tokens ({n}) exceeds "
                             f"n_positions = {self.cfg.n_positions}")
        weight = self.wte.weight
        native = weight.is_cuda and weight.dtype == torch.bfloat16
        if native and B * num_beams > LM_HEAD_MAX_ROWS:
            what, got = ("rows", B) if num_beams == 1 else (rows_name, f"{B} x {num_beams}")
            raise ValueError(f"{who}: at most {LM_HEAD_MAX_ROWS} {what} per call on the native path, got {got}")
        last = torch.tensor(lengths, device=dev) - 1
        tt_new = None
        if reply_type is not None:
            tt_new = torch.as_tensor(reply_type, dtype=torch.int64).to(dev).expand(B).contiguous()
        elif token_type_ids is not None:
            tt_new = token_type_ids[torch.arange(B, device=dev), last].contiguous()
        controls = dict(penalty=repetition_penalty, ngram=no_repeat_ngram_size, bias=bias,
                        frequency=float(frequency_penalty), presence=float(presence_penalty),
                        context_ngram=int(context_no_repeat_ngram_size))
        return B, T, lengths, n, t_max, last, tt_new, native, controls

    @staticmethod
    def _beam_args(who: str, num_beams: int, stop_ids: Sequence[int], suppress_ids: Sequence[int], sample: bool,
                   temperature: float, top_k: int, top_p: float, filters: Optional[dict] = None) -> int:
        """The argument checks the beam decoders share, before anything is launched: ``num_beams``, the stop and
        suppress list sizes and, with ``sample``, the sampling scalars and the truncation ``filters`` (keyword
        arguments of ``check_filter_args``). Returns K. Errors name ``who``."""
        from ..ops import BEAM_MAX_BEAMS, BEAM_MAX_STOP, BEAM_MAX_SUPPRESS

        K = int(num_beams)
        if not 1 <= K <= BEAM_MAX_BEAMS:
            raise ValueError(f"{who}: num_beams must be in [1, {BEAM_MAX_BEAMS}], got {num_beams}")
        if len(stop_ids) > BEAM_MAX_STOP:
            raise ValueError(f"{who}: at most {BEAM_MAX_STOP} stop_ids, got {len(stop_ids)}")
        if len(suppress_ids) > BEAM_MAX_SUPPRESS:
            raise ValueError(f"{who}: at most {BEAM_MAX_SUPPRESS} suppress_ids, got {len(suppress_ids)}")
        if sample and not temperature > 0:
            raise ValueError(f"{who}: sampling needs temperature > 0, got {temperature}")
        if sample and int(top_k) < 0:
            raise ValueError(f"{who}: top_k must be >= 0, got {top_k}")
        if sample and not 0 < top_p <= 1:
            raise ValueError(f"{who}: top_p must be in (0, 1], got {top_p}")
        if sample and filters:
            check_filter_args(who, **filters)
        return K

    def _guidance_rows(self, input_ids: torch.Tensor, token_type_ids: Optional[torch.Tensor], lengths: List[int],
                       last: torch.Tensor, tt_new: Optional[torch.Tensor], negative_prompt_ids: Optional[torch.Tensor],
                       neg_lengths: List[int], negative_token_type_ids: Optional[torch.Tensor]):
        """``generate``'s 2B prefill rows with guidance: the prompts, then the negative prompts (each row's last prompt
        token when ``negative_prompt_ids`` is None), right-padded to one width. Returns ``(ids, token types or None,
        lengths, token types of new tokens [2B] or None)``."""
        B, T = input_ids.shape
        dev = input_ids.device
        rows = torch.arange(B, device=dev)
        if negative_prompt_ids is None:
            neg, neg_tt = input_ids[rows, last][:, None], None
            if token_type_ids is not None:
                neg_tt = token_type_ids[rows, last][:, None]
        else:
            neg, neg_tt = negative_prompt_ids.to(dev), negative_token_type_ids
            if neg_tt is None and token_type_ids is not None:
                neg_tt = tt_new[:, None].expand(neg.shape)
        Tn = neg.shape[1]
        ids = torch.zeros(2 * B, max(T, Tn), dtype=input_ids.dtype, device=dev)
        ids[:B, :T], ids[B:, :Tn] = input_ids, neg
        tt = None
        if token_type_ids is not None:
            tt = torch.zeros_like(ids, dtype=token_type_ids.dtype)
            tt[:B, :T], tt[B:, :Tn] = token_type_ids, neg_tt.to(dev)
        return ids, tt, list(lengths) + list(neg_lengths), None if tt_new is None else tt_new.repeat(2)

    @torch.no_grad()
    def generate(self, input_ids: torch.Tensor, lengths: Optional[Sequence[int]] = None,
                 token_type_ids: Optional[torch.Tensor] = None, reply_type=None, max_new_tokens: int = 20,
                 temperature: float = 0.7, top_k: int = 0, top_p: float = 0.9, stop_ids: Sequence[int] = (),
                 suppress_ids: Sequence[int] = (), min_new_tokens: int = 0, seed=0, repetition_penalty: float = 1.0,
                 no_repeat_ngram_size: int = 0, prompt_lookup_num_tokens: int = 0,
                 max_matching_ngram_size: int = 2, min_p: float = 0.0, typical_p: float = 1.0,
                 epsilon_cutoff: float = 0.0, eta_cutoff: float = 0.0, assistant_model: "GPT2DoubleHeads" = None,
                 num_assistant_tokens: int = 4,
                 assistant_verification: str = "coupled", guidance_scale: float = 1.0,
                 negative_prompt_ids: Optional[torch.Tensor] = None, negative_lengths: Optional[Sequence[int]] = None,
                 negative_token_type_ids: Optional[torch.Tensor] = None, sequence_bias=None,
                 bad_words_ids=None, top_h: float = 0.0,
                 kv_cache_dtype: Optional[str] = None, frequency_penalty: float = 0.0,
                 presence_penalty: float = 0.0,
                 context_no_repeat_ngram_size: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
        """Batched, seeded top-k / top-p sampling of up to ``max_new_tokens`` tokens per row.

        ``input_ids`` [B, T] is right-padded; row b's prompt is its first ``lengths[b]`` tokens (default T).
        ``reply_type`` (an int or a [B] tensor) is the token type of the new tokens; by default each row's last prompt
        token type when ``token_type_ids`` is given. ``seed``: an int (row b uses ``seed + b``) or an int64 [B] tensor.
        While fewer than ``min_new_tokens`` tokens are generated, ``suppress_ids`` cannot be drawn; a token in
        ``stop_ids`` ends its row. ``temperature == 0`` is greedy. The draw of each token is defined in
        ``ops/sampling.py``: a row's tokens depend on its prompt, its seed and the scalars, not on the other rows.
        ``repetition_penalty`` (1: off) and ``no_repeat_ngram_size`` (0: off) act on each row's logits first, over its
        prompt and the tokens generated so far (``ops/repeats.py``). Before them, ``sequence_bias`` (HuggingFace's:
        a dict ``{tuple(ids): bias}`` or a list of ``[ids, bias]`` pairs, finite biases) adds each bias to the logit
        of a sequence's last id when the row's prompt and tokens end with the sequence's other ids, and
        ``bad_words_ids`` (a list of id lists; a one-token list in ``stop_ids`` is dropped) does the same with -inf,
        so no listed sequence is ever produced; at most ``ops.repeats.BIAS_MAX_ENTRIES`` entries of at most
        ``BIAS_MAX_LEN`` ids in all, one table for every row. ``frequency_penalty`` and ``presence_penalty`` (the
        OpenAI / vLLM penalties; any finite values, 0: off) act after the repetition penalty: each id that occurs c
        times among the row's generated tokens (the prompt does not count) loses ``c * frequency_penalty``, then
        ``presence_penalty``. ``context_no_repeat_ngram_size`` = m (0: off; ParlAI's ``beam_context_block_ngram``)
        bans, after ``no_repeat_ngram_size``, every id that would complete an m-gram found inside the row's prompt;
        m = 1 bans every prompt id. ``min_p`` (0: off), ``typical_p`` (1: off),
        ``epsilon_cutoff`` (0: off) and ``eta_cutoff`` (0: off) are HuggingFace's truncation samplers: at temperature
        > 0 they filter, in that order, the ids that top-k and top-p kept, just before the draw (inside
        ``ops.sample_tokens_`` on the native path). ``top_h`` (in (0, 1]; 0: off; 1 is on) is HuggingFace's
        entropy-bounded top-h: of the row's 100 largest values it keeps the longest prefix, by value, whose partial
        entropy stays within ``top_h`` times their entropy; it acts before top-k. At temperature 0 no filter has an
        effect.

        Returns ``(tokens, n_new)``: int64 [B, max_new_tokens] (-1 after a row stopped) and the tokens per row.

        The prompts are prefilled into a KV cache of ``max(lengths) + max_new_tokens`` positions (``ValueError`` if that
        exceeds ``n_positions``: there is no sliding window here, ``sample_sequence`` has one). On CUDA with bf16
        weights the LM head and the sampler are native kernels (``ops.lm_head_logits_``, ``ops.sample_tokens_``) and
        every token after the first replays one CUDA graph of decode step, LM head (``ops.penalize_repeats_`` when a
        repetition control, penalty or sequence bias is on) and sampler, which feeds the drawn ids back into its own
        input; the host reads the done flags once every 8 tokens, a step late, to stop early. Elsewhere the same loop
        runs eagerly with fp32 PyTorch logits, ``ops.repeats.penalize_repeats_reference`` and
        ``ops.sampling.sample_reference``.

        ``prompt_lookup_num_tokens`` = k > 0 (HuggingFace's prompt lookup decoding; greedy only, without the repetition
        controls, the penalties or the sequence bias) verifies up to k draft tokens per row and step, copied from the
        row's own prompt and reply after the earliest earlier occurrence of its last ``max_matching_ngram_size`` (or
        fewer) tokens; the result is the greedy tokens. The definition is in ``ops/lookup.py``. On the native path
        (``B·(k+1)`` at most 64 rows) every verify step replays one CUDA graph: the drafts (``ops.lookup_draft_``), the model on k + 1 slots per row
        (``ops.verify_attention_``), the LM head, the slots' arg-maxes (``ops.lookup_argmax_``) and acceptance
        (``ops.lookup_accept_``); the host polls the done flags every ``LOOKUP_POLL_PERIOD`` replays. Afterwards
        ``self.lookup_stats`` holds the rows' emitted tokens (a stop id included) and verify steps, int32 [B], and the
        graph replays issued.

        ``assistant_model`` (HuggingFace's assisted generation; a ``GPT2DoubleHeads`` with the same vocabulary, bf16 on
        the same device on the native path; not with prompt lookup or the repetition controls) drafts up to
        ``num_assistant_tokens`` = k tokens per row and round, which the model verifies in one step. Every emitted token
        is drawn from the same seed, position and step as in plain ``generate``, greedy or sampled, so given the same
        per-position logits the tokens are those of plain ``generate``; the draft changes only the speed. The definition
        is in ``ops/assisted.py``. On the native path (``B·(k+1)`` at most 64 rows) a round replays one CUDA graph: the
        draft's k + 1 decode steps with k draws (``ops.sample_slots_``), the model on k + 1 slots per row, the LM head,
        the slots' draws (arg-maxes at temperature 0) and acceptance (``ops.lookup_accept_``). Afterwards
        ``self.assist_stats`` holds what ``lookup_stats`` holds for prompt lookup.

        ``assistant_verification`` is that rule, ``"coupled"``, or ``"rejection"``: HuggingFace's rejection sampling
        (Leviathan et al. 2023), where a draft d is accepted with probability ``min(1, P(d) / Q(d))`` of the model's
        and the draft's filtered distributions and a rejection is replaced by a draw from ``max(0, P - Q)``. Each
        emitted token is then distributed as the model's, acceptance is their overlap rather than the agreement of
        two draws, and the tokens depend on the draft. On the native path the draft draws also keep their weights and
        the verify step runs ``ops.spec_slots_`` and ``ops.lookup_accept_(..., flagged=True)``. At temperature
        0 both rules are the greedy one.

        ``guidance_scale`` = g != 1 is HuggingFace's classifier-free guidance (``UnbatchedClassifierFreeGuidance
        LogitsProcessor``; the definition is in ``ops/guidance.py``; any finite g, 1: off). Each row also decodes a
        negative prompt, ``negative_prompt_ids`` [B, Tn] right-padded to ``negative_lengths`` (default Tn), by default
        the row's last prompt token alone with its token type; the negative rows consume the tokens the prompt rows
        draw. Each token's scores become ``g * (lc - lu) + lu`` of the two rows' log-softmaxes, before the repetition
        controls and sequence bias (which see the prompt rows' sequences only) and the sampler. When the prompts have
        ``token_type_ids``, negative prompts take ``negative_token_type_ids``, else the type of the new tokens; new
        tokens take the same type in both rows. Not with prompt lookup or an assistant. The cache then holds 2B rows, prompts
        first (at most ``LM_HEAD_MAX_ROWS`` on the native path), prefilled together; on the native path each graph
        replay runs the decode step and LM head on all of them and ``ops.guidance_mix_`` after the head. Prompt rows
        draw from the same seeds and positions as without guidance.

        ``kv_cache_dtype="fp8_e4m3"`` keeps the KV cache in fp8 (``ops/kvcache.py``): each cached key and value vector
        as e4m3 bytes with a power-of-two scale, half the bytes of bf16 for every decode step to read. Every cached
        position is quantized, the prompt's included; the prefill attends to the unquantized keys and values, and each
        new token to its own. On the native path the prefill quantizes through ``ops.kv_quantize_`` and every step
        runs the fp8 ``ops.decode_attention_``. Not with prompt lookup or an assistant (``ValueError``)."""
        if not temperature >= 0 or int(top_k) < 0 or not 0 < top_p <= 1:
            raise ValueError(f"generate: need temperature >= 0, top_k >= 0 and 0 < top_p <= 1, got {temperature}, "
                             f"{top_k}, {top_p}")
        check_filter_args("generate", min_p, typical_p, epsilon_cutoff, eta_cutoff, top_h)
        filters = dict(min_p=min_p, typical_p=typical_p, epsilon_cutoff=epsilon_cutoff, eta_cutoff=eta_cutoff,
                       top_h=top_h)
        from ..ops.assisted import check_verification
        check_verification("generate", assistant_verification, assistant_model)
        B0 = input_ids.shape[0] if input_ids.dim() == 2 else 0
        neg_lengths = check_guidance_args("generate", guidance_scale, B0, negative_prompt_ids, negative_lengths,
                                          negative_token_type_ids, token_type_ids, max_new_tokens, self.cfg.n_positions)
        guided = neg_lengths is not None
        speculative = assistant_model is not None or prompt_lookup_num_tokens != 0
        if speculative and kv_cache_dtype is not None:
            raise ValueError("generate: kv_cache_dtype cannot be combined with prompt_lookup_num_tokens or "
                             f"assistant_model (got {kv_cache_dtype!r}, {prompt_lookup_num_tokens}, "
                             f"{type(assistant_model).__name__})")
        if speculative and (sequence_bias or bad_words_ids):
            raise ValueError("generate: sequence_bias and bad_words_ids cannot be combined with "
                             f"prompt_lookup_num_tokens or assistant_model (got {prompt_lookup_num_tokens}, "
                             f"{type(assistant_model).__name__})")
        if speculative and (frequency_penalty != 0 or presence_penalty != 0 or context_no_repeat_ngram_size != 0):
            raise ValueError("generate: frequency_penalty, presence_penalty and context_no_repeat_ngram_size cannot be "
                             f"combined with prompt_lookup_num_tokens or assistant_model (got {frequency_penalty}, "
                             f"{presence_penalty}, {context_no_repeat_ngram_size}, {prompt_lookup_num_tokens}, "
                             f"{type(assistant_model).__name__})")
        if guided and (assistant_model is not None or prompt_lookup_num_tokens != 0):
            raise ValueError("generate: guidance_scale != 1 cannot be combined with prompt_lookup_num_tokens or "
                             f"assistant_model (got {prompt_lookup_num_tokens}, {type(assistant_model).__name__})")
        if assistant_model is not None or prompt_lookup_num_tokens != 0:
            from ..ops import LOOKUP_MAX_NGRAM, LOOKUP_MAX_TOKENS
            if assistant_model is not None:
                from ..ops.assisted import check_assist_args
                check_assist_args("generate", self, assistant_model, num_assistant_tokens, LOOKUP_MAX_TOKENS,
                                  prompt_lookup_num_tokens, repetition_penalty, no_repeat_ngram_size)
                K, ngram = num_assistant_tokens, 1
            else:
                from ..ops.lookup import check_lookup_args
                check_lookup_args("generate", prompt_lookup_num_tokens, max_matching_ngram_size, LOOKUP_MAX_TOKENS,
                                  LOOKUP_MAX_NGRAM, temperature, repetition_penalty, no_repeat_ngram_size)
                K, ngram = prompt_lookup_num_tokens, max_matching_ngram_size
            return self._generate_speculative(assistant_model, int(K), int(ngram), input_ids, lengths, token_type_ids,
                                              reply_type, max_new_tokens, temperature, top_k, top_p, stop_ids,
                                              suppress_ids, min_new_tokens, seed, filters,
                                              assistant_verification == "rejection" and temperature > 0)
        B, T, lengths, n, t_max, last, tt_new, native, controls = self._decode_setup(
            "generate", input_ids, lengths, token_type_ids, reply_type, max_new_tokens, min_new_tokens,
            repetition_penalty, no_repeat_ngram_size, num_beams=2 if guided else 1,
            rows_name="rows with guidance (batch x 2)", sequence_bias=sequence_bias, bad_words_ids=bad_words_ids,
            stop_ids=stop_ids, kv_cache_dtype=kv_cache_dtype, frequency_penalty=frequency_penalty,
            presence_penalty=presence_penalty, context_no_repeat_ngram_size=context_no_repeat_ngram_size)
        dev, V = input_ids.device, self.cfg.vocab_size
        seeds = _row_seeds(seed, B, dev)
        if guided:                                  # rows [0, B): the prompts, rows [B, 2B): the negative prompts
            ids_all, tt_all, lengths_all, tt_new = self._guidance_rows(
                input_ids, token_type_ids, lengths, last, tt_new, negative_prompt_ids, neg_lengths,
                negative_token_type_ids)
            t_max = max(lengths_all) + n
            last = torch.tensor(lengths_all, device=dev) - 1
        else:
            ids_all, tt_all, lengths_all = input_ids, token_type_ids, lengths
        R = len(lengths_all)
        cache = self.new_cache(R, t_max, kv_cache_dtype)
        h = self.hidden(ids_all, tt_all, cache=cache, lengths=lengths_all)[torch.arange(R, device=dev), last]
        tokens = torch.full((B, n), -1, dtype=torch.int64, device=dev)
        reps = _Repeats.create(input_ids, cache, V, rows=B, **controls)
        if not native:                              # CPU / not bf16: the fp64 definition on fp32 PyTorch logits
            head = self.wte.weight.float()
            done = torch.zeros(B, dtype=torch.int32)
            for i in range(n):
                if i:
                    h = self.decode_step(nxt.to(dev).repeat(R // B), tt_new, cache)
                logits = self.lm_logits(h, head)
                if guided:
                    logits = guided_scores_reference(logits[:B], logits[B:], V, guidance_scale).float()
                if reps is not None:
                    logits = reps.eager(logits, cache, nxt if i else None)
                nxt, tok, done = sample_reference(logits, V, temperature, top_k, top_p, seeds, cache.lens[:B], i,
                                                  min_new_tokens, suppress_ids, stop_ids, done, **filters)
                tokens[:, i] = tok.to(dev)
                if bool(done.all()):
                    break
            return tokens, (tokens >= 0).sum(1)

        from ..ops import guidance_mix_, lm_head_logits_, sample_tokens_

        weight = self.wte.weight
        logits = torch.empty(R, weight.shape[0], dtype=torch.float32, device=dev)
        next_ids = torch.zeros(R, dtype=torch.int64, device=dev)
        done = torch.zeros(B, dtype=torch.int32, device=dev)
        step = torch.zeros(1, dtype=torch.int32, device=dev)
        sup, stop = (torch.tensor(list(x), dtype=torch.int32, device=dev) for x in (suppress_ids, stop_ids))
        # the prompt rows (all rows without guidance)
        lg, lens, ids = logits[:B], cache.lens[:B], next_ids[:B]

        def head_and_sample(hidden):
            lm_head_logits_(hidden, weight, logits)
            if guided:
                guidance_mix_(logits, V, B, guidance_scale)
            if reps is not None:
                reps.native(lg, lens, step, ids)
            sample_tokens_(lg, V, temperature, top_k, top_p, seeds, lens, step,
                           min_new_tokens, sup, stop, done, ids, tokens, **filters)
            if guided:                              # the negative rows consume the prompt rows' tokens
                next_ids[B:].copy_(ids)

        head_and_sample(h)                          # the first token, from the prefill's last positions
        if n > 1:
            # the sampler writes each token's ids into the graph's own input buffer
            DecodeGraph(self, cache, tt_new is not None, head=head_and_sample, ids=next_ids, tt=tt_new).run(n - 1, done)
        return tokens, (tokens >= 0).sum(1)

    @torch.no_grad()
    def beam_search(self, input_ids: torch.Tensor, lengths: Optional[Sequence[int]] = None,
                    token_type_ids: Optional[torch.Tensor] = None, reply_type=None, num_beams: int = 4,
                    max_new_tokens: int = 20, length_penalty: float = 1.0, stop_ids: Sequence[int] = (),
                    suppress_ids: Sequence[int] = (), min_new_tokens: int = 0, repetition_penalty: float = 1.0,
                    no_repeat_ngram_size: int = 0, do_sample: bool = False, temperature: float = 1.0,
                    top_k: int = 0, top_p: float = 1.0, seed=0,
                    num_return_sequences: int = 1, num_beam_groups: int = 1, diversity_penalty: float = 0.0,
                    sequence_bias=None, bad_words_ids=None, min_p: float = 0.0, typical_p: float = 1.0,
                    epsilon_cutoff: float = 0.0, eta_cutoff: float = 0.0, top_h: float = 0.0,
                    kv_cache_dtype: Optional[str] = None, frequency_penalty: float = 0.0,
                    presence_penalty: float = 0.0,
                    context_no_repeat_ngram_size: int = 0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Batched beam search with ``num_beams`` beams per prompt; the definition is in ``ops/beam.py``.

        ``input_ids`` [B, T] is right-padded; item b's prompt is its first ``lengths[b]`` tokens (default T).
        ``reply_type`` and the token types of new tokens work as in ``generate``. A token in ``stop_ids`` (at most 8)
        finishes a hypothesis; while fewer than ``min_new_tokens`` tokens are generated, ``suppress_ids`` cannot be
        chosen. A hypothesis of L tokens (its stop token included) scores ``sum of log-probabilities / L **
        length_penalty``. An item stops as soon as no live beam can beat its K-th finished hypothesis, which never
        changes its result. An item's result depends on its prompt and the scalars only, not on the other items.
        ``repetition_penalty`` (1: off) and ``no_repeat_ngram_size`` (0: off) act on each beam's logits before the
        log-softmax, over its prompt and its own hypothesis (``ops/repeats.py``), so its log-probabilities are
        renormalised over the ids that remain. So do ``sequence_bias`` and ``bad_words_ids`` (as in ``generate``),
        applied first: a biased beam's log-probabilities are renormalised too, where HuggingFace adds the bias to the
        log-probabilities after normalisation. ``frequency_penalty``, ``presence_penalty`` and
        ``context_no_repeat_ngram_size`` work as in ``generate``, over each beam's own hypothesis, also before the
        log-softmax.

        ``do_sample=True`` is beam sampling (HuggingFace's ``generate(do_sample=True, num_beams=K)``; the definition is
        ``ops.beam.BeamSampleReference``): each beam's ids are filtered by ``top_k`` (0: off) and ``top_p`` at
        ``temperature`` > 0, then by ``generate``'s truncation filters ``min_p``, ``typical_p``, ``epsilon_cutoff``
        and ``eta_cutoff``, with ``top_h`` before top-k, each keeping at least ``max(2, 1 + len(stop_ids))`` ids
        (HuggingFace's ``min_tokens_to_keep``; its top-h has none), and the candidates are drawn without replacement in
        proportion to ``exp(sum of log-probabilities / temperature)`` instead of ranked; the log-probabilities are
        those of the unfiltered row, as in HuggingFace. ``seed``: an int (item b uses ``seed + b``) or an int64 [B]
        tensor; an item's result depends on its prompt, its seed and the scalars. With ``do_sample=False`` the sampling
        arguments and the filters are ignored.

        ``num_beam_groups`` = G > 1 is diverse beam search (HuggingFace 4.x's ``num_beam_groups`` /
        ``diversity_penalty``; the definition is ``ops.beam.GroupBeamReference``): the beams form G groups of
        ``num_beams / G`` that select in order each step, a candidate's score lowered by ``diversity_penalty`` (finite,
        > 0) for each new beam of an earlier group of the item with the same token; each group keeps its own
        ``num_beams / G`` finished hypotheses and the results are their union, best first. G must divide
        ``num_beams``, cannot be combined with ``do_sample`` and, for G = 1, ``diversity_penalty`` must be 0.

        Returns ``(tokens, n_new, scores)``: the ``num_return_sequences`` = r (``1 <= r <= num_beams``) best hypotheses
        of each item, as rows ``b * r + q``, best first: int64 [B·r, max_new_tokens] (the stop token excluded, padded
        with -1), their lengths int64 [B·r] and their normalised scores fp32 [B·r]. An item with fewer than r
        finished hypotheses gets rows with no tokens, length 0 and score -inf.

        Each prompt is prefilled once and its keys and values copied to its ``num_beams`` rows of a cache of
        ``max(lengths) + max_new_tokens`` positions (more than ``n_positions`` is a ``ValueError``). On CUDA with bf16
        weights every token after the first replays one CUDA graph of decode step, LM head (``ops.lm_head_logits_``),
        the repetition controls and sequence bias when on (``ops.penalize_repeats_``), selection (``ops.beam_step_``) and cache
        reordering (``ops.kv_reorder_``), at most 64 beam rows per call; the host reads the done flags once every 8
        tokens, a period late. Beam sampling takes a vocabulary of at most ``ops.SAMPLE_MAX_VOCAB`` ids there, and
        the items' seeds are a device input of the graph. Elsewhere the same loop runs eagerly with fp32 PyTorch logits,
        ``ops.repeats.penalize_repeats_reference``, ``ops.beam.GroupBeamReference`` (``BeamSampleReference`` with
        ``do_sample``) and torch indexing.

        ``kv_cache_dtype="fp8_e4m3"`` keeps the KV cache in fp8 as in ``generate``; the cache reordering then moves
        the bytes and the scales."""
        from ..ops import SAMPLE_MAX_VOCAB, BeamState
        from ..ops.beam import BeamSampleReference, GroupBeamReference, best_hypotheses, merge_finished_sets

        do_sample = bool(do_sample)
        filters = dict(min_p=min_p, typical_p=typical_p, epsilon_cutoff=epsilon_cutoff, eta_cutoff=eta_cutoff,
                       top_h=top_h)
        K = self._beam_args("beam_search", num_beams, stop_ids, suppress_ids, do_sample, temperature, top_k, top_p,
                            filters)
        R = int(num_return_sequences)
        if not 1 <= R <= K:
            raise ValueError(f"beam_search: num_return_sequences must be in [1, num_beams = {K}], got "
                             f"{num_return_sequences}")
        G, lam = int(num_beam_groups), float(diversity_penalty)
        if not 1 <= G <= K or K % G != 0:
            raise ValueError(f"beam_search: num_beam_groups must divide num_beams = {K}, got {num_beam_groups}")
        if G > 1 and (do_sample or not (math.isfinite(lam) and lam > 0)):
            raise ValueError(f"beam_search: num_beam_groups > 1 needs do_sample=False and a finite diversity_penalty "
                             f"> 0, got do_sample={do_sample}, diversity_penalty={diversity_penalty}")
        if G == 1 and lam != 0:
            raise ValueError(f"beam_search: diversity_penalty needs num_beam_groups > 1, got {diversity_penalty}")

        def start(B, n, V, dev, native):
            seeds = _row_seeds(seed, B, dev) if do_sample else None
            if not native:                          # CPU / not bf16: the fp64 definition
                if do_sample:
                    return BeamSampleReference(B, K, n, V, length_penalty, stop_ids, suppress_ids, min_new_tokens,
                                               temperature=temperature, top_k=top_k, top_p=top_p,
                                               seeds=seeds.cpu().tolist(), **filters)
                return GroupBeamReference(B, K, n, V, length_penalty, stop_ids, suppress_ids, min_new_tokens,
                                          num_beam_groups=G, diversity_penalty=lam)
            if do_sample and V > SAMPLE_MAX_VOCAB:
                raise ValueError(f"beam_search: do_sample=True needs a vocabulary of at most {SAMPLE_MAX_VOCAB} ids "
                                 f"on the native path, got {V}")
            st = BeamState(B, K, n, length_penalty, dev, sample=do_sample, groups=G)
            return st, (dict(temperature=temperature, top_k=top_k, top_p=top_p, seeds=seeds, **filters) if do_sample
                         else dict(diversity_penalty=lam))

        sel = self._beam_decode("beam_search", input_ids, lengths, token_type_ids, reply_type, K, max_new_tokens,
                                min_new_tokens, repetition_penalty, no_repeat_ngram_size, stop_ids, suppress_ids, start,
                                sequence_bias, bad_words_ids, kv_cache_dtype, frequency_penalty=frequency_penalty,
                                presence_penalty=presence_penalty,
                                context_no_repeat_ngram_size=context_no_repeat_ngram_size)
        dev, B, n = input_ids.device, input_ids.shape[0], int(max_new_tokens)
        if not isinstance(sel, tuple):
            return tuple(t.to(dev) for t in sel.result(R))
        st = sel[0]
        fin = [merge_finished_sets(sets) for sets in st.finished()]
        hist_tok = st.hist_tok.view(n, B, K).cpu().numpy()
        hist_back = st.hist_back.view(n, B, K).cpu().numpy()
        return tuple(t.to(dev) for t in best_hypotheses(fin, hist_tok, hist_back, n, R))

    @torch.no_grad()
    def stochastic_beam_search(self, input_ids: torch.Tensor, lengths: Optional[Sequence[int]] = None,
                               token_type_ids: Optional[torch.Tensor] = None, reply_type=None, num_beams: int = 4,
                               max_new_tokens: int = 20, temperature: float = 1.0, top_k: int = 0,
                               top_p: float = 1.0, stop_ids: Sequence[int] = (), suppress_ids: Sequence[int] = (),
                               min_new_tokens: int = 0, repetition_penalty: float = 1.0,
                               no_repeat_ngram_size: int = 0, seed=0, sequence_bias=None, bad_words_ids=None,
                               min_p: float = 0.0, typical_p: float = 1.0, epsilon_cutoff: float = 0.0,
                               eta_cutoff: float = 0.0, top_h: float = 0.0, kv_cache_dtype: Optional[str] = None,
                               frequency_penalty: float = 0.0, presence_penalty: float = 0.0,
                               context_no_repeat_ngram_size: int = 0):
        """Stochastic beam search (Kool, van Hoof and Welling 2019): ``num_beams`` = K distinct replies per prompt,
        drawn without replacement from the law ``generate`` samples from with the same ``temperature``, ``top_k``,
        ``top_p``, truncation filters (``min_p``, ``typical_p``, ``epsilon_cutoff``, ``eta_cutoff``, ``top_h``), stop /
        suppress / ``min_new_tokens``, repetition settings, ``sequence_bias`` and ``bad_words_ids``, the frequency,
        presence and context n-gram settings and ``max_new_tokens``; the definition
        (rules R1-R8, properties P1-P4) is ``ops.beam.StochasticBeamReference``. The first reply of an item is itself
        an exact sample of that law. ``seed``: an int (item b uses ``seed + b``) or an int64 [B] tensor; an item's
        result depends on its prompt, its seed and the scalars only. The other arguments work as in ``beam_search``,
        ``kv_cache_dtype`` included.

        Returns ``(tokens, n_new, log_probs, keys, kappa)``: rows ``b·K + q``, the largest key first, of int64 [B·K,
        max_new_tokens] (the stop token excluded, padded with -1), int64 [B·K] lengths, fp32 [B·K] log-probabilities
        under the law and fp32 [B·K] perturbed keys (rows past an item's count have no tokens, length 0 and -inf),
        and the thresholds ``kappa`` fp32 [B]. With them ``ops.beam.sbs_estimate(f, log_probs, kappa)`` is an
        unbiased estimate of the expectation of any f of the reply (exact when kappa is -inf: then the K replies are
        the whole support).

        The decode loop is ``beam_search``'s: on CUDA with bf16 weights every token after the first replays one CUDA
        graph of decode step, LM head, the repetition controls and sequence bias when on, ``ops.beam_step_`` on a
        stochastic
        ``ops.BeamState`` and ``ops.kv_reorder_``; there a vocabulary of at most ``ops.SAMPLE_MAX_VOCAB`` ids and at
        most 64 beam rows per call. Elsewhere the same loop runs eagerly through ``StochasticBeamReference``. Bad
        arguments raise ``ValueError`` naming them before anything is launched."""
        from ..ops import SAMPLE_MAX_VOCAB, BeamState
        from ..ops.beam import StochasticBeamReference, stochastic_results

        who = "stochastic_beam_search"
        filters = dict(min_p=min_p, typical_p=typical_p, epsilon_cutoff=epsilon_cutoff, eta_cutoff=eta_cutoff,
                       top_h=top_h)
        K = self._beam_args(who, num_beams, stop_ids, suppress_ids, True, temperature, top_k, top_p, filters)
        scalars = dict(temperature=temperature, top_k=top_k, top_p=top_p, **filters)

        def start(B, n, V, dev, native):
            seeds = _row_seeds(seed, B, dev)
            if not native:
                return StochasticBeamReference(B, K, n, V, stop_ids, suppress_ids, min_new_tokens,
                                               seeds=seeds.cpu().tolist(), **scalars)
            if V > SAMPLE_MAX_VOCAB:
                raise ValueError(f"{who}: the vocabulary (vocab_size = {V}) must be at most {SAMPLE_MAX_VOCAB} ids on "
                                 f"the native path")
            return BeamState(B, K, n, 1.0, dev, seeds=seeds), scalars

        sel = self._beam_decode(who, input_ids, lengths, token_type_ids, reply_type, K, max_new_tokens,
                                min_new_tokens, repetition_penalty, no_repeat_ngram_size, stop_ids, suppress_ids, start,
                                sequence_bias, bad_words_ids, kv_cache_dtype, frequency_penalty=frequency_penalty,
                                presence_penalty=presence_penalty,
                                context_no_repeat_ngram_size=context_no_repeat_ngram_size)
        dev = input_ids.device
        if not isinstance(sel, tuple):
            return tuple(t.to(dev) for t in sel.result())
        st = sel[0]
        B, n = st.batch, st.max_new
        fin = [sets[0] for sets in st.finished()]
        out = stochastic_results(fin, st.hist_tok.view(n, B, K).cpu().numpy(), st.hist_back.view(n, B, K).cpu().numpy(),
                                 n, K, st.kappa.cpu().numpy())
        return tuple(t.to(dev) for t in out)

    def _beam_decode(self, who: str, input_ids: torch.Tensor, lengths, token_type_ids, reply_type, K: int,
                     max_new_tokens: int, min_new_tokens: int, repetition_penalty: float, no_repeat_ngram_size: int,
                     stop_ids: Sequence[int], suppress_ids: Sequence[int], start, sequence_bias=None,
                     bad_words_ids=None, kv_cache_dtype: Optional[str] = None, frequency_penalty: float = 0.0,
                     presence_penalty: float = 0.0, context_no_repeat_ngram_size: int = 0):
        """The decode loop of the beam decoders. ``start(B, n, V, device, native)`` is called after the argument checks
        and before anything is launched; it returns the selector: on the native path ``(BeamState, keyword arguments
        of beam_step_)``, elsewhere a reference with ``step(logits) -> (next_ids, parent)`` and ``done``. Each prompt
        is prefilled once and its keys and values copied to its K rows; every token then takes the LM head, the
        repetition controls and sequence bias when on, the selection and the cache reordering. On the native path every token after
        the first replays one CUDA graph of them and the host reads the done flags once every 8 tokens; elsewhere
        the same loop runs eagerly with fp32 PyTorch logits and torch indexing. Returns the selector."""
        from ..ops import beam_step_, kv_reorder_, kv_reorder_scratch_numel, lm_head_logits_

        B, T, lengths, n, t_max, last, tt_new, native, controls = self._decode_setup(
            who, input_ids, lengths, token_type_ids, reply_type, max_new_tokens, min_new_tokens,
            repetition_penalty, no_repeat_ngram_size, num_beams=K, sequence_bias=sequence_bias,
            bad_words_ids=bad_words_ids, stop_ids=stop_ids, kv_cache_dtype=kv_cache_dtype,
            frequency_penalty=frequency_penalty, presence_penalty=presence_penalty,
            context_no_repeat_ngram_size=context_no_repeat_ngram_size)
        dev, V, weight = input_ids.device, self.cfg.vocab_size, self.wte.weight
        sel = start(B, n, V, dev, native)
        if tt_new is not None:
            tt_new = tt_new.repeat_interleave(K)
        # one prefill per prompt, its keys and values copied to the prompt's K rows (the beams share that region)
        pre = self.new_cache(B, T, kv_cache_dtype)
        h = self.hidden(input_ids, token_type_ids, cache=pre, lengths=lengths)[torch.arange(B, device=dev), last]
        cache = self.new_cache(B * K, t_max, kv_cache_dtype)
        cache.reset([x for x in lengths for _ in range(K)], T)
        for dst, src in zip(cache.parts, pre.parts):
            dst[:, :, :, :T].copy_(src.repeat_interleave(K, dim=1))
        del pre
        h = h.repeat_interleave(K, dim=0).contiguous()
        reps = _Repeats.create(input_ids, cache, V, **controls)
        if not native:                              # CPU / not bf16: the fp64 definition on fp32 PyTorch logits
            head = weight.float()
            for i in range(n):
                if i:
                    h = self.decode_step(nxt.to(dev), tt_new, cache)
                logits = self.lm_logits(h, head)
                if reps is not None:
                    logits = reps.eager(logits, cache, nxt if i else None)
                nxt, parent = sel.step(logits)
                rows = parent.to(dev)
                for t in cache.parts:
                    t.copy_(t[:, rows])
                if reps is not None:
                    reps.reorder(rows)
                if sel.done.all():
                    break
            return sel

        st, scalars = sel
        logits = torch.empty(B * K, weight.shape[0], dtype=torch.float32, device=dev)
        sup, stop = (torch.tensor(list(x), dtype=torch.int32, device=dev) for x in (suppress_ids, stop_ids))
        prompt_len = cache.lens.clone()
        fp8 = cache.k_scale is not None
        scratch = torch.empty(kv_reorder_scratch_numel(cache.k, n, fp8=fp8), dtype=cache.k.dtype, device=dev)

        def select(hidden):
            lm_head_logits_(hidden, weight, logits)
            if reps is not None:
                reps.native(logits, cache.lens, st.step, st.next_ids, st.parent, K)
            beam_step_(logits, V, st, min_new_tokens, sup, stop, **scalars)
            kv_reorder_(cache.k, cache.v, st.parent, prompt_len, cache.lens, n, scratch, k_scale=cache.k_scale,
                        v_scale=cache.v_scale)

        select(h)                                   # the first selection, from the prefill's last positions
        if n > 1:
            # beam_step_ writes the new beams' tokens into the graph's own input buffer
            DecodeGraph(self, cache, tt_new is not None, head=select, ids=st.next_ids, tt=tt_new).run(n - 1, st.done)
        return sel

    def _generate_speculative(self, draft: Optional["GPT2DoubleHeads"], K: int, ngram: int, input_ids, lengths,
                              token_type_ids, reply_type, max_new_tokens, temperature, top_k, top_p, stop_ids,
                              suppress_ids, min_new_tokens, seed, filters,
                              rejection: bool) -> Tuple[torch.Tensor, torch.Tensor]:
        """``generate`` verifying up to ``K`` drafts per row and step. Without ``draft`` the drafts come from prompt
        lookup of up to ``ngram`` tokens (``ops/lookup.py``, greedy only), with it from that model
        (``ops/assisted.py``). The slots' tokens are arg-maxes at temperature 0, else coupled draws or, with
        ``rejection``, rejection sampling; one acceptance follows. The stats go to ``self.lookup_stats`` or
        ``self.assist_stats``."""
        arg = "prompt_lookup_num_tokens" if draft is None else "num_assistant_tokens"
        B, T, lengths, n, t_max, last, tt_new, native, _ = self._decode_setup(
            "generate", input_ids, lengths, token_type_ids, reply_type, max_new_tokens, min_new_tokens, 1.0, 0,
            num_beams=K + 1, rows_name=f"verify rows (batch x ({arg} + 1))")
        if draft is not None and t_max > draft.cfg.n_positions:
            raise ValueError(f"generate: the longest prompt ({max(lengths)}) plus max_new_tokens ({n}) exceeds the "
                             f"assistant_model's n_positions = {draft.cfg.n_positions}")
        cfg, dev, weight, V, S = self.cfg, input_ids.device, self.wte.weight, self.cfg.vocab_size, K + 1
        seeds = _row_seeds(seed if draft is not None else 0, B, dev)     # prompt lookup is greedy and ignores seed
        tt_v = tt_new.repeat_interleave(S) if tt_new is not None else None
        cache = self.new_cache(B, t_max)
        h = self.hidden(input_ids, token_type_ids, cache=cache, lengths=lengths)[torch.arange(B, device=dev), last]
        # the prompt's last token plays the row's last emitted token x_b, whose logits the prefill gave: lens = len - 1
        cache.lens.sub_(1)
        stats = "lookup_stats" if draft is None else "assist_stats"
        if draft is not None:
            # The draft's cache has K more positions than the model's: a round runs all K + 1 draft steps, and those
            # past a row's cap write there (their positions are clamped to n_positions - 1); nothing a real slot reads.
            dc, dweight = draft.cfg, draft.wte.weight
            dcache = KVCache(dc.n_layer, B, dc.n_head, t_max + K, dc.n_embd // dc.n_head, dweight.dtype, dev)
            draft.hidden(input_ids, token_type_ids, cache=dcache, lengths=lengths)
        if not native:                              # CPU / not bf16: the definition on fp32 PyTorch logits
            from ..ops.assisted import assist_round, draw_slots, spec_slots
            from ..ops.lookup import lookup_accept, lookup_draft
            head, dhead = weight.float(), dweight.float() if draft is not None else None
            seq = torch.zeros(B, t_max, dtype=torch.int32)
            seq[:, :T] = input_ids.cpu()
            lens = cache.lens.cpu()
            emitted, done, steps = (torch.zeros(B, dtype=torch.int32) for _ in range(3))
            tokens = torch.full((B, n), -1, dtype=torch.int64)
            kw = dict(min_new=min_new_tokens, suppress_ids=suppress_ids, **filters)
            scal = (V, temperature, top_k, top_p, seeds.cpu().tolist())
            ids, nq = torch.zeros(B * S, dtype=torch.int64), torch.ones(B, dtype=torch.int32)
            g = draw_slots(self.lm_logits(h, head), *scal, lens, emitted, done, nq, **kw)   # greedy_token at T = 0
            lookup_accept(None, V, ids, nq, seq, lens, emitted, done, tokens, None, stop_ids=stop_ids, drawn=g)
            rounds = 0
            while not bool(done.all()):             # every live row emits at least one token per round
                if draft is None:
                    ids, pos, nq = lookup_draft(seq, lens, emitted, done, K, n, ngram)
                else:
                    ids, pos, nq, d_in, d_pos = assist_round(seq, lens, emitted, done, K, n, dc.n_positions)
                    dcache.lens.copy_(lens)
                    qlogits = []
                    for j in range(S):
                        hd = draft._blocks(draft._embed(d_in.to(dev), tt_new, d_pos[j].to(dev)), dcache)
                        dcache.lens.add_(1)
                        if j < K:
                            qlogits.append(draft.lm_logits(hd, dhead))
                            d = draw_slots(qlogits[-1], *scal, lens, emitted, done, nq, j, True, **kw)
                            d_in = torch.from_numpy(d[:, 0]).clamp(min=0)
                            ids.view(B, S)[:, j + 1] = d_in
                cache.lens.copy_(lens)
                hv = self._verify_hidden(ids.to(dev), pos.to(dev), tt_v, VerifyKV(cache, S, nq.to(dev)))
                acc = None
                if rejection:
                    _, acc, g = spec_slots(self.lm_logits(hv, head), torch.stack(qlogits, 1), *scal, lens, emitted,
                                           done, nq, ids, **kw)
                else:
                    g = draw_slots(self.lm_logits(hv, head), *scal, lens, emitted, done, nq, **kw)
                lookup_accept(None, V, ids, nq, seq, lens, emitted, done, tokens, steps, stop_ids=stop_ids, drawn=g,
                              accepted=acc)
                rounds += 1
            setattr(self, stats, {"emitted": emitted, "steps": steps, "replays": rounds})
            return tokens.to(dev), (tokens >= 0).sum(1).to(dev)

        from ..ops import (AssistState, LookupState, assist_round_, decode_attention_work_numel, lm_head_logits_,
                           lookup_accept_, lookup_argmax_, lookup_draft_, sample_slots_, spec_slots_)

        if draft is None:
            st = LookupState(B, K, n, t_max, ngram, dev)
        else:
            st = AssistState(B, K, n, t_max, dev, V if rejection else 0)
            dlogits = torch.empty(B, dweight.shape[0], dtype=torch.float32, device=dev)
        st.seq[:, :T] = input_ids
        logits = torch.empty(B * S, weight.shape[0], dtype=torch.float32, device=dev)
        sup, stop = (torch.tensor(list(x), dtype=torch.int32, device=dev) for x in (suppress_ids, stop_ids))
        draw = (V, temperature, top_k, top_p, seeds, st, cache.lens)

        def accept(lg, count=True):
            if temperature == 0:
                lookup_argmax_(lg, V, st, min_new_tokens, sup)
            elif rejection and count:
                spec_slots_(lg, *draw, min_new_tokens, sup, **filters)
            else:
                sample_slots_(lg, *draw, 0, min_new_tokens, sup, **filters)
            lookup_accept_(st, cache.lens, stop, count=count, flagged=rejection and count)

        lm_head_logits_(h, weight, logits[:B])      # the first token, from the prefill's last positions
        accept(logits[:B], count=False)
        replays = 0
        if n > 1:
            H = cfg.n_head
            work = torch.empty(decode_attention_work_numel(B * S, H, cfg.n_embd // H, t_max), dtype=torch.float32,
                               device=dev)
            verify = VerifyKV(cache, S, st.nq, work)

            def draft_and_verify(ids, tt, c):
                # The drafts depend on the model's state alone (a round's set-up also resets the draft cache's
                # lengths), so the warm-up step drafts for itself and leaves nothing behind.
                if draft is None:
                    lookup_draft_(st, cache.lens)
                else:
                    assist_round_(st, cache.lens, dcache.lens, dc.n_positions)
                    for j in range(S):
                        hd = draft._blocks(draft._embed(st.d_in, tt_new, st.d_pos[j]), dcache)
                        dcache.lens.add_(1)
                        if j < K:
                            lm_head_logits_(hd, dweight, dlogits)
                            sample_slots_(dlogits, *draw, j, min_new_tokens, sup, draft=True, weights=rejection,
                                          **filters)
                return self._verify_hidden(st.ids, st.pos, tt_v, verify)

            def head_and_accept(hv):
                lm_head_logits_(hv, weight, logits)
                accept(logits)

            # The drafts go into the graph's own input buffers. lookup_accept_ advances the cache by the tokens it
            # emits, up to k + 1 per replay, while the host counts one per replay. A live row emits at least one token
            # per replay, so at most n - 1 replays follow the first token and the host's lengths stay at most
            # max(lengths) + n - 1 < t_max: check_room never fires.
            graph = DecodeGraph(self, cache, tt_v is not None, head=head_and_accept, ids=st.ids, tt=tt_v,
                                step=draft_and_verify)
            replays = graph.run(n - 1, st.done, period=LOOKUP_POLL_PERIOD)
        setattr(self, stats, {"emitted": st.emitted, "steps": st.steps, "replays": replays})
        return st.tokens, (st.tokens >= 0).sum(1)

    def _verify_hidden(self, ids: torch.Tensor, pos: torch.Tensor, tt: Optional[torch.Tensor],
                       verify: "VerifyKV") -> torch.Tensor:
        """The final hidden states [B·(k+1), D] of the verify slots ``ids`` at positions ``pos`` (int64 [B·(k+1)]): the
        blocks of ``decode_step`` with attention through ``verify``. The real slots' keys and values go into the cache;
        its lengths do not move."""
        return self._blocks(self._embed(ids, tt, pos), verify)

    def _candidate_hidden(self, ids: torch.Tensor, tt: Optional[torch.Tensor], cand: "CandidateKV") -> torch.Tensor:
        """The final hidden states [B·k, D] of ``cand.top_k`` candidate tokens ``ids`` [B·k] per cache row, each at its
        row's position ``lens[b]``: the blocks of ``decode_step`` with attention through ``cand``. The cache is read
        only; its lengths do not move."""
        pos = cand.cache.lens.long().repeat_interleave(cand.top_k)
        return self._blocks(self._embed(ids, tt, pos), cand)

    @torch.no_grad()
    def contrastive_search(self, input_ids: torch.Tensor, lengths: Optional[Sequence[int]] = None,
                           token_type_ids: Optional[torch.Tensor] = None, reply_type=None, top_k: int = 4,
                           penalty_alpha: float = 0.6, max_new_tokens: int = 20, stop_ids: Sequence[int] = (),
                           suppress_ids: Sequence[int] = (), min_new_tokens: int = 0, repetition_penalty: float = 1.0,
                           no_repeat_ngram_size: int = 0, sequence_bias=None, bad_words_ids=None,
                           kv_cache_dtype: Optional[str] = None, frequency_penalty: float = 0.0,
                           presence_penalty: float = 0.0,
                           context_no_repeat_ngram_size: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
        """Batched contrastive search (Su et al., 2022; HuggingFace's ``penalty_alpha`` + ``top_k``); the definition is
        in ``ops/contrastive.py``.

        Each step takes the ``top_k`` most likely next tokens of a row, runs one decode step for each of them, and emits
        the candidate with the best ``(1 - penalty_alpha) p - penalty_alpha s``, where ``s`` is the largest cosine
        between the candidate's final hidden state and the hidden states of the row's sequence so far (its prompt
        without padding, then its emitted tokens). ``penalty_alpha = 0`` or ``top_k = 1`` is greedy decoding.
        ``input_ids``, ``lengths``, ``reply_type``, token types, ``stop_ids``, ``suppress_ids``, ``min_new_tokens``,
        the repetition controls, ``sequence_bias``, ``bad_words_ids``, ``frequency_penalty``, ``presence_penalty``,
        ``context_no_repeat_ngram_size`` (applied to the logits before the candidates are taken) and the return value
        ``(tokens, n_new)`` work as in ``generate``.

        The prompts are prefilled into a KV cache of ``max(lengths) + max_new_tokens`` positions (more than
        ``n_positions`` is a ``ValueError``) and the context is taken from the prefill's hidden states. On CUDA with
        bf16 weights (at most 64 rows) every token replays one CUDA graph: the candidate step (``ops.cand_attention_``
        attends for all k candidates over the shared cache), re-rank and commit (``ops.contrastive_rerank_``), the LM
        head on the winners, ``ops.penalize_repeats_`` when a repetition control, penalty or sequence bias is on, and
        the next candidates (``ops.contrastive_select_``);
        the host reads the done flags once every 8 tokens, a period late. Elsewhere the same loop runs eagerly:
        candidates decode through ``decode_attention`` on a k-fold copy of the rows and the selection runs in fp64
        (``ops/contrastive.py``). The cache is in the model's dtype: ``kv_cache_dtype`` other than None is a
        ``ValueError``."""
        from ..ops import CONTRASTIVE_MAX_K
        from ..ops.contrastive import check_contrastive_args, rerank_row, select_candidates

        if kv_cache_dtype is not None:
            raise ValueError(f"contrastive_search: kv_cache_dtype must be None (an fp8 cache is not supported), got "
                             f"{kv_cache_dtype!r}")
        check_contrastive_args("contrastive_search", top_k, penalty_alpha, CONTRASTIVE_MAX_K)
        K, alpha = int(top_k), float(penalty_alpha)
        B, T, lengths, n, t_max, last, tt_new, native, controls = self._decode_setup(
            "contrastive_search", input_ids, lengths, token_type_ids, reply_type, max_new_tokens, min_new_tokens,
            repetition_penalty, no_repeat_ngram_size, sequence_bias=sequence_bias, bad_words_ids=bad_words_ids,
            stop_ids=stop_ids, frequency_penalty=frequency_penalty, presence_penalty=presence_penalty,
            context_no_repeat_ngram_size=context_no_repeat_ngram_size)
        cfg, dev, weight = self.cfg, input_ids.device, self.wte.weight
        tt_cand = tt_new.repeat_interleave(K) if tt_new is not None else None
        cache = self.new_cache(B, t_max)
        hs = self.hidden(input_ids, token_type_ids, cache=cache, lengths=lengths)
        h = hs[torch.arange(B, device=dev), last].contiguous()
        V, L, H = cfg.vocab_size, cfg.n_layer, cfg.n_head
        D = cfg.n_embd
        reps = _Repeats.create(input_ids, cache, V, **controls)
        if not native:                              # CPU / not bf16: the fp64 definition on fp32 PyTorch logits
            head = weight.float()
            cand = CandidateKV(cache, K, torch.zeros(L, 2, B * K, D, dtype=weight.dtype, device=dev))
            ctx = [hs[b, :x] for b, x in enumerate(lengths)]
            stop = set(int(s) for s in stop_ids)
            done = torch.zeros(B, dtype=torch.bool)
            tokens = torch.full((B, n), -1, dtype=torch.int64)
            rows = torch.arange(B, device=dev)
            win = None
            for i in range(n):
                logits = self.lm_logits(h, head)
                if reps is not None:
                    logits = reps.eager(logits, cache, win)
                ids, probs = select_candidates(logits, V, K, i, min_new_tokens, suppress_ids, done)
                cache.check_room()
                hc = self._candidate_hidden(ids.clamp(min=0).reshape(-1).to(dev), tt_cand, cand)
                hk = hc.view(B, K, D)
                pick, win = [], torch.zeros(B, dtype=torch.int64)
                for b in range(B):
                    r = rerank_row(ids[b].numpy(), probs[b].numpy(), hk[b].double().cpu().numpy(),
                                   ctx[b].double().cpu().numpy(), alpha)
                    pick.append(b * K + r["rank"])
                    win[b] = r["token"]
                    if not done[b]:
                        if r["token"] in stop:
                            done[b] = True
                        else:
                            tokens[b, i] = r["token"]
                pick = torch.tensor(pick, device=dev)
                pos = cache.lens.long()
                cache.k[:, rows, :, pos] = cand.side[:, 0, pick].view(L, B, H, D // H).transpose(0, 1)
                cache.v[:, rows, :, pos] = cand.side[:, 1, pick].view(L, B, H, D // H).transpose(0, 1)
                cache.advance()
                h = hc[pick]
                ctx = [torch.cat([ctx[b], h[b:b + 1]]) for b in range(B)]
                if bool(done.all()):
                    break
            return tokens.to(dev), (tokens >= 0).sum(1).to(dev)

        from ..ops import (ContrastiveState, contrastive_context_init_, contrastive_rerank_, contrastive_select_,
                           lm_head_logits_)

        st = ContrastiveState(B, K, n, t_max, L, H, D // H, dev)
        contrastive_context_init_(hs.contiguous(), cache.lens, st)
        del hs
        cand = CandidateKV(cache, K, st.side, st.work)
        logits = torch.empty(B, weight.shape[0], dtype=torch.float32, device=dev)
        sup, stop = (torch.tensor(list(x), dtype=torch.int32, device=dev) for x in (suppress_ids, stop_ids))

        def select(hidden):
            lm_head_logits_(hidden, weight, logits)
            if reps is not None:
                reps.native(logits, cache.lens, st.step, st.win_ids)
            contrastive_select_(logits, V, st, min_new_tokens, sup)

        def commit_and_select(hc):
            contrastive_rerank_(hc, st, alpha, cache.k, cache.v, cache.lens, stop)
            select(st.win_h)

        select(h)                                   # the first candidates, from the prefill's last positions
        # contrastive_select_ writes the candidates into the graph's own input buffer; the commit advances the cache
        graph = DecodeGraph(self, cache, tt_cand is not None, head=commit_and_select, ids=st.next_ids, tt=tt_cand,
                            step=lambda ids, tt, c: self._candidate_hidden(ids, tt, cand))
        graph.run(n, st.done)                       # the first replay commits the first token
        return st.tokens, (st.tokens >= 0).sum(1)

    def forward(self, input_ids, token_type_ids=None, mc_token_ids=None, lm_labels=None, mc_labels=None,
                lm_coef: float = 1.0, mc_coef: float = 1.0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """-> (loss, lm_loss, mc_loss). Shapes as in the reference: [B, C, T] ids/labels, [B, C]
        mc_token_ids, [B] mc_labels; -100 labels are ignored. ``lm_loss`` is the mean LM cross-entropy whatever
        ``lm_coef`` is, reported without a gradient: the LM term reaches the parameters through ``loss`` only."""
        B, C, T = input_ids.shape
        ids = input_ids.reshape(B * C, T)
        tt = token_type_ids.reshape(B * C, T) if token_type_ids is not None else None
        drop = self._begin_dropout()
        h = self.hidden(ids, tt, drop=drop)                                   # [B*C, T, D]
        zero = torch.zeros((), dtype=torch.float32, device=h.device)
        lm_loss, mc_loss = zero, zero
        if lm_labels is not None:
            labels = lm_labels.reshape(B * C, T)
            shift_h = h[:, :-1].reshape(-1, h.shape[-1])
            shift_l = labels[:, 1:].reshape(-1)
            n_valid = (shift_l >= 0).sum()
            cap = int(self.lm_row_capacity)
            compact = 0 < cap < shift_l.numel()
            if compact:
                # scored rows first, in their original order (stable sort; static shapes, so the step
                # stays CUDA-graph capturable). Backward scatters the row gradients back.
                order = torch.argsort((shift_l < 0).to(torch.int8), stable=True)[:cap]
                shift_h = shift_h.index_select(0, order)
                shift_l = shift_l.index_select(0, order)
            # the mean's 1/n and lm_coef travel INTO the fused CE kernel, so the LM term enters `loss` with
            # coefficient 1 (the contract of _ChunkedLMLoss's direct weight-gradient path)
            n = n_valid.clamp(min=1).to(torch.float32)
            scale = (lm_coef / n).reshape(1)
            lm_term, lm_sum = _ChunkedLMLoss.apply(shift_h, self.wte.weight, shift_l, self.cfg.lm_chunk_rows,
                                                   self.cfg.vocab_size, scale)
            lm_loss = lm_sum / n                  # the mean itself, also when lm_coef is 0 and lm_term vanishes
            if compact:
                # a batch with more scored rows than the capacity must not train silently on a subset
                lm_loss = torch.where(n_valid > cap, torch.full_like(lm_loss, float("nan")), lm_loss)
                lm_term = torch.where(n_valid > cap, torch.full_like(lm_term, float("nan")), lm_term)
        if mc_token_ids is not None and mc_labels is not None:
            idx = mc_token_ids.reshape(B * C, 1, 1).expand(-1, 1, h.shape[-1])
            cls_h = h.gather(1, idx).squeeze(1)                               # [B*C, D]
            if drop is not None and self.cfg.summary_first_dropout > 0:
                cls_h = dropout(cls_h, self.cfg.summary_first_dropout, drop, site_summary(self.cfg.n_layer))
            mc_logits = self.mc_head(cls_h).view(B, C).float()
            mc_loss = F.cross_entropy(mc_logits, mc_labels)
        loss = (lm_term if lm_labels is not None else zero) + mc_coef * mc_loss
        return loss, lm_loss, mc_loss


# DecodeGraph.run's poll period for prompt-lookup generation, where one replay can emit up to k + 1 tokens per row:
# on GPT-2 small (8 rows, 64 new tokens, H100) it left 2-3 replays after the last row finished, against 9-10 at 8
LOOKUP_POLL_PERIOD = 2


class DecodeGraph:
    """``model.decode_step`` for one cache captured in a CUDA graph and replayed (the pattern of
    ``FlatDataParallel.capture``): the token ids (and token types) go through static input buffers, the cache's device
    state is read and advanced inside the graph, so one capture serves every later step of that cache, also after a new
    prefill into it. Replays give the same bits as eager steps. The returned hidden state [B, D] is a static buffer that
    the next replay overwrites.

    ``head`` runs on the step's hidden state inside the graph (the warm-up step leaves it out, so it may change state).
    ``ids`` / ``tt``: input buffers to read instead of the graph's own (``tt`` replaces the one ``token_types`` asks
    for), for a caller that fills them on the device and steps with ``replay``. ``generate`` uses all three. ``step``
    replaces ``model.decode_step`` as the captured step, called as ``step(ids, tt, cache)``; it and ``head`` together
    must leave the cache one token longer per replay (``contrastive_search``: a candidate step, then a commit)."""

    def __init__(self, model: "GPT2DoubleHeads", cache: KVCache, token_types: bool = True,
                 head: Optional[Callable] = None, ids: Optional[torch.Tensor] = None, tt: Optional[torch.Tensor] = None,
                 step: Optional[Callable] = None):
        dev = cache.lens.device
        self.cache = cache
        step = model.decode_step if step is None else step
        self.ids = torch.zeros(cache.batch, dtype=torch.long, device=dev) if ids is None else ids
        self.tt = tt if tt is not None or not token_types else torch.zeros_like(self.ids)
        lens0, host0 = cache.lens.clone(), list(cache.host_lens)
        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):                     # warm-up: allocator and cuBLAS settle; writes only slot lens[b],
            step(self.ids, self.tt, cache)             # which the next real step overwrites
        torch.cuda.current_stream(dev).wait_stream(s)
        cache.lens.copy_(lens0)
        cache.host_lens = host0
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.h = step(self.ids, self.tt, cache)
            if head is not None:
                head(self.h)
        cache.host_lens = host0                        # capturing ran the host side of a step, not the step

    def __call__(self, input_ids: torch.Tensor, token_type_ids: Optional[torch.Tensor] = None) -> torch.Tensor:
        if (token_type_ids is None) != (self.tt is None):
            raise ValueError("DecodeGraph: token types given at capture and at replay must match")
        self.ids.copy_(input_ids, non_blocking=True)
        if self.tt is not None:
            self.tt.copy_(token_type_ids, non_blocking=True)
        return self.replay()

    def replay(self) -> torch.Tensor:
        """One step on what the input buffers hold now, without copying anything into them."""
        self.cache.check_room()
        self.graph.replay()
        self.cache.advance_host()
        return self.h

    def run(self, replays: int, done: torch.Tensor, period: int = 8) -> int:
        """``replays`` replays, stopping early once every flag of ``done`` (int32, on the device) is set; returns the
        replays issued. Every ``period`` replays before the last the flags are copied to a pinned buffer, and the host
        reads that copy ``period`` replays later, when it is long finished, so the host never waits for the device."""
        flags = torch.empty(done.numel(), dtype=done.dtype, pin_memory=True)
        copied = None
        for i in range(1, replays + 1):
            self.replay()
            if i % period == 0 and i < replays:
                if copied is not None:
                    copied.synchronize()
                    if bool(flags.all()):
                        return i
                flags.copy_(done, non_blocking=True)
                copied = torch.cuda.Event()
                copied.record()
        return replays


class CachedDecoder:
    """The KV cache of a sequential sampling loop (``sample_sequence``, ``eval.convai.sample_reply``): ``restart``
    starts a sequence of B rows, ``extend`` appends one token per row; both return the last position's hidden state
    [B, D]. While the sequence fits into ``n_positions`` a token is one decode step (a ``DecodeGraph`` replay on the
    native kernel, eager otherwise); beyond that ``hidden`` runs uncached over the last ``n_positions`` tokens."""

    def __init__(self, model: "GPT2DoubleHeads"):
        self.model, self.n_pos = model, model.cfg.n_positions
        self.cache = self.graph = None

    def restart(self, ids: torch.Tensor, tt: Optional[torch.Tensor]) -> torch.Tensor:
        """A new sequence ``ids`` [B, T], token types ``tt`` [B, T] or None; prefilled into the cache if T fits."""
        self.parts, self.T = [(ids, tt)], ids.shape[1]       # the sequence in pieces, concatenated when a window needs it
        if self.T > self.n_pos:
            return self._window()
        if self.cache is None:
            self.cache = self.model.new_cache(ids.shape[0])
        return self.model.hidden(ids, tt, cache=self.cache)[:, -1]

    def extend(self, ids: torch.Tensor, tt: Optional[torch.Tensor]) -> torch.Tensor:
        """Append ``ids`` [B, 1] with token types ``tt`` [B, 1] (None if ``restart`` had none)."""
        self.parts.append((ids, tt))
        self.T += 1
        if self.T > self.n_pos:
            return self._window()
        ids, tt = ids[:, -1], tt[:, -1] if tt is not None else None   # T fits, so the cache holds all but this token
        if self.cache.work is None:
            return self.model.decode_step(ids, tt, self.cache)
        if self.graph is None:
            self.graph = DecodeGraph(self.model, self.cache, tt is not None)
        return self.graph(ids, tt)

    def _window(self) -> torch.Tensor:
        ids, tt = (torch.cat(p, 1) if p[0] is not None else None for p in zip(*self.parts))
        self.parts = [(ids, tt)]
        return self.model.hidden(ids[:, -self.n_pos:], tt[:, -self.n_pos:] if tt is not None else None)[:, -1]


@torch.no_grad()
def sample_sequence(model: "GPT2DoubleHeads", input_ids: torch.Tensor, token_type_ids: Optional[torch.Tensor] = None,
                    max_new_tokens: int = 20, temperature: float = 0.7, top_k: int = 0, top_p: float = 0.9,
                    eos_token: Optional[int] = None, reply_type: Optional[int] = None,
                    generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """Nucleus / top-k sampling of a reply, one token at a time (the decoding loop of the reference's interact.py:
    ``top_filtering`` + ``sample_sequence``, /root/reference/models/gpt2/interact.py). ``input_ids`` [1, T]; new tokens
    get ``reply_type`` as their token type when given, else the prompt's last one. The prompt is prefilled into a KV
    cache once and every new token costs one ``decode_step`` (graph-replayed on CUDA with the native kernels); once the
    sequence outgrows ``n_positions`` the window slides and each token re-runs the model over it (``CachedDecoder``)."""
    head = model.wte.weight.float()                            # the fp32 LM head, converted once per call
    dec = CachedDecoder(model)
    if token_type_ids is not None and reply_type is None:
        reply_type = int(token_type_ids[0, -1])
    out = []
    for i in range(max_new_tokens):
        h = (dec.extend(nxt, torch.full_like(nxt, reply_type) if token_type_ids is not None else None) if i
             else dec.restart(input_ids, token_type_ids))
        logits = top_filtering(model.lm_logits(h, head) / max(temperature, 1e-6), top_k, top_p)
        nxt = torch.multinomial(torch.softmax(logits, -1), 1, generator=generator)
        out.append(nxt)
        if eos_token is not None and int(nxt) == eos_token:
            break
    return torch.cat(out, 1) if out else input_ids[:, :0]


def lm_rows_needed(lm_labels: torch.Tensor, multiple: int = 256) -> int:
    """Capacity for ``GPT2DoubleHeads.lm_row_capacity`` from a (host) label tensor [B, C, T]: the number
    of scored next-token rows, rounded up to ``multiple``."""
    n = int((lm_labels[..., 1:] >= 0).sum())
    return max(multiple, (n + multiple - 1) // multiple * multiple)


def synthetic_batch(batch: int, candidates: int, seq_len: int, vocab: int, device="cpu", seed: int = 0,
                    pin: bool = False):
    """PersonaChat-shaped synthetic batch (the real set is downloaded by the reference; there is no
    network here): history tokens carry -100 labels, only the last candidate's reply is scored."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, vocab, (batch, candidates, seq_len), generator=g)
    tt = torch.randint(vocab - 5, vocab - 3, (batch, candidates, seq_len), generator=g)
    labels = torch.full((batch, candidates, seq_len), -100, dtype=torch.long)
    reply = max(1, seq_len // 4)
    labels[:, -1, -reply:] = ids[:, -1, -reply:]
    mc_token_ids = torch.full((batch, candidates), seq_len - 1, dtype=torch.long)
    mc_labels = torch.full((batch,), candidates - 1, dtype=torch.long)
    out = {"input_ids": ids, "token_type_ids": tt, "lm_labels": labels, "mc_token_ids": mc_token_ids,
           "mc_labels": mc_labels}
    if pin and torch.cuda.is_available():
        out = {k: v.pin_memory() for k, v in out.items()}
    if device != "cpu":
        out = {k: v.to(device, non_blocking=True) for k, v in out.items()}
    return out
