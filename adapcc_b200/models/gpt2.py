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

from ..ops.layers import FusedLayerNorm, FusedLinear
from ..ops.repeats import check_repeat_args, penalize_repeats_reference
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
    allocated once so a captured step reuses it."""

    def __init__(self, n_layer: int, batch: int, n_head: int, t_max: int, head_dim: int, dtype: torch.dtype, device):
        self.batch, self.t_max = int(batch), int(t_max)
        self.k = torch.zeros(n_layer, batch, n_head, t_max, head_dim, dtype=dtype, device=device)
        self.v = torch.zeros_like(self.k)
        self.lens = torch.zeros(batch, dtype=torch.int32, device=self.k.device)
        self.host_lens: List[int] = [0] * self.batch
        self.work = None
        if self.k.is_cuda and dtype == torch.bfloat16:
            from ..ops import decode_attention_work_numel
            self.work = torch.empty(decode_attention_work_numel(batch, n_head, head_dim, t_max), dtype=torch.float32,
                                    device=self.k.device)

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
                     work: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One layer of decode attention: ``qkv`` [B, 3·H·Dh] (q | k | v of each row's new token), caches [B, H, t_max, Dh],
    ``lens`` int32 [B]. Stores the new k / v at position ``lens[b]`` and returns softmax(q·K[0..lens[b]]ᵀ/√Dh)·V [B, H·Dh]
    with an fp32 softmax. With ``work`` (bf16 CUDA caches) this is the native kernel (``ops.decode_attention_``);
    otherwise the same computation in PyTorch, the reference the CPU tests use."""
    B, H, t_max, Dh = k_cache.shape
    if work is not None:
        from ..ops import decode_attention_
        out = torch.empty(B, H * Dh, dtype=qkv.dtype, device=qkv.device)
        return decode_attention_(qkv, k_cache, v_cache, lens, out, work)
    q, k, v = qkv.reshape(B, 3, H, Dh).unbind(1)
    pos = lens.long()
    rows = torch.arange(B, device=qkv.device)
    k_cache[rows, :, pos] = k
    v_cache[rows, :, pos] = v
    s = torch.einsum("bhd,bhtd->bht", q.float(), k_cache.float()) / math.sqrt(Dh)
    s = s.masked_fill(torch.arange(t_max, device=qkv.device) > pos[:, None, None], float("-inf"))
    p = torch.softmax(s, dim=-1)
    return torch.einsum("bht,bhtd->bhd", p, v_cache.float()).to(qkv.dtype).reshape(B, H * Dh)


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
    """The repetition controls of a batched decoder over the R rows of its cache: ``seq`` int32 [R, t_max] each row's
    sequence (its prompt, then its tokens), ``prompt_len`` int32 [R] the lengths after the prefill, the penalty and the
    n-gram size. ``create`` returns None when both controls are off, so then nothing is allocated or launched."""

    def __init__(self, input_ids: torch.Tensor, cache: KVCache, vocab: int, penalty: float, ngram: int):
        B, T = input_ids.shape
        self.seq = torch.zeros(cache.batch, cache.t_max, dtype=torch.int32, device=input_ids.device)
        self.seq[:, :T] = input_ids.repeat_interleave(cache.batch // B, dim=0)
        self.prompt_len = cache.lens.clone()
        self.vocab, self.penalty, self.ngram = vocab, penalty, ngram

    @classmethod
    def create(cls, input_ids: torch.Tensor, cache: KVCache, vocab: int, penalty: float,
               ngram: int) -> Optional["_Repeats"]:
        return cls(input_ids, cache, vocab, penalty, ngram) if penalty != 1.0 or ngram > 0 else None

    def eager(self, logits: torch.Tensor, cache: KVCache, consumed: Optional[torch.Tensor]) -> torch.Tensor:
        """``penalize_repeats_reference`` over every row's sequence, after storing ``consumed`` [R] (the tokens the last
        decode step consumed; None before the first one) at ``lens - 1``."""
        if consumed is not None:
            dev = self.seq.device
            self.seq[torch.arange(cache.batch, device=dev), cache.lens.long() - 1] = consumed.to(dev, torch.int32)
        return penalize_repeats_reference(logits, [self.seq[r, :x] for r, x in enumerate(cache.host_lens)],
                                          self.vocab, self.penalty, self.ngram)

    def reorder(self, rows: torch.Tensor) -> None:
        """Row r continues row ``rows[r]`` (a beam its parent)."""
        self.seq = self.seq[rows]

    def native(self, logits: torch.Tensor, lens: torch.Tensor, step: torch.Tensor, ids: torch.Tensor,
               parent: Optional[torch.Tensor] = None, group: int = 1) -> None:
        """``ops.penalize_repeats_`` on ``logits`` in place; it also stores ``ids`` and follows ``parent``."""
        from ..ops import penalize_repeats_
        penalize_repeats_(logits, self.vocab, self.seq, self.prompt_len, lens, step, ids, parent, group,
                          self.penalty, self.ngram)


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
            return self.c_proj(decode_attention(self.c_attn(h), cache.k[layer], cache.v[layer], cache.lens, cache.work))
        B, T, D = h.shape
        # split along the feature dim (views; measured 6 % faster fwd+bwd than the packed permute:
        # the backward writes dq/dk/dv straight into one [B, T, 3D] buffer layout-wise)
        q, k, v = (t.view(B, T, self.n_head, D // self.n_head).transpose(1, 2) for t in self.c_attn(h).split(D, dim=-1))
        if cache is not None:                         # prefill: keep this layer's keys and values
            cache.k[layer, :, :, :T].copy_(k.detach())
            cache.v[layer, :, :, :T].copy_(v.detach())
        a = causal_attention(q, k, v)
        return self.c_proj(a.transpose(1, 2).reshape(B, T, D))

    def forward_deferred(self, x: torch.Tensor, delta: Optional[torch.Tensor], cache: Optional["KVCache"] = None,
                         layer: int = 0):
        """Same block with every residual add fused into the LayerNorm that follows it: takes the
        residual stream ``x`` and the previous block's not-yet-added MLP output ``delta``, returns
        (stream, this block's not-yet-added MLP output)."""
        if delta is None:
            h = self.ln_1(x)
        else:
            x, h = self.ln_1.forward_add(x, delta)
        x, h = self.ln_2.forward_add(x, self._attn(h, cache, layer))
        return x, self._mlp(h)

    def forward(self, x: torch.Tensor, cache: Optional["KVCache"] = None, layer: int = 0) -> torch.Tensor:
        x = x + self._attn(self.ln_1(x), cache, layer)
        return x + self._mlp(self.ln_2(x))


def use_sink(p) -> bool:
    from ..ops.layers import _sink
    return p.is_cuda and _sink(p) is not None


class _ChunkedLMLoss(torch.autograd.Function):
    """sum over rows of CE(h @ W^T, labels), ``chunk`` rows at a time. The backward of every chunk
    is produced inside the forward pass (fused softmax-CE kernel overwrites the bf16 logits with
    their gradient), so logits never outlive a chunk and are touched twice instead of ~8 times."""

    @staticmethod
    def forward(ctx, h, weight, labels, chunk, vocab, scale=None):
        """``scale`` (1-element fp32 device tensor or None): the result is ``scale * sum of row losses`` and the
        gradients produced here already contain it — the caller promises that the returned value enters the total
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
        if scale is not None:
            total = total * scale.reshape(())
        ctx.direct, ctx.weight = direct, weight
        if direct:
            ctx.save_for_backward(grad_h)
        else:
            if grad_w is None:
                grad_w = torch.zeros_like(weight)
            ctx.save_for_backward(grad_h, grad_w)
        return total

    @staticmethod
    def backward(ctx, g):
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
        self.apply(self._init)
        for blk in self.h:                                  # GPT-2 residual-projection scaling
            for lin in (blk.c_proj, blk.c_proj2):
                nn.init.normal_(lin.weight, std=cfg.initializer_range / math.sqrt(2 * cfg.n_layer))

    def _init(self, m):
        if isinstance(m, (nn.Linear, nn.Embedding)):
            nn.init.normal_(m.weight, std=self.cfg.initializer_range)
            if isinstance(m, nn.Linear) and m.bias is not None:
                nn.init.zeros_(m.bias)

    def num_parameters(self) -> int:
        return sum(p.numel() for p in self.parameters())

    def hidden(self, input_ids: torch.Tensor, token_type_ids: Optional[torch.Tensor], cache: Optional["KVCache"] = None,
               lengths: Optional[Sequence[int]] = None) -> torch.Tensor:
        """Final-LayerNorm hidden states [N, T, D]. With ``cache`` this is also the prefill of incremental decoding:
        every layer's keys and values of positions 0..T-1 go into the cache and its lengths become ``lengths`` (the real
        length of each right-padded row; default T for all). Causal attention makes the padding invisible to the real
        tokens, and ``decode_step`` overwrites the padded slots."""
        N, T = input_ids.shape
        if cache is not None:
            cache.reset(lengths if lengths is not None else [T] * N, T)
        return self._blocks(self._embed(input_ids, token_type_ids), cache)

    def _embed(self, ids: torch.Tensor, tt: Optional[torch.Tensor], pos: Optional[torch.Tensor] = None) -> torch.Tensor:
        """wte[ids] + wpe[pos] (+ wte[tt]), added in that order: [*ids.shape, D]; ``pos`` defaults to 0..T-1 in every
        row of ids [N, T]. One ``fused_embedding_sum`` for bf16 CUDA tables if ``fused_embed``."""
        if (self.fused_embed and ids.is_cuda and self.wte.weight.dtype == torch.bfloat16
                and self.wpe.weight.dtype == torch.bfloat16):
            from ..ops import fused_embedding_sum
            if pos is None:                  # cached: a captured training step reads the same positions every replay
                N, T = ids.shape
                pos = self._pos_cache.get((N, T, ids.device))
                if pos is None:
                    pos = self._pos_cache[(N, T, ids.device)] = torch.arange(T, device=ids.device).repeat(N)
            lookups = [(0, ids), (1, pos)] + ([(0, tt)] if tt is not None else [])
            return fused_embedding_sum([self.wte.weight, self.wpe.weight], lookups).view(*ids.shape, -1)
        # the default positions broadcast over the rows, so wpe's gradient is summed over them before the lookup
        x = self.wte(ids) + self.wpe(torch.arange(ids.shape[-1], device=ids.device) if pos is None else pos)
        if tt is not None:
            x = x + self.wte(tt)
        return x

    def lm_logits(self, h: torch.Tensor, head: Optional[torch.Tensor] = None) -> torch.Tensor:
        """fp32 logits [..., vocab_size] of ``h`` [..., D] through the tied head; ``head``: a kept fp32 ``wte.weight``."""
        if head is None:
            head = self.wte.weight.float()
        return (h.float() @ head.t())[..., :self.cfg.vocab_size]

    def _blocks(self, x: torch.Tensor, cache: Optional["KVCache"]) -> torch.Tensor:
        if self.fuse_add_ln:
            delta = None
            for i, blk in enumerate(self.h):
                x, delta = blk.forward_deferred(x, delta, cache, i)
            return self.ln_f.forward_add(x, delta)[1]
        for i, blk in enumerate(self.h):
            x = blk(x, cache, i)
        return self.ln_f(x)

    def new_cache(self, batch: int, t_max: Optional[int] = None) -> "KVCache":
        """An empty KV cache for ``batch`` rows of up to ``t_max`` (default ``n_positions``) tokens, on the model's
        device and in its dtype."""
        cfg = self.cfg
        t_max = cfg.n_positions if t_max is None else int(t_max)
        if not 1 <= t_max <= cfg.n_positions:
            raise ValueError(f"new_cache: t_max must be in [1, {cfg.n_positions}], got {t_max}")
        w = self.wte.weight
        return KVCache(cfg.n_layer, batch, cfg.n_head, t_max, cfg.n_embd // cfg.n_head, w.dtype, w.device)

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
                      rows_name: str = "beam rows (batch x num_beams)"):
        """The checks and prompt quantities the batched decoders share, before anything is launched:
        ``(B, T, lengths, n, t_max, last, tt_new, native)``. ``last`` [B] is each prompt's last position, ``tt_new`` [B]
        the token type of new tokens (None without token types), and ``native`` says whether the bf16 CUDA kernels
        run; they take at most ``LM_HEAD_MAX_ROWS`` rows, ``num_beams`` per prompt (called ``rows_name`` in the error
        when more than one). Errors name ``who``."""
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
        check_repeat_args(who, repetition_penalty, no_repeat_ngram_size)
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
        return B, T, lengths, n, t_max, last, tt_new, native

    @torch.no_grad()
    def generate(self, input_ids: torch.Tensor, lengths: Optional[Sequence[int]] = None,
                 token_type_ids: Optional[torch.Tensor] = None, reply_type=None, max_new_tokens: int = 20,
                 temperature: float = 0.7, top_k: int = 0, top_p: float = 0.9, stop_ids: Sequence[int] = (),
                 suppress_ids: Sequence[int] = (), min_new_tokens: int = 0, seed=0, repetition_penalty: float = 1.0,
                 no_repeat_ngram_size: int = 0, prompt_lookup_num_tokens: int = 0,
                 max_matching_ngram_size: int = 2, min_p: float = 0.0, typical_p: float = 1.0,
                 epsilon_cutoff: float = 0.0, eta_cutoff: float = 0.0, assistant_model: "GPT2DoubleHeads" = None,
                 num_assistant_tokens: int = 4,
                 assistant_verification: str = "coupled") -> Tuple[torch.Tensor, torch.Tensor]:
        """Batched, seeded top-k / top-p sampling of up to ``max_new_tokens`` tokens per row.

        ``input_ids`` [B, T] is right-padded; row b's prompt is its first ``lengths[b]`` tokens (default T).
        ``reply_type`` (an int or a [B] tensor) is the token type of the new tokens; by default each row's last prompt
        token type when ``token_type_ids`` is given. ``seed``: an int (row b uses ``seed + b``) or an int64 [B] tensor.
        While fewer than ``min_new_tokens`` tokens are generated, ``suppress_ids`` cannot be drawn; a token in
        ``stop_ids`` ends its row. ``temperature == 0`` is greedy. The draw of each token is defined in
        ``ops/sampling.py``: a row's tokens depend on its prompt, its seed and the scalars, not on the other rows.
        ``repetition_penalty`` (1: off) and ``no_repeat_ngram_size`` (0: off) act on each row's logits first, over its
        prompt and the tokens generated so far (``ops/repeats.py``). ``min_p`` (0: off), ``typical_p`` (1: off),
        ``epsilon_cutoff`` (0: off) and ``eta_cutoff`` (0: off) are HuggingFace's truncation samplers: at temperature
        > 0 they filter, in that order, the ids that top-k and top-p kept, just before the draw (inside
        ``ops.sample_tokens_`` on the native path); at temperature 0 they have no effect.

        Returns ``(tokens, n_new)``: int64 [B, max_new_tokens] (-1 after a row stopped) and the tokens per row.

        The prompts are prefilled into a KV cache of ``max(lengths) + max_new_tokens`` positions (``ValueError`` if that
        exceeds ``n_positions``: there is no sliding window here, ``sample_sequence`` has one). On CUDA with bf16
        weights the LM head and the sampler are native kernels (``ops.lm_head_logits_``, ``ops.sample_tokens_``) and
        every token after the first replays one CUDA graph of decode step, LM head (``ops.penalize_repeats_`` when a
        repetition control is on) and sampler, which feeds the drawn ids back into its own input; the host reads the
        done flags once every 8 tokens, a step late, to stop early. Elsewhere the same loop runs eagerly with fp32
        PyTorch logits, ``ops.repeats.penalize_repeats_reference`` and ``ops.sampling.sample_reference``.

        ``prompt_lookup_num_tokens`` = k > 0 (HuggingFace's prompt lookup decoding; greedy only, without the repetition
        controls) verifies up to k draft tokens per row and step, copied from the row's own prompt and reply after the
        earliest earlier occurrence of its last ``max_matching_ngram_size`` (or fewer) tokens; the result is the greedy
        tokens. The definition is in ``ops/lookup.py``. On the native path (``B·(k+1)`` at most 64 rows) every verify
        step replays one CUDA graph: the model on k + 1 slots per row (``ops.verify_attention_``), the LM head,
        acceptance (``ops.lookup_accept_``) and the next drafts (``ops.lookup_draft_``); the host polls the done flags
        every ``LOOKUP_POLL_PERIOD`` replays. Afterwards ``self.lookup_stats`` holds the rows' emitted tokens (a stop id
        included) and verify steps, int32 [B], and the graph replays issued.

        ``assistant_model`` (HuggingFace's assisted generation; a ``GPT2DoubleHeads`` with the same vocabulary, bf16 on
        the same device on the native path; not with prompt lookup or the repetition controls) drafts up to
        ``num_assistant_tokens`` = k tokens per row and round, which the model verifies in one step. Every emitted token
        is drawn from the same seed, position and step as in plain ``generate``, greedy or sampled, so given the same
        per-position logits the tokens are those of plain ``generate``; the draft changes only the speed. The definition
        is in ``ops/assisted.py``. On the native path (``B·(k+1)`` at most 64 rows) a round replays one CUDA graph: the
        draft's k + 1 decode steps with k draws (``ops.sample_slots_``), the model on k + 1 slots per row, the LM head,
        the slots' draws and acceptance (``ops.lookup_accept_drawn_``; ``ops.lookup_accept_`` at temperature 0).
        Afterwards ``self.assist_stats`` holds what ``lookup_stats`` holds for prompt lookup.

        ``assistant_verification`` is that rule, ``"coupled"``, or ``"rejection"``: HuggingFace's rejection sampling
        (Leviathan et al. 2023), where a draft d is accepted with probability ``min(1, P(d) / Q(d))`` of the model's
        and the draft's filtered distributions and a rejection is replaced by a draw from ``max(0, P - Q)``. Each
        emitted token is then distributed as the model's, acceptance is their overlap rather than the agreement of
        two draws, and the tokens depend on the draft. On the native path the draft draws also keep their weights and
        the verify step runs ``ops.spec_slots_`` and ``ops.lookup_accept_drawn_(..., flagged=True)``. At temperature
        0 both rules are the greedy one."""
        if not temperature >= 0 or int(top_k) < 0 or not 0 < top_p <= 1:
            raise ValueError(f"generate: need temperature >= 0, top_k >= 0 and 0 < top_p <= 1, got {temperature}, "
                             f"{top_k}, {top_p}")
        check_filter_args("generate", min_p, typical_p, epsilon_cutoff, eta_cutoff)
        filters = dict(min_p=min_p, typical_p=typical_p, epsilon_cutoff=epsilon_cutoff, eta_cutoff=eta_cutoff)
        from ..ops.assisted import check_verification
        check_verification("generate", assistant_verification, assistant_model)
        if assistant_model is not None:
            from ..ops import LOOKUP_MAX_TOKENS
            from ..ops.assisted import check_assist_args
            check_assist_args("generate", self, assistant_model, num_assistant_tokens, LOOKUP_MAX_TOKENS,
                              prompt_lookup_num_tokens, repetition_penalty, no_repeat_ngram_size)
            return self._generate_assisted(assistant_model, int(num_assistant_tokens), input_ids, lengths,
                                           token_type_ids, reply_type, max_new_tokens, temperature, top_k, top_p,
                                           stop_ids, suppress_ids, min_new_tokens, seed, filters,
                                           assistant_verification == "rejection" and temperature > 0)
        K = prompt_lookup_num_tokens
        if K != 0:
            from ..ops import LOOKUP_MAX_NGRAM, LOOKUP_MAX_TOKENS
            from ..ops.lookup import check_lookup_args
            check_lookup_args("generate", K, max_matching_ngram_size, LOOKUP_MAX_TOKENS, LOOKUP_MAX_NGRAM, temperature,
                              repetition_penalty, no_repeat_ngram_size)
            return self._generate_lookup(input_ids, lengths, token_type_ids, reply_type, max_new_tokens, stop_ids,
                                         suppress_ids, min_new_tokens, int(K), int(max_matching_ngram_size))
        B, T, lengths, n, t_max, last, tt_new, native = self._decode_setup(
            "generate", input_ids, lengths, token_type_ids, reply_type, max_new_tokens, min_new_tokens,
            repetition_penalty, no_repeat_ngram_size)
        dev, V = input_ids.device, self.cfg.vocab_size
        seeds = _row_seeds(seed, B, dev)
        cache = self.new_cache(B, t_max)
        h = self.hidden(input_ids, token_type_ids, cache=cache, lengths=lengths)[torch.arange(B, device=dev), last]
        tokens = torch.full((B, n), -1, dtype=torch.int64, device=dev)
        reps = _Repeats.create(input_ids, cache, V, repetition_penalty, no_repeat_ngram_size)
        if not native:                              # CPU / not bf16: the fp64 definition on fp32 PyTorch logits
            head = self.wte.weight.float()
            done = torch.zeros(B, dtype=torch.int32)
            for i in range(n):
                if i:
                    h = self.decode_step(nxt.to(dev), tt_new, cache)
                logits = self.lm_logits(h, head)
                if reps is not None:
                    logits = reps.eager(logits, cache, nxt if i else None)
                nxt, tok, done = sample_reference(logits, V, temperature, top_k, top_p, seeds, cache.lens, i,
                                                  min_new_tokens, suppress_ids, stop_ids, done, **filters)
                tokens[:, i] = tok.to(dev)
                if bool(done.all()):
                    break
            return tokens, (tokens >= 0).sum(1)

        from ..ops import lm_head_logits_, sample_tokens_

        weight = self.wte.weight
        logits = torch.empty(B, weight.shape[0], dtype=torch.float32, device=dev)
        next_ids = torch.zeros(B, dtype=torch.int64, device=dev)
        done = torch.zeros(B, dtype=torch.int32, device=dev)
        step = torch.zeros(1, dtype=torch.int32, device=dev)
        sup, stop = (torch.tensor(list(x), dtype=torch.int32, device=dev) for x in (suppress_ids, stop_ids))

        def head_and_sample(hidden):
            lm_head_logits_(hidden, weight, logits)
            if reps is not None:
                reps.native(logits, cache.lens, step, next_ids)
            sample_tokens_(logits, V, temperature, top_k, top_p, seeds, cache.lens, step,
                           min_new_tokens, sup, stop, done, next_ids, tokens, **filters)

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
                    no_repeat_ngram_size: int = 0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Batched beam search with ``num_beams`` beams per prompt; the definition is in ``ops/beam.py``.

        ``input_ids`` [B, T] is right-padded; item b's prompt is its first ``lengths[b]`` tokens (default T).
        ``reply_type`` and the token types of new tokens work as in ``generate``. A token in ``stop_ids`` (at most 8)
        finishes a hypothesis; while fewer than ``min_new_tokens`` tokens are generated, ``suppress_ids`` cannot be
        chosen. A hypothesis of L tokens (its stop token included) scores ``sum of log-probabilities / L **
        length_penalty``. An item stops as soon as no live beam can beat its K-th finished hypothesis, which never
        changes its result. An item's result depends on its prompt and the scalars only, not on the other items.
        ``repetition_penalty`` (1: off) and ``no_repeat_ngram_size`` (0: off) act on each beam's logits before the
        log-softmax, over its prompt and its own hypothesis (``ops/repeats.py``), so its log-probabilities are
        renormalised over the ids that remain.

        Returns ``(tokens, n_new, scores)``: the best hypothesis of each item as int64 [B, max_new_tokens] (the stop
        token excluded, padded with -1), its length int64 [B] and its normalised score fp32 [B].

        Each prompt is prefilled once and its keys and values copied to its ``num_beams`` rows of a cache of
        ``max(lengths) + max_new_tokens`` positions (more than ``n_positions`` is a ``ValueError``). On CUDA with bf16
        weights every token after the first replays one CUDA graph of decode step, LM head (``ops.lm_head_logits_``),
        the repetition controls when on (``ops.penalize_repeats_``), selection (``ops.beam_step_``) and cache
        reordering (``ops.kv_reorder_``), at most 64 beam rows per call; the host reads the done flags once every 8
        tokens, a period late. Elsewhere the same loop runs eagerly with fp32 PyTorch logits,
        ``ops.repeats.penalize_repeats_reference``, ``ops.beam.BeamReference`` and torch indexing."""
        from ..ops import BEAM_MAX_BEAMS, BEAM_MAX_STOP, BEAM_MAX_SUPPRESS
        from ..ops.beam import BeamReference, best_hypotheses

        K = int(num_beams)
        if not 1 <= K <= BEAM_MAX_BEAMS:
            raise ValueError(f"beam_search: num_beams must be in [1, {BEAM_MAX_BEAMS}], got {num_beams}")
        if len(stop_ids) > BEAM_MAX_STOP or len(suppress_ids) > BEAM_MAX_SUPPRESS:
            raise ValueError(f"beam_search: at most {BEAM_MAX_STOP} stop ids and {BEAM_MAX_SUPPRESS} suppressed ids, "
                             f"got {len(stop_ids)} and {len(suppress_ids)}")
        B, T, lengths, n, t_max, last, tt_new, native = self._decode_setup(
            "beam_search", input_ids, lengths, token_type_ids, reply_type, max_new_tokens, min_new_tokens,
            repetition_penalty, no_repeat_ngram_size, num_beams=K)
        dev, V, weight = input_ids.device, self.cfg.vocab_size, self.wte.weight
        if tt_new is not None:
            tt_new = tt_new.repeat_interleave(K)
        # one prefill per prompt, its keys and values copied to the prompt's K rows (the beams share that region)
        pre = self.new_cache(B, T)
        h = self.hidden(input_ids, token_type_ids, cache=pre, lengths=lengths)[torch.arange(B, device=dev), last]
        cache = self.new_cache(B * K, t_max)
        cache.reset([x for x in lengths for _ in range(K)], T)
        cache.k[:, :, :, :T].copy_(pre.k.repeat_interleave(K, dim=1))
        cache.v[:, :, :, :T].copy_(pre.v.repeat_interleave(K, dim=1))
        del pre
        h = h.repeat_interleave(K, dim=0).contiguous()
        reps = _Repeats.create(input_ids, cache, V, repetition_penalty, no_repeat_ngram_size)
        if not native:                              # CPU / not bf16: the fp64 definition on fp32 PyTorch logits
            ref = BeamReference(B, K, n, V, length_penalty, stop_ids, suppress_ids, min_new_tokens)
            head = weight.float()
            for i in range(n):
                if i:
                    h = self.decode_step(nxt.to(dev), tt_new, cache)
                logits = self.lm_logits(h, head)
                if reps is not None:
                    logits = reps.eager(logits, cache, nxt if i else None)
                nxt, parent = ref.step(logits)
                rows = parent.to(dev)
                cache.k.copy_(cache.k[:, rows])
                cache.v.copy_(cache.v[:, rows])
                if reps is not None:
                    reps.reorder(rows)
                if ref.done.all():
                    break
            return tuple(t.to(dev) for t in ref.result())

        from ..ops import BeamState, beam_step_, kv_reorder_, kv_reorder_scratch_numel, lm_head_logits_

        st = BeamState(B, K, n, length_penalty, dev)
        logits = torch.empty(B * K, weight.shape[0], dtype=torch.float32, device=dev)
        sup, stop = (torch.tensor(list(x), dtype=torch.int32, device=dev) for x in (suppress_ids, stop_ids))
        prompt_len = cache.lens.clone()
        scratch = torch.empty(kv_reorder_scratch_numel(cache.k, n), dtype=cache.k.dtype, device=dev)

        def select(hidden):
            lm_head_logits_(hidden, weight, logits)
            if reps is not None:
                reps.native(logits, cache.lens, st.step, st.next_ids, st.parent, K)
            beam_step_(logits, V, st, min_new_tokens, sup, stop)
            kv_reorder_(cache.k, cache.v, st.parent, prompt_len, cache.lens, n, scratch)

        select(h)                                   # the first selection, from the prefill's last positions
        if n > 1:
            # beam_step_ writes the new beams' tokens into the graph's own input buffer
            DecodeGraph(self, cache, tt_new is not None, head=select, ids=st.next_ids, tt=tt_new).run(n - 1, st.done)
        count = st.fin_count.cpu().tolist()
        score, n_tok, src = st.fin_score.cpu().tolist(), st.fin_n.cpu().tolist(), st.fin_src.cpu().tolist()
        fin = [list(zip(score[b], n_tok[b], src[b]))[:count[b]] for b in range(B)]
        hist_tok = st.hist_tok.view(n, B, K).cpu().numpy()
        hist_back = st.hist_back.view(n, B, K).cpu().numpy()
        return tuple(t.to(dev) for t in best_hypotheses(fin, hist_tok, hist_back, n))

    def _generate_lookup(self, input_ids, lengths, token_type_ids, reply_type, max_new_tokens, stop_ids, suppress_ids,
                         min_new_tokens, K: int, ngram: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """``generate`` at temperature 0 with prompt lookup of up to ``K`` drafts (``ops/lookup.py``)."""
        B, T, lengths, n, t_max, last, tt_new, native = self._decode_setup(
            "generate", input_ids, lengths, token_type_ids, reply_type, max_new_tokens, min_new_tokens, 1.0, 0,
            num_beams=K + 1, rows_name="verify rows (batch x (prompt_lookup_num_tokens + 1))")
        cfg, dev, weight, V, S = self.cfg, input_ids.device, self.wte.weight, self.cfg.vocab_size, K + 1
        tt_v = tt_new.repeat_interleave(S) if tt_new is not None else None
        cache = self.new_cache(B, t_max)
        h = self.hidden(input_ids, token_type_ids, cache=cache, lengths=lengths)[torch.arange(B, device=dev), last]
        # the prompt's last token plays the row's last emitted token x_b, whose logits the prefill gave: lens = len - 1
        cache.lens.sub_(1)
        if not native:                              # CPU / not bf16: the definition on fp32 PyTorch logits
            from ..ops.lookup import lookup_accept, lookup_draft
            head = weight.float()
            seq = torch.zeros(B, t_max, dtype=torch.int32)
            seq[:, :T] = input_ids.cpu()
            lens = cache.lens.cpu()
            emitted, done, steps = (torch.zeros(B, dtype=torch.int32) for _ in range(3))
            tokens = torch.full((B, n), -1, dtype=torch.int64)
            ids, nq = torch.zeros(B * S, dtype=torch.int64), torch.ones(B, dtype=torch.int32)
            lookup_accept(self.lm_logits(h, head), V, ids, nq, seq, lens, emitted, done, tokens, None, min_new_tokens,
                          suppress_ids, stop_ids)
            while not bool(done.all()):             # every live row emits at least one token per step
                ids, pos, nq = lookup_draft(seq, lens, emitted, done, K, n, ngram)
                cache.lens.copy_(lens)
                hv = self._verify_hidden(ids.to(dev), pos.to(dev), tt_v, VerifyKV(cache, S, nq.to(dev)))
                lookup_accept(self.lm_logits(hv, head), V, ids, nq, seq, lens, emitted, done, tokens, steps,
                              min_new_tokens, suppress_ids, stop_ids)
            self.lookup_stats = {"emitted": emitted, "steps": steps, "replays": int(steps.max())}
            return tokens.to(dev), (tokens >= 0).sum(1).to(dev)

        from ..ops import LookupState, decode_attention_work_numel, lm_head_logits_, lookup_accept_, lookup_draft_

        st = LookupState(B, K, n, t_max, ngram, dev)
        st.seq[:, :T] = input_ids
        logits = torch.empty(B * S, weight.shape[0], dtype=torch.float32, device=dev)
        sup, stop = (torch.tensor(list(x), dtype=torch.int32, device=dev) for x in (suppress_ids, stop_ids))
        lm_head_logits_(h, weight, logits[:B])      # the first token, from the prefill's last positions
        lookup_accept_(logits[:B], V, st, cache.lens, min_new_tokens, sup, stop, count=False)
        lookup_draft_(st, cache.lens)
        replays = 0
        if n > 1:
            H = cfg.n_head
            work = torch.empty(decode_attention_work_numel(B * S, H, cfg.n_embd // H, t_max), dtype=torch.float32,
                               device=dev)
            verify = VerifyKV(cache, S, st.nq, work)

            def accept_and_draft(hv):
                lm_head_logits_(hv, weight, logits)
                lookup_accept_(logits, V, st, cache.lens, min_new_tokens, sup, stop)
                lookup_draft_(st, cache.lens)

            # lookup_draft_ writes the next slots into the graph's own input buffers; lookup_accept_ advances the
            # cache by the tokens it emits, up to k + 1 per replay, while the host counts one per replay. A live row
            # emits at least one token per replay, so at most n - 1 replays follow the first token and the host's
            # lengths stay at most max(lengths) + n - 1 < t_max: check_room never fires.
            graph = DecodeGraph(self, cache, tt_v is not None, head=accept_and_draft, ids=st.ids, tt=tt_v,
                                step=lambda ids, tt, c: self._verify_hidden(ids, st.pos, tt, verify))
            replays = graph.run(n - 1, st.done, period=LOOKUP_POLL_PERIOD)
        self.lookup_stats = {"emitted": st.emitted, "steps": st.steps, "replays": replays}
        return st.tokens, (st.tokens >= 0).sum(1)

    def _generate_assisted(self, draft: "GPT2DoubleHeads", K: int, input_ids, lengths, token_type_ids, reply_type,
                           max_new_tokens, temperature, top_k, top_p, stop_ids, suppress_ids, min_new_tokens, seed,
                           filters, rejection: bool) -> Tuple[torch.Tensor, torch.Tensor]:
        """``generate`` with ``draft`` proposing up to ``K`` tokens per row and round (``ops/assisted.py``), verified
        by coupled draws or, with ``rejection`` (temperature > 0), by rejection sampling."""
        B, T, lengths, n, t_max, last, tt_new, native = self._decode_setup(
            "generate", input_ids, lengths, token_type_ids, reply_type, max_new_tokens, min_new_tokens, 1.0, 0,
            num_beams=K + 1, rows_name="verify rows (batch x (num_assistant_tokens + 1))")
        dc = draft.cfg
        if t_max > dc.n_positions:
            raise ValueError(f"generate: the longest prompt ({max(lengths)}) plus max_new_tokens ({n}) exceeds the "
                             f"assistant_model's n_positions = {dc.n_positions}")
        cfg, dev, weight, V, S = self.cfg, input_ids.device, self.wte.weight, self.cfg.vocab_size, K + 1
        seeds = _row_seeds(seed, B, dev)
        tt_v = tt_new.repeat_interleave(S) if tt_new is not None else None
        cache = self.new_cache(B, t_max)
        h = self.hidden(input_ids, token_type_ids, cache=cache, lengths=lengths)[torch.arange(B, device=dev), last]
        # the prompt's last token plays the row's last emitted token x_b, whose logits the prefill gave: lens = len - 1
        cache.lens.sub_(1)
        # The draft's cache has K more positions than the model's: a round runs all K + 1 draft steps, and those past a
        # row's cap write there (their positions are clamped to n_positions - 1); nothing a real slot reads.
        dcache = KVCache(dc.n_layer, B, dc.n_head, t_max + K, dc.n_embd // dc.n_head, draft.wte.weight.dtype, dev)
        draft.hidden(input_ids, token_type_ids, cache=dcache, lengths=lengths)
        if not native:                              # CPU / not bf16: the definition on fp32 PyTorch logits
            from ..ops.assisted import assist_round, draw_slots, spec_slots
            from ..ops.lookup import lookup_accept
            head, dhead = weight.float(), draft.wte.weight.float()
            seq = torch.zeros(B, t_max, dtype=torch.int32)
            seq[:, :T] = input_ids.cpu()
            lens = cache.lens.cpu()
            emitted, done, steps = (torch.zeros(B, dtype=torch.int32) for _ in range(3))
            tokens = torch.full((B, n), -1, dtype=torch.int64)
            kw = dict(min_new=min_new_tokens, suppress_ids=suppress_ids, **filters)
            scal = (V, temperature, top_k, top_p, seeds.cpu().tolist())
            ids, nq = torch.zeros(B * S, dtype=torch.int64), torch.ones(B, dtype=torch.int32)
            g = draw_slots(self.lm_logits(h, head), *scal, lens, emitted, done, nq, **kw)
            lookup_accept(None, V, ids, nq, seq, lens, emitted, done, tokens, None, stop_ids=stop_ids, drawn=g)
            rounds = 0
            while not bool(done.all()):             # every live row emits at least one token per round
                ids, pos, nq, d_in, d_pos = assist_round(seq, lens, emitted, done, K, n, dc.n_positions)
                dcache.lens.copy_(lens)
                ids = ids.view(B, S)
                qlogits = []
                for j in range(S):
                    hd = draft._blocks(draft._embed(d_in.to(dev), tt_new, d_pos[j].to(dev)), dcache)
                    dcache.lens.add_(1)
                    if j < K:
                        qlogits.append(draft.lm_logits(hd, dhead))
                        d = draw_slots(qlogits[-1], *scal, lens, emitted, done, nq, j, True, **kw)
                        d_in = torch.from_numpy(d[:, 0]).clamp(min=0)
                        ids[:, j + 1] = d_in
                ids = ids.reshape(-1)
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
            self.assist_stats = {"emitted": emitted, "steps": steps, "replays": rounds}
            return tokens.to(dev), (tokens >= 0).sum(1).to(dev)

        from ..ops import (AssistState, assist_round_, decode_attention_work_numel, lm_head_logits_, lookup_accept_,
                           lookup_accept_drawn_, sample_slots_, spec_slots_)

        st = AssistState(B, K, n, t_max, dev, V if rejection else 0)
        st.seq[:, :T] = input_ids
        dweight = draft.wte.weight
        logits = torch.empty(B * S, weight.shape[0], dtype=torch.float32, device=dev)
        dlogits = torch.empty(B, dweight.shape[0], dtype=torch.float32, device=dev)
        sup, stop = (torch.tensor(list(x), dtype=torch.int32, device=dev) for x in (suppress_ids, stop_ids))
        draw = (V, temperature, top_k, top_p, seeds, st, cache.lens)

        def accept(lg, first=False):
            if temperature == 0:                    # greedy verification: the arg-max kernel of prompt lookup
                lookup_accept_(lg, V, st, cache.lens, min_new_tokens, sup, stop, count=not first)
            elif rejection and not first:
                spec_slots_(lg, V, temperature, top_k, top_p, seeds, st, cache.lens, min_new_tokens, sup, **filters)
                lookup_accept_drawn_(st, cache.lens, stop, flagged=True)
            else:
                sample_slots_(lg, *draw, 0, min_new_tokens, sup, **filters)
                lookup_accept_drawn_(st, cache.lens, stop, count=not first, first=first)

        lm_head_logits_(h, weight, logits[:B])      # the first token, from the prefill's last positions
        accept(logits[:B], first=True)
        replays = 0
        if n > 1:
            H = cfg.n_head
            work = torch.empty(decode_attention_work_numel(B * S, H, cfg.n_embd // H, t_max), dtype=torch.float32,
                               device=dev)
            verify = VerifyKV(cache, S, st.nq, work)

            def round_step(ids, tt, c):
                # a round depends on the model's state alone: its set-up also resets the draft cache's lengths
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

            # lookup_accept_ advances the cache by the tokens it emits, up to k + 1 per replay, while the host counts
            # one per replay; as for prompt lookup, at most n - 1 replays follow the first token, so check_room never
            # fires
            graph = DecodeGraph(self, cache, tt_v is not None, head=head_and_accept, ids=st.ids, tt=tt_v,
                                step=round_step)
            replays = graph.run(n - 1, st.done, period=LOOKUP_POLL_PERIOD)
        self.assist_stats = {"emitted": st.emitted, "steps": st.steps, "replays": replays}
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
                           no_repeat_ngram_size: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
        """Batched contrastive search (Su et al., 2022; HuggingFace's ``penalty_alpha`` + ``top_k``); the definition is
        in ``ops/contrastive.py``.

        Each step takes the ``top_k`` most likely next tokens of a row, runs one decode step for each of them, and emits
        the candidate with the best ``(1 - penalty_alpha) p - penalty_alpha s``, where ``s`` is the largest cosine
        between the candidate's final hidden state and the hidden states of the row's sequence so far (its prompt
        without padding, then its emitted tokens). ``penalty_alpha = 0`` or ``top_k = 1`` is greedy decoding.
        ``input_ids``, ``lengths``, ``reply_type``, token types, ``stop_ids``, ``suppress_ids``, ``min_new_tokens``,
        the repetition controls and the return value ``(tokens, n_new)`` work as in ``generate``.

        The prompts are prefilled into a KV cache of ``max(lengths) + max_new_tokens`` positions (more than
        ``n_positions`` is a ``ValueError``) and the context is taken from the prefill's hidden states. On CUDA with
        bf16 weights (at most 64 rows) every token replays one CUDA graph: the candidate step (``ops.cand_attention_``
        attends for all k candidates over the shared cache), re-rank and commit (``ops.contrastive_rerank_``), the LM
        head on the winners, ``ops.penalize_repeats_`` when on, and the next candidates (``ops.contrastive_select_``);
        the host reads the done flags once every 8 tokens, a period late. Elsewhere the same loop runs eagerly:
        candidates decode through ``decode_attention`` on a k-fold copy of the rows and the selection runs in fp64
        (``ops/contrastive.py``)."""
        from ..ops import CONTRASTIVE_MAX_K
        from ..ops.contrastive import check_contrastive_args, rerank_row, select_candidates

        check_contrastive_args("contrastive_search", top_k, penalty_alpha, CONTRASTIVE_MAX_K)
        K, alpha = int(top_k), float(penalty_alpha)
        B, T, lengths, n, t_max, last, tt_new, native = self._decode_setup(
            "contrastive_search", input_ids, lengths, token_type_ids, reply_type, max_new_tokens, min_new_tokens,
            repetition_penalty, no_repeat_ngram_size)
        cfg, dev, weight = self.cfg, input_ids.device, self.wte.weight
        tt_cand = tt_new.repeat_interleave(K) if tt_new is not None else None
        cache = self.new_cache(B, t_max)
        hs = self.hidden(input_ids, token_type_ids, cache=cache, lengths=lengths)
        h = hs[torch.arange(B, device=dev), last].contiguous()
        V, L, H = cfg.vocab_size, cfg.n_layer, cfg.n_head
        D = cfg.n_embd
        reps = _Repeats.create(input_ids, cache, V, repetition_penalty, no_repeat_ngram_size)
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
        mc_token_ids, [B] mc_labels; -100 labels are ignored."""
        B, C, T = input_ids.shape
        ids = input_ids.reshape(B * C, T)
        tt = token_type_ids.reshape(B * C, T) if token_type_ids is not None else None
        h = self.hidden(ids, tt)                                              # [B*C, T, D]
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
            scale = (lm_coef / n_valid.clamp(min=1).to(torch.float32)).reshape(1)
            lm_term = _ChunkedLMLoss.apply(shift_h, self.wte.weight, shift_l, self.cfg.lm_chunk_rows,
                                           self.cfg.vocab_size, scale)
            lm_loss = lm_term / lm_coef if lm_coef != 0 else lm_term
            if compact:
                # a batch with more scored rows than the capacity must not train silently on a subset
                lm_loss = torch.where(n_valid > cap, torch.full_like(lm_loss, float("nan")), lm_loss)
                lm_term = torch.where(n_valid > cap, torch.full_like(lm_term, float("nan")), lm_term)
        if mc_token_ids is not None and mc_labels is not None:
            idx = mc_token_ids.reshape(B * C, 1, 1).expand(-1, 1, h.shape[-1])
            cls_h = h.gather(1, idx).squeeze(1)                               # [B*C, D]
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
