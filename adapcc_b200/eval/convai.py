"""ConvAI2-style evaluation of the double-heads GPT-2: hits@1, perplexity, F1 — and the reply sampler they share.

The reference evaluates through ParlAI (``eval_hits`` / ``eval_ppl`` / ``eval_f1`` driving a ``TransformerAgent``,
/root/reference/models/gpt2/convai_evaluation.py:27-239), which is not available offline; the three metrics are
computed here directly on PersonaChat-schema data:

* **hits@1** — the multiple-choice head ranks the gold reply first among the utterance's candidates
  (convai_evaluation.py:122-146);
* **perplexity** — token-level ``exp(mean NLL)`` of the gold reply, and ParlAI's *word-level* variant built on
  :func:`next_word_probability` (a BPE-prefix → words table turns the model's next-token distribution into a
  distribution over dictionary words, convai_evaluation.py:160-197);
* **F1** — word-overlap F1 between a sampled reply and the gold one (ParlAI's normalisation: lower case, no
  punctuation, no articles).

Batched over candidates, no ParlAI, runs on CPU (tests) or GPU.
"""
from __future__ import annotations

import math
import re
import string
from collections import Counter, defaultdict
from typing import Dict, Iterable, List, Optional, Sequence

import torch
import torch.nn.functional as F

from ..data.personachat import IGNORE, build_input_from_segments
from ..data.tokenizer import DialogTokenizer
from ..ops.sampling import top_filtering
from ..ops.synthid import check_synthid_args, is_synthid_config


# ----------------------------------------------------------------------------------------------------------------
# model access (the training forward only returns losses)
# ----------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def mc_scores(model, input_ids: torch.Tensor, token_type_ids: torch.Tensor, mc_token_ids: torch.Tensor) -> torch.Tensor:
    """Multiple-choice logits ``[B, C]`` for ``[B, C, T]`` inputs."""
    B, C, T = input_ids.shape
    h = model.hidden(input_ids.reshape(B * C, T), token_type_ids.reshape(B * C, T))
    idx = mc_token_ids.reshape(B * C, 1, 1).expand(-1, 1, h.shape[-1])
    return model.mc_head(h.gather(1, idx).squeeze(1)).view(B, C).float()


# ----------------------------------------------------------------------------------------------------------------
# sampling
# ----------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def sample_reply(model, tokenizer: DialogTokenizer, persona, history, max_length: int = 20, min_length: int = 1,
                 temperature: float = 0.7, top_k: int = 0, top_p: float = 0.9, no_sample: bool = False,
                 device="cpu", generator: Optional[torch.Generator] = None) -> List[int]:
    """Generate a reply token by token: the input is rebuilt from persona + history + the partial reply each step, so
    speaker tokens and token types stay those of training (the reference's ``sample_sequence``, interact.py:59-87);
    special tokens end the reply, and are re-drawn while the reply is shorter than ``min_length``.

    When an input is the previous one plus the newest token, that token costs one cached decode step
    (``GPT2DoubleHeads.decode_step``, graph-replayed on CUDA with the native kernels); when history truncation moved
    the prefix, the input is prefilled into the cache again."""
    from ..models.gpt2 import CachedDecoder

    special = set(tokenizer.special_ids)
    out: List[int] = []
    head = model.wte.weight.float()                            # the fp32 LM head, converted once per call
    dec, prev = CachedDecoder(model), None
    for step in range(max_length):
        inst = build_input_from_segments(persona, history, out, tokenizer, with_eos=False, max_len=model.cfg.n_positions)
        cur = (inst.input_ids, inst.token_type_ids)
        if (prev is not None and len(cur[0]) == len(prev[0]) + 1 and cur[0][:-1] == prev[0]
                and cur[1][:-1] == prev[1]):
            h = dec.extend(torch.tensor([cur[0][-1:]], device=device), torch.tensor([cur[1][-1:]], device=device))
        else:
            h = dec.restart(torch.tensor([cur[0]], device=device), torch.tensor([cur[1]], device=device))
        prev = cur
        logits = model.lm_logits(h[0], head) / max(temperature, 1e-6)   # 1-D h: the GEMV the draws were made with
        probs = F.softmax(top_filtering(logits, top_k, top_p), dim=-1)
        nxt = int(torch.argmax(probs)) if no_sample else int(torch.multinomial(probs, 1, generator=generator))
        if step < min_length and nxt in special:
            tries = 0
            while nxt in special and float(probs.max()) < 1.0 and tries < 64:
                nxt = int(torch.multinomial(probs, 1, generator=generator))
                tries += 1
        if nxt in special:
            break
        out.append(nxt)
    return out


@torch.no_grad()
def sample_replies(model, tokenizer: DialogTokenizer, dialogs: Sequence, max_length: int = 20, min_length: int = 1,
                   temperature: float = 0.7, top_k: int = 0, top_p: float = 0.9, no_sample: bool = False,
                   device="cpu", seeds: Optional[Sequence[int]] = None, num_beams: int = 0,
                   repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0,
                   penalty_alpha: float = 0.0, prompt_lookup_num_tokens: int = 0, min_p: float = 0.0,
                   typical_p: float = 1.0, epsilon_cutoff: float = 0.0, eta_cutoff: float = 0.0,
                   assistant_model=None, num_assistant_tokens: int = 4,
                   assistant_verification: str = "coupled", beam_sample: bool = False, num_beam_groups: int = 1,
                   diversity_penalty: float = 0.0, guidance_scale: float = 1.0,
                   guidance_negative: str = "last_token", sequence_bias=None,
                   bad_words_ids=None, top_h: float = 0.0, kv_cache_dtype: Optional[str] = None,
                   frequency_penalty: float = 0.0, presence_penalty: float = 0.0,
                   context_no_repeat_ngram_size: int = 0, watermarking_config=None,
                   dola_layers=None) -> List[List[int]]:
    """The batched counterpart of :func:`sample_reply`: one reply per ``(persona, history)`` in ``dialogs``, all drawn by
    one ``GPT2DoubleHeads.generate`` call, or decoded by one ``GPT2DoubleHeads.beam_search`` call with ``num_beams``
    beams when ``num_beams > 0``, or by one ``GPT2DoubleHeads.contrastive_search`` call with ``top_k`` candidates when
    ``penalty_alpha > 0`` (the sampling arguments and seeds are then unused). Each prompt is built without a
    reply and with the history truncated so that ``max_length`` new tokens fit into ``n_positions`` up front; a new
    token takes the prompt's last token type. Special tokens end a reply and cannot be drawn while it is shorter than
    ``min_length`` (removed before the top-k / top-p filtering, where ``sample_reply`` re-draws after it).
    ``seeds``: one per dialogue (default 0, 1, ...). ``repetition_penalty`` and ``no_repeat_ngram_size`` go to
    ``generate`` / ``beam_search`` / ``contrastive_search`` (``ops/repeats.py``); the prompt counts as part of each
    reply's sequence. ``prompt_lookup_num_tokens`` > 0 (with ``no_sample``) verifies up to that many draft tokens per
    step, copied from the prompt and the reply so far; the replies are the greedy ones (``ops/lookup.py``).
    ``min_p``, ``typical_p``, ``epsilon_cutoff``, ``eta_cutoff`` and ``top_h`` go to ``generate`` (the truncation
    filters of the sampler, ``ops/sampling.py``), and to ``beam_search`` with ``beam_sample``. ``assistant_model`` (a
    draft model) and ``num_assistant_tokens`` go to ``generate`` (assisted generation, ``ops/assisted.py``): the replies are the ones drawn without it; with ``num_beams`` or
    ``penalty_alpha`` it is a ``ValueError``. ``assistant_verification="rejection"`` verifies the drafts by rejection
    sampling instead: each reply token is still drawn from the model's distribution, but not the same draw.
    ``beam_sample`` with ``num_beams > 0``: beam sampling (``beam_search(do_sample=True)``) with ``temperature``,
    ``top_k``, ``top_p``, the truncation filters and the seeds. ``num_beam_groups`` and ``diversity_penalty`` go to
    ``beam_search`` (diverse beam search, ``ops/beam.py``). ``guidance_scale`` != 1 goes to ``generate`` (classifier-free guidance,
    ``ops/guidance.py``) with each dialogue's negative prompt: ``guidance_negative="last_token"`` is the prompt's last
    token (HuggingFace's default), ``"no_persona"`` the same dialogue without the persona (built and truncated as the
    prompt is), so guidance pushes each reply towards its persona. Guidance with ``num_beams``, ``penalty_alpha``,
    prompt lookup or an assistant is a ``ValueError``. ``sequence_bias`` and ``bad_words_ids`` (HuggingFace's; token
    ids of the dialogue tokenizer) go to ``generate`` / ``beam_search`` / ``contrastive_search`` (``ops/repeats.py``);
    with prompt lookup or an assistant they are a ``ValueError``. So do ``frequency_penalty`` and
    ``presence_penalty`` (over each reply's own tokens) and ``context_no_repeat_ngram_size`` (no n-gram of the persona
    and history copied into the reply), and ``watermarking_config`` (the green-list watermark,
    ``ops/watermark.py``). ``kv_cache_dtype`` (``"fp8_e4m3"``: an fp8 KV
    cache, ``ops/kvcache.py``) goes to ``generate`` / ``beam_search``; with ``penalty_alpha``, prompt lookup or an
    assistant it is a ``ValueError``. ``dola_layers`` (``"low"``, ``"high"`` or a list of layer indices; None: off)
    goes to ``generate`` (DoLa layer-contrast decoding, ``ops/dola.py``); with ``num_beams``, ``penalty_alpha`` or
    guidance it is a ``ValueError``."""
    from ..ops.assisted import check_verification
    check_verification("sample_replies", assistant_verification, assistant_model)
    if assistant_model is not None and (num_beams > 0 or penalty_alpha > 0):
        raise ValueError("sample_replies: assistant_model drafts for sampling and greedy generation only, not with "
                         f"num_beams > 0 or penalty_alpha > 0 (got {num_beams}, {penalty_alpha})")
    if guidance_negative not in ("last_token", "no_persona"):
        raise ValueError(f"sample_replies: guidance_negative must be 'last_token' or 'no_persona', got "
                         f"{guidance_negative!r}")
    if guidance_scale != 1.0 and (num_beams > 0 or penalty_alpha > 0 or prompt_lookup_num_tokens > 0
                                  or assistant_model is not None):
        raise ValueError("sample_replies: guidance_scale != 1 works with sampling and greedy generation only, not with "
                         "num_beams > 0, penalty_alpha > 0, prompt_lookup_num_tokens > 0 or assistant_model (got "
                         f"{num_beams}, {penalty_alpha}, {prompt_lookup_num_tokens}, "
                         f"{type(assistant_model).__name__})")
    if dola_layers is not None and (num_beams > 0 or penalty_alpha > 0 or guidance_scale != 1.0):
        raise ValueError("sample_replies: dola_layers works with sampling and greedy generation only, not with "
                         f"num_beams > 0, penalty_alpha > 0 or guidance_scale != 1 (got {num_beams}, {penalty_alpha}, "
                         f"{guidance_scale})")
    pad = tokenizer.special_ids[-1]

    def padded(persona_of):
        insts = [build_input_from_segments(persona_of(persona), history, [], tokenizer, with_eos=False,
                                           max_len=model.cfg.n_positions - max_length) for persona, history in dialogs]
        lengths = [len(i.input_ids) for i in insts]
        T = max(lengths)
        ids = torch.tensor([i.input_ids + [pad] * (T - len(i.input_ids)) for i in insts], device=device)
        tt = torch.tensor([i.token_type_ids + [pad] * (T - len(i.token_type_ids)) for i in insts], device=device)
        return insts, lengths, ids, tt

    insts, lengths, ids, tt = padded(lambda persona: persona)
    guidance = {}
    if guidance_scale != 1.0:
        guidance = dict(guidance_scale=guidance_scale)
        if guidance_negative == "no_persona":
            _, n_lengths, n_ids, n_tt = padded(lambda persona: [])
            guidance.update(negative_prompt_ids=n_ids, negative_lengths=n_lengths, negative_token_type_ids=n_tt)
    reply_type = torch.tensor([i.token_type_ids[-1] for i in insts], device=device)
    seed = torch.tensor(list(seeds) if seeds is not None else range(len(insts)), dtype=torch.int64)
    special = list(tokenizer.special_ids)
    repeats = dict(repetition_penalty=repetition_penalty, no_repeat_ngram_size=no_repeat_ngram_size,
                   kv_cache_dtype=kv_cache_dtype, frequency_penalty=frequency_penalty,
                   presence_penalty=presence_penalty, context_no_repeat_ngram_size=context_no_repeat_ngram_size)
    filters = dict(min_p=min_p, typical_p=typical_p, epsilon_cutoff=epsilon_cutoff, eta_cutoff=eta_cutoff, top_h=top_h)
    if sequence_bias is not None:
        repeats["sequence_bias"] = sequence_bias
    if bad_words_ids is not None:
        repeats["bad_words_ids"] = bad_words_ids
    if watermarking_config is not None:
        repeats["watermarking_config"] = watermarking_config
    if num_beams > 0:
        sampled = dict(do_sample=True, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed,
                       **filters) if beam_sample else {}
        tokens, n_new, _ = model.beam_search(ids, lengths, tt, reply_type, num_beams=num_beams,
                                             max_new_tokens=max_length, stop_ids=special, suppress_ids=special,
                                             min_new_tokens=min_length, num_beam_groups=num_beam_groups,
                                             diversity_penalty=diversity_penalty, **repeats, **sampled)
        return [row[:k] for row, k in zip(tokens.tolist(), n_new.tolist())]
    if penalty_alpha > 0:
        tokens, n_new = model.contrastive_search(ids, lengths, tt, reply_type, top_k=top_k, penalty_alpha=penalty_alpha,
                                                 max_new_tokens=max_length, stop_ids=special, suppress_ids=special,
                                                 min_new_tokens=min_length, **repeats)
        return [row[:k] for row, k in zip(tokens.tolist(), n_new.tolist())]
    tokens, n_new = model.generate(ids, lengths, tt, reply_type, max_new_tokens=max_length,
                                   temperature=0.0 if no_sample else temperature, top_k=top_k, top_p=top_p,
                                   stop_ids=special, suppress_ids=special, min_new_tokens=min_length, seed=seed,
                                   prompt_lookup_num_tokens=prompt_lookup_num_tokens, **filters,
                                   assistant_model=assistant_model, num_assistant_tokens=num_assistant_tokens,
                                   assistant_verification=assistant_verification, **repeats, **guidance,
                                   **({} if dola_layers is None else dict(dola_layers=dola_layers)))
    return [row[:k] for row, k in zip(tokens.tolist(), n_new.tolist())]


def bad_word_ids(tokenizer, words: Sequence[str]) -> List[List[int]]:
    """``bad_words_ids`` banning each of ``words`` (surrounding blanks stripped, empty ones skipped) as the dialogue
    tokenizer encodes it both at the start of a text and after a space, each distinct encoding once."""
    out: List[List[int]] = []
    for w in words:
        w = w.strip()
        for text in (w, " " + w) if w else ():
            ids = list(tokenizer.encode(text))
            if ids and ids not in out:
                out.append(ids)
    return out


# ----------------------------------------------------------------------------------------------------------------
# metrics
# ----------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def evaluate_tensors(model, loader: Iterable[Dict[str, torch.Tensor]], device="cpu") -> Dict[str, float]:
    """hits@1 (multiple-choice accuracy), token NLL / perplexity of the gold replies over a validation loader of
    ``[B, C, T]`` batches (``data.get_data_loaders``); the same quantities the reference's training script tracks as
    ``accuracy`` / ``nll`` / ``average_ppl`` (train_gpt2_ddp.py:201-208)."""
    hits = total = 0
    nll_sum, n_tok = 0.0, 0
    for batch in loader:
        b = {k: v.to(device) for k, v in batch.items()}
        B, C, T = b["input_ids"].shape
        h = model.hidden(b["input_ids"].reshape(B * C, T), b["token_type_ids"].reshape(B * C, T))
        idx = b["mc_token_ids"].reshape(B * C, 1, 1).expand(-1, 1, h.shape[-1])
        mc = model.mc_head(h.gather(1, idx).squeeze(1)).view(B, C).float()
        hits += int((mc.argmax(-1) == b["mc_labels"]).sum())
        total += B
        gold = h.view(B, C, T, -1)[:, -1]                                   # LM labels live on the last candidate
        labels = b["lm_labels"][:, -1, 1:].reshape(-1)
        keep = labels != IGNORE
        if keep.any():
            rows = gold[:, :-1].reshape(-1, gold.shape[-1])[keep]
            nll_sum += float(F.cross_entropy(model.lm_logits(rows), labels[keep], reduction="sum"))
            n_tok += int(keep.sum())
    nll = nll_sum / max(1, n_tok)
    return {"hits@1": hits / max(1, total), "nll": nll, "ppl": math.exp(min(nll, 50.0)), "examples": total, "tokens": n_tok,
            "hits": hits, "nll_sum": nll_sum}


_ARTICLES = re.compile(r"\b(a|an|the)\b")
_PUNCT = str.maketrans({c: " " for c in string.punctuation})


def normalize_answer(s: str) -> List[str]:
    return _ARTICLES.sub(" ", s.lower().translate(_PUNCT)).split()


def f1_score(guess: str, answers: Sequence[str]) -> float:
    """Best word-overlap F1 of ``guess`` against any of ``answers``."""
    g = normalize_answer(guess)
    best = 0.0
    for a in answers:
        ref = normalize_answer(a)
        common = sum((Counter(g) & Counter(ref)).values())
        if common:
            p, r = common / len(g), common / len(ref)
            best = max(best, 2 * p * r / (p + r))
    return best


def build_prefix2words(tokenizer: DialogTokenizer, word_freq: Dict[str, int], smoothing: int = 5) -> Dict[int, Dict[str, float]]:
    """first BPE token of a word → {word: share of that prefix's (smoothed) frequency mass}."""
    table: Dict[int, Dict[str, float]] = defaultdict(dict)
    for word, freq in word_freq.items():
        table[tokenizer.first_symbol_id(" " + word)][word] = freq + smoothing
    for words in table.values():
        z = sum(words.values())
        for w in words:
            words[w] /= z
    return dict(table)


@torch.no_grad()
def next_word_probability(model, tokenizer: DialogTokenizer, persona, history, partial_out: Sequence[str],
                          prefix2words: Dict[int, Dict[str, float]], device="cpu") -> Dict[str, float]:
    """Distribution over dictionary words for the next word of the reply, given the words produced so far."""
    partial = tokenizer.encode(" " + " ".join(partial_out)) if partial_out else []
    inst = build_input_from_segments(persona, history, partial, tokenizer, with_eos=False, max_len=model.cfg.n_positions)
    ids = torch.tensor(inst.input_ids, device=device).unsqueeze(0)
    tt = torch.tensor(inst.token_type_ids, device=device).unsqueeze(0)
    probs = F.softmax(model.lm_logits(model.hidden(ids, tt)[0, -1]), dim=-1)
    dist: Dict[str, float] = {}
    for prefix, words in prefix2words.items():
        p = float(probs[prefix])
        for w, share in words.items():
            dist[w] = p * share
    return dist


@torch.no_grad()
def evaluate_dialogs(model, tokenizer: DialogTokenizer, raw_split: list, eval_type: str = "f1", max_history: int = 2,
                     max_examples: int = 0, device="cpu", seed: int = 0, batch_size: int = 0, num_beams: int = 0,
                     repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0, penalty_alpha: float = 0.0,
                     prompt_lookup_num_tokens: int = 0, min_p: float = 0.0, typical_p: float = 1.0,
                     epsilon_cutoff: float = 0.0, eta_cutoff: float = 0.0, assistant_model=None,
                     num_assistant_tokens: int = 4, assistant_verification: str = "coupled",
                     beam_sample: bool = False, num_beam_groups: int = 1, diversity_penalty: float = 0.0,
                     guidance_scale: float = 1.0, guidance_negative: str = "last_token", sequence_bias=None,
                     bad_words_ids=None, top_h: float = 0.0, kv_cache_dtype: Optional[str] = None,
                     frequency_penalty: float = 0.0, presence_penalty: float = 0.0,
                     context_no_repeat_ngram_size: int = 0, watermarking_config=None, dola_layers=None,
                     **sample_kw) -> Dict[str, float]:
    """Run one metric over a RAW (string) PersonaChat split the way an agent would see it: persona + running history,
    gold reply = last candidate. ``eval_type``: ``hits@1`` | ``ppl`` (word-level) | ``f1``.

    ``batch_size > 0`` with ``f1``: the replies are generated ``batch_size`` at a time by :func:`sample_replies`, the
    reply of example n with seed ``(seed << 32) + n``, so the draws do not depend on the batch size. That path truncates
    the history so the whole reply fits up front and applies the min-length rule before filtering: its F1 comes from a
    different sample than the sequential path's (``batch_size=0``), not from the same replies.

    ``num_beams > 0`` with ``f1``: the replies are decoded by beam search instead (:func:`sample_replies`), on that
    batched path (one example at a time when ``batch_size`` is 0); with ``beam_sample`` by beam sampling, with the
    sampling arguments and the batched path's seeds; with ``num_beam_groups`` > 1 by diverse beam search with
    ``diversity_penalty``.

    ``repetition_penalty != 1`` or ``no_repeat_ngram_size > 0`` with ``f1``: the repetition controls of
    ``generate`` / ``beam_search`` (``ops/repeats.py``), also on that batched path; so do ``sequence_bias``,
    ``bad_words_ids``, ``frequency_penalty``, ``presence_penalty`` and ``context_no_repeat_ngram_size``.

    ``penalty_alpha > 0`` with ``f1``: the replies are decoded by contrastive search with ``top_k`` candidates
    (:func:`sample_replies`), on that batched path.

    ``prompt_lookup_num_tokens > 0`` with ``f1`` and ``no_sample``: greedy replies with prompt lookup decoding
    (:func:`sample_replies`), on that batched path.

    ``min_p > 0``, ``typical_p < 1``, ``epsilon_cutoff > 0``, ``eta_cutoff > 0`` or ``top_h > 0`` with ``f1``: the
    truncation filters of ``generate``'s sampler (``ops/sampling.py``), on that batched path; with ``beam_sample``
    they filter the beams too.

    ``assistant_model`` (a draft model) with ``f1``: assisted generation with up to ``num_assistant_tokens`` drafts per
    round (``ops/assisted.py``), on that batched path; the replies are those of the batched path without it, unless
    ``assistant_verification="rejection"`` (rejection sampling: replies from the same distribution, other draws).

    ``guidance_scale != 1`` with ``f1``: classifier-free guidance against ``guidance_negative`` (``"last_token"`` or
    ``"no_persona"``, see :func:`sample_replies`), on that batched path.

    ``kv_cache_dtype="fp8_e4m3"`` with ``f1``: the replies are decoded with an fp8 KV cache (``ops/kvcache.py``), on
    that batched path; comparing F1 with and without it measures what the quantization costs.

    ``watermarking_config`` with ``f1``: the replies carry the green-list watermark (``ops/watermark.py``), on that
    batched path, and the result also holds ``watermark_z``, the mean z-score of the replies scored on their own
    (``detect_watermark`` without the prompt; replies with nothing to score are left out), and
    ``watermark_detected``, the fraction of replies it flags, next to F1: what the mark costs in F1 against how
    reliably it is found. With a SynthID ``watermarking_config`` (``ops/synthid.py``) the replies are scored by
    ``detect_synthid`` instead, on their own, and the result holds ``synthid_score``, the replies' mean weighted mean
    score (replies with nothing to score are left out), and ``synthid_detected``, the fraction it flags.

    ``dola_layers`` with ``f1``: the replies are decoded with DoLa layer contrast (``ops/dola.py``), on that batched
    path."""
    from ..ops.assisted import check_verification
    check_verification("evaluate_dialogs", assistant_verification, assistant_model)
    repeats = (repetition_penalty != 1.0 or no_repeat_ngram_size > 0 or bool(sequence_bias)
               or bool(bad_words_ids) or frequency_penalty != 0 or presence_penalty != 0
               or context_no_repeat_ngram_size > 0 or watermarking_config is not None)
    bias = {k: v for k, v in (("sequence_bias", sequence_bias), ("bad_words_ids", bad_words_ids),
                              ("watermarking_config", watermarking_config)) if v is not None}
    counts = dict(frequency_penalty=frequency_penalty, presence_penalty=presence_penalty,
                  context_no_repeat_ngram_size=context_no_repeat_ngram_size)
    lookup = prompt_lookup_num_tokens > 0
    filters = dict(min_p=min_p, typical_p=typical_p, epsilon_cutoff=epsilon_cutoff, eta_cutoff=eta_cutoff, top_h=top_h)
    filtered = min_p > 0 or typical_p < 1 or epsilon_cutoff > 0 or eta_cutoff > 0 or top_h > 0
    assisted = assistant_model is not None
    if (batch_size > 0 or num_beams > 0 or repeats or penalty_alpha > 0 or lookup or filtered
            or assisted or guidance_scale != 1.0 or kv_cache_dtype is not None
            or dola_layers is not None) and eval_type == "f1":
        return _evaluate_f1_batched(model, tokenizer, raw_split, max_history, max_examples, device, seed,
                                    max(batch_size, 1), num_beams=num_beams, repetition_penalty=repetition_penalty,
                                    no_repeat_ngram_size=no_repeat_ngram_size, penalty_alpha=penalty_alpha,
                                    prompt_lookup_num_tokens=prompt_lookup_num_tokens, **filters,
                                    assistant_model=assistant_model, num_assistant_tokens=num_assistant_tokens,
                                    assistant_verification=assistant_verification, beam_sample=beam_sample,
                                    num_beam_groups=num_beam_groups, diversity_penalty=diversity_penalty,
                                    guidance_scale=guidance_scale, guidance_negative=guidance_negative, **bias,
                                    kv_cache_dtype=kv_cache_dtype, **counts,
                                    **({} if dola_layers is None else dict(dola_layers=dola_layers)), **sample_kw)
    gen = torch.Generator(device="cpu").manual_seed(seed)
    word_freq: Counter = Counter()
    if eval_type == "ppl":
        for d in raw_split:
            for u in d["utterances"]:
                word_freq.update(normalize_answer(u["candidates"][-1]))
        table = build_prefix2words(tokenizer, word_freq)
    n = 0
    acc = 0.0
    logloss, words = 0.0, 0
    for d in raw_split:
        persona = [tokenizer.encode(p) for p in d["personality"]]
        for u in d["utterances"]:
            if max_examples and n >= max_examples:
                break
            hist = [tokenizer.encode(h) for h in u["history"][-(2 * max_history + 1):]]
            gold = u["candidates"][-1]
            if eval_type == "hits@1":
                insts = [build_input_from_segments(persona, hist, tokenizer.encode(c), tokenizer, max_len=model.cfg.n_positions)
                         for c in u["candidates"]]
                T = max(len(i.input_ids) for i in insts)
                pad = tokenizer.pad_id
                ids = torch.tensor([i.input_ids + [pad] * (T - len(i.input_ids)) for i in insts], device=device)[None]
                tt = torch.tensor([i.token_type_ids + [pad] * (T - len(i.token_type_ids)) for i in insts], device=device)[None]
                mc = torch.tensor([i.mc_token_id for i in insts], device=device)[None]
                acc += float(int(mc_scores(model, ids, tt, mc)[0].argmax()) == len(insts) - 1)
            elif eval_type == "ppl":
                said: List[str] = []
                for w in normalize_answer(gold):
                    dist = next_word_probability(model, tokenizer, persona, hist, said, table, device)
                    z = sum(dist.values()) or 1.0
                    logloss -= math.log(max(dist.get(w, 0.0) / z, 1e-7))
                    words += 1
                    said.append(w)
            else:
                out = sample_reply(model, tokenizer, persona, hist, device=device, generator=gen, **sample_kw)
                acc += f1_score(tokenizer.decode(out), [gold])
            n += 1
    if eval_type == "ppl":
        return {"ppl": math.exp(min(logloss / max(1, words), 50.0)), "words": words, "examples": n}
    return {eval_type: acc / max(1, n), "examples": n}


def _evaluate_f1_batched(model, tokenizer, raw_split, max_history, max_examples, device, seed, batch_size, **sample_kw):
    examples = []
    for d in raw_split:
        persona = [tokenizer.encode(p) for p in d["personality"]]
        for u in d["utterances"]:
            if max_examples and len(examples) >= max_examples:
                break
            hist = [tokenizer.encode(h) for h in u["history"][-(2 * max_history + 1):]]
            examples.append((persona, hist, u["candidates"][-1]))
    acc = 0.0
    wm = sample_kw.get("watermarking_config")
    z, flagged = [], 0
    for s in range(0, len(examples), batch_size):
        chunk = examples[s:s + batch_size]
        seeds = [((seed & 0x7FFFFFFF) << 32) + s + j for j in range(len(chunk))]
        replies = sample_replies(model, tokenizer, [(p, h) for p, h, _ in chunk], device=device, seeds=seeds,
                                 **sample_kw)
        acc += sum(f1_score(tokenizer.decode(r), [gold]) for r, (_, _, gold) in zip(replies, chunk))
        if wm is not None and is_synthid_config(wm):
            from ..ops.synthid import detect_synthid

            width = max(int(check_synthid_args("evaluate_dialogs", wm).ngram_len), max(len(r) for r in replies))
            ids = torch.tensor([r + [0] * (width - len(r)) for r in replies], dtype=torch.int64)
            det = detect_synthid(ids.to(device), wm, lengths=[len(r) for r in replies])
            z += [float(x) for x in det.weighted_mean_score if math.isfinite(x)]
            flagged += int(det.prediction.sum())
        elif wm is not None:
            from ..ops.watermark import detect_watermark

            width = max(1, max(len(r) for r in replies))
            ids = torch.tensor([r + [0] * (width - len(r)) for r in replies], dtype=torch.int64)
            det = detect_watermark(ids.to(device), wm, lengths=[len(r) for r in replies])
            z += [float(x) for x in det.z_score if math.isfinite(x)]
            flagged += int(det.prediction.sum())
    out = {"f1": acc / max(1, len(examples)), "examples": len(examples)}
    if wm is not None and is_synthid_config(wm):
        out.update(synthid_score=sum(z) / len(z) if z else float("nan"),
                   synthid_detected=flagged / max(1, len(examples)))
    elif wm is not None:
        out.update(watermark_z=sum(z) / len(z) if z else float("nan"),
                   watermark_detected=flagged / max(1, len(examples)))
    return out
