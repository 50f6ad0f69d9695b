"""ConvAI2-style evaluation of a fine-tuned dialogue model: ``--eval_type hits@1 | ppl | f1``
(the reference's /root/reference/models/gpt2/convai_evaluation.py, which drives ParlAI's eval_hits / eval_ppl / eval_f1;
here the three metrics are computed directly, see adapcc_b200/eval/convai.py).

    python examples/eval_gpt2_convai.py --model_checkpoint ck.pt --eval_type hits@1 [--dataset_path personachat.json]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from adapcc_b200.data import synthetic_personachat  # noqa: E402
from adapcc_b200.eval import evaluate_dialogs, load_model_from_checkpoint  # noqa: E402
from adapcc_b200.eval.convai import bad_word_ids  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--model_checkpoint", required=True, help="file written by examples/train_gpt2_personachat.py --checkpoint")
    p.add_argument("--dataset_path", default="", help="PersonaChat-schema JSON (its 'valid' split is scored); empty: synthetic")
    p.add_argument("--synthetic_dialogs", type=int, default=256)
    p.add_argument("--eval_type", default="hits@1", choices=["hits@1", "ppl", "f1"])
    p.add_argument("--max_history", type=int, default=2)
    p.add_argument("--max_examples", type=int, default=0)
    p.add_argument("--device", default="cuda" if torch.cuda.is_available() else "cpu")
    p.add_argument("--no_sample", action="store_true")
    p.add_argument("--max_length", type=int, default=20)
    p.add_argument("--min_length", type=int, default=1)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--temperature", type=float, default=0.7)
    p.add_argument("--top_k", type=int, default=20)
    p.add_argument("--top_p", type=float, default=0.9)
    p.add_argument("--batch_size", type=int, default=0,
                   help="f1: generate this many replies at a time with GPT2DoubleHeads.generate (0: one by one). The "
                        "batched path truncates history so the reply fits up front and suppresses special tokens "
                        "before filtering, so its F1 is a different sample")
    p.add_argument("--num_beams", type=int, default=0,
                   help="f1: decode the replies with GPT2DoubleHeads.beam_search and this many beams (0: sample)")
    p.add_argument("--beam_sample", action="store_true",
                   help="f1 with --num_beams: beam sampling, the beams' candidates drawn with --temperature, --top_k "
                        "and --top_p instead of ranked")
    p.add_argument("--num_beam_groups", type=int, default=1,
                   help="f1 with --num_beams: diverse beam search with this many groups of beams (1: off); needs "
                        "--diversity_penalty > 0")
    p.add_argument("--diversity_penalty", type=float, default=0.0,
                   help="f1 with --num_beam_groups > 1: score lowered per earlier group's beam with the same token")
    p.add_argument("--repetition_penalty", type=float, default=1.0,
                   help="f1: penalty on ids already in the prompt or reply (1: off); replies go through the batched path")
    p.add_argument("--no_repeat_ngram_size", type=int, default=0,
                   help="f1: never repeat an n-gram of the prompt or reply (0: off); replies go through the batched path")
    p.add_argument("--frequency_penalty", type=float, default=0.0,
                   help="f1: subtract this times the count of each id already in the reply (the prompt does not "
                        "count; 0: off); replies go through the batched path")
    p.add_argument("--presence_penalty", type=float, default=0.0,
                   help="f1: subtract this once from each id already in the reply (the prompt does not count; 0: off); "
                        "replies go through the batched path")
    p.add_argument("--context_no_repeat_ngram_size", type=int, default=0,
                   help="f1: never complete an n-gram of the persona and history (0: off); replies go through the "
                        "batched path")
    p.add_argument("--penalty_alpha", type=float, default=0.0,
                   help="f1: > 0 decodes the replies with GPT2DoubleHeads.contrastive_search, this degeneration penalty "
                        "and --top_k candidates (0: sample); replies go through the batched path")
    p.add_argument("--prompt_lookup_num_tokens", type=int, default=0,
                   help="f1 with --no_sample: verify up to this many draft tokens per step, copied from the prompt and "
                        "the reply (prompt lookup decoding; 0: off); the replies are the greedy ones")
    p.add_argument("--min_p", type=float, default=0.0,
                   help="f1: keep ids with at least this fraction of the top id's probability (0: off); replies go "
                        "through the batched path")
    p.add_argument("--typical_p", type=float, default=1.0,
                   help="f1: locally typical sampling, keep this much mass of the ids closest to the entropy (1: off); "
                        "replies go through the batched path")
    p.add_argument("--epsilon_cutoff", type=float, default=0.0,
                   help="f1: keep ids with probability at least this (0: off); replies go through the batched path")
    p.add_argument("--eta_cutoff", type=float, default=0.0,
                   help="f1: eta sampling, keep ids with probability at least min(eta, sqrt(eta) exp(-entropy)) "
                        "(0: off); replies go through the batched path")
    p.add_argument("--top_h", type=float, default=0.0,
                   help="f1: top-h, keep the most probable ids whose partial entropy stays within this fraction of the "
                        "entropy of the 100 most probable (0: off); replies go through the batched path")
    p.add_argument("--assistant_checkpoint", default="",
                   help="f1: a smaller model with the same vocabulary (a --checkpoint file) drafts tokens that the model "
                        "verifies (assisted generation); the replies are those drawn without it, through the batched path")
    p.add_argument("--num_assistant_tokens", type=int, default=4,
                   help="f1 with --assistant_checkpoint: draft tokens per verify step")
    p.add_argument("--assistant_verification", choices=("coupled", "rejection"), default="coupled",
                   help="f1 with --assistant_checkpoint: coupled draws (the replies drawn without the draft) or "
                        "rejection sampling (replies from the same distribution, more drafts accepted)")
    p.add_argument("--guidance_scale", type=float, default=1.0,
                   help="f1: classifier-free guidance scale (1: off); replies go through the batched path")
    p.add_argument("--guidance_negative", choices=("last_token", "no_persona"), default="last_token",
                   help="f1 with --guidance_scale: the negative prompt, the prompt's last token or the dialogue "
                        "without the persona")
    p.add_argument("--bad_words", default="",
                   help="f1: comma-separated words the replies may never contain, each banned as encoded with and "
                        "without a leading space; replies go through the batched path")
    p.add_argument("--watermark_bias", type=float, default=None,
                   help="f1: mark the replies with the green-list watermark, adding this to every green id's logit "
                        "(default: off); the result adds the replies' mean z-score and detected fraction")
    p.add_argument("--watermark_ratio", type=float, default=0.25, help="f1: the watermark's green-list ratio")
    p.add_argument("--watermark_scheme", choices=("lefthash", "selfhash"), default="lefthash",
                   help="f1: the watermark's seeding scheme")
    p.add_argument("--watermark_context_width", type=int, default=1,
                   help="f1: the ids before a token that seed its green list")
    p.add_argument("--kv_cache_dtype", choices=("fp8_e4m3",), default=None,
                   help="f1: keep the KV cache in fp8 (e4m3 bytes with a power-of-two scale per vector; default: the "
                        "model's dtype); replies go through the batched path")
    p.add_argument("--dola_layers", default=None,
                   help="f1: DoLa layer-contrast decoding against the candidate layers 'low', 'high' or a "
                        "comma-separated list of layer indices (default: off); replies go through the batched path")
    a = p.parse_args()
    model, tok = load_model_from_checkpoint(a.model_checkpoint, a.device,
                                            torch.bfloat16 if a.device.startswith("cuda") else None)
    if a.dataset_path:
        raw = json.load(open(a.dataset_path, encoding="utf-8"))
    else:
        raw = synthetic_personachat(n_train=a.synthetic_dialogs, n_valid=max(8, a.synthetic_dialogs // 8), n_candidates=4, seed=a.seed)
    kw = {}
    if a.eval_type == "f1":
        kw = dict(max_length=a.max_length, min_length=a.min_length, temperature=a.temperature, top_k=a.top_k, top_p=a.top_p,
                  no_sample=a.no_sample, repetition_penalty=a.repetition_penalty,
                  no_repeat_ngram_size=a.no_repeat_ngram_size, penalty_alpha=a.penalty_alpha,
                  prompt_lookup_num_tokens=a.prompt_lookup_num_tokens, min_p=a.min_p, typical_p=a.typical_p,
                  epsilon_cutoff=a.epsilon_cutoff, eta_cutoff=a.eta_cutoff, top_h=a.top_h, beam_sample=a.beam_sample,
                  num_beam_groups=a.num_beam_groups, diversity_penalty=a.diversity_penalty,
                  guidance_scale=a.guidance_scale, guidance_negative=a.guidance_negative,
                  kv_cache_dtype=a.kv_cache_dtype, frequency_penalty=a.frequency_penalty,
                  presence_penalty=a.presence_penalty, context_no_repeat_ngram_size=a.context_no_repeat_ngram_size)
        if a.dola_layers is not None:
            kw["dola_layers"] = (a.dola_layers if a.dola_layers in ("low", "high")
                                 else [int(x) for x in a.dola_layers.split(",") if x.strip()])
        if a.bad_words:
            kw["bad_words_ids"] = bad_word_ids(tok, a.bad_words.split(","))
        if a.watermark_bias is not None:
            kw["watermarking_config"] = dict(bias=a.watermark_bias, greenlist_ratio=a.watermark_ratio,
                                             seeding_scheme=a.watermark_scheme,
                                             context_width=a.watermark_context_width)
        if a.assistant_checkpoint:
            kw["assistant_model"] = load_model_from_checkpoint(
                a.assistant_checkpoint, a.device, torch.bfloat16 if a.device.startswith("cuda") else None)[0]
            kw["num_assistant_tokens"] = a.num_assistant_tokens
            kw["assistant_verification"] = a.assistant_verification
    res = evaluate_dialogs(model, tok, raw["valid"], a.eval_type, a.max_history, a.max_examples, a.device, a.seed,
                           a.batch_size, a.num_beams, **kw)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
