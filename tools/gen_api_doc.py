#!/usr/bin/env python
"""Writes docs/API.md: the public Python surface (signatures + first docstring paragraph) and the C ABI of
libadapcc.so (exported ``adapcc_*`` functions and the reference's six symbols), straight from the sources."""
import importlib
import inspect
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODULES = [
    ("adapcc_b200.adapcc", ["AdapCC"]),
    ("adapcc_b200.commu", ["CudaCommu"]),
    ("adapcc_b200.runtime.native", ["NativeComm", "load_library", "native_relay_control", "native_tree_role"]),
    ("adapcc_b200.parallel.engine", ["FlatDataParallel", "shard_of"]),
    ("adapcc_b200.parallel.ddp", None),
    ("adapcc_b200.parallel.expert_parallel", ["ExpertExchange"]),
    ("adapcc_b200.ops", None),
    ("adapcc_b200.ops.sampling", ["top_filtering", "philox4x32_10", "uniform", "keep", "reference_row",
                                  "sample_reference", "check_filter_args"]),
    ("adapcc_b200.ops.dropout", ["DropoutState", "dropout", "dropout_mask", "dropout_reference", "threshold"]),
    ("adapcc_b200.ops.beam", ["BeamReference", "BeamSampleReference", "GroupBeamReference", "best_hypotheses",
                              "merge_finished_sets", "offer_finished", "sample_keep", "philox_words", "gumbel",
                              "StochasticBeamReference", "stochastic_results", "sbs_estimate", "truncated_gumbel",
                              "start_keys"]),
    ("adapcc_b200.ops.contrastive", ["candidates_row", "max_cosine", "rerank_row", "select_candidates",
                                     "check_contrastive_args"]),
    ("adapcc_b200.ops.lookup", ["draft_row", "greedy_token", "accept_row", "lookup_draft", "lookup_accept",
                                "check_lookup_args", "mean_tokens_per_step"]),
    ("adapcc_b200.ops.assisted", ["check_assist_args", "draw_slot", "assist_round", "draw_slots", "check_verification",
                                  "filtered_probs", "spec_slot", "spec_slots"]),
    ("adapcc_b200.ops.repeats", ["penalize_repeats_reference", "banned_ngram_ids", "check_repeat_args",
                                 "finite_fp32", "check_sequence_bias_args", "SequenceBias"]),
    ("adapcc_b200.ops.guidance", ["check_guidance_args", "guided_scores_reference"]),
    ("adapcc_b200.ops.dola", ["dola_candidate_layers", "check_dola_args", "dola_scores_reference",
                              "dola_js_reference"]),
    ("adapcc_b200.ops.watermark", ["WatermarkingConfig", "check_watermark_args", "watermark_reference",
                                   "watermark_counts_reference", "detect_watermark", "WatermarkDetectorOutput"]),
    ("adapcc_b200.ops.synthid", ["SynthIDTextWatermarkingConfig", "check_synthid_args", "is_synthid_config",
                                 "synthid_flags", "synthid_counts_reference", "synthid_mask_reference",
                                 "synthid_g_values", "detect_synthid", "SynthIDDetectorOutput"]),
    ("adapcc_b200.ops.kvcache", ["quantize", "dequantize", "store_", "check_kv_cache_dtype"]),
    ("adapcc_b200.ops.layers", ["FusedLayerNorm", "FusedLinear", "linear_backward"]),
    ("adapcc_b200.ops.gemm", ["linear_act", "linear_gelu", "supported", "default_variant"]),
    ("adapcc_b200.strategy.trees", ["Tree", "Strategy"]),
    ("adapcc_b200.strategy.relay", None),
    ("adapcc_b200.synth.synthesizer", ["Synthesizer"]),
    ("adapcc_b200.synth.partrees", ["ParTrees"]),
    ("adapcc_b200.synth.solver", ["Solver"]),
    ("adapcc_b200.synth.multiround", None),
    ("adapcc_b200.synth.cost_model", None),
    ("adapcc_b200.coord.server", None),
    ("adapcc_b200.coord.client", None),
    ("adapcc_b200.topology", None),
    ("adapcc_b200.dispatcher", ["Dispatcher"]),
    ("adapcc_b200.utils.checkpoint", None),
    ("adapcc_b200.utils.fault", None),
    ("adapcc_b200.utils.gns", None),
    ("adapcc_b200.utils.meters", None),
    ("adapcc_b200.models.gpt2", ["GPT2Config", "GPT2DoubleHeads", "KVCache", "DecodeGraph", "CachedDecoder",
                                 "CandidateKV", "VerifyKV", "decode_attention", "sample_sequence", "synthetic_batch", "lm_rows_needed"]),
    ("adapcc_b200.models.vit", ["ViTConfig", "ViT"]),
    ("adapcc_b200.models.moe", None),
    ("adapcc_b200.data.tokenizer", ["DialogTokenizer"]),
    ("adapcc_b200.data.personachat", ["synthetic_personachat", "get_dataset", "build_input_from_segments", "build_tensors",
                                       "get_data_loaders"]),
    ("adapcc_b200.data.prefetch", ["PinnedPrefetcher", "micro_batch_groups"]),
    ("adapcc_b200.eval.convai", ["mc_scores", "sample_reply", "sample_replies", "evaluate_tensors", "f1_score",
                                  "next_word_probability", "evaluate_dialogs", "bad_word_ids"]),
    ("adapcc_b200.eval", ["pack_checkpoint", "load_model_from_checkpoint"]),
    ("adapcc_b200.synth.plan", None),
]


def first_par(doc):
    if not doc:
        return ""
    par = inspect.cleandoc(doc).split("\n\n")[0]
    return " ".join(par.split())


def sig(obj):
    try:
        return str(inspect.signature(obj))
    except (TypeError, ValueError):
        return "(...)"


def describe(name, obj, out, level="###"):
    if inspect.isclass(obj):
        out.append(f"{level} class `{name}{sig(obj)}`")
        d = first_par(obj.__doc__)
        if d:
            out.append(d)
        rows = []
        for mname, m in inspect.getmembers(obj):
            if mname.startswith("_") or not (inspect.isfunction(m) or inspect.ismethod(m) or isinstance(m, property)):
                continue
            if not any(mname in vars(k) for k in obj.__mro__ if k.__module__.startswith("adapcc_b200")):
                continue
            if isinstance(m, property):
                rows.append(f"* `{mname}` (property) — {first_par(m.fget.__doc__)}")
            else:
                rows.append(f"* `{mname}{sig(m)}` — {first_par(m.__doc__)}")
        out.extend(rows)
    else:
        out.append(f"* `{name}{sig(obj)}` — {first_par(obj.__doc__)}")


def main():
    out = ["# API reference (generated by `tools/gen_api_doc.py`; do not edit by hand)", "",
           "Python surface first (module by module), then the C ABI of `adapcc_b200/_C/libadapcc.so`.", ""]
    for modname, names in MODULES:
        try:
            mod = importlib.import_module(modname)
        except Exception as e:                                      # pragma: no cover
            out.append(f"## `{modname}` — import failed here: {e!r}")
            continue
        out.append(f"## `{modname}`")
        d = first_par(mod.__doc__)
        if d:
            out.append(d)
            out.append("")
        if names is None:
            names = [n for n, o in vars(mod).items() if not n.startswith("_") and getattr(o, "__module__", None) == modname
                     and (inspect.isclass(o) or inspect.isfunction(o))]
        for n in names:
            if hasattr(mod, n):
                describe(n, getattr(mod, n), out)
        out.append("")
    out.append("## C ABI (`extern \"C\"`, `adapcc_b200/csrc/*.cu|cpp`)")
    out.append("")
    csrc = os.path.join(ROOT, "adapcc_b200", "csrc")
    pat = re.compile(r"^(?:const char\*|void\*|int|long long|unsigned long long|void)\s+((?:adapcc_\w+|initThreads|exitThreads|"
                     r"allreduce|reduce|boardcast|updateActive))\s*\(([^)]*)\)", re.M | re.S)
    for fn in sorted(os.listdir(csrc)):
        if not fn.endswith((".cu", ".cpp")):
            continue
        src = open(os.path.join(csrc, fn)).read()
        hits = [(m.group(1), " ".join(m.group(2).split())) for m in pat.finditer(src)]
        if not hits:
            continue
        out.append(f"### `{fn}`")
        for name, args in hits:
            out.append(f"* `{name}({args})`")
        out.append("")
    path = os.path.join(ROOT, "docs", "API.md")
    with open(path, "w") as f:
        f.write("\n".join(out) + "\n")
    print(path, len(out), "lines")


if __name__ == "__main__":
    main()
