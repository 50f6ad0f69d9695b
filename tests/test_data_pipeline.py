"""The conversational GPT-2 workload's data path on CPU: tokenizer, PersonaChat-format inputs, loaders, prefetcher,
ConvAI metrics, and the end-to-end example (train → checkpoint → evaluate → interact)."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _free_ports(n):
    import socket

    socks = [socket.socket() for _ in range(n)]
    for s in socks:
        s.bind(("127.0.0.1", 0))
    ports = [s.getsockname()[1] for s in socks]
    for s in socks:
        s.close()
    return ports

from adapcc_b200.data import (DialogTokenizer, PinnedPrefetcher, build_input_from_segments, build_tensors,  # noqa: E402
                              corpus_of, get_data_loaders, get_dataset, synthetic_personachat)
from adapcc_b200.eval import f1_score, normalize_answer, top_filtering  # noqa: E402


@pytest.fixture(scope="module")
def corpus():
    return synthetic_personachat(24, 6, 4, seed=3)


@pytest.fixture(scope="module")
def tok(corpus):
    return DialogTokenizer.train(corpus_of(corpus), vocab_size=500, model_vocab=512)


def test_tokenizer_roundtrip_specials_and_persistence(tok, tmp_path):
    for s in ("hi , how are you today ?", "i could eat sushi every day .", "héllo wörld — 123 !!", "  two  spaces\tand\nnewline"):
        assert tok.decode(tok.encode(s)) == s
    assert tok.base_vocab <= 500 and len(tok.merges) == tok.base_vocab - 256
    assert tok.special_ids == (507, 508, 509, 510, 511) and tok.pad_id == 511        # the model's top five ids
    assert tok.convert_tokens_to_ids(["<bos>", "<pad>"]) == [507, 511]
    merged = tok.encode(" hiking")
    assert len(merged) < len(" hiking".encode())                                     # merges were learned
    p = tmp_path / "tok.json"
    tok.save(str(p))
    again = DialogTokenizer.load(str(p))
    assert again.encode("what do you do for fun ?") == tok.encode("what do you do for fun ?") and again.special_ids == tok.special_ids
    # deterministic training
    t2 = DialogTokenizer.train(corpus_of(synthetic_personachat(24, 6, 4, seed=3)), vocab_size=500, model_vocab=512)
    assert t2.merges == tok.merges
    with pytest.raises(ValueError):
        DialogTokenizer(tok.symbols, tok.merges, model_vocab=tok.base_vocab + 2)


def test_gpt2_vocab_files_are_accepted(tok, tmp_path):
    d = tmp_path / "gpt2"
    d.mkdir()
    (d / "vocab.json").write_text(json.dumps({s: i for i, s in enumerate(tok.symbols)}), encoding="utf-8")
    (d / "merges.txt").write_text("#version: 0.2\n" + "\n".join(f"{a} {b}" for a, b in tok.merges) + "\n", encoding="utf-8")
    t = DialogTokenizer.from_gpt2_files(str(d), 600)
    assert t.encode("i have a parrot .") == tok.encode("i have a parrot .") and t.special_ids[0] == 595


def test_segment_layout_matches_the_reference_semantics(tok):
    bos, eos, s1, s2, pad = tok.special_ids
    persona, history, reply = [[1, 2], [3]], [[4], [5, 6]], [7, 8]
    inst = build_input_from_segments(persona, history, reply, tok, lm_labels=True)
    # <bos> persona | <speaker?> h0 | <speaker?> h1 | <speaker?> reply <eos>   with 4 segments: tags s1? (4-0)%2=0 -> s1,
    # (4-1)%2=1 -> s2, (4-2)%2=0 -> s1
    assert inst.input_ids == [bos, 1, 2, 3, s1, 4, s2, 5, 6, s1, 7, 8, eos]
    assert inst.token_type_ids == [s1] * 4 + [s2] * 2 + [s1] * 3 + [s2] * 4             # per segment: s1, s2, s1, s2
    assert inst.lm_labels == [-100] * 10 + [7, 8, eos]                                 # only the reply, not its speaker token
    assert inst.mc_token_id == 12
    plain = build_input_from_segments(persona, history, reply, tok, lm_labels=False, with_eos=False)
    assert plain.input_ids[-1] == 8 and set(plain.lm_labels) == {-100}
    # over-long inputs lose their OLDEST history first; the persona and the reply survive
    short = build_input_from_segments(persona, history, reply, tok, lm_labels=True, max_len=11)
    assert short.input_ids == [bos, 1, 2, 3, s2, 5, 6, s1, 7, 8, eos] and len(short.input_ids) <= 11
    tail = build_input_from_segments(persona, [], list(range(20, 40)), tok, lm_labels=True, max_len=8)
    assert len(tail.input_ids) == 8 and tail.input_ids[-1] == eos and tail.mc_token_id == 7


def test_tensors_and_loaders(tok, corpus, tmp_path):
    from types import SimpleNamespace

    data = get_dataset(tok, synthetic=dict(n_train=24, n_valid=6, n_candidates=4, seed=3))
    t = build_tensors(data["train"], tok, num_candidates=2, max_history=2, personality_permutations=2)
    n_utt = sum(len(d["utterances"]) for d in data["train"])
    N, C, T = t["input_ids"].shape
    assert (N, C) == (2 * n_utt, 2) and T % 64 == 0
    assert t["mc_labels"].tolist() == [1] * N and t["mc_token_ids"].shape == (N, 2)
    assert (t["lm_labels"][:, 0] == -100).all() and (t["lm_labels"][:, 1] != -100).any(dim=-1).all()   # gold = last candidate
    eos = tok.special_ids[1]
    last = t["input_ids"].gather(2, t["mc_token_ids"].unsqueeze(-1)).squeeze(-1)
    assert (last == eos).all()                                                         # the MC head reads the <eos> position
    assert (t["input_ids"][t["lm_labels"] != -100] == t["lm_labels"][t["lm_labels"] != -100]).all()
    # validation keeps every candidate; fixed seq_len is honoured
    v = build_tensors(data["valid"], tok, num_candidates=2, seq_len=128, limit_candidates=False)
    assert v["input_ids"].shape[1:] == (4, 128)
    # cache round trip through a JSON file in the PersonaChat schema
    path = tmp_path / "pc.json"
    path.write_text(json.dumps(corpus), encoding="utf-8")
    a = SimpleNamespace(dataset_path=str(path), dataset_cache=str(tmp_path / "cache"), num_candidates=2, train_batch_size=4)
    tl, vl, ts, vs = get_data_loaders(a, tok)
    assert any(f.startswith("cache_") for f in os.listdir(tmp_path))
    tl2, *_ = get_data_loaders(a, tok)                                                 # second call reads the cache
    b = next(iter(vl))
    assert set(b) == {"input_ids", "mc_token_ids", "lm_labels", "mc_labels", "token_type_ids"} and b["input_ids"].dim() == 3
    assert len(tl) == len(tl2)
    # distributed samplers partition the training set
    _, _, s0, _ = get_data_loaders(a, tok, distributed=True, rank=0, world_size=2)
    _, _, s1, _ = get_data_loaders(a, tok, distributed=True, rank=1, world_size=2)
    assert not set(iter(s0)) & set(iter(s1))
    # the prefetcher hands out exactly the loader's batches, in order
    ref = [b for b in vl]
    got = [{k: v.clone() for k, v in b.items()} for b in PinnedPrefetcher(vl, "cpu")]
    assert len(ref) == len(got) and all(torch.equal(r[k], g[k]) for r, g in zip(ref, got) for k in r)
    static = {k: torch.zeros_like(v) for k, v in ref[0].items()}
    for r, g in zip(ref[:-1], PinnedPrefetcher(vl, "cpu", static_out=static)):        # last batch may be ragged
        assert g is static and torch.equal(static["input_ids"], r["input_ids"])
        if r["input_ids"].shape != ref[-1]["input_ids"].shape:
            break


def test_metrics_helpers():
    assert normalize_answer("The cat, a dog & an owl!") == ["cat", "dog", "owl"]
    assert f1_score("i love hiking", ["I love hiking."]) == 1.0
    assert f1_score("completely different", ["i love hiking"]) == 0.0
    assert abs(f1_score("i love pizza", ["i love hiking a lot"]) - 2 * (2 / 3) * (2 / 4) / (2 / 3 + 2 / 4)) < 1e-9
    logits = torch.tensor([2.0, 1.0, 0.5, -1.0, -3.0])
    k2 = top_filtering(logits, top_k=2, top_p=0.0)
    assert torch.isfinite(k2).tolist() == [True, True, False, False, False]
    p = top_filtering(logits, top_k=0, top_p=0.6)            # probs ~ .60 .22 .13 .03 .004: keep until the mass crosses 0.6
    assert torch.isfinite(p).tolist() == [True, True, False, False, False] or torch.isfinite(p).tolist() == [True, False, False, False, False]
    assert torch.isfinite(top_filtering(logits, 0, 0.0, threshold=0.75)).tolist() == [True, True, False, False, False]
    assert torch.equal(logits, torch.tensor([2.0, 1.0, 0.5, -1.0, -3.0]))           # input untouched


def test_top_filtering_keeps_every_token_at_top_p_1():
    # the fp32 cumulative softmax of a GPT-2-sized row passes 1.0 by rounding before its last entry: top_p = 1 must
    # not turn that into dropped tokens
    logits = torch.randn(50257, generator=torch.Generator().manual_seed(0)) * 3
    assert torch.isfinite(top_filtering(logits, top_k=0, top_p=1.0)).all()
    assert int(torch.isfinite(top_filtering(logits, top_k=40, top_p=1.0)).sum()) == 40


def test_train_evaluate_interact_end_to_end(tmp_path):
    """examples/train_gpt2_personachat.py on 2 gloo ranks (tokenizer built by rank 0, distributed loaders, DDP + the
    communicator's hook, linear lr decay, validation all-reduced, checkpoint), then the evaluation and chat scripts."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="2")
    mport, cport, sport = _free_ports(3)
    env["ADAPCC_COORD_PORT"] = str(cport)
    train = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
             "--master-port", str(mport), os.path.join(ROOT, "examples", "train_gpt2_personachat.py"), "--backend", "gloo", "--tiny",
             "--n_epochs", "2", "--synthetic_dialogs", "24", "--lr", "3e-3", "--eval_before_start", "--checkpoint", "ck.pt",
             "--port", str(sport)]
    r = subprocess.run(train, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    vals = [float(line.split("nll ")[1].split()[0]) for line in r.stdout.splitlines() if line.startswith("validation")]
    assert len(vals) == 3 and vals[-1] < vals[0] - 1.0, r.stdout[-1500:]           # before, epoch 0, epoch 1
    assert (tmp_path / "ck.pt").exists() and (tmp_path / "dialog_tokenizer.json").exists()
    for kind in ("hits@1", "ppl", "f1"):
        e = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "eval_gpt2_convai.py"), "--model_checkpoint", "ck.pt",
                            "--eval_type", kind, "--synthetic_dialogs", "24", "--max_examples", "6", "--device", "cpu"],
                           cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
        assert e.returncode == 0, e.stderr[-2000:]
        rec = json.loads(e.stdout.strip().splitlines()[-1])
        assert rec["examples"] == 6 and kind in rec and rec[kind] >= 0
    c = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "interact_gpt2.py"), "--model_checkpoint", "ck.pt",
                        "--device", "cpu", "--script", "hi there|do you have any pets ?"], cwd=tmp_path, env=env,
                       capture_output=True, text=True, timeout=600)
    assert c.returncode == 0 and c.stdout.startswith("Selected personality:") and len(c.stdout.splitlines()) == 3, c.stderr[-2000:]
    # resume: a second run starts after the last finished epoch and has nothing left to do
    r2 = subprocess.run(train, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    assert r2.returncode == 0 and "epoch 0 step" not in r2.stdout, r2.stdout[-1500:] + r2.stderr[-2000:]


def test_accuracy_benchmark_and_log_processors(tmp_path):
    """examples/accuracy_benchmark.py on 2 gloo ranks with learnable dummy data: training Acc@1 rises, validation is
    all-reduced over an exact partition, the GNS probe prints, checkpoints resume; tools/process_log.py extracts the
    Acc@1 / gns series the reference keeps as accuracy_*.txt / gns-split-all.txt."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="2")
    mport, cport, sport = _free_ports(3)
    env["ADAPCC_COORD_PORT"] = str(cport)
    base = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
            "--master-port", str(mport), os.path.join(ROOT, "examples", "accuracy_benchmark.py"), "--dummy", "--backend", "gloo",
            "-a", "resnet18", "--image_size", "32", "--classes", "10", "--dummy_size", "768", "-b", "16", "--lr", "0.05",
            "--gns_freq", "8", "-p", "4", "--port", str(sport), "--seed", "0"]
    r = subprocess.run(base + ["--epochs", "1"], cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    (tmp_path / "run.out").write_text(r.stdout)
    summary = [line for line in r.stdout.splitlines() if line.startswith(" *")]
    assert len(summary) == 1 and "(96 samples)" in summary[0]                       # 768 // 8 validation samples, each once
    val_acc1 = float(summary[0].split("Acc@1")[1].split()[0])
    assert val_acc1 > 30.0, summary                                                 # chance = 10 %
    assert (tmp_path / "checkpoint.pth.tar").exists() and (tmp_path / "model_best.pth.tar").exists()
    for metric, n_min in (("acc1", 5), ("gns", 3)):
        e = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "process_log.py"), "--metric", metric, "run.out", metric + ".txt"],
                           cwd=tmp_path, capture_output=True, text=True, timeout=60)
        assert e.returncode == 0, e.stderr
        vals = [float(x) for x in (tmp_path / (metric + ".txt")).read_text().split()]
        assert len(vals) >= n_min
        if metric == "acc1":
            assert max(vals[-3:]) > vals[0] and all(0.0 <= v <= 100.0 for v in vals)
    # resume into a second epoch, bf16 whole-model precision, early stop
    r2 = subprocess.run(base + ["--epochs", "2", "--resume", "checkpoint.pth.tar", "--stop", "3"], cwd=tmp_path, env=env,
                        capture_output=True, text=True, timeout=900)
    assert r2.returncode == 0 and "=> loaded checkpoint 'checkpoint.pth.tar' (epoch 1)" in r2.stdout, r2.stdout[-800:] + r2.stderr[-2000:]
    assert "Epoch: [1]" in r2.stdout and "Epoch: [0]" not in r2.stdout
    ev = subprocess.run(base + ["--evaluate", "--resume", "checkpoint.pth.tar", "--bfp16"], cwd=tmp_path, env=env,
                        capture_output=True, text=True, timeout=900)
    assert ev.returncode == 0 and " *   Acc@1" in ev.stdout and "Epoch:" not in ev.stdout, ev.stderr[-2000:]


def test_tokenizer_and_layout_properties(tok):
    """Property tests: any text survives encode → decode; any (persona, history, reply) yields a well-formed input."""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=150, deadline=None)
    @given(st.text(max_size=60))
    def roundtrip(text):
        ids = tok.encode(text)
        assert all(0 <= i < tok.base_vocab for i in ids)
        assert tok.decode(ids) == text.encode("utf-8", errors="replace").decode("utf-8", errors="replace")

    roundtrip()
    seg = st.lists(st.integers(0, tok.base_vocab - 1), min_size=1, max_size=12)

    @settings(max_examples=150, deadline=None)
    @given(st.lists(seg, min_size=1, max_size=4), st.lists(seg, min_size=0, max_size=5), seg, st.booleans(), st.booleans(),
           st.one_of(st.none(), st.integers(8, 64)))
    def layout(persona, history, reply, lm, eos, max_len):
        bos, eos_id, s1, s2, _ = tok.special_ids
        inst = build_input_from_segments(persona, history, reply, tok, lm_labels=lm, with_eos=eos, max_len=max_len)
        n = len(inst.input_ids)
        assert n == len(inst.token_type_ids) == len(inst.lm_labels) and inst.mc_token_id == n - 1
        if max_len is not None:
            assert n <= max_len
        assert set(inst.token_type_ids) <= {s1, s2}
        tail = list(reply) + ([eos_id] if eos else [])
        assert inst.input_ids[-min(n, len(tail)):] == tail[-min(n, len(tail)):]           # the reply always survives, at the end
        scored = [x for x in inst.lm_labels if x != -100]
        if lm:
            assert scored == tail[-len(scored):] and len(scored) <= len(tail)            # labels = (a suffix of) the reply only
        else:
            assert not scored
        if max_len is None:
            assert inst.input_ids[0] == bos and inst.input_ids.count(bos) == 1

    layout()


def test_prefetcher_handles_ragged_batches_and_any_depth():
    """The prefetcher returns exactly the loader's batches for any length / batch size / ring depth, including a shorter
    last batch (its slot is re-shaped) and an empty loader."""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=40, deadline=None)
    @given(st.integers(0, 23), st.integers(1, 7), st.integers(2, 4))
    def prop(n, bs, depth):
        data = [{"a": torch.arange(i * 3, (i + 1) * 3), "b": torch.tensor([float(i)])} for i in range(n)]
        coll = lambda items: {k: torch.stack([x[k] for x in items]) for k in ("a", "b")}          # noqa: E731
        loader = torch.utils.data.DataLoader(data, batch_size=bs, collate_fn=coll)
        ref = [b for b in loader]
        got = [{k: v.clone() for k, v in b.items()} for b in PinnedPrefetcher(loader, "cpu", depth=depth)]
        assert len(ref) == len(got) and all(torch.equal(r[k], g[k]) for r, g in zip(ref, got) for k in r)

    prop()
