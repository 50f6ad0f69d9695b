"""KV-cached GPT-2 decoding on the GPU: the decode-attention kernel against fp64 at the split boundaries, its
repeatability and batch / graph invariance, and the cached model against the uncached one on GPT-2 small."""
import copy
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24          # unit roundoff of fp32
U16 = 2.0 ** -8           # unit roundoff of bf16
NAN_BITS = 0x7FC1         # a bf16 NaN: a sentinel the kernel must neither read nor overwrite
# the split boundaries of every split length the kernel may be built with (64, 128 or 256 keys)
LENS = [0, 1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1022, 1023]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)           # the in-tree .so must be the code under test
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _inputs(dev, lens, H, Dh, t_max, seed=0, q_scale=2.0):
    """qkv [B, 3HDh]; caches with random keys / values below lens[b] and NaN sentinels from lens[b] on."""
    g = torch.Generator(device=dev).manual_seed(seed)
    B = len(lens)
    qkv = torch.randn(B, 3 * H * Dh, device=dev, generator=g)
    qkv[:, :H * Dh] *= q_scale                                      # peaked as well as flat softmax rows
    qkv = qkv.to(torch.bfloat16)
    kc = torch.randn(B, H, t_max, Dh, device=dev, generator=g).to(torch.bfloat16)
    vc = torch.randn(B, H, t_max, Dh, device=dev, generator=g).to(torch.bfloat16)
    pos = torch.arange(t_max, device=dev)
    lens_t = torch.tensor(lens, dtype=torch.int32, device=dev)
    beyond = (pos[None, :] >= lens_t[:, None].long())[:, None, :, None].expand_as(kc)
    for c in (kc, vc):
        c.view(torch.int16)[beyond] = NAN_BITS
    return qkv, kc, vc, lens_t


def _run(qkv, kc, vc, lens):
    from adapcc_b200.ops import decode_attention_, decode_attention_work_numel

    B, H, t_max, Dh = kc.shape
    out = torch.full((B, H * Dh), float("nan"), dtype=torch.bfloat16, device=kc.device)
    work = torch.empty(decode_attention_work_numel(B, H, Dh, t_max), dtype=torch.float32, device=kc.device)
    return decode_attention_(qkv, kc, vc, lens, out, work)


def _check_against_fp64(out, qkv, kc0, lens, H, Dh, vc0):
    """Per element: the fp64 result from the same bf16 inputs, against a bound from the kernel's arithmetic.

    * Scores: a bf16 x bf16 product is exact in fp32; Dh fused multiply-adds and the scale 1/sqrt(Dh) (rounded) are
      off by at most (Dh + 2) u32 * scale * sum |q k|; subtracting the running max adds u32 * |s - m| <= 2 u32 max |s|.
      So every score is off by at most e, and normalised softmax weights by a factor in [e^-2e, e^2e].
    * Weights and sums: expf is within 2 ulp (4 u32 relative); the sum of the weights and P.V accumulate n = lens + 1
      terms in fp32 (n u32 relative each, on sums of non-negative weights times |v|); the split combination rescales
      with one more expf and fma per split and divides once. (2n + 32) u32 bounds all of it relative to
      sum p|v| / sum p.
    * Then one bf16 rounding of the output (U16 relative)."""
    D = H * Dh
    B = out.shape[0]
    for b in range(B):
        L = int(lens[b])
        o = out[b].double().view(H, Dh)
        if L >= kc0.shape[2]:
            assert torch.equal(out[b].float(), torch.zeros_like(out[b].float())), b
            continue
        q = qkv[b, :D].double().view(H, Dh)
        K = torch.cat([kc0[b, :, :L].double(), qkv[b, D:2 * D].double().view(H, 1, Dh)], 1)      # [H, L + 1, Dh]
        V = torch.cat([vc0[b, :, :L].double(), qkv[b, 2 * D:].double().view(H, 1, Dh)], 1)
        scale = 1.0 / math.sqrt(Dh)
        s = torch.einsum("hd,htd->ht", q, K) * scale
        p = torch.softmax(s, -1)
        ref = torch.einsum("ht,htd->hd", p, V)
        e = (Dh + 2) * U32 * scale * torch.einsum("hd,htd->ht", q.abs(), K.abs()).amax(-1) + 4 * U32 * s.abs().amax(-1)
        mag = torch.einsum("ht,htd->hd", p, V.abs())
        n = L + 1
        err = (torch.expm1(2 * e)[:, None] + (2 * n + 32) * U32) * mag
        bound = err + U16 * (ref.abs() + err)
        bad = ~((o - ref).abs() <= bound)
        assert not bool(bad.any()), (b, L, float((o - ref).abs().max()), float(bound.min()))


@pytest.mark.parametrize("H,Dh", [(12, 64), (4, 16), (4, 128)])
def test_decode_attention_against_fp64_and_cache_bits(dev, H, Dh):
    t_max = 1024
    lens = LENS + [t_max]                                           # the last row is out of range: left alone
    qkv, kc, vc, lens_t = _inputs(dev, lens, H, Dh, t_max)
    kc0, vc0 = kc.clone(), vc.clone()
    out = _run(qkv, kc, vc, lens_t)
    torch.cuda.synchronize()
    _check_against_fp64(out, qkv, kc0, lens_t.cpu(), H, Dh, vc0)
    D = H * Dh
    for b, L in enumerate(lens):
        if L < t_max:
            # the new k / v sit at position L bit for bit; every other slot keeps its bits
            assert torch.equal(kc[b, :, L].view(torch.int16), qkv[b, D:2 * D].view(H, Dh).view(torch.int16)), b
            assert torch.equal(vc[b, :, L].view(torch.int16), qkv[b, 2 * D:].view(H, Dh).view(torch.int16)), b
            keep = torch.ones(t_max, dtype=torch.bool, device=dev)
            keep[L] = False
        else:
            keep = torch.ones(t_max, dtype=torch.bool, device=dev)
        assert torch.equal(kc[b][:, keep].view(torch.int16), kc0[b][:, keep].view(torch.int16)), b
        assert torch.equal(vc[b][:, keep].view(torch.int16), vc0[b][:, keep].view(torch.int16)), b


def test_decode_attention_is_repeatable_and_batch_invariant(dev):
    H, Dh, t_max = 12, 64, 1024
    qkv, kc, vc, lens = _inputs(dev, LENS, H, Dh, t_max, seed=3)
    a = _run(qkv, kc.clone(), vc.clone(), lens)
    b = _run(qkv, kc.clone(), vc.clone(), lens)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    for r in (0, 3, 7, len(LENS) - 1):
        alone = _run(qkv[r:r + 1].clone(), kc[r:r + 1].clone(), vc[r:r + 1].clone(), lens[r:r + 1].clone())
        assert torch.equal(alone[0].view(torch.int16), a[r].view(torch.int16)), r


def _gpt2_small(dev, seed=0):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(seed)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


def test_graph_replay_equals_eager_steps(dev):
    from adapcc_b200.models.gpt2 import DecodeGraph

    m = _gpt2_small(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    B, T, steps = 3, 100, 32
    ids = torch.randint(0, m.cfg.vocab_size, (B, T), device=dev, generator=g)
    toks = torch.randint(0, m.cfg.vocab_size, (steps, B), device=dev, generator=g)
    tts = torch.randint(m.cfg.vocab_size - 5, m.cfg.vocab_size - 3, (steps, B), device=dev, generator=g)
    lengths = [100, 37, 64]
    eager, graph = m.new_cache(B), m.new_cache(B)
    with torch.no_grad():
        m.hidden(ids, None, cache=eager, lengths=lengths)
        m.hidden(ids, None, cache=graph, lengths=lengths)
    step = DecodeGraph(m, graph, token_types=True)
    for i in range(steps):
        he = m.decode_step(toks[i], tts[i], eager)
        hg = step(toks[i], tts[i])
        assert torch.equal(he.view(torch.int16), hg.view(torch.int16)), i
    torch.cuda.synchronize()
    assert torch.equal(eager.k.view(torch.int16), graph.k.view(torch.int16))
    assert torch.equal(eager.v.view(torch.int16), graph.v.view(torch.int16))
    want = [n + steps for n in lengths]
    assert graph.lens.tolist() == want and graph.host_lens == want and eager.lens.tolist() == want


def test_cached_gpt2_small_is_as_accurate_as_uncached(dev):
    """300-token prompt, 64 teacher-forced steps: the cached bf16 hidden states are no further from an fp32 run of the
    same weights than twice the uncached bf16 path's distance."""
    m = _gpt2_small(dev)
    ref = copy.deepcopy(m).float()
    g = torch.Generator(device=dev).manual_seed(2)
    seq = torch.randint(0, m.cfg.vocab_size, (1, 300 + 64), device=dev, generator=g)
    cache = m.new_cache(1)
    err_cached = err_uncached = 0.0
    with torch.no_grad():
        m.hidden(seq[:, :300], None, cache=cache)
        for i in range(64):
            t = 300 + i
            hc = m.decode_step(seq[:, t], None, cache)[0].double()
            hu = m.hidden(seq[:, :t + 1], None)[0, -1].double()
            hr = ref.hidden(seq[:, :t + 1], None)[0, -1].double()
            err_cached = max(err_cached, float((hc - hr).abs().max()))
            err_uncached = max(err_uncached, float((hu - hr).abs().max()))
    assert err_cached <= 2 * err_uncached, (err_cached, err_uncached)


def test_greedy_generation_repeats_and_follows_the_uncached_path(dev):
    from adapcc_b200.models.gpt2 import sample_sequence

    m = _gpt2_small(dev)
    g = torch.Generator(device=dev).manual_seed(4)
    prompt = torch.randint(0, m.cfg.vocab_size, (1, 200), device=dev, generator=g)
    a = sample_sequence(m, prompt, None, max_new_tokens=32, top_k=1, top_p=1.0)
    b = sample_sequence(m, prompt, None, max_new_tokens=32, top_k=1, top_p=1.0)
    assert torch.equal(a, b)
    ids = prompt
    head = m.wte.weight.float()
    with torch.no_grad():
        for i in range(32):
            logits = (m.hidden(ids, None)[:, -1].float() @ head.t())[0, :m.cfg.vocab_size]
            top2 = torch.topk(logits, 2).values
            nxt = int(logits.argmax())
            if float(top2[0] - top2[1]) < 0.1:       # a near tie: bf16 rounding may pick either token from here on
                break
            assert int(a[0, i]) == nxt, i
            ids = torch.cat([ids, a[:, i:i + 1]], 1)
