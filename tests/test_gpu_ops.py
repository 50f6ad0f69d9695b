"""GPU numerics of the hand-written kernels against plain PyTorch fp32 references (single GPU)."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)           # the in-tree .so must be the code under test
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def test_fused_ce_matches_torch(dev):
    from adapcc_b200.ops import fused_ce_

    torch.manual_seed(0)
    rows, vocab, stride = 257, 50262, 50304
    logits = (torch.randn(rows, stride, device=dev) * 3).bfloat16()
    labels = torch.randint(0, vocab, (rows,), device=dev)
    labels[::7] = -100
    ref_in = logits.float()[:, :vocab].clone().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(ref_in, labels, ignore_index=-100, reduction="sum")
    ref.backward()
    work = logits.clone()
    row_loss = fused_ce_(work, labels, vocab)
    assert torch.allclose(row_loss.sum(), ref.detach(), rtol=2e-3)
    assert torch.all(row_loss[::7] == 0)
    got = work.float()
    assert torch.all(got[:, vocab:] == 0)
    assert torch.allclose(got[:, :vocab], ref_in.grad, atol=8e-3, rtol=2e-2)


@pytest.mark.parametrize("pdtype,gdtype", [(torch.bfloat16, torch.bfloat16), (torch.float32, torch.float32)])
def test_fused_adamw_matches_torch(dev, pdtype, gdtype):
    from adapcc_b200.ops import fused_adamw_, incr_, sumsq_

    torch.manual_seed(1)
    n = 100_003
    w0 = torch.randn(n, device=dev)
    ref_p = torch.nn.Parameter(w0.clone())
    opt = torch.optim.AdamW([ref_p], lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    param = w0.to(pdtype).clone()
    master = w0.clone()
    m = torch.zeros(n, device=dev)
    v = torch.zeros(n, device=dev)
    sumsq = torch.zeros(1, device=dev)
    step_t = torch.zeros(1, dtype=torch.int32, device=dev)
    for step in range(1, 6):
        g = torch.randn(n, device=dev) * 5
        gq = g.to(gdtype)
        ref_p.grad = gq.float().clone()
        torch.nn.utils.clip_grad_norm_([ref_p], 1.0)
        opt.step()
        sumsq.zero_()
        sumsq_(gq, sumsq)
        assert torch.allclose(sumsq, gq.float().pow(2).sum(), rtol=1e-3)
        incr_(step_t)
        fused_adamw_(param, gq, master, m, v, lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1, step=step,
                     max_norm=1.0, sumsq=sumsq, step_tensor=step_t)
    assert int(step_t.item()) == 5
    assert torch.allclose(master, ref_p.detach(), atol=2e-5, rtol=1e-4)
    tol = 1e-2 if pdtype == torch.bfloat16 else 1e-6
    assert torch.allclose(param.float(), master, atol=tol, rtol=tol)


@pytest.mark.parametrize("dtype,wire", [(torch.float32, None), (torch.float32, "bfloat16"), (torch.bfloat16, None)])
def test_collective_kernels_single_gpu_identity(dev, dtype, wire):
    """World size 1 with forced kernels: every stage (stage-in cast, barrier, reduce, stage-out)
    runs on one GPU; the result must equal the (wire-rounded) input."""
    from adapcc_b200.constants import ALLREDUCE
    from adapcc_b200.runtime.native import NativeComm

    comm = NativeComm(f"t1-{os.getpid()}-{dtype}-{wire}", 0, 1, 0, staging_bytes=8 << 20, heap_bytes=8 << 20)
    try:
        comm.set_tunable("force_kernel", 1)
        for n in (1, 17, 4099, 300_001):
            x = torch.randn(n, device=dev).to(dtype)
            want = x.to(getattr(torch, wire)).to(dtype) if wire else x
            for algo in ["one_shot", "two_shot"] + (["nvls"] if comm.multicast else []):
                y = x.clone()
                comm.all_reduce(y, op="sum", algo=algo, wire=wire)
                comm.check()
                assert torch.equal(y, want), (algo, n)
            y = x.clone()
            comm.all_reduce(y, op="avg", algo="two_shot", wire=wire)
            comm.check()
            assert torch.equal(y, want)
        # pipelined staged kernel (two sub-grids) on one GPU
        comm.set_tunable("pipe_min_bytes", 1 << 16)
        comm.set_tunable("pipe_nvls", 1)
        comm.set_tunable("pipe_piece_bytes", 1 << 16)
        for algo in ["two_shot"] + (["nvls"] if comm.multicast else []):
            y = x.clone()
            comm.all_reduce(y, op="sum", algo=algo, wire=wire)
            comm.check()
            assert torch.equal(y, want), ("pipelined", algo)
        comm.set_tunable("pipe_min_bytes", 32 << 20)
        # zero-copy path on the symmetric heap
        t = comm.symm_empty(70_000, dtype)
        src = torch.randn(70_000, device=dev).to(dtype)
        t.copy_(src)
        comm.all_reduce(t, op="sum", algo="two_shot")
        comm.check()
        assert torch.equal(t, src)
        # strategy tree with a single rank
        comm.load_strategy("<trees><root id='0' ip='a'/></trees>")
        y = x.clone()
        comm.tree_collective(ALLREDUCE, y, wire=wire, chunk_bytes=4096)
        comm.check()
        # the root hands its fp32 accumulator straight to the user tensor (no wire rounding)
        assert torch.allclose(y.float(), x.float(), atol=0, rtol=0) or torch.equal(y, want)
    finally:
        comm.close()


def test_model_gpu_matches_fp32_reference(dev):
    """bf16 model + fused chunked LM-head/CE against the same weights evaluated in fp32 PyTorch."""
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, synthetic_batch

    torch.manual_seed(0)
    cfg = GPT2Config.tiny()
    ref = GPT2DoubleHeads(cfg).to(dev)
    model = GPT2DoubleHeads(cfg).to(dev)
    model.load_state_dict(ref.state_dict())
    model = model.bfloat16()
    batch = synthetic_batch(2, 2, 48, cfg.vocab_size, device=dev)
    l_ref, lm_ref, mc_ref = ref(**batch)
    l, lm, mc = model(**batch)
    assert abs(l.item() - l_ref.item()) < 0.05 * abs(l_ref.item())
    l_ref.backward()
    l.backward()
    g_ref, g = ref.wte.weight.grad, model.wte.weight.grad.float()
    cos = torch.nn.functional.cosine_similarity(g.flatten(), g_ref.flatten(), dim=0)
    assert cos > 0.99, cos


def test_engine_trains_and_graph_matches_eager(dev):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, synthetic_batch
    from adapcc_b200.parallel.engine import FlatDataParallel

    cfg = GPT2Config.tiny()
    batch = synthetic_batch(2, 2, 32, cfg.vocab_size, device=dev)
    losses = {}
    for mode in ("eager", "graph"):
        torch.manual_seed(3)
        model = GPT2DoubleHeads(cfg).to(dev)
        eng = FlatDataParallel(model, None, world_size=1, lr=2e-3, max_norm=1.0)
        ptrs = [p.grad.data_ptr() for p in eng.params]
        out = []
        if mode == "graph":
            eng.capture(batch, warmup=0)
            for _ in range(8):
                out.append(float(eng.step_graph(batch).item()))
        else:
            for _ in range(8):
                out.append(float(eng.step(batch).item()))
        assert [p.grad.data_ptr() for p in eng.params] == ptrs      # grads stayed views of the flat buffer
        assert out[-1] < out[0] - 0.1, out
        losses[mode] = out
        eng.close()
    assert abs(losses["eager"][-1] - losses["graph"][-1]) < 0.05 * abs(losses["eager"][-1])


def test_graft_smoke(dev):
    import __graft_entry__ as g

    g.smoke()


# 4099 rows at every width (ids: the width alone), and single-row / sub-CTA / one-past-a-CTA row counts
LN_CASES = ([pytest.param(d, 4099, id=str(d)) for d in (256, 512, 768, 1024)]
            + [pytest.param(d, r, id=f"{d}-rows{r}") for d in (256, 512, 768, 1024) for r in (1, 7, 9)])


@pytest.mark.parametrize("d,rows", LN_CASES)
def test_fused_layernorm_matches_torch(dev, d, rows):
    from adapcc_b200.ops.layers import FusedLayerNorm

    torch.manual_seed(d + rows)
    ln = FusedLayerNorm(d).to(dev).bfloat16()
    with torch.no_grad():
        ln.weight.copy_(torch.randn(d) * 0.5 + 1)
        ln.bias.copy_(torch.randn(d) * 0.1)
    x = (torch.randn(rows, d, device=dev) * 2 + 0.5).bfloat16().requires_grad_(True)
    dy = torch.randn(rows, d, device=dev).bfloat16()
    y = ln(x)
    y.backward(dy)
    xr = x.detach().float().requires_grad_(True)
    wr = ln.weight.detach().float().requires_grad_(True)
    br = ln.bias.detach().float().requires_grad_(True)
    yr = torch.nn.functional.layer_norm(xr, (d,), wr, br, ln.eps)
    yr.backward(dy.float())
    assert torch.allclose(y.float(), yr, atol=3e-2, rtol=2e-2)
    assert torch.allclose(x.grad.float(), xr.grad, atol=5e-2, rtol=5e-2)
    # column reductions over 4099 rows: compare relative to the fp32 result's scale
    for got, want in ((ln.weight.grad, wr.grad), (ln.bias.grad, br.grad)):
        err = (got.float() - want).abs().max() / want.abs().max()
        assert err < 2e-2, err


@pytest.mark.parametrize("d", [256, 512, 768])
def test_fused_add_layernorm_matches_torch(dev, d):
    """(x, res) -> (x + res, LN(x + res)) and its backward with a residual-stream gradient."""
    from adapcc_b200.ops.layers import FusedLayerNorm

    torch.manual_seed(d + 1)
    rows = 2051
    ln = FusedLayerNorm(d).to(dev).bfloat16()
    with torch.no_grad():
        ln.weight.copy_(torch.randn(d) * 0.5 + 1)
        ln.bias.copy_(torch.randn(d) * 0.1)
    x = (torch.randn(rows, d, device=dev) * 2).bfloat16().requires_grad_(True)
    r = (torch.randn(rows, d, device=dev) + 0.5).bfloat16().requires_grad_(True)
    dy = torch.randn(rows, d, device=dev).bfloat16()
    ds = torch.randn(rows, d, device=dev).bfloat16()
    s, y = ln.forward_add(x, r)
    torch.autograd.backward([s, y], [ds, dy])
    # the sum is exactly the bf16 add
    assert torch.equal(s, x.detach() + r.detach())
    xr = x.detach().float().requires_grad_(True)
    rr = r.detach().float().requires_grad_(True)
    wr = ln.weight.detach().float().requires_grad_(True)
    br = ln.bias.detach().float().requires_grad_(True)
    # the same bf16-rounded sum, with the gradient passing straight through the rounding
    sr = (xr + rr) + ((xr + rr).bfloat16().float() - (xr + rr)).detach()
    yr = torch.nn.functional.layer_norm(sr, (d,), wr, br, ln.eps)
    torch.autograd.backward([sr, yr], [ds.float(), dy.float()])
    assert torch.allclose(y.float(), yr, atol=3e-2, rtol=2e-2)
    assert torch.allclose(x.grad.float(), xr.grad, atol=6e-2, rtol=5e-2)
    assert torch.equal(x.grad, r.grad)
    for got, want in ((ln.weight.grad, wr.grad), (ln.bias.grad, br.grad)):
        err = (got.float() - want).abs().max() / want.abs().max()
        assert err < 2e-2, err
    # unused sum (the final LayerNorm of the network): gradient is the plain LayerNorm one
    x2 = x.detach().clone().requires_grad_(True)
    r2 = r.detach().clone().requires_grad_(True)
    ln.zero_grad()
    ln.forward_add(x2, r2)[1].backward(dy)
    x3 = (x.detach() + r.detach()).requires_grad_(True)
    ln(x3).backward(dy)
    assert torch.equal(x2.grad, x3.grad)


def test_gpt2_fused_residual_path_matches_unfused(dev):
    """d = 256 so the fused LayerNorm kernels run; deferred-residual blocks vs plain blocks, and the
    LM head on scored rows only vs all rows, eager and under CUDA-graph capture."""
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, lm_rows_needed, synthetic_batch
    from adapcc_b200.parallel.engine import FlatDataParallel

    cfg = GPT2Config(vocab_size=1000, n_positions=64, n_embd=256, n_layer=3, n_head=4, lm_chunk_rows=96)
    torch.manual_seed(11)
    base = GPT2DoubleHeads(cfg).to(dev).bfloat16()
    batch = synthetic_batch(2, 2, 64, cfg.vocab_size, device=dev)
    need = lm_rows_needed(batch["lm_labels"], multiple=16)

    def run(fuse, cap):
        m = GPT2DoubleHeads(cfg).to(dev).bfloat16()
        m.load_state_dict(base.state_dict())
        m.fuse_add_ln, m.lm_row_capacity = fuse, cap
        loss = m(**batch)[0]
        loss.backward()
        return loss.item(), torch.cat([p.grad.float().flatten() for p in m.parameters()])

    l0, g0 = run(False, 0)
    for fuse, cap in ((True, 0), (False, need), (True, need)):
        l1, g1 = run(fuse, cap)
        assert abs(l1 - l0) < 2e-2 * abs(l0), (fuse, cap, l0, l1)
        cos = torch.nn.functional.cosine_similarity(g0, g1, dim=0)
        assert cos > 0.995, (fuse, cap, cos)
    # whole step captured in a graph with both options on
    torch.manual_seed(12)
    m = GPT2DoubleHeads(cfg).to(dev)
    m.fuse_add_ln, m.lm_row_capacity = True, need
    eng = FlatDataParallel(m, None, world_size=1, lr=2e-3, max_norm=1.0)
    eng.capture(batch, warmup=1)
    out = [float(eng.step_graph(batch).item()) for _ in range(8)]
    assert out[-1] < out[0] - 0.1, out
    eng.close()


def test_adamw_device_learning_rate_and_engine_set_lr(dev):
    """lr read from a device scalar: overrides the launch argument, and set_lr() takes effect inside a captured graph."""
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, synthetic_batch
    from adapcc_b200.ops import fused_adamw_
    from adapcc_b200.parallel.engine import FlatDataParallel

    torch.manual_seed(1)
    n = 4099
    g = torch.randn(n, device=dev)
    outs = []
    for lr_arg, lr_dev in ((3e-3, None), (123.0, 3e-3)):            # the tensor wins over a deliberately absurd argument
        p = torch.ones(n, device=dev)
        master, m, v = p.clone(), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
        lr_t = None if lr_dev is None else torch.full((1,), lr_dev, device=dev)
        fused_adamw_(p, g, master, m, v, lr=lr_arg, step=1, lr_tensor=lr_t)
        outs.append(p.clone())
    assert torch.equal(outs[0], outs[1]) and not torch.equal(outs[0], torch.ones(n, device=dev))
    cfg = GPT2Config.tiny()
    batch = synthetic_batch(2, 2, 32, cfg.vocab_size, device=dev)
    torch.manual_seed(2)
    eng = FlatDataParallel(GPT2DoubleHeads(cfg).to(dev), None, world_size=1, lr=2e-3)
    eng.capture(batch, warmup=0)
    eng.step_graph(batch)
    before = eng.flat_param.clone()
    eng.step_graph(batch)
    assert not torch.equal(before, eng.flat_param)                  # training moves the weights ...
    frozen = eng.flat_param.clone()
    eng.set_lr(0.0)
    eng.step_graph(batch)
    assert torch.equal(frozen, eng.flat_param)                      # ... until the schedule says lr = 0, same graph
    eng.close()


def test_engine_direct_grads_match_accumulated(dev):
    """Fused ops writing parameter gradients straight into the flat buffer vs autograd accumulation."""
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, synthetic_batch
    from adapcc_b200.parallel.engine import FlatDataParallel

    cfg = GPT2Config(vocab_size=1000, n_positions=64, n_embd=256, n_layer=2, n_head=4, lm_chunk_rows=96)
    batch = synthetic_batch(2, 2, 64, cfg.vocab_size, device=dev)
    grads, losses = {}, {}
    for direct in (False, True):
        torch.manual_seed(21)
        m = GPT2DoubleHeads(cfg).to(dev)
        m.fuse_add_ln = direct                              # cover both LayerNorm backward variants
        eng = FlatDataParallel(m, None, world_size=1, lr=1e-3, max_norm=1.0, direct_grads=direct)
        assert eng.direct_grads == direct
        eng.step(batch)
        grads[direct] = eng.flat_grad.float().clone()
        losses[direct] = [float(eng.step(batch).item()) for _ in range(4)]
        eng.close()
        assert not any(hasattr(p, "_adapcc_grad_sink") for p in m.parameters())
    ref = grads[False]
    assert ref.abs().max() > 0
    assert (grads[True] - ref).abs().max() <= 5e-2 * ref.abs().max()
    cos = torch.nn.functional.cosine_similarity(grads[True], ref, dim=0)
    assert cos > 0.995, cos
    assert abs(losses[True][-1] - losses[False][-1]) < 0.03 * abs(losses[False][-1])


def test_fused_linear_bias_grad(dev):
    from adapcc_b200.ops.layers import FusedLinear

    torch.manual_seed(5)
    lin = FusedLinear(768, 2304).to(dev).bfloat16()
    x = torch.randn(8, 1000, 768, device=dev).bfloat16().requires_grad_(True)
    dy = torch.randn(8, 1000, 2304, device=dev).bfloat16()
    lin(x).backward(dy)
    ref_db = dy.float().sum((0, 1))
    ref_dw = dy.float().reshape(-1, 2304).t() @ x.detach().float().reshape(-1, 768)
    assert (lin.bias.grad.float() - ref_db).abs().max() / ref_db.abs().max() < 1e-2
    assert (lin.weight.grad.float() - ref_dw).abs().max() / ref_dw.abs().max() < 2e-2
    assert x.grad is not None and x.grad.shape == x.shape


def test_moe_exchange_single_rank_matches_local_reference(dev):
    """Expert 'parallel' exchange kernels with world=1 (push/pull through the symmetric heap) must
    reproduce the pure-PyTorch local-expert path, forward and backward; two identical runs give
    bit-identical expert gradients."""
    _moe_exchange_matches_local(dev, overflow=False)


def test_moe_exchange_overflow_matches_local_reference(dev):
    """The same with most tokens dropped: the gate's bias sends every token to expert 0 and
    capacity_factor 0.5 leaves room for a quarter of them; both paths must keep the same first
    `capacity` tokens (in token order)."""
    _moe_exchange_matches_local(dev, overflow=True)


def _moe_exchange_matches_local(dev, overflow):
    from adapcc_b200.models.moe import MoEMLP
    from adapcc_b200.parallel.expert_parallel import ExpertExchange
    from adapcc_b200.runtime.native import NativeComm

    comm = NativeComm(f"moe-{os.getpid()}-{overflow}", 0, 1, 0, staging_bytes=4 << 20, heap_bytes=64 << 20)
    try:
        torch.manual_seed(11)
        E, d, h, T, k = 4, 64, 128, 96, 2
        cf = 0.5 if overflow else 2.0
        ref = MoEMLP(E, d, h, top_k=k, capacity_factor=cf).to(dev).bfloat16()
        if overflow:
            with torch.no_grad():
                ref.gate.bias[0] += 8.0
        cap = ref.capacity(T)
        ex = ExpertExchange(comm, E, cap, d)
        moe = MoEMLP(E, d, h, top_k=k, capacity_factor=cf, exchange=ex).to(dev).bfloat16()
        moe.load_state_dict(ref.state_dict())
        x = torch.randn(T, d, device=dev).bfloat16()
        x1, x2 = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        y1, y2 = ref(x1), moe(x2)
        comm.check()
        assert torch.allclose(y1.float(), y2.float(), atol=2e-2, rtol=2e-2)
        g = torch.randn_like(y1)
        y1.backward(g)
        y2.backward(g)
        comm.check()
        assert torch.allclose(x1.grad.float(), x2.grad.float(), atol=3e-2, rtol=3e-2)
        assert torch.allclose(ref.w1.grad.float(), moe.w1.grad.float(), atol=3e-2, rtol=3e-2)
        assert torch.allclose(ref.gate.weight.grad.float(), moe.gate.weight.grad.float(), atol=5e-2, rtol=5e-2)
        if overflow:
            expert = torch.topk(ref.gate(x).float(), k, dim=-1).indices.reshape(-1).to(torch.int32)
            assert int((expert == 0).sum()) > cap                       # the case really drops tokens
        first = [p.grad.clone() for p in (moe.w1, moe.w2, moe.b1, moe.b2)]
        for p in moe.parameters():
            p.grad = None
        x3 = x.clone().requires_grad_(True)
        moe(x3).backward(g)
        comm.check()
        for p, want in zip((moe.w1, moe.w2, moe.b1, moe.b2), first):
            assert torch.equal(p.grad, want)
    finally:
        comm.close()


def test_reference_c_abi_symbols(dev, tmp_path, monkeypatch):
    """The six symbols of the reference's communicator.so (initThreads / exitThreads / allreduce /
    reduce / boardcast / updateActive), called through ctypes exactly like its commu.py does."""
    import ctypes

    from adapcc_b200.runtime.native import load_library

    lib = load_library()
    for sym in ("initThreads", "exitThreads", "allreduce", "reduce", "boardcast", "updateActive"):
        assert hasattr(lib, sym)
    monkeypatch.setenv("RANK", "0")
    monkeypatch.setenv("WORLD_SIZE", "1")
    monkeypatch.setenv("LOCAL_RANK", "0")
    monkeypatch.setenv("ADAPCC_STAGING_MB", "8")
    sf = tmp_path / "s.xml"
    sf.write_text("<trees><root id='0' ip='10.0.0.1'/></trees>")
    lib.initThreads(ctypes.c_int(0), ctypes.c_char_p(str(sf).encode()), ctypes.c_int(5000 + os.getpid() % 1000))
    t = torch.ones(16, device=dev) * 3
    active = (ctypes.c_int * 1)(0)
    lib.allreduce(ctypes.c_void_p(t.data_ptr()), ctypes.c_int(16), ctypes.c_int(8), active, ctypes.c_int(1))
    assert torch.equal(t.cpu(), torch.full((16,), 3.0))
    lib.updateActive(ctypes.c_int(0))
    lib.allreduce(ctypes.c_void_p(t.data_ptr()), ctypes.c_int(16), ctypes.c_int(8), active, ctypes.c_int(1))
    assert torch.equal(t.cpu(), torch.full((16,), 3.0))
    lib.exitThreads(ctypes.c_int(0))


def test_fused_embedding_sum_matches_torch(dev):
    """One-kernel embedding sum and its sort-free backward (fixed-point accumulation of duplicate rows, in-place add
    into an existing gradient) against F.embedding on fp32 copies; two rounds: the work buffers must come back clean;
    the same backward repeated gives the same bits."""
    from adapcc_b200.ops import fused_embedding_sum

    torch.manual_seed(5)
    V, P, D, N, T = 1000, 64, 256, 4, 64
    wte = (torch.randn(V, D, device=dev) * 0.5).bfloat16().requires_grad_(True)
    wpe = (torch.randn(P, D, device=dev) * 0.5).bfloat16().requires_grad_(True)
    for rnd in range(2):
        ids = torch.randint(0, V, (N, T), device=dev)
        ids[:, :8] = 7                                               # heavy duplication of one row
        tt = torch.randint(V - 2, V, (N, T), device=dev)              # two token-type rows hit by everything
        pos = torch.arange(T, device=dev).repeat(N)
        y = fused_embedding_sum([wte, wpe], [(0, ids), (1, pos), (0, tt)])
        w32, p32 = wte.detach().float().requires_grad_(True), wpe.detach().float().requires_grad_(True)
        F = torch.nn.functional
        y_ref = F.embedding(ids.reshape(-1), w32) + F.embedding(pos, p32) + F.embedding(tt.reshape(-1), w32)
        assert torch.allclose(y.float(), y_ref, atol=2e-2, rtol=1e-2)
        dy = (torch.randn(N * T, D, device=dev) * 0.1).bfloat16()
        wte.grad = wpe.grad = None
        y.backward(dy)
        y_ref.backward(dy.float())
        for got, ref in ((wte.grad, w32.grad), (wpe.grad, p32.grad)):
            err = (got.float() - ref).abs().max()
            assert err <= 2e-2 * ref.abs().max() + 1e-3, (rnd, float(err), float(ref.abs().max()))
        untouched = torch.ones(V, dtype=torch.bool, device=dev)
        untouched[ids.reshape(-1)] = False
        untouched[tt.reshape(-1)] = False
        assert torch.all(wte.grad[untouched] == 0)
        first = (wte.grad.clone(), wpe.grad.clone())
        for _ in range(3):
            wte.grad = wpe.grad = None
            fused_embedding_sum([wte, wpe], [(0, ids), (1, pos), (0, tt)]).backward(dy)
            assert torch.equal(wte.grad, first[0]) and torch.equal(wpe.grad, first[1])


def test_fused_ce_grad_scale(dev):
    from adapcc_b200.ops import fused_ce_

    torch.manual_seed(6)
    rows, vocab, stride = 64, 1000, 1024
    logits = (torch.randn(rows, stride, device=dev) * 2).bfloat16()
    labels = torch.randint(0, vocab, (rows,), device=dev)
    labels[::5] = -100
    a, b = logits.clone(), logits.clone()
    la = fused_ce_(a, labels, vocab)
    scale = torch.tensor([0.125], device=dev)
    lb = fused_ce_(b, labels, vocab, grad_scale=scale)
    assert torch.equal(la, lb)                                       # row losses are not scaled
    assert torch.allclose(b.float(), a.float() * 0.125, atol=2e-3, rtol=2e-2)


def test_causal_attention_backward_is_repeatable(dev):
    """GPT-2's attention: same gradients as plain SDPA (up to bf16 rounding), identical bits on every repetition, and
    PyTorch's deterministic-algorithms setting left as it was."""
    from adapcc_b200.models.gpt2 import causal_attention

    torch.manual_seed(9)
    q, k, v = (torch.randn(4, 12, 512, 64, device=dev).bfloat16().requires_grad_(True) for _ in range(3))
    do = torch.randn(4, 12, 512, 64, device=dev).bfloat16()
    F = torch.nn.functional
    F.scaled_dot_product_attention(q, k, v, is_causal=True).backward(do)
    ref = [t.grad.clone() for t in (q, k, v)]
    first = None
    for _ in range(4):
        for t in (q, k, v):
            t.grad = None
        causal_attention(q, k, v).backward(do)
        got = [t.grad.clone() for t in (q, k, v)]
        for a, b in zip(got, ref):
            assert torch.allclose(a.float(), b.float(), atol=2e-2, rtol=2e-2)
        if first is None:
            first = got
        assert all(torch.equal(a, b) for a, b in zip(got, first))
    assert not torch.are_deterministic_algorithms_enabled()
