"""The wgmma GEMM's epilogue (csrc/gemm_wgmma.cu) stores through shared-memory staging buffers with TMA.

* GPU: the C entry points, called on the first M rows of larger sentinel-filled buffers, write no row past M (the
  tensor map's bounds are the only thing that clips them), with and without `pre`, for every act and every variant
  the act supports; the result equals the same call on exactly-sized buffers, and repeats bit for bit.
* Build box: the SASS of the ACT 0 / 1 kernels stores its outputs with UTMASTG and has no STG.E left.
* CPU model of the staging protocol under random schedules: a consumer warp's ring of NB buffers, TMA stores
  committed one bulk group per buffer use and reused after `cp.async.bulk.wait_group.read NB - 1`; for the aux
  epilogues, TMA loads into the ring completing on one mbarrier per buffer (parity tracked per buffer), the result
  written back in place, and a refill only after the store has read the buffer. Deliberately wrong variants must be
  caught.
"""
import ctypes
import random
import re
import shutil
import subprocess

import pytest
import torch

SENTINEL = -12288.0          # -1.5 * 2^13: exactly representable in bf16


# ---------------------------------------------------------------------------------------------- GPU: rows past M
def _ptr(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def _call(lib, x, w, b, out, pre, act, variant, colsum=None, work=None):
    m, k = x.shape
    n = w.shape[0]
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if variant == 3:
        rc = lib.adapcc_gemm_pp(_ptr(x), _ptr(w), _ptr(b), _ptr(out), _ptr(pre), _ptr(colsum), _ptr(work), m, n, k, act,
                                stream)
    else:
        rc = lib.adapcc_gemm_bias_act_v(_ptr(x), _ptr(w), _ptr(b), _ptr(out), _ptr(pre), m, n, k, act, variant, stream)
    assert rc == 0


def _cases():
    for n in (256, 128):
        for act in (0, 1, 2, 3):
            if act <= 1:
                variants = [0, 1, 2, 3] if n == 256 else [0, 1]
            elif act == 2:
                variants = [0, 3] if n == 256 else [0]
            else:
                variants = [0]
            for v in variants:
                yield n, act, v


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 127, 129, 200, 8191])
@pytest.mark.parametrize("n,act,variant", list(_cases()))
def test_no_writes_past_m(m, n, act, variant):
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from adapcc_b200.ops.gemm import _lib

    lib = _lib()
    dev = torch.device("cuda:0")
    k = 128
    torch.manual_seed(m * 7 + n + act)
    x = torch.randn(m, k, device=dev).bfloat16()
    w = (torch.randn(n, k, device=dev) / k ** 0.5).bfloat16()
    b = torch.randn(n, device=dev).bfloat16() if act != 2 else None
    big = m + 133                                   # rows past M, not a multiple of any tile
    aux_rows = torch.randn(m, n, device=dev).bfloat16()
    pre_modes = [False, True] if act <= 1 else [True]
    for with_pre in pre_modes:
        out_big = torch.full((big, n), SENTINEL, dtype=torch.bfloat16, device=dev)
        pre_big = torch.full((big, n), SENTINEL, dtype=torch.bfloat16, device=dev) if with_pre else None
        if act >= 2:
            pre_big[:m] = aux_rows                  # an input in these modes; the rows past M must stay untouched too
        colsum = work = None
        if act == 2 and variant == 3:
            colsum = torch.zeros(n, dtype=torch.float32, device=dev)
            work = torch.empty((m + 127) // 128, n, dtype=torch.float32, device=dev)
        _call(lib, x, w, b, out_big, pre_big, act, variant, colsum, work)
        # the same call on exactly-sized buffers, twice
        outs = []
        for _ in range(2):
            out = torch.empty(m, n, dtype=torch.bfloat16, device=dev)
            pre = (aux_rows.clone() if act >= 2 else torch.empty(m, n, dtype=torch.bfloat16, device=dev)) \
                if with_pre else None
            cs2 = torch.zeros(n, dtype=torch.float32, device=dev) if colsum is not None else None
            _call(lib, x, w, b, out, pre, act, variant, cs2, torch.empty_like(work) if work is not None else None)
            outs.append((out, pre, cs2))
        torch.cuda.synchronize()
        tail = f"act {act} variant {variant} n {n} pre {with_pre}"
        assert bool((out_big[m:].float() == SENTINEL).all()), "out written past M: " + tail
        if pre_big is not None:
            assert bool((pre_big[m:].float() == SENTINEL).all()), "pre written past M: " + tail
        out, pre, cs2 = outs[0]
        assert torch.equal(out_big[:m], out), tail
        if with_pre:
            assert torch.equal(pre_big[:m], pre), tail
        if colsum is not None:
            assert torch.equal(colsum, cs2), tail
        out_r, pre_r, cs_r = outs[1]                # repeat runs give identical bits
        assert torch.equal(out_r, out) and (pre is None or torch.equal(pre_r, pre)), tail
        assert cs2 is None or torch.equal(cs_r, cs2), tail
        if act <= 1:                                # and the values are the GEMM's
            u = x.float() @ w.float().t() + b.float()
            for got in ([out] if act == 0 else []) + ([pre] if with_pre else []):
                assert torch.allclose(got.float(), u, atol=3e-2, rtol=2e-2), tail


# ---------------------------------------------------------------------------------------------- build box: SASS
def test_sass_act01_kernels_store_with_tma_only():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    from adapcc_b200.build import build

    lib = build()
    sass = subprocess.run(["cuobjdump", "-sass", str(lib)], capture_output=True, text=True, timeout=600).stdout
    blocks = dict(zip(re.findall(r"Function : (\S+)", sass), re.split(r"\n\s*Function : \S+\n", sass)[1:]))
    # template arguments <BN, ACT, CLUSTER>
    act01 = {name: body for name, body in blocks.items()
             if re.search(r"gemm_bias_act_wgmma_kernelILi\d+ELi[01]ELi\d+E", name)}
    assert len(act01) == 6, sorted(act01)          # BN 128 / 256 x ACT 0 / 1 x one CTA, and BN 256 pairs x ACT 0 / 1
    for name, body in act01.items():
        assert "UTMASTG" in body, name
        assert "STG.E" not in body, name
    aux = [body for name, body in blocks.items() if re.search(r"gemm_bias_act_wgmma_kernelILi\d+ELi[23]ELi\d+E", name)]
    assert aux and all("UTMASTG" in b and "UTMALDG" in b and "LDSM" in b for b in aux)


# ---------------------------------------------------------------------------------------------- CPU protocol model
class MBar:
    def __init__(self, count):
        self.count, self.pending, self.tx, self.phase = count, count, 0, 0

    def _maybe_flip(self):
        if self.pending == 0 and self.tx == 0:
            self.phase ^= 1
            self.pending = self.count

    def arrive(self, expect_tx=0):
        self.tx += expect_tx
        self.pending -= 1
        assert self.pending >= 0
        self._maybe_flip()

    def complete_tx(self, n):
        self.tx -= n
        self._maybe_flip()

    def done(self, parity):
        return self.phase != parity


def simulate_staging(tiles, J, NB, aux, has_pre, seed, bug=None, max_steps=200_000):
    """One consumer warp over `tiles` tiles of J sub-tiles. bug: None, "ring_depth" (reuse after wait_group.read NB
    instead of NB - 1), "aux_parity" (wait on the wrong parity of a buffer's mbarrier), "refill_no_wait" (refill a
    buffer before its store has read it), "prefetch_no_wait" (load a tile's first aux sub-tiles without waiting for the
    previous tile's stores)."""
    rng = random.Random(seed)
    bufs = [None] * NB
    bars = [MBar(1) for _ in range(NB)]
    groups = []                                   # per committed bulk group: [read_done]
    tma = []                                      # pending async ops
    stored = []

    def wait_read(n):
        while not all(g[0] for g in groups[:max(0, len(groups) - n)]):
            yield

    def commit_store(b, tag):
        g = [False]
        groups.append(g)
        tma.append(("store", b, tag, g))

    def load(b, tag):
        bars[b].arrive(expect_tx=1)
        tma.append(("load", b, tag, None))

    def warp():
        epi_it, phase = 0, 0
        for t in range(tiles):
            if aux:
                # issued under the tile's first slab
                if bug != "prefetch_no_wait":
                    yield from wait_read(0)
                for b in range(NB):
                    load(b, (t, b, "aux"))
            for _ in range(rng.randint(0, 3)):    # the mainloop
                yield
            for j in range(J):
                if aux:
                    b = j % NB
                    want = ((phase >> b) & 1) ^ (1 if bug == "aux_parity" else 0)
                    while not bars[b].done(want):
                        yield
                    phase ^= 1 << b
                    assert bufs[b] == (t, j, "aux"), f"sub-tile {(t, j)} read {bufs[b]} from buffer {b}"
                    yield
                    bufs[b] = (t, j, "out")       # the result, in place
                    commit_store(b, (t, j, "out"))
                    if j + NB < J:
                        if bug != "refill_no_wait":
                            yield from wait_read(0)
                        load(b, (t, j + NB, "aux"))
                else:
                    for what in (("pre", "out") if has_pre else ("out",)):
                        yield from wait_read(NB if bug == "ring_depth" else NB - 1)
                        b = epi_it % NB
                        bufs[b] = (t, j, what)
                        yield
                        commit_store(b, (t, j, what))
                        epi_it += 1
                yield
        yield from wait_read(0)                    # cp.async.bulk.wait_group before the CTA exits

    def engine():
        while True:
            if tma and rng.random() < 0.5:
                kind, b, tag, g = tma.pop(rng.randrange(min(len(tma), 3)))   # out of order
                if kind == "store":
                    assert bufs[b] == tag, f"store of {tag} read {bufs[b]} from buffer {b}"
                    stored.append(tag)
                    g[0] = True
                else:
                    bufs[b] = tag
                    bars[b].complete_tx(1)
            yield

    w, e = warp(), engine()
    for _ in range(max_steps):
        next(e)
        try:
            for _ in range(rng.randint(1, 4)):
                next(w)
        except StopIteration:
            while tma:                              # drain
                next(e)
            what = ("out",) if aux else (("pre", "out") if has_pre else ("out",))
            assert sorted(stored) == sorted((t, j, x) for t in range(tiles) for j in range(J) for x in what)
            return
    raise TimeoutError("deadlock")


@pytest.mark.parametrize("J,NB", [(4, 1), (4, 2), (4, 4), (2, 1), (2, 2)])
@pytest.mark.parametrize("aux,has_pre", [(False, False), (False, True), (True, True)])
def test_staging_protocol_is_consistent(J, NB, aux, has_pre):
    for seed in range(25):
        simulate_staging(5, J, NB, aux, has_pre, seed)


@pytest.mark.parametrize("bug,aux,J,NB", [("ring_depth", False, 4, 2), ("ring_depth", False, 4, 1),
                                          ("aux_parity", True, 4, 4), ("aux_parity", True, 4, 2),
                                          ("refill_no_wait", True, 4, 1), ("refill_no_wait", True, 4, 2),
                                          ("prefetch_no_wait", True, 4, 4), ("prefetch_no_wait", True, 2, 2)])
def test_staging_model_catches_protocol_bugs(bug, aux, J, NB):
    caught = 0
    for seed in range(20):
        try:
            simulate_staging(5, J, NB, aux, True, seed, bug=bug, max_steps=20_000)
        except (AssertionError, TimeoutError):
            caught += 1
    assert caught >= 15, caught
