"""Model check, on CPU, of the mbarrier protocol of the GEMM in csrc/gemm_wgmma.cu (the file name predates the port).

Per CTA: one TMA producer thread and two consumer warpgroups, synchronised only through mbarriers with hand-computed
stage / phase indices. `full[s]` completes on the transferred bytes (expect_tx / complete_tx); `empty[s]` counts one
arrival per consumer warpgroup of EVERY CTA of the cluster. In a two-CTA cluster each producer loads its own A slab and
half of the W slab, which it multicasts into the same stage of both CTAs — so bytes may complete on a CTA's `full[s]`
before its own producer has posted expect_tx, and a stage may only be refilled once the consumers of both CTAs have
released it. A consumer keeps one wgmma group in flight and releases a stage when the group that read it has retired.
This reproduces those index computations as coroutines over a small mbarrier model, with an asynchronous TMA engine
(completions in any order) and an asynchronous tensor core per consumer, under random schedules, and checks that
  * a stage is never overwritten before every wgmma reading it has executed,
  * every wgmma reads exactly its own tile's and K-slab's A rows and both halves of its W slab,
  * nothing deadlocks.
Deliberately wrong variants (a wrong phase parity, a release before the wgmma group retired, a release to the local CTA
only) must be caught."""
import random
from collections import deque

import pytest

STAGES = 4


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
        assert self.pending >= 0, "more arrivals than the barrier was initialised for"
        self._maybe_flip()

    def complete_tx(self, n):
        self.tx -= n
        self._maybe_flip()

    def done(self, parity):                 # mbarrier.try_wait.parity: has the phase with this parity completed?
        return self.phase != parity


def simulate(tiles, num_kb, seed, cluster=1, bug=None, max_steps=400_000):
    """`tiles` per CTA (cluster); bug: None, "producer_parity", "acc_parity" (a consumer releases a stage as soon as its
    wgmma group is committed, while the group in flight still reads it) or "local_release" (consumers arrive only on
    their own CTA's `empty`, which then counts 2)."""
    rng = random.Random(seed)
    C, CONS = cluster, 2
    per_cta = CONS if bug == "local_release" else CONS * C
    full = [[MBar(1) for _ in range(STAGES)] for _ in range(C)]
    empty = [[MBar(per_cta) for _ in range(STAGES)] for _ in range(C)]
    smem_a = [[None] * STAGES for _ in range(C)]                  # [cta][stage] -> (tile, kb, cta)
    smem_w = [[[None] * C for _ in range(STAGES)] for _ in range(C)]  # [cta][stage][half] -> (tile, kb)
    tma_q = []
    tc_q = {(r, c): deque() for r in range(C) for c in range(CONS)}   # in-order wgmma groups per consumer
    seen = []

    def producer(r):
        it = 0
        for t in range(tiles):
            for kb in range(num_kb):
                s, ph = it % STAGES, (it // STAGES) & 1
                want = ph ^ 1 if bug != "producer_parity" else ph
                while not empty[r][s].done(want):
                    yield
                full[r][s].arrive(expect_tx=2 + 2)                # A (2 units) + the whole W slab (2 units)
                tma_q.append(("A", r, s, (t, kb, r)))
                if C == 1:
                    tma_q.append(("W", r, s, (t, kb)))
                else:
                    tma_q.append(("Wh", r, s, (t, kb)))           # half r, multicast to every CTA
                it += 1
                yield

    def consumer(r, c):
        q = tc_q[(r, c)]
        it = 0

        def release(s):
            for d in ([r] if bug == "local_release" or C == 1 else range(C)):
                empty[d][s].arrive()

        for t in range(tiles):
            prev = None
            for kb in range(num_kb):
                s, ph = it % STAGES, (it // STAGES) & 1
                while not full[r][s].done(ph):
                    yield
                q.append((s, (t, kb)))                            # wgmma group reading stage s
                if bug == "acc_parity":
                    release(s)
                else:
                    while len(q) > 1:                             # wgmma.wait_group 1
                        yield
                    if prev is not None:
                        release(prev)
                    prev = s
                it += 1
                yield
            while q:                                              # wgmma.wait_group 0
                yield
            if prev is not None and bug != "acc_parity":
                release(prev)
            seen.append((r, c, t))
            yield

    def tma_engine():
        while True:
            if tma_q and rng.random() < 0.6:
                op = tma_q.pop(rng.randrange(min(len(tma_q), 4)))  # completions in any order
                kind, r, s, what = op
                if kind == "A":
                    smem_a[r][s] = what
                    full[r][s].complete_tx(2)
                elif kind == "W":
                    smem_w[r][s][0] = what
                    full[r][s].complete_tx(2)
                else:
                    for d in range(C):
                        smem_w[d][s][r] = what
                        full[d][s].complete_tx(1)
            yield

    def tensor_core(r, c):
        q = tc_q[(r, c)]
        while True:
            if q and rng.random() < 0.5:
                s, (t, kb) = q[0]
                assert smem_a[r][s] == (t, kb, r), f"CTA {r} wgmma for {(t, kb)} found A {smem_a[r][s]} in stage {s}"
                assert smem_w[r][s] == [(t, kb)] * C, f"CTA {r} wgmma for {(t, kb)} found W {smem_w[r][s]} in stage {s}"
                q.popleft()
            yield

    roles = {f"p{r}": producer(r) for r in range(C)}
    roles.update({f"c{r}{c}": consumer(r, c) for r in range(C) for c in range(CONS)})
    engines = [tma_engine()] + [tensor_core(r, c) for r in range(C) for c in range(CONS)]
    steps = 0
    while roles:
        steps += 1
        if steps > max_steps:
            raise TimeoutError(f"deadlock: waiting roles {sorted(roles)}")
        for e in engines:
            next(e)
        name = rng.choice(sorted(roles))
        for _ in range(rng.randint(1, 6)):
            try:
                next(roles[name])
            except StopIteration:
                del roles[name]
                break
    assert sorted(seen) == sorted((r, c, t) for r in range(C) for c in range(CONS) for t in range(tiles))


@pytest.mark.parametrize("tiles,num_kb", [(1, 1), (1, 12), (2, 3), (5, 12), (7, 5), (6, 48)])
def test_persistent_pipeline_indices_are_consistent(tiles, num_kb):
    for seed in range(12):
        simulate(tiles, num_kb, seed)


@pytest.mark.parametrize("bug", ["producer_parity", "acc_parity"])
def test_model_catches_a_wrong_parity(bug):
    """producer_parity: the producer waits on the wrong phase of `empty`; acc_parity: a consumer releases a stage while
    its in-flight wgmma group still reads it."""
    caught = 0
    for seed in range(10):
        try:
            simulate(5, 12, seed, bug=bug, max_steps=40_000)
        except (AssertionError, TimeoutError):
            caught += 1
    assert caught == 10


@pytest.mark.parametrize("num_kb", [1, 5, 6, 12, 48])
def test_cta_pair_protocol_is_consistent(num_kb):
    for seed in range(15):
        simulate(3, num_kb, seed, cluster=2)


def test_cta_pair_model_catches_a_wrong_parity():
    caught = 0
    for seed in range(10):
        try:
            simulate(3, 24, seed, cluster=2, bug="producer_parity", max_steps=30_000)
        except (AssertionError, TimeoutError):
            caught += 1
    assert caught == 10


def test_cluster_model_catches_a_release_to_the_local_cta_only():
    """If consumers released a stage only in their own CTA, the peer's multicast could overwrite W under a wgmma."""
    caught = 0
    for seed in range(10):
        try:
            simulate(3, 24, seed, cluster=2, bug="local_release", max_steps=60_000)
        except (AssertionError, TimeoutError):
            caught += 1
    assert caught == 10
