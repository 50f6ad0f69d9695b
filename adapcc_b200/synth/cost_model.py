"""alpha-beta cost model over the profiler's measured latency / bandwidth matrices.

Units follow the profile dump (/root/reference/csrc/profile.cu:336-357): latency in microseconds,
bandwidth in GB/s. The model feeds (a) the tree synthesizers and (b) the per-message algorithm
choice (one-shot / two-shot / NVLS / tree) — "variant picked per chunk from the profiler's measured
link bandwidth" (BASELINE.json north star).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

from ..strategy.trees import Strategy, Tree

GB = 1e9


@dataclass
class LinkModel:
    """α–β description of a job's links: ``alpha(i, j)`` seconds and ``bw_gbs[i][j]`` GB/s per ordered pair, built from
    the profile's latency / bandwidth matrices (or uniform for what-if runs)."""

    alpha_us: List[List[float]]     # [src][dst] one-way latency, us
    bw_gbs: List[List[float]]       # [src][dst] bandwidth, GB/s

    @classmethod
    def uniform(cls, world: int, alpha_us: float = 2.0, bw_gbs: float = 700.0) -> "LinkModel":
        return cls([[0.0 if i == j else alpha_us for j in range(world)] for i in range(world)],
                   [[0.0 if i == j else bw_gbs for j in range(world)] for i in range(world)])

    @property
    def world(self) -> int:
        return len(self.bw_gbs)

    def beta(self, i: int, j: int) -> float:
        """seconds per byte on i -> j (inf when unmeasured)."""
        b = self.bw_gbs[i][j]
        return 1.0 / (b * GB) if b > 0 else float("inf")

    def alpha(self, i: int, j: int) -> float:
        return self.alpha_us[i][j] * 1e-6

    def mean_alpha(self, ranks: Optional[Sequence[int]] = None) -> float:
        rs = list(range(self.world)) if ranks is None else list(ranks)
        v = [self.alpha(i, j) for i in rs for j in rs if i != j and self.bw_gbs[i][j] > 0]
        return sum(v) / len(v) if v else 2e-6

    def min_bw(self, ranks: Optional[Sequence[int]] = None) -> float:
        rs = list(range(self.world)) if ranks is None else list(ranks)
        v = [self.bw_gbs[i][j] for i in rs for j in rs if i != j and self.bw_gbs[i][j] > 0]
        return min(v) if v else 1.0

    def is_uniform(self, tol: float = 0.25) -> bool:
        v = [self.bw_gbs[i][j] for i in range(self.world) for j in range(self.world)
             if i != j and self.bw_gbs[i][j] > 0]
        return bool(v) and (max(v) - min(v)) <= tol * max(v)


# One hop of the strategy-tree kernel costs more than a link latency: the parent polls the child's flag over NVLink
# (a round trip), then pulls; measured 44 us for a one-chunk 6-hop all-reduce on 8 B200 GPUs -> ~3.5 alpha per hop.
TREE_HOP_ALPHAS = 3.5
# The FIRST chunk of a lane crosses every hop at the rate of ONE CTA pulling over NVLink (512 threads x 16-byte loads,
# latency-bound), not at the link rate; later chunks overlap across the kernel's lanes and stream at a fraction of the link
# rate (flag polling and the staging passes share the ports). Both fitted on 8-GPU B200 measurements of the kernel with
# 3 trees (tests/golden/sweep_8xB200_r2.json) and 4 trees: every size 64 KB - 1 GiB within +-32 %.
TREE_LANE_GBS = 30.0
TREE_STREAM_EFF = 0.72


def tree_time(tree: Tree, lm: LinkModel, slice_bytes: float, chunk_bytes: float, bcast: bool = True,
              ingress_share: Optional[Dict[int, float]] = None) -> float:
    """Pipelined completion time of one reduction(+broadcast) tree over its slice.

    Per chunk a parent pulls from all its children through ONE ingress port, so its step time is
    alpha + sum_children chunk*beta; the pipeline runs at the slowest node's step time and fills in
    depth steps (reduce up, broadcast down)."""
    if not tree.nodes or slice_bytes <= 0:
        return 0.0
    chunk = max(16.0, min(chunk_bytes, slice_bytes))
    n_chunks = max(1.0, slice_bytes / chunk)
    step_max = 0.0
    lane_beta = 1.0 / (TREE_LANE_GBS * GB)

    def step(x: int, lat: float = 1.0) -> float:
        kids = tree.kids(x)
        if not kids:
            return 0.0
        share = (ingress_share or {}).get(x, 1.0)
        return lat * max(lm.alpha(c, x) for c in kids) + sum(chunk * lm.beta(c, x) for c in kids) * share

    def fill(x: int) -> float:
        # the FIRST chunk pays the full flag round trip at every level; later chunks overlap it across the CTA lanes,
        # so the steady-state step below keeps one link latency
        kids = tree.kids(x)
        if not kids:
            return 0.0
        slow = max(1.0, max(lm.beta(c, x) for c in kids) / lane_beta)        # a slower-than-a-lane link bounds the hop
        return (TREE_HOP_ALPHAS * max(lm.alpha(c, x) for c in kids) + len(kids) * chunk * lane_beta * slow
                + max(fill(c) for c in kids))

    for x in tree.nodes:
        step_max = max(step_max, step(x))
    t = fill(tree.root) + (n_chunks - 1) * step_max / TREE_STREAM_EFF
    if bcast:
        # same edges backwards; a child's pull is one flow on its own ingress
        def bfill(x: int) -> float:
            kids = tree.kids(x)
            if not kids:
                return 0.0
            return max(TREE_HOP_ALPHAS * lm.alpha(x, c) + chunk * max(lane_beta, lm.beta(x, c)) + bfill(c) for c in kids)
        egress = max((len(tree.kids(x)) for x in tree.nodes), default=1)
        bstep = max((lm.alpha(x, c) + chunk * lm.beta(x, c) * max(1, len(tree.kids(x)))
                     for x in tree.nodes for c in tree.kids(x)), default=0.0)
        t = max(t, fill(tree.root)) + bfill(tree.root) + max(0.0, (n_chunks - 1) * (bstep - step_max) / TREE_STREAM_EFF)
        _ = egress
    return t


def strategy_time(strategy: Strategy, lm: LinkModel, total_bytes: float, chunk_bytes: float,
                  bcast: bool = True) -> float:
    """Trees run concurrently on disjoint slices; nodes that are parents in several trees share
    their ingress port between them."""
    nt = len(strategy.trees)
    if nt == 0:
        return float("inf")
    load: Dict[int, int] = {}
    for t in strategy.trees:
        for x in t.nodes:
            if t.kids(x):
                load[x] = load.get(x, 0) + 1
    per = total_bytes / nt
    # + one kernel launch; user tensors are staged through the window on the way in and out
    return LAUNCH_US * 1e-6 + max(tree_time(t, lm, per, chunk_bytes, bcast, {x: float(k) for x, k in load.items()})
                                  for t in strategy.trees)


# Constants of the direct-algorithm model, calibrated on an 8-GPU B200 sweep (not yet re-fitted for H100)
# (tests/golden/allreduce_sweep_8xB200_final.json; tests/test_synth.py checks the model against that file):
LAUNCH_US = 5.2            # fixed cost of one collective kernel (launch, first touch, last-block bookkeeping)
BARRIER_ALPHAS = 1.5       # one per-CTA flag barrier = a peer store + a local poll ~ 1.5 link latencies
STAGE_PASS_US = 3.3        # latency of one staging pass (stage-in or stage-out) over the window
STAGE_GBS = 1640.0         # payload rate of a staging pass that is NOT overlapped with the link phase
STAGE_PIPELINED_GBS = 4200.0   # ... of the pipelined staged two-shot (stager CTAs overlap the link CTAs)
PIPELINE_MIN_BYTES = 32 << 20
TWO_SHOT_LINK_EFF = 0.9    # pull + push share the NVLink ports: 625 of the profiled 700 GB/s
NVLS_LINK_EFF = 0.77       # multimem.ld_reduce + multimem.st: 540 GB/s per GPU at 1 GiB


def direct_times(lm: LinkModel, nbytes: float, ranks: Optional[Sequence[int]] = None,
                 nvls: bool = True, nvls_bw_gbs: Optional[float] = None, zero_copy: bool = False) -> Dict[str, float]:
    """Estimates (seconds) for the switch-topology algorithms on a message of ``nbytes`` wire bytes.

    ``zero_copy``: the tensor lives in the symmetric heap, so the two-shot / NVLS kernels skip both staging passes
    (a one-shot is always staged: peers read the window while the result is produced)."""
    rs = list(range(lm.world)) if ranks is None else list(ranks)
    n = max(2, len(rs))
    a = lm.mean_alpha(rs)
    bw = lm.min_bw(rs) * GB
    fixed = LAUNCH_US * 1e-6 + 2 * BARRIER_ALPHAS * a

    def stage(passes: int, gbs: float = STAGE_GBS) -> float:
        return passes * (STAGE_PASS_US * 1e-6 + nbytes / (gbs * GB))

    two_shot_stage = 0.0 if zero_copy else stage(
        2, STAGE_PIPELINED_GBS if nbytes >= PIPELINE_MIN_BYTES else STAGE_GBS)
    out = {
        # stage-in, barrier, every rank pulls the other n-1 windows and writes the result directly, barrier
        "one_shot": fixed + stage(1) + (n - 1) * nbytes / bw,
        # [stage-in] barrier, pull my slice from n-1 peers, push it to n-1 peers, barrier [stage-out]
        "two_shot": fixed + two_shot_stage + 2 * (n - 1) / n * nbytes / (TWO_SHOT_LINK_EFF * bw),
    }
    if nvls:
        mb = (nvls_bw_gbs * GB) if nvls_bw_gbs else NVLS_LINK_EFF * bw
        # the switch reduces on the way in (S/n per rank) and replicates on the way out (S)
        out["nvls"] = fixed + (0.0 if zero_copy else stage(2)) + (1.0 + 1.0 / n) * nbytes / mb
    return out


def pick_algorithm(lm: LinkModel, nbytes: float, ranks=None, nvls: bool = True,
                   strategy: Optional[Strategy] = None, chunk_bytes: float = 1 << 20, zero_copy: bool = False) -> str:
    t = direct_times(lm, nbytes, ranks, nvls, zero_copy=zero_copy)
    if zero_copy:
        t.pop("one_shot", None)             # in place a one-shot would race with the peers' reads
    if strategy is not None:
        t["tree"] = strategy_time(strategy, lm, nbytes, chunk_bytes)
    return min(t, key=t.get)


def crossover_bytes(lm: LinkModel, a: str, b: str, ranks=None, nvls: bool = True) -> int:
    """Smallest power-of-two message size where algorithm ``b`` beats ``a``."""
    for p in range(8, 34):
        t = direct_times(lm, float(1 << p), ranks, nvls)
        if a in t and b in t and t[b] < t[a]:
            return 1 << p
    return 1 << 34


def best_chunk_bytes(strategy: Strategy, lm: LinkModel, total_bytes: float,
                     candidates=(16 << 10, 64 << 10, 256 << 10, 1 << 20, 4 << 20)) -> int:
    return min(candidates, key=lambda c: strategy_time(strategy, lm, total_bytes, c))
