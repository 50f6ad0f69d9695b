"""Control plane + data-plane front end (``CudaCommu``).

API and workflow parity with /root/reference/commu.py:40-435:

* primitive ids, ``init_threads`` / ``exit_threads`` workflow DETECT -> PROFILE -> SYNTHESIS ->
  transmission-context setup, ``all_reduce`` / ``reduce`` / ``boardcast``, ``update_relay``,
  ``cuda_allreduce_hook`` (torch DDP communication hook), ``clear``;
* rank 0 hosts the gRPC coordinator, every rank runs a controller thread that heartbeats once per
  step and drives relays.

What changed (GPU-first):

* a collective is ONE asynchronous kernel launch on a CUDA stream (no background pthread blocked
  inside ``initThreads``, no ``time.sleep(3)`` hand-shake, no blocking ``ctypes`` call);
* the DDP hook runs the collective on a high-priority side stream and returns a real CUDA future,
  so gradient communication overlaps the rest of backward (the reference blocks the autograd
  thread, commu.py:385-435); gradients are averaged over the active ranks inside the kernel
  (the reference returns the unscaled sum);
* the algorithm is chosen per message from the profiled alpha/beta (one-shot, two-shot, NVLS or the
  strategy's trees); fp32 buckets can travel as bf16 on the wire, cast fused into the kernel;
* CPU tensors (``--backend gloo``) run the same strategy through the reference executor.
"""
from __future__ import annotations

import json
import os
import threading
import time
from queue import Empty, Queue
from typing import List, Optional

from . import topology as topo
from .constants import (ALLGATHER, ALLREDUCE, ALLTOALL, BOARDCAST, DETECT, PROFILE, REDUCE,  # noqa: F401
                        REDUCESCATTER, RELAY_BYPASS, RELAY_FORWARD)
from .coord import Controller, Coordinator, Hooker, make_server
from .dispatcher import Dispatcher
from .strategy import Strategy, default_chunk_bytes
from .synth import LinkModel, Synthesizer, crossover_bytes

__all__ = ["CudaCommu", "ALLREDUCE", "REDUCE", "BOARDCAST", "ALLGATHER", "ALLTOALL", "REDUCESCATTER", "DETECT",
           "PROFILE"]

_DATA_PRIMS = (ALLREDUCE, REDUCE, BOARDCAST, ALLGATHER, ALLTOALL, REDUCESCATTER)


def _arg(args, name, default):
    v = getattr(args, name, None)
    return default if v is None else v


class CudaCommu:
    """The control plane of one rank: workflow stages (DETECT / PROFILE → synthesis → data-plane context), the
    collectives' Python entry points, the DDP communication hook, the controller thread (heartbeat + relay duty) and
    the coordinator clients — /root/reference/commu.py:37-435, on VMM symmetric memory and in-kernel NVLink
    transfers instead of cudaIpc staging threads."""

    def __init__(self, args, dylib, local_rank, world_rank, world_size):
        self.args = args
        self.dylib = dylib                      # kept for signature parity; ctypes handle or None
        self.local_rank, self.world_rank, self.world_size = local_rank, world_rank, world_size
        self.port = int(_arg(args, "port", 5000))
        self.init_count = 0
        self.work_dir = os.path.abspath(_arg(args, "work_dir", os.getcwd()))
        self.topo_dir = os.path.join(self.work_dir, "topology")
        os.makedirs(self.topo_dir, exist_ok=True)

        # ---- ip table (one line per rank; generated for single-node jobs) -----------------
        self.ip_table_file = os.path.join(self.topo_dir, "ip_table.txt")
        if os.path.exists(self.ip_table_file):
            self.ip_table = topo.read_ip_table(self.ip_table_file)
        else:
            self.ip_table = []
        if len(self.ip_table) != world_size:
            self.ip_table = [os.environ.get("ADAPCC_NODE_IP", "127.0.0.1")] * world_size
            if world_rank == 0:
                topo.write_ip_table(self.ip_table_file, self.ip_table)
        self.dispatcher = Dispatcher(self.ip_table)
        self.single_server = len(set(self.ip_table)) == 1
        # multi-server jobs: one NVLink domain (symmetric-memory context) per server + an inter-server leg
        self.node_ranks = [r for r, ip in enumerate(self.ip_table) if ip == self.ip_table[world_rank]]
        self.local_roots = topo.local_rank0_list(self.ip_table)
        self.node_index = self.local_roots.index(self.node_ranks[0])
        self._inter_group = None

        # ---- data-plane policy -----------------------------------------------------------------
        self.algo = _arg(args, "algo", os.environ.get("ADAPCC_ALGO", "auto"))
        self.wire_dtype = _arg(args, "wire_dtype", os.environ.get("ADAPCC_WIRE_DTYPE"))   # e.g. "bfloat16"
        self.reduce_op = _arg(args, "reduce_op", "avg")       # DDP hook; primitives default to "sum"
        self.relay_mode = RELAY_BYPASS if str(_arg(args, "relay_mode", "forward")) in ("bypass", "1") else RELAY_FORWARD
        self.is_bsp = bool(_arg(args, "bsp", True))
        if not self.is_bsp and world_rank == 0:
            # the reference's non-BSP join (a late rank re-enters mid-step, /root/reference/commu.py:427-431) marks the
            # rank active in ITS process only, so the ranks disagree on the active set; relays stay relays for the step here
            print("[adapcc] bsp=False: the non-BSP late join is not implemented; late ranks relay for the whole step (BSP)",
                  flush=True)
        self.relay_control = bool(_arg(args, "relay_control", True)) and world_size > 1
        self.staging_bytes = int(_arg(args, "staging_mb", os.environ.get("ADAPCC_STAGING_MB", 256))) << 20
        self.heap_bytes = int(_arg(args, "heap_mb", os.environ.get("ADAPCC_HEAP_MB", 0))) << 20
        self.verbose = bool(int(os.environ.get("ADAPCC_VERBOSE", "0")))
        self.nvtx = bool(int(os.environ.get("ADAPCC_NVTX", "0")))         # NVTX range per collective

        self.active_gpus = list(range(world_size))
        self.chunk_bytes: Optional[int] = None
        self.strategy: Optional[Strategy] = None
        self.link_model: Optional[LinkModel] = None
        self.synthesizer = Synthesizer(strategy_file=_arg(args, "strategy_file", None), ip_table=self.ip_table,
                                       parallel_degree=int(_arg(args, "parallel_degree", 4)),
                                       policy=_arg(args, "policy", "par-trees"),
                                       intra_policy=_arg(args, "intra_policy", "binary" if self.single_server else "chain"))
        self.native = None                      # NativeComm, created on first GPU context
        self._open_prims = set()
        self._comm_stream = None
        self._relay_stream = None

        # ---- coordinator (rank 0) + clients ------------------------------------------------------
        self.coordinator: Optional[Coordinator] = None
        self.server = None
        self.coordinator_port = int(_arg(args, "coordinator_port", os.environ.get("ADAPCC_COORD_PORT", 50051)))
        self.controller: Optional[Controller] = None
        self.hooker: Optional[Hooker] = None
        self._coord_proc = None
        if self.relay_control:
            if world_rank == 0:
                # The coordinator answers two blocking RPCs per rank per step. Hosted as a THREAD of rank 0 (the
                # reference's layout, /root/reference/commu.py:80-84) its handlers compete for rank 0's GIL with a
                # launch-bound training loop: one hand-off per 5 ms switch interval, i.e. several ms per negotiation,
                # about a training step's length. Default on CUDA jobs: a separate
                # PROCESS (same module, same protocol); `coordinator_process=False` keeps the in-process object
                # (tests and tools that read `communicator.coordinator` directly).
                as_process = bool(_arg(args, "coordinator_process",
                                       os.environ.get("ADAPCC_COORD_PROCESS", "1" if self._use_cuda() else "0") == "1"))
                if as_process and world_size > 1:
                    self._spawn_coordinator(args, world_size)
                if self._coord_proc is None:
                    self.coordinator = Coordinator(self.ip_table[0], self.coordinator_port, world_size,
                                                   relay_threshold=float(_arg(args, "relay_threshold", 0.1)),
                                                   fault_tolerant_time=float(_arg(args, "fault_tolerant_time", 10.0)))
                    self.server = make_server(self.coordinator)
                    self.server.start()
                    import sys as _sys
                    _sys.setswitchinterval(min(_sys.getswitchinterval(), 0.0005))   # faster GIL hand-off to the handlers
            rpc_timeout = float(_arg(args, "fault_tolerant_time", 10.0)) * 2 + float(_arg(args, "relay_threshold", 0.1)) + 20
            self.controller = Controller(self.ip_table[0], self.coordinator_port, timeout=rpc_timeout)
            self.hooker = Hooker(self.ip_table[0], self.coordinator_port, timeout=rpc_timeout)

        # ---- controller agent ---------------------------------------------------------------------
        self.step_queue: Queue = Queue()
        self.relay_signal_queue: Queue = Queue()
        self.bsp_queue: Queue = Queue()
        self.relay_results: List = []
        self.current_step = 0
        self.local_hook_num = 0
        self.bucket_info: List = []             # (numel, chunk_bytes, dtype) per bucket, recorded at step 1
        self.relay_buffer: List = []
        self.accumulated_bw = 0.0
        self.fault_worker_list: List[int] = []
        self.stats = {"hook_rpc_s": [], "relay_steps": 0, "ops": 0}
        self._lock = threading.Lock()
        self.controller_thread = threading.Thread(target=self._controller_thread_func, daemon=True,
                                                  name=f"adapcc-controller-{world_rank}")
        self.controller_thread.start()

    # ==========================================================================================
    # helpers
    # ==========================================================================================
    def _log(self, msg: str) -> None:
        if self.verbose:
            print(f"[Rank {self.world_rank}]{msg}", flush=True)

    def _barrier(self) -> None:
        import torch.distributed as dist

        if dist.is_available() and dist.is_initialized():
            dist.barrier()
        elif self.native is not None:
            self.native.host_barrier()

    def _spawn_coordinator(self, args, world_size: int) -> None:
        import subprocess
        import sys as _sys

        cmd = [_sys.executable, "-m", "adapcc_b200.coord.server", "--ip", str(self.ip_table[0]),
               "--port", str(self.coordinator_port), "--world_size", str(world_size),
               "--relay_threshold", str(float(_arg(args, "relay_threshold", 0.1))),
               "--fault_tolerant_time", str(float(_arg(args, "fault_tolerant_time", 10.0))),
               "--parent", str(os.getpid())]
        env = dict(os.environ)
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        env["PYTHONPATH"] = root + os.pathsep + env.get("PYTHONPATH", "")
        env["CUDA_VISIBLE_DEVICES"] = ""                    # the coordinator never touches a GPU
        try:
            proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, env=env)
            line = proc.stdout.readline()                   # "coordinator ready" once the port is bound
            if "ready" in line and proc.poll() is None:
                self._coord_proc = proc
                return
            proc.kill()
        except OSError as e:
            self._log(f"coordinator process could not start ({e}); hosting it in-process")

    def _use_cuda(self) -> bool:
        import torch

        return torch.cuda.is_available() and _arg(self.args, "backend", "nccl") != "gloo"

    def _ensure_native(self):
        if self.native is None:
            from .runtime.native import NativeComm
            from .runtime.rendezvous import unique_name

            name = unique_name(f"adapcc-{self.port}-{self.init_count}")
            if self.single_server:
                self.native = NativeComm(name, self.world_rank, self.world_size, self.local_rank,
                                         staging_bytes=self.staging_bytes, heap_bytes=self.heap_bytes)
            else:   # one context per server: ranks are numbered inside the server
                self.native = NativeComm(f"{name}-n{self.node_index}", self.node_ranks.index(self.world_rank),
                                         len(self.node_ranks), self.local_rank, staging_bytes=self.staging_bytes,
                                         heap_bytes=self.heap_bytes)
            self.native.set_tunable("relay_mode", self.relay_mode)
            self._apply_tunables()
        return self.native

    def _streams(self):
        import torch

        if self._comm_stream is None:
            self._comm_stream = torch.cuda.Stream(device=self.local_rank, priority=-1)
            self._relay_stream = torch.cuda.Stream(device=self.local_rank, priority=-1)
        return self._comm_stream, self._relay_stream

    def _tunables_path(self) -> str:
        return os.path.join(self.topo_dir, "tunables.json")

    def _apply_tunables(self) -> None:
        """Per-message algorithm thresholds derived from the last profile (rank 0 wrote them)."""
        if self.native is None or not os.path.exists(self._tunables_path()):
            return
        try:
            with open(self._tunables_path()) as f:
                t = json.load(f)
            for k in ("one_shot_max_bytes", "nvls_min_bytes", "max_blocks", "tree_blocks", "nvls_min_ranks", "ll_max_bytes"):
                if k in t:
                    self.native.set_tunable(k, int(t[k]))
        except (OSError, ValueError) as e:
            self._log(f"ignoring unreadable tunables: {e}")

    def _load_strategy(self) -> None:
        path = _arg(self.args, "strategy_file", None)
        if path and os.path.exists(path):
            self.strategy = Strategy.from_file(path, self.world_size)
            from .synth.plan import AlgoPlan
            self.plan = AlgoPlan.from_attrs(self.strategy.attrs)      # size bands written by the synthesizer
            if self.chunk_bytes is None and "chunk" in self.strategy.attrs:
                try:
                    self.chunk_bytes = int(self.strategy.attrs["chunk"])
                except ValueError:
                    pass
        elif self.strategy is None:
            from .strategy import make_strategy

            self.strategy = make_strategy(self.world_size, min(int(_arg(self.args, "parallel_degree", 4)),
                                                               self.world_size), "binary", self.ip_table)

    # ==========================================================================================
    # controller thread (relay driver + heartbeat)
    # ==========================================================================================
    def _controller_thread_func(self):
        while True:
            step = self.step_queue.get()
            if step == -1:
                break
            if not self.relay_control:
                continue
            try:
                active, status = self.controller.send_relay_request(step, self.world_rank)
            except Exception as e:  # noqa: BLE001  (coordinator gone: stop heartbeating)
                self._log(f"controller RPC failed: {e}")
                return
            if status == 0:
                # heartbeat deadline missed by somebody: the survivors ARE the new world. The reference prints and lets
                # the controller thread die (/root/reference/commu.py:151-157); here the thread keeps serving, the
                # active set is re-formed from the survivors and the coordinator stops waiting for the dead ranks.
                self.fault_worker_list = sorted(set(self.fault_worker_list) |
                                                {w for w in range(self.world_size) if w not in active})
                print(f"Fault occurs: rank {self.world_rank} alive; missing {self.fault_worker_list}", flush=True)
                self.active_gpus = sorted(a for a in active if a not in self.fault_worker_list)
                self.bsp_queue.put(step)
                continue
            self.active_gpus = sorted(active)
            self._log(f"Controller active: {active}")
            if step <= 1:
                continue
            if self.world_rank not in active:
                self.stats["relay_steps"] += 1
                self._run_as_relay(step, sorted(active))
                self.bsp_queue.put(step)

    def _run_as_relay(self, step: int, active: List[int]) -> None:
        """This rank missed the step's deadline: keep the data plane going for the others."""
        if self.native is None or not self.bucket_info:
            return
        import torch

        _, relay_stream = self._streams()
        if not self.single_server:
            # hierarchical path: every rank of a server takes part in the local legs, so a relay joins
            # the collective with a scratch buffer (it contributes nothing and discards the result)
            with torch.cuda.device(self.local_rank), torch.cuda.stream(relay_stream):
                for i, (numel, chunk_bytes, dtype) in enumerate(self.bucket_info):
                    if self.relay_buffer[i] is None:
                        self.relay_buffer[i] = torch.zeros(numel, dtype=dtype, device=f"cuda:{self.local_rank}")
                    self._collective(ALLREDUCE, self.relay_buffer[i], numel, chunk_bytes, active, self.reduce_op)
                    self.relay_signal_queue.put(step)
            relay_stream.synchronize()
            return
        with torch.cuda.device(self.local_rank), torch.cuda.stream(relay_stream):
            tree = [self._resolve_algo(n, dt, active) == "tree" for n, _, dt in self.bucket_info]
            wires = {self._wire_for(dt) or str(dt).replace("torch.", "") for _, _, dt in self.bucket_info}
            if all(tree) and self.relay_mode == RELAY_FORWARD and len(wires) == 1:
                # one persistent kernel forwards the chunks of every bucket of this step
                self.native.tree_relay_persistent([n for n, _, _ in self.bucket_info],
                                                  [c for _, c, _ in self.bucket_info], wire=wires.pop(),
                                                  op=self.reduce_op, active=active)
                for _ in self.bucket_info:
                    self.relay_signal_queue.put(step)
            else:
                for i, (numel, chunk_bytes, dtype) in enumerate(self.bucket_info):
                    if tree[i] and self.relay_mode == RELAY_FORWARD:
                        buf = self.relay_buffer[i]
                        self.native.tree_collective(ALLREDUCE, buf[:numel], op=self.reduce_op,
                                                    wire=self._wire_for(dtype), chunk_bytes=chunk_bytes, active=active)
                        self.relay_results.append(buf)
                    else:
                        self.native.skip_op()       # direct algorithms never route through a relay
                    self.relay_signal_queue.put(step)
        relay_stream.synchronize()

    # ==========================================================================================
    # workflow
    # ==========================================================================================
    def clear(self, keep_native: bool = False):
        """stop the controller and the grpc server (collective: a slower rank may still be
        negotiating its last step, so nobody tears the coordinator down before everyone arrived).
        ``keep_native``: hand the native context (symmetric buffers, heap — DDP buckets may live in it) back to
        the caller instead of destroying it; ``AdapCC.reconstruct_topology`` passes it to the next communicator."""
        if self.native is not None:
            import torch

            torch.cuda.synchronize(self.local_rank)
        self._barrier()
        self.update_relay(-1)
        if self.controller_thread.is_alive():
            self.controller_thread.join(timeout=5)
        for c in (self.controller, self.hooker):
            if c is not None:
                c.close()
        if self.server is not None:
            self.server.stop(1)
            self.server = None
        if getattr(self, "_coord_proc", None) is not None:
            self._coord_proc.terminate()
            try:
                self._coord_proc.wait(timeout=3)
            except Exception:  # noqa: BLE001
                self._coord_proc.kill()
            self._coord_proc = None
        kept = None
        if self.native is not None:
            self._barrier()
            if keep_native:
                kept = self.native
            else:
                self.native.close()
            self.native = None
        self._cleared = True
        return kept

    def adopt_native(self, native) -> None:
        """Reuse a live native context from a previous communicator (same world / device / buffer sizes): the
        strategy and the tunables of THIS communicator are (re)applied when its primitive is set up."""
        if native is None:
            return
        ok = (native.world == (self.world_size if self.single_server else len(self.node_ranks))
              and native.staging_bytes >= self.staging_bytes and native.heap_bytes >= self.heap_bytes)
        if not ok:                       # different shape: build a fresh one lazily, release the old one now
            native.close()
            return
        self.native = native
        self.native.set_tunable("relay_mode", self.relay_mode)
        self._apply_tunables()

    def _live(self):
        """The communicator that replaced this one (``reconstruct_topology``), following the chain."""
        c = self
        while getattr(c, "_cleared", False) and getattr(c, "_successor", None) is not None:
            c = c._successor
        return c

    def update_relay(self, step):
        """called once per iteration before forward: heartbeat + (for relays) data-plane duty"""
        if getattr(self, "_cleared", False) and step >= 0:
            # a closure that captured the communicator before reconstruct_topology keeps calling the cleared one:
            # forward to the live communicator, like cuda_allreduce_hook does (otherwise relay control, straggler
            # handling and the heartbeat are silently off for the rest of the run)
            live = self._live()
            if live is not self:
                return live.update_relay(step)
        self.step_queue.put(step)
        self.current_step = step
        self.local_hook_num = 0

    def init_threads(self, prim):
        """Enter a workflow stage or build a data-plane context: DETECT (native topology discovery), PROFILE (link
        micro-benchmarks), or a collective primitive (load the strategy, create the native context).
        Reference: /root/reference/commu.py:301-319."""
        if prim == DETECT:
            self._detect()
        elif prim == PROFILE:
            self._profile()
        elif prim in _DATA_PRIMS:
            self._load_strategy()
            if self._use_cuda():
                t0 = time.time()
                n = self._ensure_native()
                if self.strategy is not None:
                    n.load_strategy(self.strategy.to_xml())
                self._log("transmission context setup time=%6.2f(ms)" % ((time.time() - t0) * 1e3))
            self._open_prims.add(prim)
        else:
            raise NotImplementedError(f"primitive {prim} is not a known primitive id (0-7, see adapcc_b200/constants.py)")
        self.init_count += 1

    def exit_threads(self, prim):
        """Leave a stage: DETECT gathers the per-server files into the logical graph, PROFILE gathers the link
        records and synthesises the strategy (rank 0) and distributes it, a primitive closes its context.
        Reference: /root/reference/commu.py:321-358."""
        if prim == DETECT:
            if self.local_rank == 0:
                self.dispatcher.dispatch_detected_topo(os.path.join(self.topo_dir, "topo_detect*"), self.topo_dir)
            self._barrier()
            if self.local_rank == 0:
                self._gather_detect_graph()
            self._barrier()
        elif prim == PROFILE:
            if self.local_rank == 0:
                self.dispatcher.send_profiled_topo(os.path.join(self.topo_dir, "topo_profile*"), self.topo_dir)
            self._barrier()
            if self.world_rank == 0:
                lc_graph, bw_graph = self._gather_topo_profile()
                self._synthesis_strategy(lc_graph, bw_graph)
                sf = _arg(self.args, "strategy_file", None)
                if sf:
                    self.dispatcher.dispatch_strategy(sf, os.path.dirname(os.path.abspath(sf)))
            self._barrier()
            self._apply_tunables()
        elif prim in _DATA_PRIMS:
            self._open_prims.discard(prim)
            if self.native is not None:
                import torch

                torch.cuda.synchronize(self.local_rank)

    # -- DETECT -----------------------------------------------------------------------------------
    def _detect(self):
        if self.local_rank != 0:
            return
        path = os.path.join(self.topo_dir, f"topo_detect_{self.world_rank}.xml")
        xml = None
        if self._use_cuda():
            import ctypes

            from .runtime.native import last_error, load_library

            lib = load_library()
            buf = ctypes.create_string_buffer(1 << 20)
            n = lib.adapcc_detect_topology(self.world_rank, buf, len(buf))
            if n < 0:
                raise RuntimeError(f"topology detection failed: {last_error()}")
            xml = buf.value.decode()
        else:
            g = sum(1 for ip in self.ip_table if ip == self.ip_table[self.world_rank])
            gpus = "".join(f'<gpu id="{i}"/>' for i in range(g))
            xml = f'<topology first_rank="{self.world_rank}" gpus="{g}" nvml="0"><cpu numa="0"><pcie root="cpu">{gpus}</pcie></cpu></topology>\n'
        with open(path, "w") as f:
            f.write(xml)

    def _gather_detect_graph(self):
        from .strategy import xmlio

        r0s = topo.local_rank0_list(self.ip_table)
        groups = topo.server_groups(self.ip_table)
        files = [os.path.join(self.topo_dir, f"topo_detect_{r}.xml") for r in r0s]
        graph = topo.build_logical_graph(files, [self.ip_table[r] for r in r0s], r0s,
                                         [len(groups[r]) for r in r0s])
        lg = _arg(self.args, "logical_graph", os.path.join(self.topo_dir, "logical_graph.xml"))
        os.makedirs(os.path.dirname(os.path.abspath(lg)), exist_ok=True)
        xmlio.dump_file(graph, lg)

    # -- PROFILE ----------------------------------------------------------------------------------
    def _profile(self):
        path = os.path.join(self.topo_dir, f"topo_profile_{self.world_rank}")
        w = self.world_size
        if self._use_cuda() and w > 1:
            import ctypes

            import torch

            from .runtime.native import last_error

            n = self._ensure_native()
            nw = n.world                               # ranks of this NVLink domain (== w on one server)
            F = ctypes.c_float * nw
            lat, rd, wr, nv = F(), F(), F(), ctypes.c_float(0)
            n.lib.adapcc_profile_links.argtypes = [ctypes.c_void_p, ctypes.c_ulonglong, ctypes.c_int, F, F, F,
                                                   ctypes.POINTER(ctypes.c_float), ctypes.c_void_p]
            probe = int(os.environ.get("ADAPCC_PROFILE_MB", 64)) << 20
            with torch.cuda.device(self.local_rank):
                rc = n.lib.adapcc_profile_links(n.handle, probe, 64, lat, rd, wr, ctypes.byref(nv),
                                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
            if rc != 0:
                raise RuntimeError(f"link profiling failed: {last_error()}")
            glat, grd, gwr = [0.0] * w, [0.0] * w, [0.0] * w
            members = list(range(w)) if self.single_server else self.node_ranks
            for j, g in enumerate(members):
                glat[g], grd[g], gwr[g] = lat[j], rd[j], wr[j]
            if not self.single_server:
                self._profile_inter_server(glat, grd)
            topo.write_profile(path, self.world_rank, w, glat, grd, gwr, float(nv.value))
        else:
            lat = [0.0 if d == self.world_rank else 50.0 for d in range(w)]
            bw = [0.0 if d == self.world_rank else 1.0 for d in range(w)]
            topo.write_profile(path, self.world_rank, w, lat, bw)

    def _profile_inter_server(self, lat_us, bw_gbs, nbytes: int = 16 << 20):
        """Inter-server probes between the local roots, N-1 rounds like the reference's
        MPI_Isend/Irecv rounds (/root/reference/csrc/profile.cu:220-334): in round i server s sends to
        server (s+i)%N and receives from (s-i)%N; bandwidth from one large message, latency from small
        ping-pongs. Only the local roots measure; their rows carry the server-to-server numbers."""
        import torch
        import torch.distributed as dist

        roots = self.local_roots
        N = len(roots)
        if self.world_rank not in roots or N < 2:
            return
        s = roots.index(self.world_rank)
        dev = torch.device("cuda", self.local_rank)
        big = torch.empty(nbytes // 4, device=dev)
        small = torch.zeros(16, device=dev)
        for i in range(1, N):
            dst, src = roots[(s + i) % N], roots[(s - i) % N]
            for buf, reps, kind in ((small, 20, "lat"), (big, 3, "bw")):
                for w in dist.batch_isend_irecv([dist.P2POp(dist.isend, buf, dst),
                                                 dist.P2POp(dist.irecv, torch.empty_like(buf), src)]):
                    w.wait()                        # warm-up: connection setup is not link latency
                torch.cuda.synchronize()
                t0 = time.time()
                for _ in range(reps):
                    ops = [dist.P2POp(dist.isend, buf, dst), dist.P2POp(dist.irecv, torch.empty_like(buf), src)]
                    for w in dist.batch_isend_irecv(ops):
                        w.wait()
                torch.cuda.synchronize()
                dt = (time.time() - t0) / reps
                if kind == "lat":
                    lat_us[dst] = dt * 1e6
                else:
                    bw_gbs[dst] = buf.numel() * 4 / dt / 1e9

    def _gather_topo_profile(self):
        files = [os.path.join(self.topo_dir, f"topo_profile_{r}") for r in range(self.world_size)]
        lc_graph, bw_graph, ext = topo.read_profiles(files, self.world_size)
        self.accumulated_bw = topo.accumulated_bandwidth(bw_graph)
        self._profile_ext = ext
        return lc_graph, bw_graph

    def _synthesis_strategy(self, lc_graph, bw_graph):
        self.synthesizer.set_ip_info(self.ip_table)
        self.synthesizer.set_parallel_degree(int(_arg(self.args, "parallel_degree", 4)))
        self.synthesizer.set_latency_graph(lc_graph)
        self.synthesizer.set_bandwidth_graph(bw_graph)
        self.chunk_bytes = self.synthesizer.generate_strategy("reduce")
        self.link_model = LinkModel(lc_graph, bw_graph)
        # The rent/buy rule keeps the reference's constants (100*8/1024 GB per step over 50 GB/s x world,
        # /root/reference/proto/rpc_server.py:41-42 — the reference computes the profiled sum too, commu.py:266-269, and
        # never hands it over): with the profiled NVSwitch bandwidth a collective costs so little that the leader would stop
        # waiting after ~0.2 ms and ordinary arrival jitter would turn healthy ranks into relays. Opt in with
        # args.rent_from_profile (in-process coordinator only).
        if self.coordinator is not None and self.accumulated_bw > 0 and bool(_arg(self.args, "rent_from_profile", False)):
            self.coordinator.set_traffic(self.coordinator.accumulated_size, self.accumulated_bw)
        ext = getattr(self, "_profile_ext", {"nvls": []})
        nvls = max(ext.get("nvls", [0.0]) or [0.0])
        # ---- the per-message algorithm plan: every variant scored over the size axis with the PROFILED alpha / beta /
        # NVLS bandwidth; the winners travel as size bands inside the strategy XML (all ranks execute the same
        # decision) and as thresholds for the native runtime's own policy (synth/plan.py) -------------------------------
        from .strategy.trees import Strategy as _Strategy
        from .synth.plan import build_plan
        path = _arg(self.args, "strategy_file", None)
        strat = None
        try:
            strat = _Strategy.from_file(path, self.world_size) if path and os.path.exists(path) else None
        except Exception as e:  # noqa: BLE001
            self._log(f"plan: cannot re-read the synthesised strategy ({e})")
        have_nvls = nvls > 0 or bool(self.native is not None and self.native.multicast)
        plan = build_plan(self.link_model, strat, nvls=have_nvls, nvls_bw_gbs=nvls or None,
                          ll=os.environ.get("ADAPCC_LL", "1") != "0" and self.world_size > 1)
        if strat is not None:
            strat.attrs.update(plan.to_attrs())
            strat.save(path, compact=True)
        tun = {
            "one_shot_max_bytes": min(max(crossover_bytes(self.link_model, "one_shot", "two_shot", nvls=False), 16 << 10),
                                      4 << 20),
            "nvls_bw_gbs": nvls,
            "p2p_bw_gbs": self.link_model.min_bw(),
            "alpha_us": self.link_model.mean_alpha() * 1e6,
            "bands": plan.to_attrs()["bands"], "bands_zc": plan.to_attrs()["bands_zc"],
        }
        tun.update(plan.tunables())
        if not self.link_model.is_uniform() or self.world_size <= 2:
            tun["nvls_min_ranks"] = 3 if self.world_size > 2 else 99      # 2 ranks: a two-shot moves fewer bytes
        with open(self._tunables_path(), "w") as f:
            json.dump(tun, f, indent=1)
        self._log(f"algorithm plan: staged [{tun['bands']}] zero-copy [{tun['bands_zc']}]")

    # ==========================================================================================
    # data plane
    # ==========================================================================================
    def _wire_for(self, dtype) -> Optional[str]:
        import torch

        if self.wire_dtype and dtype == torch.float32:
            return self.wire_dtype
        return None

    def _resolve_algo(self, numel, dtype, active, tensor=None, wire=None) -> str:
        """The data-plane variant for this message. Explicit request (``args.algo``) first; then the strategy's own
        ``algo=`` attribute; then the synthesizer's size bands (``bands`` / ``bands_zc`` of the strategy XML, built from
        the profile: synth/plan.py) — 'tree' there means the synthesised trees are executed hop by hop; without a plan
        the native runtime's threshold policy ('auto'). Multi-server strategies are always honoured as trees."""
        if self.algo != "auto":
            return self.algo
        if self.strategy is not None and self.strategy.attrs.get("algo") in ("tree", "one_shot", "two_shot", "nvls"):
            return self.strategy.attrs["algo"]
        if not self.single_server:
            return "tree"
        plan = getattr(self, "plan", None)
        if plan is None:
            return "auto"
        import torch

        esize = (getattr(torch, wire) if isinstance(wire, str) else dtype).itemsize      # per hook call: no tensor allocation
        n = self.native
        zero_copy = bool(tensor is not None and n is not None and wire is None and n.in_heap(tensor))
        return plan.pick(int(numel) * esize, zero_copy=zero_copy, all_active=len(active) == self.world_size,
                         nvls=bool(n is not None and n.multicast), ll=bool(n is not None and n.has_ll),
                         tree=self.strategy is not None)

    def _collective(self, prim, buffer, size, chunk_bytes, active_gpus, op, root=None):
        import torch

        size = int(buffer.numel() if size is None else size)
        active = sorted(set(self.active_gpus if active_gpus is None else [int(a) for a in active_gpus]))
        flat = buffer.view(-1)[:size] if size != buffer.numel() else buffer.view(-1)
        if chunk_bytes is None:
            chunk_bytes = self.chunk_bytes or default_chunk_bytes(size * buffer.element_size())
        self.stats["ops"] += 1
        self.stats["bytes"] = self.stats.get("bytes", 0) + size * buffer.element_size()
        if not buffer.is_cuda:
            from .strategy.cpu_executor import tree_collective_cpu

            if self.strategy is None:
                self._load_strategy()
            tree_collective_cpu(prim, flat, self.strategy, self.world_rank, self.world_size, active=active, op=op,
                                chunk_bytes=int(chunk_bytes), relay_mode=self.relay_mode)
            return buffer
        n = self._ensure_native()
        if not self.single_server:
            self._hierarchical(n, prim, flat, active, op, root)
            return buffer
        wire = self._wire_for(buffer.dtype)
        algo = self._resolve_algo(size, buffer.dtype, active, tensor=flat, wire=wire)
        if algo == "ll" and prim != ALLREDUCE:
            algo = "auto"
        if self.nvtx:
            torch.cuda.nvtx.range_push(f"adapcc.prim{prim}.{algo}.{size * buffer.element_size()}B")
        try:
            self._launch(n, prim, flat, algo, wire, chunk_bytes, active, op, root)
        finally:
            if self.nvtx:
                torch.cuda.nvtx.range_pop()
        return buffer

    def _inter_server_group(self):
        import torch.distributed as dist

        if self._inter_group is None:
            self._inter_group = dist.new_group(ranks=self.local_roots)     # collective over ALL ranks
        return self._inter_group

    def _hierarchical(self, n, prim, flat, active, op, root):
        """Multi-server data plane: every server is one NVLink domain handled by our kernels; the
        local roots meet over the inter-server fabric (torch.distributed / NCCL-IB):
            all-reduce = reduce to the local root -> inter-server all-reduce of the roots -> local
            broadcast;  reduce / broadcast analogously. The reference moves inter-server chunks with
            CUDA-aware MPI point-to-point (/root/reference/csrc/trans.cu:75-99); the strategy's
            cross-server tree edges collapse onto this two-level scheme."""
        import torch
        import torch.distributed as dist

        group = self._inter_server_group()
        me = self.world_rank
        my_local = self.node_ranks.index(me)
        all_local = list(range(len(self.node_ranks)))
        i_am_root = my_local == 0
        red = "max" if op == "max" else "sum"
        rop = dist.ReduceOp.MAX if red == "max" else dist.ReduceOp.SUM
        root = active[0] if root is None else root
        root_node_root = next(r0 for r0 in self.local_roots if self.ip_table[r0] == self.ip_table[root])

        def identity():
            return torch.zeros_like(flat) if red == "sum" else torch.full_like(flat, float("-inf"))

        if prim == BOARDCAST:
            if self.ip_table[root] == self.ip_table[me]:
                r_local = self.node_ranks.index(root)
                if r_local != 0:                       # bring the data to this server's local root first
                    if my_local in (0, r_local):
                        n.broadcast(flat, root=r_local, active=sorted({0, r_local}))
                    else:
                        n.skip_op()
            if i_am_root:
                dist.broadcast(flat, src=root_node_root, group=group)
            n.broadcast(flat, root=0, active=all_local)
            return

        # ---- ALLREDUCE / REDUCE: (1) reduce inside the server to its local root ----------------------
        mine_active = me in active
        local = sorted(self.node_ranks.index(r) for r in active if r in self.node_ranks)
        members = sorted(set(local) | {0}) if local else []
        keep_own = (not mine_active) or (prim == REDUCE and me != root)   # my tensor must survive untouched
        work = flat
        if my_local in members and (not mine_active):
            work = identity()                           # the collecting root contributes nothing itself
        elif i_am_root and keep_own:
            work = flat.clone()
        if members:
            n.reduce(work, root=0, op=red, algo="auto", active=members)
        # ---- (2) the local roots meet over the inter-server fabric -----------------------------------
        if i_am_root:
            if not members:
                work = identity()
            if prim == ALLREDUCE:
                dist.all_reduce(work, op=rop, group=group)
            else:
                dist.reduce(work, dst=root_node_root, op=rop, group=group)
            if op == "avg":
                work.mul_(1.0 / max(1, len(active)))
        # ---- (3) hand the result out inside the server --------------------------------------------
        if prim == ALLREDUCE:
            if i_am_root:
                n.broadcast(work, root=0, active=all_local)
                if mine_active and work is not flat:
                    flat.copy_(work)
            else:
                n.broadcast(flat if mine_active else torch.empty_like(flat), root=0, active=all_local)
        elif self.ip_table[root] == self.ip_table[me]:
            r_local = self.node_ranks.index(root)
            if r_local != 0:                            # result is on the local root; `root` wants it
                if my_local == 0:
                    n.broadcast(work, root=0, active=sorted({0, r_local}))
                elif my_local == r_local:
                    n.broadcast(flat, root=0, active=sorted({0, r_local}))
                else:
                    n.skip_op()
            elif i_am_root and work is not flat:
                flat.copy_(work)

    def _launch(self, n, prim, flat, algo, wire, chunk_bytes, active, op, root):
        if algo == "tree":
            n.tree_collective(prim, flat, op=op, wire=wire, chunk_bytes=int(chunk_bytes), active=active)
        elif prim == ALLREDUCE:
            n.all_reduce(flat, op=op, algo=algo, wire=wire, active=active)
        elif prim == REDUCE:
            n.reduce(flat, root=(active[0] if root is None else root), op=op, algo=algo, wire=wire, active=active)
        else:
            n.broadcast(flat, root=(active[0] if root is None else root), active=active)

    # @buffer: torch tensor (device or host), @size: number of elements, @chunk_bytes: pipelining
    # granularity in bytes, @active_gpus: world ranks taking part (reference signature).
    def all_reduce(self, buffer, size=None, chunk_bytes=None, active_gpus=None, op="sum"):
        """In-place all-reduce of ``buffer[:size]`` over ``active_gpus`` (reference signature, /root/reference/commu.py:360-365);
        ``op``: sum | avg | max. Asynchronous on the current CUDA stream; host tensors go through the CPU executor."""
        return self._collective(ALLREDUCE, buffer, size, chunk_bytes, active_gpus, op)

    def reduce(self, buffer, size=None, chunk_bytes=None, active_gpus=None, op="sum", root=None):
        """In-place reduce to ``root`` (default: the first active rank; tree algorithm: each tree's root)."""
        return self._collective(REDUCE, buffer, size, chunk_bytes, active_gpus, op, root)

    def boardcast(self, buffer, size=None, chunk_bytes=None, active_gpus=None, root=None):
        """Broadcast from ``root`` (default: the first active rank); ``broadcast`` is an alias."""
        return self._collective(BOARDCAST, buffer, size, chunk_bytes, active_gpus, "sum", root)

    broadcast = boardcast

    def reduce_scatter(self, buffer, size=None, op="sum"):
        """In-place reduce-scatter over all ranks; returns ``(lo, hi)``: the element range of ``buffer[:size]`` that holds
        this rank's reduced shard afterwards (16-byte packs dealt out contiguously, ``parallel.engine.shard_of``)."""
        from .parallel.shards import reduce_scatter

        return reduce_scatter(self, buffer, size, op)

    def all_gather(self, buffer, size=None):
        """In-place all-gather, the inverse of :meth:`reduce_scatter`: rank r's shard of ``buffer[:size]`` is valid on
        entry, the whole range on exit."""
        from .parallel.shards import all_gather

        return all_gather(self, buffer, size)

    def synchronize(self):
        """Wait for the data plane and raise if a device-side wait timed out."""
        if self.native is not None:
            import torch

            for s in (self._comm_stream, self._relay_stream, torch.cuda.current_stream(self.local_rank)):
                if s is not None:
                    self.native.check(s)

    # ==========================================================================================
    # DDP communication hook
    # ==========================================================================================
    def cuda_allreduce_hook(self, state: object, bucket):
        """torch DDP communication hook (``ddp.register_comm_hook(None, communicator.cuda_allreduce_hook)``): the first
        bucket of a step negotiates the active set with the coordinator (relay control), every bucket is reduced on a
        side stream by our kernels and returned as a CUDA future — unlike the reference's blocking hook
        (/root/reference/commu.py:385-435), backward keeps running."""
        import torch

        if getattr(self, "_cleared", False):
            # DDP keeps the bound method it was given at register_comm_hook time; after reconstruct_topology that is
            # a cleared communicator -> hand the bucket to the live one (the reference re-creates the communicator
            # the same way, /root/reference/adapcc.py:64-68, and leaves the hook dangling)
            live = self._live()
            if live is not self:
                return live.cuda_allreduce_hook(state, bucket)
        if self.local_hook_num == 0 and self.relay_control:
            t0 = time.time()
            try:
                self.active_gpus = sorted(self.hooker.send_ready_request(self.current_step, self.world_rank))
            except Exception as e:  # noqa: BLE001  coordinator unreachable: degrade to a plain all-reduce
                self._log(f"hook RPC failed ({e}); treating every rank as active")
                self.active_gpus = list(range(self.world_size))
            self.stats["hook_rpc_s"].append(time.time() - t0)
        self.local_hook_num += 1
        buffer = bucket.buffer()
        size = int(buffer.numel())
        total_bytes = buffer.element_size() * size
        chunk_bytes = default_chunk_bytes(total_bytes)
        self._log(f"hook active: {self.active_gpus}; tensor number {size}, {total_bytes} bytes, chunk bytes {chunk_bytes}")

        if not buffer.is_cuda:
            self.all_reduce(buffer, size, chunk_bytes, self.active_gpus, op=self.reduce_op)
            fut = torch.futures.Future()
            fut.set_result(buffer)
            return fut

        active = self.active_gpus
        i_am_active = self.world_rank in active
        if self.current_step == 1:
            if self.local_hook_num == 1:             # first bucket of step 1: (re)learn the layout from scratch
                self.bucket_info.clear()
                self.relay_buffer.clear()
            self.bucket_info.append((size, chunk_bytes, buffer.dtype))
            if self.relay_control and self.relay_mode == RELAY_FORWARD and self._resolve_algo(size, buffer.dtype, active) == "tree":
                self.relay_buffer.append(torch.zeros(size, dtype=buffer.dtype, device=buffer.device))
            else:
                self.relay_buffer.append(None)
        comm_stream, relay_stream = self._streams()
        comm_stream.wait_stream(torch.cuda.current_stream(buffer.device))
        comm_stream.wait_stream(relay_stream)     # relay duty of earlier steps precedes this step's ops (op sequence)
        with torch.cuda.stream(comm_stream):
            if i_am_active or self.current_step <= 1:
                self.all_reduce(buffer, size, chunk_bytes, active if self.current_step > 1 else list(range(self.world_size)),
                                op=self.reduce_op)
            # relays (BSP): this rank's own un-reduced gradient is used for its local update; the
            # controller thread keeps the data plane consistent (skip / forward) on the relay stream
            fut = torch.futures.Future(devices=[buffer.device])
            fut.set_result(buffer)
        if not i_am_active and self.current_step > 1 and self.local_hook_num == max(1, len(self.bucket_info)):
            try:
                self.bsp_queue.get(timeout=60)
            except Empty:
                pass
        return fut
