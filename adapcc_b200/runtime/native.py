"""ctypes binding of ``libadapcc.so`` (the native runtime).

The reference binds ``communicator.so`` with ``ctypes.CDLL`` and passes raw ``data_ptr()``s
(/root/reference/adapcc.py:17-24, /root/reference/commu.py:124-134). We keep that shape — one
C ABI, no torch C++ extension in the way — but the calls are asynchronous launches on a CUDA
stream instead of blocking thread hand-offs.
"""
from __future__ import annotations

import ctypes
import os
import threading
from ctypes import c_char_p, c_int, c_longlong, c_ulonglong, c_void_p
from pathlib import Path
from typing import Optional, Sequence

from ..constants import ALGO_IDS, DTYPE_IDS, OP_IDS

_LIB = None
_LIB_LOCK = threading.Lock()
_LIB_PATH = Path(__file__).resolve().parent.parent / "_C" / "libadapcc.so"


class NativeError(RuntimeError):
    pass


def lib_path() -> Path:
    return _LIB_PATH


def load_library(build_if_missing: bool = True) -> ctypes.CDLL:
    """Load (building in-tree first if needed) the native runtime. Fails loudly."""
    global _LIB
    with _LIB_LOCK:
        if _LIB is not None:
            return _LIB
        if not _LIB_PATH.exists():
            if not build_if_missing:
                raise NativeError(f"{_LIB_PATH} is missing; run `python -m adapcc_b200.build`")
            from .. import build as _build

            _build.build()
        lib = ctypes.CDLL(str(_LIB_PATH), mode=ctypes.RTLD_GLOBAL)
        lib.adapcc_last_error.restype = c_char_p
        lib.adapcc_launch_count.restype = c_longlong
        lib.adapcc_ctx_create.restype = c_void_p
        lib.adapcc_ctx_create.argtypes = [c_char_p, c_int, c_int, c_int, c_ulonglong, c_ulonglong]
        lib.adapcc_ctx_destroy.argtypes = [c_void_p]
        lib.adapcc_ctx_info.argtypes = [c_void_p, ctypes.POINTER(c_int)]
        lib.adapcc_ctx_heap_ptr.restype = c_void_p
        lib.adapcc_ctx_heap_ptr.argtypes = [c_void_p]
        lib.adapcc_ctx_heap_bytes.restype = c_ulonglong
        lib.adapcc_ctx_heap_bytes.argtypes = [c_void_p]
        lib.adapcc_ctx_staging_bytes.restype = c_ulonglong
        lib.adapcc_ctx_staging_bytes.argtypes = [c_void_p]
        lib.adapcc_ctx_heap_mc_ptr.restype = c_void_p
        lib.adapcc_ctx_heap_mc_ptr.argtypes = [c_void_p]
        lib.adapcc_ctx_peer_heap_ptr.restype = c_void_p
        lib.adapcc_ctx_peer_heap_ptr.argtypes = [c_void_p, c_int]
        lib.adapcc_ctx_peer_staging_ptr.restype = c_void_p
        lib.adapcc_ctx_peer_staging_ptr.argtypes = [c_void_p, c_int]
        lib.adapcc_ctx_last_algo.argtypes = [c_void_p]
        lib.adapcc_pool_bind.argtypes = [c_void_p, c_ulonglong]
        lib.adapcc_pool_offset.restype = c_ulonglong
        lib.adapcc_ctx_set_tunable.argtypes = [c_void_p, c_int, c_longlong]
        lib.adapcc_ctx_load_strategy.argtypes = [c_void_p, c_char_p]
        lib.adapcc_ctx_load_strategy_text.argtypes = [c_void_p, c_char_p]
        ip = ctypes.POINTER(c_int)
        lib.adapcc_allreduce.argtypes = [c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_int, c_int,
                                         c_int, ip, c_int, c_void_p]
        lib.adapcc_reduce.argtypes = [c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_int, c_int, c_int,
                                      c_int, ip, c_int, c_void_p]
        lib.adapcc_broadcast.argtypes = [c_void_p, c_void_p, c_longlong, c_int, c_int, ip, c_int, c_void_p]
        lib.adapcc_tree_collective.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_longlong, c_int, c_int,
                                               c_int, c_longlong, ip, c_int, c_void_p]
        lib.adapcc_tree_relay_persistent.argtypes = [c_void_p, c_int, ctypes.POINTER(c_longlong),
                                                     ctypes.POINTER(c_longlong), c_int, c_int, ip, c_int, c_void_p]
        lib.adapcc_alltoall.argtypes = [c_void_p, c_void_p, c_void_p, c_longlong, c_int, ip, c_int, c_void_p]
        lib.adapcc_skip_op.argtypes = [c_void_p, c_void_p]
        lib.adapcc_barrier.argtypes = [c_void_p, ctypes.POINTER(c_int), c_int, c_void_p]
        lib.adapcc_allreduce_ll.argtypes = [c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_int, c_void_p]
        lib.adapcc_ctx_has_ll.argtypes = [c_void_p]
        lib.adapcc_ctx_check.argtypes = [c_void_p, c_void_p]
        lib.adapcc_ctx_host_barrier.argtypes = [c_void_p]
        lib.adapcc_relay_control.argtypes = [c_char_p, c_int, c_int, c_int, ip, c_int, ip, c_int]
        lib.adapcc_tree_role.argtypes = [c_char_p, c_int, c_int, c_int, ip, c_int, c_int, c_int, ip, c_int]
        _LIB = lib
        return lib


def last_error() -> str:
    lib = load_library()
    e = lib.adapcc_last_error()
    return e.decode("utf-8", "replace") if e else ""


def _check(rc: int, what: str) -> None:
    if rc != 0:
        raise NativeError(f"{what} failed: {last_error()}")


def _int_array(values: Sequence[int]):
    arr = (c_int * max(1, len(values)))(*values)
    return arr


TUNABLE_KEYS = {"max_blocks": 0, "one_shot_max_bytes": 1, "nvls_min_bytes": 2, "relay_mode": 3,
                "timeout_ms": 4, "tree_blocks": 5, "tree_chunk_max_bytes": 6, "nvls_min_ranks": 7, "force_kernel": 8, "pipe_min_bytes": 9, "pipe_stagers": 10,
                "pipe_links": 11, "pipe_piece_bytes": 12, "pipe_nvls": 13, "ll_max_bytes": 14}


class _CudaArray:
    """Minimal __cuda_array_interface__ holder so torch can view native symmetric memory."""

    def __init__(self, ptr: int, nbytes: int, owner):
        self.__cuda_array_interface__ = {
            "shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None,
        }
        self._owner = owner


class NativeComm:
    """One native communicator context (symmetric windows + signal pads + kernels)."""

    def __init__(self, name: str, rank: int, world: int, device: int, staging_bytes: int = 256 << 20,
                 heap_bytes: int = 0):
        self.lib = load_library()
        self.rank, self.world, self.device = rank, world, device
        h = self.lib.adapcc_ctx_create(name.encode(), rank, world, device, staging_bytes, heap_bytes)
        if not h:
            raise NativeError(f"adapcc_ctx_create(rank={rank}, world={world}, dev={device}) failed: {last_error()}")
        self.handle = c_void_p(h)
        self._heap_off = 0
        info = (c_int * 8)()
        self.lib.adapcc_ctx_info(self.handle, info)
        self.symm_backend = {0: "vmm", 1: "cuda_ipc"}.get(info[0], str(info[0]))
        self.multicast = bool(info[1])
        self.heap_multicast = bool(info[2])

    # -- lifecycle ---------------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "handle", None) is not None and self.handle.value:
            self.lib.adapcc_ctx_destroy(self.handle)
            self.handle = c_void_p(None)

    def __del__(self):  # best effort; explicit close() is collective and preferred
        pass

    # -- configuration -----------------------------------------------------------------
    def set_tunable(self, key: str, value: int) -> None:
        _check(self.lib.adapcc_ctx_set_tunable(self.handle, TUNABLE_KEYS[key], int(value)), f"set_tunable({key})")

    def load_strategy(self, path_or_text: str) -> int:
        if path_or_text.lstrip().startswith("<"):
            _check(self.lib.adapcc_ctx_load_strategy_text(self.handle, path_or_text.encode()), "load_strategy_text")
        else:
            _check(self.lib.adapcc_ctx_load_strategy(self.handle, os.fspath(path_or_text).encode()), "load_strategy")
        info = (c_int * 8)()
        self.lib.adapcc_ctx_info(self.handle, info)
        return info[5]

    @property
    def last_algo(self) -> int:
        return self.lib.adapcc_ctx_last_algo(self.handle)

    @property
    def staging_bytes(self) -> int:
        return int(self.lib.adapcc_ctx_staging_bytes(self.handle))

    @property
    def heap_bytes(self) -> int:
        return int(self.lib.adapcc_ctx_heap_bytes(self.handle))

    # -- symmetric heap ------------------------------------------------------------------
    def heap_tensor(self, nbytes: Optional[int] = None, offset: int = 0):
        """uint8 torch view of (part of) this rank's symmetric heap."""
        import torch

        base = self.lib.adapcc_ctx_heap_ptr(self.handle)
        if not base:
            raise NativeError("context has no symmetric heap (heap_bytes=0)")
        total = self.heap_bytes
        nbytes = total - offset if nbytes is None else nbytes
        if offset + nbytes > total:
            raise NativeError(f"heap view [{offset}, {offset + nbytes}) exceeds {total} bytes")
        with torch.cuda.device(self.device):
            return torch.as_tensor(_CudaArray(base + offset, nbytes, self), device=f"cuda:{self.device}")

    def symm_empty(self, numel: int, dtype):
        """Bump-allocate a tensor inside the symmetric heap (same offset on every rank as long as
        every rank performs the same sequence of allocations). Collectives on such tensors are
        zero-copy: peers read/write them directly over NVLink."""
        import torch

        esize = torch.empty((), dtype=dtype).element_size()
        nbytes = numel * esize
        off = (self._heap_off + 255) // 256 * 256
        t = self.heap_tensor(nbytes, off).view(dtype)
        self._heap_off = off + nbytes
        return t

    def heap_reset(self) -> None:
        self._heap_off = 0

    def mem_pool(self):
        """A ``torch.cuda.MemPool`` whose blocks come from this context's symmetric heap. Tensors
        allocated under ``torch.cuda.use_mem_pool(pool)`` (e.g. DDP's gradient buckets) are then
        reduced zero-copy. Every rank must allocate the same sequence of sizes."""
        import torch

        if getattr(self, "_pool", None) is None:
            self.lib.adapcc_pool_bind(self.handle, (self._heap_off + 511) // 512 * 512)
            alloc = torch.cuda.memory.CUDAPluggableAllocator(str(lib_path()), "adapcc_pool_alloc", "adapcc_pool_free")
            self._pool_allocator = alloc
            self._pool = torch.cuda.MemPool(alloc.allocator())
        return self._pool

    def heap_offset(self, tensor) -> int:
        """Byte offset of a heap tensor inside the symmetric heap (the same on every rank)."""
        base = self.lib.adapcc_ctx_heap_ptr(self.handle) or 0
        if not self.in_heap(tensor):
            raise NativeError("tensor is not inside the symmetric heap")
        return tensor.data_ptr() - base

    def heap_mc_ptr(self) -> int:
        """Multicast alias of the heap base (0 when no multicast object is bound)."""
        return int(self.lib.adapcc_ctx_heap_mc_ptr(self.handle) or 0)

    def peer_heap_ptr(self, r: int) -> int:
        return int(self.lib.adapcc_ctx_peer_heap_ptr(self.handle, int(r)) or 0)

    def device_barrier(self, active=None, stream=None) -> None:
        """One-CTA device-side barrier among ``active`` on ``stream`` (orders peer stores before later kernels)."""
        arr, n = self._active(active)
        _check(self.lib.adapcc_barrier(self.handle, arr, n, self._stream_ptr(stream)), "device_barrier")

    def in_heap(self, tensor) -> bool:
        base = self.lib.adapcc_ctx_heap_ptr(self.handle) or 0
        p = tensor.data_ptr()
        return bool(base) and base <= p and p + tensor.numel() * tensor.element_size() <= base + self.heap_bytes

    # -- collectives ---------------------------------------------------------------------
    @staticmethod
    def _stream_ptr(stream) -> c_void_p:
        import torch

        s = torch.cuda.current_stream() if stream is None else stream
        return c_void_p(s.cuda_stream)

    def _active(self, active):
        act = list(range(self.world)) if active is None else [int(a) for a in active]
        return _int_array(act), len(act)

    @staticmethod
    def _dt(t) -> int:
        return DTYPE_IDS[str(t.dtype).replace("torch.", "")]

    def all_reduce(self, tensor, out=None, op: str = "sum", algo: str = "auto", wire: Optional[str] = None,
                   active=None, stream=None):
        out = tensor if out is None else out
        dt = self._dt(tensor)
        if algo == "ll":
            return self.all_reduce_ll(tensor, out=out, op=op, stream=stream)
        wd = dt if wire is None else DTYPE_IDS[wire]
        arr, n = self._active(active)
        _check(self.lib.adapcc_allreduce(self.handle, c_void_p(tensor.data_ptr()), c_void_p(out.data_ptr()),
                                         tensor.numel(), dt, wd, OP_IDS[op], ALGO_IDS[algo], arr, n,
                                         self._stream_ptr(stream)), "all_reduce")
        return out

    @property
    def has_ll(self) -> bool:
        return bool(self.lib.adapcc_ctx_has_ll(self.handle))

    def all_reduce_ll(self, tensor, out=None, op: str = "sum", stream=None):
        """Low-latency all-reduce (csrc/kernels_ll.cuh): every rank takes part, message <= 32 KB, flag-in-data lines
        pushed into every peer's LL buffer — no barrier (about half the latency of the barrier kernels at 1 KB).
        ``algo="auto"`` picks it for such messages; the buffer exists unless the job runs with ``ADAPCC_LL=0``."""
        out = tensor if out is None else out
        _check(self.lib.adapcc_allreduce_ll(self.handle, c_void_p(tensor.data_ptr()), c_void_p(out.data_ptr()),
                                            tensor.numel(), self._dt(tensor), OP_IDS[op], self._stream_ptr(stream)),
               "all_reduce_ll")
        return out

    def reduce(self, tensor, root: int, out=None, op: str = "sum", algo: str = "auto",
               wire: Optional[str] = None, active=None, stream=None):
        out = tensor if out is None else out
        dt = self._dt(tensor)
        wd = dt if wire is None else DTYPE_IDS[wire]
        arr, n = self._active(active)
        _check(self.lib.adapcc_reduce(self.handle, c_void_p(tensor.data_ptr()), c_void_p(out.data_ptr()),
                                      tensor.numel(), dt, wd, OP_IDS[op], ALGO_IDS[algo], int(root), arr, n,
                                      self._stream_ptr(stream)), "reduce")
        return out

    def reduce_scatter_(self, tensor, op: str = "sum", algo: str = "auto", stream=None):
        """In-place reduce-scatter over all ranks: afterwards elements ``[lo, hi)`` of ``tensor`` (the returned
        range, this rank's slice under the direct kernels' partition) hold the reduction; the rest of the tensor
        is unspecified. It is the direct reduce kernel with root = self, so it moves half the bytes of an
        all-reduce. (Used by the engine's sharded-optimizer mode and ``AdapCC.reducescatter``.)"""
        from ..parallel.engine import shard_of

        self.reduce(tensor, root=self.rank, op=op, algo=algo, stream=stream)
        return shard_of(0, tensor.numel(), self.rank, self.world, 16 // tensor.element_size())

    def all_gather_(self, tensor, stream=None):
        """In-place all-gather, the inverse of :meth:`reduce_scatter_`: on entry rank r's shard of ``tensor`` is valid,
        on exit every rank holds every shard. Composed of one direct broadcast per shard (``world`` launches of the
        validated broadcast kernel — multimem.st when multicast is bound); a single-kernel version is only worth
        writing where this shows up in a profile (the sharded optimizer broadcasts from inside its own kernel)."""
        from ..parallel.engine import shard_of

        epp = 16 // tensor.element_size()
        flat = tensor.view(-1)
        for r in range(self.world):
            lo, hi = shard_of(0, flat.numel(), r, self.world, epp)
            if hi > lo:
                self.broadcast(flat[lo:hi], root=r, stream=stream)
        return tensor

    def broadcast(self, tensor, root: int, active=None, stream=None):
        arr, n = self._active(active)
        _check(self.lib.adapcc_broadcast(self.handle, c_void_p(tensor.data_ptr()), tensor.numel(),
                                         self._dt(tensor), int(root), arr, n, self._stream_ptr(stream)),
               "broadcast")
        return tensor

    def tree_collective(self, prim: int, tensor, out=None, op: str = "sum", wire: Optional[str] = None,
                        chunk_bytes: int = 1 << 20, active=None, stream=None):
        out = tensor if out is None else out
        dt = self._dt(tensor)
        wd = dt if wire is None else DTYPE_IDS[wire]
        arr, n = self._active(active)
        _check(self.lib.adapcc_tree_collective(self.handle, int(prim), c_void_p(tensor.data_ptr()),
                                               c_void_p(out.data_ptr()), tensor.numel(), dt, wd, OP_IDS[op],
                                               int(chunk_bytes), arr, n, self._stream_ptr(stream)),
               "tree_collective")
        return out

    def all_to_all(self, tensor, out=None, active=None, stream=None):
        """Dense all-to-all of equal splits: block p of ``tensor`` goes to rank p, block r of the result
        comes from rank r (``torch.distributed.all_to_all_single`` semantics)."""
        import torch

        arr, n = self._active(active)
        if tensor.numel() % n:
            raise NativeError(f"all_to_all: {tensor.numel()} elements do not split over {n} ranks")
        out = torch.empty_like(tensor) if out is None else out
        _check(self.lib.adapcc_alltoall(self.handle, c_void_p(tensor.data_ptr()), c_void_p(out.data_ptr()),
                                        tensor.numel() // n, self._dt(tensor), arr, n, self._stream_ptr(stream)),
               "all_to_all")
        return out

    def tree_relay_persistent(self, counts, chunk_bytes, wire: str = "float32", op: str = "sum", active=None,
                              stream=None) -> None:
        """Relay duty for a whole step (all gradient buckets) in one persistent kernel launch."""
        n = len(counts)
        c_arr = (c_longlong * max(1, n))(*[int(x) for x in counts])
        k_arr = (c_longlong * max(1, n))(*[int(x) for x in chunk_bytes])
        arr, na = self._active(active)
        _check(self.lib.adapcc_tree_relay_persistent(self.handle, n, c_arr, k_arr, DTYPE_IDS[wire], OP_IDS[op], arr, na,
                                                     self._stream_ptr(stream)), "tree_relay_persistent")

    def skip_op(self, stream=None) -> None:
        _check(self.lib.adapcc_skip_op(self.handle, self._stream_ptr(stream)), "skip_op")

    def check(self, stream=None) -> None:
        """Synchronise the stream and raise if any device-side wait timed out."""
        rc = self.lib.adapcc_ctx_check(self.handle, self._stream_ptr(stream))
        if rc != 0:
            raise NativeError(f"collective failed: {last_error()}")

    def host_barrier(self) -> None:
        _check(self.lib.adapcc_ctx_host_barrier(self.handle), "host_barrier")


# ---- pure host queries (usable on the CPU-only box) -------------------------------------
def native_relay_control(xml_text: str, world: int, tree: int, rank: int, active: Sequence[int]):
    lib = load_library()
    out = (c_int * 64)()
    arr = _int_array(list(active))
    n = lib.adapcc_relay_control(xml_text.encode(), world, tree, rank, arr, len(active), out, 64)
    if n < 0:
        raise NativeError(last_error())
    return {"has_recv": bool(out[0]), "has_local": bool(out[1]), "has_kernel": bool(out[2]),
            "has_send": bool(out[3]), "active_recvs": [out[5 + i] for i in range(out[4])], "n_trees": n}


def native_tree_role(xml_text: str, world: int, tree: int, rank: int, active: Sequence[int], prim: int,
                     relay_mode: int = 0):
    lib = load_library()
    out = (c_int * 64)()
    arr = _int_array(list(active))
    n = lib.adapcc_tree_role(xml_text.encode(), world, tree, rank, arr, len(active), prim, relay_mode, out, 64)
    if n < 0:
        raise NativeError(last_error())
    return {"parent": out[0], "flags": out[1], "children": [out[3 + i] for i in range(out[2])], "n_trees": n}
