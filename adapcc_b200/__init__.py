"""adapcc_b200 — a Hopper-native adaptive collective-communication library.

Capabilities and API of JoeyYoung/adapcc (``AdapCC.init/setup/clear``, ``communicator.all_reduce /
reduce / boardcast``, ``cuda_allreduce_hook`` for torch DDP, XML strategy/topology files, strategy
synthesizer, on-the-fly link profiling, relay/straggler control, ``reconstruct_topology``),
re-designed for H100 servers over NVLink / NVSwitch: the collectives are hand-written sm_90a kernels
that move data with in-kernel peer loads/stores and NVLS multimem instructions on VMM symmetric
memory, fused with the bucket's cast/scale/reduction.
"""
from .constants import (ALLGATHER, ALLREDUCE, ALLTOALL, BOARDCAST, DETECT, PROFILE, REDUCE,  # noqa: F401
                        REDUCESCATTER)

__version__ = "0.1.0"


def __getattr__(name):  # lazy: keep `import adapcc_b200` light (no torch / grpc import)
    if name == "AdapCC":
        from .adapcc import AdapCC
        return AdapCC
    if name == "CudaCommu":
        from .commu import CudaCommu
        return CudaCommu
    raise AttributeError(name)
