"""`import comm_core` — the reference's native module name (common/comm_core/src/comm_core.cpp:12-37), as a drop-in.

    import comm_core
    comm_core.init()                       # process group (torchrun env://) + symmetric-memory runtime
    comm = comm_core.Communicator(1)       # nstreams
    comm.reduceScatter(send, recv); comm.allGather(recv, out); comm.allReduce(t); comm.synchronize()

``Communicator`` is :class:`dear_pytorch_b200.parallel.comm.Comm`: the same method names (``bcast, reduce, allReduce,
allReduceRB, allReduceRSAG, reduceScatter, allGather, multiBcast, sendrecv, synchronize, barrier, syncStream,
getNumOfFreeStreams, destroy, reload``) on the fused sm_90a kernels of ``dear_pytorch_b200._C`` (or on
torch.distributed for the gloo / nccl backends).  ``barriar`` keeps the reference's spelling.
"""
from dear_pytorch_b200 import init, rank, size, barrier  # noqa: F401
from dear_pytorch_b200.parallel.comm import Comm as Communicator  # noqa: F401

barriar = barrier
