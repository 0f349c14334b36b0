"""dear_pytorch_b200 — an H100-native DeAR (decoupled all-reduce) data-parallel engine.

Public API (same surface as the reference package ``dear``, dear/__init__.py:3-9)::

    import dear_pytorch_b200 as dear          # or simply: import dear
    dear.init()
    optimizer = dear.DistributedOptimizer(torch.optim.SGD(...), model)
    dear.broadcast_parameters(model.state_dict(), root_rank=0)
    ...  zero_grad -> forward -> loss -> backward -> step  ...
    avg = dear.allreduce(metric_tensor)

plus what the reference lacks: ``local_rank()``, ``shutdown()``, ``synchronize()``,
checkpointing (``save_checkpoint`` / ``load_checkpoint``) and a CUDA-graph step wrapper.
"""
from .runtime import (init, shutdown, rank, size, local_rank, local_size, backend, device, barrier,  # noqa: F401
                      is_initialized, communicator)
from .parallel.optimizer import DistributedOptimizer, DearEngine, THRESHOLD, NUM_NEARBY_LAYERS  # noqa: F401
from .parallel.grad_scaler import GradScaler  # noqa: F401
from .parallel.collectives import (allreduce, allreduce_, broadcast_, broadcast_parameters,  # noqa: F401
                                   broadcast_optimizer_state, allgather)
from .utils.checkpoint import save_checkpoint, load_checkpoint  # noqa: F401
from .utils.train import TrainStep  # noqa: F401

__version__ = "0.1.0"
