"""`import dear` — drop-in alias of :mod:`dear_pytorch_b200` (reference package name, dear/__init__.py:3-9)."""
from dear_pytorch_b200 import *  # noqa: F401,F403
from dear_pytorch_b200 import (init, shutdown, rank, size, local_rank, local_size, DistributedOptimizer,  # noqa: F401
                               broadcast_parameters, broadcast_optimizer_state, allreduce, GradScaler)
