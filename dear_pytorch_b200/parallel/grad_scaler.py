"""Dynamic loss scaling for the fused DeAR path, with the interface of ``torch.amp.GradScaler``.

The reference's mixed-precision loop (examples/mnist/pytorch_mnist.py:63-83 of the reference) is::

    scaler.scale(loss).backward(); optimizer.synchronize(); scaler.unscale_(optimizer)
    with optimizer.skip_synchronize(): scaler.step(optimizer)
    scaler.update()

Here the gradients never surface as tensors: Kernel A consumes them during back-propagation and Kernel B applies the
update.  So the whole scaler runs on the device, from a state the engine owns (``DearEngine.attach_scaler``):

* Kernel A multiplies the reduced gradient by ``1/scale`` together with its ``1/P`` and flags a non-finite result;
* the first update kernel of the step ORs every rank's flag at its entry rendezvous, skips the step on every rank when
  one is set, and applies torch's rule to the scale (back off on overflow, grow after ``growth_interval`` clean steps);
* the other update kernels of the step follow that decision.

Nothing synchronises the host, and a CUDA graph of the training step replays the whole protocol.  ``unscale_`` and
``update()`` therefore have nothing left to do; they exist so that torch's call sequence runs unchanged.
"""
from __future__ import annotations

import torch

from .optimizer import DearEngine


def _map(fn, obj):
    if torch.is_tensor(obj):
        return fn(obj)
    if isinstance(obj, (list, tuple)):
        return type(obj)(_map(fn, o) for o in obj)
    raise ValueError("outputs must be a Tensor or a list/tuple of Tensors")


class GradScaler:
    """``torch.amp.GradScaler`` for a DeAR ``DistributedOptimizer`` (same method names and state-dict keys)."""

    def __init__(self, optimizer, init_scale: float = 2.0 ** 16, growth_factor: float = 2.0, backoff_factor: float = 0.5,
                 growth_interval: int = 2000, enabled: bool = True):
        engine = getattr(optimizer, "_dear", None)
        if not isinstance(engine, DearEngine):
            raise TypeError("dear.GradScaler needs a dear.DistributedOptimizer (the loss scale is applied inside its fused "
                            "kernels); got %s.  Use torch.amp.GradScaler for other optimizers." % type(optimizer).__name__)
        if not init_scale > 0:
            raise ValueError("init_scale must be positive")
        if not growth_factor > 1.0:
            raise ValueError("growth_factor should be > 1")
        if not 0.0 < backoff_factor < 1.0:
            raise ValueError("backoff_factor should be in (0, 1)")
        if int(growth_interval) < 1:
            raise ValueError("growth_interval should be a positive integer")
        self._optimizer = optimizer
        self._engine = engine
        self._enabled = bool(enabled)
        self._config = {"growth_factor": float(growth_factor), "backoff_factor": float(backoff_factor),
                        "growth_interval": int(growth_interval)}      # what a disabled scaler reports, like torch
        if self._enabled:
            engine.attach_scaler(float(init_scale), float(growth_factor), float(backoff_factor), int(growth_interval))

    def _check(self, optimizer):
        if optimizer is not self._optimizer:
            raise ValueError("this GradScaler belongs to another optimizer")

    def is_enabled(self) -> bool:
        return self._enabled

    def scale(self, outputs):
        """``outputs * scale`` with the device-resident scale (a tensor op, so it can be captured in a CUDA graph)."""
        if not self._enabled:
            return outputs
        s = self._engine.scaler_scale()
        return _map(lambda t: t * s, outputs)

    def unscale_(self, optimizer) -> None:
        """No-op: the ``1/scale`` is a factor of the reduce-scatter epilogue."""
        self._check(optimizer)

    def step(self, optimizer, *args, **kwargs):
        """``optimizer.step()``; whether the update is applied is decided on the GPU (no host synchronisation)."""
        self._check(optimizer)
        return optimizer.step(*args, **kwargs)

    def update(self, new_scale=None) -> None:
        """Growth and backoff already happened on the device.  ``new_scale`` (float or 1-element tensor) replaces
        that step's rule, like torch: the scale becomes ``new_scale`` and the growth tracker goes back to its value
        before the step."""
        if not self._enabled or new_scale is None:
            return
        if torch.is_tensor(new_scale):
            if new_scale.numel() != 1:
                raise ValueError("new_scale should be a 1-element tensor")
            new_scale = float(new_scale)
        eng = self._engine
        eng.write_scaler(scale=new_scale)
        # (stream-ordered after the step's deciding kernel by write_scaler; no host synchronisation)
        eng.amp[eng._AMP_I32["growth_tracker"]].copy_(eng.amp[eng._AMP_I32["prev_growth_tracker"]])

    def get_scale(self) -> float:
        """Current scale (synchronises the host); 1.0 when disabled."""
        return self._engine.read_scaler()["scale"] if self._enabled else 1.0

    def _get_growth_tracker(self) -> int:
        return self._engine.read_scaler()["growth_tracker"] if self._enabled else 0

    def get_growth_factor(self) -> float:
        return self._engine.read_scaler()["growth_factor"] if self._enabled else self._config["growth_factor"]

    def get_backoff_factor(self) -> float:
        return self._engine.read_scaler()["backoff_factor"] if self._enabled else self._config["backoff_factor"]

    def get_growth_interval(self) -> int:
        return self._engine.read_scaler()["growth_interval"] if self._enabled else self._config["growth_interval"]

    def state_dict(self) -> dict:
        """torch.amp.GradScaler's keys, so a checkpoint loads into either scaler."""
        if not self._enabled:
            return {}
        st = self._engine.read_scaler()
        return {"scale": st["scale"], "growth_factor": st["growth_factor"], "backoff_factor": st["backoff_factor"],
                "growth_interval": st["growth_interval"], "_growth_tracker": st["growth_tracker"]}

    def load_state_dict(self, state_dict: dict) -> None:
        if not self._enabled:
            return
        if len(state_dict) == 0:
            raise RuntimeError("The source state dict is empty, possibly because it was saved from a disabled instance "
                               "of GradScaler.")
        self._engine.write_scaler(scale=float(state_dict["scale"]), growth_factor=float(state_dict["growth_factor"]),
                                  backoff_factor=float(state_dict["backoff_factor"]),
                                  growth_interval=int(state_dict["growth_interval"]),
                                  growth_tracker=int(state_dict["_growth_tracker"]),
                                  prev_growth_tracker=int(state_dict["_growth_tracker"]))
