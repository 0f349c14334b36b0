"""Native op loader.

The compiled extension ``dear_pytorch_b200._C`` (built in-tree by
``python setup.py build_ext --inplace`` or ``__graft_entry__.build()``) holds
the sm_90a kernels and the C++ runtime.  On a machine with a GPU the
extension is mandatory: there is no silent PyTorch fallback for the fused
path (``require_native`` raises).  On CPU-only machines the same extension
provides the host-emulation backend.
"""
from __future__ import annotations

import importlib
import os

_C = None
_import_error = None


def native():
    """Return the compiled extension module or ``None`` if it is not built."""
    global _C, _import_error
    if _C is None and _import_error is None:
        try:
            import torch  # noqa: F401  (loads libtorch / libc10 first)
            import torch.distributed  # noqa: F401  (registers the c10d::Store pybind type)
            _C = importlib.import_module("dear_pytorch_b200._C")
        except Exception as exc:  # pragma: no cover - depends on the build
            _import_error = exc
    return _C


def require_native():
    mod = native()
    if mod is None:
        raise RuntimeError(
            "dear_pytorch_b200._C is not built (%r). Build it in-tree with "
            "`python setup.py build_ext --inplace` (or `python -c 'import __graft_entry__ as g; g.build()'`)."
            % (_import_error,))
    return mod


def native_path():
    mod = native()
    return None if mod is None else os.path.abspath(mod.__file__)
