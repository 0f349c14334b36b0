"""Build the native runtime in-tree:  python setup.py build_ext --inplace

Produces dear_pytorch_b200/_C.*.so (runtime, collectives, fused BN / LN kernels) and dear_pytorch_b200/_tc.*.so
(hand-written wgmma / TMA GEMMs with fused epilogues) -- sm_90a (H100) only; no other architecture is built.
The reference's counterpart is common/comm_core/setup.py:16-44 (NCCL+MPI); this
extension links neither.
"""
import glob
import os

from setuptools import find_packages, setup
from torch.utils.cpp_extension import BuildExtension, CUDAExtension

ROOT = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join("dear_pytorch_b200", "csrc")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xptxas", "-v",
    "--expt-relaxed-constexpr",
]
CXX_FLAGS = ["-O2", "-std=c++17", "-Wno-unused-function"]

ext = CUDAExtension(
    name="dear_pytorch_b200._C",
    sources=[os.path.join(CSRC, f) for f in
             ("bindings.cpp", "communicator.cpp", "symm_mem.cpp", "emu.cpp", "kernels.cu", "rs_pipe.cu", "bn_act.cu", "ln_fused.cu")],
    include_dirs=[os.path.join(ROOT, CSRC)],
    extra_compile_args={"cxx": CXX_FLAGS, "nvcc": NVCC_FLAGS},
    libraries=["rt"],
)



tc_ext = CUDAExtension(
    name="dear_pytorch_b200._tc",
    # hand-written wgmma / TMA kernels (raw PTX; no CUTLASS headers needed)
    sources=[os.path.join(CSRC, "tc_bindings.cpp"), os.path.join(CSRC, "tc_ffn_hw.cu")],
    include_dirs=[os.path.join(ROOT, CSRC)],
    extra_compile_args={"cxx": CXX_FLAGS, "nvcc": NVCC_FLAGS},
)

setup(
    name="dear_pytorch_b200",
    version="0.1.0",
    packages=find_packages(include=["dear_pytorch_b200", "dear_pytorch_b200.*", "dear"]),
    py_modules=["comm_core"],               # drop-in for the reference's native module name
    ext_modules=[ext, tc_ext],
    cmdclass={"build_ext": BuildExtension.with_options(use_ninja=True)},
)
