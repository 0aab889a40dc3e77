"""In-tree build of the atomo_b200 native extension for sm_90a (H100).

    python setup.py build_ext --inplace      ->  atomo_b200/_C*.so

The arch is passed as an explicit -gencode (bypassing torch's arch list);
-lineinfo keeps profiler source views mapped to the .cu files.
"""
import os

from setuptools import setup
from torch.utils.cpp_extension import BuildExtension, CUDAExtension

os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
here = os.path.dirname(os.path.abspath(__file__))
src = os.path.join("atomo_b200", "csrc")
sources = [os.path.join(src, f) for f in (
    "bindings.cpp", "symm_heap.cpp", "svd_kernels.cu", "ps_kernels.cu", "qsgd_kernels.cu",
    "entrywise_kernels.cu", "ext_kernels.cu", "gemm_kernels.cu", "bn_kernels.cu", "v2_encode.cu", "v2_ps.cu",
    "v2_qsgd.cu", "v2_entrywise.cu", "v2_topk.cu", "v2_sign.cu", "v2_signum.cu", "v2_fp8.cu", "v2_hadamard.cu", "v2_powersgd.cu", "v2_stats.cu", "v2_feedback.cu", "v2_accum.cu", "v2_momentum.cu", "v2_layerwise.cu", "v2_clip.cu", "v2_ema.cu", "v2_lion.cu", "data_kernels.cu")]

nvcc_flags = ["-O3", "-lineinfo", "-std=c++17", "--use_fast_math",
              "-gencode", "arch=compute_90a,code=sm_90a"]

setup(
    name="atomo_b200",
    version="0.1.0",
    packages=["atomo_b200"],
    ext_modules=[CUDAExtension("atomo_b200._C", sources,
                               extra_compile_args={"cxx": ["-O3", "-std=c++17"], "nvcc": nvcc_flags})],
    cmdclass={"build_ext": BuildExtension.with_options(use_ninja=True)},
)
