#!/usr/bin/env python
"""Rebuild the reference's own CUDA extension (selective_scan_cuda_core) for sm_90a into oracle/_ref/.
TEST / BASELINE INFRASTRUCTURE ONLY -- the "kernel to beat", and the source of tests/golden/scan_ref_kernel.npz.

Sources are compiled where they lie in a checkout of the reference project next to this repository (../reference, or
$VMB_REFERENCE_DIR; nothing is copied):
  Mamba/kernels/selective_scan/csrc/selective_scan/cus/{selective_scan.cpp, selective_scan_core_fwd.cu, selective_scan_core_bwd.cu}
with the reference's own nvcc flags (setup.py:115-131) except the -gencode list (setup.py:62-65 -> compute_90a/sm_90a).
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.environ.get("VMB_REFERENCE_DIR") or os.path.join(os.path.dirname(ROOT), "reference")
REF = os.path.join(REF_DIR, "Mamba", "kernels", "selective_scan", "csrc", "selective_scan")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


def main():
    if not os.path.isdir(REF):
        print("reference sources not present; skipping")
        return
    so = os.path.join(OUT, "selective_scan_cuda_core.so")
    if os.path.exists(so):
        print("already built:", so)
        return
    os.makedirs(OUT, exist_ok=True)
    from torch.utils.cpp_extension import load
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "4")
    load(name="selective_scan_cuda_core",
         sources=[f"{REF}/cus/selective_scan.cpp", f"{REF}/cus/selective_scan_core_fwd.cu", f"{REF}/cus/selective_scan_core_bwd.cu"],
         extra_include_paths=[REF],
         extra_cflags=["-O3", "-std=c++17"],
         extra_cuda_cflags=["-O3", "-std=c++17", "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__",
                            "-U__CUDA_NO_BFLOAT16_OPERATORS__", "-U__CUDA_NO_BFLOAT16_CONVERSIONS__",
                            "-U__CUDA_NO_BFLOAT162_OPERATORS__", "-U__CUDA_NO_BFLOAT162_CONVERSIONS__",
                            "--expt-relaxed-constexpr", "--expt-extended-lambda", "--use_fast_math",
                            "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo"],
         build_directory=OUT, verbose=False, is_python_module=False)
    for f in os.listdir(OUT):  # keep only the .so
        if not f.endswith(".so"):
            os.remove(os.path.join(OUT, f))
    print("built", so)


if __name__ == "__main__":
    main()
