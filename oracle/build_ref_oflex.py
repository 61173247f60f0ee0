#!/usr/bin/env python
"""Rebuild the reference's `selective_scan_cuda_oflex` and `selective_scan_cuda_ndstate` extensions for sm_90a into oracle/_ref/.
TEST INFRASTRUCTURE ONLY -- the source of tests/golden/scan_ref_kernel_oflex.npz (oracle/ref_kernel_golden_oflex.py).

The sibling of oracle/build_ref.py (which builds selective_scan_cuda_core) with the same recipe: sources are compiled where they lie
in a checkout of the reference project next to this repository (../reference, or $VMB_REFERENCE_DIR; nothing is copied):
  Mamba/kernels/selective_scan/csrc/selective_scan/cusoflex/{selective_scan_oflex.cpp, selective_scan_core_fwd.cu, selective_scan_core_bwd.cu}
  Mamba/kernels/selective_scan/csrc/selective_scan/cusndstate/{selective_scan_ndstate.cpp, selective_scan_core_fwd.cu, selective_scan_core_bwd.cu}
with the reference's own nvcc flags (setup.py:115-131) except the -gencode list (setup.py:62-65 -> compute_90a/sm_90a).
Both compile unmodified.  Skipped when no checkout is present.
"""
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.environ.get("VMB_REFERENCE_DIR") or os.path.join(os.path.dirname(ROOT), "reference")
REF = os.path.join(REF_DIR, "Mamba", "kernels", "selective_scan", "csrc", "selective_scan")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")
MODULES = {"selective_scan_cuda_oflex": ("cusoflex", "selective_scan_oflex.cpp"),
           "selective_scan_cuda_ndstate": ("cusndstate", "selective_scan_ndstate.cpp")}
NVCC_FLAGS = ["-O3", "-std=c++17", "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__",
              "-U__CUDA_NO_BFLOAT16_OPERATORS__", "-U__CUDA_NO_BFLOAT16_CONVERSIONS__",
              "-U__CUDA_NO_BFLOAT162_OPERATORS__", "-U__CUDA_NO_BFLOAT162_CONVERSIONS__",
              "--expt-relaxed-constexpr", "--expt-extended-lambda", "--use_fast_math",
              "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo"]


def main():
    if not os.path.isdir(REF):
        print("reference sources not present; skipping")
        return
    from torch.utils.cpp_extension import load
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "4")
    for name, (sub, cpp) in MODULES.items():
        so = os.path.join(OUT, name + ".so")
        if os.path.exists(so):
            print("already built:", so)
            continue
        work = os.path.join(OUT, "_build_" + name)  # one build directory per module: the ninja files do not collide
        os.makedirs(work, exist_ok=True)
        load(name=name,
             sources=[f"{REF}/{sub}/{cpp}", f"{REF}/{sub}/selective_scan_core_fwd.cu", f"{REF}/{sub}/selective_scan_core_bwd.cu"],
             extra_include_paths=[REF], extra_cflags=["-O3", "-std=c++17"], extra_cuda_cflags=NVCC_FLAGS,
             build_directory=work, verbose=False, is_python_module=False)
        shutil.move(os.path.join(work, name + ".so"), so)  # keep only the .so
        shutil.rmtree(work)
        print("built", so)


if __name__ == "__main__":
    main()
