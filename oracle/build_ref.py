"""Compile the REFERENCE's own CUDA kernels for sm_90a from the sources where they lie under
/root/reference, outputs only into oracle/_ref/ (git-ignored, travels to the GPU box).

    python oracle/build_ref.py [exllamav2] [marlin]

These are the on-box baselines the north_star names (reference Marlin TFLOPS at M>=64, exllamav2 decode)
and an additional parity witness on the GPU.  TEST/BENCH INFRASTRUCTURE: never imported by the product.
No reference source is copied into this repository; the reference's setup.py is not run
(source lists follow /root/reference/setup.py:172-246).
"""
import os
import sys

REF = "/root/reference/autogptq_extension"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")

EXTS = {
    "exllamav2_kernels": [f"{REF}/exllamav2/ext.cpp", f"{REF}/exllamav2/cuda/q_matrix.cu", f"{REF}/exllamav2/cuda/q_gemm.cu"],
    "autogptq_marlin_cuda": [f"{REF}/marlin/marlin_cuda.cpp", f"{REF}/marlin/marlin_cuda_kernel.cu", f"{REF}/marlin/marlin_repack.cu"],
}
ALIASES = {"exllamav2": "exllamav2_kernels", "marlin": "autogptq_marlin_cuda"}


def build(name):
    from torch.utils import cpp_extension

    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("CXX", "/usr/bin/g++")
    os.environ.setdefault("MAX_JOBS", "4")
    bdir = os.path.join(OUT, name)
    os.makedirs(bdir, exist_ok=True)
    cpp_extension.load(name=name, sources=EXTS[name], build_directory=bdir, verbose=True, is_python_module=False,
                       extra_cuda_cflags=["-O3", "--expt-relaxed-constexpr", "-lineinfo"])
    print("built", os.path.join(bdir, name + ".so"))


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit("reference tree not present (the GPU box only uses the prebuilt oracle/_ref)")
    for a in (sys.argv[1:] or ["exllamav2", "marlin"]):
        build(ALIASES.get(a, a))
