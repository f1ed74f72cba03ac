"""Builds lib/libfsr1_b200.so (the C-ABI library with the sm_90a kernels for H100) in-tree with nvcc.

    python fidelityfx-fsr_b200/build.py [--force]

nvcc cross-compiles for sm_90a without a GPU; the resulting .so is git-ignored.  cudart is linked
statically so the library loads in a process that has no CUDA driver (symbol-export tests) and next
to torch's own runtime.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = [os.path.join(HERE, "csrc", f) for f in
       ("fsr1_direct.cu", "fsr1_easu_tiled.cu", "fsr1_easu_f32.cu", "fsr1_rcas_packed.cu", "fsr1_rcas_in.cu", "fsr1_rcas_f32.cu", "fsr1_href.cu", "fsr1_hx2.cu", "fsr1_pointwise.cu", "fsr1_shard.cu", "fsr1_fused.cu", "fsr1_capi.cu")]
DEPS = SRC + [os.path.join(HERE, "csrc", "fsr1_common.cuh"), os.path.join(HERE, "csrc", "fsr1_easu_common.cuh"), os.path.join(HERE, "csrc", "fsr1_easu_quad.cuh"), os.path.join(HERE, "csrc", "fsr1_rcas_math.cuh"), os.path.join(HERE, "csrc", "fsr1_post.cuh"), os.path.join(HERE, "csrc", "fsr1_r11.cuh"),
              os.path.join(HERE, "..", "include", "fsr1_b200.h"),
              os.path.join(HERE, "..", "include", "fsr1_host.h"), os.path.abspath(__file__)]  # this file: the flags
OUT = os.path.join(HERE, "lib", "libfsr1_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
         "-Xcompiler", "-fPIC", "-shared", "-cudart", "static"]


def up_to_date():
    if not os.path.exists(OUT):
        return False
    t = os.path.getmtime(OUT)
    return all(os.path.getmtime(d) <= t for d in DEPS)


def build(force=False, verbose=False):
    if not force and up_to_date():
        return OUT
    if not os.path.exists(NVCC):
        if os.path.exists(OUT):
            return OUT  # GPU box without a toolkit: use the prebuilt library
        raise RuntimeError("nvcc not found at %s and no prebuilt %s" % (NVCC, OUT))
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT] + SRC
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed building %s" % OUT)
    if verbose:
        sys.stderr.write(r.stderr)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
