"""Builds the in-tree native libraries (nvcc, sm_90a only).

`python -m sceneverse_b200.build` or `__graft_entry__.build()`.  nvcc cross-compiles without a
GPU; the resulting .so files live in sceneverse_b200/lib/ (git-ignored).
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "sceneverse_b200", "csrc")
LIBDIR = os.path.join(ROOT, "sceneverse_b200", "lib")
INCLUDE = os.path.join(ROOT, "include")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]

# library name -> sources (relative to csrc/)
LIBS = {
    "libsvpointops.so": ["pointops.cu", "sa_sample.cu", "fps_coop.cu", "scene_prep.cu", "eval_targets.cu"],
    "libsvgps.so": ["gps_common.cu", "sa_mlp.cu", "gemm.cu", "attention.cu", "attention_bwd.cu", "pairwise_locs.cu", "cross_entropy.cu", "norm_allgather.cu", "layer_norm.cu", "colsum.cu", "train_ops.cu", "pn_train.cu", "qa_ops.cu", "eval_metrics.cu"],
}


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_all(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    headers = [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)] + \
              [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    built = []
    for lib, srcs in LIBS.items():
        out = os.path.join(LIBDIR, lib)
        srcs = [os.path.join(CSRC, s) for s in srcs]
        if force or _newer(out, srcs + headers):
            tmp = out + ".%d.tmp" % os.getpid()
            cmd = [nvcc] + NVCC_FLAGS + ["-I" + INCLUDE, "-I" + CSRC, "-o", tmp] + srcs
            if verbose:
                print(" ".join(cmd), flush=True)
            subprocess.check_call(cmd)
            os.replace(tmp, out)
            built.append(out)
    return built


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv, verbose=True))
