"""Build libb200gs.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python gaussian-splatting-lightning_b200/build.py [--force] [--verbose]
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libb200gs.so")
SOURCES = ["api.cu", "project.cu", "binning.cu", "blend.cu", "loss.cu", "optim.cu", "knn.cu", "mcmc.cu", "isect.cu", "bilagrid.cu", "appearance.cu", "exposure.cu", "depth_loss.cu", "visibility.cu", "gauss_reg.cu", "normal_reg.cu", "similarity_reg.cu", "glossy.cu", "swag.cu", "gs4d.cu"]
HEADERS = [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "geometry.cuh"), os.path.join(CSRC, "onesweep.cuh"), os.path.join(CSRC, "knn_grid.h"), os.path.join(CSRC, "ssim.cuh"), os.path.join(CSRC, "sh.cuh"), os.path.join(CSRC, "warp_mma.cuh"),
           os.path.join(os.path.dirname(HERE), "include", "b200gs.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17"] + ARCH + ["-lineinfo", "--use_fast_math",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"] + os.environ.get("B200GS_NVCC_FLAGS", "").split()


def _stale(obj, src):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    return any(os.path.getmtime(p) > t for p in [src] + HEADERS)


def build(force=False, verbose=False):
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    # objects and library built with other flags (another architecture) are never reused: the flags are part of the key
    stamp, flags = os.path.join(HERE, "build", "flags.txt"), " ".join([NVCC] + FLAGS)
    if not os.path.exists(stamp) or open(stamp).read() != flags:
        force = True
        if os.path.exists(stamp):
            os.remove(stamp)
    objs, procs = [], []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(HERE, "build", s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, src):
            cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            print(f"--- {s} ---\n{out}")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    if procs or not os.path.exists(OUT):
        cmd = [NVCC, "-shared"] + ARCH + ["-Xcompiler", "-fPIC", "-o", OUT] + objs
        subprocess.check_call(cmd)
    with open(stamp, "w") as f:
        f.write(flags)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
