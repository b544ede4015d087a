"""Build libtw_b200.so (hand-written sm_90a CUDA for the H100 + C ABI) in-tree with nvcc.

    python -m traceweaver_b200.csrc.build [--force] [--verbose] [--prof | --timeline]

--prof builds libtw_b200_prof.so, with the phase counters of the scoring, stitch and refit kernels
(TW_PROFILE_PHASES; scripts/phase_profile.py reads them); --timeline builds libtw_b200_timeline.so,
with the stitch kernel's warp timeline (TW_STITCH_TIMELINE; scripts/stitch_timeline.py).  The product
never loads these measurement builds: a script loads one when TW_B200_SO names it.

nvcc cross-compiles without a GPU; the .so files are build products and stay out of git."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-shared", "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "-Xptxas", "-v",
         "-Wno-deprecated-gpu-targets"]


def sources():
    return sorted(glob.glob(os.path.join(HERE, "*.cu")))


def stale(out):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    deps = sources() + glob.glob(os.path.join(HERE, "*.cuh")) + \
        [os.path.join(PKG, "..", "include", "traceweaver_b200.h"), os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, defines=(), name=None):
    """libtw_b200.so, or libtw_b200_<name>.so compiled with -D<d> for every d in `defines`."""
    if defines and not name:
        raise ValueError("a build with extra defines needs a name of its own")
    suffix = f"_{name}" if name else ""
    out = os.path.join(PKG, f"libtw_b200{suffix}.so")
    if not force and not stale(out):
        return out
    cmd = [NVCC] + FLAGS + [f"-D{d}" for d in defines] + ["-o", out] + sources()
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    log = os.path.join(HERE, f"build{suffix}.log")
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + res.stdout)
    if verbose or res.returncode != 0:
        print(res.stdout)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed ({res.returncode}); see {log}")
    return out


if __name__ == "__main__":
    name, defines = None, ()
    if "--prof" in sys.argv:
        name, defines = "prof", ("TW_PROFILE_PHASES",)
    elif "--timeline" in sys.argv:
        name, defines = "timeline", ("TW_STITCH_TIMELINE",)
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv, defines=defines, name=name))
