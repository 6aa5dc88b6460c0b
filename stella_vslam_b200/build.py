"""In-tree build of libb200vslam.so (nvcc, sm_90a only).  Called by __graft_entry__.build().

The .so and the objects under build/ are build products (git-ignored).
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200vslam.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "-diag-suppress", "177"]
# per-file flags: the ORB kernels restate fp32 arithmetic that must never be contracted to FMA
SOURCES = {
    "abi_common.cu": [],
    "orb_kernels.cu": ["-fmad=false"],
    "match_kernels.cu": [],
    "lba_kernels.cu": [],
    # the rectification maps are built on the host in double; keep the host compiler from contracting them to FMA
    "rectify_kernels.cu": ["-Xcompiler", "-ffp-contract=off"],
    "random_array.cu": [],
    "pnp_kernels.cu": [],
    "essential_kernels.cu": [],
    "twoview_kernels.cu": [],
    # reproject_to_image (camera_model.cuh) is plain double arithmetic that must not be contracted, as in orb_kernels.cu
    "initialize_kernels.cu": ["-fmad=false"],
    # the pose-graph Jacobian is a central difference at delta 1e-9: no contraction on either side, as in tests/pgo_oracle.c
    "pgo_kernels.cu": ["-fmad=false", "-Xcompiler", "-ffp-contract=off"],
    # the transform optimiser's Jacobian is the same central difference (tests/transform_oracle.c)
    "transform_kernels.cu": ["-fmad=false", "-Xcompiler", "-ffp-contract=off"],
}


def nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _stale(out, deps):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    objs = []
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".inc", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "b200vslam.h"))
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for src, extra in SOURCES.items():
        sp = os.path.join(CSRC, src)
        if not os.path.exists(sp):
            continue
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, [sp] + headers):
            cmd = [nvcc()] + ARCH + COMMON + extra + ["-c", sp, "-o", obj]
            if verbose:
                print(" ".join(cmd), file=sys.stderr)
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
        if verbose and out.strip():
            print(out, file=sys.stderr)
    if force or procs or _stale(LIB, objs):
        cmd = [nvcc()] + ARCH + ["-shared", "-o", LIB] + objs + ["-cudart", "static", "-ldl"]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
