"""Build libdpb200.so in-tree with nvcc for sm_90a (H100) (no torch extension machinery: the library is a plain
C-ABI shared object, loaded with ctypes)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdpb200.so")
SOURCES = ["api.cu", "gemm_simt.cu", "norm.cu", "pointwise.cu", "optim.cu", "conv_tc.cu", "conv_bf16.cu", "fid.cu"]


def _newer(src_paths, target):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(p) > t for p in src_paths)


def build(force=False, verbose=False):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps = srcs + [os.path.join(CSRC, "common.cuh"), os.path.join(ROOT, "include", "dpb200.h")]
    deps += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    if not force and not _newer(deps, LIB):
        return LIB
    have_tc = os.path.exists(os.path.join(CSRC, "conv_tc.cu"))
    objs = []
    for s in srcs:
        o = s[:-3] + ".o"
        if force or _newer([s] + [d for d in deps if not d.endswith(".cu")], o):
            cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
                   "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-c", s, "-o", o]
            if have_tc:
                cmd.insert(1, "-DDPB200_HAVE_TC")
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                raise RuntimeError("nvcc failed for %s" % s)
            if verbose:
                sys.stderr.write(r.stderr)
        objs.append(o)
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
