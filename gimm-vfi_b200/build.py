"""In-tree build of the native library (nvcc cross-compiles sm_90a without a GPU)."""
import os
import time
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["ops_pointwise.cu", "corr.cu", "conv.cu", "conv_tc.cu", "conv_halo.cu", "conv_wide.cu", "corr_gemm.cu", "hyponet.cu", "ops_tokens.cu", "flowformer.cu", "engine.cu", "c_api.cu"]
OUT = os.path.join(HERE, "libgimmvfi_b200.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
              "-diag-suppress", "550"]


def _stale(out, srcs):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    deps = list(srcs) + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    deps.append(os.path.join(os.path.dirname(HERE), "include", "gimmvfi_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build_cuda(force=False, verbose=False) -> str:
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    if not force and not _stale(OUT, srcs):
        return OUT
    nvcc = os.environ.get("NVCC", "nvcc")
    t_start = time.time()   # the library is stamped with the time the build STARTED: a source edited while nvcc runs stays newer than it
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for s in srcs:
        o = os.path.join(HERE, "build", os.path.basename(s) + ".o")
        objs.append(o)
        cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o] + (["-Xptxas", "-v"] if verbose else [])
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out.decode(errors="replace"))
        if p.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    subprocess.check_call([nvcc, "-shared", "-o", OUT] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
    os.utime(OUT, (t_start, t_start))
    return OUT


if __name__ == "__main__":
    print(build_cuda(force="--force" in sys.argv, verbose="-v" in sys.argv))
