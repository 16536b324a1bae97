"""In-tree build of libb200meters.so (C ABI of include/b200meters.h) for the H100 (sm_90a).

    python meters.lv2_b200/build.py [--force] [--verbose]

Every .cu under csrc/ is compiled with
    nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false
(no FMA contraction: the per-sample pipelines must round exactly like the reference's SSE2 build,
Makefile:35 of the reference; kernels that want FMA call fmaf()/__fma_rn explicitly) and linked into
meters.lv2_b200/libb200meters.so next to this file, where the package loads it from.  nvcc cross-compiles
without a GPU.
"""
import concurrent.futures as cf
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libb200meters.so")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC,-O2,-ffp-contract=off,-fno-fast-math,-fvisibility=hidden",
    "-Xptxas", "-v", "-I", os.path.join(HERE, "..", "include"),
]


def _newer(src, dst, extra=()):
    if not os.path.exists(dst):
        return True
    t = os.path.getmtime(dst)
    return any(os.path.getmtime(p) > t for p in (src, *extra))


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(HERE, "..", "include", "b200meters.h"))
    hdrs.append(os.path.abspath(__file__))
    jobs = []
    for s in srcs:
        src, obj = os.path.join(CSRC, s), os.path.join(OBJ, s[:-3] + ".o")
        if force or _newer(src, obj, hdrs):
            jobs.append((src, obj))

    def run(job):
        src, obj = job
        p = subprocess.run([NVCC, *FLAGS, "-c", src, "-o", obj], capture_output=True, text=True)
        return job, p

    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for (src, obj), p in ex.map(run, jobs):
                log = (p.stdout + p.stderr)
                with open(obj[:-2] + ".ptxas.log", "w") as f:
                    f.write(log)
                if p.returncode != 0:
                    sys.stderr.write(log)
                    raise RuntimeError("nvcc failed on %s" % src)
                if verbose:
                    sys.stderr.write(log)
    objs = [os.path.join(OBJ, s[:-3] + ".o") for s in srcs]
    if jobs or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a",
               "-Xcompiler", "-fPIC", "-Xlinker", "--no-undefined"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        if p.returncode != 0:
            sys.stderr.write(p.stdout + p.stderr)
            raise RuntimeError("link failed")
    # the plain-C LV2 host used for per-instance throughput measurements (meters.lv2_b200/host/lv2_host.c)
    hsrc, hbin = os.path.join(HERE, "host", "lv2_host.c"), os.path.join(HERE, "host", "lv2_host")
    if os.path.exists(hsrc) and (force or _newer(hsrc, hbin)):
        p = subprocess.run(["gcc", "-O2", "-Wall", "-o", hbin, hsrc, "-ldl", "-lpthread"], capture_output=True, text=True)
        if p.returncode != 0:
            sys.stderr.write(p.stdout + p.stderr)
            raise RuntimeError("gcc failed on %s" % hsrc)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
