"""In-tree build of libxflow_b200.so (C++ host + hand-written sm_90a CUDA for the H100, one shared library).

    python -m xflow_b200.build [--force]

nvcc cross-compiles for sm_90a without a GPU.  The .so and the object files are build products
(git-ignored): every checkout builds them.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "xflow_b200", "csrc")
LIBDIR = os.path.join(ROOT, "xflow_b200", "lib")
LIB = os.path.join(LIBDIR, "libxflow_b200.so")
OBJDIR = os.path.join(ROOT, "build", "obj")

CU_SOURCES = ["kernels.cu", "step.cu", "step_lazy.cu", "step_fmc.cu", "step_mvm.cu", "step_ffm.cu", "step_det.cu", "capi.cu", "comm.cu", "mg_kernels.cu", "ingest.cu", "metric.cu", "admit.cu", "evict.cu", "weight.cu", "checkpoint.cu", "serve.cu", "rank.cu", "delta.cu", "validate.cu", "group_metric.cu"]
CC_SOURCES = ["loader.cc", "metrics.cc", "worker.cc"]
HEADERS = ["table.cuh", "mg.cuh", "serve.cuh", "forward.cuh", "metric.cuh", "kernels.h", "internal.h", "hash.h", os.path.join(ROOT, "include", "xflow_b200.h"),
           os.path.join(ROOT, "include", "xflow", "xflow.h")]

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden,-ffp-contract=off",
          "-I" + os.path.join(ROOT, "include"), "-I" + CSRC]


def _newer(src, dst):
    return (not os.path.exists(dst)) or os.path.getmtime(src) > os.path.getmtime(dst)


def build(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    # objects compiled with other flags (another architecture above all) are never reused
    stamp = os.path.join(OBJDIR, "flags")
    flags = " ".join([NVCC] + ARCH + COMMON)
    if not os.path.exists(stamp) or open(stamp).read() != flags:
        force = True
    hdr_paths = [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    hdr_paths = [h for h in hdr_paths if os.path.exists(h)]
    hdr_mtime = max(os.path.getmtime(h) for h in hdr_paths)
    objs = []
    procs = []
    for src in CU_SOURCES + CC_SOURCES:
        sp = os.path.join(CSRC, src)
        if not os.path.exists(sp):
            continue
        obj = os.path.join(OBJDIR, src + ".o")
        objs.append(obj)
        if force or _newer(sp, obj) or os.path.getmtime(obj) < hdr_mtime:
            cmd = [NVCC] + ARCH + COMMON + (["-x", "cu"] if src.endswith(".cc") else []) + ["-c", sp, "-o", obj]
            if verbose:
                print(" ".join(cmd))
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write("---- %s ----\n%s\n" % (src, out.decode(errors="replace")))
        elif verbose and out:
            sys.stderr.write(out.decode(errors="replace"))
    if failed:
        raise RuntimeError("nvcc failed")
    if force or procs or not os.path.exists(LIB):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-lpthread", "-ldl"]
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
    with open(stamp, "w") as f:
        f.write(flags)
    # the reference's CLI (src/model/main.cc) on top of the library
    bindir = os.path.join(ROOT, "xflow_b200", "bin")
    os.makedirs(bindir, exist_ok=True)
    exe = os.path.join(bindir, "xflow_lr")
    main_cc = os.path.join(CSRC, "main.cc")
    if force or _newer(main_cc, exe) or _newer(LIB, exe):
        subprocess.check_call([os.environ.get("CXX_HOST", "g++"), "-O2", "-std=c++17", "-I" + os.path.join(ROOT, "include"),
                               main_cc, "-o", exe, "-L" + LIBDIR, "-lxflow_b200", "-Wl,-rpath," + LIBDIR])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
