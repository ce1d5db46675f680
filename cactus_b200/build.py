"""Build libbarb200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m cactus_b200.build
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libbarb200.so")
SOURCES = ["poa_kernel.cu", "poa_trace_kernel.cu", "guide_tree.cu", "barb200.cu", "host_bar.cpp", "host_end_trace.cpp","pecan.cu", "pecan_plan.cpp", "mum_anchor.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC,-fopenmp,-O3,-Wall,-Wno-unused-function", "-Xptxas", "-v"]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    # every file under csrc/ (sources AND headers) plus the public header: an edited .cuh must never leave a stale library behind
    deps = glob.glob(os.path.join(CSRC, "*")) + [os.path.join(HERE, "..", "include", "barb200.h"), os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, extra_flags=None, out_path=None):
    """extra_flags / out_path: development aid (A/B builds of differently tuned kernels into another file; see scripts/)"""
    if out_path is None and not force and not needs_build():
        return LIB
    objs = []
    bdir = os.path.join(HERE, "_build" if out_path is None else "_build_" + os.path.basename(out_path))
    os.makedirs(bdir, exist_ok=True)
    procs = []
    for s in SOURCES:
        o = os.path.join(bdir, os.path.splitext(s)[0] + ".o")
        cmd = [NVCC] + FLAGS + list(extra_flags or []) + ["-x", "cu", "-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(o)
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError("nvcc failed on %s" % s)
        if verbose:
            sys.stderr.write(out)
    target = LIB if out_path is None else out_path
    cmd = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", target] + objs + ["-Xcompiler", "-fopenmp", "-lcudart", "-lgomp"]
    subprocess.check_call(cmd)
    return target


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
