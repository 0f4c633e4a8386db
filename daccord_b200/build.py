"""Build the sm_90a (H100) C-ABI library (and the host tools) in-tree with nvcc / g++."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BUILD = os.path.join(HERE, "_build")
LIB = os.path.join(BUILD, "libdaccord_b200.so")
HOST_LIB = os.path.join(BUILD, "libdaccord_host.so")
CLOCKS_LIB = os.path.join(BUILD, "libdaccord_b200_clocks.so")      # measurement build (build_stage_clocks), never loaded by the package
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-fmad=false",
              "-Xcompiler", "-fPIC,-O3,-ffp-contract=off,-fopenmp", "-shared"]


def _newer(out, deps):
    return (not os.path.exists(out)) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps if os.path.exists(d))


def _nvcc(out, defines, force, verbose):
    csrc = os.path.join(HERE, "csrc")
    deps = [os.path.join(csrc, f) for f in os.listdir(csrc) if os.path.isfile(os.path.join(csrc, f))] + [os.path.join(ROOT, "include", "daccord_b200.h")]
    if force or _newer(out, deps):
        srcs = [os.path.join(csrc, f) for f in sorted(os.listdir(csrc)) if f.endswith(".cu")]
        cmd = ["nvcc"] + NVCC_FLAGS + defines + (["-Xptxas", "-v"] if verbose else []) + ["-o", out] + srcs + ["-lcudart", "-lgomp"]
        env = dict(os.environ)
        env["PATH"] = "/usr/bin:" + env.get("PATH", "")      # system g++ (the /opt/gcc wrapper lacks libgomp.spec)
        subprocess.check_call(cmd, env=env)


def build_stage_clocks(force=False, verbose=False):
    """the library with per-stage clocks in the window kernels (-DDCU_STAGE_CLOCKS), for tools/stage_clocks.py only"""
    os.makedirs(BUILD, exist_ok=True)
    _nvcc(CLOCKS_LIB, ["-DDCU_STAGE_CLOCKS"], force, verbose)
    return CLOCKS_LIB


def build(force=False, verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    csrc = os.path.join(HERE, "csrc")
    _nvcc(LIB, [], force, verbose)
    host_src = os.path.join(csrc, "host", "hostlib.cpp")  # noqa
    host_deps = [os.path.join(csrc, "host", f) for f in os.listdir(os.path.join(csrc, "host"))] + [os.path.join(ROOT, "include", "daccord_b200.h"),
                                                                                               os.path.join(csrc, "profile_core.cuh"),
                                                                                               os.path.join(csrc, "inqual_core.cuh"),
                                                                                               os.path.join(csrc, "exqual_core.cuh"),
                                                                                               os.path.join(csrc, "proper_core.cuh")]
    if force or _newer(HOST_LIB, host_deps):
        subprocess.check_call(["/usr/bin/g++", "-O3", "-g", "-std=c++17", "-march=x86-64-v2", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                               "-o", HOST_LIB, host_src])
    cli = os.path.join(BUILD, "daccord")
    if force or _newer(cli, host_deps + [LIB]):
        subprocess.check_call(["/usr/bin/g++", "-O3", "-g", "-std=c++17", "-march=x86-64-v2", "-ffp-contract=off", "-fopenmp", "-pthread", "-o", cli,
                               os.path.join(csrc, "host", "daccord_main.cpp"), "-L" + BUILD, "-ldaccord_b200", "-Wl,-rpath,$ORIGIN"])
    iqv = os.path.join(BUILD, "computeintrinsicqv")
    if force or _newer(iqv, host_deps + [LIB]):
        subprocess.check_call(["/usr/bin/g++", "-O3", "-g", "-std=c++17", "-march=x86-64-v2", "-ffp-contract=off", "-fopenmp", "-pthread", "-o", iqv,
                               os.path.join(csrc, "host", "computeintrinsicqv.cpp"), "-L" + BUILD, "-ldaccord_b200", "-Wl,-rpath,$ORIGIN"])
    xqv = os.path.join(BUILD, "computeextrinsicqv")
    if force or _newer(xqv, host_deps + [LIB]):
        subprocess.check_call(["/usr/bin/g++", "-O3", "-g", "-std=c++17", "-march=x86-64-v2", "-ffp-contract=off", "-fopenmp", "-pthread", "-o", xqv,
                               os.path.join(csrc, "host", "computeextrinsicqv.cpp"), "-L" + BUILD, "-ldaccord_b200", "-Wl,-rpath,$ORIGIN"])
    lfa = os.path.join(BUILD, "lasfilteralignments")
    if force or _newer(lfa, host_deps + [LIB]):
        subprocess.check_call(["/usr/bin/g++", "-O3", "-g", "-std=c++17", "-march=x86-64-v2", "-ffp-contract=off", "-fopenmp", "-pthread", "-o", lfa,
                               os.path.join(csrc, "host", "lasfilteralignments.cpp"), "-L" + BUILD, "-ldaccord_b200", "-Wl,-rpath,$ORIGIN"])
    return LIB


if __name__ == "__main__":
    print((build_stage_clocks if "--stage-clocks" in sys.argv else build)(force="--force" in sys.argv, verbose="-v" in sys.argv))
