"""Builds libnnnoiseless_b200.so (hand-written sm_90a CUDA kernels + the C ABI of include/rnnoise.h).

In-tree build with nvcc (cross-compiles without a GPU):
    python -m nnnoiseless_b200.build [--force]
The .so is git-ignored but travels to the GPU box with the tree.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# NNB_VARIANT=prof builds a second library with the clock64 phase profiles of the pitch kernel and the wgmma GRU kernel
# compiled in (lib/libnnnoiseless_b200_prof.so, selected at run time with NNB_LIB=<path>); the default build is untouched.
VARIANT = os.environ.get("NNB_VARIANT", "")
OBJ = os.path.join(HERE, "_obj" + ("_" + VARIANT if VARIANT else ""))
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libnnnoiseless_b200%s.so" % ("_" + VARIANT if VARIANT else ""))
VARIANT_FLAGS = {"": [], "prof": ["-DPITCH_PROFILE", "-DRNN_TC_PROFILE"]}[VARIANT]
WEIGHTS = os.path.join(HERE, "data", "weights.rnn")
BINDIR = os.path.join(HERE, "bin")
CLI = os.path.join(BINDIR, "nnnoiseless-b200")
CLI_SRC = os.path.join(HERE, "..", "cli", "nnnoiseless_cli.cpp")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]

# (source, extra flags).  exact.cu is the order-exact pitch path: no FMA contraction.
UNITS = [
    ("exact.cu", ["-fmad=false"]),
    ("pitch.cu", ["-fmad=false"]),
    ("train.cu", ["-fmad=false"]),
    ("fit.cu", []),
    ("spectral_warp.cu", []),
    ("rnn_mma.cu", []),
    ("rnn_tc.cu", []),
    ("frontend.cu", []),
    ("resample_stream.cu", []),
    ("state.cu", []),
    ("host.cu", []),
]
HEADERS = ["abi.hpp", "common.cuh", "fft480.cuh", "model.hpp", "audio_io.hpp", "owners.hpp", os.path.join("..", "..", "include", "rnnoise.h")]


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(LIBDIR, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS] + [os.path.abspath(__file__)]
    objs = []
    logs = []
    for src, extra in UNITS:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src + ".o")
        objs.append(o)
        if force or _newer(o, [s] + hdrs):
            cmd = [NVCC] + ARCH + COMMON + extra + VARIANT_FLAGS + os.environ.get("NNB_EXTRA_NVCC", "").split() + ["-c", s, "-o", o]
            r = subprocess.run(cmd, capture_output=True, text=True)
            logs.append(r.stderr)
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                raise RuntimeError("nvcc failed on " + src)
            if verbose:
                sys.stderr.write(r.stderr)
    s = os.path.join(CSRC, "model.cpp")
    o = os.path.join(OBJ, "model.cpp.o")
    objs.append(o)
    if force or _newer(o, [s, WEIGHTS] + hdrs):
        cmd = ["g++", "-O2", "-std=c++17", "-fPIC", '-DNNB_WEIGHTS_PATH="%s"' % WEIGHTS, "-c", s, "-o", o]
        subprocess.run(cmd, check=True)
    s = os.path.join(CSRC, "audio_io.cpp")
    o = os.path.join(OBJ, "audio_io.cpp.o")
    objs.append(o)
    if force or _newer(o, [s] + hdrs):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-Wall", "-c", s, "-o", o], check=True)
    if force or _newer(LIB, objs):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs
        subprocess.run(cmd, check=True)
    # the command-line front-end (src/nnnoiseless.rs): a thin main() over rnnoise_denoise_files
    os.makedirs(BINDIR, exist_ok=True)
    if not VARIANT and (force or _newer(CLI, [CLI_SRC, LIB] + hdrs)):
        cmd = ["g++", "-O2", "-std=c++17", "-Wall", CLI_SRC, "-o", CLI, "-L" + LIBDIR, "-lnnnoiseless_b200",
               "-Wl,-rpath,$ORIGIN/../lib"]
        subprocess.run(cmd, check=True)
    with open(os.path.join(OBJ, "ptxas.log"), "a") as f:
        f.write("".join(logs))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
