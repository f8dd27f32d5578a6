"""Build the SIMT-emulator harness (test infrastructure): product kernels compiled as C++ for the CPU."""
import os
import subprocess

_DIR = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_DIR))
_CSRC = os.path.join(_ROOT, "cyberfabric-core_b200", "csrc")
SO = os.path.join(_DIR, "_build", "libcfbpe_sim.so")


def build(force=False):
    srcs = [os.path.join(_DIR, "sim_harness.cpp"), os.path.join(_CSRC, "vocab.cpp")]
    deps = srcs + [os.path.join(_DIR, "cusim.h")] + [os.path.join(_CSRC, f) for f in os.listdir(_CSRC)]
    if not force and os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return SO
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    tmp = SO + ".%d.tmp" % os.getpid()       # another process may be loading SO: it sees the old library or the whole new one
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-fno-omit-frame-pointer",
           "-Wall", "-Wno-unused-function", "-Wno-unknown-pragmas", "-DCFBPE_SIM=1", "-o", tmp] + srcs
    subprocess.check_call(cmd)
    os.replace(tmp, SO)
    return SO


if __name__ == "__main__":
    print(build(force=True))
