"""Build the SIMT-emulator harness (test infrastructure): product kernels compiled as C++ for the CPU.

`build(sanitize=True)` builds the same sources with the alignment sanitizer into a second library: a misaligned load (a uint4
from an address that is not 16-byte aligned, as a GPU would fault on) stops the process with "runtime error: ... misaligned
address".  Load it in a child process only."""
import os
import subprocess
import sys

_DIR = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_DIR))
_CSRC = os.path.join(_ROOT, "cyberfabric-core_b200", "csrc")
SO = os.path.join(_DIR, "_build", "libcfbpe_sim.so")
SO_SANITIZE = os.path.join(_DIR, "_build", "libcfbpe_sim_align.so")


def build(force=False, sanitize=False):
    so = SO_SANITIZE if sanitize else SO
    srcs = [os.path.join(_DIR, "sim_harness.cpp"), os.path.join(_CSRC, "vocab.cpp")]
    deps = srcs + [os.path.join(_DIR, "cusim.h")] + [os.path.join(_CSRC, f) for f in os.listdir(_CSRC)]
    if not force and os.path.exists(so) and all(os.path.getmtime(so) >= os.path.getmtime(d) for d in deps):
        return so
    os.makedirs(os.path.dirname(so), exist_ok=True)
    tmp = so + ".%d.tmp" % os.getpid()       # another process may be loading the library: it sees the old one or the whole new one
    san = ["-fsanitize=alignment", "-fno-sanitize-recover=alignment"] if sanitize else []
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-fno-omit-frame-pointer",
           "-Wall", "-Wno-unused-function", "-Wno-unknown-pragmas", "-DCFBPE_SIM=1"] + san + ["-o", tmp] + srcs
    subprocess.check_call(cmd)
    os.replace(tmp, so)
    return so


if __name__ == "__main__":
    print(build(force=True, sanitize="--sanitize" in sys.argv[1:]))
