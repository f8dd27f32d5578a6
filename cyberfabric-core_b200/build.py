"""Build libcfbpe.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
import os
import subprocess
import sys

_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_DIR, "csrc")
SO = os.path.join(_DIR, "cfbpe", "libcfbpe.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def source_hash():
    """sha256 over csrc/* and include/cfbpe.h (what libcfbpe.so is built from)"""
    import hashlib
    h = hashlib.sha256()
    files = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC)) + [os.path.join(_DIR, "..", "include", "cfbpe.h")]
    for f in files:
        h.update(os.path.basename(f).encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()[:16]


def needs_build():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(_DIR, "..", "include", "cfbpe.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, defines=(), out=None):
    """defines/out: build an experimental variant (A/B timing of kernel parameters) next to the product library"""
    if out is None and not force and not needs_build():
        return SO
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
           "-Xcompiler", "-fPIC,-fvisibility=hidden,-O2", "-shared", "--cudart", "shared",
           "-Xptxas", "-v" if verbose else "-O3", '-DCFBPE_SRC_HASH="%s"' % source_hash(),
           os.path.join(CSRC, "cfbpe.cu"), os.path.join(CSRC, "vocab.cpp"), "-o", out or SO] + ["-D" + d for d in defines]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode:
        raise RuntimeError("nvcc failed")
    return out or SO


if __name__ == "__main__":
    print(build(force=True, verbose="-v" in sys.argv))
