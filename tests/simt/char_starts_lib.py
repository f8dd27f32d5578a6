"""Build and bind the SIMT-emulator entry of cfbpe_encode_batch_char_starts (test infrastructure; tests/simt/sim_char_starts.cpp).
The vocabularies are simlib.SimVocab objects: their packed table blobs go to the call."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import build as _build  # noqa: E402
import simlib  # noqa: E402

UNIT_CODEPOINT, UNIT_UTF16 = 0, 1      # what a unit start counts (cfbpe_encode_batch_char_starts)
SRC = os.path.join(_build._DIR, "sim_char_starts.cpp")
SO = os.path.join(_build._DIR, "_build", "libcfbpe_sim_char_starts.so")
_lib = None


def build(force=False):
    deps = [SRC, os.path.join(_build._DIR, "cusim.h")] + [os.path.join(_build._CSRC, f) for f in os.listdir(_build._CSRC)]
    if not force and os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return SO
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    tmp = SO + ".%d.tmp" % os.getpid()       # another process may be loading the library: it sees the old one or the whole new one
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-Wl,--no-undefined",
                           "-Wall", "-Wno-unused-function", "-Wno-unknown-pragmas", "-DCFBPE_SIM=1", "-o", tmp, SRC])
    os.replace(tmp, SO)
    return SO


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.sim_encode_batch_char_starts.restype = C.c_int
        L.sim_encode_batch_char_starts.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                                   C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def encode_char_starts(vocabs, prompts, unit, vocab_ids=None, out_cap=None, null=None):
    """encode with token starts in `unit`: (rc, ids, starts, offsets, counts, lens); vocabs: simlib.SimVocab objects; null: "ids",
    "starts" or "lens" to pass as NULL"""
    data, offs = simlib.pack(prompts)
    n = len(prompts)
    cap = int(offs[-1]) + 1 if out_cap is None else out_cap
    ids = np.zeros(max(cap, 1), dtype=np.uint32)
    starts = np.full(max(cap, 1), 0xFFFFFFFF, dtype=np.uint32)
    out_off = np.zeros(n + 1, dtype=np.uint64)
    counts = np.zeros(max(n, 1), dtype=np.uint32)
    lens = np.full(max(n, 1), 0xFFFFFFFF, dtype=np.uint32)
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    blobs = [v.blob() for v in vocabs]                   # (kept alive for the call)
    barr = (C.c_void_p * len(blobs))(*[b.ctypes.data for b in blobs])
    rc = lib().sim_encode_batch_char_starts(barr, len(blobs), n, data.ctypes.data, offs.ctypes.data,
                                            None if vid is None else vid.ctypes.data, unit, None if null == "ids" else ids.ctypes.data,
                                            None if null == "starts" else starts.ctypes.data, cap, out_off.ctypes.data, counts.ctypes.data,
                                            None if null == "lens" else lens.ctypes.data)
    n_tok = int(out_off[-1]) if rc == 0 else 0
    return rc, ids[:n_tok], starts[:n_tok], out_off, counts[:n], lens[:n]
