"""Build and bind the SIMT-emulator entry of cfbpe_encode_batch_lossy (test infrastructure; tests/simt/sim_lossy.cpp).
The vocabularies are simlib.SimVocab objects: their packed table blobs go to the call."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import build as _build  # noqa: E402
import simlib  # noqa: E402

SRC = os.path.join(_build._DIR, "sim_lossy.cpp")
SO = os.path.join(_build._DIR, "_build", "libcfbpe_sim_lossy.so")
GUARDS = {"none": 0, "after": 1, "before": 2}     # where a guard page lies around the batch (sim_lossy.cpp, PlacedBytes)
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
        L.sim_encode_batch_lossy.restype = C.c_int
        L.sim_encode_batch_lossy.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_char_p, C.c_uint32, C.c_uint32,
                                             C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_int)]
        _lib = L
    return _lib


def encode_batch_lossy(vocabs, prompts, vocab_ids=None, out_cap=None, max_bytes=None, counts_only=False, misalign=0, fill=b"\0",
                       guard="none"):
    """cfbpe_encode_batch_lossy on the emulator: {"rc", "ids" (per prompt; None with counts_only), "offsets", "counts", "replaced",
    "repaired" (the repair ran), "r" (per prompt: the repaired bytes, when it ran), "dirty_lanes", "growth" (the scan's status)}.
    vocabs: simlib.SimVocab objects; misalign / fill / guard: where the batch's bytes lie (guard "after": exactly 32 bytes of
    padding, then an unmapped page; "before": an unmapped page before the first byte's page)"""
    data, offs = simlib.pack(prompts)
    total = int(offs[-1])
    n = len(prompts)
    cap = 3 * total + 1 if out_cap is None else out_cap
    ids = np.zeros(max(cap, 1), dtype=np.uint32)
    out_off = np.zeros(n + 1, dtype=np.uint64)
    counts = np.zeros(max(n, 1), dtype=np.uint32)
    replaced = np.full(max(n, 1), 0xFFFFFFFF, dtype=np.uint32)
    r = np.zeros(max(3 * total, 1), dtype=np.uint8)
    r_off = np.zeros(n + 1, dtype=np.uint64)
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    blobs = [v.blob() for v in vocabs]                   # (kept alive for the call)
    barr = (C.c_void_p * len(blobs))(*[b.ctypes.data for b in blobs])
    status = C.c_uint64(0)
    repaired = C.c_int(0)
    rc = lib().sim_encode_batch_lossy(barr, len(blobs), n, data.ctypes.data, offs.ctypes.data, None if vid is None else vid.ctypes.data,
                                      None if counts_only else ids.ctypes.data, cap, out_off.ctypes.data, counts.ctypes.data,
                                      replaced.ctypes.data, (1 << 32) - 4097 if max_bytes is None else max_bytes, misalign, bytes(fill),
                                      len(fill), GUARDS[guard], r.ctypes.data, r.size, r_off.ctypes.data, C.byref(status), C.byref(repaired))
    out = {"rc": rc, "offsets": out_off, "counts": counts[:n].tolist(), "replaced": replaced[:n].tolist(), "repaired": bool(repaired.value),
           "dirty_lanes": status.value >> 36, "growth": status.value & ((1 << 36) - 1), "ids": None, "r": None}
    if rc == 0 and not counts_only:
        out["ids"] = [ids[int(out_off[i]):int(out_off[i + 1])].tolist() for i in range(n)]
    if repaired.value:
        out["r"] = [r[int(r_off[i]):int(r_off[i + 1])].tobytes() for i in range(n)]
    return out
