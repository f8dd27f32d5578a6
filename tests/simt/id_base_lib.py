"""Build and bind the SIMT-emulator entries of id bases (test infrastructure; tests/simt/sim_id_base.cpp): encode cut into sub-batches
and rebased, special encode with the rebase before the splice, decode under bases, and the check of specials against a base's range.
The vocabularies are simlib.SimVocab objects: their packed table blobs go to the calls."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import build as _build  # noqa: E402
import simlib  # noqa: E402

SRC = os.path.join(_build._DIR, "sim_id_base.cpp")
SO = os.path.join(_build._DIR, "_build", "libcfbpe_sim_id_base.so")
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
        vp = C.c_void_p
        L.sim_encode_based.restype = C.c_int
        L.sim_encode_based.argtypes = [vp, C.c_uint32, vp, C.c_uint32, vp, vp, vp, vp, C.c_uint32, vp, C.c_uint64, vp]
        L.sim_encode_special_based.restype = C.c_int
        L.sim_encode_special_based.argtypes = [vp, C.c_uint32, vp, vp, vp, vp, vp, C.c_uint32, vp, vp, vp, vp, C.c_uint64, vp, C.POINTER(C.c_int)]
        L.sim_decode_based.restype = C.c_int
        L.sim_decode_based.argtypes = [vp, C.c_uint32, vp, vp, vp, vp, vp, C.c_uint32, vp, vp, vp, vp, C.c_uint64, vp]
        L.sim_special_in_id_range.restype = C.c_int
        L.sim_special_in_id_range.argtypes = [C.c_uint32, vp, vp, vp, C.c_uint32, C.c_uint32]
        _lib = L
    return _lib


def _blobs(vocabs):
    blobs = [v.blob() for v in vocabs]
    return blobs, (C.c_void_p * len(blobs))(*[b.ctypes.data for b in blobs])


def _bases(bases):
    return None if bases is None else np.ascontiguousarray(bases, dtype=np.uint32)


def _specials(specials_per_vocab, n_vocabs):
    """[{str: id} or None per vocabulary] -> (n, bytes, offsets, ids) arrays for special_tables (all None: no tables)"""
    if specials_per_vocab is None:
        return None, None, None, None
    n = np.zeros(n_vocabs, dtype=np.uint32)
    toks, ids = [], []
    for v, sp in enumerate(specials_per_vocab):
        for t, i in (sp or {}).items():
            toks.append(t.encode("utf-8"))
            ids.append(i)
        n[v] = len(sp or {})
    offs = np.zeros(len(toks) + 1 + n_vocabs, dtype=np.uint64)     # (each vocabulary's offsets start where the last one ended)
    offs[1:len(toks) + 1] = np.cumsum([len(t) for t in toks]) if toks else []
    return n, np.frombuffer(b"".join(toks) + b"\0", dtype=np.uint8).copy(), offs, np.asarray(ids + [0], dtype=np.uint32)


def encode(vocabs, prompts, bases=None, vocab_ids=None, cuts=None):
    """cfbpe_encode_batch as a pipelined host call with sub-batches at prompt indices `cuts` (None: one pass), rebased by
    `bases` (one per slot; None: not rebased) -> (rc, ids per prompt)"""
    data, offs = simlib.pack(prompts)
    n = len(prompts)
    cuts = np.asarray([0, n] if cuts is None else [0] + list(cuts) + [n], dtype=np.uint32)
    cap = int(offs[-1]) + 1
    ids = np.zeros(cap, dtype=np.uint32)
    out_off = np.zeros(n + 1, dtype=np.uint64)
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    blobs, barr = _blobs(vocabs)
    b = _bases(bases)
    rc = lib().sim_encode_based(barr, len(blobs), None if b is None else b.ctypes.data, n, data.ctypes.data, offs.ctypes.data,
                                None if vid is None else vid.ctypes.data, cuts.ctypes.data, len(cuts) - 1, ids.ctypes.data, cap, out_off.ctypes.data)
    return rc, ([ids[int(out_off[i]):int(out_off[i + 1])].tolist() for i in range(n)] if rc == 0 else None)


def encode_special(vocabs, prompts, specials, bases=None, vocab_ids=None):
    """cfbpe_encode_batch_special with every special allowed, rebased by `bases` -> (rc, ids per prompt, spliced)"""
    data, offs = simlib.pack(prompts)
    n = len(prompts)
    cap = int(offs[-1]) + 1
    ids = np.zeros(cap, dtype=np.uint32)
    out_off = np.zeros(n + 1, dtype=np.uint64)
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    blobs, barr = _blobs(vocabs)
    b = _bases(bases)
    ns, sb, so, si = _specials(specials, len(vocabs))
    spliced = C.c_int(0)
    rc = lib().sim_encode_special_based(barr, len(blobs), None if b is None else b.ctypes.data, ns.ctypes.data, sb.ctypes.data, so.ctypes.data,
                                        si.ctypes.data, n, data.ctypes.data, offs.ctypes.data, None if vid is None else vid.ctypes.data,
                                        ids.ctypes.data, cap, out_off.ctypes.data, C.byref(spliced))
    return rc, ([ids[int(out_off[i]):int(out_off[i + 1])].tolist() for i in range(n)] if rc == 0 else None), bool(spliced.value)


def decode(vocabs, seqs, bases=None, specials=None, vocab_ids=None):
    """decode of id sequences under `bases` with `specials` -> (rc, bytes per sequence)"""
    n = len(seqs)
    ids = np.asarray([i for s in seqs for i in s] + [0], dtype=np.uint32)
    id_off = np.zeros(n + 1, dtype=np.uint64)
    id_off[1:] = np.cumsum([len(s) for s in seqs]) if seqs else []
    cap = 64 * (len(ids) + 1)
    out = np.zeros(cap, dtype=np.uint8)
    out_off = np.zeros(n + 1, dtype=np.uint64)
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    blobs, barr = _blobs(vocabs)
    b = _bases(bases)
    ns, sb, so, si = _specials(specials, len(vocabs))
    rc = lib().sim_decode_based(barr, len(blobs), None if b is None else b.ctypes.data, None if ns is None else ns.ctypes.data,
                                None if sb is None else sb.ctypes.data, None if so is None else so.ctypes.data, None if si is None else si.ctypes.data,
                                n, ids.ctypes.data, id_off.ctypes.data, None if vid is None else vid.ctypes.data, out.ctypes.data, cap, out_off.ctypes.data)
    return rc, ([out[int(out_off[i]):int(out_off[i + 1])].tobytes() for i in range(n)] if rc == 0 else None)


def special_in_id_range(specials, base, n_ranks):
    """index of the first special of {str: id} whose id is an ordinary id under `base`, or -1"""
    ns, sb, so, si = _specials([specials], 1)
    return lib().sim_special_in_id_range(int(ns[0]), sb.ctypes.data, so.ctypes.data, si.ctypes.data, base, n_ranks)
