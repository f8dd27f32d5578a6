"""ctypes binding of the special-token emulator harness (test infrastructure; tests/simt/sim_special.cpp)."""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import build_special as _build  # noqa: E402

EINVAL, ENOSPC, EILSEQ, EBADMSG = -22, -28, -84, -74
ORDINARY, ALLOW, DISALLOW = 0, 1, 2
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(_build.build())
        L.sim_vocab_build.restype = C.c_void_p
        L.sim_vocab_build.argtypes = [C.c_char_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p, C.c_size_t]
        L.sim_vocab_free.argtypes = [C.c_void_p]
        L.sim_specials_build.restype = C.c_void_p
        L.sim_specials_build.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_char_p, C.c_size_t]
        L.sim_specials_free.argtypes = [C.c_void_p]
        L.sim_encode_batch_special.restype = C.c_int
        L.sim_encode_batch_special.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint64)]
        L.sim_decode_batch_special.restype = C.c_int
        L.sim_decode_batch_special.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_uint64, C.c_void_p]
        _lib = L
    return _lib


class Vocab:
    def __init__(self, file_bytes, pattern, max_ranks):
        err = C.create_string_buffer(256)
        self._h = lib().sim_vocab_build(file_bytes, len(file_bytes), 0, pattern, max_ranks, err, 256)
        if not self._h:
            raise ValueError(err.value.decode())

    def __del__(self):
        if getattr(self, "_h", None):
            lib().sim_vocab_free(self._h)


class Specials:
    """the special-token table of one vocabulary ({str or bytes: id}, order = special index)"""

    def __init__(self, specials):
        toks = [t.encode("utf-8") if isinstance(t, str) else bytes(t) for t in specials]
        self.tokens = toks
        offs = np.zeros(len(toks) + 1, dtype=np.uint64)
        if toks:
            offs[1:] = np.cumsum([len(t) for t in toks])
        data = np.frombuffer(b"".join(toks) + b"\0", dtype=np.uint8).copy()
        ids = np.asarray([int(v) for v in specials.values()] + [0], dtype=np.uint32)
        rc = C.c_int(0)
        err = C.create_string_buffer(256)
        self._h = lib().sim_specials_build(len(toks), data.ctypes.data, offs.ctypes.data, ids.ctypes.data, C.byref(rc), err, 256)
        self.rc, self.err = rc.value, err.value.decode()

    def __del__(self):
        if getattr(self, "_h", None):
            lib().sim_specials_free(self._h)


def pack(prompts):
    offs = np.zeros(len(prompts) + 1, dtype=np.uint64)
    if prompts:
        offs[1:] = np.cumsum([len(p) for p in prompts], dtype=np.uint64)
    data = np.frombuffer(b"".join(prompts) + b"\0" * 64, dtype=np.uint8).copy()
    return data, offs


def encode_batch_special(vocabs, specials, prompts, modes=None, vocab_ids=None, out_cap=None, max_prompts=1 << 20, counts_only=False):
    """(rc, per-prompt id lists, counts, bad (prompt, index), n_stretches)"""
    data, offs = pack(prompts)
    total = int(offs[-1])
    cap = total + 1 if out_cap is None else out_cap
    ids = np.zeros(max(cap, 1), dtype=np.uint32)
    out_off = np.zeros(len(prompts) + 1, dtype=np.uint64)
    counts = np.zeros(max(len(prompts), 1), dtype=np.uint32)
    vh = (C.c_void_p * len(vocabs))(*[v._h for v in vocabs])
    sh = (C.c_void_p * len(vocabs))(*[None if s is None else s._h for s in specials])
    keep = [None if m is None else np.ascontiguousarray(m, dtype=np.uint8) for m in (modes or [])]
    marr = (C.c_void_p * 8)(*([None if m is None else m.ctypes.data for m in keep] + [None] * (8 - len(keep)))) if modes is not None else None
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    bad = np.zeros(2, dtype=np.uint32)
    nst = C.c_uint64(0)
    rc = lib().sim_encode_batch_special(vh, sh, len(vocabs), marr, len(prompts), data.ctypes.data, offs.ctypes.data,
                                        None if vid is None else vid.ctypes.data, None if counts_only else ids.ctypes.data, cap,
                                        out_off.ctypes.data, counts.ctypes.data, max_prompts, bad.ctypes.data, C.byref(nst))
    out = None
    if rc == 0 and not counts_only:
        out = [ids[int(out_off[i]):int(out_off[i + 1])].tolist() for i in range(len(prompts))]
    return rc, out, counts[:len(prompts)].tolist(), (int(bad[0]), int(bad[1])), nst.value, out_off


def decode_batch(vocabs, specials, seqs, vocab_ids=None):
    ids = np.asarray([i for s in seqs for i in s] + [0], dtype=np.uint32)
    io = np.zeros(len(seqs) + 1, dtype=np.uint64)
    io[1:] = np.cumsum([len(s) for s in seqs])
    cap = (len(ids) + 1) * 300
    out = np.zeros(cap, dtype=np.uint8)
    out_off = np.zeros(len(seqs) + 1, dtype=np.uint64)
    vh = (C.c_void_p * len(vocabs))(*[v._h for v in vocabs])
    sh = (C.c_void_p * len(vocabs))(*[None if s is None else s._h for s in specials])
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    rc = lib().sim_decode_batch_special(vh, sh, len(vocabs), len(seqs), ids.ctypes.data, io.ctypes.data,
                                        None if vid is None else vid.ctypes.data, out.ctypes.data, cap, out_off.ctypes.data)
    if rc:
        return rc, None
    return rc, [bytes(out[int(out_off[i]):int(out_off[i + 1])]) for i in range(len(seqs))]
