"""ctypes binding of the SIMT-emulator harness (test infrastructure; tests/simt/sim_harness.cpp)."""
import contextlib
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import build as _build  # noqa: E402

EINVAL, ENOENT, ENOSPC, EILSEQ, EBADMSG = -22, -2, -28, -84, -74
ORDINARY, ALLOW, DISALLOW = 0, 1, 2             # special-token modes
GUARDS = {"none": 0, "after": 1, "before": 2}   # sim_batch_layout's guard pages
SANITIZE_ENV = "CFBPE_SIM_SANITIZE"             # "1": this process loads the alignment-sanitizer build (build.py)
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(_build.build(sanitize=os.environ.get(SANITIZE_ENV) == "1"))
        L.sim_batch_layout.restype = C.c_int
        L.sim_batch_layout.argtypes = [C.c_uint32, C.c_char_p, C.c_uint32, C.c_uint32]
        L.sim_vocab_build.restype = C.c_void_p
        L.sim_vocab_build.argtypes = [C.c_char_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p, C.c_size_t]
        L.sim_vocab_free.argtypes = [C.c_void_p]
        L.sim_vocab_info.argtypes = [C.c_void_p, C.c_void_p]
        L.sim_piece_lookup.restype = C.c_uint32
        L.sim_piece_lookup.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32]
        L.sim_pair_lookup.restype = C.c_uint32
        L.sim_pair_lookup.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        L.sim_run_end.restype = C.c_uint64
        L.sim_run_end.argtypes = [C.c_uint32, C.c_char_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32]
        L.sim_split.restype = C.c_int
        L.sim_split.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.sim_encode_batch.restype = C.c_int
        L.sim_encode_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        L.sim_decode_batch.restype = C.c_int
        L.sim_decode_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_uint64, C.c_void_p]
        L.sim_specials_build.restype = C.c_void_p
        L.sim_specials_build.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_char_p, C.c_size_t]
        L.sim_specials_free.argtypes = [C.c_void_p]
        L.sim_encode_batch_special.restype = C.c_int
        L.sim_encode_batch_special.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint64)]
        L.sim_truncate_batch.restype = C.c_int
        L.sim_truncate_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                         C.c_void_p, C.c_void_p, C.c_void_p]
        L.sim_chunk_batch.restype = C.c_int
        L.sim_chunk_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                      C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_int]
        L.sim_plan_sub_batches.restype = C.c_int
        L.sim_plan_sub_batches.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_void_p]
        L.sim_split_fixups.restype = C.c_ulonglong
        L.sim_split_fixups.argtypes = [C.c_int]
        L.sim_vocab_blob.restype = C.c_uint64
        L.sim_vocab_blob.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        L.sim_validate_blob.restype = C.c_int
        L.sim_validate_blob.argtypes = [C.c_void_p, C.c_uint64, C.c_char_p, C.c_size_t]
        L.sim_dbg_counter.restype = C.c_ulonglong
        L.sim_dbg_counter.argtypes = [C.c_uint32, C.c_int]
        L.sim_workspace_layout.restype = None
        L.sim_workspace_layout.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p]
        _lib = L
    return _lib


def set_batch_layout(misalign=0, fill=b"\0", guard="none"):
    """where every later call puts its batch (sim_harness.cpp, SimBytes): the first prompt byte at an address = misalign (mod 16),
    `fill` repeated over the bytes before it and the padding after the last prompt byte; guard "after": exactly 32 bytes of
    padding, then an unmapped page (misalign not used); "before": an unmapped page just before the misalign leading bytes"""
    assert lib().sim_batch_layout(misalign, bytes(fill), len(fill), GUARDS[guard]) == 0, (misalign, fill, guard)


@contextlib.contextmanager
def batch_layout(misalign=0, fill=b"\0", guard="none"):
    """set_batch_layout for the calls in the block, then the default again (aligned, 64 zero bytes, no guard)"""
    set_batch_layout(misalign, fill, guard)
    try:
        yield
    finally:
        set_batch_layout()


def validate_blob(blob: np.ndarray):
    """(rc, message) of the check cfbpe_vocab_import runs on a packed table blob"""
    err = C.create_string_buffer(256)
    b = np.ascontiguousarray(blob, dtype=np.uint8)
    rc = lib().sim_validate_blob(b.ctypes.data, b.size, err, 256)
    return rc, err.value.decode()


def split_fixups(reset=False):
    """K1 threads that stopped in S_W_U and were finished by pretok_fixup_kernel, in sim_split calls so far"""
    return int(lib().sim_split_fixups(1 if reset else 0))


def dbg_counter(i, reset=False):
    """path counters of csrc/bpe_kernels.cuh (emulator build only): which path did the kernels take"""
    return int(lib().sim_dbg_counter(i, 1 if reset else 0))


class SimVocab:
    def __init__(self, file_bytes, fmt, pattern, max_ranks=0):
        err = C.create_string_buffer(256)
        self._h = lib().sim_vocab_build(file_bytes, len(file_bytes), fmt, pattern, max_ranks, err, 256)
        if not self._h:
            raise ValueError(err.value.decode())
        info = (C.c_uint32 * 6)()
        lib().sim_vocab_info(self._h, info)
        self.n_ranks, self.pattern_id, self.max_token_len, self.n_pair_entries = info[0], info[1], info[2], info[3]
        self.table_bytes = info[4] | (info[5] << 32)

    def __del__(self):
        if getattr(self, "_h", None):
            lib().sim_vocab_free(self._h)
            self._h = None

    def blob(self) -> np.ndarray:
        """the packed tables (what cfbpe_vocab_export hands out)"""
        n = int(lib().sim_vocab_blob(self._h, None, 0))
        out = np.empty(n, dtype=np.uint8)
        lib().sim_vocab_blob(self._h, out.ctypes.data, n)
        return out

    def piece_lookup(self, b: bytes):
        return lib().sim_piece_lookup(self._h, b, len(b))

    def pair_lookup(self, l, r):
        return lib().sim_pair_lookup(self._h, l, r)


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


def _handles(objs):
    """the C array of the SimVocab / Specials handles (None: a NULL entry)"""
    return (C.c_void_p * len(objs))(*[None if o is None else o._h for o in objs])


def pack(prompts):
    """list[bytes] -> (uint8 array, uint64 offsets)"""
    offs = np.zeros(len(prompts) + 1, dtype=np.uint64)
    if prompts:
        offs[1:] = np.cumsum([len(p) for p in prompts], dtype=np.uint64)
    data = np.frombuffer(b"".join(prompts), dtype=np.uint8).copy() if prompts else np.zeros(0, np.uint8)
    return data, offs


def run_end(data: bytes, pos, pe, byte=None):
    """K1's bulk run scanners on data placed by the current layout: the end of the run of `byte` (same_byte_run_end) or, with
    byte None, of ASCII digits (ascii_digit_run_end) that starts at pos, bounded by pe"""
    return int(lib().sim_run_end(1 if byte is None else 0, bytes(data), len(data), pos, pe, 0 if byte is None else byte))


def split(patterns, prompts, vocab_ids=None):
    """piece END offsets per prompt (relative to the prompt) from the K1 bitmask"""
    data, offs = pack(prompts)
    total = int(offs[-1])
    nw = (total + 31) // 32
    bits = np.zeros(nw + 2, dtype=np.uint32)
    pats = np.asarray(patterns, dtype=np.uint32)
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    rc = lib().sim_split(pats.ctypes.data, len(pats), len(prompts), data.ctypes.data, offs.ctypes.data,
                         None if vid is None else vid.ctypes.data, bits.ctypes.data)
    flags = np.unpackbits(bits.view(np.uint8), bitorder="little")[:total]
    out = []
    for i in range(len(prompts)):
        a, b = int(offs[i]), int(offs[i + 1])
        starts = np.nonzero(flags[a:b])[0]
        ends = list(starts[1:]) + ([b - a] if b > a else [])
        out.append([int(e) for e in ends])
    return rc, out


def encode_batch(vocabs, prompts, vocab_ids=None, out_cap=None, starts=None):
    """(rc, ids, offsets, counts, long pieces); starts: an array of out_cap entries that receives the token starts, or None"""
    data, offs = pack(prompts)
    total = int(offs[-1])
    cap = total + 1 if out_cap is None else out_cap
    ids = np.zeros(max(cap, 1), dtype=np.uint32)
    out_off = np.zeros(len(prompts) + 1, dtype=np.uint64)
    counts = np.zeros(max(len(prompts), 1), dtype=np.uint32)
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    nlong = C.c_uint64(0)
    rc = lib().sim_encode_batch(_handles(vocabs), len(vocabs), len(prompts), data.ctypes.data, offs.ctypes.data,
                                None if vid is None else vid.ctypes.data, ids.ctypes.data,
                                None if starts is None else starts.ctypes.data, cap, out_off.ctypes.data, counts.ctypes.data,
                                C.byref(nlong))
    return rc, ids, out_off, counts[:len(prompts)], nlong.value


def encode_starts(vocabs, prompts, vocab_ids=None, out_cap=None):
    """encode with token starts: (rc, ids, starts, offsets, counts)"""
    cap = sum(len(p) for p in prompts) + 1 if out_cap is None else out_cap
    starts = np.full(max(cap, 1), 0xFFFFFFFF, dtype=np.uint32)
    rc, ids, out_off, counts, _ = encode_batch(vocabs, prompts, vocab_ids, cap, starts)
    n_tok = int(out_off[-1])
    return rc, ids[:n_tok], starts[:n_tok], out_off, counts


def encode_batch_special(vocabs, specials, prompts, modes=None, vocab_ids=None, out_cap=None, max_prompts=1 << 20, counts_only=False):
    """(rc, per-prompt id lists, counts, bad (prompt, index), n_stretches, offsets)"""
    data, offs = pack(prompts)
    total = int(offs[-1])
    cap = total + 1 if out_cap is None else out_cap
    ids = np.zeros(max(cap, 1), dtype=np.uint32)
    out_off = np.zeros(len(prompts) + 1, dtype=np.uint64)
    counts = np.zeros(max(len(prompts), 1), dtype=np.uint32)
    keep = [None if m is None else np.ascontiguousarray(m, dtype=np.uint8) for m in (modes or [])]
    marr = (C.c_void_p * 8)(*([None if m is None else m.ctypes.data for m in keep] + [None] * (8 - len(keep)))) if modes is not None else None
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    bad = np.zeros(2, dtype=np.uint32)
    nst = C.c_uint64(0)
    rc = lib().sim_encode_batch_special(_handles(vocabs), _handles(specials), len(vocabs), marr, len(prompts), data.ctypes.data,
                                        offs.ctypes.data, None if vid is None else vid.ctypes.data,
                                        None if counts_only else ids.ctypes.data, cap, out_off.ctypes.data, counts.ctypes.data,
                                        max_prompts, bad.ctypes.data, C.byref(nst))
    out = None
    if rc == 0 and not counts_only:
        out = [ids[int(out_off[i]):int(out_off[i + 1])].tolist() for i in range(len(prompts))]
    return rc, out, counts[:len(prompts)].tolist(), (int(bad[0]), int(bad[1])), nst.value, out_off


def truncate(vocabs, prompts, budgets, mode, vocab_ids=None, null=None):
    """(rc, cut, kept, counts); null: the name of an argument to pass as NULL"""
    data, offs = pack(prompts)
    n = len(prompts)
    bud = np.ascontiguousarray(np.broadcast_to(np.asarray(budgets, dtype=np.uint64), (n,)).astype(np.uint32)) if n else np.zeros(1, np.uint32)
    cut = np.full(max(n, 1), 0xFFFFFFFF, dtype=np.uint32)
    kept = np.full(max(n, 1), 0xFFFFFFFF, dtype=np.uint32)
    counts = np.zeros(max(n, 1), dtype=np.uint32)
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    rc = lib().sim_truncate_batch(_handles(vocabs), len(vocabs), n, data.ctypes.data, offs.ctypes.data,
                                  None if vid is None else vid.ctypes.data, None if null == "budgets" else bud.ctypes.data, mode,
                                  None if null == "cut" else cut.ctypes.data, None if null == "kept" else kept.ctypes.data,
                                  counts.ctypes.data)
    return rc, cut[:n], kept[:n], counts[:n]


def chunk(vocabs, prompts, n_tok, overlap, vocab_ids=None, cap=None, device_form=False, null=None):
    """(rc, spans [cap, 2], chunk offsets [n + 1], counts); cap: the byte bound by default; null: an argument to pass as NULL"""
    data, offs = pack(prompts)
    n = len(prompts)
    if cap is None:
        ln = np.array([len(p) for p in prompts], dtype=np.int64)
        step = max(n_tok - overlap, 1)
        cap = int((ln > 0).sum() + ((np.maximum(ln - n_tok, 0) + step - 1) // step).sum())
    spans = np.full((max(cap, 1), 2), 0xFFFFFFFF, dtype=np.uint32)
    coffs = np.full(n + 1, 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
    counts = np.zeros(max(n, 1), dtype=np.uint32)
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    rc = lib().sim_chunk_batch(_handles(vocabs), len(vocabs), n, data.ctypes.data, offs.ctypes.data, None if vid is None else vid.ctypes.data,
                               n_tok, overlap, None if null == "spans" else spans.ctypes.data, cap,
                               None if null == "offsets" else coffs.ctypes.data, counts.ctypes.data, int(device_form))
    return rc, spans, coffs, counts[:n]


def decode_batch(vocabs, ids, id_offsets, vocab_ids=None, out_cap=None, specials=None):
    """the decode kernels on the emulator: (rc, bytes uint8, byte offsets uint64 n+1); specials: the vocabularies' Specials
    tables (None entries allowed), or None"""
    ids = np.ascontiguousarray(ids, dtype=np.uint32)
    id_offsets = np.ascontiguousarray(id_offsets, dtype=np.uint64)
    n = len(id_offsets) - 1
    cap = int(out_cap) if out_cap is not None else int(len(ids)) * 260 + 64
    out = np.zeros(max(cap, 1), dtype=np.uint8)
    out_off = np.zeros(n + 1, dtype=np.uint64)
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    rc = lib().sim_decode_batch(_handles(vocabs), None if specials is None else _handles(specials), len(vocabs), n, ids.ctypes.data,
                                id_offsets.ctypes.data, None if vid is None else vid.ctypes.data, out.ctypes.data, cap,
                                out_off.ctypes.data)
    return rc, out[:int(out_off[n])] if rc == 0 else out[:0], out_off


WS_KINDS = ["flag_words", "per_byte", "long_list", "scan_tiles", "miss0", "miss1", "miss2", "fix_list", "piece_tiles", "block_prompt"]
WS_BUFFERS = ["piece_bits", "tok_bits", "pstart_bits", "ids_by_pos", "lscratch.rank", "lscratch.aux0", "lscratch.aux1", "dense.by_piece",
              "dense.extras", "long_list", "tile_counts", "tile_base", "miss.list[0]", "miss.list[1]", "miss.list[2]", "fix_list",
              "dense.tile_pieces", "dense.piece_base", "block_prompt"]


class _Layout(C.Structure):
    _fields_ = [("n_buffers", C.c_uint64), ("kind", C.c_uint64 * 32), ("elem", C.c_uint64 * 32), ("start", C.c_uint64 * 32),
                ("alloc", C.c_uint64 * 32), ("extent", C.c_uint64 * len(WS_KINDS)), ("long_cap", C.c_uint64), ("fix_cap", C.c_uint64),
                ("extras_cap", C.c_uint64), ("miss_cap", C.c_uint64 * 3), ("bytes_at", C.c_uint64), ("bytes_alloc", C.c_uint64),
                ("offsets_at", C.c_uint64), ("offsets_alloc", C.c_uint64)]


def workspace_layout(o0, length, k, p0, max_bytes, max_prompts, max_chunks=64):
    """csrc/pipeline.cuh: where a pipelined call puts sub-batch k (length bytes from byte o0, prompts from p0) in a lane.
    buffers: {name: (kind, element bytes, first element, lane allocation)}; extent: {kind: workspace_extent(length)}"""
    r = _Layout()
    lib().sim_workspace_layout(o0, length, k, p0, max_bytes, max_prompts, max_chunks, C.byref(r))
    assert r.n_buffers == len(WS_BUFFERS)
    return {"buffers": {name: (WS_KINDS[r.kind[i]], r.elem[i], r.start[i], r.alloc[i]) for i, name in enumerate(WS_BUFFERS)},
            "extent": dict(zip(WS_KINDS, list(r.extent))),
            "caps": {"long_list": r.long_cap, "fix_list": r.fix_cap, "per_byte": r.extras_cap,
                     "miss0": r.miss_cap[0], "miss1": r.miss_cap[1], "miss2": r.miss_cap[2]},
            "bytes_at": r.bytes_at, "bytes_alloc": r.bytes_alloc, "offsets_at": r.offsets_at, "offsets_alloc": r.offsets_alloc}


def plan_sub_batches(offsets, chunk, max_chunks=64):
    """csrc/subbatch.h:plan_sub_batches -> list of prompt indices cut[0..nc]"""
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    cut = np.zeros(max_chunks + 1, dtype=np.uint32)
    nc = lib().sim_plan_sub_batches(offsets.ctypes.data, len(offsets) - 1, int(chunk), max_chunks, cut.ctypes.data)
    return cut[:nc + 1].tolist()
