"""ctypes binding of libcfbpe.so (include/cfbpe.h).  No fallback: if the CUDA library is not
built or no sm_90 device is present, loading / creating a context raises."""
import ctypes as C
import os

import numpy as np

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # effective if CUDA is not initialised yet; see csrc/cfbpe.cu:cfbpe_create
_DIR = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("CFBPE_SO_VARIANT") or os.path.join(_DIR, "libcfbpe.so")   # CFBPE_SO_VARIANT: A/B builds (tools only)

OK, ENOENT, EIO, ENOMEM, ENODEV, EINVAL, ENOSPC, EILSEQ, EBADMSG = 0, -2, -5, -12, -19, -22, -28, -84, -74
SPECIAL_ORDINARY, SPECIAL_ALLOW, SPECIAL_DISALLOW = 0, 1, 2      # what an occurrence of a special token means in one call
MAX_SPECIALS, MAX_SPECIAL_LEN = 4096, 64
TRUNCATE_HEAD, TRUNCATE_TAIL = 0, 1      # keep the first / the last tokens of every prompt (cfbpe_truncate_batch)
UNIT_CODEPOINT, UNIT_UTF16 = 0, 1        # what a unit start counts (cfbpe_encode_batch_char_starts)
FORMAT_TIKTOKEN, FORMAT_TEKKEN_JSON = 0, 1
PATTERN_CL100K, PATTERN_O200K, PATTERN_LLAMA3, PATTERN_TEKKEN = 0, 1, 2, 3
PATTERN_IDS = {"cl100k": 0, "o200k": 1, "llama3": 2, "tekken": 3}
MAX_VOCABS = 8
NUM_KERNELS = 10
KERNEL_NAMES = ["pretok_split", "bpe_encode", "bpe_long", "flag_count", "tile_scan", "emit_compact", "bpe_list", "long_scan", "bpe_merge", "reserved"]

# every symbol include/cfbpe.h declares (checked by tests/test_abi.py without a GPU)
EXPORTS = [
    "cfbpe_abi_version", "cfbpe_build_id", "cfbpe_create", "cfbpe_destroy", "cfbpe_last_error", "cfbpe_vocab_load",
    "cfbpe_vocab_get_info", "cfbpe_vocab_export", "cfbpe_vocab_import", "cfbpe_encode_batch", "cfbpe_count_batch",
    "cfbpe_encode_batch_device", "cfbpe_device_status", "cfbpe_host_alloc", "cfbpe_host_free",
    "cfbpe_profile_enable", "cfbpe_profile_read", "cfbpe_decode_batch",
    "cfbpe_vocab_set_specials", "cfbpe_encode_batch_special", "cfbpe_encode_batch_special_device",
    "cfbpe_encode_batch_starts", "cfbpe_encode_batch_starts_device",
    "cfbpe_encode_batch_char_starts", "cfbpe_encode_batch_char_starts_device",
    "cfbpe_truncate_batch", "cfbpe_truncate_batch_device",
    "cfbpe_chunk_batch", "cfbpe_chunk_batch_device",
    "cfbpe_encode_batch_lossy", "cfbpe_encode_batch_lossy_device",
    "cfbpe_vocab_set_id_base", "cfbpe_vocab_get_id_base",
]


MAX_DEVICES = 8


class Config(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("device", C.c_int32), ("max_batch_bytes", C.c_uint64),
                ("max_prompts", C.c_uint32), ("flags", C.c_uint32),
                ("devices", C.c_int32 * MAX_DEVICES), ("n_devices", C.c_uint32), ("n_workspaces", C.c_uint32)]


class VocabInfo(C.Structure):
    _fields_ = [("n_ranks", C.c_uint32), ("pattern_id", C.c_uint32), ("max_token_len", C.c_uint32),
                ("n_pair_entries", C.c_uint32), ("table_bytes", C.c_uint64)]


class Profile(C.Structure):
    _fields_ = [("kernel_ms", C.c_float * NUM_KERNELS), ("kernel_launches", C.c_uint32 * NUM_KERNELS),
                ("h2d_ms", C.c_float), ("d2h_ms", C.c_float), ("total_ms", C.c_float),
                ("n_tokens", C.c_uint64), ("n_bytes", C.c_uint64), ("n_long_pieces", C.c_uint64),
                ("n_long_bytes", C.c_uint64), ("n_long_tokens", C.c_uint64),
                ("n_miss_pieces", C.c_uint64), ("n_list_pieces", C.c_uint64), ("n_list_parts", C.c_uint64), ("n_extra_tokens", C.c_uint64)]


_lib = None


def load():
    """dlopen libcfbpe.so; raises if the extension has not been built (python __graft_entry__.py build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise RuntimeError("libcfbpe.so is not built (%s); run `python -c 'import __graft_entry__ as g; g.build()'`. "
                           "There is no CPU fallback." % SO_PATH)
    L = C.CDLL(SO_PATH)
    vp, u8p = C.c_void_p, C.c_void_p
    L.cfbpe_abi_version.restype = C.c_int
    L.cfbpe_build_id.restype = C.c_char_p
    # refuse a binary that was not built from the sources next to it (a failed rebuild must not go unnoticed)
    bpy = os.path.join(os.path.dirname(_DIR), "build.py")
    if os.path.exists(bpy) and os.path.isdir(os.path.join(os.path.dirname(_DIR), "csrc")):
        import importlib.util
        spec = importlib.util.spec_from_file_location("cfbpe_build", bpy)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        want, got = mod.source_hash(), L.cfbpe_build_id().decode()
        if want != got and not os.environ.get("CFBPE_SO_VARIANT"):
            raise RuntimeError("libcfbpe.so is stale (built from %s, sources are %s): rebuild with "
                               "`python -c 'import __graft_entry__ as g; g.build()'`" % (got, want))
    L.cfbpe_create.restype = C.c_int
    L.cfbpe_create.argtypes = [C.POINTER(Config), C.POINTER(vp)]
    L.cfbpe_destroy.argtypes = [vp]
    L.cfbpe_destroy.restype = None
    L.cfbpe_last_error.restype = C.c_char_p
    L.cfbpe_last_error.argtypes = [vp]
    L.cfbpe_vocab_load.restype = C.c_int
    L.cfbpe_vocab_load.argtypes = [vp, C.c_uint32, C.c_char_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32]
    L.cfbpe_vocab_get_info.restype = C.c_int
    L.cfbpe_vocab_get_info.argtypes = [vp, C.c_uint32, C.POINTER(VocabInfo)]
    L.cfbpe_vocab_export.restype = C.c_int
    L.cfbpe_vocab_export.argtypes = [vp, C.c_uint32, u8p, C.c_uint64, C.POINTER(C.c_uint64)]
    L.cfbpe_vocab_import.restype = C.c_int
    L.cfbpe_vocab_import.argtypes = [vp, C.c_uint32, u8p, C.c_uint64]
    L.cfbpe_encode_batch.restype = C.c_int
    L.cfbpe_encode_batch.argtypes = [vp, C.c_uint32, u8p, vp, u8p, vp, C.c_uint64, vp, vp]
    L.cfbpe_count_batch.restype = C.c_int
    L.cfbpe_count_batch.argtypes = [vp, C.c_uint32, u8p, vp, u8p, vp]
    L.cfbpe_decode_batch.restype = C.c_int
    L.cfbpe_decode_batch.argtypes = [vp, C.c_uint32, vp, vp, u8p, vp, C.c_uint64, vp]
    L.cfbpe_encode_batch_device.restype = C.c_int
    L.cfbpe_encode_batch_device.argtypes = [vp, C.c_uint32, vp, C.c_uint64, vp, vp, vp, C.c_uint64, vp, vp,
                                            C.POINTER(C.c_uint64), vp]
    L.cfbpe_encode_batch_starts.restype = C.c_int
    L.cfbpe_encode_batch_starts.argtypes = [vp, C.c_uint32, u8p, vp, u8p, vp, vp, C.c_uint64, vp, vp]
    L.cfbpe_encode_batch_starts_device.restype = C.c_int
    L.cfbpe_encode_batch_starts_device.argtypes = [vp, C.c_uint32, vp, C.c_uint64, vp, vp, vp, vp, C.c_uint64, vp, vp,
                                                   C.POINTER(C.c_uint64), vp]
    L.cfbpe_encode_batch_char_starts.restype = C.c_int
    L.cfbpe_encode_batch_char_starts.argtypes = [vp, C.c_uint32, u8p, vp, u8p, C.c_uint32, vp, vp, C.c_uint64, vp, vp, vp]
    L.cfbpe_encode_batch_char_starts_device.restype = C.c_int
    L.cfbpe_encode_batch_char_starts_device.argtypes = [vp, C.c_uint32, vp, C.c_uint64, vp, vp, C.c_uint32, vp, vp, C.c_uint64, vp, vp,
                                                        vp, C.POINTER(C.c_uint64), vp]
    L.cfbpe_truncate_batch.restype = C.c_int
    L.cfbpe_truncate_batch.argtypes = [vp, C.c_uint32, u8p, vp, u8p, vp, C.c_uint32, vp, vp, vp]
    L.cfbpe_truncate_batch_device.restype = C.c_int
    L.cfbpe_truncate_batch_device.argtypes = [vp, C.c_uint32, vp, C.c_uint64, vp, vp, vp, C.c_uint32, vp, vp, vp, vp]
    L.cfbpe_chunk_batch.restype = C.c_int
    L.cfbpe_chunk_batch.argtypes = [vp, C.c_uint32, u8p, vp, u8p, C.c_uint32, C.c_uint32, vp, C.c_uint64, vp, vp]
    L.cfbpe_chunk_batch_device.restype = C.c_int
    L.cfbpe_chunk_batch_device.argtypes = [vp, C.c_uint32, vp, C.c_uint64, vp, vp, C.c_uint32, C.c_uint32, vp, C.c_uint64, vp, vp,
                                           C.POINTER(C.c_uint64), vp]
    L.cfbpe_vocab_set_specials.restype = C.c_int
    L.cfbpe_vocab_set_specials.argtypes = [vp, C.c_uint32, C.c_uint32, u8p, vp, vp]
    L.cfbpe_vocab_set_id_base.restype = C.c_int
    L.cfbpe_vocab_set_id_base.argtypes = [vp, C.c_uint32, C.c_uint32]
    L.cfbpe_vocab_get_id_base.restype = C.c_int
    L.cfbpe_vocab_get_id_base.argtypes = [vp, C.c_uint32, C.POINTER(C.c_uint32)]
    L.cfbpe_encode_batch_special.restype = C.c_int
    L.cfbpe_encode_batch_special.argtypes = [vp, C.c_uint32, u8p, vp, u8p, vp, vp, C.c_uint64, vp, vp, vp]
    L.cfbpe_encode_batch_special_device.restype = C.c_int
    L.cfbpe_encode_batch_special_device.argtypes = [vp, C.c_uint32, vp, C.c_uint64, vp, vp, vp, vp, C.c_uint64, vp, vp,
                                                    C.POINTER(C.c_uint64), vp, vp]
    L.cfbpe_encode_batch_lossy.restype = C.c_int
    L.cfbpe_encode_batch_lossy.argtypes = [vp, C.c_uint32, u8p, vp, u8p, vp, C.c_uint64, vp, vp, vp]
    L.cfbpe_encode_batch_lossy_device.restype = C.c_int
    L.cfbpe_encode_batch_lossy_device.argtypes = [vp, C.c_uint32, vp, C.c_uint64, vp, vp, vp, C.c_uint64, vp, vp, vp,
                                                  C.POINTER(C.c_uint64), vp]
    L.cfbpe_device_status.restype = C.c_int
    L.cfbpe_device_status.argtypes = [vp, vp]
    L.cfbpe_host_alloc.restype = vp
    L.cfbpe_host_alloc.argtypes = [vp, C.c_size_t]
    L.cfbpe_host_free.restype = None
    L.cfbpe_host_free.argtypes = [vp, vp]
    L.cfbpe_profile_enable.restype = C.c_int
    L.cfbpe_profile_enable.argtypes = [vp, C.c_int]
    L.cfbpe_profile_read.restype = C.c_int
    L.cfbpe_profile_read.argtypes = [vp, C.POINTER(Profile)]
    _lib = L
    return L


class NativeError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("cfbpe error %d: %s" % (code, msg))
        self.code = code


class PinnedArray:
    """numpy view over page-locked host memory owned by the library (cfbpe_host_alloc)."""

    def __init__(self, ctx, shape, dtype):
        self._ctx = ctx
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) if not isinstance(shape, int) else shape
        self.nbytes = max(n * dtype.itemsize, 1)
        self.ptr = load().cfbpe_host_alloc(ctx._h, self.nbytes)
        if not self.ptr:
            raise NativeError(ENOMEM, "cfbpe_host_alloc failed")
        buf = (C.c_uint8 * self.nbytes).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=dtype, count=n).reshape(shape)

    def free(self):
        if self.ptr and self._ctx._h:
            self.array = None
            load().cfbpe_host_free(self._ctx._h, self.ptr)
        self.ptr = None


class Context:
    """One context: one device (`device`) or several (`devices`: a host batch is sharded over them, NCCL inside the library),
    `n_workspaces` independent workspaces per device (that many calls run concurrently).  max_batch_bytes is per device."""

    def __init__(self, device=0, max_batch_bytes=0, max_prompts=0, devices=None, n_workspaces=1):
        self._h = None
        L = load()
        cfg = Config(C.sizeof(Config), device, max_batch_bytes, max_prompts, 0)
        if devices:
            if len(devices) > MAX_DEVICES:
                raise NativeError(EINVAL, "at most %d devices" % MAX_DEVICES)
            for i, d in enumerate(devices):
                cfg.devices[i] = int(d)
            cfg.n_devices = len(devices)
            device = int(devices[0])
        cfg.n_workspaces = int(n_workspaces)
        self.devices = list(devices) if devices else [device]
        self.n_workspaces = int(n_workspaces)
        h = C.c_void_p()
        rc = L.cfbpe_create(C.byref(cfg), C.byref(h))
        if rc != OK:
            raise NativeError(rc, "cfbpe_create failed (no sm_90 device visible?)" if rc == ENODEV else
                              ("cfbpe_create failed: " + L.cfbpe_last_error(None).decode("utf-8", "replace")))
        self._h = h
        self.device = device

    def close(self):
        if self._h:
            load().cfbpe_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != OK:
            raise NativeError(rc, load().cfbpe_last_error(self._h).decode("utf-8", "replace"))

    # ---- vocab
    def vocab_load(self, vocab_id, file_bytes, fmt, pattern_id, max_ranks=0):
        self._check(load().cfbpe_vocab_load(self._h, vocab_id, file_bytes, len(file_bytes), fmt, pattern_id, max_ranks))

    def vocab_info(self, vocab_id):
        vi = VocabInfo()
        self._check(load().cfbpe_vocab_get_info(self._h, vocab_id, C.byref(vi)))
        return {"n_ranks": vi.n_ranks, "pattern_id": vi.pattern_id, "max_token_len": vi.max_token_len,
                "n_pair_entries": vi.n_pair_entries, "table_bytes": vi.table_bytes}

    def vocab_export(self, vocab_id) -> np.ndarray:
        size = C.c_uint64(0)
        self._check(load().cfbpe_vocab_export(self._h, vocab_id, None, 0, C.byref(size)))
        buf = np.empty(size.value, dtype=np.uint8)
        self._check(load().cfbpe_vocab_export(self._h, vocab_id, buf.ctypes.data, size.value, C.byref(size)))
        return buf

    def vocab_import(self, vocab_id, blob: np.ndarray):
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        self._check(load().cfbpe_vocab_import(self._h, vocab_id, blob.ctypes.data, blob.size))

    # ---- host-buffer API
    @staticmethod
    def _check_inputs(data, offsets, vocab_ids, what="bytes", dtype=np.uint8):
        """The C ABI takes pointers without lengths: what it cannot check is checked here (the Rust binding does the same on
        its slices) -- dtypes, contiguity, offsets[n] inside the buffer, one vocab id per prompt."""
        def bad(msg):
            return NativeError(EINVAL, msg)
        if not isinstance(offsets, np.ndarray) or offsets.dtype != np.uint64 or offsets.ndim != 1 or len(offsets) < 1 or not offsets.flags.c_contiguous:
            raise bad("offsets must be a C-contiguous uint64 array of n+1 entries")
        if not isinstance(data, np.ndarray) or data.dtype != dtype or data.ndim != 1 or not data.flags.c_contiguous:
            raise bad("%s must be a C-contiguous 1-D %s array" % (what, np.dtype(dtype).name))
        n = len(offsets) - 1
        if int(offsets[n]) > data.size:
            raise bad("offsets[n] = %d exceeds len(%s) = %d" % (int(offsets[n]), what, data.size))
        if vocab_ids is not None:
            if not isinstance(vocab_ids, np.ndarray) or vocab_ids.dtype != np.uint8 or vocab_ids.ndim != 1 or len(vocab_ids) < n or not vocab_ids.flags.c_contiguous:
                raise bad("vocab_ids must be a C-contiguous uint8 array with one entry per prompt")
        return n

    def encode_batch(self, data: np.ndarray, offsets: np.ndarray, vocab_ids=None, out_ids=None, out_offsets=None,
                     out_counts=None):
        n = self._check_inputs(data, offsets, vocab_ids)
        total = int(offsets[n])
        if out_ids is None:
            out_ids = np.empty(max(total, 1), dtype=np.uint32)
        if out_offsets is None:
            out_offsets = np.empty(n + 1, dtype=np.uint64)
        if out_counts is None:
            out_counts = np.empty(max(n, 1), dtype=np.uint32)
        vid = None if vocab_ids is None else vocab_ids.ctypes.data
        rc = load().cfbpe_encode_batch(self._h, n, data.ctypes.data if data.size else None, offsets.ctypes.data, vid,
                                       out_ids.ctypes.data, out_ids.size, out_offsets.ctypes.data,
                                       out_counts.ctypes.data)
        self._check(rc)
        return out_ids[:int(out_offsets[n])], out_offsets, out_counts[:n]

    def encode_batch_starts(self, data: np.ndarray, offsets: np.ndarray, vocab_ids=None, out_ids=None, out_starts=None,
                            out_offsets=None, out_counts=None):
        """encode_batch plus each token's byte offset within its prompt: (ids, starts uint32, offsets, counts).  Token k of prompt i
        covers bytes[offsets_in[i] + starts[k] .. offsets_in[i] + end), end = starts[k + 1] or the prompt's length for its last token."""
        n = self._check_inputs(data, offsets, vocab_ids)
        total = int(offsets[n])
        if out_ids is None:
            out_ids = np.empty(max(total, 1), dtype=np.uint32)
        if out_starts is None:
            out_starts = np.empty(out_ids.size, dtype=np.uint32)
        if out_starts.dtype != np.uint32 or out_starts.size < out_ids.size or not out_starts.flags.c_contiguous:
            raise NativeError(EINVAL, "out_starts must be a C-contiguous uint32 array with room for as many entries as out_ids")
        if out_offsets is None:
            out_offsets = np.empty(n + 1, dtype=np.uint64)
        if out_counts is None:
            out_counts = np.empty(max(n, 1), dtype=np.uint32)
        vid = None if vocab_ids is None else vocab_ids.ctypes.data
        rc = load().cfbpe_encode_batch_starts(self._h, n, data.ctypes.data if data.size else None, offsets.ctypes.data, vid,
                                              out_ids.ctypes.data, out_starts.ctypes.data, out_ids.size, out_offsets.ctypes.data,
                                              out_counts.ctypes.data)
        self._check(rc)
        nt = int(out_offsets[n])
        return out_ids[:nt], out_starts[:nt], out_offsets, out_counts[:n]

    def encode_batch_char_starts(self, data: np.ndarray, offsets: np.ndarray, unit=UNIT_CODEPOINT, vocab_ids=None, out_ids=None,
                                 out_starts=None, out_offsets=None, out_counts=None, out_lens=None):
        """encode_batch plus each token's start within its prompt in `unit` (UNIT_CODEPOINT: str indices, UNIT_UTF16: UTF-16 code
        units): (ids, starts uint32, offsets, counts, lens uint32 -- every prompt's length in the unit).  A token's start is that of
        the character holding its first byte, so byte tokens of one character share it: their spans are empty."""
        n = self._check_inputs(data, offsets, vocab_ids)
        total = int(offsets[n])
        if out_ids is None:
            out_ids = np.empty(max(total, 1), dtype=np.uint32)
        if out_starts is None:
            out_starts = np.empty(out_ids.size, dtype=np.uint32)
        if out_starts.dtype != np.uint32 or out_starts.size < out_ids.size or not out_starts.flags.c_contiguous:
            raise NativeError(EINVAL, "out_starts must be a C-contiguous uint32 array with room for as many entries as out_ids")
        if out_offsets is None:
            out_offsets = np.empty(n + 1, dtype=np.uint64)
        if out_counts is None:
            out_counts = np.empty(max(n, 1), dtype=np.uint32)
        if out_lens is None:
            out_lens = np.empty(max(n, 1), dtype=np.uint32)
        elif not isinstance(out_lens, np.ndarray) or out_lens.dtype != np.uint32 or out_lens.size < n or not out_lens.flags.c_contiguous:
            raise NativeError(EINVAL, "out_lens must be a C-contiguous uint32 array with one entry per prompt")
        vid = None if vocab_ids is None else vocab_ids.ctypes.data
        rc = load().cfbpe_encode_batch_char_starts(self._h, n, data.ctypes.data if data.size else None, offsets.ctypes.data, vid, int(unit),
                                                   out_ids.ctypes.data, out_starts.ctypes.data, out_ids.size, out_offsets.ctypes.data,
                                                   out_counts.ctypes.data, out_lens.ctypes.data)
        self._check(rc)
        nt = int(out_offsets[n])
        return out_ids[:nt], out_starts[:nt], out_offsets, out_counts[:n], out_lens[:n]

    @staticmethod
    def budget_array(budgets, n):
        """an int (every prompt) or one budget per prompt -> a C-contiguous uint32 array of max(n, 1) entries"""
        if isinstance(budgets, (int, np.integer)):
            if not 0 <= int(budgets) <= 0xFFFFFFFF:
                raise NativeError(EINVAL, "a token budget must be in 0 .. 2^32 - 1")
            return np.full(max(n, 1), int(budgets), dtype=np.uint32)
        b = np.asarray(budgets)
        if b.ndim != 1 or len(b) != n or (b.size and (b.dtype.kind not in "iu" or int(b.min()) < 0 or int(b.max()) > 0xFFFFFFFF)):
            raise NativeError(EINVAL, "budgets must be one integer in 0 .. 2^32 - 1 per prompt")
        return np.ascontiguousarray(b, dtype=np.uint32) if n else np.zeros(1, dtype=np.uint32)

    def truncate_batch(self, data: np.ndarray, offsets: np.ndarray, budgets, mode=TRUNCATE_HEAD, vocab_ids=None, out_cut=None,
                       out_kept=None, out_counts=None):
        """cfbpe_truncate_batch: (cut, kept, counts), uint32 each, one entry per prompt.  budgets: an int or one per prompt.
        TRUNCATE_HEAD keeps bytes[offsets[i] .. offsets[i] + cut[i]), TRUNCATE_TAIL keeps bytes[offsets[i] + cut[i] .. offsets[i + 1])."""
        n = self._check_inputs(data, offsets, vocab_ids)
        bud = self.budget_array(budgets, n)
        outs = []
        for a in (out_cut, out_kept, out_counts):
            if a is None:
                a = np.empty(max(n, 1), dtype=np.uint32)
            elif not isinstance(a, np.ndarray) or a.dtype != np.uint32 or a.size < n or not a.flags.c_contiguous:
                raise NativeError(EINVAL, "out_cut, out_kept and out_counts must be C-contiguous uint32 arrays with one entry per prompt")
            outs.append(a)
        vid = None if vocab_ids is None else vocab_ids.ctypes.data
        self._check(load().cfbpe_truncate_batch(self._h, n, data.ctypes.data if data.size else None, offsets.ctypes.data, vid,
                                                bud.ctypes.data, mode, outs[0].ctypes.data, outs[1].ctypes.data, outs[2].ctypes.data))
        return outs[0][:n], outs[1][:n], outs[2][:n]

    @staticmethod
    def chunk_bound(offsets: np.ndarray, chunk_tokens: int, overlap_tokens: int = 0) -> int:
        """chunks a batch can have at most (include/cfbpe.h, cfbpe_chunk_batch): the chunk formula with c = each prompt's byte length"""
        ln = np.diff(np.asarray(offsets, dtype=np.int64))
        step = chunk_tokens - overlap_tokens
        if chunk_tokens < 1 or step < 1:
            return 0
        return int((ln > 0).sum() + ((np.maximum(ln - chunk_tokens, 0) + step - 1) // step).sum())

    def chunk_batch(self, data: np.ndarray, offsets: np.ndarray, chunk_tokens: int, overlap_tokens: int = 0, vocab_ids=None,
                    out_counts=None):
        """cfbpe_chunk_batch: (spans, chunk_offsets, counts).  spans: uint32 [chunks, 2], (begin, end) of every chunk within its
        prompt; prompt i's chunks are spans[chunk_offsets[i] .. chunk_offsets[i + 1]] (uint64, n + 1); counts: uint32 tokens a
        prompt.  chunk_cap is the byte bound (chunk_bound), so the call never needs a second try."""
        n = self._check_inputs(data, offsets, vocab_ids)
        if not (isinstance(chunk_tokens, (int, np.integer)) and isinstance(overlap_tokens, (int, np.integer))
                and 0 <= int(chunk_tokens) <= 0xFFFFFFFF and 0 <= int(overlap_tokens) <= 0xFFFFFFFF):
            raise NativeError(EINVAL, "chunk_tokens and overlap_tokens must be integers in 0 .. 2^32 - 1")
        cap = self.chunk_bound(offsets, int(chunk_tokens), int(overlap_tokens))
        spans = np.empty((max(cap, 1), 2), dtype=np.uint32)
        coffs = np.zeros(n + 1, dtype=np.uint64)
        if out_counts is None:
            out_counts = np.empty(max(n, 1), dtype=np.uint32)
        elif not isinstance(out_counts, np.ndarray) or out_counts.dtype != np.uint32 or out_counts.size < n or not out_counts.flags.c_contiguous:
            raise NativeError(EINVAL, "out_counts must be a C-contiguous uint32 array with one entry per prompt")
        vid = None if vocab_ids is None else vocab_ids.ctypes.data
        self._check(load().cfbpe_chunk_batch(self._h, n, data.ctypes.data if data.size else None, offsets.ctypes.data, vid,
                                             int(chunk_tokens), int(overlap_tokens), spans.ctypes.data, cap, coffs.ctypes.data,
                                             out_counts.ctypes.data))
        return spans[:int(coffs[n])], coffs, out_counts[:n]

    def count_batch(self, data: np.ndarray, offsets: np.ndarray, vocab_ids=None, out_counts=None):
        n = self._check_inputs(data, offsets, vocab_ids)
        if out_counts is None:
            out_counts = np.empty(max(n, 1), dtype=np.uint32)
        vid = None if vocab_ids is None else vocab_ids.ctypes.data
        self._check(load().cfbpe_count_batch(self._h, n, data.ctypes.data if data.size else None, offsets.ctypes.data,
                                             vid, out_counts.ctypes.data))
        return out_counts[:n]

    def decode_batch(self, ids: np.ndarray, id_offsets: np.ndarray, vocab_ids=None, out_cap=None, out_bytes=None, out_offsets=None):
        """ids (uint32, packed) + id_offsets (uint64, n+1) -> (bytes uint8, byte offsets uint64 n+1).
        out_bytes / out_offsets: caller's buffers (pinned ones make the download several times faster)"""
        n = self._check_inputs(ids, id_offsets, vocab_ids, "ids", np.uint32)
        if out_offsets is None:
            out_offsets = np.zeros(n + 1, dtype=np.uint64)
        vid = None if vocab_ids is None else vocab_ids.ctypes.data
        if out_bytes is not None:
            self._check(load().cfbpe_decode_batch(self._h, n, ids.ctypes.data if ids.size else None, id_offsets.ctypes.data, vid,
                                                  out_bytes.ctypes.data, out_bytes.size, out_offsets.ctypes.data))
            return out_bytes[:int(out_offsets[n])], out_offsets
        cap = int(out_cap) if out_cap is not None else max(int(len(ids)) * 8 + 64, 64)
        while True:
            out = np.empty(max(cap, 1), dtype=np.uint8)
            rc = load().cfbpe_decode_batch(self._h, n, ids.ctypes.data if ids.size else None, id_offsets.ctypes.data, vid,
                                           out.ctypes.data, cap, out_offsets.ctypes.data)
            if rc == ENOSPC and out_cap is None:
                cap = int(out_offsets[n])
                continue
            self._check(rc)
            return out[:int(out_offsets[n])], out_offsets

    # ---- device-buffer API (raw pointers; torch tensors pass .data_ptr())
    def encode_batch_device(self, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_ids, out_cap,
                            d_out_offsets, d_out_counts, stream=0, sync=True):
        nt = C.c_uint64(0)
        rc = load().cfbpe_encode_batch_device(self._h, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids,
                                              d_out_ids, out_cap, d_out_offsets, d_out_counts,
                                              C.byref(nt) if sync else None, stream)
        self._check(rc)
        return nt.value if sync else None

    def encode_batch_starts_device(self, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_ids, d_out_starts, out_cap,
                                   d_out_offsets, d_out_counts, stream=0, sync=True):
        """cfbpe_encode_batch_starts_device on raw device pointers (d_out_starts: room for out_cap uint32); the id count when sync"""
        nt = C.c_uint64(0)
        rc = load().cfbpe_encode_batch_starts_device(self._h, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_ids,
                                                     d_out_starts, out_cap, d_out_offsets, d_out_counts,
                                                     C.byref(nt) if sync else None, stream)
        self._check(rc)
        return nt.value if sync else None

    def encode_batch_char_starts_device(self, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, unit, d_out_ids, d_out_starts, out_cap,
                                        d_out_offsets, d_out_counts, d_out_lens, stream=0, sync=True):
        """cfbpe_encode_batch_char_starts_device on raw device pointers (d_out_starts: room for out_cap uint32; d_out_lens: n_prompts
        uint32 or None); the id count when sync, else fully asynchronous"""
        nt = C.c_uint64(0)
        rc = load().cfbpe_encode_batch_char_starts_device(self._h, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, int(unit), d_out_ids,
                                                          d_out_starts, out_cap, d_out_offsets, d_out_counts, d_out_lens,
                                                          C.byref(nt) if sync else None, stream)
        self._check(rc)
        return nt.value if sync else None

    def truncate_batch_device(self, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_budgets, mode, d_out_cut, d_out_kept,
                              d_out_counts, stream=0):
        """cfbpe_truncate_batch_device on raw device pointers (uint32 budgets, cuts, kept counts, counts: n_prompts each; counts
        may be None).  Asynchronous: its errors come from device_status, called from the same thread before its next device call."""
        self._check(load().cfbpe_truncate_batch_device(self._h, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_budgets,
                                                       mode, d_out_cut, d_out_kept, d_out_counts, stream))

    def chunk_batch_device(self, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, chunk_tokens, overlap_tokens, d_out_spans,
                           chunk_cap, d_out_chunk_offsets, d_out_counts, stream=0, sync=True):
        """cfbpe_chunk_batch_device on raw device pointers (d_out_spans: room for chunk_cap pairs of uint32; d_out_chunk_offsets:
        n_prompts + 1 uint64; d_out_counts: n_prompts uint32 or None); the chunk count when sync, else fully asynchronous"""
        nc = C.c_uint64(0)
        rc = load().cfbpe_chunk_batch_device(self._h, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, chunk_tokens, overlap_tokens,
                                             d_out_spans, chunk_cap, d_out_chunk_offsets, d_out_counts, C.byref(nc) if sync else None, stream)
        self._check(rc)
        return nc.value if sync else None

    # ---- special tokens
    @staticmethod
    def pack_specials(specials):
        """{str: id} (tiktoken's special_tokens; dict order = special index) -> (bytes uint8, offsets uint64 n+1, ids uint32)"""
        toks = [t.encode("utf-8") for t in specials]
        offs = np.zeros(len(toks) + 1, dtype=np.uint64)
        if toks:
            offs[1:] = np.cumsum([len(t) for t in toks])
        data = np.frombuffer(b"".join(toks), dtype=np.uint8).copy() if toks else np.zeros(1, np.uint8)
        ids = np.asarray([int(v) for v in specials.values()], dtype=np.uint32) if toks else np.zeros(1, np.uint32)
        return data, offs, ids

    def vocab_set_specials(self, vocab_id, specials):
        """register {token string: id} as the special tokens of vocabulary slot `vocab_id` (replaces the earlier set; {} clears it)"""
        data, offs, ids = self.pack_specials(specials)
        self._check(load().cfbpe_vocab_set_specials(self._h, vocab_id, len(specials), data.ctypes.data, offs.ctypes.data, ids.ctypes.data))

    def vocab_set_id_base(self, vocab_id, base):
        """ordinary token of rank r of slot `vocab_id` -> id base + r in every id a call returns or decode takes (0: ids are ranks)"""
        self._check(load().cfbpe_vocab_set_id_base(self._h, vocab_id, int(base)))

    def vocab_id_base(self, vocab_id):
        out = C.c_uint32(0)
        self._check(load().cfbpe_vocab_get_id_base(self._h, vocab_id, C.byref(out)))
        return out.value

    @staticmethod
    def _modes_arg(modes):
        """modes: None (every special of every vocabulary DISALLOWED) or a sequence indexed by vocabulary slot of None / uint8 arrays
        of one SPECIAL_* byte per registered special -> (ctypes array or None, arrays kept alive)"""
        if modes is None:
            return None, []
        if len(modes) > MAX_VOCABS:
            raise NativeError(EINVAL, "modes names more than %d vocabularies" % MAX_VOCABS)
        keep = [None if m is None else np.ascontiguousarray(m, dtype=np.uint8) for m in modes]
        arr = (C.c_void_p * MAX_VOCABS)(*([None if m is None else m.ctypes.data for m in keep] + [None] * (MAX_VOCABS - len(keep))))
        return arr, keep

    def encode_batch_special(self, data: np.ndarray, offsets: np.ndarray, vocab_ids=None, modes=None, out_ids=None, out_offsets=None,
                             out_counts=None, counts_only=False):
        """tiktoken's encode(allowed_special / disallowed_special) for every prompt: (ids, offsets, counts).  modes: see _modes_arg.
        NativeError EBADMSG (with .bad = (prompt, special index)) when a prompt spells a DISALLOWED special."""
        n = self._check_inputs(data, offsets, vocab_ids)
        total = int(offsets[n])
        if out_ids is None and not counts_only:
            out_ids = np.empty(max(total, 1), dtype=np.uint32)
        if out_offsets is None:
            out_offsets = np.empty(n + 1, dtype=np.uint64)
        if out_counts is None:
            out_counts = np.empty(max(n, 1), dtype=np.uint32)
        marr, _keep = self._modes_arg(modes)
        bad = (C.c_uint32 * 2)()
        vid = None if vocab_ids is None else vocab_ids.ctypes.data
        rc = load().cfbpe_encode_batch_special(self._h, n, data.ctypes.data if data.size else None, offsets.ctypes.data, vid, marr,
                                               None if counts_only else out_ids.ctypes.data, 0 if counts_only else out_ids.size,
                                               out_offsets.ctypes.data, out_counts.ctypes.data, bad)
        self._check_special(rc, bad)
        return (None if counts_only else out_ids[:int(out_offsets[n])]), out_offsets, out_counts[:n]

    def encode_batch_special_device(self, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_ids, out_cap,
                                    d_out_offsets, d_out_counts, modes=None, stream=0, sync=True):
        """cfbpe_encode_batch_special_device on raw device pointers; returns the id count when sync"""
        nt = C.c_uint64(0)
        marr, _keep = self._modes_arg(modes)
        bad = (C.c_uint32 * 2)()
        rc = load().cfbpe_encode_batch_special_device(self._h, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, marr,
                                                      d_out_ids, out_cap, d_out_offsets, d_out_counts,
                                                      C.byref(nt) if sync else None, bad, stream)
        self._check_special(rc, bad)
        return nt.value if sync else None

    def _check_special(self, rc, bad):
        if rc != OK:
            e = NativeError(rc, load().cfbpe_last_error(self._h).decode("utf-8", "replace"))
            e.bad = (int(bad[0]), int(bad[1])) if rc == EBADMSG else None
            raise e

    # ---- bytes that are not valid UTF-8
    def encode_batch_lossy(self, data: np.ndarray, offsets: np.ndarray, vocab_ids=None, out_ids=None, out_offsets=None, out_counts=None,
                           out_replaced=None, counts_only=False):
        """encode every prompt as b.decode("utf-8", "replace") would be encoded: (ids, offsets, counts, replaced).  replaced: uint32,
        the U+FFFD the decode inserted into each prompt (0: valid UTF-8).  counts_only: ids is None."""
        n = self._check_inputs(data, offsets, vocab_ids)
        total = int(offsets[n])
        if out_ids is None and not counts_only:
            out_ids = np.empty(max(3 * total, 1), dtype=np.uint32)      # (the repaired text is at most 3 bytes a byte)
        if out_offsets is None:
            out_offsets = np.empty(n + 1, dtype=np.uint64)
        if out_counts is None:
            out_counts = np.empty(max(n, 1), dtype=np.uint32)
        if out_replaced is None:
            out_replaced = np.empty(max(n, 1), dtype=np.uint32)
        elif not isinstance(out_replaced, np.ndarray) or out_replaced.dtype != np.uint32 or out_replaced.size < n or not out_replaced.flags.c_contiguous:
            raise NativeError(EINVAL, "out_replaced must be a C-contiguous uint32 array with one entry per prompt")
        vid = None if vocab_ids is None else vocab_ids.ctypes.data
        rc = load().cfbpe_encode_batch_lossy(self._h, n, data.ctypes.data if data.size else None, offsets.ctypes.data, vid,
                                             None if counts_only else out_ids.ctypes.data, 0 if counts_only else out_ids.size,
                                             out_offsets.ctypes.data, out_counts.ctypes.data, out_replaced.ctypes.data)
        self._check(rc)
        return (None if counts_only else out_ids[:int(out_offsets[n])]), out_offsets, out_counts[:n], out_replaced[:n]

    def encode_batch_lossy_device(self, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_ids, out_cap, d_out_offsets,
                                  d_out_counts, d_out_replaced, stream=0, sync=True):
        """cfbpe_encode_batch_lossy_device on raw device pointers (d_out_replaced: n_prompts uint32 or None); the id count when sync.
        The call synchronises `stream` once after its scan either way."""
        nt = C.c_uint64(0)
        rc = load().cfbpe_encode_batch_lossy_device(self._h, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_ids, out_cap,
                                                    d_out_offsets, d_out_counts, d_out_replaced, C.byref(nt) if sync else None, stream)
        self._check(rc)
        return nt.value if sync else None

    def device_status(self, stream=0):
        """sync `stream` and raise the error of this thread's last device call on this context (sync=False calls report only here);
        host calls, decode and other threads' calls do not change it"""
        self._check(load().cfbpe_device_status(self._h, stream))

    def pinned(self, shape, dtype):
        return PinnedArray(self, shape, dtype)

    def profile_enable(self, on=True):
        self._check(load().cfbpe_profile_enable(self._h, 1 if on else 0))

    def profile_read(self):
        p = Profile()
        self._check(load().cfbpe_profile_read(self._h, C.byref(p)))
        return {"kernel_ms": {KERNEL_NAMES[i]: p.kernel_ms[i] for i in range(NUM_KERNELS)},
                "kernel_launches": {KERNEL_NAMES[i]: p.kernel_launches[i] for i in range(NUM_KERNELS)},
                "h2d_ms": p.h2d_ms, "d2h_ms": p.d2h_ms, "total_ms": p.total_ms, "n_tokens": p.n_tokens,
                "n_bytes": p.n_bytes, "n_long_pieces": p.n_long_pieces, "n_long_bytes": p.n_long_bytes,
                "n_long_tokens": p.n_long_tokens, "n_miss_pieces": p.n_miss_pieces, "n_list_pieces": p.n_list_pieces,
                "n_list_parts": p.n_list_parts, "n_extra_tokens": p.n_extra_tokens}
