"""Chunking (chunk_scan / chunk_emit, csrc/bpe_kernels.cuh) on the CPU SIMT emulator, against a reference built here from live
tiktoken 0.12.0: encode_ordinary, the tokens' byte lengths and the snap of include/cfbpe.h (cfbpe_chunk_batch)."""
import base64
import ctypes as C
import os
import random
import sys

import numpy as np
import pytest

import fuzzgen
import simlib
from conftest import COMBOS, golden_cases

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))
import build_chunk  # noqa: E402

EINVAL, ENOENT, ENOSPC, EILSEQ = -22, -2, -28, -84
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_chunk.build())
        L.sim_vocab_build.restype = C.c_void_p
        L.sim_vocab_build.argtypes = [C.c_char_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p, C.c_size_t]
        L.sim_vocab_free.argtypes = [C.c_void_p]
        L.sim_chunk_batch.restype = C.c_int
        L.sim_chunk_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                      C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_int]
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


def chunk(vocabs, prompts, n_tok, overlap, vocab_ids=None, cap=None, device_form=False, null=None):
    """(rc, spans [cap, 2], chunk offsets [n + 1], counts); cap: the byte bound by default; null: an argument to pass as NULL"""
    data, offs = simlib.pack(prompts)
    n = len(prompts)
    if cap is None:
        ln = np.array([len(p) for p in prompts], dtype=np.int64)
        step = max(n_tok - overlap, 1)
        cap = int((ln > 0).sum() + ((np.maximum(ln - n_tok, 0) + step - 1) // step).sum())
    spans = np.full((max(cap, 1), 2), 0xFFFFFFFF, dtype=np.uint32)
    coffs = np.full(n + 1, 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
    counts = np.zeros(max(n, 1), dtype=np.uint32)
    vh = (C.c_void_p * len(vocabs))(*[v._h for v in vocabs])
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    dbuf = np.concatenate([data, np.zeros(8, np.uint8)])
    rc = lib().sim_chunk_batch(vh, len(vocabs), n, dbuf.ctypes.data, offs.ctypes.data, None if vid is None else vid.ctypes.data,
                               n_tok, overlap, None if null == "spans" else spans.ctypes.data, cap,
                               None if null == "offsets" else coffs.ctypes.data, counts.ctypes.data, int(device_form))
    return rc, spans, coffs, counts[:n]


def is_cont(b):
    return 0x80 <= b < 0xC0


def reference(enc, prompt: bytes, n_tok: int, overlap: int):
    """[(begin, end)] of every chunk and the count, by the contract, from live tiktoken"""
    ids = enc.encode_ordinary(prompt.decode("utf-8"))
    c, ln = len(ids), len(prompt)
    lens = [len(enc.decode_single_token_bytes(t)) for t in ids]
    x = [0] + list(np.cumsum(lens)) if c else [0]

    def F(j):
        if j >= c:
            return ln
        p = int(x[j])
        while 0 < p < ln and is_cont(prompt[p]):
            p -= 1
        return p
    step = n_tok - overlap
    k = 0 if c == 0 else 1 if c <= n_tok else 1 + -(-(c - n_tok) // step)
    return [(F(q * step), F(min(q * step + n_tok, c))) for q in range(k)], c


@pytest.fixture(scope="module")
def encs(tekken_bytes):
    tiktoken = pytest.importorskip("tiktoken")
    from oracle import patterns as PT
    lines = tekken_bytes.splitlines()
    out = {}
    for pat, n in COMBOS:
        ranks = {base64.b64decode(l.split()[0]): i for i, l in enumerate(lines[:n])}
        out[pat] = tiktoken.Encoding("live%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks, special_tokens={})
    return out


@pytest.fixture(scope="module")
def vocabs(tekken_bytes):
    return {pat: Vocab(tekken_bytes, pat, n) for pat, n in COMBOS}


def check(encs, vocabs, prompts, n_tok, overlap, pats, vocab_ids=None, device_form=False):
    """the emulator equals the reference for every prompt; returns the reference rows"""
    rc, spans, coffs, counts = chunk([vocabs[p] for p in pats], prompts, n_tok, overlap, vocab_ids, device_form=device_form)
    assert rc == 0
    rows = []
    for i, p in enumerate(prompts):
        enc = encs[pats[0] if vocab_ids is None else pats[int(vocab_ids[i])]]
        want, c = reference(enc, p, n_tok, overlap)
        got = [tuple(int(v) for v in s) for s in spans[int(coffs[i]):int(coffs[i + 1])]]
        assert (got, int(counts[i])) == (want, c), (i, n_tok, overlap, p[:60])
        rows.append((want, c))
    assert int(coffs[0]) == 0 and int(coffs[-1]) == sum(len(w) for w, _ in rows)
    return rows


@pytest.mark.parametrize("pat,n_ranks", COMBOS)
def test_golden_cases(golden, encs, vocabs, pat, n_ranks):
    cases = golden_cases(golden)
    for n_tok, overlap in ((7, 2), (512, 64), (2, 0)):
        check(encs, vocabs, cases, n_tok, overlap, [pat], device_form=n_tok == 7)


@pytest.mark.parametrize("n_tok", [1, 2, 3, 7, 512])
def test_sizes_and_overlaps(encs, vocabs, n_tok):
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(5 + n_tok, 40, max_atoms=30)] + [b"Hello, world! " * 12, "日本語のテキスト".encode()]
    for overlap in sorted({0, 1, n_tok - 1} & set(range(n_tok))):
        for device_form in (False, True):
            check(encs, vocabs, prompts, n_tok, overlap, [0], device_form=device_form)


def test_counts_at_the_edges(encs, vocabs):
    """c = 0 (no chunk), c = N (one), c = N + 1 (two); empty prompts between others"""
    base = "the quick brown fox jumps over the lazy dog " * 3
    ids = encs[0].encode_ordinary(base)
    n_tok = 9
    exact = encs[0].decode(ids[:n_tok]).encode()
    plus1 = encs[0].decode(ids[:n_tok + 1]).encode()
    assert len(encs[0].encode_ordinary(exact.decode())) == n_tok and len(encs[0].encode_ordinary(plus1.decode())) == n_tok + 1
    prompts = [b"", exact, b"", plus1, b"", b"x"]
    rows = check(encs, vocabs, prompts, n_tok, 0, [0])
    assert [len(w) for w, _ in rows] == [0, 1, 0, 2, 0, 1]
    rows = check(encs, vocabs, prompts, n_tok, 3, [0])
    assert [len(w) for w, _ in rows] == [0, 1, 0, 2, 0, 1]
    rc, spans, coffs, counts = chunk([vocabs[0]], [b"", b"", b""], 4, 1)
    assert rc == 0 and coffs.tolist() == [0, 0, 0, 0] and counts.tolist() == [0, 0, 0]


def multibyte_texts(seed, count):
    """text whose byte-level tokens end inside characters: CJK Extension B ideographs (4 bytes, rare: byte pieces) and emoji"""
    rng = random.Random(seed)
    ext_b = [chr(0x20000 + rng.randrange(0xA6DF)) for _ in range(64)]
    emoji = ["\U0001f600", "\U0001f9d1‍\U0001f4bb", "\U0001f3f3️‍\U0001f308", "\U0001fae0", "❤️"]
    out = []
    for _ in range(count):
        parts = []
        for _ in range(rng.randint(1, 30)):
            r = rng.random()
            parts.append(rng.choice(ext_b) if r < 0.45 else rng.choice(emoji) if r < 0.75 else rng.choice([" ", "a", "文", " the", "\n"]))
        out.append("".join(parts))
    return out


def test_boundaries_inside_characters_are_snapped(encs, vocabs):
    prompts = [t.encode() for t in multibyte_texts(99, 200)]
    for pat in (0, 1):
        moved = 0
        for n_tok, overlap in ((1, 0), (2, 1), (5, 0), (5, 2)):
            rows = check(encs, vocabs, prompts, n_tok, overlap, [pat])
            for (want, c), p in zip(rows, prompts):
                ids = encs[pat].encode_ordinary(p.decode())
                x = np.cumsum([0] + [len(encs[pat].decode_single_token_bytes(t)) for t in ids])
                step = n_tok - overlap
                moved += sum(1 for q, (b, _) in enumerate(want) if b != int(x[q * step]))
                for b, e in want:
                    p[b:e].decode("utf-8")                             # valid UTF-8, always
                    assert b <= e
        assert moved >= 20, (pat, moved)                               # the data holds token starts inside characters


def test_no_overlap_tiles_and_chunk0_is_the_head_cut(encs, vocabs):
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(71, 60, max_atoms=40)] + [t.encode() for t in multibyte_texts(3, 40)]
    for n_tok in (1, 3, 16):
        rows = check(encs, vocabs, prompts, n_tok, 0, [0])
        for (want, c), p in zip(rows, prompts):
            if not c:
                continue
            assert want[0][0] == 0 and want[-1][1] == len(p)
            assert all(want[k][1] == want[k + 1][0] for k in range(len(want) - 1))
            assert b"".join(p[b:e] for b, e in want) == p
            # chunk 0 ends where truncation to the first n_tok tokens (CFBPE_TRUNCATE_HEAD) cuts
            ids = encs[0].encode_ordinary(p.decode())
            cut = len(encs[0].decode_bytes(ids[:n_tok]))
            while 0 < cut < len(p) and is_cont(p[cut]):
                cut -= 1
            assert want[0][1] == cut


def test_mixed_vocabulary_batch(encs, vocabs):
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(31, 120, max_atoms=40)] + [s.encode() for s in fuzzgen.long_runs(2)[:30]]
    vid = np.array([i % 4 for i in range(len(prompts))], dtype=np.uint8)
    pats = [p for p, _ in COMBOS]
    for n_tok, overlap in ((4, 1), (64, 0)):
        check(encs, vocabs, prompts, n_tok, overlap, pats, vocab_ids=vid)


def test_long_prompt_beside_short_ones(encs, vocabs):
    """a prompt with thousands of chunks, spread over the emit grid's threads, among short and empty ones"""
    rng = random.Random(23)
    big = "".join(rng.choice(["\U00020b9f", "x", " ", "\U0001f600", "é", "word "]) for _ in range(6000)).encode()
    prompts = [b"short one", big, b"", "中文".encode()]
    for n_tok, overlap in ((3, 0), (8, 5)):
        rows = check(encs, vocabs, prompts, n_tok, overlap, [0], device_form=True)
        assert len(rows[1][0]) > 1000


def test_enospc_at_the_cap(encs, vocabs):
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(12, 30, max_atoms=30)]
    need = sum(len(reference(encs[0], p, 5, 1)[0]) for p in prompts)
    for device_form in (False, True):
        rc, spans, coffs, _ = chunk([vocabs[0]], prompts, 5, 1, cap=need - 1, device_form=device_form)
        assert rc == ENOSPC and int(coffs[-1]) == need
        if device_form:                              # the chunks below the cap are written, the rest are not
            rc2, full, coffs2, _ = chunk([vocabs[0]], prompts, 5, 1, cap=need, device_form=True)
            assert np.array_equal(spans[:need - 1], full[:need - 1])
        rc, spans, coffs, _ = chunk([vocabs[0]], prompts, 5, 1, cap=need, device_form=device_form)
        assert rc == 0 and int(coffs[-1]) == need


def test_error_codes(vocabs):
    prompts = [b"hello world", b"more text"]
    assert chunk([vocabs[0]], prompts, 0, 0)[0] == EINVAL
    assert chunk([vocabs[0]], prompts, 4, 4)[0] == EINVAL
    assert chunk([vocabs[0]], prompts, 4, 9)[0] == EINVAL
    for null in ("spans", "offsets"):
        assert chunk([vocabs[0]], prompts, 4, 1, null=null)[0] == EINVAL
    assert chunk([vocabs[0]], [b"ok", b"bad \xff utf-8"], 4, 0)[0] == EILSEQ
    assert chunk([vocabs[0]], prompts, 4, 0, vocab_ids=np.array([0, 5], np.uint8))[0] == ENOENT


def test_service_over_the_emulator_equals_the_host_default(encs, vocabs):
    """LlmGatewayTokenizerService.chunk over a plugin whose chunk_batch is the emulated device path equals the same service over the
    trait's host default (encode_batch with starts, then chunk_spans), and rebuilds the reference's chunks"""
    from cfbpe import plugin as P

    class Starts(P.TokenizerPluginClient):          # the default chunk_batch, over exact ids and starts from tiktoken
        def encode_batch(self, ctx, req):
            assert req.with_starts
            n = len(req.offsets) - 1
            ids, starts, counts = [], [], []
            for i in range(n):
                t = bytes(req.bytes[int(req.offsets[i]):int(req.offsets[i + 1])]).decode()
                e = encs[0].encode_ordinary(t)
                ln = [len(encs[0].decode_single_token_bytes(x)) for x in e]
                ids += e
                starts += np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(int).tolist() if e else []
                counts.append(len(e))
            off = np.zeros(n + 1, np.uint64)
            off[1:] = np.cumsum(counts)
            return P.EncodeBatchResponse(np.array(ids, np.uint32), off, np.array(counts, np.uint32), np.array(starts, np.uint32))

    class Emulated(P.TokenizerPluginClient):
        def chunk_batch(self, ctx, req, chunk_tokens, overlap_tokens=0):
            n_tok, overlap = P._chunk_args(chunk_tokens, overlap_tokens)
            n = len(req.offsets) - 1
            prompts = [bytes(req.bytes[int(req.offsets[i]):int(req.offsets[i + 1])]) for i in range(n)]
            rc, spans, coffs, counts = chunk([vocabs[0]], prompts, n_tok, overlap)
            assert rc == 0
            return P.ChunkBatchResponse(spans[:int(coffs[-1])], coffs, counts)

    def service(plugin):
        hub = P.ClientHub()
        inst = P.PluginInstance("gts.emulated", "cyberfabric", 0)
        hub.register_scoped(P.TokenizerPluginClient, inst.id, plugin)
        return P.LlmGatewayTokenizerService(hub, [inst])

    texts = fuzzgen.fuzz_strings(88, 80, max_atoms=40) + multibyte_texts(5, 40) + ["", "Hello, world! " * 20]
    sec = P.SecurityContext.anonymous()
    a, b = service(Emulated()), service(Starts())
    for n_tok, overlap in ((1, 0), (6, 2), (50, 0)):
        got = a.chunk(sec, "x", texts, n_tok, overlap)
        assert got == b.chunk(sec, "x", texts, n_tok, overlap)
        for t, chunks in zip(texts, got):
            want, _ = reference(encs[0], t.encode(), n_tok, overlap)
            assert chunks == [t.encode()[x:y].decode() for x, y in want]
            if overlap == 0:
                assert "".join(chunks) == t
    for bad in ((0, 0), (4, 4), (4, -1), (2.5, 0)):
        for svc in (a, b):
            with pytest.raises(P.InvalidInput):
                svc.chunk(sec, "x", texts, *bad)
