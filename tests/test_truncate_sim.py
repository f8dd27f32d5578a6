"""Truncation to token budgets (truncate / truncate_long, csrc/bpe_kernels.cuh) on the CPU SIMT emulator, against a reference
built here from live tiktoken 0.12.0: decode_bytes of the first / last k ids, moved to a character boundary (include/cfbpe.h,
cfbpe_truncate_batch)."""
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
import build_truncate  # noqa: E402

HEAD, TAIL = 0, 1
EINVAL, ENOENT, EILSEQ = -22, -2, -84
MAX_BUDGET = 2 ** 32 - 1
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_truncate.build())
        L.sim_vocab_build.restype = C.c_void_p
        L.sim_vocab_build.argtypes = [C.c_char_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p, C.c_size_t]
        L.sim_vocab_free.argtypes = [C.c_void_p]
        L.sim_truncate_batch.restype = C.c_int
        L.sim_truncate_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                         C.c_void_p, C.c_void_p, C.c_void_p]
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


def truncate(vocabs, prompts, budgets, mode, vocab_ids=None, null=None):
    """(rc, cut, kept, counts); null: the name of an argument to pass as NULL"""
    data, offs = simlib.pack(prompts)
    n = len(prompts)
    bud = np.ascontiguousarray(np.broadcast_to(np.asarray(budgets, dtype=np.uint64), (n,)).astype(np.uint32)) if n else np.zeros(1, np.uint32)
    cut = np.full(max(n, 1), 0xFFFFFFFF, dtype=np.uint32)
    kept = np.full(max(n, 1), 0xFFFFFFFF, dtype=np.uint32)
    counts = np.zeros(max(n, 1), dtype=np.uint32)
    vh = (C.c_void_p * len(vocabs))(*[v._h for v in vocabs])
    vid = None if vocab_ids is None else np.ascontiguousarray(vocab_ids, dtype=np.uint8)
    dbuf = np.concatenate([data, np.zeros(8, np.uint8)])
    rc = lib().sim_truncate_batch(vh, len(vocabs), n, dbuf.ctypes.data, offs.ctypes.data, None if vid is None else vid.ctypes.data,
                                  None if null == "budgets" else bud.ctypes.data, mode, None if null == "cut" else cut.ctypes.data,
                                  None if null == "kept" else kept.ctypes.data, counts.ctypes.data)
    return rc, cut[:n], kept[:n], counts[:n]


def is_cont(b):
    return 0x80 <= b < 0xC0


def reference(enc, prompt: bytes, budget: int, mode: int):
    """(cut, kept, count, x) by the contract, from live tiktoken: x is the unsnapped token boundary"""
    ids = enc.encode_ordinary(prompt.decode("utf-8"))
    c, n = len(ids), len(prompt)
    k = min(budget, c)
    lens = [len(enc.decode_single_token_bytes(t)) for t in ids]
    if mode == HEAD:
        x = len(enc.decode_bytes(ids[:k]))
        cut = x
        while 0 < cut < n and is_cont(prompt[cut]):
            cut -= 1
        ends = np.cumsum(lens) if c else np.zeros(0, np.int64)
        kept = int((ends <= cut).sum())
    else:
        x = n - len(enc.decode_bytes(ids[c - k:]))
        cut = x
        while cut < n and is_cont(prompt[cut]):
            cut += 1
        st = np.concatenate([[0], np.cumsum(lens)[:-1]]) if c else np.zeros(0, np.int64)
        kept = int((st >= cut).sum())
    return cut, kept, c, x


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


def budget_kinds(c, rng):
    """the budgets every prompt is checked with: 0, 1, c - 1, c, c + 1, 2^32 - 1, about half, any"""
    return [0, 1, max(c - 1, 0), c, c + 1, MAX_BUDGET, c // 2, rng.randint(0, c + 2)]


def check(encs, vocabs, prompts, budgets, mode, pats, vocab_ids=None):
    """the emulator equals the reference for every prompt; returns the reference rows"""
    rc, cut, kept, counts = truncate([vocabs[p] for p in pats], prompts, budgets, mode, vocab_ids)
    assert rc == 0
    rows = []
    for i, p in enumerate(prompts):
        enc = encs[pats[0] if vocab_ids is None else pats[int(vocab_ids[i])]]
        want = reference(enc, p, int(budgets[i]), mode)
        assert (int(cut[i]), int(kept[i]), int(counts[i])) == want[:3], (i, mode, int(budgets[i]), p[:60])
        rows.append(want)
    return rows


@pytest.mark.parametrize("mode", [HEAD, TAIL])
@pytest.mark.parametrize("pat,n_ranks", COMBOS)
def test_golden_cases(golden, encs, vocabs, pat, n_ranks, mode):
    cases = golden_cases(golden)
    rng = random.Random(pat * 2 + mode)
    counts = [len(encs[pat].encode_ordinary(p.decode())) for p in cases]
    budgets = np.array([budget_kinds(c, rng)[(i + mode) % 8] for i, c in enumerate(counts)], dtype=np.uint64)
    check(encs, vocabs, cases, budgets, mode, [pat])


def test_budget_edges(encs, vocabs):
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(5, 60, max_atoms=30)] + [b"Hello, world! " * 12, "日本語のテキスト".encode()]
    rng = random.Random(3)
    counts = [len(encs[0].encode_ordinary(p.decode())) for p in prompts]
    for kind in range(8):
        budgets = np.array([budget_kinds(c, rng)[kind] for c in counts], dtype=np.uint64)
        for mode in (HEAD, TAIL):
            rows = check(encs, vocabs, prompts, budgets, mode, [0])
            for (cut, kept, c, _), p, bgt in zip(rows, prompts, budgets):
                if bgt == 0:
                    assert (cut, kept) == ((0 if mode == HEAD else len(p)), 0)
                if bgt >= c:
                    assert (cut, kept) == ((len(p) if mode == HEAD else 0), c)


def test_empty_prompts_long_pieces_and_layouts(encs, vocabs):
    rng = random.Random(17)
    letters = "abcdefghijklmnopqrstuvwxyz"
    long_one = "".join(rng.choice(letters) for _ in range(40)) + " " * 300 + "".join(rng.choice(letters) for _ in range(600))
    long_one += " " + "=" * 3000 + " end" + "".join(rng.choice("etaoin") for _ in range(270))
    prompts = [b"", b"", b"a", b"", long_one.encode(), b"", b"x" * 1023, "中" * 700, b"tail"]
    prompts = [p if isinstance(p, bytes) else p.encode() for p in prompts]
    for pat in (0, 3):
        counts = [len(encs[pat].encode_ordinary(p.decode())) for p in prompts]
        for kind in (1, 2, 6):
            budgets = np.array([budget_kinds(c, rng)[kind] for c in counts], dtype=np.uint64)
            for mode in (HEAD, TAIL):
                check(encs, vocabs, prompts, budgets, mode, [pat])
    rc, cut, kept, counts = truncate([vocabs[0]], [b"", b"", b""], 5, TAIL)
    assert rc == 0 and cut.tolist() == [0, 0, 0] and kept.tolist() == [0, 0, 0] and counts.tolist() == [0, 0, 0]


def test_mixed_vocabulary_batch(encs, vocabs):
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(31, 200, max_atoms=40)] + [s.encode() for s in fuzzgen.long_runs(2)[:40]]
    vid = np.array([i % 4 for i in range(len(prompts))], dtype=np.uint8)
    pats = [p for p, _ in COMBOS]
    rng = random.Random(8)
    counts = [len(encs[pats[v]].encode_ordinary(p.decode())) for p, v in zip(prompts, vid)]
    budgets = np.array([budget_kinds(c, rng)[i % 8] for i, c in enumerate(counts)], dtype=np.uint64)
    for mode in (HEAD, TAIL):
        check(encs, vocabs, prompts, budgets, mode, pats, vocab_ids=vid)


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


def test_cuts_inside_characters_are_snapped(encs, vocabs):
    texts = multibyte_texts(99, 300)
    prompts = [t.encode() for t in texts]
    rng = random.Random(4)
    for pat in (0, 1):
        counts = [len(encs[pat].encode_ordinary(t)) for t in texts]
        budgets = np.array([rng.randint(1, max(c - 1, 1)) for c in counts], dtype=np.uint64)
        for mode in (HEAD, TAIL):
            rows = check(encs, vocabs, prompts, budgets, mode, [pat])
            moved = [(cut, kept, c, x, b) for (cut, kept, c, x), b in zip(rows, budgets) if cut != x]
            # the data holds token boundaries inside characters, and the cut moved off them (dropping the tokens it cut through)
            assert len(moved) >= 20, (pat, mode, len(moved))
            assert all(kept < min(int(b), c) for cut, kept, c, x, b in moved)
            for (cut, kept, c, x), p in zip(rows, prompts):
                kept_text = p[:cut] if mode == HEAD else p[cut:]
                kept_text.decode("utf-8")                         # valid UTF-8, always


def test_long_prompt_spread_over_warps(encs, vocabs):
    """a prompt with more ids to sum than one warp takes (truncate_long: parts, the last to arrive finishes) beside short ones"""
    rng = random.Random(23)
    big = "".join(rng.choice(["\U00020b9f", "\U0002a6d6", "x", " ", "\U0001f600", "é"]) for _ in range(12000)).encode()
    prompts = [b"short one", big, "中文".encode(), big[:20000].decode("utf-8", "ignore").encode()]
    counts = [len(encs[0].encode_ordinary(p.decode())) for p in prompts]
    assert counts[1] > 4 * 4096, counts                       # half the ids of the big prompt are several warps' parts
    for mode in (HEAD, TAIL):
        for frac in (0.5, 0.3, 0.8):
            budgets = np.array([int(c * frac) for c in counts], dtype=np.uint64)
            check(encs, vocabs, prompts, budgets, mode, [0])


def test_error_codes(vocabs):
    prompts = [b"hello world", b"more text"]
    for mode in (2, 0xFFFFFFFF):
        assert truncate([vocabs[0]], prompts, 3, mode)[0] == EINVAL
    for null in ("budgets", "cut", "kept"):
        assert truncate([vocabs[0]], prompts, 3, HEAD, null=null)[0] == EINVAL
    assert truncate([vocabs[0]], [b"ok", b"bad \xff utf-8"], 3, HEAD)[0] == EILSEQ
    assert truncate([vocabs[0]], prompts, 3, TAIL, vocab_ids=np.array([0, 5], np.uint8))[0] == ENOENT


def test_service_over_the_emulator_equals_the_host_default(encs, vocabs):
    """LlmGatewayTokenizerService.truncate over a plugin whose truncate_batch is the emulated device path equals the same service
    over the trait's host default (encode_batch with starts), and rebuilds what the reference keeps"""
    from cfbpe import plugin as P

    class Starts(P.TokenizerPluginClient):          # the default truncate_batch, over exact ids and starts from tiktoken
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
        def truncate_batch(self, ctx, req, budgets, keep="head"):
            n = len(req.offsets) - 1
            prompts = [bytes(req.bytes[int(req.offsets[i]):int(req.offsets[i + 1])]) for i in range(n)]
            rc, cut, kept, counts = truncate([vocabs[0]], prompts, P._budgets(budgets, n), P._truncate_mode(keep))
            assert rc == 0
            return P.TruncateBatchResponse(cut, kept, counts)

    def service(plugin):
        hub = P.ClientHub()
        inst = P.PluginInstance("gts.emulated", "cyberfabric", 0)
        hub.register_scoped(P.TokenizerPluginClient, inst.id, plugin)
        return P.LlmGatewayTokenizerService(hub, [inst])

    texts = fuzzgen.fuzz_strings(88, 120, max_atoms=40) + multibyte_texts(5, 60) + ["", "Hello, world! " * 20]
    sec = P.SecurityContext.anonymous()
    a, b = service(Emulated()), service(Starts())
    rng = random.Random(6)
    per_text = [rng.randint(0, 40) for _ in texts]
    for keep, mode in (("head", HEAD), ("tail", TAIL)):
        for budgets in (7, per_text, 0, MAX_BUDGET):
            got = a.truncate(sec, "x", texts, budgets, keep)
            assert got == b.truncate(sec, "x", texts, budgets, keep)
            for t, (kept_text, kept, count), bgt in zip(texts, got, np.broadcast_to(np.asarray(budgets), (len(texts),))):
                cut, want_kept, c, _ = reference(encs[0], t.encode(), int(bgt), mode)
                want_text = t.encode()[:cut] if mode == HEAD else t.encode()[cut:]
                assert (kept_text.encode(), kept, count) == (want_text, want_kept, c)
    with pytest.raises(P.InvalidInput):
        a.truncate(sec, "x", texts, 5, "middle")
    with pytest.raises(P.InvalidInput):
        b.truncate(sec, "x", texts, -1, "head")
