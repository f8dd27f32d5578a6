"""Token starts in code points and UTF-16 units (unit_len / unit_tile_scan / unit_emit, csrc/bpe_kernels.cuh) on the CPU SIMT
emulator: code-point starts are live tiktoken 0.12.0's `decode_with_offsets`, UTF-16 starts are the UTF-16 length of the text
before the character that holds the token's first byte, the lengths are len(text) and its UTF-16 length, and the ids / offsets /
counts are those of the plain path."""
import base64

import numpy as np
import pytest

import fuzzgen
import simlib
import vocab_shapes as VS
from cfbpe.plugin import unit_starts
from char_starts_lib import UNIT_CODEPOINT, UNIT_UTF16, encode_char_starts
from conftest import COMBOS, golden_cases
from simlib import EINVAL, ENOSPC

UNITS = {"codepoint": UNIT_CODEPOINT, "utf16": UNIT_UTF16}
MULTILINGUAL = ["Grüße aus Köln", "日本語のテキストです。", "Привет, мир!", "مرحبا بالعالم", "नमस्ते दुनिया", "한국어 텍스트",
                "emoji 😀👍🏽🎉 and flags 🇩🇪🇯🇵", "family 👨‍👩‍👧‍👦 zwj", "CJK Ext B 𠀀𠀁𠀂𪚥 and 𝔘𝔫𝔦𝔠𝔬𝔡𝔢", "math 𝑥² + 𝑦² = 𝑧²",
                "mixed aé中😀 \n1 𐍈 ẞ", "😀" * 40, "𠀀" * 33, "é" * 300, ""]


@pytest.fixture(scope="module")
def vocabs(tekken_bytes):
    return {pat: simlib.SimVocab(tekken_bytes, 0, pat, n) for pat, n in COMBOS}


def by_formula(p: bytes, x: int, unit: str) -> int:
    """units before the character that holds byte x of p: len(b[:F(x)].decode()) in code points or UTF-16 units"""
    while 0 < x < len(p) and p[x] & 0xC0 == 0x80:
        x -= 1
    t = p[:x].decode()
    return len(t) if unit == "codepoint" else len(t.encode("utf-16-le")) // 2


def check(vs, prompts, vocab_ids=None, formula=False):
    """both units: ids / offsets / counts equal the plain path's, starts and lengths equal unit_starts (and, with formula, the
    per-token formula); returns the code-point starts and the offsets"""
    prc, pids, poff, pcounts, _ = simlib.encode_batch(vs, prompts, vocab_ids=vocab_ids)
    assert prc == 0
    brc, _, bstarts, _, _ = simlib.encode_starts(vs, prompts, vocab_ids)
    assert brc == 0
    data, offs = simlib.pack(prompts)
    out = None
    for name, unit in UNITS.items():
        rc, ids, starts, off, counts, lens = encode_char_starts(vs, prompts, unit, vocab_ids)
        assert rc == 0
        assert np.array_equal(off, poff) and np.array_equal(counts, pcounts)
        assert np.array_equal(ids, pids[:int(poff[-1])])
        want, want_lens = unit_starts(data, offs, off, bstarts, name)
        assert np.array_equal(starts, want), name
        assert np.array_equal(lens, want_lens), name
        for i, p in enumerate(prompts):
            t = p.decode()
            assert int(lens[i]) == (len(t) if name == "codepoint" else len(t.encode("utf-16-le")) // 2)
            a, b = int(off[i]), int(off[i + 1])
            st = starts[a:b].astype(np.int64)
            assert (b == a) or (st[0] == 0 and np.all(np.diff(st) >= 0) and st[-1] <= int(lens[i]))
            if formula:
                assert st.tolist() == [by_formula(p, int(x), name) for x in bstarts[a:b]], (name, i)
        if name == "codepoint":
            out = (starts, off)
    return out


@pytest.mark.parametrize("pat,n_ranks", COMBOS)
def test_golden_fuzz_multilingual(golden, vocabs, pat, n_ranks):
    prompts = golden_cases(golden) + [s.encode() for s in fuzzgen.fuzz_strings(50 + pat, 300, max_atoms=40)]
    prompts += [t.encode() for t in MULTILINGUAL] + [b"", b"", b"x", b""]
    check([vocabs[pat]], prompts, formula=True)


@pytest.mark.parametrize("pat,n_ranks", COMBOS)
def test_against_live_tiktoken_decode_with_offsets(tekken_bytes, vocabs, pat, n_ranks):
    tiktoken = pytest.importorskip("tiktoken")
    from oracle import patterns as PT
    ranks = {base64.b64decode(l.split()[0]): i for i, l in enumerate(tekken_bytes.splitlines()[:n_ranks])}
    enc = tiktoken.Encoding("live%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks, special_tokens={})
    texts = fuzzgen.fuzz_strings(800 + pat, 250, max_atoms=40) + fuzzgen.long_runs(pat)[:30] + MULTILINGUAL
    starts, off = check([vocabs[pat]], [t.encode() for t in texts])
    for i, t in enumerate(texts):
        a, b = int(off[i]), int(off[i + 1])
        text, want = enc.decode_with_offsets(enc.encode_ordinary(t))
        assert text == t
        assert starts[a:b].tolist() == want, repr(t)


@pytest.mark.parametrize("name", ["utf8_random", "scattered_bytes"])
def test_vocab_shapes_that_split_characters(name):
    """rank files whose tokens start and end inside characters (several byte tokens of one character share a start)"""
    rf, texts = VS.shape(name)
    texts = texts[:400] + MULTILINGUAL
    for pat in (0, 3):
        v = simlib.SimVocab(rf, 0, pat)
        check([v], [t.encode() for t in texts], formula=True)


def test_tiles_and_prompts_across_tiles(vocabs):
    """prompts that span several 2048-token tiles, tiles that hold many prompt starts, and empty prompts between them"""
    rng = np.random.default_rng(5)
    alphabet = list("ab é中😀𠀀\n")
    long_t = "".join(rng.choice(alphabet, 9000))
    prompts = [long_t.encode(), b"", "😀".encode() * 2100, b""] + [("x%d 中" % i).encode() for i in range(3000)]
    prompts += [b"", long_t[:5000].encode(), b""]
    check([vocabs[0]], prompts)
    check([vocabs[0]], [b"", b"", b""])


def test_mixed_vocabulary_batch(vocabs):
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(31, 300, max_atoms=40)] + [t.encode() for t in MULTILINGUAL]
    vid = np.array([i % 4 for i in range(len(prompts))], dtype=np.uint8)
    check([vocabs[p] for p, _ in COMBOS], prompts, vocab_ids=vid)


def test_errors(vocabs):
    prompts = [b"hello world, this is a test", "and more 😀".encode()]
    for unit in (UNIT_CODEPOINT, UNIT_UTF16):
        rc, _, _, off, _, _ = encode_char_starts([vocabs[0]], prompts, unit, out_cap=2)
        assert rc == ENOSPC and int(off[-1]) == int(simlib.encode_batch([vocabs[0]], prompts)[2][-1])
    assert encode_char_starts([vocabs[0]], prompts, 2)[0] == EINVAL
    assert encode_char_starts([vocabs[0]], prompts, 0xFFFFFFFF)[0] == EINVAL
    assert encode_char_starts([vocabs[0]], prompts, UNIT_UTF16, null="ids")[0] == EINVAL
    assert encode_char_starts([vocabs[0]], prompts, UNIT_CODEPOINT, null="starts")[0] == EINVAL
    rc, _, starts, _, _, _ = encode_char_starts([vocabs[0]], prompts, UNIT_UTF16, null="lens")     # the lengths are optional
    assert rc == 0 and starts[0] == 0


def test_encode_with_offsets_units_over_the_emulator(vocabs):
    """LlmGatewayTokenizerService.encode_with_offsets(unit=...): spans slice every str back into exactly its text, through a
    plugin that honours starts_unit and through the trait default (byte starts converted on the host)"""
    from cfbpe import plugin as P

    class Emulated(P.TokenizerPluginClient):
        def __init__(self, units):
            self.units = units

        def encode_batch(self, ctx, req):
            n = len(req.offsets) - 1
            prompts = [bytes(req.bytes[int(req.offsets[i]):int(req.offsets[i + 1])]) for i in range(n)]
            if self.units and req.with_starts and req.starts_unit != "byte":
                rc, ids, starts, off, counts, lens = encode_char_starts([vocabs[0]], prompts, UNITS[req.starts_unit])
                assert rc == 0
                return P.EncodeBatchResponse(ids, off, counts, starts, lens)
            rc, ids, starts, off, counts = simlib.encode_starts([vocabs[0]], prompts)
            assert rc == 0
            return P.EncodeBatchResponse(ids, off, counts, starts if req.with_starts else None)

        def encode_batch_unit_starts(self, ctx, req):
            return self.encode_batch(ctx, req) if self.units else super().encode_batch_unit_starts(ctx, req)

    texts = fuzzgen.fuzz_strings(89, 200, max_atoms=40) + MULTILINGUAL + ["Hello, 世界! 😀 " * 20]
    for units in (True, False):
        hub = P.ClientHub()
        inst = P.PluginInstance("gts.emulated", "cyberfabric", 0)
        hub.register_scoped(P.TokenizerPluginClient, inst.id, Emulated(units))
        svc = P.LlmGatewayTokenizerService(hub, [inst])
        for unit in ("byte", "codepoint", "utf16"):
            got = svc.encode_with_offsets(P.SecurityContext.anonymous(), "x", texts, unit=unit)
            for t, (ids, spans) in zip(texts, got):
                s = t.encode() if unit == "byte" else t if unit == "codepoint" else t.encode("utf-16-le")
                w = 2 if unit == "utf16" else 1
                assert len(ids) == len(spans)
                assert type(s)().join(s[int(a) * w:int(e) * w] for a, e in spans) == s, (unit, t)
                assert all(int(a) <= int(e) for a, e in spans)
        with pytest.raises(P.InvalidInput):
            svc.encode_with_offsets(P.SecurityContext.anonymous(), "x", texts, unit="utf32")
