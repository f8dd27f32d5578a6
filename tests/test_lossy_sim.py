"""Encode of bytes that are not valid UTF-8 (utf8_scan / utf8_repair_emit / utf8_repair_offsets, csrc/utf8_repair.cuh) on the CPU
SIMT emulator: the repaired batch is CPython's b.decode("utf-8", "replace").encode("utf-8") prompt by prompt, every prompt's
replacement count is the number of times CPython calls a decode error handler on it (once per maximal subpart), and the ids are
the oracle's on the repaired text.  A batch of valid UTF-8 is never repaired."""
import codecs
import random

import numpy as np
import pytest

import fuzzgen
import simlib
from conftest import COMBOS
from lossy_lib import encode_batch_lossy
from simlib import EINVAL, ENOSPC

_calls = [0]


def _count_replace(exc):
    _calls[0] += 1
    return "�", exc.end


codecs.register_error("cfbpe_test_count_replace", _count_replace)


def cpython(p: bytes):
    """(R(p), U+FFFD inserted) by CPython"""
    _calls[0] = 0
    r = p.decode("utf-8", "cfbpe_test_count_replace").encode("utf-8")
    return r, _calls[0]


# one sample of every class of ill-formed input (the Unicode Standard, table 3-7)
STRAYS = [b"\x80", b"\xbf", b"\x80\xbf\x80", b"\xa0\xa0\xa0\xa0\xa0"]
BAD_LEADS = [b"\xc0", b"\xc1", b"\xf5", b"\xf8", b"\xfe", b"\xff", b"\xc0\xaf", b"\xc1\xbf", b"\xf5\x80\x80\x80", b"\xff\xbf"]
OVERLONGS = [b"\xe0\x80\x80", b"\xe0\x9f\xbf", b"\xf0\x80\x80\x80", b"\xf0\x8f\xbf\xbf"]
SURROGATES = [b"\xed\xa0\x80", b"\xed\xbf\xbf", b"\xed\xa0\x80\xed\xb0\x80"]
ABOVE_MAX = [b"\xf4\x90\x80\x80", b"\xf4\xbf\xbf\xbf"]
CUT_SHORT = [b"\xc3", b"\xdf", b"\xe2", b"\xe2\x82", b"\xef\xbf", b"\xf0", b"\xf0\x9f", b"\xf0\x9f\x98", b"\xf4\x8f\xbf", b"\xe0\xa0", b"\xed\x9f"]
CLASSES = {"stray": STRAYS, "bad_lead": BAD_LEADS, "overlong": OVERLONGS, "surrogate": SURROGATES, "above_max": ABOVE_MAX, "cut_short": CUT_SHORT}
AFTER = {"ascii": b"a b", "lead": "é€😀".encode(), "end": b""}
MULTILINGUAL = ["Grüße aus Köln", "日本語のテキストです。", "Привет, мир!", "مرحبا بالعالم", "emoji 😀👍🏽🎉", "𠀀𠀁𪚥", "a�b"]


@pytest.fixture(scope="module")
def vocabs(tekken_bytes):
    return {pat: simlib.SimVocab(tekken_bytes, 0, pat, n) for pat, n in COMBOS}


def check(vs, ov, pat, prompts, expect_repair=None, **layout):
    """the lossy call against CPython and the oracle on the repaired text (layout: where the batch's bytes lie, as
    lossy_lib.encode_batch_lossy takes it); returns the call's result"""
    out = encode_batch_lossy([vs], prompts, **layout)
    assert out["rc"] == 0
    want = [cpython(p) for p in prompts]
    assert out["replaced"] == [k for _, k in want]
    dirty = any(k for _, k in want)
    assert out["repaired"] == dirty and (out["dirty_lanes"] > 0) == dirty
    if expect_repair is not None:
        assert dirty == expect_repair
    if dirty:
        assert out["r"] == [r for r, _ in want]
        assert out["growth"] == sum(len(r) for r, _ in want) - sum(len(p) for p in prompts)
    else:
        assert out["growth"] == 0
    for i, (r, _) in enumerate(want):
        assert out["ids"][i] == ov.encode(pat, r).tolist(), (pat, prompts[i], r)
    assert out["counts"] == [len(x) for x in out["ids"]]
    return out


def at_every_lane_offset(body: bytes, lead_in=b"x"):
    """prompts that put `body` at every absolute batch position mod 32 (a 16-byte lane and the next), each after a lead-in of
    ASCII"""
    prompts, cur = [], 0
    for k in range(32):
        f = (k - cur) % 32 + 1
        p = lead_in * f + body
        prompts.append(p)
        cur += len(p)
    return prompts


@pytest.mark.parametrize("cls", sorted(CLASSES))
@pytest.mark.parametrize("after", sorted(AFTER))
def test_each_class_at_every_offset(vocabs, oracle_vocabs, cls, after):
    for bad in CLASSES[cls]:
        check(vocabs[3], oracle_vocabs[3], 3, at_every_lane_offset(bad + AFTER[after]), expect_repair=True)


def test_the_header_examples(vocabs, oracle_vocabs):
    for bad, n, r in [(b"\xf0\x9f\x98", 1, "�"), (b"\xed\xa0\x80", 3, "�" * 3), (b"\xc0\xaf", 2, "�" * 2),
                      (b"\xf4\x90\x80\x80", 4, "�" * 4), (b"\xf0\x9f\x98\x61", 1, "�a")]:
        out = check(vocabs[0], oracle_vocabs[0], 0, [bad])
        assert out["replaced"] == [n] and out["r"] == [r.encode()]


def test_sequences_never_span_prompts(vocabs, oracle_vocabs):
    """a lead byte that ends prompt i is a subpart of its own; the continuation bytes that open prompt i + 1 are strays"""
    for a, b in [(b"\xe2", b"\x82\xac"), (b"\xe2\x82", b"\xac"), (b"\xf0\x9f", b"\x98\x80"), (b"\xf0\x9f\x98", b"\x80"), (b"\xc3", b"\xa9")]:
        for f in range(32):
            prompts = [b"y" * f + b"abc" + a, b + b"def", b"", b + a, b]
            out = check(vocabs[1], oracle_vocabs[1], 1, prompts, expect_repair=True)
            assert out["replaced"][0] == 1 and out["replaced"][1] == len(b)


def test_empty_only_bad_and_existing_replacement_characters(vocabs, oracle_vocabs):
    prompts = [b"", b"\xff" * 40, b"", b"\x80" * 17, "a�b".encode() + b"\xff", "�".encode() * 5, b"", b"\xed\xa0\x80" * 11, b""]
    out = check(vocabs[2], oracle_vocabs[2], 2, prompts, expect_repair=True)
    assert out["replaced"] == [0, 40, 0, 17, 1, 0, 0, 33, 0]
    assert check(vocabs[2], oracle_vocabs[2], 2, [b"", b"", b""], expect_repair=False)["ids"] == [[], [], []]
    assert check(vocabs[2], oracle_vocabs[2], 2, [], expect_repair=False)["ids"] == []


def test_clean_batches_are_not_repaired(vocabs, oracle_vocabs):
    """valid UTF-8: a zero status, no repair, no replacement, and the ids of the strict path"""
    prompts = [t.encode() for t in fuzzgen.fuzz_strings(4711, 120, max_atoms=30)] + [t.encode() for t in MULTILINGUAL]
    for pat in (0, 3):
        out = check(vocabs[pat], oracle_vocabs[pat], pat, prompts, expect_repair=False)
        assert out["dirty_lanes"] == 0 and out["growth"] == 0 and not out["repaired"] and set(out["replaced"]) == {0}
        rc, ids, off, counts, _ = simlib.encode_batch([vocabs[pat]], prompts)
        assert rc == 0 and np.array_equal(out["offsets"], off) and out["counts"] == counts.tolist()


def _fuzz_prompt(rng: random.Random) -> bytes:
    parts = []
    for _ in range(rng.randrange(0, 12)):
        k = rng.randrange(6)
        if k == 0:
            parts.append(bytes(rng.randrange(256) for _ in range(rng.randrange(1, 9))))
        elif k == 1:
            parts.append(bytes(rng.choice([0x80, 0xBF, 0xC0, 0xC2, 0xE0, 0xED, 0xEF, 0xF0, 0xF4, 0xF5, 0xFF, 0x41]) for _ in range(rng.randrange(1, 6))))
        elif k == 2:
            t = rng.choice(MULTILINGUAL).encode()
            a = rng.randrange(len(t) + 1)
            parts.append(t[a:a + rng.randrange(1, 20)])        # cut anywhere, inside a character too
        else:
            parts.append(rng.choice(MULTILINGUAL).encode())
    return b"".join(parts)


@pytest.mark.parametrize("seed", range(6))
def test_fuzz_random_bytes_in_multilingual_text(vocabs, oracle_vocabs, seed):
    rng = random.Random(1000 + seed)
    pat = COMBOS[seed % len(COMBOS)][0]
    prompts = [_fuzz_prompt(rng) for _ in range(rng.randrange(20, 80))]
    check(vocabs[pat], oracle_vocabs[pat], pat, prompts)


def test_fuzz_at_odd_alignments_with_garbage_past_the_end(vocabs, oracle_vocabs):
    """the batch's first byte at every alignment, non-ASCII bytes before it and past its end: no result depends on them, and
    nothing is read more than 32 bytes past the end (guard page)"""
    rng = random.Random(77)
    for misalign in range(16):
        prompts = [_fuzz_prompt(rng) for _ in range(12)] + [b"abc\xe2"]
        check(vocabs[0], oracle_vocabs[0], 0, prompts, misalign=misalign, fill=b"\x82\xac\xbf\xf0", guard="before")
        check(vocabs[0], oracle_vocabs[0], 0, prompts, fill=b"\x80\x9f\xbf", guard="after")


def test_several_vocabularies(vocabs, oracle_vocabs):
    rng = random.Random(5)
    prompts = [_fuzz_prompt(rng) for _ in range(40)]
    vids = np.array([i % 4 for i in range(len(prompts))], dtype=np.uint8)
    vs = [vocabs[p] for p, _ in COMBOS]
    out = encode_batch_lossy(vs, prompts, vocab_ids=vids)
    assert out["rc"] == 0
    for i, p in enumerate(prompts):
        r, k = cpython(p)
        assert out["replaced"][i] == k
        assert out["ids"][i] == oracle_vocabs[int(vids[i])].encode(int(vids[i]), r).tolist()


def test_counts_only_enospc_and_the_repaired_size_limit(vocabs):
    prompts = [b"ab\xffcd", b"\xc0" * 10, "日本".encode()]
    full = encode_batch_lossy([vocabs[0]], prompts)
    assert full["rc"] == 0
    co = encode_batch_lossy([vocabs[0]], prompts, counts_only=True)
    assert co["rc"] == 0 and co["counts"] == full["counts"] and np.array_equal(co["offsets"], full["offsets"]) and co["ids"] is None
    need = int(full["offsets"][-1])
    ns = encode_batch_lossy([vocabs[0]], prompts, out_cap=need - 1)
    assert ns["rc"] == ENOSPC and int(ns["offsets"][-1]) == need
    r_total = sum(len(cpython(p)[0]) for p in prompts)
    assert encode_batch_lossy([vocabs[0]], prompts, max_bytes=r_total)["rc"] == 0
    assert encode_batch_lossy([vocabs[0]], prompts, max_bytes=r_total - 1)["rc"] == EINVAL
