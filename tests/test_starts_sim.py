"""Token byte starts (starts_len / starts_emit, csrc/bpe_kernels.cuh) on the CPU SIMT emulator: every start is the exclusive
prefix sum of the byte lengths of the prompt's tokens before it, the ids / offsets / counts are those of the plain path, and the
starts give live tiktoken 0.12.0's `decode_with_offsets` under its own byte -> character rule."""
import base64
import random

import numpy as np
import pytest

import fuzzgen
import simlib
from conftest import COMBOS, golden_cases
from simlib import ENOSPC, encode_starts


@pytest.fixture(scope="module")
def vocabs(tekken_bytes):
    return {pat: simlib.SimVocab(tekken_bytes, 0, pat, n) for pat, n in COMBOS}


@pytest.fixture(scope="module")
def tok_lens(tekken_bytes):
    """byte length of every rank of the committed rank file (each slot keeps a prefix of it)"""
    return np.array([len(base64.b64decode(l.split()[0])) for l in tekken_bytes.splitlines()], dtype=np.int64)


def check(vocabs, lens, prompts, vocab_ids=None):
    """starts obey the prefix-sum rule; ids, offsets and counts equal the plain path's"""
    rc, ids, starts, off, counts = encode_starts(vocabs, prompts, vocab_ids)
    assert rc == 0
    prc, pids, poff, pcounts, _ = simlib.encode_batch(vocabs, prompts, vocab_ids=vocab_ids)
    assert prc == 0
    assert np.array_equal(off, poff)
    assert np.array_equal(ids, pids[:int(poff[-1])])
    assert np.array_equal(counts, pcounts)
    for i, p in enumerate(prompts):
        a, b = int(off[i]), int(off[i + 1])
        ln = lens[ids[a:b]]
        assert int(ln.sum()) == len(p), i
        want = np.concatenate([[0], np.cumsum(ln)[:-1]]) if b > a else np.zeros(0, np.int64)
        assert np.array_equal(starts[a:b].astype(np.int64), want), (i, p[:80])
    return ids, starts, off


@pytest.mark.parametrize("pat,n_ranks", COMBOS)
def test_golden_cases_starts_and_parity(golden, vocabs, tok_lens, pat, n_ranks):
    cases = golden_cases(golden)
    check([vocabs[pat]], tok_lens, cases)


def test_layouts(vocabs, tok_lens):
    rng = random.Random(11)
    words = [s.encode() for s in fuzzgen.fuzz_strings(3, 400, max_atoms=4)]
    prompts = [w for w in words[:300]]                        # many prompts inside one 1 KiB window, empty ones among them
    prompts += [b"", b"", b"a", b"", b" "]
    used = sum(len(p) for p in prompts)
    pad = (-used) % 1024
    prompts.append(b"x" * (pad - 1) + b"." if pad else b"")  # ... so that the next prompt starts at the first bit of a window
    prompts.append(b"Hello world")
    used = sum(len(p) for p in prompts)
    prompts.append(b"y" * ((31 - used) % 32 + 32))            # the next one starts at the last byte of a word
    assert sum(len(p) for p in prompts) % 32 == 31
    prompts.append(b"q and more")
    letters = "abcdefghijklmnopqrstuvwxyz"
    long_one = "".join(rng.choice(letters) for _ in range(40)) + " " + " " * 300 + "".join(rng.choice(letters) for _ in range(600))
    long_one += " " + "=" * 3000 + " end" + "".join(rng.choice("etaoin") for _ in range(270))
    prompts.append(long_one.encode())                         # several windows; pieces > 32 B and > 256 B (ids by position)
    prompts += [b"", b"tail"]
    for pat in (0, 3):
        check([vocabs[pat]], tok_lens, prompts)


def test_empty_prompts_only_and_edges(vocabs, tok_lens):
    check([vocabs[0]], tok_lens, [b"", b"", b""])
    check([vocabs[0]], tok_lens, [b"", b"a", b"", b"", b"bc", b""])
    check([vocabs[0]], tok_lens, [b"x" * 1024, b"y" * 1023, b"", b"z"])


def test_mixed_vocabulary_batch(vocabs, tok_lens):
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(31, 300, max_atoms=40)] + [s.encode() for s in fuzzgen.long_runs(2)[:40]]
    vid = np.array([i % 4 for i in range(len(prompts))], dtype=np.uint8)
    check([vocabs[p] for p, _ in COMBOS], tok_lens, prompts, vocab_ids=vid)


def test_out_cap_too_small(vocabs):
    rc, _, _, off, _ = encode_starts([vocabs[0]], [b"hello world, this is a test", b"and more"], out_cap=2)
    assert rc == ENOSPC and int(off[-1]) > 2


@pytest.mark.parametrize("pat,n_ranks", COMBOS)
def test_against_live_tiktoken_decode_with_offsets(tekken_bytes, vocabs, pat, n_ranks):
    tiktoken = pytest.importorskip("tiktoken")
    from oracle import patterns as PT
    ranks = {base64.b64decode(l.split()[0]): i for i, l in enumerate(tekken_bytes.splitlines()[:n_ranks])}
    enc = tiktoken.Encoding("live%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks, special_tokens={})
    texts = fuzzgen.fuzz_strings(700 + pat, 250, max_atoms=40) + fuzzgen.long_runs(pat)[:30]
    prompts = [t.encode() for t in texts]
    rc, ids, starts, off, _ = encode_starts([vocabs[pat]], prompts)
    assert rc == 0
    for i, (t, p) in enumerate(zip(texts, prompts)):
        a, b = int(off[i]), int(off[i + 1])
        want_ids = enc.encode_ordinary(t)
        assert ids[a:b].tolist() == want_ids
        text, want = enc.decode_with_offsets(want_ids)
        assert text == t
        # tiktoken's rule: characters (non-continuation bytes) before the token's first byte, one less when that byte is a
        # continuation byte (the token starts inside a character)
        got = []
        for s in starts[a:b].tolist():
            chars = sum(1 for c in p[:s] if not 0x80 <= c < 0xC0)
            got.append(max(0, chars - (1 if 0x80 <= p[s] < 0xC0 else 0)))
        assert got == want, repr(t)


def test_encode_with_offsets_service_over_the_emulator(vocabs):
    """LlmGatewayTokenizerService.encode_with_offsets: spans rebuild every text; a plugin without starts is refused"""
    from cfbpe import plugin as P

    class Emulated(P.TokenizerPluginClient):
        def __init__(self, with_starts=True):
            self.with_starts = with_starts

        def encode_batch(self, ctx, req):
            n = len(req.offsets) - 1
            prompts = [bytes(req.bytes[int(req.offsets[i]):int(req.offsets[i + 1])]) for i in range(n)]
            rc, ids, starts, off, counts = encode_starts([vocabs[0]], prompts)
            assert rc == 0
            return P.EncodeBatchResponse(ids, off, counts, starts if (req.with_starts and self.with_starts) else None)

    texts = fuzzgen.fuzz_strings(88, 200, max_atoms=40) + ["", "Hello, world! " * 20]
    for with_starts in (True, False):
        hub = P.ClientHub()
        inst = P.PluginInstance("gts.emulated", "cyberfabric", 0)
        hub.register_scoped(P.TokenizerPluginClient, inst.id, Emulated(with_starts))
        svc = P.LlmGatewayTokenizerService(hub, [inst])
        if not with_starts:
            with pytest.raises(P.ServiceUnavailable):
                svc.encode_with_offsets(P.SecurityContext.anonymous(), "x", texts)
            continue
        got = svc.encode_with_offsets(P.SecurityContext.anonymous(), "x", texts)
        for t, (ids, spans) in zip(texts, got):
            b = t.encode()
            assert len(ids) == len(spans)
            assert b"".join(b[int(s):int(e)] for s, e in spans) == b
            assert all(int(s) < int(e) for s, e in spans)
