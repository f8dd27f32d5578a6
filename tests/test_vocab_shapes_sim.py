"""Rank files shaped like real ones (tests/vocab_shapes.py: bytes at scattered ranks, tokens of up to 255 bytes, more than
2^20 ranks, random ranks over multi-byte UTF-8, lengths at every kernel threshold) on the CPU SIMT emulator and the oracle,
against live tiktoken 0.12.0 built from the same rank file.  The path counters check that each shape reached the code it is
meant for."""
import os
import random

import numpy as np
import pytest

import fuzzgen
import simlib
import vocab_shapes as VS
from oracle import oracle
from test_chunk_sim import reference as chunk_reference
from test_truncate_sim import HEAD, TAIL, reference as truncate_reference

PATTERNS = [0, 1, 2, 3]
LIST_COUNTERS = (0, 2)          # bpe_list_kernel took a big piece
GLOBAL_LIST_PATH = 5            # bpe_long_kernel's list rounds on a piece in global memory


def tiktoken_encoding(rf, pat, name="shape"):
    tiktoken = pytest.importorskip("tiktoken")
    from oracle import patterns as PT
    return tiktoken.Encoding(name, pat_str=PT.PATTERNS[pat], mergeable_ranks={t: i for i, t in enumerate(VS.tokens_of(rf))},
                             special_tokens={})


@pytest.fixture(scope="module")
def shapes():
    return {name: VS.shape(name) for name in VS.SHAPES}


@pytest.fixture(scope="module")
def encs(shapes):
    cache = {}

    def get(name, pat):
        if (name, pat) not in cache:
            cache[(name, pat)] = tiktoken_encoding(shapes[name][0], pat, "%s%d" % (name, pat))
        return cache[(name, pat)]
    return get


def want_batch(enc, texts):
    want = enc.encode_ordinary_batch(texts, num_threads=min(8, os.cpu_count() or 1))
    off = np.zeros(len(texts) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(w) for w in want])
    ids = np.concatenate([np.asarray(w, dtype=np.uint32) for w in want]) if want else np.zeros(0, np.uint32)
    return ids, off, np.array([len(w) for w in want], dtype=np.uint32)


def reset_counters():
    for i in range(8):
        simlib.dbg_counter(i, reset=True)


@pytest.mark.parametrize("pat", PATTERNS)
@pytest.mark.parametrize("name", VS.SHAPES)
def test_emulator_matches_tiktoken(shapes, encs, name, pat):
    rf, texts = shapes[name]
    sv = simlib.SimVocab(rf, 0, pat, 0)
    want_ids, want_off, want_counts = want_batch(encs(name, pat), texts)
    reset_counters()
    rc, ids, off, counts, nlong = simlib.encode_batch([sv], [t.encode() for t in texts])
    assert rc == 0
    assert np.array_equal(off, want_off)
    bad = [i for i in range(len(texts)) if not np.array_equal(ids[int(off[i]):int(off[i + 1])], want_ids[int(off[i]):int(off[i + 1])])]
    assert not bad, (name, pat, len(bad), texts[bad[0]][:80] if bad else None)
    assert np.array_equal(counts, want_counts)
    assert nlong > 0                                                    # pieces of more than 32 bytes went to K2b / K2c
    if name in ("long_tokens", "runs_to_255", "thresholds"):
        assert sv.max_token_len == 255
    if name == "over_2_20":
        assert sv.n_ranks > VS.K_LIST_MAX_RANK + 4000 and int(want_ids.max()) >= 1 << 20
        assert all(simlib.dbg_counter(i) == 0 for i in LIST_COUNTERS)   # bpe_list_kernel stays out above kListMaxRank ...
        assert simlib.dbg_counter(GLOBAL_LIST_PATH) > 0                 # ... so pieces of 257..4096 bytes take the global path
    if name == "thresholds":
        assert simlib.dbg_counter(GLOBAL_LIST_PATH) > 0                 # pieces of 4097 bytes
        assert any(simlib.dbg_counter(i) > 0 for i in LIST_COUNTERS)   # and of 257..4096 in bpe_list_kernel


@pytest.mark.parametrize("name", VS.SHAPES)
def test_oracle_matches_tiktoken(shapes, encs, name):
    """the oracle is the reference of the full-size GPU tests: it has to be right on these shapes too"""
    rf, texts = shapes[name]
    ov = oracle.OracleVocab(rf)
    data, offs = simlib.pack([t.encode() for t in texts])
    for pat in PATTERNS:
        ids, off, counts = oracle.encode_batch([ov], [pat], data, offs, nthreads=os.cpu_count())
        want_ids, want_off, want_counts = want_batch(encs(name, pat), texts)
        assert np.array_equal(off, want_off) and np.array_equal(ids, want_ids) and np.array_equal(counts, want_counts), (name, pat)


def eight_vocabularies(shapes):
    """eight rank orders of the union of the scattered-bytes and UTF-8 shapes, patterns 0..3 twice; texts of both shapes"""
    toks = list(dict.fromkeys(VS.tokens_of(shapes["utf8_random"][0]) + VS.tokens_of(shapes["scattered_bytes"][0])))
    rfs = []
    for v in range(8):
        order = list(toks)
        random.Random(100 + v).shuffle(order)
        rfs.append(VS.rank_file(order))
    texts = shapes["utf8_random"][1][:600] + shapes["scattered_bytes"][1][:600]
    random.Random(9).shuffle(texts)
    vid = np.array([(i * 5 + i // 7) % 8 for i in range(len(texts))], dtype=np.uint8)   # changes from prompt to prompt
    return rfs, [v % 4 for v in range(8)], texts, vid


def test_eight_vocabularies_in_one_batch(shapes):
    rfs, pats, texts, vid = eight_vocabularies(shapes)
    assert set(vid.tolist()) == set(range(8)) and all(vid[i] != vid[i + 1] for i in range(len(vid) - 1))
    encs = [tiktoken_encoding(rf, p, "v%d" % v) for v, (rf, p) in enumerate(zip(rfs, pats))]
    svs = [simlib.SimVocab(rf, 0, p, 0) for rf, p in zip(rfs, pats)]
    rc, ids, off, counts, nlong = simlib.encode_batch(svs, [t.encode() for t in texts], vocab_ids=vid)
    assert rc == 0 and nlong > 0
    for i, t in enumerate(texts):
        assert ids[int(off[i]):int(off[i + 1])].tolist() == encs[vid[i]].encode_ordinary(t), (i, int(vid[i]), t[:60])


def starts_by_tiktoken_rule(prompt: bytes, starts):
    """tiktoken's decode_with_offsets: characters before the token's first byte, one less when it starts inside a character"""
    out = []
    for s in starts:
        chars = sum(1 for c in prompt[:s] if not 0x80 <= c < 0xC0)
        out.append(max(0, chars - (1 if 0x80 <= prompt[s] < 0xC0 else 0)))
    return out


@pytest.mark.parametrize("pat", [0, 1])
@pytest.mark.parametrize("name", ["utf8_random", "scattered_bytes"])
def test_starts_truncate_chunk_and_decode(shapes, encs, name, pat):
    rf, texts = shapes[name]
    enc = encs(name, pat)
    sv = simlib.SimVocab(rf, 0, pat, 0)
    texts = texts[:500] + texts[-6:]
    prompts = [t.encode() for t in texts]
    rc, ids, starts, off, counts = simlib.encode_starts([sv], prompts)
    assert rc == 0
    inside = 0
    for i, (t, p) in enumerate(zip(texts, prompts)):
        a, b = int(off[i]), int(off[i + 1])
        want_ids = enc.encode_ordinary(t)
        assert ids[a:b].tolist() == want_ids
        text, want = enc.decode_with_offsets(want_ids)
        assert text == t
        assert starts_by_tiktoken_rule(p, starts[a:b].tolist()) == want, t[:60]
        inside += sum(1 for s in starts[a:b].tolist() if 0x80 <= p[s] < 0xC0)
    assert inside > 100                                                 # tokens that start inside a character
    # decode inverts encode
    rc, dec, doff = simlib.decode_batch([sv], ids, off)
    assert rc == 0 and bytes(dec) == b"".join(prompts) and np.array_equal(doff, simlib.pack(prompts)[1])
    # truncation and chunks against the contracts of include/cfbpe.h
    rng = random.Random(pat)
    budgets = np.array([rng.randint(0, max(int(c), 1) + 1) for c in counts], dtype=np.uint64)
    for mode in (HEAD, TAIL):
        rc, cut, kept, tcounts = simlib.truncate([sv], prompts, budgets, mode)
        assert rc == 0
        for i, p in enumerate(prompts):
            assert (int(cut[i]), int(kept[i]), int(tcounts[i])) == truncate_reference(enc, p, int(budgets[i]), mode)[:3], (i, mode)
    for n_tok, overlap in ((1, 0), (3, 1), (16, 5)):
        rc, spans, coffs, ccounts = simlib.chunk([sv], prompts, n_tok, overlap)
        assert rc == 0
        for i, p in enumerate(prompts):
            want, c = chunk_reference(enc, p, n_tok, overlap)
            got = [tuple(int(v) for v in s) for s in spans[int(coffs[i]):int(coffs[i + 1])]]
            assert (got, int(ccounts[i])) == (want, c), (i, n_tok, overlap)


def test_load_limits():
    """kMaxRank = 2^21 - 2 ranks load, and encode the top ids; one rank more, a rank of 2^21 - 1 and a token of 256 bytes are
    refused (EINVAL)"""
    sv = simlib.SimVocab(VS.big_rank_file(VS.K_MAX_RANK), 0, 0, 0)
    assert sv.n_ranks == VS.K_MAX_RANK
    last = VS.top_ranks(VS.K_MAX_RANK, 40)
    prompts = [t for _, t in last] + [b" ".join(t for _, t in last)]
    rc, ids, off, counts, _ = simlib.encode_batch([sv], prompts)
    assert rc == 0
    assert [int(ids[int(off[i])]) for i in range(40)] == [r for r, _ in last] and counts[:40].tolist() == [1] * 40
    ov = oracle.OracleVocab(VS.big_rank_file(VS.K_MAX_RANK))
    assert np.array_equal(ids[int(off[40]):int(off[41])], ov.encode(0, prompts[40]))
    del sv, ov
    with pytest.raises(ValueError, match="vocab size out of range"):
        simlib.SimVocab(VS.big_rank_file(VS.K_MAX_RANK + 1), 0, 0, 0)
    small = VS.tokens_of(VS.shape("runs_to_255")[0])
    with pytest.raises(ValueError, match="rank too large"):
        simlib.SimVocab(VS.rank_file(small) + b"YWJjZA== %d\n" % (VS.K_MAX_RANK + 1), 0, 0, 0)
    simlib.SimVocab(VS.rank_file(small + [b"b" * 255]), 0, 0, 0)
    with pytest.raises(ValueError, match="longer than 255"):
        simlib.SimVocab(VS.rank_file(small + [b"b" * 256]), 0, 0, 0)


@pytest.mark.parametrize("pat", PATTERNS)
def test_every_scalar_value_through_the_split(pat):
    """K1's UTF-8 decode and class lookup for every code point, in five contexts, against the oracle's split"""
    for k in range(len(fuzzgen.SCALAR_CONTEXTS)):
        strs = [s.encode() for s in fuzzgen.every_scalar_value(k)]
        rc, ends = simlib.split([pat], strs)
        assert rc == 0
        bad = [(p, e) for p, e in zip(strs, ends) if oracle.split(pat, p).tolist() != e]
        assert not bad, (k, len(bad), bad[:1])
