"""Text made of each benchmark slot's own vocabulary (cfbpe.workload.make_vocab_text) on the CPU SIMT emulator and the oracle,
against live tiktoken 0.12.0 built from the same ranks: every token alone and under the variants of TOKEN_VARIANTS (short-table,
long-table and whole-piece lookups of every token length, and misses of the same lengths), and letter-only words of each script
joined into single pieces of exactly 12 .. 20 000 bytes (merge trees of many rounds over real ranks, in bpe_list and in
bpe_long's global-memory path)."""
import os

import numpy as np
import pytest

import simlib
from conftest import COMBOS
from oracle import oracle
from test_vocab_shapes_sim import GLOBAL_LIST_PATH, LIST_COUNTERS, reset_counters, tiktoken_encoding

SLOTS = range(len(COMBOS))
# every slot encodes each token alone and under one other variant (the GPU test runs every variant on every slot)
SLOT_VARIANTS = {0: ("alone", "letter_changed"), 1: ("alone", "after_space"), 2: ("alone", "doubled"), 3: ("alone", "letter_after")}
LONG_PIECES = (9000, 20000)     # emulated slowly: one script a slot (the GPU test runs them in every script)


def rank_file(tekken_bytes, slot):
    return b"\n".join(tekken_bytes.splitlines()[:COMBOS[slot][1]])


def prompts_of(data, offs):
    return [bytes(data[int(offs[i]):int(offs[i + 1])]) for i in range(len(offs) - 1)]


def live_want(enc, texts):
    """live tiktoken's (ids uint32, offsets uint64 n+1, counts uint32) of a batch, one encode_ordinary call a text
    (encode_ordinary_batch spends most of its time handing hundreds of thousands of tiny texts to threads)"""
    want = [enc.encode_ordinary(t) for t in texts]
    off = np.zeros(len(texts) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(w) for w in want])
    ids = np.fromiter((i for w in want for i in w), dtype=np.uint32, count=int(off[-1]))
    return ids, off, np.diff(off).astype(np.uint32)


def mismatch(slot, data, offs, ids, off, want_ids, want_off):
    """None when two encodings of a batch agree, else what a person needs to cut the failure down: the slot (a number, or a
    word for a batch of several), the first prompt whose tokens differ, its first 80 bytes, and the first token of it that
    differs"""
    off, want_off = np.asarray(off, dtype=np.int64), np.asarray(want_off, dtype=np.int64)
    ids, want_ids = np.asarray(ids)[:off[-1]], np.asarray(want_ids)[:want_off[-1]]
    if np.array_equal(off, want_off) and np.array_equal(ids, want_ids):
        return None
    n = len(offs) - 1
    count_bad = np.nonzero(np.diff(off) != np.diff(want_off))[0]
    i = int(count_bad[0]) if len(count_bad) else n
    m = int(off[i])                                     # the prompts before i have the same counts, so the same offsets
    diff = np.nonzero(ids[:m] != want_ids[:m])[0]
    if len(diff):
        i = int(np.searchsorted(off, diff[0], side="right")) - 1
    got, want = ids[off[i]:off[i + 1]].tolist(), want_ids[want_off[i]:want_off[i + 1]].tolist()
    k = next((j for j, (a, b) in enumerate(zip(got, want)) if a != b), min(len(got), len(want)))
    return ("slot %s, prompt %d of %d: %r...: token %d is %s, want %s (%d tokens, want %d)"
            % (slot, i, n, bytes(data[int(offs[i]):int(offs[i]) + 80]), k, got[k] if k < len(got) else "missing",
               want[k] if k < len(want) else "none", len(got), len(want)))


@pytest.fixture(scope="module")
def slot_refs(tekken_bytes):
    """slot -> (SimVocab, OracleVocab, live tiktoken encoding) of the slot's ranks and pattern"""
    cache = {}

    def get(slot):
        if slot not in cache:
            pat, n = COMBOS[slot]
            cache[slot] = (simlib.SimVocab(tekken_bytes, 0, pat, n), oracle.OracleVocab(tekken_bytes, n),
                           tiktoken_encoding(rank_file(tekken_bytes, slot), pat, "slot%d" % slot))
        return cache[slot]
    return get


def check_emulator_and_oracle(slot, refs, data, offs):
    sv, ov, enc = refs
    prompts = prompts_of(data, offs)
    want_ids, want_off, want_counts = live_want(enc, [p.decode() for p in prompts])
    rc, ids, off, counts, nlong = simlib.encode_batch([sv], prompts)
    assert rc == 0
    msg = mismatch(slot, data, offs, ids, off, want_ids, want_off)
    assert msg is None, msg
    assert np.array_equal(counts, want_counts)
    oids, ooff, _ = oracle.encode_batch([ov], [COMBOS[slot][0]], data, offs, nthreads=os.cpu_count())
    msg = mismatch(slot, data, offs, oids, ooff, want_ids, want_off)
    assert msg is None, "oracle: " + msg
    return want_ids, nlong


@pytest.mark.parametrize("slot", SLOTS)
def test_every_token(tekken_bytes, slot_refs, slot):
    from cfbpe import workload as W
    data, offs = W.make_vocab_text(tekken_bytes, COMBOS[slot][1], slot, "tokens", variants=SLOT_VARIANTS[slot])
    want_ids, nlong = check_emulator_and_oracle(slot, slot_refs(slot), data, offs)
    assert nlong > 0                                                    # tokens of 33..78 bytes: the whole-piece lookup in K2b
    assert len(offs) - 1 > COMBOS[slot][1]                              # every valid token, and the variant


@pytest.mark.parametrize("slot", SLOTS)
def test_word_pieces(tekken_bytes, slot_refs, slot):
    from cfbpe import workload as W
    pat, n = COMBOS[slot]
    short = tuple(L for L in W.PIECE_LENGTHS if L not in LONG_PIECES)
    data, offs = W.make_vocab_text(tekken_bytes, n, slot, "pieces", lengths=short, per_length=lambda L: 1)
    d2, o2 = W.make_vocab_text(tekken_bytes, n, slot, "pieces", lengths=LONG_PIECES, per_length=lambda L: 1,
                               scripts=(W.PIECE_SCRIPTS[slot],))
    prompts = prompts_of(data, offs) + prompts_of(d2, o2)
    assert sorted(set(len(p) for p in prompts)) == sorted(W.PIECE_LENGTHS)
    assert all(oracle.split(pat, p).tolist() == [len(p)] for p in prompts)     # one piece each under the slot's pattern
    data, offs = simlib.pack(prompts)
    reset_counters()
    _, nlong = check_emulator_and_oracle(slot, slot_refs(slot), data, offs)
    assert nlong > 0
    assert any(simlib.dbg_counter(i) > 0 for i in LIST_COUNTERS)       # pieces of 257..4096 bytes in bpe_list_kernel
    assert simlib.dbg_counter(GLOBAL_LIST_PATH) > 0                     # and of more in bpe_long_kernel's global-memory path


def test_generator(tekken_bytes):
    """make_vocab_text is seeded, and each kind is what it says"""
    from cfbpe import workload as W
    n = COMBOS[0][1]
    toks = W.vocab_tokens(tekken_bytes, n)
    have = set(toks)
    valid = [t for t in toks if W._utf8(t) is not None]
    per = {}
    for v in W.TOKEN_VARIANTS:
        per[v] = prompts_of(*W.make_vocab_text(tekken_bytes, n, 5, "tokens", variants=(v,)))
    assert per["alone"] == valid and per["after_space"] == [b" " + t for t in valid] and per["doubled"] == [t + t for t in valid]
    assert all(p[:-1] == t and p[-1:].isalpha() for p, t in zip(per["letter_after"], valid))
    with_letter = [t for t in valid if any(chr(c).isalpha() and c < 128 for c in t)]
    assert len(per["letter_changed"]) > 0.99 * len(with_letter)        # (some short tokens are tokens with any letter changed)
    for p in per["letter_changed"]:
        assert p not in have and p.decode()
    a = W.make_vocab_text(tekken_bytes, n, 9, "diverse", n_prompts=3000)
    b = W.make_vocab_text(tekken_bytes, n, 9, "diverse", n_prompts=3000)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    lens = np.diff(a[1].astype(np.int64))
    assert len(lens) == 3000 and lens.min() >= 8 and lens.max() <= 4096
    prompts = prompts_of(*a)
    for p in prompts:
        p.decode()                                                      # cut at character boundaries
    assert sum(1 for p in prompts if p[:1].isalpha() and p[-1:].isalpha()) > 100   # and inside words, not only between them
    for distinct in (30, 1000):                                        # pools of short words still fill every prompt
        for seed in range(4):
            _, offs = W.make_vocab_text(tekken_bytes, n, seed, "diverse", n_prompts=200, distinct=distinct)
            lens = np.diff(offs.astype(np.int64))
            assert len(lens) == 200 and lens.min() >= 8 and lens.max() <= 4096
