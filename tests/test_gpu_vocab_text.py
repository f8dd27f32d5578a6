"""Text made of each benchmark slot's own vocabulary (cfbpe.workload.make_vocab_text) through libcfbpe.so on the H100.

  * every token of each slot under every variant, and letter-only word pieces of 12 .. 20 000 bytes in every script: the host
    call, the device entry point, and one batch whose vocabulary changes from prompt to prompt, against live tiktoken 0.12.0;
  * decode of every id of each slot, against the rank file;
  * full-size batches of words drawn uniformly from the whole vocabulary (65 536 prompts, ~134 MB; a quarter of that on slots
    1 and 2, and one batch of all four slots): the pipelined host call, the device entry point, count, byte starts and unit
    starts, against the multi-threaded oracle (test_vocab_shapes_sim.py checks the oracle against live tiktoken).  The
    profile counters show that each batch reached the merge kernels harder than the benchmark corpus does."""
import base64
import json
import os

import numpy as np
import pytest

from conftest import COMBOS
from oracle import oracle
from test_gpu_starts import check_starts
from test_vocab_shapes_sim import tiktoken_encoding
from test_vocab_text_sim import live_want, mismatch, rank_file

pytestmark = pytest.mark.gpu

SLOTS = range(len(COMBOS))
MAX_BYTES = 160 << 20
FULL_PROMPTS = {0: 65536, 1: 16384, 2: 16384, 3: 65536}
CONFIG3_MISSES_PER_MB = 4.0e6 / 134.0    # DESIGN.md, K2a/K2m: BASELINE.json config 3 has 4.0 M miss pieces in its 134 MB


@pytest.fixture(scope="module")
def ctx(tekken_bytes):
    """one context with the four benchmark slots loaded"""
    from cfbpe import _native as N
    c = N.Context(0, MAX_BYTES, 1 << 20)
    for slot, (pat, n) in enumerate(COMBOS):
        c.vocab_load(slot, tekken_bytes, N.FORMAT_TIKTOKEN, pat, n)
    yield c
    c.close()


@pytest.fixture(scope="module")
def encs(tekken_bytes):
    return [tiktoken_encoding(rank_file(tekken_bytes, slot), pat, "slot%d" % slot) for slot, (pat, _) in enumerate(COMBOS)]


@pytest.fixture(scope="module")
def tok_lens(tekken_bytes):
    return np.array([len(base64.b64decode(l.split()[0])) for l in tekken_bytes.splitlines()], dtype=np.int64)


def token_text(tekken_bytes, slot):
    """every token of the slot under every variant, then the word pieces of every script: (bytes, offsets)"""
    from cfbpe import workload as W
    t = W.make_vocab_text(tekken_bytes, COMBOS[slot][1], slot, "tokens")
    p = W.make_vocab_text(tekken_bytes, COMBOS[slot][1], slot, "pieces")
    offs = np.concatenate([t[1], p[1][1:] + t[1][-1]])
    return np.concatenate([t[0], p[0]]), offs


def texts_of(data, offs):
    return [bytes(data[int(offs[i]):int(offs[i + 1])]).decode() for i in range(len(offs) - 1)]


@pytest.fixture(scope="module")
def token_batches(tekken_bytes, encs):
    """slot -> (bytes, offsets, live tiktoken's ids, offsets, counts)"""
    cache = {}

    def get(slot):
        if slot not in cache:
            data, offs = token_text(tekken_bytes, slot)
            cache[slot] = (data, offs) + live_want(encs[slot], texts_of(data, offs))
        return cache[slot]
    return get


def check(slot, data, offs, got, want):
    ids, off, counts = got
    want_ids, want_off, want_counts = want
    msg = mismatch(slot, data, offs, ids, off, want_ids, want_off)
    assert msg is None, msg
    assert np.array_equal(np.asarray(counts, dtype=np.uint32), want_counts), slot


def device_encode(c, data, offs, vid, profile=False):
    """cfbpe_encode_batch_device on torch buffers: (ids, offsets, counts) as numpy, and the profile when asked for"""
    import torch
    dev = torch.device("cuda:0")
    n = len(offs) - 1
    d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).to(dev)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    d_vid = torch.from_numpy(np.ascontiguousarray(vid)).to(dev)
    d_ids = torch.full((len(data) + 1,), -1, dtype=torch.int32, device=dev)
    d_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    d_cnt = torch.zeros(n, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    if profile:
        c.profile_enable(True)
    try:
        nt = c.encode_batch_device(n, d_bytes.data_ptr(), int(offs[-1]), d_offs.data_ptr(), d_vid.data_ptr(), d_ids.data_ptr(),
                                   d_ids.numel(), d_off.data_ptr(), d_cnt.data_ptr(), stream, sync=True)
        prof = c.profile_read() if profile else None
    finally:
        if profile:
            c.profile_enable(False)
    off = d_off.cpu().numpy().astype(np.uint64)
    assert nt == int(off[-1])
    return (d_ids[:nt].cpu().numpy().view(np.uint32), off, d_cnt.cpu().numpy().view(np.uint32)), prof


@pytest.mark.parametrize("slot", SLOTS)
def test_every_token_and_word_pieces_host_call(ctx, token_batches, slot):
    data, offs, *want = token_batches(slot)
    check(slot, data, offs, ctx.encode_batch(data, offs, np.full(len(offs) - 1, slot, np.uint8)), want)


@pytest.mark.parametrize("slot", SLOTS)
def test_every_token_and_word_pieces_device_entry_point(ctx, token_batches, slot):
    data, offs, *want = token_batches(slot)
    got, _ = device_encode(ctx, data, offs, np.full(len(offs) - 1, slot, np.uint8))
    check(slot, data, offs, got, want)


def test_every_token_and_word_pieces_four_slots_in_one_batch(ctx, token_batches, encs):
    """slot 1's batch (its 150 000 ranks hold every other slot's) with the vocabulary cycling 0, 1, 2, 3 from prompt to prompt"""
    data, offs = token_batches(1)[:2]
    n = len(offs) - 1
    vid = (np.arange(n) % 4).astype(np.uint8)
    texts = texts_of(data, offs)
    want = [None] * n
    for slot in SLOTS:
        for i in range(slot, n, 4):
            want[i] = encs[slot].encode_ordinary(texts[i])
    want_off = np.zeros(n + 1, dtype=np.uint64)
    want_off[1:] = np.cumsum([len(w) for w in want])
    want_ids = np.fromiter((i for w in want for i in w), dtype=np.uint32, count=int(want_off[-1]))
    want = (want_ids, want_off, np.diff(want_off).astype(np.uint32))
    check("0..3 cycling", data, offs, ctx.encode_batch(data, offs, vid), want)
    check("0..3 cycling", data, offs, device_encode(ctx, data, offs, vid)[0], want)


@pytest.mark.parametrize("slot", SLOTS)
def test_decode_every_id(ctx, tekken_bytes, slot):
    from cfbpe import workload as W
    toks = W.vocab_tokens(tekken_bytes, COMBOS[slot][1])
    n = len(toks)
    dec, doff = ctx.decode_batch(np.arange(n, dtype=np.uint32), np.arange(n + 1, dtype=np.uint64), np.full(n, slot, np.uint8))
    assert bytes(dec) == b"".join(toks)
    assert np.array_equal(np.diff(doff.astype(np.int64)), [len(t) for t in toks])


def full_size(tekken_bytes, slot, n_prompts, vid=None):
    """a diverse batch from the slot's vocabulary and the oracle's encoding of it (vid: each prompt's slot; None: `slot`)"""
    from cfbpe import workload as W
    data, offs = W.make_vocab_text(tekken_bytes, COMBOS[slot][1], 100 + slot, "diverse", n_prompts=n_prompts)
    vocabs = [oracle.OracleVocab(tekken_bytes, n) for _, n in COMBOS]
    if vid is None:
        vid = np.full(n_prompts, slot, np.uint8)
    want = oracle.encode_batch(vocabs, [pat for pat, _ in COMBOS], data, offs, vid, nthreads=os.cpu_count())
    return data, offs, vid, want


def check_reach(name, prof):
    """print the profile counters of a full-size batch and check that it reached what it is for"""
    keys = ("n_bytes", "n_tokens", "n_miss_pieces", "n_extra_tokens", "n_long_pieces", "n_list_pieces", "n_list_parts")
    print(json.dumps({"batch": name, **{k: int(prof[k]) for k in keys},
                      "miss_pieces_per_MB": round(prof["n_miss_pieces"] / (prof["n_bytes"] / 1e6))}), flush=True)
    assert prof["n_miss_pieces"] / (prof["n_bytes"] / 1e6) > CONFIG3_MISSES_PER_MB
    assert prof["n_list_pieces"] > 0
    assert prof["n_extra_tokens"] > 0


@pytest.mark.parametrize("slot", SLOTS)
def test_full_size_diverse_batch(ctx, tekken_bytes, tok_lens, slot):
    from cfbpe import _native as N
    from cfbpe import plugin as P
    n = FULL_PROMPTS[slot]
    data, offs, vid, want = full_size(tekken_bytes, slot, n)
    if n == 65536:
        assert int(offs[-1]) > 130e6
    check(slot, data, offs, ctx.encode_batch(data, offs, vid), want)       # pipelined: above 4 MB, profiling off
    got, prof = device_encode(ctx, data, offs, vid, profile=True)
    check(slot, data, offs, got, want)
    check_reach("slot %d" % slot, prof)
    assert np.array_equal(ctx.count_batch(data, offs, vid), want[2])
    ids, starts, off, counts = ctx.encode_batch_starts(data, offs, vid)
    check(slot, data, offs, (ids, off, counts), want)
    check_starts(ids, starts, off, counts, offs, tok_lens)
    for unit, name in ((N.UNIT_CODEPOINT, "codepoint"), (N.UNIT_UTF16, "utf16")):
        want_starts, want_lens = P.unit_starts(data, offs, off, starts, name)
        uids, ustarts, uoff, ucounts, ulens = ctx.encode_batch_char_starts(data, offs, unit, vid)
        check(slot, data, offs, (uids, uoff, ucounts), want)
        assert np.array_equal(ustarts, want_starts), (slot, name)
        assert np.array_equal(ulens, want_lens), (slot, name)


def test_full_size_four_slots_in_one_batch(ctx, tekken_bytes):
    """words of slot 1's 150 000 ranks, the vocabulary cycling 0, 1, 2, 3 from prompt to prompt"""
    n = 65536
    data, offs, vid, want = full_size(tekken_bytes, 1, n, (np.arange(n) % 4).astype(np.uint8))
    check("0..3 cycling", data, offs, ctx.encode_batch(data, offs, vid), want)
    got, prof = device_encode(ctx, data, offs, vid, profile=True)
    check("0..3 cycling", data, offs, got, want)
    check_reach("four slots", prof)
    assert np.array_equal(ctx.count_batch(data, offs, vid), want[2])
