"""Rank files shaped like real ones (tests/vocab_shapes.py) through libcfbpe.so on the GPU, against live tiktoken 0.12.0 (and
the oracle, multi-threaded, for the 32 MB batch): one-shot host calls, the pipelined host path, the device entry point, eight
vocabularies in one batch, starts / truncate / chunk / decode, the load limits, and every Unicode scalar value."""
import os
import random

import numpy as np
import pytest

import fuzzgen
import vocab_shapes as VS
from conftest import COMBOS, pack
from test_chunk_sim import reference as chunk_reference
from test_truncate_sim import HEAD, TAIL, reference as truncate_reference
from test_vocab_shapes_sim import PATTERNS, eight_vocabularies, starts_by_tiktoken_rule, tiktoken_encoding, want_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def shapes():
    return {name: VS.shape(name) for name in VS.SHAPES}


@pytest.fixture(scope="module")
def wants(shapes):
    """(shape, pattern) -> tiktoken's (ids, offsets, counts) of the shape's texts"""
    return {(name, pat): want_batch(tiktoken_encoding(shapes[name][0], pat), shapes[name][1]) for name in VS.SHAPES for pat in PATTERNS}


def context(rf, max_bytes=16 << 20, max_prompts=1 << 16):
    """a context with the rank file in slots 0..3 under patterns 0..3"""
    from cfbpe import _native as N
    c = N.Context(0, max_bytes, max_prompts)
    for pat in PATTERNS:
        c.vocab_load(pat, rf, N.FORMAT_TIKTOKEN, pat, 0)
    return c


def check_host(c, texts, wants, name):
    data, offs = pack([t.encode() for t in texts])
    for pat in PATTERNS:
        ids, off, counts = c.encode_batch(data, offs, np.full(len(texts), pat, np.uint8))
        want_ids, want_off, want_counts = wants[(name, pat)]
        assert np.array_equal(off, want_off), (name, pat)
        assert np.array_equal(ids, want_ids), (name, pat)
        assert np.array_equal(counts, want_counts), (name, pat)


@pytest.mark.parametrize("name", VS.SHAPES)
def test_one_shot_host_calls(shapes, wants, name):
    rf, texts = shapes[name]
    c = context(rf)
    check_host(c, texts, wants, name)
    info = c.vocab_info(0)
    assert info["n_ranks"] == len(VS.tokens_of(rf))
    c.close()


@pytest.mark.parametrize("name", VS.SHAPES)
def test_pipelined_host_path(shapes, wants, name, monkeypatch):
    """tiny sub-batches: seams everywhere, long pieces across them"""
    monkeypatch.setenv("CFBPE_PIPE_CHUNK_BYTES", "20000")
    monkeypatch.setenv("CFBPE_PIPE_MIN_BYTES", "1")
    rf, texts = shapes[name]
    c = context(rf, 1 << 20)
    check_host(c, texts, wants, name)
    c.close()


@pytest.mark.parametrize("name", VS.SHAPES)
def test_device_entry_point(shapes, wants, name):
    import torch
    rf, texts = shapes[name]
    c = context(rf)
    data, offs = pack([t.encode() for t in texts])
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    n = len(texts)
    d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).to(dev)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    for pat in PATTERNS:
        d_vid = torch.full((n,), pat, dtype=torch.uint8, device=dev)
        d_ids = torch.full((len(data) + 1,), -1, dtype=torch.int32, device=dev)
        d_out = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        d_cnt = torch.zeros(n, dtype=torch.int32, device=dev)
        nt = c.encode_batch_device(n, d_bytes.data_ptr(), int(offs[-1]), d_offs.data_ptr(), d_vid.data_ptr(), d_ids.data_ptr(),
                                   d_ids.numel(), d_out.data_ptr(), d_cnt.data_ptr(), stream, sync=True)
        want_ids, want_off, want_counts = wants[(name, pat)]
        assert nt == len(want_ids)
        assert np.array_equal(d_out.cpu().numpy().astype(np.uint64), want_off), (name, pat)
        assert np.array_equal(d_ids[:nt].cpu().numpy().view(np.uint32), want_ids), (name, pat)
        assert np.array_equal(d_cnt.cpu().numpy().astype(np.uint32), want_counts), (name, pat)
    c.close()


def test_eight_vocabularies_in_one_batch(shapes):
    from cfbpe import _native as N
    rfs, pats, texts, vid = eight_vocabularies(shapes)
    c = N.Context(0, 16 << 20, 1 << 16)
    for v, (rf, p) in enumerate(zip(rfs, pats)):
        c.vocab_load(v, rf, N.FORMAT_TIKTOKEN, p, 0)
    encs = [tiktoken_encoding(rf, p) for rf, p in zip(rfs, pats)]
    data, offs = pack([t.encode() for t in texts])
    ids, off, counts = c.encode_batch(data, offs, vid)
    for i, t in enumerate(texts):
        assert ids[int(off[i]):int(off[i + 1])].tolist() == encs[vid[i]].encode_ordinary(t), (i, int(vid[i]), t[:60])
    c.close()


@pytest.mark.parametrize("name", ["utf8_random", "scattered_bytes"])
def test_starts_truncate_chunk_and_decode(shapes, name):
    rf, texts = shapes[name]
    c = context(rf)
    for pat in (0, 1):
        enc = tiktoken_encoding(rf, pat)
        prompts = [t.encode() for t in texts]
        data, offs = pack(prompts)
        vid = np.full(len(prompts), pat, np.uint8)
        ids, starts, off, counts = c.encode_batch_starts(data, offs, vid)
        for i, (t, p) in enumerate(zip(texts, prompts)):
            a, b = int(off[i]), int(off[i + 1])
            want_ids = enc.encode_ordinary(t)
            assert ids[a:b].tolist() == want_ids
            assert starts_by_tiktoken_rule(p, starts[a:b].tolist()) == enc.decode_with_offsets(want_ids)[1], t[:60]
        dec, doff = c.decode_batch(ids, off, vid)
        assert bytes(dec) == bytes(data) and np.array_equal(doff, offs)
        rng = random.Random(pat)
        budgets = np.array([rng.randint(0, int(k) + 1) for k in counts], dtype=np.uint32)
        for mode in (HEAD, TAIL):
            cut, kept, tcounts = c.truncate_batch(data, offs, budgets, mode, vid)
            for i, p in enumerate(prompts):
                assert (int(cut[i]), int(kept[i]), int(tcounts[i])) == truncate_reference(enc, p, int(budgets[i]), mode)[:3], (i, mode)
        for n_tok, overlap in ((1, 0), (3, 1), (16, 5)):
            spans, coffs, ccounts = c.chunk_batch(data, offs, n_tok, overlap, vid)
            for i, p in enumerate(prompts):
                want, k = chunk_reference(enc, p, n_tok, overlap)
                got = [tuple(int(v) for v in s) for s in spans[int(coffs[i]):int(coffs[i + 1])]]
                assert (got, int(ccounts[i])) == (want, k), (i, n_tok, overlap)
    c.close()


def test_32mb_of_big_pieces_over_2_20_ranks():
    """more than 32 MB of letter words of 257..4096 bytes on the 2^20 + 2^19-rank vocabulary: every piece in bpe_long_kernel's
    global-memory path at once (many warps), against the oracle"""
    from cfbpe import _native as N
    from oracle import oracle
    rf, _ = VS.over_2_20()
    rng = np.random.default_rng(20)
    lens = rng.integers(257, 4097, size=16000)
    data = np.frombuffer(b"abcdefgh", np.uint8)[rng.integers(0, 8, size=int(lens.sum()))].copy()
    offs = np.zeros(len(lens) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    assert int(offs[-1]) >= 32 << 20
    want_ids, want_off, want_counts = oracle.encode_batch([oracle.OracleVocab(rf)], [0], data, offs, nthreads=os.cpu_count())
    assert int(want_ids.max()) >= 1 << 20
    c = N.Context(0, 40 << 20, 1 << 16)
    c.vocab_load(0, rf, N.FORMAT_TIKTOKEN, 0, 0)
    ids, off, counts = c.encode_batch(data, offs)
    assert np.array_equal(off, want_off)
    assert np.array_equal(ids, want_ids)
    assert np.array_equal(counts, want_counts)
    c.close()


def test_load_limits():
    from cfbpe import _native as N
    c = N.Context(0, 1 << 20, 1024)
    c.vocab_load(0, VS.big_rank_file(VS.K_MAX_RANK), N.FORMAT_TIKTOKEN, 0, 0)
    assert c.vocab_info(0)["n_ranks"] == VS.K_MAX_RANK
    last = VS.top_ranks(VS.K_MAX_RANK, 40)
    ids, off, counts = c.encode_batch(*pack([t for _, t in last]))
    assert ids.tolist() == [r for r, _ in last]
    small = VS.tokens_of(VS.shape("runs_to_255")[0])
    for bad in (VS.big_rank_file(VS.K_MAX_RANK + 1), VS.rank_file(small + [b"b" * 256])):
        with pytest.raises(N.NativeError) as ei:
            c.vocab_load(1, bad, N.FORMAT_TIKTOKEN, 0, 0)
        assert ei.value.code == N.EINVAL
    c.close()


def test_every_scalar_value_through_the_tekken_slots(tekken_bytes):
    """K1's UTF-8 decode and class lookup on the device for every code point, in five contexts, under each slot's pattern"""
    from cfbpe import _native as N
    c = N.Context(0, 64 << 20, 1 << 18)
    for slot, (pat, n) in enumerate(COMBOS):
        c.vocab_load(slot, tekken_bytes, N.FORMAT_TIKTOKEN, pat, n)
    for slot, (pat, n) in enumerate(COMBOS):
        enc = tiktoken_encoding(b"\n".join(tekken_bytes.splitlines()[:n]), pat)
        for k in range(len(fuzzgen.SCALAR_CONTEXTS)):
            texts = fuzzgen.every_scalar_value(k)
            want_ids, want_off, want_counts = want_batch(enc, texts)
            data, offs = pack([t.encode() for t in texts])
            ids, off, counts = c.encode_batch(data, offs, np.full(len(texts), slot, np.uint8))
            assert np.array_equal(off, want_off), (pat, k)
            assert np.array_equal(ids, want_ids), (pat, k)
    c.close()
