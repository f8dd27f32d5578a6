"""Single pieces at bpe_long_kernel's part limit (kListMax = 65 535) on the CPU SIMT emulator, and the heap-ordered reference
merge (tests/long_piece_ref.py) that checks pieces of MiB size on the GPU, pinned to the oracle and to live tiktoken.

The boundary pieces are cheap to merge (a handful of merges in a run of filler), so the emulator runs them at full size; the
path counter shows whether bpe_long_kernel's list rounds ran on each, which the ids alone cannot show."""
import base64
import random

import pytest

import long_piece_ref as LR
import simlib
import synth_vocab
from conftest import COMBOS
from oracle import oracle
from oracle import patterns as PT

GLOBAL_LIST_PATH = 5            # bpe_long_kernel's list rounds on a piece in global memory


def random_pieces(rng, alphabet, sizes):
    return ["".join(rng.choice(alphabet) for _ in range(n)).encode() for n in sizes]


def test_heap_reference_matches_oracle_and_tiktoken(tekken_bytes):
    """merge() equals the oracle's merge loop on random-rank vocabularies (merged tokens may rank below their parts) and on
    the Tekken stand-in slots, and live tiktoken on the stand-in slots, on pieces of up to 20 000 bytes"""
    rng = random.Random(11)
    for seed in range(6):
        alphabet = b"abcdefgh"[:3 + seed]
        rf = synth_vocab.make_rank_file(seed, alphabet=alphabet, n_extra=40 + 60 * seed, max_len=6)
        ranks, ov = LR.ranks_of(rf), oracle.OracleVocab(rf)
        sizes = [1, 2, 3, 7, 33, 100, 257, 1000, 4097, 8000]
        pieces = random_pieces(rng, alphabet.decode(), sizes)
        pieces += [(alphabet[:k] * 4000)[:n] for k in (1, 2, 3) for n in (5, 64, 2500, 8000)]
        for p in pieces:
            assert LR.merge(ranks, p) == ov.encode(0, p).tolist(), (seed, len(p), p[:40])
    tiktoken = pytest.importorskip("tiktoken")
    lines = tekken_bytes.splitlines()
    for pat, n in COMBOS:
        ranks, ov = LR.ranks_of(tekken_bytes, n), oracle.OracleVocab(tekken_bytes, n)
        assert ranks == {t: i for i, t in enumerate(LR.ranks_of(b"\n".join(lines[:n])))}    # rank = line number
        enc = tiktoken.Encoding("huge%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks, special_tokens={})
        pieces = random_pieces(rng, "abcdefghijklmnopqrstuvwxyz", (1, 40, 4097, 20000))
        pieces += random_pieces(rng, "ACGT", (8000, 20000)) + [b"a" * 20000, ("abcab" * 4000).encode()]
        pieces += ["".join(chr(rng.randint(0x4E00, 0x9FA5)) for _ in range(3000)).encode(), ("ก" * 2000).encode()]
        for p in pieces:
            want = enc.encode_ordinary(p.decode())
            assert oracle.split(pat, p).tolist() == [len(p)], (pat, p[:20])    # one piece
            assert LR.merge(ranks, p) == want, (pat, len(p), p[:40])
            if len(p) <= 8000:
                assert ov.encode(pat, p).tolist() == want, (pat, len(p))


def test_heap_reference_takes_ties_leftmost():
    """equal ranks: the leftmost pair first, also when an earlier merge creates the tie"""
    toks = [bytes([b]) for b in range(256)] + [b"ab", b"ba", b"abab", b"bab"]
    ranks = {t: i for i, t in enumerate(toks)}
    ov = oracle.OracleVocab(b"".join(base64.b64encode(t) + b" %d\n" % i for i, t in enumerate(toks)))
    for p in (b"ab" * 9, b"b" + b"ab" * 9, b"aba", b"bab", b"babab", b"ab" * 9 + b"a"):
        assert LR.merge(ranks, p) == ov.encode(0, p).tolist(), p


@pytest.fixture(scope="module")
def boundary():
    rf = LR.boundary_rank_file()
    return simlib.SimVocab(rf, 0, 0, 0), LR.ranks_of(rf), oracle.OracleVocab(rf)


@pytest.mark.parametrize("m,merges,list_rounds", LR.BOUNDARY_CASES,
                         ids=["m%d-%s" % (m, "+".join(g)) for m, g, _ in LR.BOUNDARY_CASES])
def test_pieces_at_the_list_limit(boundary, m, merges, list_rounds):
    """a piece with m parts after its first batched round, between two ordinary prompts: ids against the heap reference and
    the oracle, and the list rounds ran exactly when the parts left with a pair are at most kListMax"""
    sv, ranks, ov = boundary
    piece = LR.boundary_piece(m, merges)
    want = LR.merge(ranks, piece)
    assert len(want) == m - len(merges)
    assert want == ov.encode(0, piece).tolist()
    prompts = [b"ab cd xy zz", piece, b"xyab qq"]
    for i in range(8):
        simlib.dbg_counter(i, reset=True)
    rc, ids, off, counts, nlong = simlib.encode_batch([sv], prompts)
    assert rc == 0
    diff = LR.first_difference(ids[int(off[1]):int(off[2])], want)
    assert diff is None, (m, merges, diff)
    for i in (0, 2):
        assert ids[int(off[i]):int(off[i + 1])].tolist() == LR.encode(ranks, 0, prompts[i]), i
    assert counts.tolist() == [int(off[i + 1] - off[i]) for i in range(3)]
    assert simlib.dbg_counter(GLOBAL_LIST_PATH) == (1 if list_rounds else 0), (m, merges)
