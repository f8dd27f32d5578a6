"""Single pieces of 20 001 bytes to 4 MiB through libcfbpe.so on the GPU, against the heap-ordered reference merge
(tests/long_piece_ref.py), and against the oracle up to 65 537 bytes.

Letter runs are one piece under every pattern, so a DNA or protein sequence, a Thai or CJK passage or a run of one letter
reaches bpe_long_kernel whole: past 65 535 parts it stays in batched rounds (kListMax), and K3, starts, truncate and chunk see
one piece with up to two million tokens.  Every case sits in one batch between ordinary prompts of every vocabulary, so
offsets, tiles and ranks after a huge piece are checked too.  Each entry point runs the whole batch once."""
import os
import random

import numpy as np
import pytest

import fuzzgen
import long_piece_ref as LR
import synth_vocab
import vocab_shapes as VS
from conftest import pack

pytestmark = pytest.mark.gpu

LOWER = "abcdefghijklmnopqrstuvwxyz"
PROTEIN = "ACDEFGHIKLMNPQRSTVWY"
ORACLE_MAX = 65537                    # the oracle's merge loop is quadratic: it checks the reference up to here
MAX_BATCH_BYTES = 16 << 20


@pytest.fixture(scope="module")
def slots(tekken_bytes):
    """slot -> (name, rank file, pattern, max ranks): the cl100k and Tekken stand-ins, a random-rank vocabulary (merged tokens
    may rank below their parts), 2^20 + 2^19 ranks (bpe_list_kernel stays out, ids >= 2^20) and the kListMax boundary tokens"""
    return [("cl100k", tekken_bytes, 0, 100256),
            ("tekken", tekken_bytes, 3, 130072),
            ("random-rank", synth_vocab.make_rank_file(21, alphabet=b"abcdefghijkl", n_extra=1500, max_len=7), 0, 0),
            ("over_2_20", VS.over_2_20()[0], 0, 0),
            ("boundary", LR.boundary_rank_file(), 0, 0)]


def huge_cases():
    """[(slot, kind, piece bytes)]"""
    rng = random.Random(2026)

    def rnd(alphabet, n):
        return "".join(rng.choice(alphabet) for _ in range(n)).encode()

    def period_with_foreign(n):
        s = bytearray(("abcab" * (n // 5 + 1))[:n].encode())
        for _ in range(8):
            s[rng.randrange(n)] = ord("z")
        return bytes(s)

    cases = []
    for slot in (0, 1):
        cases += [(slot, "random letters", rnd(LOWER, n)) for n in (20001, 65535, 65536, 65537, 100000)]
    cases += [(0, "ACGT", rnd("ACGT", 65536)), (1, "ACGT", rnd("ACGT", 1 << 20)),
              (0, "protein", rnd(PROTEIN, 100000)), (1, "protein", rnd(PROTEIN, 262144)),
              (0, "one letter", b"e" * 65537),
              (0, "period with foreign letters", period_with_foreign(1 << 20)),
              (1, "period with foreign letters", period_with_foreign(100000)),
              (0, "Thai letters", "".join(chr(rng.randint(0xE01, 0xE2E)) for _ in range(33334)).encode()),
              (1, "CJK letters", "".join(chr(rng.randint(0x4E00, 0x9FA5)) for _ in range(21846)).encode()),
              (2, "random letters", rnd("abcdefghijkl", 65537)), (2, "random letters", rnd("abcdefghijkl", 100000)),
              (3, "random letters", rnd("abcdefgh", 65536))]
    # not here: pieces that stay above kListMax parts for tens of thousands of merges of distinct ranks.  A batched round takes
    # one rank, so such a piece costs one warp-wide pass per merge: 100 000 random letters over the 2^20 + 2^19 ranks take
    # about 26 s on an H100 (700 W) while 65 536 take 2.4 s.
    cases += [(4, "boundary m=%d %s" % (m, "+".join(g)), LR.boundary_piece(m, g)) for m, g, _ in LR.BOUNDARY_CASES]
    rng.shuffle(cases)
    cases.insert(len(cases) // 2, (1, "one letter", b"a" * (4 << 20)))       # the 4 MiB prompt, in the middle of the batch
    return cases


@pytest.fixture(scope="module")
def batch(slots):
    """the prompts (every huge piece between ordinary prompts of every slot), their labels, vocabulary ids and the reference
    ids, offsets and token starts"""
    from oracle import oracle
    ranks = [LR.ranks_of(rf, n) for _, rf, _, n in slots]
    tok_len = []
    for r in ranks:
        ln = np.zeros(max(r.values()) + 1, dtype=np.int64)
        ln[list(r.values())] = [len(t) for t in r.keys()]
        tok_len.append(ln)
    ordinary = iter(fuzzgen.fuzz_strings(77, 4000, max_atoms=30))
    prompts, labels, vid = [], [], []

    def add_ordinary(k):
        for _ in range(k):
            slot = len(prompts) % len(slots)
            prompts.append(next(ordinary).encode())
            labels.append((slots[slot][0], "ordinary", len(prompts[-1])))
            vid.append(slot)
    for slot, kind, piece in huge_cases():
        add_ordinary(3)
        assert oracle.split(slots[slot][2], piece).tolist() == [len(piece)], (slot, kind)    # one piece
        prompts.append(piece)
        labels.append((slots[slot][0], kind, len(piece)))
        vid.append(slot)
    add_ordinary(3)
    prompts.append(b"DNA: " + prompts[-4][:70000].upper() + b".\n")      # a huge piece inside a prompt
    labels.append((slots[vid[-4]][0], "inside a prompt", len(prompts[-1])))
    vid.append(vid[-4])
    add_ordinary(3)
    assert sum(len(p) for p in prompts) <= MAX_BATCH_BYTES

    want = [np.asarray(LR.encode(ranks[v], slots[v][2], p), dtype=np.uint32) for v, p in zip(vid, prompts)]
    # the reference against the oracle wherever the oracle's quadratic merge loop finishes in time
    for slot, (_, rf, pat, n) in enumerate(slots):
        small = [i for i in range(len(prompts)) if vid[i] == slot and len(prompts[i]) <= ORACLE_MAX]
        data, offs = pack([prompts[i] for i in small])
        ids, off, _ = oracle.encode_batch([oracle.OracleVocab(rf, n)], [pat], data, offs, nthreads=os.cpu_count())
        for k, i in enumerate(small):
            assert LR.first_difference(want[i], ids[int(off[k]):int(off[k + 1])]) is None, labels[i]
    data, offs = pack(prompts)
    want_off = np.zeros(len(prompts) + 1, dtype=np.uint64)
    want_off[1:] = np.cumsum([len(w) for w in want])
    starts = []
    for v, w in zip(vid, want):
        ends = np.cumsum(tok_len[v][w.astype(np.int64)])
        starts.append(np.concatenate([[0], ends[:-1]]).astype(np.uint32) if len(w) else np.zeros(0, np.uint32))
    return dict(prompts=prompts, labels=labels, vid=np.asarray(vid, dtype=np.uint8), data=data, offs=offs, want_ids=np.concatenate(want),
                want_off=want_off, want_counts=np.diff(want_off).astype(np.uint32), want_starts=np.concatenate(starts))


def context(slots):
    from cfbpe import _native as N
    c = N.Context(0, MAX_BATCH_BYTES, 1 << 12)
    for slot, (_, rf, pat, n) in enumerate(slots):
        c.vocab_load(slot, rf, N.FORMAT_TIKTOKEN, pat, n)
    return c


@pytest.fixture(scope="module")
def ctx(slots):
    c = context(slots)
    yield c
    c.close()


def check_ids(b, ids, off, what):
    """every prompt's ids equal the reference; a failure names the entry point, the slot, the kind, the size and the first
    token that differs"""
    assert len(off) == len(b["want_off"])
    for i, label in enumerate(b["labels"]):
        diff = LR.first_difference(ids[int(off[i]):int(off[i + 1])], b["want_ids"][int(b["want_off"][i]):int(b["want_off"][i + 1])])
        assert diff is None, (what, i) + label + (diff,)
    assert np.array_equal(off, b["want_off"]), what


def check_per_prompt(b, got, want, what):
    bad = [i for i in range(len(b["labels"])) if not np.array_equal(got[i], want[i])]
    assert not bad, (what, len(bad), bad[0]) + b["labels"][bad[0]] + (got[bad[0]], want[bad[0]])


def test_host_encode(batch, ctx):
    ids, off, counts = ctx.encode_batch(batch["data"], batch["offs"], batch["vid"])
    check_ids(batch, ids, off, "encode_batch")
    assert np.array_equal(counts, batch["want_counts"])


def test_pipelined_host_encode(batch, slots, monkeypatch):
    """sub-batches of about 1 MiB: more than one before and after the 4 MiB prompt, huge pieces at their seams"""
    monkeypatch.setenv("CFBPE_PIPE_CHUNK_BYTES", str(1 << 20))
    monkeypatch.setenv("CFBPE_PIPE_MIN_BYTES", "1")
    c = context(slots)
    try:
        ids, off, counts = c.encode_batch(batch["data"], batch["offs"], batch["vid"])
    finally:
        c.close()
    check_ids(batch, ids, off, "pipelined encode_batch")
    assert np.array_equal(counts, batch["want_counts"])


def test_device_encode(batch, ctx):
    import torch
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    data, offs, n = batch["data"], batch["offs"], len(batch["labels"])
    d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).to(dev)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    d_vid = torch.from_numpy(batch["vid"]).to(dev)
    d_ids = torch.full((len(data) + 1,), -1, dtype=torch.int32, device=dev)
    d_out = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    d_cnt = torch.zeros(n, dtype=torch.int32, device=dev)
    ctx.encode_batch_device(n, d_bytes.data_ptr(), int(offs[-1]), d_offs.data_ptr(), d_vid.data_ptr(), d_ids.data_ptr(), d_ids.numel(),
                            d_out.data_ptr(), d_cnt.data_ptr(), stream, sync=False)
    ctx.device_status(stream)
    off = d_out.cpu().numpy().astype(np.uint64)
    check_ids(batch, d_ids[:int(off[-1])].cpu().numpy().view(np.uint32), off, "encode_batch_device")
    assert np.array_equal(d_cnt.cpu().numpy().astype(np.uint32), batch["want_counts"])


def test_count(batch, ctx):
    counts = ctx.count_batch(batch["data"], batch["offs"], batch["vid"])
    check_per_prompt(batch, counts, batch["want_counts"], "count_batch")


def test_starts(batch, ctx):
    """each token's byte offset within its prompt: the sums of the reference tokens' lengths"""
    ids, starts, off, counts = ctx.encode_batch_starts(batch["data"], batch["offs"], batch["vid"])
    check_ids(batch, ids, off, "encode_batch_starts")
    wo = batch["want_off"]
    check_per_prompt(batch, [starts[int(off[i]):int(off[i + 1])] for i in range(len(counts))],
                     [batch["want_starts"][int(wo[i]):int(wo[i + 1])] for i in range(len(counts))], "starts")


def budgets(batch):
    """half of every huge prompt's tokens (the cut falls inside the piece), any number for the ordinary prompts"""
    rng = random.Random(5)
    return np.array([c // 2 if kind != "ordinary" else rng.randint(0, int(c) + 1) for (_, kind, _), c in zip(batch["labels"], batch["want_counts"])],
                    dtype=np.uint32)


@pytest.mark.parametrize("mode", ["head", "tail"])
def test_truncate(batch, ctx, mode):
    from cfbpe import _native as N
    from cfbpe import plugin as P
    bud = budgets(batch)
    cut, kept, counts = ctx.truncate_batch(batch["data"], batch["offs"], bud, N.TRUNCATE_HEAD if mode == "head" else N.TRUNCATE_TAIL,
                                           batch["vid"])
    want_cut, want_kept = P.truncate_cuts(batch["data"], batch["offs"], batch["want_off"], batch["want_starts"], bud, mode == "tail")
    check_per_prompt(batch, cut, want_cut, "truncate %s: cut" % mode)
    check_per_prompt(batch, kept, want_kept, "truncate %s: kept" % mode)
    check_per_prompt(batch, counts, batch["want_counts"], "truncate %s: counts" % mode)
    huge = [i for i, (_, kind, _) in enumerate(batch["labels"]) if kind != "ordinary"]
    assert all(0 < int(cut[i]) < len(batch["prompts"][i]) for i in huge)      # every cut inside the huge piece


@pytest.mark.parametrize("n_tok,overlap", [(4096, 0), (30000, 10000)])
def test_chunk(batch, ctx, n_tok, overlap):
    from cfbpe import plugin as P
    spans, coffs, counts = ctx.chunk_batch(batch["data"], batch["offs"], n_tok, overlap, batch["vid"])
    want_spans, want_coffs = P.chunk_spans(batch["data"], batch["offs"], batch["want_off"], batch["want_starts"], n_tok, overlap)
    check_per_prompt(batch, [spans[int(coffs[i]):int(coffs[i + 1])] for i in range(len(counts))],
                     [want_spans[int(want_coffs[i]):int(want_coffs[i + 1])] for i in range(len(counts))], "chunk %d/%d" % (n_tok, overlap))
    check_per_prompt(batch, counts, batch["want_counts"], "chunk counts")


def test_random_letters_262144(slots):
    """a quarter-MiB random-letter piece: about 110 000 merges, all of them in one-warp batched rounds (the part count stays
    above kListMax to the end)"""
    from cfbpe import _native as N
    piece = "".join(random.Random(262144).choice(LOWER) for _ in range(262144)).encode()
    prompts = [b"before it", piece, b"after it"]
    c = N.Context(0, 1 << 20, 16)
    try:
        c.vocab_load(0, slots[0][1], N.FORMAT_TIKTOKEN, slots[0][2], slots[0][3])
        ids, off, counts = c.encode_batch(*pack(prompts))
    finally:
        c.close()
    ranks = LR.ranks_of(slots[0][1], slots[0][3])
    for i, p in enumerate(prompts):
        diff = LR.first_difference(ids[int(off[i]):int(off[i + 1])], LR.encode(ranks, 0, p))
        assert diff is None, (i, len(p), diff)
    assert int(counts[1]) > LR.K_LIST_MAX
