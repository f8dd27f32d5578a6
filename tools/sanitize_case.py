#!/usr/bin/env python3
"""A small but path-complete encode workload for `compute-sanitizer --tool memcheck|racecheck|synccheck|initcheck`
(SURVEY.md section 5).  Fuzz prompts, long and periodic pieces, cased runs that take the fix-up path, two vocabularies in one
batch, the one-shot and the pipelined host path, count-only and decode -- each result checked against the oracle, so that a run
under the sanitizer is also a parity run.  Usage (GPU box):
    compute-sanitizer --tool memcheck  --log-file sanitizer_memcheck.log  python tools/sanitize_case.py
    compute-sanitizer --tool racecheck --log-file sanitizer_racecheck.log python tools/sanitize_case.py small
"""
import os
import sys

os.environ.setdefault("CFBPE_ALLOW_STAND_IN", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "cyberfabric-core_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import random

import numpy as np

import fuzzgen
from cfbpe import _native as N
from oracle import oracle

small = len(sys.argv) > 1 and sys.argv[1] == "small"
tekken = open(os.path.join(ROOT, "vocabs", "tekken_240911.tiktoken"), "rb").read()
ovs = [oracle.OracleVocab(tekken, 100256), oracle.OracleVocab(tekken, 130072)]
pats = [0, 3]

rng = random.Random(7)
prompts = [s.encode() for s in fuzzgen.fuzz_strings(99, 150 if small else 1200, max_atoms=40)]
prompts += [s.encode() for s in fuzzgen.long_runs(3)[: (20 if small else 200)]]
letters = "abcdefghijklmnopqrstuvwxyzABCDEFGH"
for n in ([40, 300, 1500] if small else [33, 64, 257, 600, 1500, 4096, 9000]):
    prompts.append("".join(rng.choice(letters) for _ in range(n)).encode())
    prompts.append(("xyz" * n)[:n].encode())
    prompts.append(("中文A字" * n)[:n].encode())
    prompts.append((" " * n + "x").encode())
    prompts.append("".join(rng.choice("0123456789") for _ in range(n)).encode())
prompts += [b"", b"a", b""]
offs = np.zeros(len(prompts) + 1, dtype=np.uint64)
offs[1:] = np.cumsum([len(p) for p in prompts])
data = np.frombuffer(b"".join(prompts), dtype=np.uint8).copy()
vid = (np.arange(len(prompts)) % 2).astype(np.uint8)
want_ids, want_off, want_counts = oracle.encode_batch(ovs, pats, data, offs, vocab_ids=vid, nthreads=os.cpu_count())

for pipelined in (False, True):
    if pipelined:
        os.environ["CFBPE_PIPE_CHUNK_BYTES"] = "30000"
        os.environ["CFBPE_PIPE_MIN_BYTES"] = "1"
    c = N.Context(0, 8 << 20, 1 << 14)
    c.vocab_load(0, tekken, N.FORMAT_TIKTOKEN, 0, 100256)
    c.vocab_load(1, tekken, N.FORMAT_TIKTOKEN, 3, 130072)
    ids, off, counts = c.encode_batch(data, offs, vid)
    assert np.array_equal(off, want_off) and np.array_equal(ids, want_ids) and np.array_equal(counts, want_counts)
    assert np.array_equal(c.count_batch(data, offs, vid), want_counts)
    dec, doff = c.decode_batch(ids, off, vid)
    assert np.array_equal(doff, offs) and bytes(dec) == bytes(data)
    c.close()
    print("sanitize_case: %s host path ok (%d prompts, %d bytes, %d ids)" % ("pipelined" if pipelined else "one-shot", len(prompts), len(data), len(ids)))
