"""Special-token encode at its table's limits and on prompts dense with matches (csrc/specials.cuh, specials.h) on the CPU
SIMT emulator, against one plain reference (special_sets.reference) and, where its leftmost-longest rule cannot differ from
tiktoken's leftmost-first alternation, against live tiktoken 0.12.0 `Encoding.encode`: the sets of special_sets.py on the
cl100k and Tekken slots under three policies, eight vocabularies with their own sets in one batch, the max_prompts boundary,
counts only, ENOSPC, decode of every id of a full table, and disallowed specials at index 2048 and above."""
import base64
import random

import numpy as np
import pytest

import special_sets as SS
from conftest import COMBOS

import simlib as S

tiktoken = pytest.importorskip("tiktoken")

SLOTS = (COMBOS[0], COMBOS[3])          # the cl100k (pattern 0) and Tekken (pattern 3) slots


def walk_witness(kept_all, offsets):
    """what special_walk met in a call: (most kept matches in one 32-bit candidate word of the batch, most kept matches of one
    prompt in one 1 KiB trip, most trips of one prompt that hold a kept match, words that hold the kept matches of two prompts)"""
    words, trips, n_trips, owners = {}, {}, 0, {}
    for i, kept in enumerate(kept_all):
        lo = int(offsets[i])
        ts = set()
        for a, _, _ in kept:
            w = (lo + a) >> 5
            words[w] = words.get(w, 0) + 1
            owners.setdefault(w, set()).add(i)
            t = (w - (lo >> 5)) >> 5
            trips[(i, t)] = trips.get((i, t), 0) + 1
            ts.add(t)
        n_trips = max(n_trips, len(ts))
    shared = sum(len(o) > 1 for o in owners.values())
    return max(words.values(), default=0), max(trips.values(), default=0), n_trips, shared


def run(vocabs, specials, modes, prompts, vocab_ids, tables, encoders, **kw):
    """one emulator call against the reference; EBADMSG must name the reference's prompt and index.  Returns (reference,
    n_stretches, offsets)"""
    want = SS.reference(tables, modes, prompts, vocab_ids, encoders)
    rc, got, counts, bad, nst, off = S.encode_batch_special(vocabs, specials, prompts, modes=modes, vocab_ids=vocab_ids, **kw)
    if want[0] == "bad":
        assert rc == S.EBADMSG and bad == want[1:], (rc, bad, want[1:])
        return want, None, None
    assert rc == 0
    n_kept = sum(len(k) for k in want[2])
    assert nst == len(prompts) + 2 * n_kept          # the stretch path ran iff some match was kept
    for i, (g, c, w) in enumerate(zip(got, counts, want[1])):
        assert g == w, (i, prompts[i][:300])
        assert c == len(w)
    return want, nst, off


def tiktoken_pin(ranks_of_pat, pat, specials, modes, texts):
    """assert the reference equals live tiktoken Encoding.encode on every text that has no position holding two specials"""
    from oracle import patterns as PT
    enc = tiktoken.Encoding("pin%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks_of_pat, special_tokens=specials)
    T = SS.Table(specials)
    names = T.names
    allowed = set() if modes is None else {t for t, m in zip(names, modes) if m == SS.ALLOW}
    disallowed = set(names) if modes is None else {t for t, m in zip(names, modes) if m == SS.DISALLOW}
    f = SS.ordinary(enc)
    n = 0
    for t in texts:
        p = t.encode()
        bad, kept, amb = SS.cut(T, modes, p)
        if amb:
            continue
        n += 1
        if bad is not None:
            with pytest.raises(ValueError):
                enc.encode(t, allowed_special=allowed, disallowed_special=disallowed)
            continue
        want, at = [], 0
        for a, b, k in kept:
            want += f(p[at:a]) + [T.ids[k]]
            at = b
        assert enc.encode(t, allowed_special=allowed, disallowed_special=disallowed) == want + f(p[at:]), t
    return n


# ---- fixtures -----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sim_vocabs(tekken_bytes):
    return {pat: S.SimVocab(tekken_bytes, 0, pat, n) for pat, n in COMBOS}


@pytest.fixture(scope="module")
def ranks(tekken_bytes):
    lines = tekken_bytes.splitlines()
    return {pat: {base64.b64decode(l.split()[0]): i for i, l in enumerate(lines[:n])} for pat, n in COMBOS}


@pytest.fixture(scope="module")
def encoders(ranks):
    """pattern id -> encode_ordinary (cached) of a tiktoken Encoding without special tokens"""
    from oracle import patterns as PT
    return {pat: SS.ordinary(tiktoken.Encoding("plain%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks[pat], special_tokens={}))
            for pat, _ in COMBOS}


@pytest.fixture(scope="module")
def sets():
    return {name: SS.special_set(name) for name in SS.SETS}


@pytest.fixture(scope="module")
def tables(sets):
    return {name: (SS.Table(sets[name][0]), S.Specials(sets[name][0])) for name in SS.SETS}


# ---- the sets one at a time ---------------------------------------------------------------------------------------------
def test_sets_are_what_they_claim(sets):
    sp, _ = sets["all_lengths"]
    assert sorted(len(t.encode()) for t in sp) == list(range(1, 65)) and SS.is_prefix_free(sp)
    assert {len(c.encode()) for t in sp for c in t} == {1, 2, 3, 4}
    sp, _ = sets["max_table"]
    ids = list(sp.values())
    assert len(sp) == SS.MAX_SPECIALS and len(set(ids)) == len(ids) and 0 in ids and 0xFFFFFFFE in ids
    assert sum(i < 100000 for i in ids) >= 100 and max(len(t.encode()) for t in sp) == 64
    sp, _ = sets["overlaps"]
    names = list(sp)
    a, d = names[0], names[2]
    assert d in a and not a.startswith(d) and names[5] in names[3] + names[3] and names[5] not in names[3]


@pytest.mark.parametrize("policy", SS.POLICIES)
@pytest.mark.parametrize("pat,n_ranks", SLOTS)
@pytest.mark.parametrize("name", SS.SETS)
def test_set_against_the_reference(sim_vocabs, encoders, ranks, sets, tables, name, pat, n_ranks, policy):
    specials, texts = sets[name]
    T, sp = tables[name]
    assert sp.rc == 0, sp.err
    modes = SS.policy_modes(policy, len(specials))
    ml = None if modes is None else [modes]
    prompts = [t.encode() for t in texts]
    want, nst, off = run([sim_vocabs[pat]], [sp], ml, prompts, None, [T], [encoders[pat]])
    if policy != "allow_all":
        assert want[0] == "bad"                      # every set spells a DISALLOWED special somewhere
        prompts, _ = SS.without_bad([T], ml, prompts, None)
        want, nst, off = run([sim_vocabs[pat]], [sp], ml, prompts, None, [T], [encoders[pat]])
    assert want[0] == "ok"
    starts = np.cumsum([0] + [len(p) for p in prompts])
    kept = [(int(starts[i]) + a, b - a, k) for i, ks in enumerate(want[2]) for a, b, k in ks]
    if policy == "allow_all":
        assert nst > len(prompts)
        if name == "all_lengths":                    # every length kept; the 64-byte one (64 probes) at every lane offset
            assert {n for _, n, _ in kept} == set(range(1, 65))
            assert {q % 16 for q, n, _ in kept if n == 64} == set(range(16))
        if name == "max_table":
            assert len({k for _, _, k in kept}) == SS.MAX_SPECIALS
        if name == "dense":
            per_word, per_trip, trips, shared = walk_witness(want[2], starts)
            assert per_word == 32 and per_trip > 32 and trips >= 64 and shared > 0, (per_word, per_trip, trips, shared)
    if pat == 0:
        n = tiktoken_pin(ranks[pat], pat, specials, modes, texts)
        assert n == len(texts) if SS.is_prefix_free(specials) else n > 0


# ---- eight vocabularies in one batch ------------------------------------------------------------------------------------
def test_eight_vocabularies_with_their_own_sets(sim_vocabs, encoders, sets, tables):
    prompts, vid = SS.eight_vocab_batch(sets, 8, 1500)
    modes, tabs = SS.eight_vocab_modes(sets)
    sps = [None if name is None else tables[name][1] for _, name, _ in SS.EIGHT]
    vocabs = [sim_vocabs[pat] for pat, _, _ in SS.EIGHT]
    encs = [encoders[pat] for pat, _, _ in SS.EIGHT]
    want, _, _ = run(vocabs, sps, modes, prompts, vid, tabs, encs)
    assert want[0] == "bad"
    prompts, vid = SS.without_bad(tabs, modes, prompts, vid)
    assert len(prompts) > 800 and set(vid.tolist()) == set(range(8))
    want, nst, _ = run(vocabs, sps, modes, prompts, vid, tabs, encs)
    kept_slots = {int(vid[i]) for i, ks in enumerate(want[2]) if ks}
    assert kept_slots == {0, 1, 2, 3, 4, 7} and nst > len(prompts)
    # a DISALLOWED special of slot 7 in the batch's last prompt: its index (12 bits beside the slot in bad_inv) comes back
    T7 = tabs[7]
    k = max(k for k in range(len(T7.toks)) if modes[7][k] == SS.DISALLOW)
    rc, _, _, bad, _, _ = S.encode_batch_special(vocabs, sps, prompts + [b"x " + T7.toks[k]], modes=modes,
                                                 vocab_ids=np.append(vid, 7).astype(np.uint8))
    assert rc == S.EBADMSG and bad == (len(prompts), k)


# ---- sizing, counts, ENOSPC ---------------------------------------------------------------------------------------------
def dense_batch(sets):
    return [t.encode() for t in sets["dense"][1] if len(t) <= 4096][:400]


def test_max_prompts_boundary_on_a_dense_batch(sim_vocabs, encoders, sets, tables):
    T, sp = tables["dense"]
    allow = [SS.policy_modes("allow_all", len(T.toks))]
    prompts = dense_batch(sets)
    want = SS.reference([T], allow, prompts, None, [encoders[0]])
    need = len(prompts) + 2 * sum(len(k) for k in want[2])
    assert need > 4 * len(prompts)
    rc, got, _, _, nst, _ = S.encode_batch_special([sim_vocabs[0]], [sp], prompts, modes=allow, max_prompts=need)
    assert rc == 0 and nst == need and got == want[1]
    rc, *_ = S.encode_batch_special([sim_vocabs[0]], [sp], prompts, modes=allow, max_prompts=need - 1)
    assert rc == S.EINVAL


def test_counts_only_and_enospc_on_a_dense_batch(sim_vocabs, encoders, sets, tables):
    T, sp = tables["dense"]
    allow = [SS.policy_modes("allow_all", len(T.toks))]
    prompts = dense_batch(sets)
    want = SS.reference([T], allow, prompts, None, [encoders[0]])
    counts = [len(w) for w in want[1]]
    total = sum(counts)
    rc, _, got_counts, _, _, off = S.encode_batch_special([sim_vocabs[0]], [sp], prompts, modes=allow, counts_only=True)
    assert rc == 0 and got_counts == counts and off.tolist() == np.cumsum([0] + counts).tolist()
    rc, _, _, _, _, off = S.encode_batch_special([sim_vocabs[0]], [sp], prompts, modes=allow, out_cap=total - 1)
    assert rc == S.ENOSPC and int(off[-1]) == total
    rc, got, _, _, _, _ = S.encode_batch_special([sim_vocabs[0]], [sp], prompts, modes=allow, out_cap=total)
    assert rc == 0 and got == want[1]


# ---- decode and the index of a disallowed special -----------------------------------------------------------------------
def decode(vocab, sp, seqs):
    io = np.cumsum([0] + [len(s) for s in seqs]).astype(np.uint64)
    rc, out, off = S.decode_batch([vocab], [i for s in seqs for i in s], io, specials=[sp])
    return rc, [bytes(out[int(off[i]):int(off[i + 1])]) for i in range(len(seqs))] if rc == 0 else None


@pytest.mark.parametrize("pat,n_ranks", SLOTS)
def test_decode_every_id_of_a_full_table(sim_vocabs, ranks, tables, pat, n_ranks):
    """every special id of the 4096-entry table, ascending and shuffled: an id below n_ranks is the ordinary token"""
    T, sp = tables["max_table"]
    token = {i: t for t, i in ranks[pat].items()}
    by_id = {i: (token[i] if i < n_ranks else T.toks[k]) for k, i in enumerate(T.ids)}
    assert sum(i < n_ranks for i in by_id) >= 100
    rng = random.Random(pat)
    for order in (sorted(by_id), rng.sample(sorted(by_id), len(by_id))):
        seqs, i = [], 0
        while i < len(order):
            n = rng.randint(1, 40)
            seqs.append(order[i:i + n])
            i += n
        rc, back = decode(sim_vocabs[pat], sp, seqs)
        assert rc == 0
        assert back == [b"".join(by_id[i] for i in s) for s in seqs]
    ids = set(T.ids)
    for missing in (n_ranks, 0xFFFFFFFF, next(i for i in range(n_ranks + 1, 1 << 32) if i not in ids), max(ids) - 1):
        if missing in ids:
            continue
        rc, _ = decode(sim_vocabs[pat], sp, [[T.ids[0] if T.ids[0] >= n_ranks else 0], [missing]])
        assert rc == S.EINVAL, missing


def test_disallowed_special_at_a_high_index_is_reported(sim_vocabs, tables):
    T, sp = tables["max_table"]
    for k in (2047, 2048, 3000, 4095):
        modes = np.full(len(T.toks), SS.ALLOW, np.uint8)
        modes[k] = SS.DISALLOW
        other = T.toks[(k + 1) % len(T.toks)]
        prompts = [b"clean " + other, other + b" x" + T.toks[k] + b"y " + other, T.toks[k]]
        rc, _, _, bad, _, _ = S.encode_batch_special([sim_vocabs[0]], [sp], prompts, modes=[modes])
        assert rc == S.EBADMSG and bad == (1, k), (k, bad)
