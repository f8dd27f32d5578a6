"""Encode with special tokens (csrc/specials.cuh) on the CPU SIMT emulator, against live tiktoken 0.12.0
`Encoding.encode(text, allowed_special=..., disallowed_special=...)` built on the committed Tekken ranks, and -- where tiktoken's
choice is undefined (one special a prefix of another) -- against the host cut of the plugin trait's default."""
import base64
import random

import numpy as np
import pytest

import fuzzgen
from conftest import COMBOS

import simspecial as S

tiktoken = pytest.importorskip("tiktoken")

# ids above every slot's ranks (the stand-in vocabularies have at most 150 000 ranks)
SPECIALS = {"<|endoftext|>": 200000, "<|fim_prefix|>": 200001, "<|endofprompt|>": 200002, "<|eot_id|>": 200003,
            "<|start_header_id|>": 200004, "<|end_header_id|>": 200005, "<|é中|>": 200006, "\U0001f600!": 200007}
KEYS = list(SPECIALS)


@pytest.fixture(scope="module")
def vocabs(tekken_bytes):
    return {pat: S.Vocab(tekken_bytes, pat, n) for pat, n in COMBOS}


@pytest.fixture(scope="module")
def encodings(tekken_bytes):
    from oracle import patterns as PT
    lines = tekken_bytes.splitlines()
    out = {}
    for pat, n in COMBOS:
        ranks = {base64.b64decode(l.split()[0]): i for i, l in enumerate(lines[:n])}
        out[pat] = tiktoken.Encoding("live%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks, special_tokens=SPECIALS)
    return out


def modes_for(allowed, disallowed, specials=SPECIALS):
    return np.array([S.DISALLOW if t in disallowed else (S.ALLOW if t in allowed else S.ORDINARY) for t in specials], dtype=np.uint8)


def texts_with_specials(seed, n):
    rng = random.Random(seed)
    base = fuzzgen.fuzz_strings(seed, n, max_atoms=30)
    out = []
    for i, t in enumerate(base):
        k, k2 = rng.choice(KEYS), rng.choice(KEYS)
        cut = rng.randint(0, len(t))
        out.append([t, k + t, t + k, t[:cut] + k + t[cut:] + k2 + k2, k, t[:cut] + " \n  " + k + "   " + t[cut:], k + k2 + k][i % 7])
    return out


@pytest.mark.parametrize("pat,n_ranks", COMBOS)
def test_allowed_all_against_live_tiktoken(vocabs, encodings, pat, n_ranks):
    """fuzz texts with specials spliced in (at the start, the end, inside, adjacent, alone, after whitespace), every pattern"""
    enc = encodings[pat]
    texts = texts_with_specials(500 + pat, 240) + ["", "   ", "x" + KEYS[0], " \n\n" + KEYS[1] + "\n\n "]
    sp = S.Specials(SPECIALS)
    rc, got, counts, _, nst, _ = S.encode_batch_special([vocabs[pat]], [sp], [t.encode() for t in texts], modes=[modes_for(set(SPECIALS), set())])
    assert rc == 0
    assert nst > len(texts)                     # the stretch path ran
    for t, g, c in zip(texts, got, counts):
        want = enc.encode(t, allowed_special="all")
        assert g == want, repr(t)
        assert c == len(want)


@pytest.mark.parametrize("pat,n_ranks", COMBOS[:2])
def test_some_allowed_rest_ordinary_against_live_tiktoken(vocabs, encodings, pat, n_ranks):
    enc = encodings[pat]
    allowed = {KEYS[0], KEYS[3], KEYS[6]}
    texts = texts_with_specials(900 + pat, 200)
    sp = S.Specials(SPECIALS)
    rc, got, _, _, _, _ = S.encode_batch_special([vocabs[pat]], [sp], [t.encode() for t in texts], modes=[modes_for(allowed, set())])
    assert rc == 0
    for t, g in zip(texts, got):
        assert g == enc.encode(t, allowed_special=allowed, disallowed_special=()), repr(t)


def test_default_policy_on_clean_text_takes_the_fast_path(vocabs, encodings):
    """modes NULL = every special DISALLOWED (tiktoken's default): text without specials gives encode_ordinary's ids, no stretches"""
    enc = encodings[0]
    texts = [t for t in fuzzgen.fuzz_strings(77, 300, max_atoms=40) if "<|" not in t] + ["a <| b |> c <|endoftex"]
    rc, got, _, _, nst, _ = S.encode_batch_special([vocabs[0]], [S.Specials(SPECIALS)], [t.encode() for t in texts])
    assert rc == 0 and nst == len(texts)
    for t, g in zip(texts, got):
        assert g == enc.encode(t), repr(t)


def test_disallowed_reports_lowest_prompt_and_leftmost_special(vocabs):
    sp = S.Specials(SPECIALS)
    prompts = [b"clean", b"x <|fim_prefix|> and <|endoftext|>", b"<|endoftext|>"]
    rc, _, _, bad, _, _ = S.encode_batch_special([vocabs[0]], [sp], prompts)
    assert rc == S.EBADMSG and bad == (1, KEYS.index("<|fim_prefix|>"))
    # DISALLOWED inside an ALLOWED occurrence still fails: tiktoken searches the raw text
    inner = {"<|a<|x|>b|>": 300, "<|x|>": 301}
    rc, _, _, bad, _, _ = S.encode_batch_special([vocabs[0]], [S.Specials(inner)], [b"ok", b"<|a<|x|>b|>"],
                                                 modes=[np.array([S.ALLOW, S.DISALLOW], np.uint8)])
    assert rc == S.EBADMSG and bad == (1, 1)
    # a disallowed special wins over malformed UTF-8 in an earlier prompt
    rc, _, _, bad, _, _ = S.encode_batch_special([vocabs[0]], [sp], [b"\xff\xfe", b"a<|eot_id|>"])
    assert rc == S.EBADMSG and bad == (1, KEYS.index("<|eot_id|>"))
    # ... and malformed UTF-8 alone is still EILSEQ
    rc, *_ = S.encode_batch_special([vocabs[0]], [sp], [b"\xff\xfe", b"a<|eot_id|>"], modes=[modes_for(set(SPECIALS), set())])
    assert rc == S.EILSEQ


def test_occurrence_across_a_prompt_boundary_does_not_match(vocabs, encodings):
    enc = encodings[0]
    prompts = ["abc <|endof", "text|> def", "<|eot_id", "|>"]
    rc, got, _, _, _, _ = S.encode_batch_special([vocabs[0]], [S.Specials(SPECIALS)], [p.encode() for p in prompts])
    assert rc == 0                               # (nothing disallowed is found: no prompt holds a whole special)
    for p, g in zip(prompts, got):
        assert g == enc.encode_ordinary(p)


def test_prefix_sharing_and_overlapping_sets_against_the_host_cut(vocabs):
    """one special a prefix of another, overlapping occurrences: leftmost, then longest, then non-overlapping (the host cut)"""
    from cfbpe import plugin as P
    specials = {"<|a|>": 1000000, "<|a|>b": 1000001, "<|a|>bc": 1000002, "a|><|a": 1000003, "|><": 1000004, "x": 1000005}
    specials.update({"<|reserved_special_token_%d|>" % i: 1000100 + i for i in range(250)})
    rng = random.Random(5)
    atoms = list(specials) + ["a", "b", "c", "<|", "|>", " ", "\n", "<|reserved_special_token_", "|>b"]
    texts = ["".join(rng.choice(atoms) for _ in range(rng.randint(0, 14))) for _ in range(300)]

    class Plain(P.TokenizerPluginClient):        # the host cut over the emulator's ordinary path
        def encode_batch(self, ctx, req):
            n = len(req.offsets) - 1
            prompts = [bytes(req.bytes[int(req.offsets[i]):int(req.offsets[i + 1])]) for i in range(n)]
            rc, got, counts, _, _, off = S.encode_batch_special([vocabs[0]], [None], prompts)
            assert rc == 0
            return P.EncodeBatchResponse(np.array([i for g in got for i in g], np.uint32), off, np.array(counts, np.uint32))

    allowed = {t for i, t in enumerate(specials) if i % 3 != 2}
    want = Plain().encode_batch_special(P.SecurityContext.anonymous(), P.EncodeBatchRequest(P.VocabRef("x"), *P.pack_texts(texts)),
                                        specials, allowed, set())
    rc, got, _, _, _, off = S.encode_batch_special([vocabs[0]], [S.Specials(specials)], [t.encode() for t in texts],
                                                   modes=[modes_for(allowed, set(), specials)])
    assert rc == 0
    assert np.array_equal(off, want.offsets)
    assert [i for g in got for i in g] == want.ids.tolist()


def test_multi_vocabulary_batch_with_its_own_sets(vocabs, encodings):
    sp0 = {"<|endoftext|>": 200000, "<|eot_id|>": 200003}
    sp3 = {"[INST]": 300001, "[/INST]": 300002}
    texts = ["a<|endoftext|>b[INST]", "[INST] hi [/INST]<|eot_id|>", "<|eot_id|>x", "plain [/INST]"]
    vid = [0, 1, 0, 1]
    rc, got, _, _, _, _ = S.encode_batch_special([vocabs[0], vocabs[3]], [S.Specials(sp0), S.Specials(sp3)], [t.encode() for t in texts],
                                                 modes=[np.array([1, 1], np.uint8), np.array([1, 0], np.uint8)], vocab_ids=vid)
    assert rc == 0
    e0 = tiktoken.Encoding("v0", pat_str=encodings[0]._pat_str, mergeable_ranks=encodings[0]._mergeable_ranks, special_tokens=sp0)
    e3 = tiktoken.Encoding("v3", pat_str=encodings[3]._pat_str, mergeable_ranks=encodings[3]._mergeable_ranks, special_tokens=sp3)
    assert got[0] == e0.encode(texts[0], allowed_special="all")
    assert got[1] == e3.encode(texts[1], allowed_special={"[INST]"}, disallowed_special=())
    assert got[2] == e0.encode(texts[2], allowed_special="all")
    assert got[3] == e3.encode(texts[3], allowed_special={"[INST]"}, disallowed_special=())


def test_limits_counts_only_and_enospc(vocabs):
    sp = S.Specials(SPECIALS)
    allow = [modes_for(set(SPECIALS), set())]
    prompts = [b"<|eot_id|><|eot_id|>", b"a<|eot_id|>"]
    rc, *_ = S.encode_batch_special([vocabs[0]], [sp], prompts, modes=allow, max_prompts=2 + 2 * 3 - 1)
    assert rc == S.EINVAL                        # 2 prompts + 2 x 3 matches = 8 stretches
    rc, got, counts, _, nst, _ = S.encode_batch_special([vocabs[0]], [sp], prompts, modes=allow, max_prompts=8)
    assert rc == 0 and nst == 8 and got[0] == [200003, 200003] and got[1][-1] == 200003 and counts == [2, len(got[1])]
    rc, _, counts2, _, _, _ = S.encode_batch_special([vocabs[0]], [sp], prompts, modes=allow, counts_only=True)
    assert rc == 0 and counts2 == counts
    rc, _, _, _, _, off = S.encode_batch_special([vocabs[0]], [sp], prompts, modes=allow, out_cap=2)
    assert rc == S.ENOSPC and int(off[-1]) == sum(counts)


def test_registration_errors():
    assert S.Specials({"<|a|>": 1, "<|b|>": 2}).rc == 0
    assert S.Specials({}).rc == 0
    for bad in ({"<|a|>": 1, b"<|a|>": 2}, {"": 1}, {"x" * 65: 1}, {b"\xff<|a|>": 1}, {b"\xed\xa0\x80": 1}, {"a": 1, "b": 1},
                {"a": 0xFFFFFFFF}, {"t%d" % i: i for i in range(4097)}):
        t = S.Specials(bad)
        assert t.rc == S.EINVAL, bad
        assert t.err


def test_decode_round_trip_of_special_ids(vocabs, encodings):
    sp = S.Specials(SPECIALS)
    texts = texts_with_specials(4242, 60)
    rc, got, _, _, _, _ = S.encode_batch_special([vocabs[0]], [sp], [t.encode() for t in texts], modes=[modes_for(set(SPECIALS), set())])
    assert rc == 0
    rc, back = S.decode_batch([vocabs[0]], [sp], got)
    assert rc == 0 and back == [t.encode() for t in texts]
    rc, _ = S.decode_batch([vocabs[0]], [sp], [[999999]])
    assert rc == S.EINVAL                        # neither an ordinary nor a special id
    rc, _ = S.decode_batch([vocabs[0]], [None], [[200000]])
    assert rc == S.EINVAL                        # no table: the id is unknown, as before
