"""Id bases (cfbpe_vocab_set_id_base) on the SIMT emulator: the rebase kernel after the encode pass -- one vocabulary, mixed vocabularies
whose unbased ids must stay exactly the ranks, sub-batches of a pipelined call, special stretches whose control ids pass through
unshifted -- and the decode mapping at the edges of [base, base + n_ranks).  Reference: the C oracle's ranks."""
import random

import numpy as np
import pytest

import fuzzgen
import id_base_lib as IB
import simlib

TEKKEN, CL100K = 3, 0
N_TEK, N_CL = 130072, 100256


@pytest.fixture(scope="module")
def vocabs(tekken_bytes):
    """slot 0: the cl100k stand-in (ids stay ranks), slot 1: Tekken as Mistral numbers it"""
    return [simlib.SimVocab(tekken_bytes, 0, CL100K, N_CL), simlib.SimVocab(tekken_bytes, 0, TEKKEN, N_TEK)]


@pytest.fixture(scope="module")
def oracles(tekken_bytes):
    from oracle import oracle
    return [oracle.OracleVocab(tekken_bytes, N_CL), oracle.OracleVocab(tekken_bytes, N_TEK)]


PATS = [CL100K, TEKKEN]
CONTROLS = {"<unk>": 0, "<s>": 1, "</s>": 2, "[INST]": 3, "[/INST]": 4, "[TOOL_CONTENT]": 19, "<SPECIAL_999>": 999}


def _prompts(seed, n):
    return [s.encode() for s in fuzzgen.fuzz_strings(seed, n, max_atoms=30)] + [b"", b"x", b" " * 40, "naïve café 你好".encode()]


def _ranks(oracles, vid, p):
    return [int(x) for x in oracles[vid].encode(PATS[vid], p)]


@pytest.mark.parametrize("cuts", [None, [1], [7, 50, 51, 150]])
def test_one_vocabulary_adds_its_base(vocabs, oracles, cuts):
    prompts = _prompts(1, 200)
    rc, ids = IB.encode(vocabs[1:], prompts, bases=[1000], cuts=cuts)
    assert rc == 0
    for p, got in zip(prompts, ids):
        assert got == [r + 1000 for r in _ranks(oracles, 1, p)]


@pytest.mark.parametrize("cuts", [None, [3, 90, 91, 200]])
@pytest.mark.parametrize("bases", [[0, 1000], [5, 1000], [0, 0xFFFFFFFF - N_TEK]])
def test_mixed_vocabularies(vocabs, oracles, cuts, bases):
    """each prompt gets its own vocabulary's base; a vocabulary with base 0 keeps exactly the ids it had without bases"""
    prompts = _prompts(2, 240)
    rng = random.Random(3)
    vid = [rng.randrange(2) for _ in prompts]
    rc, plain = IB.encode(vocabs, prompts, bases=None, vocab_ids=vid, cuts=cuts)
    assert rc == 0
    rc, based = IB.encode(vocabs, prompts, bases=bases, vocab_ids=vid, cuts=cuts)
    assert rc == 0
    for p, v, a, b in zip(prompts, vid, plain, based):
        assert a == _ranks(oracles, v, p)
        assert b == [r + bases[v] for r in a]


def _split_specials(text, specials):
    """tiktoken's cut: leftmost occurrence, longest there -> [(is_special, str)]"""
    out, pos = [], 0
    toks = sorted(specials, key=len, reverse=True)
    while True:
        hits = [(text.find(t, pos), -len(t), t) for t in toks if text.find(t, pos) >= 0]
        if not hits:
            break
        at, _, t = min(hits)
        if at > pos:
            out.append((False, text[pos:at]))
        out.append((True, t))
        pos = at + len(t)
    if pos < len(text):
        out.append((False, text[pos:]))
    return out


def test_special_stretches_keep_their_ids(vocabs, oracles):
    """the ordinary pass's ids are rebased before the splice: text ids are base + rank, a control token's id is as registered"""
    rng = random.Random(4)
    texts = fuzzgen.fuzz_strings(5, 120, max_atoms=12)
    prompts = ["".join(rng.choice([t, "<s>", "[INST]", "[/INST]", "</s>", " ", "<SPECIAL_999>"]) for t in rng.sample(texts, 4)) for _ in range(120)]
    prompts += ["[INST][/INST]", "<s>", "", "no control token here"]
    rc, ids, spliced = IB.encode_special(vocabs, [p.encode() for p in prompts], [None, CONTROLS], bases=[0, 1000], vocab_ids=[1] * len(prompts))
    assert rc == 0 and spliced
    for p, got in zip(prompts, ids):
        want = []
        for is_sp, s in _split_specials(p, CONTROLS):
            want += [CONTROLS[s]] if is_sp else [r + 1000 for r in _ranks(oracles, 1, s.encode())]
        assert got == want, p
    # no control token in any prompt: the ordinary path, then the rebase
    plain = [b"hello world", b"", "déjà vu".encode()]
    rc, ids, spliced = IB.encode_special(vocabs, plain, [None, CONTROLS], bases=[0, 1000], vocab_ids=[1, 1, 1])
    assert rc == 0 and not spliced
    assert ids == [[r + 1000 for r in _ranks(oracles, 1, p)] for p in plain]


def test_decode_at_the_edges_of_the_range(vocabs, tekken_bytes):
    from cfbpe import workload as W
    toks = W.vocab_tokens(tekken_bytes, N_TEK)
    tek = vocabs[1:]
    base = 1000
    edges = {base - 1: None, base: toks[0], base + 1: toks[1], base + N_TEK - 1: toks[-1], base + N_TEK: None}
    for i, want in edges.items():
        rc, out = IB.decode(tek, [[i]], bases=[base])
        assert (rc, out) == ((0, [want]) if want is not None else (simlib.EINVAL, None)), i
    # control ids below the base and a special past the range resolve through the special table
    past = dict(CONTROLS, **{"<past>": base + N_TEK})
    seq = [1, 3, base + 100, 4, base + N_TEK - 1, 2, base + N_TEK, 999, 0]
    rc, out = IB.decode(tek, [seq, [], [base]], bases=[base], specials=[past])
    assert rc == 0
    assert out == [b"<s>[INST]" + toks[100] + b"[/INST]" + toks[-1] + b"</s><past><SPECIAL_999><unk>", b"", toks[0]]
    # base 0: an id below n_ranks is the ordinary token, as it always was (a special registered on it does not change that)
    rc, out = IB.decode(tek, [[0, 5, N_TEK - 1]], bases=[0], specials=[{"<zero>": 0}])
    assert (rc, out) == (0, [toks[0] + toks[5] + toks[-1]])
    rc, _ = IB.decode(tek, [[N_TEK]], bases=[0])
    assert rc == simlib.EINVAL
    # mixed: each sequence decodes under its vocabulary's base
    rc, out = IB.decode(vocabs, [[7], [1007], [7]], bases=[0, 1000], vocab_ids=[0, 1, 0])
    assert (rc, out) == (0, [toks[7], toks[7], toks[7]])
    rc, _ = IB.decode(vocabs, [[7], [7]], bases=[0, 1000], vocab_ids=[0, 1])
    assert rc == simlib.EINVAL


def test_specials_may_not_take_ordinary_ids():
    """cfbpe_vocab_set_id_base / cfbpe_vocab_set_specials refuse a special whose id is base + a rank (special_in_id_range)"""
    n = 500
    assert IB.special_in_id_range({"<a>": 0, "<b>": 499, "<c>": 1000}, 0, n) == -1          # base 0: no rule, as before
    assert IB.special_in_id_range({"<a>": 0, "<b>": 999, "<c>": 1000 + n}, 1000, n) == -1
    assert IB.special_in_id_range({"<a>": 0, "<b>": 1000}, 1000, n) == 1
    assert IB.special_in_id_range({"<b>": 1000 + n - 1, "<a>": 3}, 1000, n) == 0
    ctl = {t: i for i, t in enumerate(["<unk>", "<s>", "</s>"] + ["<SPECIAL_%d>" % k for k in range(3, 1000)])}
    assert IB.special_in_id_range(ctl, 1000, N_TEK) == -1 and IB.special_in_id_range(ctl, 999, N_TEK) == 999
