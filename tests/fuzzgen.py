"""Seeded generator of nasty pre-tokenizer inputs (test infrastructure).

Covers the edge cases SURVEY.md H1 lists: contractions in every case incl. U+017F,
digit runs, CR/LF/other-whitespace mixes (U+0085, U+00A0, U+2028, U+3000), combining
marks, titlecase / modifier letters, astral code points, '/' and newline trailers."""
import random

ATOMS = {
    "lower": list("abcdefghijklmnopqrstuvwxyz") + ["é", "ß", "ſ", "я", "λ", "ö"],
    "upper": list("ABCDEFGHIJKLMNOPQRSTUVWXYZ") + ["É", "Я", "Λ", "Ö", "K"],
    "title": ["ǅ", "ǈ", "ᾈ"],
    "other_letter": ["中", "文", "日", "本", "語", "한", "글", "ع", "ر",
                     "ب", "א", "ב", "ʰ", "ˀ", "\U00020000", "\U00010400"],
    "mark": ["́", "̀", "̈", "ा", "⃝", "\U000e0100"],
    "digit": list("0123456789") + ["٣", "５", "Ⅷ", "²", "½", "\U0001d7d8"],
    "space": [" "],
    "ws": ["\t", " ", "", " ", "　", "\x0b", "\x0c", " "],
    "crlf": ["\n", "\r", "\r\n", "\n\n"],
    "punct": list("!\"#$%&()*+,-.:;<=>?@[\\]^_`{|}~") + ["…", "—", "«", "€", "\U0001f600",
                                                          "\U0001f3f3️", "‍", "\x00", "\x1f", "\x7f"],
    "apos": ["'"],
    "slash": ["/"],
    "contr": ["'s", "'S", "'t", "'T", "'re", "'RE", "'rE", "'ve", "'Ve", "'m", "'M", "'ll", "'LL", "'lL", "'d", "'D",
              "'ſ", "'l", "'r", "'v", "'", "''s", "'sx", "'lll"],
}
KINDS = list(ATOMS)
WEIGHTS = [10, 6, 1, 4, 3, 5, 8, 3, 4, 6, 3, 2, 4]


def fuzz_string(rng: random.Random, max_atoms=24) -> str:
    n = rng.randint(0, max_atoms)
    out = []
    kind = rng.choices(KINDS, WEIGHTS)[0]
    for _ in range(n):
        if rng.random() < 0.45:
            kind = rng.choices(KINDS, WEIGHTS)[0]
        out.append(rng.choice(ATOMS[kind]))
    return "".join(out)


def fuzz_strings(seed: int, count: int, max_atoms=24):
    rng = random.Random(seed)
    return [fuzz_string(rng, max_atoms) for _ in range(count)]


SCALAR_CONTEXTS = [lambda c: c, lambda c: "a" + c + "b", lambda c: " " + c + c + "'s", lambda c: "A" + c + "1",
                   lambda c: "!" + c + "\n"]


def every_scalar_value(context: int, per_prompt=16):
    """all 1 112 064 Unicode scalar values (every code point but the surrogates), in order, each wrapped in one of the five
    SCALAR_CONTEXTS (alone, between letters, doubled after a space with a contraction, between a capital and a digit,
    after punctuation before a newline), per_prompt of them a prompt"""
    f = SCALAR_CONTEXTS[context]
    cps = [c for c in range(0x110000) if not 0xD800 <= c <= 0xDFFF]
    return ["".join(f(chr(c)) for c in cps[i:i + per_prompt]) for i in range(0, len(cps), per_prompt)]


def long_runs(seed: int):
    """adversarial long single-class runs and repeats"""
    rng = random.Random(seed)
    out = []
    for ch in ["a", "A", "aB", "ab", " ", "\n", " \n", "1", "!", "'s", "́", "中", "á", "/", "\t",
               "é", "\U0001f600", "!\n/"]:
        for n in [1, 2, 3, 4, 7, 31, 32, 33, 64, 100, 257]:
            out.append(ch * n)
    for _ in range(40):
        a = rng.choice("abcdefgh")
        b = rng.choice("abcdefgh ")
        out.append((a + b) * rng.randint(5, 80) + rng.choice(["", " ", "\n", "x"]))
    return out
