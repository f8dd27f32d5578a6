"""Seeded special-token sets shaped to reach the branches of the special-token kernels (test infrastructure).

The realistic eight-token set the other special tests use has a few lengths of 8..19 bytes, one shared first byte and a
16-slot hash table.  The sets below go where it does not: every length 1..64 (64 hash probes a position), the full
4096-entry table with long probe chains and ids over the whole uint32 range, one-byte specials (every bm2 bit of their first
byte), prompts that are nothing but matches (many marks per bit word, many 1 KiB walk trips, prompt seams inside a word),
and specials that overlap and contain one another.  Each set returns (specials, texts): {token str: id} in special-index
order, and prompts built to reach the branch the set is about.  The mixed policy of the tests gives special k the mode
MIXED[k % 3]; `overlaps` orders its specials by that rule.

`reference` is what a special-token encode call must return, computed in plain Python without the GPU, the emulator or the
plugin: DISALLOWED anywhere fails the call; else the leftmost ALLOWED occurrence, the longest one there, is kept and the search
resumes after it; the text between kept specials is encoded by a given ordinary encoder (live tiktoken, or the oracle)."""
import random

import numpy as np

MAX_SPECIALS = 4096        # specials.h: kMaxSpecials
MAX_LEN = 64               # kMaxSpecialLen
ABOVE = 1 << 20            # ids from here up are above the ranks of every stand-in slot (at most 150 000)
ORDINARY, ALLOW, DISALLOW = 0, 1, 2     # CFBPE_SPECIAL_*
MIXED = (ALLOW, ORDINARY, DISALLOW)    # the mixed policy: special k gets MIXED[k % 3]
POLICIES = ("allow_all", "mixed", "default")
SETS = ("all_lengths", "max_table", "one_byte", "dense", "overlaps")
CHARS = ["a", "Z", "<", "|", "é", "ß", "中", "ー", "😀", "𝄞"]     # 1-, 2-, 3- and 4-byte UTF-8
FILLER = "qwxy .,\n'"                                               # no special of these sets starts with one of these


def _chars_of(rng, n_bytes, chars=CHARS):
    """a random string of exactly n_bytes UTF-8 bytes over chars"""
    out, n = [], 0
    while n < n_bytes:
        c = rng.choice([c for c in chars if len(c.encode()) <= n_bytes - n])
        out.append(c)
        n += len(c.encode())
    return "".join(out)


def _filler(rng, n_bytes):
    return "".join(rng.choice(FILLER) for _ in range(n_bytes))


def near_misses(s):
    """s with its last byte changed (still valid UTF-8), and s without its last character"""
    b = bytearray(s.encode())
    b[-1] = (ord("q") if b[-1] != ord("q") else ord("w")) if b[-1] < 0x80 else 0x80 + ((b[-1] - 0x80 + 1) & 63)
    return [b.decode(), s[:-1]]


def is_prefix_free(toks):
    bs = sorted(t.encode() for t in toks)
    return all(not bs[i + 1].startswith(bs[i]) for i in range(len(bs) - 1))


def all_lengths(seed=11):
    """one special of every length 1..64 bytes over ASCII and 2-, 3-, 4-byte characters, none a prefix of another.  Texts:
    each special at every offset mod 16 of the batch (every prompt is a multiple of 16 bytes, so prompt offsets are batch
    offsets mod 16), ending at the prompt's last byte, as a whole prompt, its near misses, and all 64 in one prompt"""
    rng = random.Random(seed)
    toks = ["@"]
    for n in range(2, MAX_LEN + 1):
        while True:
            t = _chars_of(rng, n)
            if not any(t.encode().startswith(u.encode()) for u in toks):
                break
        toks.append(t)
    specials = {t: ABOVE + 17 * k for k, t in enumerate(toks)}
    texts = []
    for t in toks:
        for o in range(16):
            body = _filler(rng, o) + t
            texts.append(body + _filler(rng, (-len(body.encode())) % 16))
        texts += [_filler(rng, rng.randint(1, 20)) + t, t, t + t]
        texts += [_filler(rng, rng.randint(0, 5)) + m for m in near_misses(t)]
    order = list(toks)
    rng.shuffle(order)
    texts.append(" ".join(order))
    texts.append("".join(order))
    return specials, texts


def max_table(seed=12):
    """4096 specials: families that share their first one and two bytes (<|r_N|>, <|reserved_special_token_N|>, [INST_N])
    and a few hundred random ones, so the hash table (8192 slots) holds long probe chains.  Ids spread over the whole uint32
    range except 0xFFFFFFFF, 0 and 0xFFFFFFFE among them, a hundred of them below 100 000 (ordinary ranks of every slot).
    Texts: every special at least once, and family members that are not specials"""
    rng = random.Random(seed)
    toks = ["<|r_%d|>" % i for i in range(1800)] + ["<|reserved_special_token_%d|>" % i for i in range(1200)]
    toks += ["[INST_%d]" % i for i in range(700)]
    seen = set(toks)
    while len(toks) < MAX_SPECIALS:
        t = _chars_of(rng, rng.randint(2, MAX_LEN))
        if t not in seen:
            seen.add(t)
            toks.append(t)
    rng.shuffle(toks)
    ids = set(rng.sample(range(1, 100000), 100)) | {0, 0xFFFFFFFE}
    while len(ids) < MAX_SPECIALS:
        ids.add(rng.randrange(100000, 0xFFFFFFFF))
    ids = list(ids)
    rng.shuffle(ids)
    specials = dict(zip(toks, ids))
    order = list(toks)
    rng.shuffle(order)
    texts, i = [], 0
    while i < len(order):
        k = rng.randint(1, 24)
        texts.append("".join(_filler(rng, rng.randint(0, 3)) + t for t in order[i:i + k]))
        i += k
    texts += ["<|r_%d|> <|r_%d" % (rng.randrange(1800, 10 ** 6), rng.randrange(1800)) for _ in range(100)]
    texts += ["[INST_%d][INST_%d" % (rng.randrange(700, 10 ** 5), rng.randrange(700)) for _ in range(60)]
    texts += ["<|reserved_special_token_%d|>" % rng.randrange(1200, 10 ** 4) for _ in range(60)]
    return specials, texts


def one_byte(seed=13):
    """the one-byte specials "@" and "~" beside longer specials that start with the same byte.  Texts: a one-byte special
    inside text, as the prompt's last byte, as a whole prompt, in runs"""
    rng = random.Random(seed)
    toks = ["@", "~", "@home", "@@", "~>", "~~~", "@é", "home~"]
    specials = {t: ABOVE + 1000 + k for k, t in enumerate(toks)}
    atoms = toks + ["home", "a", "x", " ", "é", "\n", "ho", ">"]
    texts = ["@", "~", "a@", "a~", "@a", "x@y", "é@é", "é~", "@é", "@\n", "hom@", "home@", "@home", "@hom", "~~", "~~~~~",
             "@" * 33, "~" * 65, "a " * 20 + "@", "q" * 15 + "~" + "q" * 16]
    texts += ["".join(rng.choice(atoms) for _ in range(rng.randint(1, 30))) for _ in range(400)]
    return specials, texts


def dense(seed=14):
    """short specials and texts that are nothing but matches: runs of thousands of adjacent specials (32 marks in a bit
    word), "aa" over runs of "a" of every parity (every position a candidate, every other one dropped), prompts of 1..64 KiB
    whose marks cross many 32-word walk trips, and hundreds of prompts of 1..7 bytes (several prompts to a bit word)"""
    rng = random.Random(seed)
    toks = ["aa", "|", "<s>", "</s>", "中", "é|", "[x]"]
    specials = {t: ABOVE + 2000 + k for k, t in enumerate(toks)}
    adjacent = ["|", "<s>", "</s>", "中", "[x]"]          # no special spans the seam of two of these
    texts = ["".join(rng.choice(adjacent) for _ in range(rng.randint(2000, 5000))) for _ in range(4)]
    texts += ["|" * n for n in (31, 32, 33, 64, 1024, 1025, 3000)]
    texts += ["a" * n for n in range(1, 70)] + ["a" * n for n in (1023, 1024, 2047, 2048, 4097)]
    texts += ["b" + "a" * n + "|" for n in (62, 63, 64, 65)]
    for kib in (1, 2, 4, 16, 64):
        parts, n = [], 0
        while n < kib * 1024:
            p = rng.choice(["a" * rng.randint(1, 300), rng.choice(adjacent) * rng.randint(1, 100), "é", "x"])
            parts.append(p)
            n += len(p.encode())
        texts.append("".join(parts))
    texts += ["".join(rng.choice(["a", "|", "aa", "<s>", "x", "é"]) for _ in range(rng.randint(1, 3)))[:7] for _ in range(600)]
    return specials, texts


def overlaps(seed=15):
    """specials that overlap and contain one another, ordered so that the mixed policy (MIXED[k % 3]) makes them ALLOWED,
    ORDINARY, DISALLOWED in turn: a DISALLOWED special inside an ALLOWED one (im_start in <|im_start|>), one straddling two
    adjacent ALLOWED occurrences (|><|), ORDINARY ones inside, around and across ALLOWED ones.  Texts: random strings of
    the specials and their pieces"""
    rng = random.Random(seed)
    toks = ["<|im_start|>", "start|>", "im_start",            # A, O, D: D inside A, O a suffix of A
            "<|im_end|>", "<|im", "|><|",                    # A, O (prefix of A), D across two A
            "end|>x", "x<|im", "<|im_end|>x",                # A, O, D (A a prefix of D)
            "<|", "d|><|i", "zz",                            # A (prefix of A), O across two A, D
            "q|", "<|im_start|><|im_end|>", "|q"]            # A, O (two A back to back), D
    specials = {t: ABOVE + 3000 + k for k, t in enumerate(toks)}
    atoms = toks + ["<", "|", ">", "im", "_", "start", "end", "x", "z", "q", " ", "\n", "é"]
    texts = ["<|im_start|>", "<|im_start|><|im_start|>", "<|im_end|>x", "<|im_start|><|im_end|>", "x<|im_end|>",
             "end|><|im_start|>", "q|q", "zz", "<|<|im", "start|>"]
    texts += ["".join(rng.choice(atoms) for _ in range(rng.randint(1, 24))) for _ in range(600)]
    return specials, texts


class Table:
    """a special set as the reference reads it: bytes -> index, ids, the distinct lengths (longest first), the first bytes"""

    def __init__(self, specials):
        self.names = list(specials)
        self.toks = [t.encode() for t in specials]
        self.ids = [int(v) for v in specials.values()]
        self.index = {t: k for k, t in enumerate(self.toks)}
        self.lens = sorted({len(t) for t in self.toks}, reverse=True)
        self.first = frozenset(t[0] for t in self.toks)


def policy_modes(policy, n):
    """the mode bytes of a policy over n specials (None: tiktoken's default, every special DISALLOWED)"""
    if policy == "default":
        return None
    if policy == "allow_all":
        return np.full(n, ALLOW, np.uint8)
    return np.array([MIXED[k % 3] for k in range(n)], np.uint8)


def cut(T, modes, text: bytes):
    """one prompt: (bad, kept, ambiguous).  bad: the index of the longest DISALLOWED special at the leftmost position that
    holds one, or None; kept: [(start, end, index)] of the ALLOWED occurrences kept -- the leftmost, the longest there, the
    search resuming after it; ambiguous: some position holds two specials (tiktoken's alternation may pick another one)"""
    n, kept, last, ambiguous = len(text), [], 0, False
    if T is None:
        return None, kept, False
    for p in range(n):
        if text[p] not in T.first:
            continue
        allow, hits = None, 0
        for L in T.lens:
            k = T.index.get(text[p:p + L]) if p + L <= n else None
            if k is None:
                continue
            hits += 1
            m = DISALLOW if modes is None else modes[k]
            if m == DISALLOW:
                return k, None, False
            if m == ALLOW and allow is None:
                allow = (p, p + L, k)
        ambiguous = ambiguous or hits > 1
        if allow and p >= last:
            kept.append(allow)
            last = allow[1]
    return None, kept, ambiguous


def reference(tables, modes, prompts, vocab_ids, encoders):
    """What encode_batch_special must return.  tables[v]: Table of vocabulary v (None: no specials); modes[v]: its mode bytes
    (modes or modes[v] None: every special DISALLOWED); encoders[v](bytes) -> the ordinary ids of a text stretch.
    ("bad", prompt, index) for the lowest prompt that holds a DISALLOWED special; else ("ok", ids per prompt, kept per prompt)."""
    ids, kept_all = [], []
    for i, p in enumerate(prompts):
        v = 0 if vocab_ids is None else int(vocab_ids[i])
        bad, kept, _ = cut(tables[v], None if modes is None else modes[v], p)
        if bad is not None:
            return "bad", i, bad
        out, at = [], 0
        for a, b, k in kept:
            out += encoders[v](p[at:a]) + [tables[v].ids[k]]
            at = b
        ids.append(out + encoders[v](p[at:]))
        kept_all.append(kept)
    return "ok", ids, kept_all


def ordinary(enc):
    """encode_ordinary of a text stretch (bytes), cached"""
    cache = {}

    def f(b):
        if b not in cache:
            cache[b] = enc.encode_ordinary(b.decode())
        return cache[b]
    return f


def without_bad(tables, modes, prompts, vocab_ids):
    """the prompts (and their vocabulary ids) that hold no DISALLOWED special"""
    keep = []
    for i, p in enumerate(prompts):
        v = 0 if vocab_ids is None else int(vocab_ids[i])
        if cut(tables[v], None if modes is None else modes[v], p)[0] is None:
            keep.append(i)
    return [prompts[i] for i in keep], None if vocab_ids is None else np.asarray(vocab_ids, np.uint8)[keep]


# slot -> (pattern of its vocabulary, its special set or None, its policy) of a batch over eight vocabularies: slot 5 has no
# specials, slot 6's modes are all ORDINARY (it is left out of first_bytes: its specials stay text)
EIGHT = [(0, "dense", "allow_all"), (1, "one_byte", "mixed"), (2, "all_lengths", "allow_all"), (3, "overlaps", "mixed"),
         (0, "max_table", "allow_all"), (1, None, None), (2, "one_byte", "ordinary"), (3, "all_lengths", "mixed")]


def eight_vocab_batch(sets, seed, n_prompts, max_len=2048):
    """prompts (bytes) whose vocabulary changes on every prompt, each drawn from its slot's set (slot 5: the dense set's
    texts), and their vocabulary ids"""
    rng = random.Random(seed)
    pools = [[t for t in sets[name or "dense"][1] if len(t.encode()) <= max_len] for _, name, _ in EIGHT]
    vid, prompts = [], []
    for _ in range(n_prompts):
        v = rng.choice([s for s in range(8) if not vid or s != vid[-1]])
        vid.append(v)
        prompts.append(rng.choice(pools[v]).encode())
    return prompts, np.array(vid, np.uint8)


def eight_vocab_modes(sets):
    """(mode bytes per slot, Table per slot as the reference sees it: None where no special is looked for)"""
    modes, tabs = [], []
    for _, name, policy in EIGHT:
        if name is None:
            modes.append(None)
            tabs.append(None)
            continue
        n = len(sets[name][0])
        modes.append(np.zeros(n, np.uint8) if policy == "ordinary" else policy_modes(policy, n))
        tabs.append(Table(sets[name][0]) if policy != "ordinary" else None)
    return modes, tabs


def special_set(name):
    """(specials {str: id}, texts) of one of SETS"""
    return globals()[name]()
