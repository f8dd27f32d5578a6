"""Seeded rank files shaped like real ones where the Tekken stand-in and synth_vocab.py are not (test infrastructure).

Real rank files (cl100k_base, o200k_base, Llama 3) differ from the stand-in in ways the kernels have branches for: single
bytes at scattered ranks, tokens of up to 255 bytes, more than 2^20 ranks, random rank orders over multi-byte UTF-8.  Each
shape below returns (rank_file_bytes, texts): a rank file in the tiktoken format and prompts built to reach the code path the
shape is about.  Everything is seeded; the big vocabularies are built once per process (cached)."""
import base64
import functools
import itertools
import random

K_MAX_RANK = (1 << 21) - 2          # vocab.cpp: kMaxRank, the most ranks a vocabulary may have
K_LIST_MAX_RANK = (1 << 20) - 1     # bpe_kernels.cuh: kListMaxRank, bpe_list_kernel's limit (rank << 12 in 32 bits)
THRESHOLDS = (12, 13, 32, 33, 256, 257, 4096, 4097)   # kShortMaxLen, K2a / K2b, kBigPiece / kMedSmem, kDeferMaxParts
SHAPES = ("scattered_bytes", "long_tokens", "runs_to_255", "over_2_20", "utf8_random", "thresholds")
UTF8_ALPHABET = "aé中😀 '\n1"


def rank_file(tokens) -> bytes:
    """the tiktoken format: '<base64> <rank>' a line, rank = position in tokens"""
    return b"".join(base64.b64encode(t) + b" %d\n" % i for i, t in enumerate(tokens))


def tokens_of(rf: bytes):
    return [base64.b64decode(l.split()[0]) for l in rf.splitlines() if l.strip()]


def _add(seen, out, t):
    if t and t not in seen:
        seen.add(t)
        out.append(t)
        return True
    return False


def _with_bytes_scattered(rng, tokens):
    """the 256 single bytes (those not already tokens) shuffled in among the tokens: merged tokens rank below some bytes"""
    have = set(tokens)
    out = list(tokens) + [bytes([b]) for b in range(256) if bytes([b]) not in have]
    rng.shuffle(out)
    return out


def scattered_bytes(seed=1):
    """cl100k-like: the bytes permuted among ~3000 merged tokens (ASCII words, spaces, and the UTF-8 of é / 中 / 😀 with pieces
    of them), so byte2id and the bytepair index hold ids that are not the byte values"""
    rng = random.Random(seed)
    alpha = [c.encode() for c in "etaoin shrdlu"] + ["é".encode(), "中".encode(), "😀".encode(), b"\xe4\xb8", b"\x9f\x98"]
    seen, toks = set(), []
    while len(toks) < 3000:
        t = b"".join(rng.choice(alpha) for _ in range(rng.randint(1, 4)))
        _add(seen, toks, t[:rng.randint(2, 8)])
    toks = _with_bytes_scattered(rng, toks)
    chars = "etaoin shrdlu" * 3 + "é中😀.,\n'"
    texts = ["".join(rng.choice(chars) for _ in range(rng.randint(0, 200))) for _ in range(1200)]
    texts += ["".join(rng.choice(chars) for _ in range(n)) for n in (300, 700, 1500, 5000)]
    return rank_file(toks), texts


def _collision_family(rng, n, count, alpha=b"ab"):
    """count tokens of n bytes with the same first 12 bytes and last 4 bytes: long_hash sees only those and the length, so
    all of them land on one hash and only the byte comparison tells them apart"""
    head = bytes(rng.choice(alpha) for _ in range(12))
    tail = bytes(rng.choice(alpha) for _ in range(4))
    fam = set()
    while len(fam) < count:
        fam.add(head + bytes(rng.choice(alpha) for _ in range(n - 16)) + tail)
    return sorted(fam)


def long_tokens(seed=2):
    """tokens of every length 2..255 over 'ab' (most longer ones unreachable by any merge: only the whole-piece lookup finds
    them), plus hash-collision families; texts: every long token alone (and after a space), family members that are not
    tokens, and random 'ab' words"""
    rng = random.Random(seed)
    seen, toks = set(), []
    for n in range(2, 256):
        k = 0
        while k < min(6 if n <= 40 else 2, 2 ** n):
            k += _add(seen, toks, bytes(rng.choice(b"ab") for _ in range(n)))
    misses = []
    for n in (20, 21, 40, 79, 100, 128, 200, 254, 255):
        fam = _collision_family(rng, n, 12)
        for t in fam[:8]:
            _add(seen, toks, t)
        misses += [t for t in fam[8:] if t not in seen]          # same hash as eight tokens, not a token
    while len(toks) < 2000:
        _add(seen, toks, bytes(rng.choice(b"ab") for _ in range(rng.randint(2, 12))))
    toks = _with_bytes_scattered(rng, toks)
    longs = [t for t in toks if len(t) > 12]
    texts = [t.decode() for t in longs] + [" " + t.decode() for t in longs[::3]] + [t.decode() for t in misses]
    texts += ["".join(rng.choice("ab") for _ in range(rng.randint(1, 600))) for _ in range(400)]
    texts += [" ".join(rng.choice(longs).decode() for _ in range(rng.randint(2, 6))) for _ in range(100)]
    return rank_file(toks), texts


def runs_to_255(seed=3):
    """'a' * k and ' ' + 'a' * k for every length k up to 255 bytes, in merge order: BPE reaches every one of them by merges
    (the longest through pairs of long tokens); texts: every run length up to 700"""
    toks = [bytes([b]) for b in range(256)] + [b"a" * k for k in range(2, 256)] + [b" " + b"a" * k for k in range(1, 255)]
    texts = ["a" * k for k in range(1, 701)] + [" " + "a" * k for k in range(1, 701)] + ["b" + "a" * k + " a" for k in range(250, 260)]
    return rank_file(toks), texts


@functools.lru_cache(maxsize=1)
def _big_tokens(seed=4):
    """every string of 2..7 letters over 'abcdefgh' (2 396 736), shuffled: more than kMaxRank of them"""
    rng = random.Random(seed)
    toks = [bytes(t) for n in range(2, 8) for t in itertools.product(b"abcdefgh", repeat=n)]
    rng.shuffle(toks)
    return toks


def big_rank_file(n_ranks: int) -> bytes:
    """the 256 bytes, then the shuffled letter strings, n_ranks in all (up to kMaxRank + 1)"""
    return rank_file([bytes([b]) for b in range(256)] + _big_tokens()[:n_ranks - 256])


def top_ranks(n_ranks: int, count: int):
    """[(id, token bytes)] of the count highest ranks of big_rank_file(n_ranks)"""
    return [(r, _big_tokens()[r - 256]) for r in range(n_ranks - 1, n_ranks - 1 - count, -1)]


@functools.lru_cache(maxsize=1)
def over_2_20(seed=5):
    """2^20 + 2^19 ranks: bpe_list_kernel stays out (kListMaxRank), pieces of 257..4096 bytes take bpe_long_kernel's
    global-memory path, and a third of the merges have ids >= 2^20 (in every packed key); texts: letter words of every size
    class, and periodic ones (batched rounds)"""
    rng = random.Random(seed)
    rf = big_rank_file((1 << 20) + (1 << 19))
    texts = []
    for n in (1, 2, 5, 7, 8, 13, 30, 33, 100, 256, 257, 300, 1000, 2500, 4096, 4097, 6000):
        for _ in range(6 if n < 1000 else 3):
            texts.append("".join(rng.choice("abcdefgh") for _ in range(n)))
    texts += [" ".join("".join(rng.choice("abcdefgh") for _ in range(rng.randint(1, 12))) for _ in range(rng.randint(1, 40)))
              for _ in range(300)]
    texts += [("".join(rng.choice("abcdefgh") for _ in range(rng.randint(1, 4)))) * rng.choice([20, 70, 200, 1200])
              for _ in range(40)]
    return rf, texts


def utf8_random(seed=6):
    """random ranks over the UTF-8 of 'aé中😀 \\'\\n1': tokens that are parts of characters, tokens that span characters,
    tokens no merge reaches, bytes scattered; texts over the same alphabet, some of them long single pieces"""
    rng = random.Random(seed)
    ab = [c.encode() for c in UTF8_ALPHABET]
    seen, toks = set(), []
    while len(toks) < 2500:
        t = b"".join(rng.choice(ab) for _ in range(rng.randint(1, 5)))
        if rng.random() < 0.3:
            t = t[rng.randint(0, 2):]                       # starts inside a character
        if rng.random() < 0.3:
            t = t[:len(t) - rng.randint(0, 2)]              # ends inside one
        _add(seen, toks, t)
    toks = _with_bytes_scattered(rng, toks)
    texts = ["".join(rng.choice(UTF8_ALPHABET) for _ in range(rng.randint(0, 300))) for _ in range(1200)]
    texts += ["".join(rng.choice("aé中😀") for _ in range(n)) for n in (40, 70, 90, 200, 1100)]   # letters: one piece each
    texts += ["中" * n for n in (11, 86, 1366)] + ["😀" * n for n in (8, 64, 65, 1024)]
    return rank_file(toks), texts


def thresholds(seed=7):
    """tokens and pieces of every length on either side of the kernels' thresholds (THRESHOLDS, and 254 / 255, the longest
    token): each token length once as a whole piece and once as a miss of the same length"""
    rng = random.Random(seed)
    seen, toks = set(), []
    while len(toks) < 600:
        _add(seen, toks, bytes(rng.choice(b"xyz") for _ in range(rng.randint(2, 7))))
    present = []
    for n in (11, 12, 13, 14, 31, 32, 33, 34, 254, 255):
        k = 0
        while k < 3:
            t = bytes(rng.choice(b"xyz") for _ in range(n))
            if _add(seen, toks, t):
                present.append(t)
                k += 1
    toks = _with_bytes_scattered(rng, toks)
    texts = []
    for t in present:
        texts.append(t.decode())
        i = rng.randrange(len(t))
        miss = t[:i] + (b"x" if t[i] != ord("x") else b"y") + t[i + 1:]
        if miss not in seen:
            texts.append(miss.decode())
    for n in THRESHOLDS + (254, 255):
        for _ in range(4):
            texts.append("".join(rng.choice("xyz") for _ in range(n)))
        texts.append("x" * n)
        texts.append(("xyz" * n)[:n])
        texts.append(" " * (n - 1) + "x")              # a whitespace piece of n - 1 bytes, then a one-letter word
    texts.append(" ".join(texts[:40]))
    return rank_file(toks), texts


def shape(name):
    """(rank_file_bytes, texts) of one of SHAPES"""
    return globals()[name]()
