"""Synthetic prompt batches for BASELINE.json's five configurations (SURVEY.md section 8(d)).

There is no network and no text corpus on the box, and /root/reference is not on the GPU box,
so prompts are drawn from corpora assembled from what ships with the image, deterministically:

  english       CPython's own documentation strings (`pydoc_data.topics`, ~0.5 MB of technical English)
  code          CPython standard-library sources (argparse.py, typing.py, ...)
  multilingual  pseudo-sentences of real words: the vocabulary's own whole-word tokens in Cyrillic,
                Greek, Arabic, Hebrew, Devanagari, Thai, Hangul, Kana and CJK, joined the way each script
                joins words, sprinkled with that script's punctuation
  digits/ws     numbers, tables, indentation runs
  adversarial   single-character runs and long random "words" (one piece per prompt: the worst case of
                the merge loop, SURVEY.md H3)

Mix (by prompt): 80 % english(+code 1:4), 10 % multilingual, 5 % digits/whitespace, 5 % adversarial.
Prompts are UTF-8-boundary-snapped slices; generator = numpy PCG64 with the seed SURVEY.md names.
"""
from __future__ import annotations

import base64
import hashlib
import os
import sysconfig
import unicodedata

import numpy as np

from . import vocabs as V

_SCRIPTS = ["CYRILLIC", "GREEK", "ARABIC", "HEBREW", "DEVANAGARI", "THAI", "HANGUL", "HIRAGANA", "KATAKANA", "CJK"]
_SPACELESS = {"THAI", "HIRAGANA", "KATAKANA", "CJK"}
_PUNCT = {"CJK": ["，", "。", "、", "？"], "HIRAGANA": ["、", "。"], "KATAKANA": ["・", "。"],
          "ARABIC": ["،", "."], "default": [",", ".", ";", "?", "!"]}

_cache = {}


def _english() -> bytes:
    import pydoc_data.topics as T
    return "\n\n".join(T.topics[k] for k in sorted(T.topics)).encode("utf-8")


def _code() -> bytes:
    std = sysconfig.get_paths()["stdlib"]
    out = []
    for name in ["argparse.py", "typing.py", "dataclasses.py", "json/decoder.py", "textwrap.py", "heapq.py", "bisect.py"]:
        p = os.path.join(std, name)
        if os.path.exists(p):
            with open(p, "rb") as f:
                out.append(f.read())
    return b"\n".join(out)


def _script_of(word: str):
    s = None
    for ch in word:
        if not ch.isalpha():
            return None
        try:
            nm = unicodedata.name(ch)
        except ValueError:
            return None
        sc = next((x for x in _SCRIPTS if nm.startswith(x)), None)
        if sc is None or (s is not None and sc != s):
            return None
        s = sc
    return s


def _multilingual(seed: int, target_bytes: int = 1 << 20) -> bytes:
    words = {s: [] for s in _SCRIPTS}
    with open(V.TEKKEN_FILE, "rb") as f:
        for line in f:
            tok = base64.b64decode(line.split()[0])
            if len(tok) < 4:
                continue
            try:
                w = tok.decode("utf-8")
            except UnicodeDecodeError:
                continue
            w = w.lstrip(" ")
            sc = _script_of(w) if w else None
            if sc:
                words[sc].append(w)
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    size = 0
    scripts = [s for s in _SCRIPTS if len(words[s]) >= 20]
    while size < target_bytes:
        sc = scripts[int(rng.integers(len(scripts)))]
        ws = words[sc]
        n = int(rng.integers(4, 24))
        sep = "" if sc in _SPACELESS else " "
        sent = sep.join(ws[int(i)] for i in rng.integers(len(ws), size=n))
        p = _PUNCT.get(sc, _PUNCT["default"])
        sent += p[int(rng.integers(len(p)))] + ("\n" if rng.random() < 0.15 else " ")
        b = sent.encode("utf-8")
        out.append(b)
        size += len(b)
    return b"".join(out)


def _digits_ws(seed: int, target_bytes: int = 1 << 19) -> bytes:
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    size = 0
    while size < target_bytes:
        k = int(rng.integers(5))
        if k == 0:
            s = " ".join(str(int(x)) for x in rng.integers(0, 10 ** int(rng.integers(1, 12)), size=8)) + "\n"
        elif k == 1:
            s = " " * int(rng.integers(1, 24)) + "x = %d;\n" % int(rng.integers(1 << 30))
        elif k == 2:
            s = "\t".join("%.4f" % x for x in rng.random(6)) + "\r\n"
        elif k == 3:
            s = "\n" * int(rng.integers(1, 5)) + "  - item %d:  %s\n" % (int(rng.integers(1000)), "=" * int(rng.integers(1, 20)))
        else:
            v = [int(x) for x in rng.integers(1, 28, size=5)]
            s = "2026-%02d-%02dT%02d:%02d:%02dZ 0x%08x %d%%\n" % (v[0] % 12 + 1, v[1], v[2] % 24, v[3], v[4], int(rng.integers(1 << 31)), int(rng.integers(101)))
        b = s.encode()
        out.append(b)
        size += len(b)
    return b"".join(out)


def corpora(seed: int):
    key = ("corpora", seed)
    if key not in _cache:
        _cache[key] = {
            "english": _english(), "code": _code(),
            "multilingual": _multilingual(seed * 7919 + 1), "digits_ws": _digits_ws(seed * 7919 + 2),
        }
    return _cache[key]


def _snap_tables(buf: np.ndarray):
    """next_start[i]: first char start >= i ; prev_start[i]: last char start <= i (i in 0..n)"""
    n = len(buf)
    is_start = np.ones(n + 1, dtype=bool)
    is_start[:n] = (buf & 0xC0) != 0x80
    idx = np.arange(n + 1, dtype=np.int64)
    prev_start = np.maximum.accumulate(np.where(is_start, idx, 0))
    nxt = np.where(is_start, idx, n)
    next_start = np.minimum.accumulate(nxt[::-1])[::-1]
    return next_start, prev_start


def _slices(buf: bytes, lengths: np.ndarray, rng) -> list:
    a = np.frombuffer(buf, dtype=np.uint8)
    n = len(a)
    ns, ps = _snap_tables(a)
    starts = rng.integers(0, max(n - 1, 1), size=len(lengths))
    out = []
    for s0, ln in zip(starts, lengths):
        s = int(ns[int(s0)])
        e = int(ps[min(s + int(ln), n)])
        if e <= s:
            s = 0
            e = int(ps[min(int(ln), n)])
        out.append(a[s:e])
    return out


def _adversarial(lengths: np.ndarray, rng) -> list:
    letters = np.frombuffer(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ", dtype=np.uint8)
    out = []
    for ln in lengths:
        ln = int(ln)
        k = int(rng.integers(4))
        if k == 0:      # one repeated character
            ch = b"a !\n0"[int(rng.integers(5))]
            out.append(np.full(ln, ch, dtype=np.uint8))
        elif k == 1:    # one long random "word"
            out.append(letters[rng.integers(len(letters), size=ln)])
        elif k == 2:    # short period repeats: abababab...
            per = letters[rng.integers(len(letters), size=int(rng.integers(2, 5)))]
            out.append(np.resize(per, ln))
        else:           # long lowercase word
            out.append(letters[rng.integers(26, size=ln)])
    return out


def make_batch(n_prompts: int, min_len: int, max_len: int, seed: int, mix=(0.80, 0.10, 0.05, 0.05)):
    """returns (bytes uint8, offsets uint64 n+1, meta dict).  Lengths are i.i.d. uniform integers in
    [min_len, max_len] before UTF-8 boundary snapping; meta reports the realised total."""
    rng = np.random.Generator(np.random.PCG64(seed))
    C = corpora(seed)
    lengths = rng.integers(min_len, max_len + 1, size=n_prompts)
    kind = rng.choice(4, size=n_prompts, p=list(mix))
    parts = [None] * n_prompts
    eng = C["english"] + b"\n\n" + C["code"]
    for k, src in ((0, eng), (1, C["multilingual"]), (2, C["digits_ws"])):
        idx = np.nonzero(kind == k)[0]
        if len(idx):
            for i, sl in zip(idx, _slices(src, lengths[idx], rng)):
                parts[i] = sl
    idx = np.nonzero(kind == 3)[0]
    if len(idx):
        for i, sl in zip(idx, _adversarial(lengths[idx], rng)):
            parts[i] = sl
    offs = np.zeros(n_prompts + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(p) for p in parts], dtype=np.uint64)
    data = np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint8)
    meta = {"n_prompts": n_prompts, "total_bytes": int(offs[-1]), "min_len": min_len, "max_len": max_len, "seed": seed,
            "mix": {"english+code": mix[0], "multilingual": mix[1], "digits_ws": mix[2], "adversarial": mix[3]},
            "sha256": hashlib.sha256(data.tobytes()).hexdigest()[:16]}
    return np.ascontiguousarray(data), offs, meta


# BASELINE.json configs -> concrete inputs (SURVEY.md 8(d)); vocab names resolve through cfbpe.vocabs
CONFIGS = {
    1: dict(name="1x512B cl100k", n=1, min_len=512, max_len=512, seed=1, vocabs=["cl100k_base"]),
    2: dict(name="1Kx512B cl100k", n=1024, min_len=512, max_len=512, seed=2, vocabs=["cl100k_base"]),
    3: dict(name="64K mixed 8-4096B cl100k", n=65536, min_len=8, max_len=4096, seed=3, vocabs=["cl100k_base"]),
    4: dict(name="16Kx1KiB o200k", n=16384, min_len=1024, max_len=1024, seed=4, vocabs=["o200k_base"]),
    5: dict(name="256 tenants x 256 prompts, vocab = tenant mod 3", n=65536, min_len=8, max_len=4096, seed=5,
            vocabs=["cl100k_base", "o200k_base", "llama3"], tenants=256),
}


def make_config(cfg_id: int, scale: float = 1.0):
    """(bytes, offsets, vocab_ids or None, meta) of a BASELINE.json config; scale < 1 shrinks n_prompts (tests)."""
    c = CONFIGS[cfg_id]
    n = max(1, int(round(c["n"] * scale)))
    data, offs, meta = make_batch(n, c["min_len"], c["max_len"], c["seed"])
    vid = None
    if "tenants" in c:
        per = max(1, n // c["tenants"])
        tenant = np.minimum(np.arange(n) // per, c["tenants"] - 1)
        vid = (tenant % len(c["vocabs"])).astype(np.uint8)
    meta.update(config=cfg_id, name=c["name"], vocabs=c["vocabs"])
    return data, offs, vid, meta


# ---- text made of a vocabulary's own tokens (make_vocab_text)
#
# The corpora above are a few MB tiled to the batch size, so a full-size batch holds few distinct pieces and looks up a small
# share of the vocabulary.  make_vocab_text builds text from the rank file itself: every token, long letter-only pieces of
# exact lengths, and batches of words drawn uniformly from the whole vocabulary.

VOCAB_TEXT_KINDS = ("tokens", "pieces", "diverse")
TOKEN_VARIANTS = ("alone", "after_space", "doubled", "letter_changed", "letter_after")
PIECE_LENGTHS = (12, 13, 32, 33, 76, 77, 256, 257, 4096, 4097, 9000, 20000)   # either side of the kernels' length thresholds
PIECE_SCRIPTS = ("ASCII",) + tuple(_SCRIPTS)
_LETTERS = b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ"
_SEPARATORS = [b" "] * 6 + [b"\n"] * 2 + [b", ", b". ", b".\n", b"; ", b": ", b" (", b") ", b"-", b"/", b"\t", b"\n\n", b"? ", b"! ",
                                          b" \"", b"\" ", b"'", b" = ", b"_", b"  "]


def vocab_tokens(file_bytes: bytes, max_ranks: int = 0) -> list:
    """the token bytes of ranks 0 .. max_ranks - 1 of a tiktoken rank file (every rank when max_ranks is 0), in rank order"""
    lines = [l for l in file_bytes.splitlines() if l.strip()]
    return [base64.b64decode(l.split()[0]) for l in (lines[:max_ranks] if max_ranks else lines)]


def _utf8(t: bytes):
    try:
        return t.decode("utf-8")
    except UnicodeDecodeError:
        return None


def vocab_words(toks) -> list:
    """the word pool of the diverse batches: every valid-UTF-8 token, stripped, that is not empty, holds no white space and no
    U+FFFD, in rank order, duplicates dropped"""
    out = {}
    for t in toks:
        s = _utf8(t)
        if s is None:
            continue
        s = s.strip()
        if s and not any(c.isspace() for c in s) and "�" not in s:
            out.setdefault(s.encode(), None)
    return list(out)


def letter_words(toks) -> dict:
    """script -> the vocabulary's letter-only words in it, stripped and lower-cased: every character a lower-case, modifier or
    other letter (Ll, Lm, Lo), so that every pattern keeps a run of them in one piece ("ASCII": a-z only)"""
    out = {s: {} for s in PIECE_SCRIPTS}
    for t in toks:
        s = _utf8(t)
        if s is None:
            continue
        w = s.strip().lower()
        if not w or not all(unicodedata.category(c) in ("Ll", "Lm", "Lo") for c in w):
            continue
        sc = "ASCII" if w.isascii() else _script_of(w)
        if sc:
            out[sc].setdefault(w.encode(), None)
    return {s: list(v) for s, v in out.items()}


def _pack(prompts):
    offs = np.zeros(len(prompts) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(p) for p in prompts], dtype=np.uint64)
    data = np.frombuffer(b"".join(prompts), dtype=np.uint8).copy() if prompts else np.zeros(0, np.uint8)
    return data, offs


def _token_prompts(toks, rng, variants):
    """every valid-UTF-8 token under each variant: alone, after a space, doubled, with one ASCII letter changed so that it is
    no token (a miss of the token's length; tokens without an ASCII letter have none), followed by a letter"""
    have = set(toks)
    valid = [t for t in toks if _utf8(t) is not None]
    out = []
    for v in variants:
        if v == "alone":
            out += valid
        elif v == "after_space":
            out += [b" " + t for t in valid]
        elif v == "doubled":
            out += [t + t for t in valid]
        elif v == "letter_after":
            out += [t + bytes([_LETTERS[int(k)]]) for t, k in zip(valid, rng.integers(26, size=len(valid)))]
        elif v == "letter_changed":
            for t in valid:
                pos = [i for i, c in enumerate(t) if c in _LETTERS]
                if not pos:
                    continue
                i = pos[int(rng.integers(len(pos)))]
                for k in rng.permutation(len(_LETTERS)):
                    m = t[:i] + bytes([_LETTERS[int(k)]]) + t[i + 1:]
                    if m not in have:
                        out.append(m)
                        break
        else:
            raise ValueError("unknown token variant %r" % v)
    return out


def _piece_prompts(toks, rng, lengths, per_length, scripts):
    """letter-only words of one script concatenated with no separator into pieces of exactly L bytes, for each of `scripts` with
    20 words or more (a piece is cut at a character boundary and filled up with ASCII letters)"""
    words = letter_words(toks)
    ascii_words = words["ASCII"]
    out = []
    for sc in scripts:
        ws = words[sc]
        if len(ws) < 20:
            continue
        for L in lengths:
            for _ in range(per_length(L)):
                buf = bytearray()
                while len(buf) < L:
                    buf += ws[int(rng.integers(len(ws)))]
                end = L
                while end < len(buf) and (buf[end] & 0xC0) == 0x80:
                    end -= 1
                del buf[end:]
                while len(buf) < L:
                    buf += ascii_words[int(rng.integers(len(ascii_words)))][:L - len(buf)]
                out.append(bytes(buf))
    return out


def _gather(pool: np.ndarray, pool_off: np.ndarray, idx: np.ndarray) -> np.ndarray:
    """the concatenation of the pool entries idx (pool entry k = pool[pool_off[k]:pool_off[k + 1]])"""
    lens = (pool_off[1:] - pool_off[:-1])[idx]
    starts = pool_off[:-1][idx]
    out = np.empty(int(lens.sum()), dtype=np.uint8)
    pos = 0
    for a in range(0, len(idx), 1 << 20):
        ln, st = lens[a:a + (1 << 20)], starts[a:a + (1 << 20)]
        tot = int(ln.sum())
        out[pos:pos + tot] = pool[np.repeat(st - (np.cumsum(ln) - ln), ln) + np.arange(tot)]
        pos += tot
    return out


def _diverse_text(words, rng, target_bytes, glue_share, run_share):
    """words drawn uniformly from `words`, each followed by a separator: a space, line break or punctuation, a digit group, or
    nothing (a share glue_share of them); plus runs of 40..2000 words joined with no separator, about one in 1 / run_share
    words starting one.  Returns at least target_bytes bytes."""
    digits = [(b" " if rng.random() < 0.7 else b"") + str(int(x)).encode() + (b" " if rng.random() < 0.5 else b",")
              for x in rng.integers(0, 10 ** rng.integers(1, 13, size=256))]
    seps = [b""] + _SEPARATORS + digits
    pool_words, off_words = _pack(words)
    pool_seps, off_seps = _pack(seps)
    pool = np.concatenate([pool_words, pool_seps])
    pool_off = np.concatenate([off_words, off_seps[1:] + off_words[-1]]).astype(np.int64)
    n = int(target_bytes / float(np.diff(off_words).mean()) * 1.05) + 64     # enough without the separators, almost always
    idx = np.empty(2 * n, dtype=np.int64)
    idx[0::2] = rng.integers(len(words), size=n)
    kind = rng.random(n)
    sep = np.where(kind < glue_share, 0, np.where(kind < glue_share + 0.05, 1 + len(_SEPARATORS) + rng.integers(len(digits), size=n),
                                                   1 + rng.integers(len(_SEPARATORS), size=n)))
    runs = np.nonzero(rng.random(n) < run_share)[0]
    run_len = rng.integers(40, 2001, size=len(runs))
    for r, k in zip(runs, run_len):
        sep[r:r + k - 1] = 0
    idx[1::2] = len(words) + sep
    text = _gather(pool, pool_off, idx)
    item_at = np.zeros(2 * n + 1, dtype=np.int64)         # item j of idx is text[item_at[j]:item_at[j + 1]]
    np.cumsum((pool_off[1:] - pool_off[:-1])[idx], out=item_at[1:])
    # lower-case the ASCII letters of each run, so that its letter words stay one piece under the patterns that split at a
    # change of case (the punctuation, digits and other scripts among its words still split it)
    for r, k in zip(runs, run_len):
        seg = text[int(item_at[2 * r]):int(item_at[min(2 * (r + k) - 1, 2 * n)])]
        seg[(seg >= 65) & (seg <= 90)] += 32
    if len(text) < target_bytes:
        text = np.concatenate([text, _diverse_text(words, rng, target_bytes - len(text), glue_share, run_share)])
    return text


def make_vocab_text(file_bytes: bytes, max_ranks: int, seed: int, kind: str, variants=TOKEN_VARIANTS, lengths=PIECE_LENGTHS,
                    per_length=lambda L: 4 if L <= 257 else 1, scripts=PIECE_SCRIPTS, n_prompts=65536, min_len=8, max_len=4096, distinct=0,
                    glue_share=0.08, run_share=2e-4):
    """(bytes uint8, offsets uint64 n+1) of text made of the tokens of ranks 0 .. max_ranks - 1 of a tiktoken rank file, seeded.

      "tokens"   every token that is valid UTF-8 as its own prompt, once per variant of TOKEN_VARIANTS named in `variants`
      "pieces"   letter-only words of one script concatenated into single pieces of exactly L bytes: for each script of
                 `scripts` (PIECE_SCRIPTS names them all) and L of `lengths`, per_length(L) pieces
      "diverse"  n_prompts prompts of min_len..max_len bytes (lengths drawn uniformly, cuts at character boundaries) cut from one
                 text of words drawn uniformly from the vocab_words pool (its first `distinct` words when distinct > 0),
                 joined by spaces, line breaks, punctuation and digit groups, with a share of separator-free runs
    """
    toks = vocab_tokens(file_bytes, max_ranks)
    rng = np.random.Generator(np.random.PCG64(seed))
    if kind == "tokens":
        return _pack(_token_prompts(toks, rng, variants))
    if kind == "pieces":
        return _pack(_piece_prompts(toks, rng, lengths, per_length, scripts))
    if kind != "diverse":
        raise ValueError("kind must be one of %s" % (VOCAB_TEXT_KINDS,))
    words = vocab_words(toks)
    if distinct:
        words = words[:distinct]
    if max_len - min_len < 6:
        raise ValueError("max_len must exceed min_len by 6 bytes or more")
    # each cut moves forward by 0..3 bytes to the next character boundary, so a prompt is its drawn length -3..+3 bytes
    lens = rng.integers(min_len + 3, max_len - 2, size=n_prompts)
    text = _diverse_text(words, rng, int(lens.sum()) + 4, glue_share, run_share)
    cut = np.cumsum(lens)
    for _ in range(3):
        cut += (text[cut] & 0xC0) == 0x80
    offs = np.zeros(n_prompts + 1, dtype=np.uint64)
    offs[1:] = cut
    return np.ascontiguousarray(text[:int(offs[-1])]), offs
