"""The device entry points' two promises about the caller's bytes (include/cfbpe.h): d_bytes may sit at any address, and the 32
bytes after the last prompt byte are read but their contents do not matter.  On the CPU SIMT emulator every entry point (split,
encode with and without starts, special in every mode, truncate, chunk in both forms) runs with the batch placed at every
address mod 16, followed by adversarial padding, and against guard pages just past the 32 bytes and just before the first byte;
its results must equal live tiktoken 0.12.0's on the prompt bytes alone (the oracle's split for the piece ends) and, for the
batch moved through every alignment, the default layout's.

The sweeps that can stop the process -- a guard page hit, or a misaligned vector load under the alignment sanitizer
(tests/simt/build.py) -- run in a child process: `python tests/test_buffer_layout_sim.py --child`."""
import base64
import functools
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from conftest import COMBOS, TEKKEN_PATH          # (first: conftest puts tests/simt and the repository root on sys.path)
import fuzzgen
import simlib as S
from oracle import oracle
from test_chunk_sim import reference as chunk_reference
from test_truncate_sim import HEAD, TAIL, reference as truncate_reference

SPECIALS = {"<|endoftext|>": 200000, "<|eot_id|>": 200003}
SPECIAL_SUFFIX = b"text|>"                        # "...<|endof" followed by this padding would read as <|endoftext|>
N_TOK, OVERLAP = 7, 2                             # chunk size and overlap of every chunk call
FILLS = [b"\x00", b"\xff", b"\x80", b"a", b"s", b" ", b"\n", b"0", SPECIAL_SUFFIX,
         bytes(random.Random(5).randrange(256) for _ in range(61))]
FILLER = b"some filler words, then 12 digits: 345678 and more"
CONFIGS = 5                                       # 0..3: one vocabulary, pattern COMBOS[i]; 4: two vocabularies, the last prompt in the second


def endings():
    """last prompts whose end is where a kernel that reads past it would go wrong"""
    rng = random.Random(11)

    def letters(n):
        return "".join(rng.choice("abcdefghijklmnopqrstuvwxyz") for _ in range(n)).encode()
    out = []
    for n in (1, 2, 15, 16, 17, 200):                                   # \s+(?!\S) looks ahead
        out += [b"word" + b" " * n, b"word" + b"\n" * n]
    out += [b"line\r", b"don x'", b"hello worldly", b"SHOUTING LOUDLY"]   # 'x + s: a contraction; the caps run: the W_U fix-up
    out += [b"n " + b"7" * k for k in (1, 2, 3, 4)] + [b"n " + b"1234567890" * 13]        # ascii_digit_run_end
    out += [b"=" * 130, b"x" + b"-" * 300]                                                  # same_byte_run_end
    out += [b" " + letters(n - 1) for n in (12, 13, 16, 17, 32, 33, 257, 4097)]            # one piece of n bytes
    out += ["café".encode(), "文中".encode(), "hi \U0001f600".encode()]                   # a 2-, 3-, 4-byte character last
    out += [b"hi <|endoftext|>", b"hi <|endof"]                                             # a special, a special's prefix
    return out


class Env:
    """the four slots' vocabularies on the emulator, their live tiktoken encodings and the special table"""

    def __init__(self, tekken_bytes, tiktoken):
        from oracle import patterns as PT
        lines = tekken_bytes.splitlines()
        self.vocabs = [S.SimVocab(tekken_bytes, 0, pat, n) for pat, n in COMBOS]
        self.encs = []
        for pat, n in COMBOS:
            ranks = {base64.b64decode(l.split()[0]): i for i, l in enumerate(lines[:n])}
            self.encs.append(tiktoken.Encoding("live%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks, special_tokens=SPECIALS))
        self.specials = S.Specials(SPECIALS)
        self.encode_ordinary = functools.lru_cache(maxsize=None)(lambda slot, p: self.encs[slot].encode_ordinary(p.decode()))

    def config(self, cfg, n):
        """(slot of every prompt, vocabularies of the call, vocab_ids or None)"""
        if cfg < 4:
            return [cfg] * n, [self.vocabs[cfg]], None
        vid = np.array([i % 2 for i in range(n)], np.uint8) if n != 2 else np.array([0, 1], np.uint8)
        return [(0, 3)[v] for v in vid], [self.vocabs[0], self.vocabs[3]], vid


def call_modes(m, n_vocabs):
    """per-vocabulary special modes of a call: vocabulary k uses mode (m + k) % 3 for every special"""
    return [np.full(len(SPECIALS), (m + k) % 3, np.uint8) for k in range(n_vocabs)]


def call_all(env, cfg, prompts, budgets, variant=None):
    """every emulator entry point on one batch, in the current layout: {entry: result as plain lists}.  variant k (0..7) takes
    one form of each of encode (with or without starts), truncate (HEAD, TAIL) and chunk (host, device form); None: all forms"""
    slots, vs, vid = env.config(cfg, len(prompts))
    forms = [(k & 1, (k >> 1) & 1, (k >> 2) & 1) for k in (range(8) if variant is None else [variant])]
    r = {"split": S.split([v.pattern_id for v in vs], prompts, vid)}
    if any(f[0] == 0 for f in forms):
        rc, ids, off, counts, _ = S.encode_batch(vs, prompts, vid)
        r["encode"] = (rc,) + ((ids[:int(off[-1])].tolist(), off.tolist(), counts.tolist()) if rc == 0 else ())
    if any(f[0] == 1 for f in forms):
        rc, ids, starts, off, counts = S.encode_starts(vs, prompts, vid)
        r["starts"] = (rc,) + ((ids.tolist(), starts.tolist(), off.tolist(), counts.tolist()) if rc == 0 else ())
    for m in (S.ORDINARY, S.ALLOW, S.DISALLOW):
        rc, got, counts, bad, _, _ = S.encode_batch_special(vs, [env.specials] * len(vs), prompts, call_modes(m, len(vs)), vid,
                                                            max_prompts=4 * len(prompts) + 8)
        r["special", m] = (rc, got, counts if rc == 0 else None, bad if rc == S.EBADMSG else None)
    for mode in sorted({f[1] for f in forms}):
        rc, cut, kept, counts = S.truncate(vs, prompts, budgets, mode, vid)
        r["truncate", mode] = (rc,) + ((cut.tolist(), kept.tolist(), counts.tolist()) if rc == 0 else ())
    for form in sorted({f[2] for f in forms}):
        rc, spans, coffs, counts = S.chunk(vs, prompts, N_TOK, OVERLAP, vid, device_form=bool(form))
        r["chunk", form] = (rc,) + ((spans[:int(coffs[-1])].tolist(), coffs.tolist(), counts.tolist()) if rc == 0 else ())
    return r


def special_reference(env, slot, m, p):
    """(ids, or None when a disallowed special occurs, the index of the leftmost such special) by tiktoken's rules"""
    t = p.decode()
    if m == S.ALLOW:
        return env.encs[slot].encode(t, allowed_special="all"), None
    if m == S.DISALLOW:
        found = [(t.find(k), i) for i, k in enumerate(SPECIALS) if k in t]
        if found:
            return None, min(found)[1]
    return env.encode_ordinary(slot, p), None


def check_reference(env, cfg, prompts, budgets, r):
    """the results of call_all equal the oracle's split and live tiktoken on the prompt bytes alone"""
    slots, vs, _ = env.config(cfg, len(prompts))
    want = [env.encode_ordinary(s, p) for s, p in zip(slots, prompts)]
    flat = [t for w in want for t in w]
    counts = [len(w) for w in want]
    assert r["split"] == (0, [oracle.split(COMBOS[s][0], p).tolist() for s, p in zip(slots, prompts)])
    offsets = np.concatenate([[0], np.cumsum(counts)]).tolist()
    if "encode" in r:
        assert r["encode"] == (0, flat, offsets, counts)
    if "starts" in r:
        starts = []
        for s, w in zip(slots, want):
            ln = np.array([len(env.encs[s].decode_single_token_bytes(t)) for t in w], np.int64)
            starts += (np.cumsum(ln) - ln).tolist()
        assert r["starts"] == (0, flat, starts, offsets, counts)
    for m in (S.ORDINARY, S.ALLOW, S.DISALLOW):
        rows = [special_reference(env, s, (m + (0 if len(vs) == 1 else (s == 3))) % 3, p) for s, p in zip(slots, prompts)]
        bad = [(i, b) for i, (_, b) in enumerate(rows) if b is not None]
        rc, got, _, got_bad = r["special", m]
        if bad:
            assert (rc, got_bad) == (S.EBADMSG, bad[0]), m
        else:
            assert (rc, got) == (0, [ids for ids, _ in rows]), m
    for mode in (HEAD, TAIL):
        if ("truncate", mode) in r:
            rows = [truncate_reference(env.encs[s], p, int(b), mode)[:3] for s, p, b in zip(slots, prompts, budgets)]
            assert r["truncate", mode] == (0,) + tuple(list(x) for x in zip(*rows)), mode
    spans, coffs = [], [0]
    for s, p in zip(slots, prompts):
        w, _ = chunk_reference(env.encs[s], p, N_TOK, OVERLAP)
        spans += [list(x) for x in w]
        coffs.append(coffs[-1] + len(w))
    for form in (0, 1):
        if ("chunk", form) in r:
            assert r["chunk", form] == (0, spans, coffs, counts), form


def padding_cases(env):
    """[(cfg, prompts, budgets, fill)]: a filler prompt, then an ending, the filler's length moving the batch end through every
    residue mod 16; every ending meets every residue and every fill; the last prompt's truncate budget is 0, 1, c - 1, c or c + 5"""
    rng = random.Random(7)
    out = []
    for ei, last in enumerate(endings()):
        fills = list(range(len(FILLS)))
        rng.shuffle(fills)
        fills += [rng.randrange(len(FILLS)) for _ in range(16 - len(FILLS))]
        for r in range(16):
            prompts = [FILLER[:4 + (r - 4 - len(last)) % 16], last]
            cfg = (ei + r) % CONFIGS
            c = len(env.encode_ordinary(env.config(cfg, 2)[0][1], last))
            budgets = [3, [0, 1, max(c - 1, 0), c, c + 5][(ei + 3 * r) % 5]]
            out.append((cfg, prompts, budgets, FILLS[fills[r]]))
    return out


def alignment_batch():
    """one mixed batch: fuzz strings, long runs, every ending (one of them last)"""
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(404, 60, max_atoms=30) + fuzzgen.long_runs(4)[:24]] + endings()
    rng = random.Random(9)
    body = prompts[:-1]
    rng.shuffle(body)
    return body + prompts[-1:]


def padding_sweep(env, guard="none"):
    """every padding case with its fill after the batch, one variant of each entry point a case (every variant at every ending):
    the references.  guard "after": exactly 32 bytes of padding, then an unmapped page"""
    for k, (cfg, prompts, budgets, fill) in enumerate(padding_cases(env)):
        with S.batch_layout(0, fill, guard):
            got = call_all(env, cfg, prompts, budgets, variant=k % 8)
        try:
            check_reference(env, cfg, prompts, budgets, got)
        except AssertionError as e:
            raise AssertionError((guard, cfg, fill[:8], len(prompts[0]), prompts[-1][-40:])) from e


def alignment_sweep(env, guard="none"):
    """the mixed batch at every address mod 16, fills and variants rotating, over two vocabularies and over one: the default
    layout's results, which are the references.  guard "before": an unmapped page just before the leading bytes"""
    prompts = alignment_batch()
    budgets = [(i * 7) % 40 for i in range(len(prompts))]
    for cfg in (4, 1):
        want = call_all(env, cfg, prompts, budgets)
        check_reference(env, cfg, prompts, budgets, want)
        for m in range(16):
            fill = FILLS[(m + cfg) % len(FILLS)]
            with S.batch_layout(m, fill, guard):
                got = call_all(env, cfg, prompts, budgets, variant=(m + cfg) % 8)
            for key in got:
                assert got[key] == want[key], (guard, key, cfg, m, fill[:8])


@pytest.fixture(scope="module")
def env(tekken_bytes):
    return Env(tekken_bytes, pytest.importorskip("tiktoken"))


def test_padding_sweep(env):
    padding_sweep(env)


def test_alignment_sweep(env):
    alignment_sweep(env)


def run_end_sweep(guard="none"):
    """K1's bulk run scanners (same_byte_run_end, ascii_digit_run_end), which load whole 16-byte groups once aligned, against a
    plain scan: at every address mod 16 and every run length around the 16- and 128-byte loops, with the bytes past pe
    continuing the run (the padding, or the next prompt), the end is pe, or the first byte in [pos, pe) that breaks the run"""
    for byte in (ord(" "), ord("\n"), None):
        c = b"7" if byte is None else bytes([byte])
        for m in range(16):
            for n in (1, 15, 16, 17, 127, 128, 129, 143, 300):
                for pos in (0, 9):
                    if pos >= n:
                        continue
                    data = b"x" * pos + c * (n - pos)
                    k = pos + (n - pos) // 2
                    with S.batch_layout(m, c, guard):
                        assert S.run_end(data, pos, n, byte) == n, (c, m, n, pos)
                        assert S.run_end(data + c * 40, pos, n, byte) == n, (c, m, n, pos)
                        assert S.run_end(data[:k] + b"y" + data[k + 1:], pos, n, byte) == k, (c, m, n, pos)


def test_run_scanners_stop_at_the_prompt_end():
    run_end_sweep()


def continued_runs():
    """(prompt, next prompt) pairs where the next prompt's first bytes continue the run that ends the prompt: the bytes a kernel
    reads past a prompt's end are another prompt's text, as in a window of a resident corpus or in a pipelined lane"""
    return [(b"n " + b"7" * 200, b"7" * 40), (b"n " + b"1234567890" * 13, b"1234567890" * 5 + b" x"), (b"n " + b"0" * 17, b"0" * 20),
            (b"x" + b" " * 150, b"     y"), (b"x" + b"\n" * 150, b"\n\n\n\n y"), (b"y" + b" " * 130, b" " * 40 + b"z"),
            (b"w" + b"\t" * 140, b"\t" * 30 + b"!")]


def test_runs_that_continue_into_the_next_prompt(env):
    """a whitespace or digit run at a prompt's end that the next prompt continues, the prompt's end at every residue mod 16: the
    bulk run scanners (same_byte_run_end, ascii_digit_run_end) stop at the prompt's end, so the next prompt is split on its own"""
    for i, (run, nxt) in enumerate(continued_runs()):
        for r in range(16):
            prompts = [FILLER[:4 + (r - 4 - len(run)) % 16], run, nxt]
            cfg, budgets = (i + r) % CONFIGS, [1, 2, 3]
            got = call_all(env, cfg, prompts, budgets, variant=(i + r) % 8)
            try:
                check_reference(env, cfg, prompts, budgets, got)
            except AssertionError as e:
                raise AssertionError((cfg, r, run[-8:], nxt[:8])) from e


def test_utf8_at_the_end_is_judged_on_the_prompt_bytes(env):
    """a last prompt ending in the first two bytes of a 3-byte character is malformed even when the padding completes it; a
    valid last prompt followed by continuation bytes is not"""
    for cfg in range(CONFIGS):
        for last, fill, bad in ((b"ok \xe4\xb8", b"\xad", True), (b"ok \xe4\xb8\xad", b"\x80", False), (b"ok", b"\x80\xbf", False)):
            prompts = [b"a prompt", last]
            for m in (0, 7, 15):
                with S.batch_layout(m, fill):
                    r = call_all(env, cfg, prompts, [2, 1])
                rcs = {key: v[0] for key, v in r.items()}
                want = S.EILSEQ if bad else 0
                assert rcs == {key: want for key in rcs}, (cfg, last, m)


def test_layout_setter_refuses_bad_layouts():
    assert S.lib().sim_batch_layout(16, b"\0", 1, 0) == S.EINVAL
    assert S.lib().sim_batch_layout(0, b"", 0, 0) == S.EINVAL
    assert S.lib().sim_batch_layout(0, b"\0", 1, 3) == S.EINVAL


def test_guard_pages_and_alignment_sanitizer_in_a_child():
    """the sweeps against guard pages and under the alignment sanitizer, in a child process (a hit stops it)"""
    pytest.importorskip("tiktoken")
    import build as simt_build
    simt_build.build(sanitize=True)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=dict(os.environ, **{S.SANITIZE_ENV: "1"}),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, "child exit %d\n--- stdout\n%s\n--- stderr\n%s" % (r.returncode, r.stdout[-3000:], r.stderr[-6000:])
    assert "child: ok" in r.stdout


if __name__ == "__main__" and sys.argv[1:] == ["--child"]:
    assert os.environ.get(S.SANITIZE_ENV) == "1"
    import tiktoken
    with open(TEKKEN_PATH, "rb") as f:
        child_env = Env(f.read(), tiktoken)
    alignment_sweep(child_env, "before")
    padding_sweep(child_env, "after")
    run_end_sweep("after")
    print("child: ok")
