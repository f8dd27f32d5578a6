"""Every kind of call after every other on one lane, and the status a device call leaves for cfbpe_device_status.

A context with n_workspaces = 1 runs every call on one lane: host calls, device calls and decode share its workspace, its byte and
id buffers and its status word, and several calls reuse each other's scratch (special and decode use ids_by_pos, lossy puts the
repaired bytes in the lane's byte buffer, chunk rewrites the status's token count).  Each kind of call here is checked, bit for
bit, against a reference built without the library, right after every other kind and along a seeded random walk:
  ids          the C oracle's ranks plus the slot's id base
  byte starts  cumulative token lengths from the rank file
  unit starts, truncate cuts, chunk spans   the host contracts of cfbpe.plugin applied to those starts
  lossy        repair_utf8, then the oracle;   special   the leftmost-longest host cut (special_sets.cut), then the oracle
  decode       the token bytes
The status tests check that cfbpe_device_status reports the calling thread's last device call on that context, whatever ran on
the lane, on other contexts or on other threads since."""
import os
import random
import threading

import numpy as np
import pytest

import fuzzgen
import special_sets as SS
from conftest import pack

pytestmark = pytest.mark.gpu

TEK_BASE = 1000
SLOTS = [(0, 100256, 0), (3, 130072, TEK_BASE), (1, 150000, 0)]   # (pattern, ranks, id base): cl100k, Tekken, o200k stand-ins
O200K_SPECIALS = {"<|endoftext|>": 199999, "<|endofprompt|>": 200018, "<|im_start|>": 200264, "<|im_end|>": 200265}
SENTINEL = 0xFFFFFFFF          # fills every output buffer: what a call must leave past its results
TAIL = 16                      # entries of room past the results
CHUNKS = [(7, 0), (16, 5)]     # (N, S) of the chunk kinds


def _load(c, tekken_bytes, controls):
    from cfbpe import _native as N
    for slot, (pat, n, base) in enumerate(SLOTS):
        c.vocab_load(slot, tekken_bytes, N.FORMAT_TIKTOKEN, pat, n)
        if base:
            c.vocab_set_id_base(slot, base)
    c.vocab_set_specials(1, controls)
    c.vocab_set_specials(2, O200K_SPECIALS)
    return c


@pytest.fixture(scope="module")
def controls():
    from cfbpe import vocabs as V
    return V.control_tokens(V.SPECS["mistral_tekken"])


@pytest.fixture(scope="module")
def ctx(tekken_bytes, controls):
    """one lane; small sub-batches, so that a host call on the big batch pipelines and one on the small batch runs in one pass"""
    from cfbpe import _native as N
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("CFBPE_PIPE_CHUNK_BYTES", str(192 << 10))
        mp.setenv("CFBPE_PIPE_MIN_BYTES", str(1 << 20))
        c = N.Context(0, max_batch_bytes=16 << 20, max_prompts=1 << 14, n_workspaces=1)
    yield _load(c, tekken_bytes, controls)
    c.close()


@pytest.fixture(scope="module")
def plain_ctx(tekken_bytes, controls):
    """one lane, default pipelining: every host call on the batches of the status tests runs in one pass"""
    from cfbpe import _native as N
    c = N.Context(0, max_batch_bytes=16 << 20, max_prompts=1 << 14, n_workspaces=1)
    yield _load(c, tekken_bytes, controls)
    c.close()


# ---------------------------------------------------------------------------------------------------------------------------
# batches
# ---------------------------------------------------------------------------------------------------------------------------
class Batch:
    def __init__(self, prompts, vid, budgets=None):
        self.prompts, self.vid = list(prompts), np.asarray(vid, np.uint8)
        self.data, self.offs = pack(self.prompts)
        self.n, self.total = len(self.prompts), int(self.offs[-1])
        self.budgets = budgets
        self._dev = None

    def dev(self):
        """the batch in device memory (bytes padded by 64), cached"""
        import torch
        if self._dev is None:
            d = torch.device("cuda:0")
            b = torch.zeros(self.total + 64, dtype=torch.uint8, device=d)
            if self.total:
                b[:self.total] = torch.from_numpy(self.data).to(d)
            self._dev = (b, torch.from_numpy(self.offs.astype(np.int64)).to(d), torch.from_numpy(self.vid.copy()).to(d),
                         torch.from_numpy(self.budgets.astype(np.int32)).to(d) if self.budgets is not None else None)
        return self._dev


def _char_cut(p: bytes, rng):
    """a character boundary of p, drawn"""
    cuts = [i for i in range(len(p) + 1) if i == len(p) or p[i] & 0xC0 != 0x80]
    return rng.choice(cuts)


def _family(prompts, vid, seed, specials):
    """clean, one malformed byte, specials spelled in: Batches over the same prompts and vocabularies"""
    rng = random.Random(seed)
    k = max(range(len(prompts)), key=lambda i: len(prompts[i]))
    bad = list(prompts)
    at = _char_cut(bad[k], rng)
    bad[k] = bad[k][:at] + b"\xff" + bad[k][at:]
    spec = []
    for p, v in zip(prompts, vid):
        toks = specials[int(v)]
        if toks and (len(prompts) == 1 or rng.random() < 0.5):
            for _ in range(rng.randint(1, 3)):
                at = _char_cut(p, rng)
                p = p[:at] + rng.choice(toks).encode() + p[at:]
        spec.append(p)
    budgets = np.array([rng.choice([0, 1, 2, 3, 5, 17, 64, 1 << 20]) for _ in prompts], np.uint32)
    return {"clean": Batch(prompts, vid, budgets), "bad": Batch(bad, vid), "spec": Batch(spec, vid)}


@pytest.fixture(scope="module")
def fams(controls):
    from cfbpe import workload as W
    specials = [[], list(controls)[:40] + ["<s>", "[INST]", "[/INST]"], list(O200K_SPECIALS)]
    rng = np.random.default_rng(5)
    ml, mo, _ = W.make_batch(60, 8, 900, seed=21)
    multi = [bytes(ml[int(mo[i]):int(mo[i + 1])]) for i in range(len(mo) - 1)]
    small = [s.encode() for s in fuzzgen.fuzz_strings(31, 220, max_atoms=40)] + [s.encode() for s in fuzzgen.long_runs(3)[::5]] + multi
    random.Random(6).shuffle(small)
    small = [b""] + small[:150] + [b"", b""] + small[150:] + [b""]
    bd, bo, _ = W.make_batch(1400, 8, 3600, seed=22)         # ~2.5 MB: a dozen sub-batches a host call on ctx
    big = [bytes(bd[int(bo[i]):int(bo[i + 1])]) for i in range(len(bo) - 1)]
    one = [max(multi, key=len) * 3]
    return {"small": _family(small, rng.integers(0, 3, len(small)), 1, specials),
            "big": _family(big, rng.integers(0, 3, len(big)), 2, specials),
            "one": _family(one, [1], 3, specials)}


# ---------------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------------
class Ref:
    def __init__(self, tekken_bytes, controls):
        from cfbpe import workload as W
        from oracle import oracle
        self.oracle = oracle
        self.vocabs = [oracle.OracleVocab(tekken_bytes, n) for _, n, _ in SLOTS]
        self.patterns = [p for p, _, _ in SLOTS]
        self.bases = np.array([b for _, _, b in SLOTS], np.int64)
        self.tok_len = np.array([len(t) for t in W.vocab_tokens(tekken_bytes, max(n for _, n, _ in SLOTS))], np.int64)
        self.tables = [None, SS.Table(controls), SS.Table(O200K_SPECIALS)]
        self.n_specials = [0, len(controls), len(O200K_SPECIALS)]
        self.memo = {}

    def _m(self, key, f):
        if key not in self.memo:
            self.memo[key] = f()
        return self.memo[key]

    def encode(self, b):
        """(ids, id offsets, counts, byte starts) of a valid batch"""
        def f():
            r, io, cnt = self.oracle.encode_batch(self.vocabs, self.patterns, b.data, b.offs, b.vid, nthreads=os.cpu_count())
            tp = np.repeat(np.arange(b.n), cnt.astype(np.int64))
            ids = (r.astype(np.int64) + self.bases[b.vid[tp]]).astype(np.uint32)
            ln = self.tok_len[r]
            excl = np.cumsum(ln) - ln
            assert int(ln.sum()) == b.total                     # the token bytes tile the batch
            starts = (excl - b.offs[tp].astype(np.int64)).astype(np.uint32)
            return ids, io, cnt.astype(np.uint32), starts
        return self._m(("enc", id(b)), f)

    def repaired(self, b):
        from cfbpe import plugin as P
        def f():
            data, offs, rep = P.repair_utf8(b.data, b.offs)
            rb = Batch([bytes(data[int(offs[i]):int(offs[i + 1])]) for i in range(b.n)], b.vid)
            return rb, rep
        return self._m(("rep", id(b)), f)

    def special(self, b, allow):
        """("bad", prompt, index) or ("ok", ids, offsets, counts) of encode_batch_special: allow -> every special ALLOWED, else
        tiktoken's default (every special DISALLOWED)"""
        def f():
            modes = [None] + [np.full(k, SS.ALLOW, np.uint8) for k in self.n_specials[1:]] if allow else None

            def enc(v):
                return lambda s: (self.vocabs[v].encode(self.patterns[v], s).astype(np.int64) + self.bases[v]).tolist()
            res = SS.reference(self.tables, modes, b.prompts, b.vid, [enc(v) for v in range(len(SLOTS))])
            if res[0] == "bad":
                return res
            per = res[1]
            io = np.zeros(b.n + 1, np.uint64)
            io[1:] = np.cumsum([len(p) for p in per])
            return "ok", np.array([i for p in per for i in p], np.uint32), io, np.array([len(p) for p in per], np.uint32)
        return self._m(("spec", id(b), allow), f)


@pytest.fixture(scope="module")
def ref(tekken_bytes, controls):
    return Ref(tekken_bytes, controls)


# ---------------------------------------------------------------------------------------------------------------------------
# the call catalogue: name -> (run(ctx, fam, stream) -> (rc, outputs), expect(ref, fam) -> (rc, outputs))
# ---------------------------------------------------------------------------------------------------------------------------
def _rc(f, *a, **k):
    """(rc, result, the exception or None) of a binding call"""
    from cfbpe import _native as N
    try:
        return N.OK, f(*a, **k), None
    except N.NativeError as e:
        return e.code, None, e


def _fill(n, dtype=np.uint32):
    return np.full(n, SENTINEL, dtype)


def _tfill(n, dtype=None):
    import torch
    return torch.full((max(n, 1),), -1, dtype=dtype or torch.int32, device="cuda:0")


def _u32(t, n=None):
    a = t.cpu().numpy()
    return (a.view(np.uint32) if a.dtype == np.int32 else a.astype(np.uint64))[:n]


def _tail():
    return np.full(TAIL, SENTINEL, np.uint32)


def _device(ctx, call, sync, stream):
    """a device call, then (async) cfbpe_device_status on its stream: the first error"""
    rc, r, _ = _rc(call, sync)
    if rc:
        return rc, {}
    if rc == 0 and not sync:
        rc, _, _ = _rc(ctx.device_status, stream)
    return rc, r


# -- host kinds
def run_encode(ctx, F, s):
    b = F["clean"]
    ids, io = _fill(b.total + TAIL), np.zeros(b.n + 1, np.uint64)
    rc, r, _ = _rc(ctx.encode_batch, b.data, b.offs, b.vid, ids, io)
    if rc:
        return rc, {}
    nt = int(io[-1])
    return rc, dict(ids=ids[:nt], offsets=io, counts=r[2], tail=ids[nt:nt + TAIL])


def exp_encode(R, F):
    ids, io, cnt, _ = R.encode(F["clean"])
    return 0, dict(ids=ids, offsets=io, counts=cnt, tail=_tail())


def run_starts(ctx, F, s):
    b = F["clean"]
    ids, st = _fill(b.total + TAIL), _fill(b.total + TAIL)
    rc, r, _ = _rc(ctx.encode_batch_starts, b.data, b.offs, b.vid, ids, st)
    if rc:
        return rc, {}
    nt = int(r[2][-1])
    return rc, dict(ids=r[0], starts=r[1], offsets=r[2], counts=r[3], tail=st[nt:nt + TAIL])


def exp_starts(R, F):
    ids, io, cnt, st = R.encode(F["clean"])
    return 0, dict(ids=ids, starts=st, offsets=io, counts=cnt, tail=_tail())


def _units(unit):
    def run(ctx, F, s):
        from cfbpe import _native as N
        b = F["clean"]
        rc, r, _ = _rc(ctx.encode_batch_char_starts, b.data, b.offs, N.UNIT_UTF16 if unit == "utf16" else N.UNIT_CODEPOINT, b.vid)
        if rc:
            return rc, {}
        return rc, dict(ids=r[0], starts=r[1], offsets=r[2], counts=r[3], lens=r[4])

    def exp(R, F):
        from cfbpe import plugin as P
        b = F["clean"]
        ids, io, cnt, st = R.encode(b)
        us, lens = P.unit_starts(b.data, b.offs, io, st, unit)
        return 0, dict(ids=ids, starts=us, offsets=io, counts=cnt, lens=lens)
    return run, exp


def run_count(ctx, F, s):
    b = F["clean"]
    rc, r, _ = _rc(ctx.count_batch, b.data, b.offs, b.vid)
    if rc:
        return rc, {}
    return rc, dict(counts=r)


def exp_count(R, F):
    return 0, dict(counts=R.encode(F["clean"])[2])


def _exp_truncate(R, F, tail):
    from cfbpe import plugin as P
    b = F["clean"]
    _, io, cnt, st = R.encode(b)
    cut, kept = R._m(("trunc", id(b), tail), lambda: P.truncate_cuts(b.data, b.offs, io, st, b.budgets, tail))
    return 0, dict(cut=cut, kept=kept, counts=cnt)


def _truncate(tail):
    def run(ctx, F, s):
        from cfbpe import _native as N
        b = F["clean"]
        rc, r, _ = _rc(ctx.truncate_batch, b.data, b.offs, b.budgets, N.TRUNCATE_TAIL if tail else N.TRUNCATE_HEAD, b.vid)
        if rc:
            return rc, {}
        return rc, dict(cut=r[0], kept=r[1], counts=r[2])
    return run, lambda R, F: _exp_truncate(R, F, tail)


def _exp_chunk(R, F, n, s):
    from cfbpe import plugin as P
    b = F["clean"]
    _, io, cnt, st = R.encode(b)
    spans, coffs = R._m(("chunk", id(b), n, s), lambda: P.chunk_spans(b.data, b.offs, io, st, n, s))
    return 0, dict(spans=spans.reshape(-1), coffs=coffs, counts=cnt)


def _chunk(n, s_):
    def run(ctx, F, s):
        b = F["clean"]
        rc, r, _ = _rc(ctx.chunk_batch, b.data, b.offs, n, s_, b.vid)
        if rc:
            return rc, {}
        return rc, dict(spans=r[0].reshape(-1), coffs=r[1], counts=r[2])
    return run, lambda R, F: _exp_chunk(R, F, n, s_)


def _modes(R, allow):
    return [None] + [np.full(k, SS.ALLOW, np.uint8) for k in R.n_specials[1:]] if allow else None


def _exp_special(R, F, variant, allow):
    from cfbpe import _native as N
    res = R.special(F[variant], allow)
    if res[0] == "bad":
        return N.EBADMSG, dict(bad=np.array(res[1:], np.int64))
    return 0, dict(ids=res[1], offsets=res[2], counts=res[3])


def _special(variant, allow):
    def run(ctx, F, s):
        b = F[variant]
        rc, r, e = _rc(ctx.encode_batch_special, b.data, b.offs, b.vid, _modes(REF[0], allow))
        if e is not None and e.bad is not None:
            return rc, dict(bad=np.array(e.bad, np.int64))
        return rc, (dict(ids=r[0], offsets=r[1], counts=r[2]) if r else {})
    return run, lambda R, F: _exp_special(R, F, variant, allow)


def _exp_lossy(R, F, variant):
    b = F[variant]
    rb, rep = R.repaired(b)
    ids, io, cnt, _ = R.encode(rb)
    return 0, dict(ids=ids, offsets=io, counts=cnt, replaced=rep)


def _lossy(variant):
    def run(ctx, F, s):
        b = F[variant]
        rc, r, _ = _rc(ctx.encode_batch_lossy, b.data, b.offs, b.vid)
        if rc:
            return rc, {}
        return rc, dict(ids=r[0], offsets=r[1], counts=r[2], replaced=r[3])
    return run, lambda R, F: _exp_lossy(R, F, variant)


def _decode_input(R, F, unknown):
    ids, io, _, _ = R.encode(F["clean"])
    ids = ids.copy()
    if unknown:
        ids[len(ids) // 2] = 0xFFFFFFF0          # past every slot's ranks and base, and no registered special
    return ids, io


def _decode(unknown):
    def run(ctx, F, s):
        b = F["clean"]
        ids, io = _decode_input(REF[0], F, unknown)
        out = np.full(b.total + TAIL, 0xAB, np.uint8)
        rc, r, _ = _rc(ctx.decode_batch, ids, io, b.vid, out_bytes=out)
        if rc:
            return rc, {}
        return rc, ({} if unknown else dict(bytes=r[0], offsets=r[1], tail=out[b.total:]))

    def exp(R, F):
        from cfbpe import _native as N
        b = F["clean"]
        if unknown:
            return N.EINVAL, {}
        return 0, dict(bytes=b.data, offsets=b.offs, tail=np.full(TAIL, 0xAB, np.uint8))
    return run, exp


def run_eilseq(ctx, F, s):
    b = F["bad"]
    rc, _, _ = _rc(ctx.encode_batch, b.data, b.offs, b.vid)
    return rc, {}


def exp_eilseq(R, F):
    from cfbpe import _native as N
    return N.EILSEQ, {}


def run_enospc(ctx, F, s):
    b = F["clean"]
    need = int(REF[0].encode(b)[1][-1])
    ids, io = _fill(need - 1 + TAIL), np.zeros(b.n + 1, np.uint64)
    rc, _, _ = _rc(ctx.encode_batch, b.data, b.offs, b.vid, ids[:need - 1], io)
    return rc, dict(need=io[-1:], tail=ids[need - 1:])


def exp_enospc(R, F):
    from cfbpe import _native as N
    return N.ENOSPC, dict(need=R.encode(F["clean"])[1][-1:], tail=_tail())


# -- device kinds: the same calls on device memory, synchronous or sync=False + cfbpe_device_status
def _dev_encode(form, sync, variant="clean", cap_short=False):
    """form: plain, starts, utf16 (with lengths), special (all allowed), lossy (U+FFFD counts out)"""
    def run(ctx, F, s):
        import torch
        from cfbpe import _native as N
        b = F[variant]
        d_b, d_o, d_v, _ = b.dev()
        if form == "lossy":
            need = int(REF[0].encode(REF[0].repaired(b)[0])[1][-1])
        elif form == "special":
            need = int(REF[0].special(b, True)[2][-1])
        else:
            need = int(REF[0].encode(b)[1][-1])
        cap = need - 1 if cap_short else need
        ids, st, off, cnt, aux = _tfill(cap + TAIL), _tfill(cap + TAIL), _tfill(b.n + 1, torch.int64), _tfill(b.n), _tfill(b.n)
        a = (b.n, d_b.data_ptr(), b.total, d_o.data_ptr(), d_v.data_ptr())
        if form == "plain":
            call = lambda y: ctx.encode_batch_device(*a, ids.data_ptr(), cap, off.data_ptr(), cnt.data_ptr(), s, y)
        elif form == "starts":
            call = lambda y: ctx.encode_batch_starts_device(*a, ids.data_ptr(), st.data_ptr(), cap, off.data_ptr(), cnt.data_ptr(), s, y)
        elif form == "utf16":
            call = lambda y: ctx.encode_batch_char_starts_device(*a, N.UNIT_UTF16, ids.data_ptr(), st.data_ptr(), cap, off.data_ptr(),
                                                                 cnt.data_ptr(), aux.data_ptr(), s, y)
        elif form == "special":
            call = lambda y: ctx.encode_batch_special_device(*a, ids.data_ptr(), cap, off.data_ptr(), cnt.data_ptr(), _modes(REF[0], True), s, y)
        else:
            call = lambda y: ctx.encode_batch_lossy_device(*a, ids.data_ptr(), cap, off.data_ptr(), cnt.data_ptr(), aux.data_ptr(), s, y)
        rc, nt = _device(ctx, call, sync, s)
        o = _u32(off)
        if cap_short:
            return rc, dict(need=o[-1:], tail=_u32(ids)[cap:cap + TAIL])
        out = dict(ids=_u32(ids)[:need], offsets=o, counts=_u32(cnt, b.n), tail=_u32(ids)[need:need + TAIL])
        if sync:
            out["n"] = np.array([nt], np.int64)
        if form in ("starts", "utf16"):
            out["starts"] = _u32(st)[:need]
        if form in ("utf16", "lossy"):
            out["aux"] = _u32(aux, b.n)
        return rc, out

    def exp(R, F):
        from cfbpe import _native as N
        from cfbpe import plugin as P
        b = F[variant]
        if form == "lossy":
            rb, rep = R.repaired(b)
            ids, io, cnt, _ = R.encode(rb)
        elif form == "special":
            _, ids, io, cnt = R.special(b, True)
        else:
            ids, io, cnt, st = R.encode(b)
        if cap_short:
            return N.ENOSPC, dict(need=io[-1:], tail=_tail())
        out = dict(ids=ids, offsets=io, counts=cnt, tail=_tail())
        if sync:
            out["n"] = np.array([len(ids)], np.int64)
        if form == "starts":
            out["starts"] = st
        if form == "utf16":
            out["starts"], out["aux"] = P.unit_starts(b.data, b.offs, io, st, "utf16")
        if form == "lossy":
            out["aux"] = rep
        return 0, out
    return run, exp


def _dev_eilseq(sync):
    def run(ctx, F, s):
        import torch
        b = F["bad"]
        d_b, d_o, d_v, _ = b.dev()
        ids, off = _tfill(b.total + TAIL), _tfill(b.n + 1, torch.int64)
        rc, _ = _device(ctx, lambda y: ctx.encode_batch_device(b.n, d_b.data_ptr(), b.total, d_o.data_ptr(), d_v.data_ptr(), ids.data_ptr(),
                                                               b.total + TAIL, off.data_ptr(), None, s, y), sync, s)
        return rc, {}
    return run, exp_eilseq


def _dev_truncate(tail):
    def run(ctx, F, s):
        from cfbpe import _native as N
        b = F["clean"]
        d_b, d_o, d_v, d_bud = b.dev()
        cut, kept, cnt = _tfill(b.n + TAIL), _tfill(b.n + TAIL), _tfill(b.n + TAIL)
        rc, _ = _device(ctx, lambda y: ctx.truncate_batch_device(b.n, d_b.data_ptr(), b.total, d_o.data_ptr(), d_v.data_ptr(), d_bud.data_ptr(),
                                                                 N.TRUNCATE_TAIL if tail else N.TRUNCATE_HEAD, cut.data_ptr(), kept.data_ptr(),
                                                                 cnt.data_ptr(), s), False, s)
        c, k, n_ = _u32(cut), _u32(kept), _u32(cnt)
        return rc, dict(cut=c[:b.n], kept=k[:b.n], counts=n_[:b.n], tail=np.concatenate([c[b.n:], k[b.n:], n_[b.n:]]))

    def exp(R, F):
        rc, out = _exp_truncate(R, F, tail)
        out["tail"] = np.full(3 * TAIL, SENTINEL, np.uint32)
        return rc, out
    return run, exp


def _dev_chunk(n, s_, sync, cap_short=False):
    def run(ctx, F, s):
        import torch
        b = F["clean"]
        d_b, d_o, d_v, _ = b.dev()
        need = len(_exp_chunk(REF[0], F, n, s_)[1]["spans"]) // 2
        cap = need - 1 if cap_short else need
        spans, coffs, cnt = _tfill(2 * (cap + TAIL)), _tfill(b.n + 1, torch.int64), _tfill(b.n)
        rc, nc = _device(ctx, lambda y: ctx.chunk_batch_device(b.n, d_b.data_ptr(), b.total, d_o.data_ptr(), d_v.data_ptr(), n, s_,
                                                               spans.data_ptr(), cap, coffs.data_ptr(), cnt.data_ptr(), s, y), sync, s)
        sp = _u32(spans)
        if cap_short:
            return rc, dict(need=_u32(coffs)[-1:], tail=sp[2 * cap:])
        out = dict(spans=sp[:2 * need], coffs=_u32(coffs), counts=_u32(cnt, b.n), tail=sp[2 * need:])
        if sync:
            out["n"] = np.array([nc], np.int64)
        return rc, out

    def exp(R, F):
        from cfbpe import _native as N
        rc, out = _exp_chunk(R, F, n, s_)
        if cap_short:
            return N.ENOSPC, dict(need=out["coffs"][-1:], tail=np.full(2 * TAIL, SENTINEL, np.uint32))
        out["tail"] = np.full(2 * TAIL, SENTINEL, np.uint32)
        if sync:
            out["n"] = np.array([len(out["spans"]) // 2], np.int64)
        return rc, out
    return run, exp


REF = [None]     # the module's Ref, for the runners that size their buffers from it


def _catalogue():
    k = {"encode": (run_encode, exp_encode), "starts": (run_starts, exp_starts), "units_cp": _units("codepoint"),
         "units_utf16": _units("utf16"), "count": (run_count, exp_count), "truncate_head": _truncate(False),
         "truncate_tail": _truncate(True), "chunk_s0": _chunk(*CHUNKS[0]), "chunk_overlap": _chunk(*CHUNKS[1]),
         "special_default": _special("clean", False), "special_allowed": _special("spec", True),
         "special_disallowed": _special("spec", False), "lossy_clean": _lossy("clean"), "lossy_repair": _lossy("bad"),
         "decode": _decode(False), "decode_unknown": _decode(True), "encode_eilseq": (run_eilseq, exp_eilseq),
         "encode_enospc": (run_enospc, exp_enospc)}
    for sync in (True, False):
        t = "sync" if sync else "async"
        k["dev_encode_" + t] = _dev_encode("plain", sync)
        k["dev_starts_" + t] = _dev_encode("starts", sync)
        k["dev_units_utf16_" + t] = _dev_encode("utf16", sync)
        k["dev_special_allowed_" + t] = _dev_encode("special", sync, "spec")
        k["dev_lossy_repair_" + t] = _dev_encode("lossy", sync, "bad")
        k["dev_chunk_overlap_" + t] = _dev_chunk(*CHUNKS[1], sync)
        k["dev_eilseq_" + t] = _dev_eilseq(sync)
        k["dev_enospc_" + t] = _dev_encode("plain", sync, cap_short=True)
    k["dev_truncate_head_async"] = _dev_truncate(False)
    k["dev_truncate_tail_async"] = _dev_truncate(True)
    k["dev_chunk_enospc_async"] = _dev_chunk(*CHUNKS[0], False, cap_short=True)
    return k


KINDS = _catalogue()


def _check(ctx, ref, fams, kind, fam, stream, where=""):
    run, exp = KINDS[kind]
    want_rc, want = ref._m(("want", kind, fam), lambda: exp(ref, fams[fam]))
    rc, got = run(ctx, fams[fam], stream)
    assert rc == want_rc, "%s on %s%s: rc %d, want %d" % (kind, fam, where, rc, want_rc)
    for key, w in want.items():
        g = got.get(key)
        assert g is not None and np.array_equal(np.asarray(g), np.asarray(w)), "%s on %s%s: %s differs" % (kind, fam, where, key)


@pytest.fixture(scope="module")
def world(ctx, ref, fams):
    import torch
    REF[0] = ref
    return ctx, ref, fams, torch.cuda.current_stream().cuda_stream


@pytest.mark.parametrize("first", sorted(KINDS))
def test_every_kind_after_every_other(world, first):
    """`first` on the big batch (a host call pipelines), then every kind on the small batch (a host call runs in one pass): both
    exact, whatever the lane kept from the call before"""
    ctx, ref, fams, s = world
    for then in sorted(KINDS):
        _check(ctx, ref, fams, first, "big", s, " (first)")
        _check(ctx, ref, fams, then, "small", s, " after %s on big" % first)


def test_random_walk(world):
    """a seeded walk of 4000 calls over kinds x batches, each one checked"""
    ctx, ref, fams, s = world
    rng = random.Random(2024)
    names = sorted(KINDS)
    prev = "start"
    for step in range(4000):
        kind = rng.choice(names)
        fam = rng.choices(["small", "one", "big"], [6, 3, 1])[0]
        _check(ctx, ref, fams, kind, fam, s, " at step %d after %s" % (step, prev))
        prev = "%s on %s" % (kind, fam)


# ---------------------------------------------------------------------------------------------------------------------------
# what cfbpe_device_status reports
# ---------------------------------------------------------------------------------------------------------------------------
def _status(c, stream):
    return _rc(c.device_status, stream)[0]


def _async_encode(c, b, stream, cap=None):
    """encode_batch_device(sync=False) of b; the output buffers are returned, to live until the call is done"""
    import torch
    d_b, d_o, d_v, _ = b.dev()
    cap = b.total + 1 if cap is None else cap
    ids, off = torch.empty(max(cap, 1), dtype=torch.int32, device=d_b.device), torch.empty(b.n + 1, dtype=torch.int64, device=d_b.device)
    c.encode_batch_device(b.n, d_b.data_ptr(), b.total, d_o.data_ptr(), d_v.data_ptr(), ids.data_ptr(), cap, off.data_ptr(), None, stream,
                          sync=False)
    return ids, off


# host kinds that each run in one pass on plain_ctx's lane and rewrite its status word
ONE_PASS_HOST_KINDS = ["encode", "starts", "units_utf16", "count", "truncate_tail", "chunk_overlap", "lossy_repair", "special_allowed",
                       "special_disallowed", "decode", "decode_unknown", "encode_eilseq"]


@pytest.fixture(scope="module")
def status_world(plain_ctx, ref, fams):
    import torch
    REF[0] = ref
    return plain_ctx, ref, fams, torch.cuda.current_stream().cuda_stream


def test_status_survives_host_calls_and_decode(status_world):
    """case 1: an async device encode on malformed bytes, then a host call or decode on the lane: cfbpe_device_status is EILSEQ"""
    from cfbpe import _native as N
    c, ref, fams, s = status_world
    for kind in ONE_PASS_HOST_KINDS:
        for fam in ("one", "small"):
            bufs = _async_encode(c, fams["small"]["bad"], s)
            _check(c, ref, fams, kind, fam, s, " between a device call and device_status")
            assert _status(c, s) == N.EILSEQ, "%s on %s" % (kind, fam)
            del bufs


def test_status_keeps_its_own_out_cap(status_world):
    """case 2: an async device encode whose ids exactly fill out_cap, then a one-pass host call with more ids: OK"""
    c, ref, fams, s = status_world
    b = Batch(fams["small"]["clean"].prompts[:6], fams["small"]["clean"].vid[:6])
    need = int(ref.encode(b)[1][-1])
    assert 0 < need < int(ref.encode(fams["one"]["clean"])[1][-1])
    ids, off = _async_encode(c, b, s, cap=need)
    _check(c, ref, fams, "encode", "one", s)
    assert _status(c, s) == 0
    assert np.array_equal(_u32(ids), ref.encode(b)[0])


def test_status_not_taken_from_decode(status_world):
    """case 3: a clean async device call, then decode with an unknown id (EINVAL for decode): cfbpe_device_status is OK"""
    c, ref, fams, s = status_world
    bufs = _async_encode(c, fams["small"]["clean"], s)
    _check(c, ref, fams, "decode_unknown", "small", s)
    assert _status(c, s) == 0
    del bufs


def test_chunk_status_keeps_its_chunk_cap(status_world):
    """case 4: an async device chunk call over chunk_cap, then a one-pass host chunk call with fewer tokens than that chunk_cap:
    cfbpe_device_status is ENOSPC"""
    import torch
    from cfbpe import _native as N
    c, ref, fams, s = status_world
    b = fams["small"]["clean"]
    n, s_ = CHUNKS[0]
    need = len(_exp_chunk(ref, fams["small"], n, s_)[1]["spans"]) // 2
    few = Batch([b"Hello there, world"], [0])
    assert int(ref.encode(few)[1][-1]) <= need - 1
    d_b, d_o, d_v, _ = b.dev()
    spans, coffs = torch.empty(2 * need, dtype=torch.int32, device="cuda:0"), torch.empty(b.n + 1, dtype=torch.int64, device="cuda:0")
    c.chunk_batch_device(b.n, d_b.data_ptr(), b.total, d_o.data_ptr(), d_v.data_ptr(), n, s_, spans.data_ptr(), need - 1, coffs.data_ptr(),
                         None, s, sync=False)
    spans_h, coffs_h, _ = c.chunk_batch(few.data, few.offs, n, s_, few.vid)
    assert len(coffs_h) == 2 and int(coffs_h[-1]) >= 1
    assert _status(c, s) == N.ENOSPC
    assert int(_u32(coffs)[-1]) == need


def test_status_is_per_context(status_world, tekken_bytes):
    """case 5: two live contexts: an async bad call on A does not show in cfbpe_device_status(B), and A still reports it"""
    from cfbpe import _native as N
    c, ref, fams, s = status_world
    other = N.Context(0, max_batch_bytes=1 << 20, max_prompts=1 << 10)
    try:
        other.vocab_load(0, tekken_bytes, N.FORMAT_TIKTOKEN, SLOTS[0][0], SLOTS[0][1])
        assert _status(other, s) == 0                                   # no device call on it yet
        good = Batch([b"Hello", b" world"], [0, 0])
        keep = _async_encode(other, good, s)
        bad = _async_encode(c, fams["small"]["bad"], s)
        assert _status(other, s) == 0
        assert _status(c, s) == N.EILSEQ
        assert _status(other, s) == 0
        del keep, bad
    finally:
        other.close()


def _two_threads(c1, c2, bad, good, one, device1=0):
    """thread 1: an async bad device call on c1; then thread 2: a clean async device call and one-pass host calls on c2; then each
    reads its status.  Returns (thread 1's, thread 2's)."""
    import torch
    from cfbpe import _native as N
    out, e1, e2, errs = {}, threading.Event(), threading.Event(), []

    def t1():
        try:
            with torch.cuda.device(device1):
                st = torch.cuda.Stream()
                with torch.cuda.stream(st):
                    keep = _async_encode(c1, bad, st.cuda_stream)
                e1.set()
                e2.wait(120)
                out[1] = _status(c1, st.cuda_stream)
                del keep
        except Exception as e:           # pragma: no cover - reported below
            errs.append(e)
            e1.set()

    def t2():
        try:
            e1.wait(120)
            st = torch.cuda.Stream(device=0)
            with torch.cuda.stream(st):
                keep = _async_encode(c2, good, st.cuda_stream)
            rc, _, _ = _rc(c2.decode_batch, np.array([0xFFFFFFF0], np.uint32), np.array([0, 1], np.uint64), one.vid)
            assert rc == N.EINVAL
            c2.encode_batch(one.data, one.offs, one.vid)
            e2.set()
            out[2] = _status(c2, st.cuda_stream)
            del keep
        except Exception as e:           # pragma: no cover - reported below
            errs.append(e)
            e2.set()
    ts = [threading.Thread(target=t1), threading.Thread(target=t2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs
    return out[1], out[2]


def test_status_is_per_thread(status_world):
    """case 6: two threads on the one-lane context: thread 1's async bad call is reported to thread 1 (EILSEQ) after thread 2's
    calls took the lane, and thread 2 gets OK"""
    import torch
    from cfbpe import _native as N
    c, ref, fams, s = status_world
    for b in (fams["small"]["bad"], fams["small"]["clean"]):
        b.dev()
    torch.cuda.synchronize()
    r1, r2 = _two_threads(c, c, fams["small"]["bad"], fams["small"]["clean"], fams["one"]["clean"])
    assert (r1, r2) == (N.EILSEQ, 0)


def test_status_is_per_thread_on_two_devices(tekken_bytes, controls, fams, ref):
    """case 6 on a two-device context: thread 1 calls on device 1, thread 2 on device 0"""
    import torch
    from cfbpe import _native as N
    if torch.cuda.device_count() < 2:
        pytest.skip("one device")
    REF[0] = ref
    c = _load(N.Context(devices=[0, 1], max_batch_bytes=16 << 20, max_prompts=1 << 14, n_workspaces=1), tekken_bytes, controls)
    try:
        bad = fams["small"]["bad"]
        d1 = torch.device("cuda:1")
        with torch.cuda.device(1):
            bad1 = Batch(bad.prompts, bad.vid)
            d_b = torch.zeros(bad.total + 64, dtype=torch.uint8, device=d1)
            d_b[:bad.total] = torch.from_numpy(bad.data).to(d1)
            bad1._dev = (d_b, torch.from_numpy(bad.offs.astype(np.int64)).to(d1), torch.from_numpy(bad.vid.copy()).to(d1), None)
        fams["small"]["clean"].dev()
        torch.cuda.synchronize(0)
        torch.cuda.synchronize(1)
        r1, r2 = _two_threads(c, c, bad1, fams["small"]["clean"], fams["one"]["clean"], device1=1)
        assert (r1, r2) == (N.EILSEQ, 0)
    finally:
        c.close()


def test_a_later_device_call_replaces_the_status(status_world):
    """case 7: the status is that of the thread's LAST device call: bad then clean is OK, clean then bad is EILSEQ"""
    from cfbpe import _native as N
    c, ref, fams, s = status_world
    a = _async_encode(c, fams["small"]["bad"], s)
    b = _async_encode(c, fams["small"]["clean"], s)
    assert _status(c, s) == 0
    a = _async_encode(c, fams["small"]["clean"], s)
    b = _async_encode(c, fams["small"]["bad"], s)
    assert _status(c, s) == N.EILSEQ
    assert _status(c, s) == N.EILSEQ              # reading it does not clear it
    del a, b
