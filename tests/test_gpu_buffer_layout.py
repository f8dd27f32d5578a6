"""The device entry points on caller buffers laid out as include/cfbpe.h allows (d_bytes at any address, 32 bytes of padding
whose contents do not matter), windows of a batch that stays on the device, and host calls over a lane whose byte buffer holds
adversarial bytes from an earlier call, on the H100: equal to the host call on the same prompts and to the oracle.
The same layouts run on the CPU emulator, under the alignment sanitizer and against guard pages, in test_buffer_layout_sim.py."""
import numpy as np
import pytest

import fuzzgen
from conftest import pack
from test_buffer_layout_sim import FILLER, FILLS, SPECIALS, endings

pytestmark = pytest.mark.gpu

PATS = ((0, 100256), (3, 130072))
N_TOK, OVERLAP = 7, 2
HEAD, TAIL = 0, 1
CHUNK = 4096                     # sub-batch bytes of the pipelined context (CFBPE_PIPE_CHUNK_BYTES)


def context(tekken_bytes, max_bytes=8 << 20, max_prompts=1 << 16):
    from cfbpe import _native as N
    c = N.Context(0, max_bytes, max_prompts)
    for slot, (pat, n) in enumerate(PATS):
        c.vocab_load(slot, tekken_bytes, N.FORMAT_TIKTOKEN, pat, n)
        c.vocab_set_specials(slot, SPECIALS)
    return c


def modes_for(m):
    """per-vocabulary modes: slot k uses mode (m + k) % 3 (ORDINARY, ALLOW, DISALLOW) for every special"""
    return [np.full(len(SPECIALS), (m + k) % 3, np.uint8) for k in range(len(PATS))]


def host_all(c, data, offs, vid, budgets):
    """every host entry point: {entry: numpy results, or ("error", code[, bad])}"""
    from cfbpe import _native as N
    r = {}

    def run(key, f):
        try:
            r[key] = tuple(np.array(x) for x in f())
        except N.NativeError as e:
            r[key] = ("error", e.code, getattr(e, "bad", None))
    run("encode", lambda: c.encode_batch(data, offs, vid))
    run("starts", lambda: c.encode_batch_starts(data, offs, vid))
    for m in range(3):
        run(("special", m), lambda: c.encode_batch_special(data, offs, vid, modes_for(m)))
    for mode in (HEAD, TAIL):
        run(("truncate", mode), lambda: c.truncate_batch(data, offs, budgets, mode, vid))
    run("chunk", lambda: c.chunk_batch(data, offs, N_TOK, OVERLAP, vid))
    return r


def device_all(c, n, d_bytes, total, d_offs, d_vid, budgets, sync):
    """the device entry points on d_bytes (total bytes) and device offsets, in host_all's form; sync False: asynchronous, then
    device_status"""
    import torch
    from cfbpe import _native as N
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    vid = None if d_vid is None else d_vid.data_ptr()
    cap = total + 1
    r = {}

    def outs():
        return (torch.full((cap,), -1, dtype=torch.int32, device=dev), torch.zeros(n + 1, dtype=torch.int64, device=dev),
                torch.zeros(max(n, 1), dtype=torch.int32, device=dev))

    def u32(t):
        return t.cpu().numpy().view(np.uint32)

    def finish(key, f):
        try:
            f()
            if not sync:
                c.device_status(stream)
            torch.cuda.synchronize()
            return True
        except N.NativeError as e:
            torch.cuda.synchronize()
            r[key] = ("error", e.code, getattr(e, "bad", None))
            return False
    ids, off, cnt = outs()
    if finish("encode", lambda: c.encode_batch_device(n, d_bytes, total, d_offs, vid, ids.data_ptr(), cap, off.data_ptr(), cnt.data_ptr(),
                                                      stream, sync)):
        o = off.cpu().numpy().astype(np.uint64)
        r["encode"] = (u32(ids)[:int(o[-1])], o, u32(cnt)[:n])
    ids, off, cnt = outs()
    st = torch.full((cap,), -1, dtype=torch.int32, device=dev)
    if finish("starts", lambda: c.encode_batch_starts_device(n, d_bytes, total, d_offs, vid, ids.data_ptr(), st.data_ptr(), cap, off.data_ptr(),
                                                             cnt.data_ptr(), stream, sync)):
        o = off.cpu().numpy().astype(np.uint64)
        r["starts"] = (u32(ids)[:int(o[-1])], u32(st)[:int(o[-1])], o, u32(cnt)[:n])
    for m in range(3):
        ids, off, cnt = outs()
        if finish(("special", m), lambda: c.encode_batch_special_device(n, d_bytes, total, d_offs, vid, ids.data_ptr(), cap, off.data_ptr(),
                                                                        cnt.data_ptr(), modes_for(m), stream, sync)):
            o = off.cpu().numpy().astype(np.uint64)
            r["special", m] = (u32(ids)[:int(o[-1])], o, u32(cnt)[:n])
    d_bud = torch.from_numpy(np.asarray(budgets, np.uint32).view(np.int32)).to(dev)
    for mode in (HEAD, TAIL):
        cut, kept, cnt = (torch.full((max(n, 1),), -1, dtype=torch.int32, device=dev) for _ in range(3))
        if finish(("truncate", mode), lambda: c.truncate_batch_device(n, d_bytes, total, d_offs, vid, d_bud.data_ptr(), mode, cut.data_ptr(),
                                                                      kept.data_ptr(), cnt.data_ptr(), stream)):
            r["truncate", mode] = (u32(cut)[:n], u32(kept)[:n], u32(cnt)[:n])
    ccap = max(total, 1)
    spans = torch.full((ccap, 2), -1, dtype=torch.int32, device=dev)
    coffs = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    cnt = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
    if finish("chunk", lambda: c.chunk_batch_device(n, d_bytes, total, d_offs, vid, N_TOK, OVERLAP, spans.data_ptr(), ccap, coffs.data_ptr(),
                                                    cnt.data_ptr(), stream, sync)):
        co = coffs.cpu().numpy().astype(np.uint64)
        r["chunk"] = (u32(spans)[:int(co[-1])], co, u32(cnt)[:n])
    return r


def assert_same(got, want, what):
    assert got.keys() == want.keys(), what
    for key in want:
        g, w = got[key], want[key]
        if isinstance(w[0], str):                        # ("error", code, bad)
            assert g == w, (what, key)
        else:
            assert not isinstance(g[0], str) and len(g) == len(w), (what, key, g)
            for a, b in zip(g, w):
                assert np.array_equal(np.asarray(a, np.int64), np.asarray(b, np.int64)), (what, key)


def placed(data, m, fill):
    """a device buffer with the batch at byte offset m, fill before it and exactly 32 bytes of fill after it; (buffer, d_bytes)"""
    import torch

    def tile(k):
        return (fill * (k // len(fill) + 1))[:k]
    host = np.frombuffer(tile(m) + data.tobytes() + tile(32), np.uint8).copy()
    buf = torch.from_numpy(host).to("cuda:0")
    return buf, buf.data_ptr() + m


@pytest.fixture(scope="module")
def ctx(tekken_bytes):
    c = context(tekken_bytes)
    yield c
    c.close()


@pytest.fixture
def make_context(tekken_bytes):
    """context(...) for one test; every context it made is closed at teardown, whether the test passed or not"""
    made = []

    def make(**kw):
        made.append(context(tekken_bytes, **kw))
        return made[-1]
    yield make
    for c in made:
        c.close()


def test_every_device_entry_point_at_every_alignment(ctx, oracle_vocabs):
    """fuzz prompts, a filler and a crafted ending last, at every address mod 16 and every fill, two vocabularies, specials
    registered: the host call on the same prompts, whose ids are the oracle's"""
    import torch
    base = [s.encode() for s in fuzzgen.fuzz_strings(808, 24, max_atoms=20)]
    ends = endings()
    rng = np.random.default_rng(4)
    for i, last in enumerate(ends):
        prompts = base + [FILLER[:4 + (i - 4 - len(last)) % 16], last]
        data, offs = pack(prompts)
        vid = (np.arange(len(prompts)) % 2).astype(np.uint8)
        vid[-1] = i % 2
        budgets = rng.integers(0, 12, len(prompts)).astype(np.uint32)
        c = len(oracle_vocabs[PATS[vid[-1]][0]].encode(PATS[vid[-1]][0], last))
        budgets[-1] = [0, 1, max(c - 1, 0), c, c + 5][i % 5]
        want = host_all(ctx, data, offs, vid, budgets)
        for p in range(len(prompts)):
            pat = PATS[vid[p]][0]
            got = want["encode"][0][int(want["encode"][1][p]):int(want["encode"][1][p + 1])]
            assert np.array_equal(got, oracle_vocabs[pat].encode(pat, prompts[p])), (i, p)
        d_offs = torch.from_numpy(offs.astype(np.int64)).to("cuda:0")
        d_vid = torch.from_numpy(vid).to("cuda:0")
        for m in range(16):
            fill = FILLS[(i + m) % len(FILLS)]
            buf, d_bytes = placed(data, m, fill)
            for sync in (True, False):
                got = device_all(ctx, len(prompts), d_bytes, int(offs[-1]), d_offs.data_ptr(), d_vid, budgets, sync)
                assert_same(got, want, (i, m, fill[:8], sync))
            del buf


def test_windows_of_a_resident_corpus(make_context):
    """config 2 on the device; windows [i0, i1) passed as d_bytes = corpus + offsets[i0] with rebased offsets: the matching
    slice of the whole-batch call"""
    import torch
    from cfbpe import workload as W
    data, offs, _, _ = W.make_config(2, 1.0)
    n = len(offs) - 1
    c = make_context(max_bytes=16 << 20)
    vid = (np.arange(n) % 2).astype(np.uint8)
    budgets = np.random.default_rng(2).integers(0, 200, n).astype(np.uint32)
    corpus = torch.from_numpy(np.concatenate([data, np.frombuffer(FILLS[2] * 32, np.uint8)])).to("cuda:0")
    all_offs = torch.from_numpy(offs.astype(np.int64)).to("cuda:0")
    whole = device_all(c, n, corpus.data_ptr(), int(offs[-1]), all_offs.data_ptr(), torch.from_numpy(vid).to("cuda:0"), budgets, True)
    rng = np.random.default_rng(12)
    windows = [(0, n), (0, 1), (n - 1, n), (1, 2)] + [tuple(sorted(rng.choice(n + 1, 2, replace=False))) for _ in range(12)]
    for i0, i1 in windows:
        o0 = int(offs[i0])
        d_offs = torch.from_numpy((offs[i0:i1 + 1] - offs[i0]).astype(np.int64)).to("cuda:0")
        d_vid = torch.from_numpy(vid[i0:i1].copy()).to("cuda:0")
        for sync in (True, False):
            got = device_all(c, i1 - i0, corpus.data_ptr() + o0, int(offs[i1]) - o0, d_offs.data_ptr(), d_vid, budgets[i0:i1], sync)
            for key in ("encode", "starts", ("special", 0), ("truncate", HEAD), ("truncate", TAIL), "chunk"):
                assert_same({key: got[key]}, {key: _window(whole[key], key, i0, i1)}, (i0, i1, sync))


def _window(res, key, i0, i1):
    """prompts [i0, i1) of a whole-batch result, offsets rebased"""
    if key in ("encode", ("special", 0)):
        ids, off, cnt = res
        return ids[int(off[i0]):int(off[i1])], off[i0:i1 + 1] - off[i0], cnt[i0:i1]
    if key == "starts":
        ids, st, off, cnt = res
        return ids[int(off[i0]):int(off[i1])], st[int(off[i0]):int(off[i1])], off[i0:i1 + 1] - off[i0], cnt[i0:i1]
    if key == "chunk":
        spans, co, cnt = res
        return spans[int(co[i0]):int(co[i1])], co[i0:i1 + 1] - co[i0], cnt[i0:i1]
    return tuple(x[i0:i1] for x in res)


def stale_batches():
    """batches whose pipelined sub-batches (csrc/subbatch.h, CHUNK bytes) end at every residue mod 16 of the lane's byte buffer,
    one of them a byte before the next sub-batch's first byte (the smallest gap)"""
    import simlib
    out, ends, gaps = [], set(), set()
    for seed in range(400):
        rng = np.random.default_rng(seed)
        prompts = [s.encode() for s in fuzzgen.fuzz_strings(seed, int(rng.integers(150, 260)), max_atoms=30)]
        ending = endings()
        for k in rng.choice(len(ending), 12, replace=False):
            prompts.insert(int(rng.integers(0, len(prompts))), ending[k])
        data, offs = pack(prompts)
        cut = simlib.plan_sub_batches(offs, CHUNK, 64)
        new_ends, new_gaps = set(), set()
        for k in range(len(cut) - 2):
            o0, o1, o2 = (int(offs[cut[j]]) for j in (k, k + 1, k + 2))
            at0 = simlib.workspace_layout(o0, o1 - o0, k, cut[k], 1 << 20, 1 << 16)["bytes_at"]
            at1 = simlib.workspace_layout(o1, o2 - o1, k + 1, cut[k + 1], 1 << 20, 1 << 16)["bytes_at"]
            new_ends.add((at0 + o1 - o0) % 16)
            new_gaps.add(at1 - (at0 + o1 - o0))
        if not (new_ends - ends or (1 in new_gaps and 1 not in gaps)):
            continue
        ends |= new_ends
        gaps |= new_gaps
        out.append((prompts, data, offs))
        if len(ends) == 16 and 1 in gaps:
            break
    assert len(ends) == 16 and 1 in gaps and min(gaps) >= 1, (sorted(ends), sorted(gaps))
    return out


@pytest.mark.parametrize("pipelined", [False, True])
def test_host_calls_over_stale_lane_bytes(make_context, oracle_vocabs, monkeypatch, pipelined):
    """after a call that leaves 80 80 ... (it fails with EILSEQ), spaces, digits or a special's suffix in the lane's byte buffer,
    host calls one-shot and pipelined (sub-batch gaps of 1 to 31 bytes): the oracle's ids, and truncate / chunk equal to the
    one-shot context's"""
    from cfbpe import _native as N
    batches = stale_batches()
    ref = make_context()
    if pipelined:
        monkeypatch.setenv("CFBPE_PIPE_MIN_BYTES", "1")
        monkeypatch.setenv("CFBPE_PIPE_CHUNK_BYTES", str(CHUNK))
    c = make_context()
    for bi, (prompts, data, offs) in enumerate(batches):
        n = len(prompts)
        vid = (np.arange(n) % 2).astype(np.uint8)
        budgets = np.random.default_rng(bi).integers(0, 40, n).astype(np.uint32)
        want = host_all(ref, data, offs, vid, budgets)
        for fill in (b"\x80", b" ", b"0", b"text|>"):
            junk = np.frombuffer(fill * ((len(data) + 2048) // len(fill)), np.uint8).copy()     # covers every sub-batch's slot
            jo = np.array([0, len(junk)], np.uint64)
            if fill == b"\x80":
                with pytest.raises(N.NativeError) as ei:
                    c.encode_batch(junk, jo)
                assert ei.value.code == N.EILSEQ
            else:
                c.encode_batch(junk, jo)
            got = host_all(c, data, offs, vid, budgets)
            assert_same(got, want, (bi, fill, pipelined))
            ids, off, _ = got["encode"]
            for p in range(n):
                pat = PATS[vid[p]][0]
                assert np.array_equal(ids[int(off[p]):int(off[p + 1])], oracle_vocabs[pat].encode(pat, prompts[p])), (bi, p, fill)
