"""Token starts in code points and UTF-16 units on the H100 (cfbpe_encode_batch_char_starts / _device): against live tiktoken 0.12.0
`decode_with_offsets`, against the host reference (cfbpe.plugin.unit_starts over the byte starts) at full size and on every
Unicode scalar value, and the ids / offsets / counts of cfbpe_encode_batch on the same inputs, in every form a host call takes
(one shot, profiling, pipelined in large and tiny sub-batches, several lanes, several devices) and through the device entry point."""
import base64
import ctypes as C
import threading

import numpy as np
import pytest

import fuzzgen
from conftest import COMBOS, pack

pytestmark = pytest.mark.gpu

UNITS = ("codepoint", "utf16")
MULTILINGUAL = ["Grüße aus Köln", "日本語のテキストです。", "Привет, мир!", "مرحبا بالعالم", "emoji 😀👍🏽🎉 🇩🇪", "family 👨‍👩‍👧‍👦",
                "CJK Ext B 𠀀𠀁𠀂𪚥 𝔘𝔫𝔦𝔠𝔬𝔡𝔢", "😀" * 40, "𠀀" * 33, ""]


def native_unit(unit):
    from cfbpe import _native as N
    return {"codepoint": N.UNIT_CODEPOINT, "utf16": N.UNIT_UTF16}[unit]


def context(tekken_bytes, pats=((0, 100256),), max_bytes=8 << 20, max_prompts=1 << 16, **kw):
    from cfbpe import _native as N
    c = N.Context(0, max_bytes, max_prompts, **kw)
    for slot, (pat, n) in enumerate(pats):
        c.vocab_load(slot, tekken_bytes, N.FORMAT_TIKTOKEN, pat, n)
    return c


def check_against_plain(c, data, offs, vid=None, units=UNITS):
    """both units: ids / offsets / counts equal cfbpe_encode_batch's, starts and lengths equal unit_starts over the byte starts"""
    from cfbpe.plugin import unit_starts
    ids, off, counts = (x.copy() for x in c.encode_batch(data, offs, vid))
    _, bstarts, _, _ = (x.copy() for x in c.encode_batch_starts(data, offs, vid))
    out = {}
    for unit in units:
        uids, starts, uoff, ucounts, lens = c.encode_batch_char_starts(data, offs, native_unit(unit), vid)
        assert np.array_equal(uids, ids) and np.array_equal(uoff, off) and np.array_equal(ucounts, counts)
        want, want_lens = unit_starts(data, offs, off, bstarts, unit)
        assert np.array_equal(starts, want), unit
        assert np.array_equal(lens, want_lens), unit
        out[unit] = (starts.copy(), lens.copy())
    return ids, off, out


@pytest.mark.parametrize("pat,n_ranks", COMBOS)
def test_against_live_tiktoken(tekken_bytes, pat, n_ranks):
    tiktoken = pytest.importorskip("tiktoken")
    from oracle import patterns as PT
    ranks = {base64.b64decode(l.split()[0]): i for i, l in enumerate(tekken_bytes.splitlines()[:n_ranks])}
    enc = tiktoken.Encoding("live%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks, special_tokens={})
    texts = fuzzgen.fuzz_strings(950 + pat, 3000, max_atoms=48) + fuzzgen.long_runs(pat) + MULTILINGUAL + ["", "x"]
    c = context(tekken_bytes, ((pat, n_ranks),))
    data, offs = pack([t.encode() for t in texts])
    ids, off, got = check_against_plain(c, data, offs)
    starts, lens = got["codepoint"]
    for i, t in enumerate(texts):
        a, b = int(off[i]), int(off[i + 1])
        assert ids[a:b].tolist() == enc.encode_ordinary(t)
        assert starts[a:b].tolist() == enc.decode_with_offsets(ids[a:b].tolist())[1], repr(t)
        assert int(lens[i]) == len(t) and int(got["utf16"][1][i]) == len(t.encode("utf-16-le")) // 2
    c.close()


def test_config3_full_size_pipelined(tekken_bytes):
    """BASELINE.json config 3 at full size (65 536 prompts, ~134 MB): a pipelined host call against the numpy reference"""
    from cfbpe import workload as W
    data, offs, _, _ = W.make_config(3, 1.0)
    assert int(offs[-1]) > 100 << 20 and len(offs) - 1 == 65536
    c = context(tekken_bytes, max_bytes=160 << 20, max_prompts=1 << 17)
    check_against_plain(c, data, offs)
    c.close()


def test_one_shot_and_profiling(tekken_bytes):
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(43, 2000, max_atoms=60) + fuzzgen.long_runs(3) + MULTILINGUAL] + [b"", b"a", b""]
    data, offs = pack(prompts)
    assert int(offs[-1]) < 4 << 20                          # below the pipelining threshold: one pass
    vid = (np.arange(len(prompts)) % 2).astype(np.uint8)
    c = context(tekken_bytes, ((0, 100256), (3, 130072)))
    check_against_plain(c, data, offs, vid)
    c.profile_enable(True)
    check_against_plain(c, data, offs, vid)
    assert c.profile_read()["n_tokens"] > 0
    c.close()


def test_tiny_sub_batches(tekken_bytes, monkeypatch):
    """sub-batches of a few KiB: many prompts, each sub-batch's lengths at its prompts' places"""
    monkeypatch.setenv("CFBPE_PIPE_MIN_BYTES", "1")
    monkeypatch.setenv("CFBPE_PIPE_CHUNK_BYTES", "4096")
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(44, 3000, max_atoms=30) + MULTILINGUAL * 20] + [b"", "😀".encode() * 3000, b""]
    c = context(tekken_bytes, ((0, 100256), (3, 130072)))
    data, offs = pack(prompts)
    check_against_plain(c, data, offs, (np.arange(len(prompts)) % 2).astype(np.uint8))
    c.close()


def test_every_unicode_scalar_value(tekken_bytes):
    """every scalar value U+0000 .. U+10FFFF (no surrogates) once, in prompts of 1000 characters, through every stand-in slot"""
    cps = [c for c in range(0x110000) if not 0xD800 <= c < 0xE000]
    texts = ["".join(map(chr, cps[i:i + 1000])) for i in range(0, len(cps), 1000)]
    data, offs = pack([t.encode() for t in texts])
    c = context(tekken_bytes, tuple(COMBOS), max_bytes=16 << 20)
    for slot in range(len(COMBOS)):
        vid = np.full(len(texts), slot, dtype=np.uint8)
        _, _, got = check_against_plain(c, data, offs, vid)
        assert got["codepoint"][1].tolist() == [len(t) for t in texts]
        assert got["utf16"][1].tolist() == [len(t.encode("utf-16-le")) // 2 for t in texts]
    c.close()


def test_device_entry_point_equals_host_call(tekken_bytes):
    import torch
    from cfbpe import workload as W
    data, offs, _, _ = W.make_config(2, 1.0)
    c = context(tekken_bytes, max_bytes=64 << 20, max_prompts=1 << 17)
    dev = torch.device("cuda:0")
    n = len(offs) - 1
    d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).to(dev)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    stream = torch.cuda.current_stream().cuda_stream
    for unit in UNITS:
        ids, starts, off, counts, lens = (x.copy() for x in c.encode_batch_char_starts(data, offs, native_unit(unit)))
        for sync in (True, False):
            d_ids = torch.zeros(len(data) + 1, dtype=torch.int32, device=dev)
            d_starts = torch.full((len(data) + 1,), -1, dtype=torch.int32, device=dev)
            d_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
            d_counts = torch.zeros(n, dtype=torch.int32, device=dev)
            d_lens = torch.full((n,), -1, dtype=torch.int32, device=dev)
            nt = c.encode_batch_char_starts_device(n, d_bytes.data_ptr(), int(offs[-1]), d_offs.data_ptr(), None, native_unit(unit),
                                                   d_ids.data_ptr(), d_starts.data_ptr(), d_ids.numel(), d_off.data_ptr(), d_counts.data_ptr(),
                                                   d_lens.data_ptr(), stream, sync=sync)
            if sync:
                assert nt == len(ids)
            else:
                c.device_status(stream)
            m = len(ids)
            assert np.array_equal(d_ids[:m].cpu().numpy().view(np.uint32), ids)
            assert np.array_equal(d_starts[:m].cpu().numpy().view(np.uint32), starts)
            assert np.array_equal(d_off.cpu().numpy().astype(np.uint64), off)
            assert np.array_equal(d_counts.cpu().numpy().view(np.uint32), counts)
            assert np.array_equal(d_lens.cpu().numpy().view(np.uint32), lens)
        # the lengths are optional on the device too
        d_starts = torch.full((len(data) + 1,), -1, dtype=torch.int32, device=dev)
        c.encode_batch_char_starts_device(n, d_bytes.data_ptr(), int(offs[-1]), d_offs.data_ptr(), None, native_unit(unit), d_ids.data_ptr(),
                                          d_starts.data_ptr(), d_ids.numel(), d_off.data_ptr(), d_counts.data_ptr(), None, stream)
        assert np.array_equal(d_starts[:len(ids)].cpu().numpy().view(np.uint32), starts)
    c.close()


def test_errors(tekken_bytes):
    from cfbpe import _native as N
    c = context(tekken_bytes)
    L = N.load()
    data, offs = pack([b"hello world", "more text 😀 here".encode()])
    ids = np.zeros(64, np.uint32)
    starts = np.zeros(64, np.uint32)
    o = np.zeros(3, np.uint64)
    cnt = np.zeros(2, np.uint32)
    lens = np.zeros(2, np.uint32)
    args = lambda unit, i, s: (c._h, 2, data.ctypes.data, offs.ctypes.data, None, unit, i, s, 64, o.ctypes.data, cnt.ctypes.data, lens.ctypes.data)
    assert L.cfbpe_encode_batch_char_starts(*args(N.UNIT_CODEPOINT, ids.ctypes.data, None)) == N.EINVAL
    assert L.cfbpe_encode_batch_char_starts(*args(N.UNIT_UTF16, None, starts.ctypes.data)) == N.EINVAL
    assert L.cfbpe_encode_batch_char_starts(*args(2, ids.ctypes.data, starts.ctypes.data)) == N.EINVAL
    nt = C.c_uint64(0)
    assert L.cfbpe_encode_batch_char_starts_device(c._h, 0, None, 0, None, None, N.UNIT_UTF16, None, None, 0, None, None, None, C.byref(nt),
                                                   None) == N.EINVAL
    assert L.cfbpe_encode_batch_char_starts_device(c._h, 0, None, 0, None, None, 7, None, None, 0, None, None, None, C.byref(nt), None) == N.EINVAL
    want_n = len(c.encode_batch(data, offs)[0])
    for unit in (N.UNIT_CODEPOINT, N.UNIT_UTF16):
        with pytest.raises(N.NativeError) as ei:
            c.encode_batch_char_starts(data, offs, unit, out_ids=np.zeros(2, np.uint32), out_offsets=o)
        assert ei.value.code == N.ENOSPC and int(o[2]) == want_n
    with pytest.raises(N.NativeError) as ei:
        c.encode_batch_char_starts(*pack([b"fine", b"bad \xff here"]), N.UNIT_UTF16)
    assert ei.value.code == N.EILSEQ
    _, st, _, _, ln = c.encode_batch_char_starts(data, offs, N.UNIT_UTF16)       # the context works after the failures
    assert st.tolist()[:1] == [0] and ln.tolist() == [11, len("more text 😀 here".encode("utf-16-le")) // 2]
    c.close()


def test_two_threads_on_two_lanes(tekken_bytes):
    from cfbpe.plugin import unit_starts
    c = context(tekken_bytes, max_bytes=16 << 20, max_prompts=1 << 17, n_workspaces=2)
    batches = [pack([s.encode() for s in fuzzgen.fuzz_strings(seed, 20000, max_atoms=40) + MULTILINGUAL]) for seed in (7, 8)]
    want = []
    for d, o in batches:
        ids, bst, off, _ = (x.copy() for x in c.encode_batch_starts(d, o))
        want.append((ids, off, unit_starts(d, o, off, bst, "utf16")))
    errors = []

    def run(k):
        try:
            d, o = batches[k]
            for _ in range(6):
                if k == 0:
                    ids, st, off, _, lens = c.encode_batch_char_starts(d, o, native_unit("utf16"))
                    assert np.array_equal(st, want[k][2][0]) and np.array_equal(lens, want[k][2][1])
                else:
                    ids, off, _ = c.encode_batch(d, o)
                assert np.array_equal(ids, want[k][0]) and np.array_equal(off, want[k][1])
        except Exception as e:          # noqa: BLE001 -- reported below
            errors.append(e)
    th = [threading.Thread(target=run, args=(k,)) for k in (0, 1)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
    c.close()


@pytest.mark.skipif("__import__('torch').cuda.device_count() < 2")
@pytest.mark.parametrize("mode", ["shards", "round_robin"])
def test_multi_device(tekken_bytes, mode, monkeypatch):
    import torch
    if mode == "round_robin":
        monkeypatch.setenv("CFBPE_PIPE_MIN_BYTES", "1")
        monkeypatch.setenv("CFBPE_PIPE_CHUNK_BYTES", str(64 << 10))
    else:
        monkeypatch.setenv("CFBPE_NO_PEER", "1")
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(79, 40000, max_atoms=60) + fuzzgen.long_runs(5) + MULTILINGUAL] + [b"", b"x", b""]
    data, offs = pack(prompts)
    vid = (np.arange(len(prompts)) % 2).astype(np.uint8)
    pats = ((0, 100256), (3, 130072))
    one = context(tekken_bytes, pats, max_bytes=64 << 20, max_prompts=1 << 17)
    _, _, want = check_against_plain(one, data, offs, vid)
    one.close()
    c = context(tekken_bytes, pats, max_bytes=64 << 20, max_prompts=1 << 17, devices=list(range(min(torch.cuda.device_count(), 8))))
    _, _, got = check_against_plain(c, data, offs, vid)
    for unit in UNITS:
        assert np.array_equal(got[unit][0], want[unit][0]) and np.array_equal(got[unit][1], want[unit][1])
    c.close()


def test_encode_with_offsets_spans_slice_each_string():
    from cfbpe import plugin as P
    plug = P.GpuBpeTokenizerPlugin(device=0, vocab_names=("cl100k_base", "tekken"), max_batch_bytes=8 << 20, max_prompts=1 << 16,
                                   allow_stand_in=True)
    hub = P.ClientHub()
    hub.register_scoped(P.TokenizerPluginClient, plug.instance.id, plug)
    svc = P.LlmGatewayTokenizerService(hub, [plug.instance])
    ctx = P.SecurityContext.anonymous()
    texts = fuzzgen.fuzz_strings(1235, 800, max_atoms=40) + MULTILINGUAL + ["Hello, 世界! 😀 " * 40]
    for model in ("cl100k_base", "tekken"):
        plain = svc.encode(ctx, model, texts)
        for unit in ("byte", "codepoint", "utf16"):
            got = svc.encode_with_offsets(ctx, model, texts, unit=unit)
            for t, (ids, spans), want_ids in zip(texts, got, plain):
                s = t.encode() if unit == "byte" else t if unit == "codepoint" else t.encode("utf-16-le")
                w = 2 if unit == "utf16" else 1
                assert np.array_equal(ids, want_ids)
                assert type(s)().join(s[int(a) * w:int(e) * w] for a, e in spans) == s, (unit, t)
                assert all(int(a) <= int(e) for a, e in spans)
    plug.close()
