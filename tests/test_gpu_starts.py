"""Token byte starts on the H100 (cfbpe_encode_batch_starts / _device): against live tiktoken 0.12.0 `decode_with_offsets`, the
prefix-sum rule at full size, and the ids / offsets / counts of cfbpe_encode_batch on the same inputs, in every form a host call
takes (one shot, profiling, pipelined, several lanes, several devices)."""
import base64
import ctypes as C
import os
import threading

import numpy as np
import pytest

import fuzzgen
from conftest import COMBOS, pack

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tok_lens(tekken_bytes):
    """byte length of every rank of the committed rank file (every slot, stand-ins included, keeps a prefix of it)"""
    return np.array([len(base64.b64decode(l.split()[0])) for l in tekken_bytes.splitlines()], dtype=np.int64)


def context(tekken_bytes, pats=((0, 100256),), max_bytes=8 << 20, max_prompts=1 << 16, **kw):
    from cfbpe import _native as N
    c = N.Context(0, max_bytes, max_prompts, **kw)
    for slot, (pat, n) in enumerate(pats):
        c.vocab_load(slot, tekken_bytes, N.FORMAT_TIKTOKEN, pat, n)
    return c


def check_starts(ids, starts, off, counts, offs, tok_lens):
    """every start = the bytes of the prompt's tokens before it (numpy, whole batch at once)"""
    lens = tok_lens[ids]
    excl = np.cumsum(lens) - lens                          # byte position of every token in the batch
    prompt_start = np.repeat(offs[:-1].astype(np.int64), counts.astype(np.int64))
    assert np.array_equal(starts.astype(np.int64), excl - prompt_start)
    assert int(lens.sum()) == int(offs[-1])


def check_against_plain(c, data, offs, vid, tok_lens):
    ids, off, counts = c.encode_batch(data, offs, vid)
    ids, off, counts = ids.copy(), off.copy(), counts.copy()
    sids, starts, soff, scounts = c.encode_batch_starts(data, offs, vid)
    assert np.array_equal(sids, ids) and np.array_equal(soff, off) and np.array_equal(scounts, counts)
    check_starts(sids, starts, soff, scounts, offs, tok_lens)
    return sids, starts, soff


@pytest.mark.parametrize("pat,n_ranks", COMBOS)
def test_against_live_tiktoken(tekken_bytes, pat, n_ranks):
    tiktoken = pytest.importorskip("tiktoken")
    from oracle import patterns as PT
    ranks = {base64.b64decode(l.split()[0]): i for i, l in enumerate(tekken_bytes.splitlines()[:n_ranks])}
    enc = tiktoken.Encoding("live%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks, special_tokens={})
    texts = fuzzgen.fuzz_strings(900 + pat, 3000, max_atoms=48) + fuzzgen.long_runs(pat) + ["", "x"]
    prompts = [t.encode() for t in texts]
    c = context(tekken_bytes, ((pat, n_ranks),))
    ids, starts, off, _ = c.encode_batch_starts(*pack(prompts))
    for i, (t, p) in enumerate(zip(texts, prompts)):
        a, b = int(off[i]), int(off[i + 1])
        want_ids = enc.encode_ordinary(t)
        assert ids[a:b].tolist() == want_ids
        _, want = enc.decode_with_offsets(want_ids)
        got = []
        for s in starts[a:b].tolist():      # tiktoken's byte -> character rule
            chars = sum(1 for ch in p[:s] if not 0x80 <= ch < 0xC0)
            got.append(max(0, chars - (1 if 0x80 <= p[s] < 0xC0 else 0)))
        assert got == want, repr(t)
    c.close()


def test_config3_full_size_pipelined(tekken_bytes, tok_lens):
    """BASELINE.json config 3 at full size (65 536 prompts, ~134 MB): a pipelined host call"""
    from cfbpe import workload as W
    data, offs, _, _ = W.make_config(3, 1.0)
    assert int(offs[-1]) > 100 << 20 and len(offs) - 1 == 65536
    c = context(tekken_bytes, max_bytes=160 << 20, max_prompts=1 << 17)
    check_against_plain(c, data, offs, None, tok_lens)
    c.close()


def test_one_shot_and_profiling(tekken_bytes, tok_lens):
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(41, 2000, max_atoms=60) + fuzzgen.long_runs(3)] + [b"", b"a", b""]
    data, offs = pack(prompts)
    assert int(offs[-1]) < 4 << 20                          # below the pipelining threshold: one pass
    vid = (np.arange(len(prompts)) % 2).astype(np.uint8)
    c = context(tekken_bytes, ((0, 100256), (3, 130072)))
    check_against_plain(c, data, offs, vid, tok_lens)
    c.profile_enable(True)
    check_against_plain(c, data, offs, vid, tok_lens)
    assert c.profile_read()["n_tokens"] > 0
    c.close()


def test_device_entry_point_equals_host_call(tekken_bytes, tok_lens):
    import torch
    from cfbpe import workload as W
    data, offs, _, _ = W.make_config(2, 1.0)
    c = context(tekken_bytes, max_bytes=64 << 20, max_prompts=1 << 17)
    ids, starts, off, counts = c.encode_batch_starts(data, offs)
    dev = torch.device("cuda:0")
    n = len(offs) - 1
    d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).to(dev)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    stream = torch.cuda.current_stream().cuda_stream
    for sync in (True, False):
        d_ids = torch.zeros(len(data) + 1, dtype=torch.int32, device=dev)
        d_starts = torch.full((len(data) + 1,), -1, dtype=torch.int32, device=dev)
        d_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        d_counts = torch.zeros(n, dtype=torch.int32, device=dev)
        nt = c.encode_batch_starts_device(n, d_bytes.data_ptr(), int(offs[-1]), d_offs.data_ptr(), None, d_ids.data_ptr(), d_starts.data_ptr(),
                                          d_ids.numel(), d_off.data_ptr(), d_counts.data_ptr(), stream, sync=sync)
        if sync:
            assert nt == len(ids)
        else:
            c.device_status(stream)
        m = len(ids)
        assert np.array_equal(d_ids[:m].cpu().numpy().view(np.uint32), ids)
        assert np.array_equal(d_starts[:m].cpu().numpy().view(np.uint32), starts)
        assert np.array_equal(d_off.cpu().numpy().astype(np.uint64), off)
        assert np.array_equal(d_counts.cpu().numpy().view(np.uint32), counts)
    c.close()


def test_errors(tekken_bytes):
    from cfbpe import _native as N
    c = context(tekken_bytes)
    L = N.load()
    data, offs = pack([b"hello world", b"more text here"])
    ids = np.zeros(64, np.uint32)
    starts = np.zeros(64, np.uint32)
    o = np.zeros(3, np.uint64)
    cnt = np.zeros(2, np.uint32)
    assert L.cfbpe_encode_batch_starts(c._h, 2, data.ctypes.data, offs.ctypes.data, None, ids.ctypes.data, None, 64, o.ctypes.data,
                                       cnt.ctypes.data) == N.EINVAL
    assert L.cfbpe_encode_batch_starts(c._h, 2, data.ctypes.data, offs.ctypes.data, None, None, starts.ctypes.data, 64, o.ctypes.data,
                                       cnt.ctypes.data) == N.EINVAL
    nt = C.c_uint64(0)
    assert L.cfbpe_encode_batch_starts_device(c._h, 0, None, 0, None, None, None, None, 0, None, None, C.byref(nt), None) == N.EINVAL
    want_n = len(c.encode_batch(data, offs)[0])
    with pytest.raises(N.NativeError) as ei:
        c.encode_batch_starts(data, offs, out_ids=np.zeros(2, np.uint32), out_offsets=o)
    assert ei.value.code == N.ENOSPC and int(o[2]) == want_n
    with pytest.raises(N.NativeError) as ei:
        c.encode_batch_starts(*pack([b"fine", b"bad \xff here"]))
    assert ei.value.code == N.EILSEQ
    _, st, _, _ = c.encode_batch_starts(data, offs)           # the context works after the failures
    assert st.tolist()[:1] == [0]
    c.close()


def test_two_threads_on_two_lanes(tekken_bytes, tok_lens):
    c = context(tekken_bytes, max_bytes=16 << 20, max_prompts=1 << 17, n_workspaces=2)
    batches = [pack([s.encode() for s in fuzzgen.fuzz_strings(seed, 20000, max_atoms=40)]) for seed in (5, 6)]
    want = [c.encode_batch(d, o) for d, o in batches]
    want = [(a.copy(), b.copy(), x.copy()) for a, b, x in want]
    errors = []

    def run(k):
        try:
            d, o = batches[k]
            for _ in range(6):
                if k == 0:
                    ids, st, off, counts = c.encode_batch_starts(d, o)
                    check_starts(ids, st, off, counts, o, tok_lens)
                else:
                    ids, off, counts = c.encode_batch(d, o)
                assert np.array_equal(ids, want[k][0]) and np.array_equal(off, want[k][1]) and np.array_equal(counts, want[k][2])
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
def test_multi_device(tekken_bytes, tok_lens, mode, monkeypatch):
    import torch
    if mode == "round_robin":
        monkeypatch.setenv("CFBPE_PIPE_MIN_BYTES", "1")
        monkeypatch.setenv("CFBPE_PIPE_CHUNK_BYTES", str(64 << 10))
    else:
        monkeypatch.setenv("CFBPE_NO_PEER", "1")
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(78, 40000, max_atoms=60) + fuzzgen.long_runs(5)] + [b"", b"x", b""]
    data, offs = pack(prompts)
    vid = (np.arange(len(prompts)) % 2).astype(np.uint8)
    one = context(tekken_bytes, ((0, 100256), (3, 130072)), max_bytes=64 << 20, max_prompts=1 << 17)
    want = one.encode_batch(data, offs, vid)
    want = tuple(x.copy() for x in want)
    one.close()
    c = context(tekken_bytes, ((0, 100256), (3, 130072)), max_bytes=64 << 20, max_prompts=1 << 17,
                devices=list(range(min(torch.cuda.device_count(), 8))))
    ids, st, off, counts = c.encode_batch_starts(data, offs, vid)
    assert np.array_equal(ids, want[0]) and np.array_equal(off, want[1]) and np.array_equal(counts, want[2])
    check_starts(ids, st, off, counts, offs, tok_lens)
    c.close()


def test_encode_with_offsets_spans_rebuild_each_text():
    from cfbpe import plugin as P
    plug = P.GpuBpeTokenizerPlugin(device=0, vocab_names=("cl100k_base", "tekken"), max_batch_bytes=8 << 20, max_prompts=1 << 16,
                                   allow_stand_in=True)
    hub = P.ClientHub()
    hub.register_scoped(P.TokenizerPluginClient, plug.instance.id, plug)
    svc = P.LlmGatewayTokenizerService(hub, [plug.instance])
    ctx = P.SecurityContext.anonymous()
    texts = fuzzgen.fuzz_strings(1234, 800, max_atoms=40) + ["", "Hello, world! " * 40]
    for model in ("cl100k_base", "tekken"):
        got = svc.encode_with_offsets(ctx, model, texts)
        plain = svc.encode(ctx, model, texts)
        for t, (ids, spans), want_ids in zip(texts, got, plain):
            b = t.encode()
            assert np.array_equal(ids, want_ids)
            assert b"".join(b[int(s):int(e)] for s, e in spans) == b
            assert all(int(s) < int(e) for s, e in spans)
    plug.close()
