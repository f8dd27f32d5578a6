"""Chunking on the H100 (cfbpe_chunk_batch / _device): against live tiktoken 0.12.0 under all four patterns, and against the
trait's host default (the chunks from cfbpe_encode_batch_starts, cfbpe.plugin.chunk_spans) at full size, in every form a host call
takes (one shot, profiling, pipelined over many sub-batches, several lanes, several devices) and on the device entry point."""
import base64
import random
import threading

import numpy as np
import pytest

import fuzzgen
from conftest import COMBOS, pack

pytestmark = pytest.mark.gpu
HEAD = 0


def context(tekken_bytes, pats=((0, 100256),), max_bytes=8 << 20, max_prompts=1 << 16, **kw):
    from cfbpe import _native as N
    c = N.Context(0, max_bytes, max_prompts, **kw)
    for slot, (pat, n) in enumerate(pats):
        c.vocab_load(slot, tekken_bytes, N.FORMAT_TIKTOKEN, pat, n)
    return c


def reference(enc, prompt: bytes, n_tok: int, overlap: int):
    """[(begin, end)] of every chunk by the contract, from live tiktoken"""
    ids = enc.encode_ordinary(prompt.decode("utf-8"))
    c, ln = len(ids), len(prompt)
    x = np.concatenate([[0], np.cumsum([len(enc.decode_single_token_bytes(t)) for t in ids])]).astype(np.int64)

    def F(j):
        if j >= c:
            return ln
        p = int(x[j])
        while 0 < p < ln and 0x80 <= prompt[p] < 0xC0:
            p -= 1
        return p
    step = n_tok - overlap
    k = 0 if c == 0 else 1 if c <= n_tok else 1 + -(-(c - n_tok) // step)
    return [(F(q * step), F(min(q * step + n_tok, c))) for q in range(k)]


def host_default(c, data, offs, vid, n_tok, overlap):
    """the trait's default: encode with starts, then the chunks on the host"""
    from cfbpe import plugin as P
    _, starts, off, counts = c.encode_batch_starts(data, offs, vid)
    spans, coffs = P.chunk_spans(data, offs, off, starts, n_tok, overlap)
    return spans, coffs, counts.copy()


def check_against_host_default(c, data, offs, vid, sizes=((512, 0), (512, 64))):
    for n_tok, overlap in sizes:
        want = host_default(c, data, offs, vid, n_tok, overlap)
        got = c.chunk_batch(data, offs, n_tok, overlap, vid)
        for g, w in zip(got, want):
            assert np.array_equal(g, w), (n_tok, overlap)


@pytest.mark.parametrize("pat,n_ranks", COMBOS)
def test_against_live_tiktoken(tekken_bytes, pat, n_ranks):
    tiktoken = pytest.importorskip("tiktoken")
    from oracle import patterns as PT
    ranks = {base64.b64decode(l.split()[0]): i for i, l in enumerate(tekken_bytes.splitlines()[:n_ranks])}
    enc = tiktoken.Encoding("live%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks, special_tokens={})
    rng = random.Random(pat)
    ext = ["".join(chr(0x20000 + rng.randrange(0xA6DF)) + rng.choice(["\U0001f600", " ", "a", "文"]) for _ in range(rng.randint(1, 20)))
           for _ in range(300)]
    texts = fuzzgen.fuzz_strings(900 + pat, 1500, max_atoms=48) + fuzzgen.long_runs(pat) + ext + ["", "x"]
    prompts = [t.encode() for t in texts]
    data, offs = pack(prompts)
    c = context(tekken_bytes, ((pat, n_ranks),))
    for n_tok, overlap in ((1, 0), (3, 2), (7, 3), (64, 0)):
        spans, coffs, counts = c.chunk_batch(data, offs, n_tok, overlap)
        for i, p in enumerate(prompts):
            got = [tuple(int(v) for v in s) for s in spans[int(coffs[i]):int(coffs[i + 1])]]
            assert got == reference(enc, p, n_tok, overlap), (n_tok, overlap, texts[i])
    c.close()


def test_config3_full_size_pipelined(tekken_bytes):
    """BASELINE.json config 3 at full size (65 536 prompts, ~134 MB): a pipelined host call"""
    from cfbpe import workload as W
    data, offs, _, _ = W.make_config(3, 1.0)
    assert int(offs[-1]) > 100 << 20 and len(offs) - 1 == 65536
    c = context(tekken_bytes, max_bytes=160 << 20, max_prompts=1 << 17)
    check_against_host_default(c, data, offs, None)
    c.close()


def test_many_sub_batches(tekken_bytes, monkeypatch):
    """sub-batches of 64 KiB: the chunk offsets chain over dozens of them on the device"""
    monkeypatch.setenv("CFBPE_PIPE_MIN_BYTES", "1")
    monkeypatch.setenv("CFBPE_PIPE_CHUNK_BYTES", str(64 << 10))
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(61, 20000, max_atoms=60) + fuzzgen.long_runs(4)] + [b"", b"x", b""]
    data, offs = pack(prompts)
    vid = (np.arange(len(prompts)) % 2).astype(np.uint8)
    c = context(tekken_bytes, ((0, 100256), (3, 130072)), max_bytes=16 << 20, max_prompts=1 << 17)
    check_against_host_default(c, data, offs, vid, ((512, 0), (512, 64), (5, 2), (1, 0)))
    c.close()


def test_one_shot_and_profiling(tekken_bytes):
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(41, 2000, max_atoms=60) + fuzzgen.long_runs(3)] + [b"", b"a", b""]
    big = "".join(random.Random(2).choice(["\U00020b9f", "x", " ", "é", "\U0001f600"]) for _ in range(40000)).encode()
    prompts.insert(7, big)
    data, offs = pack(prompts)
    assert int(offs[-1]) < 4 << 20                          # below the pipelining threshold: one pass
    vid = (np.arange(len(prompts)) % 2).astype(np.uint8)
    c = context(tekken_bytes, ((0, 100256), (3, 130072)))
    check_against_host_default(c, data, offs, vid, ((512, 0), (512, 64), (2, 1)))
    c.profile_enable(True)
    check_against_host_default(c, data, offs, vid, ((512, 64),))
    assert c.profile_read()["n_tokens"] > 0
    c.close()


def test_64mib_single_prompt(tekken_bytes):
    """one 64 MiB prompt: its tens of thousands of chunks are spread over the emit grid"""
    from cfbpe import workload as W
    data, offs, _, _ = W.make_config(3, 1.0)
    one = np.ascontiguousarray(data[:int(offs[np.searchsorted(offs, 64 << 20) - 1])])
    assert (60 << 20) < one.size <= 64 << 20
    prompts_off = np.array([0, 3, 3 + one.size], dtype=np.uint64)
    both = np.concatenate([np.frombuffer(b"abc", np.uint8), one])
    c = context(tekken_bytes, max_bytes=80 << 20, max_prompts=1 << 10)
    check_against_host_default(c, both, prompts_off, None)
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
    for n_tok, overlap in ((512, 0), (100, 30)):
        spans, coffs, counts = c.chunk_batch(data, offs, n_tok, overlap)
        m = int(coffs[-1])
        for sync in (True, False):
            d_spans = torch.full((m + 5, 2), -1, dtype=torch.int32, device=dev)
            d_coffs = torch.full((n + 1,), -1, dtype=torch.int64, device=dev)
            d_counts = torch.zeros(n, dtype=torch.int32, device=dev)
            got = c.chunk_batch_device(n, d_bytes.data_ptr(), int(offs[-1]), d_offs.data_ptr(), None, n_tok, overlap, d_spans.data_ptr(),
                                       m + 5, d_coffs.data_ptr(), d_counts.data_ptr() if sync else None, stream, sync)
            if sync:
                assert got == m
            else:
                c.device_status(stream)                        # raises on an error
            assert np.array_equal(d_spans[:m].cpu().numpy().view(np.uint32), spans)
            assert (d_spans[m:].cpu().numpy() == -1).all()
            assert np.array_equal(d_coffs.cpu().numpy().view(np.uint64), coffs)
            if sync:
                assert np.array_equal(d_counts.cpu().numpy().view(np.uint32), counts)
        # a cap one below the count: ENOSPC, synchronously with n_chunks, else from device_status; the chunks below the cap are written
        from cfbpe import _native as N
        for sync in (True, False):
            d_spans = torch.full((m, 2), -1, dtype=torch.int32, device=dev)
            d_coffs = torch.zeros(n + 1, dtype=torch.int64, device=dev)
            with pytest.raises(N.NativeError) as ei:
                c.chunk_batch_device(n, d_bytes.data_ptr(), int(offs[-1]), d_offs.data_ptr(), None, n_tok, overlap, d_spans.data_ptr(),
                                     m - 1, d_coffs.data_ptr(), None, stream, sync)
                c.device_status(stream)
            assert ei.value.code == N.ENOSPC
            assert np.array_equal(d_spans[:m - 1].cpu().numpy().view(np.uint32), spans[:m - 1])
            assert (d_spans[m - 1].cpu().numpy() == -1).all() and int(d_coffs[-1].item()) == m
    c.close()


def test_chunk0_ends_at_the_head_cut(tekken_bytes):
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(13, 3000, max_atoms=60)]
    prompts += ["".join(random.Random(k).choice(["\U00020b9f", "x", " ", "\U0001f600"]) for _ in range(200)).encode() for k in range(50)]
    data, offs = pack(prompts)
    c = context(tekken_bytes)
    for n_tok in (1, 2, 3, 17, 512):
        spans, coffs, counts = c.chunk_batch(data, offs, n_tok, 0)
        cut, _, _ = c.truncate_batch(data, offs, n_tok, HEAD)
        has = counts > 0
        assert np.array_equal(spans[coffs[:-1][has].astype(np.int64), 1], cut[has])
        ends = np.diff(offs)
        last = coffs[1:][has].astype(np.int64) - 1
        assert np.array_equal(spans[last, 1].astype(np.uint64), ends[has])          # the last chunk ends at the prompt's end
    c.close()


def test_errors(tekken_bytes):
    from cfbpe import _native as N
    c = context(tekken_bytes)
    L = N.load()
    data, offs = pack([b"hello world", b"more text here"])
    spans = np.zeros((8, 2), np.uint32)
    coffs = np.zeros(3, np.uint64)
    args = [data.ctypes.data, offs.ctypes.data, None]
    assert L.cfbpe_chunk_batch(c._h, 2, *args, 0, 0, spans.ctypes.data, 8, coffs.ctypes.data, None) == N.EINVAL
    assert L.cfbpe_chunk_batch(c._h, 2, *args, 4, 4, spans.ctypes.data, 8, coffs.ctypes.data, None) == N.EINVAL
    assert L.cfbpe_chunk_batch(c._h, 2, *args, 4, 1, None, 8, coffs.ctypes.data, None) == N.EINVAL
    assert L.cfbpe_chunk_batch(c._h, 2, *args, 4, 1, spans.ctypes.data, 8, None, None) == N.EINVAL
    assert L.cfbpe_chunk_batch_device(c._h, 0, None, 0, None, None, 0, 0, None, 0, None, None, None, None) == N.EINVAL
    assert L.cfbpe_chunk_batch(c._h, 2, *args, 1, 0, spans.ctypes.data, 1, coffs.ctypes.data, None) == N.ENOSPC
    need = int(coffs[2])                                    # one-token chunks: as many as tokens
    assert need == len(c.encode_batch(data, offs)[0]) and need > 1
    big = np.zeros((need, 2), np.uint32)
    assert L.cfbpe_chunk_batch(c._h, 2, *args, 1, 0, big.ctypes.data, need, coffs.ctypes.data, None) == N.OK
    with pytest.raises(N.NativeError) as ei:
        c.chunk_batch(*pack([b"fine", b"bad \xff here"]), 4)
    assert ei.value.code == N.EILSEQ
    with pytest.raises(N.NativeError) as ei:
        c.chunk_batch(data, offs, 4, 0, np.array([0, 3], np.uint8))
    assert ei.value.code == N.ENOENT
    sp, co, cnt = c.chunk_batch(data, offs, 2)              # the context works after the failures
    assert co.tolist() == [0, -(-int(cnt[0]) // 2), -(-int(cnt[0]) // 2) - (-int(cnt[1]) // 2)]
    c.close()


def test_two_threads_on_two_lanes(tekken_bytes):
    c = context(tekken_bytes, max_bytes=16 << 20, max_prompts=1 << 17, n_workspaces=2)
    batches = [pack([s.encode() for s in fuzzgen.fuzz_strings(seed, 20000, max_atoms=40)]) for seed in (5, 6)]
    want_enc = [tuple(x.copy() for x in c.encode_batch(d, o)) for d, o in batches]
    want_chunks = [tuple(x.copy() for x in c.chunk_batch(d, o, 16, 4)) for d, o in batches]
    errors = []

    def run(k):
        try:
            d, o = batches[k]
            for _ in range(6):
                if k == 0:
                    got = c.chunk_batch(d, o, 16, 4)
                    assert all(np.array_equal(g, w) for g, w in zip(got, want_chunks[0]))
                else:
                    got = c.encode_batch(d, o)
                    assert all(np.array_equal(g, w) for g, w in zip(got, want_enc[1]))
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
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(78, 40000, max_atoms=60) + fuzzgen.long_runs(5)] + [b"", b"x", b""]
    data, offs = pack(prompts)
    vid = (np.arange(len(prompts)) % 2).astype(np.uint8)
    one = context(tekken_bytes, ((0, 100256), (3, 130072)), max_bytes=64 << 20, max_prompts=1 << 17)
    want = [tuple(x.copy() for x in one.chunk_batch(data, offs, n, s, vid)) for n, s in ((512, 64), (3, 1))]
    one.close()
    c = context(tekken_bytes, ((0, 100256), (3, 130072)), max_bytes=64 << 20, max_prompts=1 << 17,
                devices=list(range(min(torch.cuda.device_count(), 8))))
    for (n, s), w in zip(((512, 64), (3, 1)), want):
        got = c.chunk_batch(data, offs, n, s, vid)
        assert all(np.array_equal(g, x) for g, x in zip(got, w))
    c.close()


def test_plugin_device_path_equals_trait_default():
    """GpuBpeTokenizerPlugin.chunk_batch (the device call) equals TokenizerPluginClient.chunk_batch (encode with starts, the chunks
    on the host) on the same plugin and inputs; the service's chunks join back into the texts"""
    from cfbpe import plugin as P
    plug = P.GpuBpeTokenizerPlugin(device=0, vocab_names=("cl100k_base", "tekken"), max_batch_bytes=8 << 20, max_prompts=1 << 16,
                                   allow_stand_in=True)
    sec = P.SecurityContext.anonymous()
    texts = fuzzgen.fuzz_strings(1234, 800, max_atoms=40) + ["", "Hello, world! " * 40, "\U00020000\U0001f600" * 30]
    data, offs = P.pack_texts(texts)
    for model in ("cl100k_base", "tekken"):
        req = P.EncodeBatchRequest(P.VocabRef(model), data, offs)
        for n_tok, overlap in ((5, 0), (9, 4), (512, 64)):
            dev = plug.chunk_batch(sec, req, n_tok, overlap)
            host = P.TokenizerPluginClient.chunk_batch(plug, sec, req, n_tok, overlap)
            assert np.array_equal(dev.spans, host.spans) and np.array_equal(dev.chunk_offsets, host.chunk_offsets)
            assert np.array_equal(dev.counts, host.counts)
    hub = P.ClientHub()
    hub.register_scoped(P.TokenizerPluginClient, plug.instance.id, plug)
    svc = P.LlmGatewayTokenizerService(hub, [plug.instance])
    for t, chunks in zip(texts, svc.chunk(sec, "cl100k_base", texts, 7)):
        assert "".join(chunks) == t
    plug.close()
