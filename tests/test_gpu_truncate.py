"""Truncation to token budgets on the H100 (cfbpe_truncate_batch / _device): against live tiktoken 0.12.0 under all four patterns,
and against the trait's host default (the cut from cfbpe_encode_batch_starts, cfbpe.plugin.truncate_cuts) at full size, in every
form a host call takes (one shot, profiling, pipelined, several lanes, several devices) and on the device entry point."""
import base64
import random
import threading

import numpy as np
import pytest

import fuzzgen
from conftest import COMBOS, pack

pytestmark = pytest.mark.gpu
HEAD, TAIL = 0, 1


def context(tekken_bytes, pats=((0, 100256),), max_bytes=8 << 20, max_prompts=1 << 16, **kw):
    from cfbpe import _native as N
    c = N.Context(0, max_bytes, max_prompts, **kw)
    for slot, (pat, n) in enumerate(pats):
        c.vocab_load(slot, tekken_bytes, N.FORMAT_TIKTOKEN, pat, n)
    return c


def reference(enc, prompt: bytes, budget: int, mode: int):
    """(cut, kept, count) by the contract: decode_bytes of the first / last k ids, moved to a character boundary"""
    ids = enc.encode_ordinary(prompt.decode("utf-8"))
    c, n = len(ids), len(prompt)
    k = min(budget, c)
    lens = np.array([len(enc.decode_single_token_bytes(t)) for t in ids], dtype=np.int64)
    if mode == HEAD:
        cut = len(enc.decode_bytes(ids[:k]))
        while 0 < cut < n and 0x80 <= prompt[cut] < 0xC0:
            cut -= 1
        return cut, int((np.cumsum(lens) <= cut).sum()), c
    cut = n - len(enc.decode_bytes(ids[c - k:]))
    while cut < n and 0x80 <= prompt[cut] < 0xC0:
        cut += 1
    return cut, int(((np.cumsum(lens) - lens) >= cut).sum()), c


def host_default(c, data, offs, vid, budgets, mode):
    """the trait's default: encode with starts, then the cut on the host"""
    from cfbpe import plugin as P
    _, starts, off, counts = c.encode_batch_starts(data, offs, vid)
    cut, kept = P.truncate_cuts(data, offs, off, starts, budgets, mode == TAIL)
    return cut, kept, counts.copy()


def check_against_host_default(c, data, offs, vid, budgets):
    for mode in (HEAD, TAIL):
        want = host_default(c, data, offs, vid, budgets, mode)
        got = c.truncate_batch(data, offs, budgets, mode, vid)
        for g, w in zip(got, want):
            assert np.array_equal(g, w), mode


def half_cut_budgets(c, data, offs, vid, seed):
    """budgets that cut about half the prompts: between 0.5x and 1.5x of each prompt's count"""
    counts = c.count_batch(data, offs, vid).astype(np.int64)
    rng = np.random.default_rng(seed)
    return (counts * rng.uniform(0.5, 1.5, len(counts))).astype(np.uint32)


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
    counts = c.count_batch(data, offs)
    for mode in (HEAD, TAIL):
        budgets = np.array([[0, 1, max(int(n) - 1, 0), int(n), int(n) + 1, 2 ** 32 - 1, int(n) // 2, rng.randint(0, int(n) + 1)][i % 8]
                            for i, n in enumerate(counts)], dtype=np.uint32)
        cut, kept, cnt = c.truncate_batch(data, offs, budgets, mode)
        for i, p in enumerate(prompts):
            assert (int(cut[i]), int(kept[i]), int(cnt[i])) == reference(enc, p, int(budgets[i]), mode), (mode, int(budgets[i]), texts[i])
    c.close()


def test_config3_full_size_pipelined(tekken_bytes):
    """BASELINE.json config 3 at full size (65 536 prompts, ~134 MB): a pipelined host call, about half the prompts cut"""
    from cfbpe import workload as W
    data, offs, _, _ = W.make_config(3, 1.0)
    assert int(offs[-1]) > 100 << 20 and len(offs) - 1 == 65536
    c = context(tekken_bytes, max_bytes=160 << 20, max_prompts=1 << 17)
    budgets = half_cut_budgets(c, data, offs, None, 3)
    counts = c.count_batch(data, offs)
    assert 0.35 < float((budgets < counts).mean()) < 0.65
    check_against_host_default(c, data, offs, None, budgets)
    check_against_host_default(c, data, offs, None, np.full(len(offs) - 1, 512, np.uint32))
    c.close()


def test_one_shot_and_profiling(tekken_bytes):
    prompts = [s.encode() for s in fuzzgen.fuzz_strings(41, 2000, max_atoms=60) + fuzzgen.long_runs(3)] + [b"", b"a", b""]
    big = "".join(random.Random(2).choice(["\U00020b9f", "x", " ", "é", "\U0001f600"]) for _ in range(40000)).encode()
    prompts.insert(7, big)                                   # more ids to sum than one warp takes: truncate_long
    data, offs = pack(prompts)
    assert int(offs[-1]) < 4 << 20                          # below the pipelining threshold: one pass
    vid = (np.arange(len(prompts)) % 2).astype(np.uint8)
    c = context(tekken_bytes, ((0, 100256), (3, 130072)))
    budgets = half_cut_budgets(c, data, offs, vid, 1)
    budgets[7] = c.count_batch(data, offs, vid)[7] // 2
    check_against_host_default(c, data, offs, vid, budgets)
    c.profile_enable(True)
    check_against_host_default(c, data, offs, vid, budgets)
    assert c.profile_read()["n_tokens"] > 0
    c.close()


def test_device_entry_point_equals_host_call(tekken_bytes):
    import torch
    from cfbpe import workload as W
    data, offs, _, _ = W.make_config(2, 1.0)
    c = context(tekken_bytes, max_bytes=64 << 20, max_prompts=1 << 17)
    budgets = half_cut_budgets(c, data, offs, None, 2)
    dev = torch.device("cuda:0")
    n = len(offs) - 1
    d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).to(dev)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    d_bud = torch.from_numpy(budgets.view(np.int32)).to(dev)
    stream = torch.cuda.current_stream().cuda_stream
    for mode in (HEAD, TAIL):
        want = c.truncate_batch(data, offs, budgets, mode)
        for sync in (True, False):
            d_cut = torch.full((n,), -1, dtype=torch.int32, device=dev)
            d_kept = torch.full((n,), -1, dtype=torch.int32, device=dev)
            d_counts = torch.zeros(n, dtype=torch.int32, device=dev)
            c.truncate_batch_device(n, d_bytes.data_ptr(), int(offs[-1]), d_offs.data_ptr(), None, d_bud.data_ptr(), mode,
                                    d_cut.data_ptr(), d_kept.data_ptr(), d_counts.data_ptr() if sync else None, stream)
            if sync:
                c.device_status(stream)                        # raises on an error
            assert np.array_equal(d_cut.cpu().numpy().view(np.uint32), want[0])      # (.cpu() waits for the stream)
            assert np.array_equal(d_kept.cpu().numpy().view(np.uint32), want[1])
            if sync:
                assert np.array_equal(d_counts.cpu().numpy().view(np.uint32), want[2])
    c.close()


def test_errors(tekken_bytes):
    from cfbpe import _native as N
    c = context(tekken_bytes)
    L = N.load()
    data, offs = pack([b"hello world", b"more text here"])
    bud = np.array([1, 2], np.uint32)
    cut = np.zeros(2, np.uint32)
    kept = np.zeros(2, np.uint32)
    args = [data.ctypes.data, offs.ctypes.data, None]
    assert L.cfbpe_truncate_batch(c._h, 2, *args, bud.ctypes.data, 2, cut.ctypes.data, kept.ctypes.data, None) == N.EINVAL
    assert L.cfbpe_truncate_batch(c._h, 2, *args, None, 0, cut.ctypes.data, kept.ctypes.data, None) == N.EINVAL
    assert L.cfbpe_truncate_batch(c._h, 2, *args, bud.ctypes.data, 1, None, kept.ctypes.data, None) == N.EINVAL
    assert L.cfbpe_truncate_batch(c._h, 2, *args, bud.ctypes.data, 1, cut.ctypes.data, None, None) == N.EINVAL
    assert L.cfbpe_truncate_batch_device(c._h, 0, None, 0, None, None, None, 0, None, None, None, None) == N.EINVAL
    assert L.cfbpe_truncate_batch_device(c._h, 1, None, 0, None, None, bud.ctypes.data, 7, cut.ctypes.data, kept.ctypes.data, None, None) == N.EINVAL
    with pytest.raises(N.NativeError) as ei:
        c.truncate_batch(*pack([b"fine", b"bad \xff here"]), 1)
    assert ei.value.code == N.EILSEQ
    with pytest.raises(N.NativeError) as ei:
        c.truncate_batch(data, offs, 1, HEAD, np.array([0, 3], np.uint8))
    assert ei.value.code == N.ENOENT
    with pytest.raises(N.NativeError) as ei:
        c.truncate_batch(data, offs, -1)
    assert ei.value.code == N.EINVAL
    ct, kp, cnt = c.truncate_batch(data, offs, 1)            # the context works after the failures
    assert kp.tolist() == [1, 1] and all(0 < int(x) for x in ct) and cnt.tolist() == c.count_batch(data, offs).tolist()
    c.close()


def test_two_threads_on_two_lanes(tekken_bytes):
    c = context(tekken_bytes, max_bytes=16 << 20, max_prompts=1 << 17, n_workspaces=2)
    batches = [pack([s.encode() for s in fuzzgen.fuzz_strings(seed, 20000, max_atoms=40)]) for seed in (5, 6)]
    budgets = [half_cut_budgets(c, d, o, None, 9) for d, o in batches]
    want_enc = [tuple(x.copy() for x in c.encode_batch(d, o)) for d, o in batches]
    want_cut = [tuple(x.copy() for x in c.truncate_batch(d, o, b, TAIL)) for (d, o), b in zip(batches, budgets)]
    errors = []

    def run(k):
        try:
            d, o = batches[k]
            for _ in range(6):
                if k == 0:
                    got = c.truncate_batch(d, o, budgets[0], TAIL)
                    assert all(np.array_equal(g, w) for g, w in zip(got, want_cut[0]))
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
    budgets = half_cut_budgets(one, data, offs, vid, 4)
    want = [tuple(x.copy() for x in one.truncate_batch(data, offs, budgets, m, vid)) for m in (HEAD, TAIL)]
    one.close()
    c = context(tekken_bytes, ((0, 100256), (3, 130072)), max_bytes=64 << 20, max_prompts=1 << 17,
                devices=list(range(min(torch.cuda.device_count(), 8))))
    for m in (HEAD, TAIL):
        got = c.truncate_batch(data, offs, budgets, m, vid)
        assert all(np.array_equal(g, w) for g, w in zip(got, want[m]))
    c.close()


def test_plugin_device_path_equals_trait_default():
    """GpuBpeTokenizerPlugin.truncate_batch (the device call) equals TokenizerPluginClient.truncate_batch (encode with starts, the
    cut on the host) on the same plugin and inputs; the service's texts are the prompts' kept bytes"""
    from cfbpe import plugin as P
    plug = P.GpuBpeTokenizerPlugin(device=0, vocab_names=("cl100k_base", "tekken"), max_batch_bytes=8 << 20, max_prompts=1 << 16,
                                   allow_stand_in=True)
    sec = P.SecurityContext.anonymous()
    texts = fuzzgen.fuzz_strings(1234, 800, max_atoms=40) + ["", "Hello, world! " * 40, "\U00020000\U0001f600" * 30]
    data, offs = P.pack_texts(texts)
    rng = np.random.default_rng(0)
    for model in ("cl100k_base", "tekken"):
        req = P.EncodeBatchRequest(P.VocabRef(model), data, offs)
        for keep in ("head", "tail"):
            for budgets in (5, rng.integers(0, 30, len(texts))):
                dev = plug.truncate_batch(sec, req, budgets, keep)
                host = P.TokenizerPluginClient.truncate_batch(plug, sec, req, budgets, keep)
                assert np.array_equal(dev.cut, host.cut) and np.array_equal(dev.kept, host.kept) and np.array_equal(dev.counts, host.counts)
    hub = P.ClientHub()
    hub.register_scoped(P.TokenizerPluginClient, plug.instance.id, plug)
    svc = P.LlmGatewayTokenizerService(hub, [plug.instance])
    for keep in ("head", "tail"):
        for t, (kept_text, kept, count) in zip(texts, svc.truncate(sec, "cl100k_base", texts, 9, keep)):
            assert (t.startswith(kept_text) if keep == "head" else t.endswith(kept_text))
            assert kept <= min(9, count)
    plug.close()
