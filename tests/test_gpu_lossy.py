"""Encode of bytes that are not valid UTF-8 on the H100 (cfbpe_encode_batch_lossy / _device): ids, offsets and counts against live
tiktoken 0.12.0 `encode_ordinary(b.decode("utf-8", "replace"))`, replacement counts against CPython's decoder, valid batches
bit-identical to cfbpe_encode_batch, the host, device and counts-only forms against each other, the errors the call can give,
caller buffers at odd alignments, several devices, and the plugin's errors="replace" against the trait's host default."""
import base64
import codecs
import random

import numpy as np
import pytest

import fuzzgen
from conftest import COMBOS, pack

pytestmark = pytest.mark.gpu

MULTILINGUAL = ["Grüße aus Köln", "日本語のテキストです。", "Привет, мир!", "مرحبا بالعالم", "emoji 😀👍🏽🎉 🇩🇪", "𠀀𠀁𪚥", "a�b", ""]
CASES = [b"\x80", b"\xbf\x80", b"\xc0\xaf", b"\xc1", b"\xf5\x80", b"\xff", b"\xe0\x80\x80", b"\xf0\x8f\xbf\xbf", b"\xed\xa0\x80",
         b"\xf4\x90\x80\x80", b"\xc3", b"\xe2\x82", b"\xf0\x9f\x98", b"\xf0\x9f\x98a", b"\xe2\x82\xe2\x82\xac"]
_calls = [0]


def _count(exc):
    _calls[0] += 1
    return "�", exc.end


codecs.register_error("cfbpe_gpu_test_count_replace", _count)


def cpython(p: bytes):
    """(the text b.decode("utf-8", "replace"), U+FFFD inserted)"""
    _calls[0] = 0
    t = p.decode("utf-8", "cfbpe_gpu_test_count_replace")
    return t, _calls[0]


def fuzz_prompt(rng: random.Random) -> bytes:
    parts = []
    for _ in range(rng.randrange(0, 14)):
        k = rng.randrange(6)
        if k == 0:
            parts.append(bytes(rng.randrange(256) for _ in range(rng.randrange(1, 9))))
        elif k == 1:
            parts.append(rng.choice(CASES))
        elif k == 2:
            t = rng.choice(MULTILINGUAL).encode()
            a = rng.randrange(len(t) + 1)
            parts.append(t[a:a + rng.randrange(1, 20)])
        else:
            parts.append(rng.choice(MULTILINGUAL + fuzzgen.fuzz_strings(rng.randrange(1 << 30), 1, max_atoms=12)).encode())
    return b"".join(parts)


def case_prompts():
    """every case after every ASCII lead-in of 0 .. 31 bytes, before ASCII, before a lead and at the prompt's end, and a lead
    that ends one prompt with the continuation bytes that open the next"""
    out = []
    for bad in CASES:
        for f in range(32):
            out += [b"x" * f + bad + b" y", b"x" * f + bad + "é".encode(), b"x" * f + bad]
    out += [b"abc\xe2", b"\x82\xacdef", b"\xf0\x9f", b"\x98\x80", b"", b"\xff" * 50]
    return out


def context(tekken_bytes, pats=((0, 100256),), max_bytes=8 << 20, max_prompts=1 << 16, **kw):
    from cfbpe import _native as N
    c = N.Context(0, max_bytes, max_prompts, **kw)
    for slot, (pat, n) in enumerate(pats):
        c.vocab_load(slot, tekken_bytes, N.FORMAT_TIKTOKEN, pat, n)
    return c


def repaired(prompts):
    """CPython's repair of every prompt: (bytes, offsets, replaced)"""
    texts = [cpython(p) for p in prompts]
    data, offs = pack([t.encode() for t, _ in texts])
    return data, offs, np.array([k for _, k in texts], dtype=np.uint32)


@pytest.mark.parametrize("pat,n_ranks", COMBOS)
def test_against_live_tiktoken(tekken_bytes, pat, n_ranks):
    tiktoken = pytest.importorskip("tiktoken")
    from oracle import patterns as PT
    ranks = {base64.b64decode(l.split()[0]): i for i, l in enumerate(tekken_bytes.splitlines()[:n_ranks])}
    enc = tiktoken.Encoding("live%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks, special_tokens={})
    rng = random.Random(31 + pat)
    prompts = case_prompts() + [fuzz_prompt(rng) for _ in range(1500)] + [t.encode() for t in fuzzgen.fuzz_strings(pat, 300, max_atoms=30)]
    c = context(tekken_bytes, ((pat, n_ranks),))
    data, offs = pack(prompts)
    ids, off, counts, rep = c.encode_batch_lossy(data, offs)
    for i, p in enumerate(prompts):
        t, k = cpython(p)
        a, b = int(off[i]), int(off[i + 1])
        assert ids[a:b].tolist() == enc.encode_ordinary(t), (p, t)
        assert int(counts[i]) == b - a and int(rep[i]) == k, p
    c.close()


def test_valid_batches_are_bit_identical_to_the_strict_call(tekken_bytes):
    from cfbpe import workload as W
    c = context(tekken_bytes, max_bytes=40 << 20)
    for data, offs in [pack([t.encode() for t in fuzzgen.fuzz_strings(7, 2000, max_atoms=40) + MULTILINGUAL]), W.make_config(3, 0.2)[:2]]:
        ids, off, counts = (x.copy() for x in c.encode_batch(data, offs))
        lids, loff, lcounts, rep = c.encode_batch_lossy(data, offs)
        assert np.array_equal(lids, ids) and np.array_equal(loff, off) and np.array_equal(lcounts, counts)
        assert not rep.any()
    c.close()


def test_a_large_batch_with_strays_equals_the_strict_call_on_the_repaired_bytes(tekken_bytes):
    """config-3 prompts, a stray byte in 1 % of them and in every one: the lossy call against cfbpe_encode_batch on CPython's repair"""
    from cfbpe import workload as W
    data, offs = W.make_config(3, 0.25)[:2]
    raw = data.tobytes()
    n = len(offs) - 1
    c = context(tekken_bytes, max_bytes=64 << 20, max_prompts=1 << 17)
    for every in (100, 1):
        prompts = [raw[int(offs[i]):int(offs[i + 1])] for i in range(n)]
        for i in range(0, n, every):
            cut = len(prompts[i]) // 2
            while 0 < cut < len(prompts[i]) and prompts[i][cut] & 0xC0 == 0x80:
                cut -= 1
            prompts[i] = prompts[i][:cut] + b"\xff" + prompts[i][cut:]
        d2, o2 = pack(prompts)
        rd, ro, want_rep = repaired(prompts)
        ids, off, counts = (x.copy() for x in c.encode_batch(rd, ro))
        lids, loff, lcounts, rep = c.encode_batch_lossy(d2, o2)
        assert np.array_equal(rep, want_rep)
        assert np.array_equal(loff, off) and np.array_equal(lcounts, counts) and np.array_equal(lids, ids)
    c.close()


def _device_call(c, data, offs, m=0, fill=b"\0", counts_only=False, sync=True, replaced=True):
    """the device form on a buffer with the batch at byte offset m, `fill` before it and exactly 32 bytes of fill after it"""
    import torch
    dev = torch.device("cuda:0")
    total, n = int(offs[-1]), len(offs) - 1
    host = np.frombuffer((fill * (m // len(fill) + 1))[:m] + data.tobytes()[:total] + (fill * (32 // len(fill) + 1))[:32], dtype=np.uint8)
    buf = torch.from_numpy(host.copy()).to(dev)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    cap = 3 * total + 1
    d_ids = torch.full((cap,), -1, dtype=torch.int32, device=dev)
    d_off = torch.full((n + 1,), -1, dtype=torch.int64, device=dev)
    d_cnt = torch.full((max(n, 1),), -1, dtype=torch.int32, device=dev)
    d_rep = torch.full((max(n, 1),), -1, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    nt = c.encode_batch_lossy_device(n, buf.data_ptr() + m, total, d_offs.data_ptr(), None, None if counts_only else d_ids.data_ptr(), cap,
                                     d_off.data_ptr(), d_cnt.data_ptr(), d_rep.data_ptr() if replaced else None, stream, sync)
    if not sync:
        torch.cuda.synchronize()
        c.device_status(stream)
    off = d_off.cpu().numpy().view(np.uint64)
    if sync:
        assert nt == int(off[-1])
    ids = None if counts_only else d_ids.cpu().numpy().view(np.uint32)[:int(off[-1])]
    return ids, off, d_cnt.cpu().numpy().view(np.uint32)[:n], d_rep.cpu().numpy().view(np.uint32)[:n]


def test_host_device_and_counts_only_agree(tekken_bytes):
    rng = random.Random(8)
    prompts = case_prompts() + [fuzz_prompt(rng) for _ in range(800)]
    data, offs = pack(prompts)
    _, _, want_rep = repaired(prompts)
    c = context(tekken_bytes)
    ids, off, counts, rep = (x.copy() for x in c.encode_batch_lossy(data, offs))
    assert np.array_equal(rep, want_rep)
    _, coff, ccounts, crep = c.encode_batch_lossy(data, offs, counts_only=True)
    assert np.array_equal(coff, off) and np.array_equal(ccounts, counts) and np.array_equal(crep, rep)
    for kw in ({}, {"sync": False}, {"counts_only": True}, {"replaced": False}):
        dids, doff, dcounts, drep = _device_call(c, data, offs, **kw)
        assert np.array_equal(doff, off) and np.array_equal(dcounts, counts), kw
        if "counts_only" not in kw:
            assert np.array_equal(dids, ids), kw
        if "replaced" not in kw:
            assert np.array_equal(drep, rep), kw
    c.close()


def test_device_form_at_odd_alignments_with_garbage_past_the_end(tekken_bytes):
    rng = random.Random(9)
    prompts = [fuzz_prompt(rng) for _ in range(300)] + [b"tail \xe2\x82"]
    data, offs = pack(prompts)
    c = context(tekken_bytes)
    ids, off, counts, rep = (x.copy() for x in c.encode_batch_lossy(data, offs))
    for m in range(16):
        for fill in (b"\0", b"\x80\xbf", b"\xf0\x9f\x98", b"\xff"):
            dids, doff, dcounts, drep = _device_call(c, data, offs, m=m, fill=fill)
            assert np.array_equal(dids, ids) and np.array_equal(doff, off), (m, fill)
            assert np.array_equal(dcounts, counts) and np.array_equal(drep, rep), (m, fill)
    c.close()


def test_enospc_writes_the_needed_count(tekken_bytes):
    from cfbpe import _native as N
    prompts = [b"ab\xffcd efg", b"\xc0" * 10, "日本語".encode()]
    data, offs = pack(prompts)
    c = context(tekken_bytes)
    ids, off, _, _ = c.encode_batch_lossy(data, offs)
    need = int(off[-1])
    out_ids = np.zeros(need - 1, dtype=np.uint32)
    out_off = np.zeros(len(prompts) + 1, dtype=np.uint64)
    with pytest.raises(N.NativeError) as e:
        c.encode_batch_lossy(data, offs, out_ids=out_ids, out_offsets=out_off)
    assert e.value.code == N.ENOSPC and int(out_off[-1]) == need
    c.close()


def test_a_repair_over_max_batch_bytes_is_einval_and_writes_nothing(tekken_bytes):
    import torch
    from cfbpe import _native as N
    c = context(tekken_bytes, max_bytes=4096, max_prompts=64)
    prompts = [b"ok", b"\xff" * 1500, b"\x80" * 500]          # 2002 bytes, repaired 6002
    data, offs = pack(prompts)
    outs = [np.full(3 * 2002, 7, np.uint32), np.full(4, 7, np.uint64), np.full(3, 7, np.uint32), np.full(3, 7, np.uint32)]
    with pytest.raises(N.NativeError) as e:
        c.encode_batch_lossy(data, offs, None, *outs)
    assert e.value.code == N.EINVAL and "6002" in str(e.value)
    assert all((a == 7).all() for a in outs)
    with pytest.raises(N.NativeError) as e:
        _device_call(c, data, offs)
    assert e.value.code == N.EINVAL
    torch.cuda.synchronize()
    ok = [b"ok", b"\xff" * 1300]                               # repaired 3902: fits
    d2, o2 = pack(ok)
    ids, off, counts, rep = c.encode_batch_lossy(d2, o2)
    assert rep.tolist() == [0, 1300]
    c.close()


def test_several_devices_match_one(tekken_bytes):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from cfbpe import _native as N
    rng = random.Random(10)
    prompts = case_prompts() + [fuzz_prompt(rng) for _ in range(3000)]
    data, offs = pack(prompts)
    one = context(tekken_bytes)
    want = [x.copy() for x in one.encode_batch_lossy(data, offs)]
    one.close()
    multi = N.Context(devices=list(range(min(torch.cuda.device_count(), 4))), max_batch_bytes=8 << 20, max_prompts=1 << 16)
    multi.vocab_load(0, tekken_bytes, N.FORMAT_TIKTOKEN, 0, 100256)
    got = multi.encode_batch_lossy(data, offs)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
    multi.close()


def test_plugin_replace_matches_the_trait_default():
    from cfbpe import plugin as P
    plug = P.GpuBpeTokenizerPlugin(device=0, vocab_names=("cl100k_base", "tekken"), max_batch_bytes=8 << 20, max_prompts=1 << 16,
                                   allow_stand_in=True)
    ctx = P.SecurityContext.anonymous()
    rng = random.Random(11)
    prompts = case_prompts() + [fuzz_prompt(rng) for _ in range(500)]
    data, offs = pack(prompts)
    for name in ("cl100k_base", "tekken"):
        req = P.EncodeBatchRequest(P.VocabRef(name), data, offs, errors="replace")
        got = plug.encode_batch(ctx, req)
        want = P.TokenizerPluginClient.encode_batch_lossy(plug, ctx, req)
        assert np.array_equal(got.ids, want.ids) and np.array_equal(got.offsets, want.offsets)
        assert np.array_equal(got.counts, want.counts) and np.array_equal(got.replaced, want.replaced)
        creq = P.CountTokensRequest(P.VocabRef(name), data, offs, errors="replace")
        assert np.array_equal(plug.count_tokens(ctx, creq), P.TokenizerPluginClient.count_tokens_lossy(plug, ctx, creq))
        with pytest.raises(P.InvalidInput):
            plug.encode_batch(ctx, P.EncodeBatchRequest(P.VocabRef(name), data, offs, with_starts=True, errors="replace"))
        with pytest.raises(P.InvalidInput):
            plug.encode_batch(ctx, P.EncodeBatchRequest(P.VocabRef(name), data, offs))      # strict: malformed UTF-8 is refused
    plug.close()
