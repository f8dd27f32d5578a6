"""Encode with special tokens on the H100 (cfbpe_encode_batch_special / _device, csrc/specials.cuh): against live tiktoken 0.12.0
`Encoding.encode(text, allowed_special=...)`, against the host cut of the plugin trait's default, and against the ordinary path."""
import base64
import random
import threading

import numpy as np
import pytest

import fuzzgen
from conftest import COMBOS, pack

pytestmark = pytest.mark.gpu

SLOT_NAMES = {0: "cl100k_base", 1: "o200k_base", 2: "llama3", 3: "tekken"}
SPECIALS = {"<|endoftext|>": 200000, "<|fim_prefix|>": 200001, "<|endofprompt|>": 200002, "<|eot_id|>": 200003,
            "<|start_header_id|>": 200004, "<|end_header_id|>": 200005, "<|é中|>": 200006, "\U0001f600!": 200007}
KEYS = list(SPECIALS)
ALLOW_ALL = np.ones(len(SPECIALS), np.uint8)


@pytest.fixture(scope="module")
def plug():
    from cfbpe import plugin as P
    p = P.GpuBpeTokenizerPlugin(device=0, vocab_names=("cl100k_base", "o200k_base", "llama3", "tekken"),
                                max_batch_bytes=160 << 20, max_prompts=1 << 20, allow_stand_in=True)
    for slot in range(4):
        p.ctx.vocab_set_specials(slot, SPECIALS)
        p._specials[slot] = dict(SPECIALS)
    yield p
    p.close()


@pytest.fixture(scope="module")
def ctx():
    from cfbpe import plugin as P
    return P.SecurityContext.anonymous()


def _encoding(tekken_bytes, pat, n_ranks, special):
    tiktoken = pytest.importorskip("tiktoken")
    from oracle import patterns as PT
    lines = tekken_bytes.splitlines()[:n_ranks]
    ranks = {base64.b64decode(l.split()[0]): i for i, l in enumerate(lines)}
    return tiktoken.Encoding("live%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks, special_tokens=special)


def texts_with_specials(seed, n):
    rng = random.Random(seed)
    out = []
    for i, t in enumerate(fuzzgen.fuzz_strings(seed, n, max_atoms=30)):
        k, k2 = rng.choice(KEYS), rng.choice(KEYS)
        cut = rng.randint(0, len(t))
        out.append([t, k + t, t + k, t[:cut] + k + t[cut:] + k2 + k2, k, t[:cut] + " \n  " + k + "   " + t[cut:], k + k2 + k][i % 7])
    return out


def split(ids, offs):
    return [ids[int(offs[i]):int(offs[i + 1])].tolist() for i in range(len(offs) - 1)]


def host_cut(plug, ctx, texts_or_packed, allowed, disallowed=frozenset()):
    """the plugin trait's default (host cut over the GPU plugin's encode_batch): the reference where tiktoken is not"""
    from cfbpe import plugin as P
    data, offs = texts_or_packed if isinstance(texts_or_packed, tuple) else P.pack_texts(texts_or_packed)
    return P.TokenizerPluginClient.encode_batch_special(plug, ctx, P.EncodeBatchRequest(P.VocabRef("cl100k_base"), data, offs),
                                                        SPECIALS, set(allowed), set(disallowed))


def inject(data, offs, per_prompt, seed):
    """the prompts of a packed batch with about `per_prompt` allowed specials each, at character boundaries"""
    rng = random.Random(seed)
    out = []
    for i in range(len(offs) - 1):
        t = bytes(data[int(offs[i]):int(offs[i + 1])]).decode("utf-8")
        for _ in range(rng.randint(0, 2 * per_prompt)):
            c = rng.randint(0, len(t))
            t = t[:c] + rng.choice(KEYS) + t[c:]
        out.append(t)
    return out


@pytest.mark.parametrize("pat,n_ranks", COMBOS)
def test_against_live_tiktoken(plug, tekken_bytes, pat, n_ranks):
    enc = _encoding(tekken_bytes, pat, n_ranks, SPECIALS)
    texts = texts_with_specials(700 + pat, 3000) + ["", " \n\n" + KEYS[1] + "\n\n "]
    data, offs = pack([t.encode() for t in texts])
    vid = np.full(len(texts), pat, np.uint8)
    ids, o, c = plug.ctx.encode_batch_special(data, offs, vid, [None] * pat + [ALLOW_ALL])
    got = split(ids, o)
    for t, g, k in zip(texts, got, c):
        want = enc.encode(t, allowed_special="all")
        assert g == want, repr(t)
        assert k == len(want)
    allowed = {KEYS[0], KEYS[3], KEYS[6]}
    m = np.array([1 if k in allowed else 0 for k in KEYS], np.uint8)
    ids, o, _ = plug.ctx.encode_batch_special(data, offs, vid, [None] * pat + [m])
    for t, g in zip(texts, split(ids, o)):
        assert g == enc.encode(t, allowed_special=allowed, disallowed_special=()), repr(t)


def test_multi_vocabulary_batch_with_own_sets_and_modes(tekken_bytes):
    from cfbpe import _native as N
    from cfbpe import vocabs as V
    c = N.Context(0, 8 << 20, 1 << 12)
    sp = [{"<|endoftext|>": 200000, "<|eot_id|>": 200003}, {"[INST]": 300001, "[/INST]": 300002}]
    for slot, name in enumerate(("cl100k_base", "tekken")):
        rv = V.resolve(name, allow_stand_in=True)
        c.vocab_load(slot, rv.file_bytes, rv.spec.fmt, rv.pattern_id, rv.max_ranks)
        c.vocab_set_specials(slot, sp[slot])
    texts = ["a<|endoftext|>b[INST]", "[INST] hi [/INST]<|eot_id|>", "<|eot_id|>x", "plain [/INST]"] * 50
    vid = np.array([0, 1, 0, 1] * 50, np.uint8)
    data, offs = pack([t.encode() for t in texts])
    ids, o, _ = c.encode_batch_special(data, offs, vid, [np.array([1, 1], np.uint8), np.array([1, 0], np.uint8)])
    e0 = _encoding(tekken_bytes, 0, 100256, sp[0])
    e3 = _encoding(tekken_bytes, 3, 130072, sp[1])
    for t, v, g in zip(texts, vid, split(ids, o)):
        want = e0.encode(t, allowed_special="all") if v == 0 else e3.encode(t, allowed_special={"[INST]"}, disallowed_special=())
        assert g == want, t
    c.close()


@pytest.mark.parametrize("size", ["small", "pipelined", "bench"])
def test_host_calls_against_the_host_cut(plug, ctx, size):
    """below and above the 4 MiB one-shot limit of cfbpe_encode_batch, and the bench batch (config 3) with specials injected"""
    from cfbpe import workload as W
    if size == "small":
        texts = texts_with_specials(11, 2000)
    else:
        data, offs, _, _ = W.make_config(3, 0.06 if size == "pipelined" else 1.0)
        texts = inject(data, offs, 5, 3)
    from cfbpe import plugin as P
    data, offs = P.pack_texts(texts)
    assert (size == "small") == (int(offs[-1]) < (4 << 20))
    want = host_cut(plug, ctx, (data, offs), set(SPECIALS))
    ids, o, c = plug.ctx.encode_batch_special(data, offs, None, [ALLOW_ALL])
    assert np.array_equal(o, want.offsets)
    assert np.array_equal(c, want.counts)
    assert np.array_equal(ids, want.ids)


def test_device_entry_point_equals_host(plug):
    import torch
    texts = texts_with_specials(21, 4000)
    data, offs = pack([t.encode() for t in texts])
    ids, o, c = plug.ctx.encode_batch_special(data, offs, None, [ALLOW_ALL])
    total, n = int(offs[-1]), len(offs) - 1
    d_bytes = torch.zeros(total + 64, dtype=torch.uint8, device="cuda")
    d_bytes[:total] = torch.from_numpy(data)
    d_offs = torch.from_numpy(offs.view(np.int64)).cuda()
    d_ids = torch.zeros(total + 1, dtype=torch.int32, device="cuda")
    d_oo = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    d_cc = torch.zeros(n, dtype=torch.int32, device="cuda")
    nt = plug.ctx.encode_batch_special_device(n, d_bytes.data_ptr(), total, d_offs.data_ptr(), None, d_ids.data_ptr(), total + 1,
                                              d_oo.data_ptr(), d_cc.data_ptr(), modes=[ALLOW_ALL], stream=torch.cuda.current_stream().cuda_stream)
    assert nt == len(ids)
    assert np.array_equal(d_oo.cpu().numpy().view(np.uint64), o)
    assert np.array_equal(d_cc.cpu().numpy().view(np.uint32), c)
    assert np.array_equal(d_ids[:nt].cpu().numpy().view(np.uint32), ids)
    # asynchronous form: the offsets carry the total, device_status reports no error
    d_oo.zero_()
    plug.ctx.encode_batch_special_device(n, d_bytes.data_ptr(), total, d_offs.data_ptr(), None, d_ids.data_ptr(), total + 1,
                                         d_oo.data_ptr(), None, modes=[ALLOW_ALL], stream=torch.cuda.current_stream().cuda_stream, sync=False)
    plug.ctx.device_status(torch.cuda.current_stream().cuda_stream)
    assert np.array_equal(d_oo.cpu().numpy().view(np.uint64), o)


def test_counts_only_enospc_ebadmsg_and_einval(plug):
    from cfbpe import _native as N
    texts = texts_with_specials(31, 500)
    data, offs = pack([t.encode() for t in texts])
    ids, o, c = plug.ctx.encode_batch_special(data, offs, None, [ALLOW_ALL])
    _, o2, c2 = plug.ctx.encode_batch_special(data, offs, None, [ALLOW_ALL], counts_only=True)
    assert np.array_equal(c2, c) and np.array_equal(o2, o)
    with pytest.raises(N.NativeError) as ei:
        plug.ctx.encode_batch_special(data, offs, None, [ALLOW_ALL], out_ids=np.empty(len(ids) - 1, np.uint32))
    assert ei.value.code == N.ENOSPC and str(len(ids)) in str(ei.value)
    bad = [b"clean", b"also clean", b"x <|fim_prefix|> and <|endoftext|>", b"<|endoftext|>"]
    d, of = pack(bad)
    with pytest.raises(N.NativeError) as ei:
        plug.ctx.encode_batch_special(d, of)                 # tiktoken's default: every special disallowed
    assert ei.value.code == N.EBADMSG and ei.value.bad == (2, KEYS.index("<|fim_prefix|>")) and "<|fim_prefix|>" in str(ei.value)
    with pytest.raises(N.NativeError) as ei:                 # a disallowed special wins over malformed UTF-8
        plug.ctx.encode_batch_special(*pack([b"\xff", b"a<|eot_id|>"]))
    assert ei.value.code == N.EBADMSG and ei.value.bad == (1, KEYS.index("<|eot_id|>"))
    small = N.Context(0, 1 << 20, 8)
    from cfbpe import vocabs as V
    rv = V.resolve("cl100k_base", allow_stand_in=True)
    small.vocab_load(0, rv.file_bytes, rv.spec.fmt, rv.pattern_id, rv.max_ranks)
    small.vocab_set_specials(0, SPECIALS)
    small.encode_batch_special(*pack([b"<|eot_id|>a", b"b<|eot_id|>"]), None, [ALLOW_ALL])     # 2 + 2 x 2 = 6 stretches
    with pytest.raises(N.NativeError) as ei:
        small.encode_batch_special(*pack([b"<|eot_id|>a<|eot_id|>", b"b<|eot_id|><|eot_id|>"]), None, [ALLOW_ALL])
    assert ei.value.code == N.EINVAL and "max_prompts" in str(ei.value)
    small.close()


def test_fast_path_equals_encode_batch(plug):
    from cfbpe import workload as W
    data, offs, _, _ = W.make_config(3, 0.25)
    ids, o, c = plug.ctx.encode_batch(data, offs)
    ids2, o2, c2 = plug.ctx.encode_batch_special(data, offs)       # every special disallowed, none present
    assert np.array_equal(o2, o) and np.array_equal(c2, c) and np.array_equal(ids2, ids)


def test_decode_round_trip_of_special_ids(plug):
    texts = texts_with_specials(41, 1500)
    data, offs = pack([t.encode() for t in texts])
    ids, o, _ = plug.ctx.encode_batch_special(data, offs, None, [ALLOW_ALL])
    assert any(int(i) >= 200000 for i in ids)
    out, bo = plug.ctx.decode_batch(ids, o)
    assert bytes(out) == bytes(data) and np.array_equal(bo, offs)


def test_set_specials_racing_encode_on_two_lanes(tekken_bytes):
    from cfbpe import _native as N
    from cfbpe import vocabs as V
    c = N.Context(0, 8 << 20, 1 << 14, n_workspaces=2)
    rv = V.resolve("cl100k_base", allow_stand_in=True)
    c.vocab_load(0, rv.file_bytes, rv.spec.fmt, rv.pattern_id, rv.max_ranks)
    c.vocab_set_specials(0, SPECIALS)
    enc = _encoding(tekken_bytes, 0, 100256, SPECIALS)
    texts = texts_with_specials(51, 400)
    data, offs = pack([t.encode() for t in texts])
    want = [enc.encode(t, allowed_special="all") for t in texts]
    errors = []
    stop = threading.Event()

    def encoder():
        try:
            while not stop.is_set():
                ids, o, _ = c.encode_batch_special(data, offs, None, [ALLOW_ALL])
                assert split(ids, o) == want
        except Exception as e:   # noqa: BLE001
            errors.append(e)

    th = [threading.Thread(target=encoder) for _ in range(3)]
    for t in th:
        t.start()
    for _ in range(30):
        c.vocab_set_specials(0, SPECIALS)          # the same set again: calls see either table, both right
    stop.set()
    for t in th:
        t.join()
    assert not errors, errors[0]
    c.close()


def test_two_devices_shard_form(tekken_bytes):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from cfbpe import _native as N
    from cfbpe import vocabs as V
    c = N.Context(devices=[0, 1], max_batch_bytes=8 << 20, max_prompts=1 << 14)
    rv = V.resolve("cl100k_base", allow_stand_in=True)
    c.vocab_load(0, rv.file_bytes, rv.spec.fmt, rv.pattern_id, rv.max_ranks)
    c.vocab_set_specials(0, SPECIALS)
    enc = _encoding(tekken_bytes, 0, 100256, SPECIALS)
    texts = texts_with_specials(61, 2000)
    data, offs = pack([t.encode() for t in texts])
    ids, o, _ = c.encode_batch_special(data, offs, None, [ALLOW_ALL])
    assert split(ids, o) == [enc.encode(t, allowed_special="all") for t in texts]
    with pytest.raises(N.NativeError) as ei:
        c.encode_batch_special(*pack([b"a"] * 1500 + [b"<|eot_id|>"]))
    assert ei.value.code == N.EBADMSG and ei.value.bad == (1500, KEYS.index("<|eot_id|>"))
    c.close()


def test_plugin_override_equals_the_host_cut_default(plug, ctx):
    from cfbpe import plugin as P
    texts = texts_with_specials(71, 1500)
    for allowed in (set(SPECIALS), {KEYS[0], KEYS[4]}):
        disallowed = set()
        data, offs = P.pack_texts(texts)
        req = P.EncodeBatchRequest(P.VocabRef("cl100k_base"), data, offs)
        got = plug.encode_batch_special(ctx, req, SPECIALS, allowed, disallowed)
        want = P.TokenizerPluginClient.encode_batch_special(plug, ctx, req, SPECIALS, allowed, disallowed)
        assert np.array_equal(got.offsets, want.offsets) and np.array_equal(got.ids, want.ids)
    with pytest.raises(P.InvalidInput) as ei:
        plug.encode_batch_special(ctx, P.EncodeBatchRequest(P.VocabRef("cl100k_base"), *P.pack_texts(["x <|eot_id|>"])), SPECIALS, set(), set(SPECIALS))
    assert "<|eot_id|>" in str(ei.value)
