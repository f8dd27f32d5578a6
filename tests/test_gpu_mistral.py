"""Mistral's Tekken ids on the H100: the slot loaded with id base 1000 and mistral_common's control tokens returns exactly
Tekkenizer.encode(s, bos=False, eos=False) from every encode entry point and its device form, decode takes those ids back, and
control ids decode to their text.  Reference: live mistral_common when it imports; else its golden file (tests/mistral_ref.py) and,
for the large batches, the C oracle's ranks + 1000 (the golden file shows the two agree)."""
import os

import numpy as np
import pytest

import mistral_ref as MR
from conftest import pack

pytestmark = pytest.mark.gpu

BASE, N_TEK = MR.ID_BASE, MR.N_RANKS


@pytest.fixture(scope="module")
def controls():
    from cfbpe import vocabs as V
    return V.control_tokens(V.SPECS["mistral_tekken"])


@pytest.fixture(scope="module")
def ctx(tekken_bytes, controls):
    """slot 0: the cl100k stand-in (ids = ranks), slot 1: Mistral's Tekken (base 1000 + control tokens)"""
    from cfbpe import _native as N
    c = N.Context(0, max_batch_bytes=160 << 20, max_prompts=1 << 19)
    c.vocab_load(0, tekken_bytes, N.FORMAT_TIKTOKEN, N.PATTERN_IDS["cl100k"], 100256)
    c.vocab_load(1, tekken_bytes, N.FORMAT_TIKTOKEN, N.PATTERN_IDS["tekken"], N_TEK)
    c.vocab_set_id_base(1, BASE)
    c.vocab_set_specials(1, controls)
    yield c
    c.close()


@pytest.fixture(scope="module")
def tek_oracle(tekken_bytes):
    from oracle import oracle
    return oracle.OracleVocab(tekken_bytes, N_TEK)


def _reference(texts, tek_oracle):
    """Tekkenizer ids of `texts`, packed: (ids, offsets)"""
    mt = MR.live_tokenizer()
    if mt is not None:
        per = [mt.instruct_tokenizer.tokenizer.encode(t, bos=False, eos=False) for t in texts]
    else:
        per = [(tek_oracle.encode(3, t.encode()).astype(np.int64) + BASE).tolist() for t in texts]
    offs = np.concatenate([[0], np.cumsum([len(p) for p in per])]).astype(np.uint64)
    return np.asarray([i for p in per for i in p], dtype=np.uint32), offs


def _fuzz():
    """(bytes, offsets, Tekkenizer ids, id offsets) of the fuzz strings: live, or the golden file"""
    texts = MR.fuzz_texts()
    data, offs = pack([t.encode() for t in texts])
    mt = MR.live_tokenizer()
    if mt is not None:
        per = [mt.instruct_tokenizer.tokenizer.encode(t, bos=False, eos=False) for t in texts]
        return data, offs, np.asarray([i for p in per for i in p], dtype=np.uint32), np.concatenate([[0], np.cumsum([len(p) for p in per])]).astype(np.uint64)
    g = MR.golden()
    assert np.array_equal(g["text_bytes"], data)
    return data, offs, g["ids"], g["id_offsets"]


def _every_entry_point(ctx, data, offs, want, want_off):
    """host and device forms of every encode call that returns ids, on slot 1, against (want, want_off)"""
    import torch
    from cfbpe import _native as N
    n = len(offs) - 1
    vid = np.ones(max(n, 1), dtype=np.uint8)
    ids, o, _ = ctx.encode_batch(data, offs, vid)
    assert np.array_equal(o, want_off) and np.array_equal(ids, want)
    ids, starts, o, _ = ctx.encode_batch_starts(data, offs, vid)
    assert np.array_equal(o, want_off) and np.array_equal(ids, want)
    ids, starts, o, _, _ = ctx.encode_batch_char_starts(data, offs, N.UNIT_UTF16, vid)
    assert np.array_equal(o, want_off) and np.array_equal(ids, want)
    ids, o, _, rep = ctx.encode_batch_lossy(data, offs, vid)
    assert np.array_equal(o, want_off) and np.array_equal(ids, want) and not rep.any()
    modes = [None, np.zeros(BASE, dtype=np.uint8)]          # every control token ORDINARY: its spelling is text
    ids, o, _ = ctx.encode_batch_special(data, offs, vid, modes)
    assert np.array_equal(o, want_off) and np.array_equal(ids, want)
    dev = torch.device("cuda:0")
    total = int(offs[-1])
    d_bytes = torch.zeros(total + 64, dtype=torch.uint8, device=dev)
    d_bytes[:total] = torch.from_numpy(data[:total].copy()).to(dev)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    d_vid = torch.from_numpy(vid.copy()).to(dev)
    cap = total + 1
    stream = torch.cuda.current_stream().cuda_stream
    for form in ("plain", "starts", "char_starts", "lossy", "special"):
        d_ids = torch.full((cap,), -1, dtype=torch.int32, device=dev)
        d_st = torch.full((cap,), -1, dtype=torch.int32, device=dev)
        d_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        d_cnt = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        args = (n, d_bytes.data_ptr(), total, d_offs.data_ptr(), d_vid.data_ptr())
        if form == "plain":
            nt = ctx.encode_batch_device(*args, d_ids.data_ptr(), cap, d_off.data_ptr(), d_cnt.data_ptr(), stream)
        elif form == "starts":
            nt = ctx.encode_batch_starts_device(*args, d_ids.data_ptr(), d_st.data_ptr(), cap, d_off.data_ptr(), d_cnt.data_ptr(), stream)
        elif form == "char_starts":
            nt = ctx.encode_batch_char_starts_device(*args, N.UNIT_CODEPOINT, d_ids.data_ptr(), d_st.data_ptr(), cap, d_off.data_ptr(),
                                                     d_cnt.data_ptr(), None, stream)
        elif form == "lossy":
            nt = ctx.encode_batch_lossy_device(*args, d_ids.data_ptr(), cap, d_off.data_ptr(), d_cnt.data_ptr(), None, stream)
        else:
            nt = ctx.encode_batch_special_device(*args, d_ids.data_ptr(), cap, d_off.data_ptr(), d_cnt.data_ptr(), modes, stream)
        torch.cuda.synchronize()
        assert nt == len(want), form
        assert np.array_equal(d_off.cpu().numpy().astype(np.uint64), want_off), form
        assert np.array_equal(d_ids[:nt].cpu().numpy().view(np.uint32), want), form


def test_fuzz_strings_every_entry_point(ctx):
    data, offs, want, want_off = _fuzz()
    _every_entry_point(ctx, data, offs, want, want_off)
    dec, doffs = ctx.decode_batch(want, want_off, np.ones(len(offs) - 1, dtype=np.uint8))
    assert np.array_equal(doffs, offs) and np.array_equal(dec, data)


def test_every_token_of_the_vocabulary(ctx, tekken_bytes, tek_oracle):
    from cfbpe import workload as W
    data, offs = W.make_vocab_text(tekken_bytes, N_TEK, 7, "tokens", variants=("alone", "after_space"))
    texts = [bytes(data[int(offs[i]):int(offs[i + 1])]).decode("utf-8") for i in range(len(offs) - 1)]
    want, want_off = _reference(texts, tek_oracle)
    _every_entry_point(ctx, data, offs, want, want_off)


def test_config3_full_size(ctx, tek_oracle):
    """BASELINE.json config 3 at full size on the Mistral slot: every id, through the pipelined host path and the device path"""
    from cfbpe import workload as W
    data, offs, _, _ = W.make_config(3, 1.0)
    n = len(offs) - 1
    mt = MR.live_tokenizer()
    if mt is not None:
        from concurrent.futures import ThreadPoolExecutor
        tek = mt.instruct_tokenizer.tokenizer
        texts = [bytes(data[int(offs[i]):int(offs[i + 1])]).decode("utf-8") for i in range(n)]
        with ThreadPoolExecutor(os.cpu_count()) as ex:
            per = list(ex.map(lambda t: tek.encode(t, bos=False, eos=False), texts, chunksize=512))
        want_off = np.concatenate([[0], np.cumsum([len(p) for p in per])]).astype(np.uint64)
        want = np.fromiter((i for p in per for i in p), dtype=np.uint32, count=int(want_off[-1]))
    else:
        from oracle import oracle
        want, want_off, _ = oracle.encode_batch([tek_oracle], [3], data, offs, nthreads=os.cpu_count())
        want = want + np.uint32(BASE)
    vid = np.ones(n, dtype=np.uint8)
    ids, o, _ = ctx.encode_batch(data, offs, vid)
    assert np.array_equal(o, want_off) and np.array_equal(ids, want)
    import torch
    dev = torch.device("cuda:0")
    d_bytes = torch.zeros(len(data) + 64, dtype=torch.uint8, device=dev)
    d_bytes[:len(data)] = torch.from_numpy(data).to(dev)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    d_ids = torch.empty(len(data) + 1, dtype=torch.int32, device=dev)
    d_off = torch.empty(n + 1, dtype=torch.int64, device=dev)
    d_vid = torch.from_numpy(vid).to(dev)
    nt = ctx.encode_batch_device(n, d_bytes.data_ptr(), len(data), d_offs.data_ptr(), d_vid.data_ptr(), d_ids.data_ptr(), len(data) + 1,
                                 d_off.data_ptr(), None, torch.cuda.current_stream().cuda_stream)
    assert nt == len(want)
    assert np.array_equal(d_ids[:nt].cpu().numpy().view(np.uint32), want)
    dec, doffs = ctx.decode_batch(want, want_off, vid)
    assert np.array_equal(doffs, offs) and np.array_equal(dec, data)


def test_control_tokens_allowed_and_decoded(ctx, controls, tek_oracle):
    """allowed control tokens become their registered ids (below the base); the text between them is base + rank"""
    texts = ["<s>[INST]Hi there[/INST]Hello!</s>[INST]Be brief.\n\nCount me[/INST]", "[TOOL_CONTENT]x<SPECIAL_999>", "plain", ""]
    data, offs = pack([t.encode() for t in texts])
    vid = np.ones(len(texts), dtype=np.uint8)
    ids, o, _ = ctx.encode_batch_special(data, offs, vid, [None, np.ones(BASE, dtype=np.uint8)])
    mt = MR.live_tokenizer()
    if mt is not None:
        from mistral_common.tokens.tokenizers.base import SpecialTokenPolicy
        tek = mt.instruct_tokenizer.tokenizer
        for i, t in enumerate(texts):
            got = ids[int(o[i]):int(o[i + 1])].tolist()
            assert tek.decode(got, special_token_policy=SpecialTokenPolicy.KEEP) == t
            assert all(x >= BASE or x in controls.values() for x in got)
    first = ids[int(o[0]):int(o[1])].tolist()
    assert first == [1, 3, 37133, 2156, 4, 22177, 1033, 2, 3, 5934, 13426, 1338, 6669, 1639, 4]   # encode_chat_completion's ids of it
    dec, doffs = ctx.decode_batch(ids, o, vid)
    assert np.array_equal(doffs, offs) and np.array_equal(dec, data)
    dec, _ = ctx.decode_batch(np.arange(BASE, dtype=np.uint32), np.array([0, BASE], dtype=np.uint64), vid[:1])
    assert bytes(dec).decode() == "".join(controls)


def test_set_id_base_and_specials_refusals(ctx, tekken_bytes, controls):
    from cfbpe import _native as N
    c = N.Context(0, max_batch_bytes=1 << 20, max_prompts=1 << 10)
    try:
        with pytest.raises(N.NativeError) as e:
            c.vocab_set_id_base(0, 1000)                                  # not loaded
        assert e.value.code == N.ENOENT
        c.vocab_load(0, tekken_bytes, N.FORMAT_TIKTOKEN, N.PATTERN_IDS["tekken"], N_TEK)
        assert c.vocab_id_base(0) == 0
        with pytest.raises(N.NativeError) as e:
            c.vocab_set_id_base(0, 0xFFFFFFFF - N_TEK + 1)                # base + n_ranks past 0xFFFFFFFF
        assert e.value.code == N.EINVAL
        c.vocab_set_id_base(0, 0xFFFFFFFF - N_TEK)
        c.vocab_set_specials(0, {"<x>": 5})                                # base 0 rules are unchanged: an id below n_ranks is allowed
        c.vocab_set_id_base(0, 0)
        c.vocab_set_specials(0, {"<x>": 5})
        with pytest.raises(N.NativeError) as e:
            c.vocab_set_id_base(0, 1)                                      # would make special 5 an ordinary id
        assert e.value.code == N.EINVAL and c.vocab_id_base(0) == 0
        c.vocab_set_specials(0, controls)
        c.vocab_set_id_base(0, BASE)
        with pytest.raises(N.NativeError) as e:
            c.vocab_set_specials(0, {"<x>": BASE + N_TEK - 1})
        assert e.value.code == N.EINVAL
        c.vocab_set_specials(0, {"<x>": BASE + N_TEK, "<y>": BASE - 1})
        c.vocab_load(0, tekken_bytes, N.FORMAT_TIKTOKEN, N.PATTERN_IDS["tekken"], N_TEK)   # a load resets the base ...
        assert c.vocab_id_base(0) == 0
        c.vocab_set_id_base(0, BASE)
        c.vocab_import(0, c.vocab_export(0))                                               # ... and so does an import
        assert c.vocab_id_base(0) == 0
    finally:
        c.close()


def test_plugin_speaks_mistral_ids(controls):
    """the registry's Mistral models get the Mistral slot: encode, special encode and decode in Mistral's ids; the raw-rank slot
    beside it is unchanged"""
    from cfbpe import plugin as P
    plug = P.GpuBpeTokenizerPlugin(device=0, vocab_names=("tekken", "mistral_tekken"), max_batch_bytes=8 << 20, max_prompts=1 << 12)
    try:
        c = P.SecurityContext.anonymous()
        data, offs = pack([b"Hi there", b"Count me"])
        raw = plug.encode_batch(c, P.EncodeBatchRequest(P.VocabRef("tekken"), data, offs))
        for model in ("mistral::mistral-nemo", "mistral::pixtral-12b"):
            r = plug.encode_batch(c, P.EncodeBatchRequest(P.VocabRef(model), data, offs))
            assert np.array_equal(r.ids, raw.ids + np.uint32(BASE)) and np.array_equal(r.offsets, raw.offsets)
            d = plug.decode_batch(c, P.DecodeBatchRequest(P.VocabRef(model), np.array([1, 3] + r.ids.tolist() + [4], dtype=np.uint32),
                                                          np.array([0, len(r.ids) + 3], dtype=np.uint64)))
            assert bytes(d.bytes) == b"<s>[INST]Hi thereCount me[/INST]"
            s = plug.encode_batch_special(c, P.EncodeBatchRequest(P.VocabRef(model), *pack([b"<s>[INST]Hi there[/INST]"])), controls,
                                          {"<s>", "[INST]", "[/INST]"}, set())
            assert s.ids.tolist() == [1, 3, 37133, 2156, 4]
    finally:
        plug.close()


def test_two_devices():
    """a two-device context: sharded and round-robin host calls rebase per shard / sub-batch"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one device")
    from cfbpe import _native as N
    from cfbpe import workload as W
    from oracle import oracle
    tb = open(os.path.join(MR.ROOT, "vocabs", "tekken_240911.tiktoken"), "rb").read()
    c = N.Context(devices=[0, 1], max_batch_bytes=96 << 20, max_prompts=1 << 17)
    try:
        c.vocab_load(0, tb, N.FORMAT_TIKTOKEN, N.PATTERN_IDS["cl100k"], 100256)
        c.vocab_load(1, tb, N.FORMAT_TIKTOKEN, N.PATTERN_IDS["tekken"], N_TEK)
        c.vocab_set_id_base(1, BASE)
        data, offs, _, _ = W.make_config(3, 0.25)
        n = len(offs) - 1
        vid = (np.arange(n) % 2).astype(np.uint8)
        ovs = [oracle.OracleVocab(tb, 100256), oracle.OracleVocab(tb, N_TEK)]
        ids, o, _ = c.encode_batch(data, offs, vid)
        for i in np.random.default_rng(1).integers(0, n, size=400):
            want = ovs[vid[i]].encode([0, 3][vid[i]], bytes(data[int(offs[i]):int(offs[i + 1])])).astype(np.int64) + (BASE if vid[i] else 0)
            assert np.array_equal(ids[int(o[i]):int(o[i + 1])], want)
    finally:
        c.close()
