"""Mistral's Tekken models without a GPU: the registry entry and its control tokens, the "mistral" chat template against
mistral_common's encode_chat_completion (live when it imports, else its golden counts), and the importer on a tokenizer.json whose
mergeable ids start at a base."""
import base64
import json

import numpy as np
import pytest

import mistral_ref as MR
from cfbpe import importers as I
from cfbpe import plugin as P
from cfbpe import vocabs as V


def test_registry_maps_mistral_models_to_mistral_ids():
    spec = V.SPECS["mistral_tekken"]
    assert (spec.pattern, spec.n_ranks, spec.id_base) == ("tekken", MR.N_RANKS, MR.ID_BASE)
    assert V.for_model("mistral::mistral-nemo") == V.for_model("mistral::pixtral-12b") == "mistral_tekken"
    assert V.SPECS["tekken"].id_base == 0 and not V.SPECS["tekken"].controls
    ctl = V.control_tokens(spec)
    assert len(ctl) == MR.ID_BASE and list(ctl.values()) == list(range(MR.ID_BASE))
    assert [t for t, i in ctl.items() if i in (0, 1, 2, 3, 4, 19, 20, 999)] == \
        ["<unk>", "<s>", "</s>", "[INST]", "[/INST]", "[TOOL_CONTENT]", "<SPECIAL_20>", "<SPECIAL_999>"]
    mt = MR.live_tokenizer()
    if mt is not None:
        tek = mt.instruct_tokenizer.tokenizer
        assert list(ctl) == [tek.id_to_piece(i) for i in range(tek.num_special_tokens)]


def test_nemo_and_pixtral_files_share_the_ranks():
    """Mistral NeMo's tekken_240718 and Pixtral's tekken_240911 hold the same first 130072 ranks as the committed rank file"""
    pytest.importorskip("mistral_common")
    import os
    import mistral_common
    ours = [base64.b64decode(l.split()[0]) for l in open(os.path.join(MR.ROOT, "vocabs", "tekken_240911.tiktoken"), "rb").read().splitlines()[:MR.N_RANKS]]
    for name in ("tekken_240718.json", "tekken_240911.json"):
        with open(os.path.join(os.path.dirname(mistral_common.__file__), "data", name)) as f:
            j = json.load(f)
        assert j["config"]["default_num_special_tokens"] == MR.ID_BASE and j["config"]["default_vocab_size"] == MR.ID_BASE + MR.N_RANKS
        assert [base64.b64decode(v["token_bytes"]) for v in j["vocab"][:MR.N_RANKS]] == ours, name


@pytest.fixture(scope="module")
def service(tekken_bytes):
    from oracle import oracle
    ov = oracle.OracleVocab(tekken_bytes, MR.N_RANKS)

    class OraclePlugin(P.TokenizerPluginClient):
        def count_tokens(self, ctx, req):
            return oracle.encode_batch([ov], [3], req.bytes, req.offsets, nthreads=2)[2]

    hub = P.ClientHub()
    inst = P.PluginInstance("gts.x.core.modkit.plugin.v1~x.llmgw.tokenizer.plugin.v1~test.oracle.v1", "cyberfabric", 10)
    hub.register_scoped(P.TokenizerPluginClient, inst.id, OraclePlugin())
    return P.LlmGatewayTokenizerService(hub, [inst], vendor="cyberfabric")


def test_mistral_template_counts_as_mistral_common(service):
    convs = MR.conversations()
    mt = MR.live_tokenizer()
    if mt is not None:
        want = [MR.mistral_count(mt, c) for c in convs]
    else:
        g = MR.golden()
        assert bytes(g["conversations"]).decode("utf-8") == MR.conversations_json(convs)
        want = g["conversation_counts"].tolist()
    ctx = P.SecurityContext.anonymous()
    tpl = P.CHAT_TEMPLATES["mistral-v3"]
    assert sum(w >= 0 for w in want) >= 250
    for conv, w in zip(convs, want):
        if w < 0:                           # mistral_common refuses the order of these messages
            with pytest.raises(P.InvalidInput):
                service.count_chat_tokens(ctx, "mistral::mistral-nemo", conv, tpl)
        else:
            assert service.count_chat_tokens(ctx, "mistral::mistral-nemo", conv, tpl).input_tokens == w, conv
    # what encode_chat_completion makes of this conversation: <s>[INST]Hi there[/INST]Hello!</s>[INST]Be brief.\n\nCount me[/INST]
    msg = lambda role, t: {"role": role, "content": [{"type": "text", "text": t}]}
    conv = [msg("system", "Be brief."), msg("user", "Hi there"), msg("assistant", "Hello!"), msg("user", "Count me")]
    texts, n_ctl = P.mistral_instruct_texts(conv)
    assert texts == ["Hi there", "Hello!", "Be brief.\n\nCount me"] and n_ctl == 6
    assert service.count_chat_tokens(ctx, "mistral::mistral-nemo", conv, tpl).input_tokens == 15


def test_importer_takes_ids_from_a_base(tekken_bytes):
    """a byte-level tokenizer.json with 1000 control tokens first and the mergeable tokens from id 1000 (the layout of Hugging Face's
    Mistral NeMo files), built from the committed ranks: the importer returns the rank file and the base, and Hugging Face's
    tokenizers library, reading the same file, gives ids = 1000 + the oracle's ranks"""
    tokenizers = pytest.importorskip("tokenizers")
    from oracle import oracle
    b2u = I.bytes_to_unicode()
    enc = lambda t: "".join(b2u[b] for b in t)
    toks = [base64.b64decode(l.split()[0]) for l in tekken_bytes.splitlines()[:3000]]
    rank = {t: i for i, t in enumerate(toks)}
    keep, merges = [], []
    for t in toks:                           # the tokens whose merge order is their rank order (the importer's condition)
        if len(t) == 1:
            keep.append(t)
            continue
        parts = [bytes([b]) for b in t]
        while len(parts) > 2:                # replay rank-by-bytes merging below t's own rank
            best = min(((rank.get(parts[i] + parts[i + 1], 1 << 30), i) for i in range(len(parts) - 1)))
            if best[0] >= rank[t]:
                break
            parts[best[1]:best[1] + 2] = [parts[best[1]] + parts[best[1] + 1]]
        if len(parts) == 2 and all(p in set(keep) for p in parts):
            keep.append(t)
            merges.append(enc(parts[0]) + " " + enc(parts[1]))
    assert len(keep) > 1500
    rank_file = b"".join(base64.b64encode(t) + b" " + str(i).encode() + b"\n" for i, t in enumerate(keep))
    controls = ["<unk>", "<s>", "</s>", "[INST]", "[/INST]"] + ["<SPECIAL_%d>" % k for k in range(5, 1000)]
    vocab = {c: i for i, c in enumerate(controls)}
    vocab.update({enc(t): 1000 + i for i, t in enumerate(keep)})
    j = {"version": "1.0", "model": {"type": "BPE", "vocab": vocab, "merges": merges, "byte_fallback": False, "ignore_merges": False},
         "added_tokens": [{"id": i, "content": c, "special": True, "single_word": False, "lstrip": False, "rstrip": False, "normalized": False}
                          for i, c in enumerate(controls)],
         "pre_tokenizer": {"type": "ByteLevel", "add_prefix_space": False, "trim_offsets": False, "use_regex": True},
         "decoder": {"type": "ByteLevel", "add_prefix_space": False, "trim_offsets": False, "use_regex": True}}
    data = json.dumps(j).encode()
    out, meta = I.hf_tokenizer_json_to_rank_file(data)
    assert out == rank_file and meta["id_base"] == 1000 and meta["n_ranks"] == len(keep)
    assert meta["special_tokens"] == {c: i for i, c in enumerate(controls)}
    hf = tokenizers.Tokenizer.from_str(data.decode())
    ov = oracle.OracleVocab(rank_file, len(keep))
    for text in ["hello world", "the cat sat on the mat", "abcabc", "  spaced   out  ", "tokenizer"]:
        words = text.split(" ")
        for k, w in enumerate(words):
            piece = ((" " if k else "") + w).encode()
            if not piece.strip():
                continue
            got = hf.encode(piece.decode(), add_special_tokens=False).ids     # (one word: one pre-token under either pattern)
            assert np.array_equal(np.asarray(got) - 1000, ov.encode(0, piece)), (piece, got)
    base0 = json.loads(data)
    base0["model"]["vocab"] = {enc(t): i for i, t in enumerate(keep)}
    base0["added_tokens"] = []
    out0, meta0 = I.hf_tokenizer_json_to_rank_file(json.dumps(base0).encode())
    assert out0 == rank_file and meta0["id_base"] == 0
