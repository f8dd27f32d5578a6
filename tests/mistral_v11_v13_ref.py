"""The Mistral instruct V11 and V13 reference of the V11 / V13 template tests: mistral_common (1.11) when it imports, else the
golden file that tools/gen_mistral_v13_data.py wrote from it (tests/golden/mistral_v11_v13.npz).  Also the seeded conversations
both use: the text-only, tool and V7 conversations of the earlier tests, and conversations built around what V11 and V13 do
differently.

mistral_common ships no V11 or V13 Tekken file, and tekken_240911 has no [ARGS] or [CALL_ID] control token.  The reference
tokenizer is therefore tekken_240911 declared as version v11 or v13, with two of its unused control slots renamed: ARGS_SLOT
becomes [ARGS] and CALL_ID_SLOT becomes [CALL_ID].  Counts do not depend on which slots these are (each control token counts one),
and parity is pinned on this stand-in only, not on any V11 or V13 model's own tekken.json."""
import json
import os
import random

import numpy as np

import fuzzgen
import mistral_ref as MR
import mistral_tools_ref as MTR
import mistral_v7_ref as R7

GOLDEN = os.path.join(MR.ROOT, "tests", "golden", "mistral_v11_v13.npz")
VERSIONS = (11, 13)
ARGS_SLOT, CALL_ID_SLOT = 20, 21        # <SPECIAL_20> and <SPECIAL_21> of tekken_240911: the first two unused control slots


def live_tokenizer(version):
    """mistral_common's MistralTokenizer of tekken_240911.json as a Tekken file of `version` (11 or 13) with [ARGS] and [CALL_ID]
    at ARGS_SLOT and CALL_ID_SLOT: InstructTokenizerV11 or V13, MistralRequestValidatorV13 (default mode) and
    InstructRequestNormalizerV13, as mistral_common pairs them for these versions; None when mistral_common does not import"""
    mt = MR.live_tokenizer()
    if mt is None:
        return None
    from mistral_common.protocol.instruct.normalize import InstructRequestNormalizerV13
    from mistral_common.protocol.instruct.validator import MistralRequestValidatorV13
    from mistral_common.tokens.tokenizers.base import TokenizerVersion
    from mistral_common.tokens.tokenizers.instruct import InstructTokenizerV11, InstructTokenizerV13
    from mistral_common.tokens.tokenizers.mistral import MistralTokenizer
    from mistral_common.tokens.tokenizers.tekken import Tekkenizer
    base = mt.instruct_tokenizer.tokenizer
    specials = list(Tekkenizer.DEPRECATED_SPECIAL_TOKENS)
    assert [s["rank"] for s in specials] == list(range(ARGS_SLOT))      # the slots follow the named control tokens
    specials += [{"rank": ARGS_SLOT, "token_str": "[ARGS]", "is_control": True},
                 {"rank": CALL_ID_SLOT, "token_str": "[CALL_ID]", "is_control": True}]
    with open(base.file_path, encoding="utf-8") as f:
        model = json.load(f)
    tok = Tekkenizer(model["vocab"], specials, pattern=model["config"]["pattern"], vocab_size=model["config"]["default_vocab_size"],
                     num_special_tokens=model["config"]["default_num_special_tokens"], version=TokenizerVersion("v%d" % version),
                     name="tekken_240911_v%d" % version)
    instruct = {11: InstructTokenizerV11, 13: InstructTokenizerV13}[version]
    return MistralTokenizer(instruct(tok), validator=MistralRequestValidatorV13(), request_normalizer=InstructRequestNormalizerV13.normalizer())


def requests():
    """every (conversation, tools) pair the golden file holds: the text-only conversations of mistral_ref, the tool conversations
    of mistral_tools_ref, the V7 conversations of mistral_v7_ref and v13_conversations()"""
    return R7.requests() + v13_conversations()


def golden_counts():
    """(requests(), mistral_common's V7, V11 and V13 count of each; -1 for a refusal), from the golden file, whose requests must be
    the generators'"""
    reqs = requests()
    g = np.load(GOLDEN)
    assert bytes(g["requests"]).decode("utf-8") == MR.conversations_json(reqs)
    return reqs, g["v7_counts"].tolist(), g["v11_counts"].tolist(), g["v13_counts"].tolist()


def mistral_count(tok, conv, tools):
    """mistral_v7_ref.mistral_count under V11 or V13, or -1 when mistral_common refuses the request; InstructTokenizerV13 refuses
    a tool call whose id is "null" with an assertion"""
    try:
        return R7.mistral_count(tok, conv, tools)
    except AssertionError:
        return -1


def _text(role, *texts):
    return {"role": role, "content": [{"type": "text", "text": t} for t in texts]}


def v13_conversations(seed=53, n=480):
    """n (conversation, tools) pairs in the gateway's form around what V11 and V13 do otherwise than V7: assistant turns of one to
    four calls, with ids and with "null" ids (refused by V13), some with one id twice (refused); tools with one user turn and
    with several, so that the first and the last user message differ; results in the order of the calls or another, some that
    answer a call twice, answer no call of the assistant message before them or leave one unanswered (refused); result content
    that is JSON, JSON in other spacing, not JSON, non-ASCII or empty; system messages, text beside calls and prefix turns."""
    rng = random.Random(seed)
    pool = fuzzgen.fuzz_strings(seed, 200, max_atoms=8) + ["", " ", "Zürich ☀ 東京", "[ARGS]", "[CALL_ID]", "[TOOL_CALLS]",
                                                          "[TOOL_RESULTS]", "trailing   ", "\n\nafter breaks"]
    ids = [i for i in MTR.GOOD_IDS if i != "null"] + ["a1b2c3d4e", "Zz9Yy8Xx7", "123456789"]

    def content():
        k = rng.random()
        if k < 0.35:
            return json.dumps(MTR._json_value(rng, pool), ensure_ascii=rng.random() < 0.5)
        if k < 0.5:
            return json.dumps(MTR._json_value(rng, pool), indent=rng.choice([None, 2]), separators=rng.choice([(",", ":"), (" , ", " : ")]))
        if k < 0.6:
            return ""
        return rng.choice(pool + ["東京 ☀ 21°C", "ok", "  {\"a\" : 1}  ", "[1, 2", "NaN", "1E5", "\"quoted\"", "null"])

    def calls(k, bad):
        cids = rng.sample(ids, k)
        if bad and rng.random() < 0.3:
            cids[-1] = "null"                                     # no id: V11 prints none, V13 refuses it
        elif bad and k > 1 and rng.random() < 0.3:
            cids[-1] = cids[0]                                    # one id twice in one message: refused
        return [{"type": "tool_call", "tool_call": {"id": c, "name": rng.choice(MTR.GOOD_NAMES),
                                                    "arguments": {rng.choice(MTR.TOOL_KEYS): MTR._json_value(rng, pool)
                                                                  for _ in range(rng.randint(0, 3))}}} for c in cids]

    def results(cs, bad):
        rids = [c["tool_call"]["id"] for c in cs if c["tool_call"]["id"] != "null"]
        if rng.random() < 0.5:
            rng.shuffle(rids)                                     # answered in another order than called
        if bad:
            k = rng.random()
            if k < 0.3 and rids:
                rids.append(rids[0])                              # one call answered twice
            elif k < 0.6 and rids:
                rids[-1] = rng.choice([i for i in ids if i not in rids])      # an id no call of the turn has
            elif k < 0.8 and rids:
                rids.pop()                                        # one call left unanswered
        return [{"role": "tool", "content": [{"type": "tool_result", "tool_result": {"tool_call_id": r, "content": content()}}]}
                for r in rids]

    out = []
    for _ in range(n):
        bad = rng.random() < 0.3                                  # this conversation may break a rule of V11's or V13's
        tools = [{"type": "unified", "name": rng.choice(MTR.GOOD_NAMES), "description": rng.choice(pool),
                  "parameters": {"json_schema": MTR._schema(rng, pool)}} for _ in range(rng.choice([0, 1, 1, 2, 3]))]
        conv = [_text("system", rng.choice(pool)) for _ in range(rng.choice([0, 0, 1, 2]))]
        for _ in range(rng.choice([1, 1, 2, 3, 4])):              # several user turns: the tools' place differs in V13
            conv.append(_text("user", *[rng.choice(pool) for _ in range(rng.choice([1, 1, 2]))]))
            if rng.random() < 0.15:
                conv.append(_text("system", rng.choice(pool)))
            if rng.random() < 0.2:
                conv.append(_text("assistant", rng.choice(pool) + "ok "))
                continue
            for _ in range(rng.choice([1, 1, 2])):                # one or two rounds of calls and their results
                cs = calls(rng.choice([1, 1, 2, 3, 4]), bad)
                if rng.random() < 0.3:
                    conv.append({"role": "assistant", "content": [{"type": "text", "text": rng.choice(pool) + " "}] + cs})
                else:
                    conv.append({"role": "assistant", "content": cs})
                conv += results(cs, bad)
            if rng.random() < 0.5:
                conv.append(_text("assistant", rng.choice(pool) + "done"))
        k = rng.random()
        if k < 0.4:
            conv.append(_text("user", rng.choice(pool)))
        elif k < 0.6:                                             # a call without an id, unanswered, then a user turn
            c = calls(1, False)[0]
            c["tool_call"]["id"] = "null"
            conv += [{"role": "assistant", "content": [c]}, _text("user", rng.choice(pool))]
        elif k < 0.8 and conv[-1]["role"] != "assistant":         # the start of the reply, text or calls
            parts = [{"type": "text", "text": rng.choice(pool) + "{"}] if rng.random() < 0.5 else calls(1, bad)
            conv.append({"role": "assistant", "prefix": True, "content": parts})
        if bad and rng.random() < 0.15 and conv[0]["role"] == "user" and len(conv) > 1:
            conv.insert(0, {"role": "assistant", "content": calls(1, False)})    # calls in the first message: not checked
        out.append((conv, tools))
    return out
