"""The Mistral instruct V7 reference of the V7 template tests: mistral_common (1.11) when it imports, else the golden file that
tools/gen_mistral_v7_data.py wrote from it (tests/golden/mistral_v7.npz).  Also the seeded conversations both use: the text-only
and tool conversations of the V3 tests, and conversations built around what V7 does differently."""
import json
import os
import random

import numpy as np

import fuzzgen
import mistral_ref as MR
import mistral_tools_ref as MTR

GOLDEN = os.path.join(MR.ROOT, "tests", "golden", "mistral_v7.npz")


def live_v7_tokenizer():
    """mistral_common's MistralTokenizer of tekken_240911.json with InstructTokenizerV7, the V7 validator (MistralRequestValidatorV5,
    default mode) and the V7 request normalizer; None when mistral_common does not import"""
    mt = MR.live_tokenizer()
    if mt is None:
        return None
    from mistral_common.protocol.instruct.normalize import InstructRequestNormalizerV7
    from mistral_common.protocol.instruct.validator import MistralRequestValidatorV5
    from mistral_common.tokens.tokenizers.instruct import InstructTokenizerV7
    from mistral_common.tokens.tokenizers.mistral import MistralTokenizer
    return MistralTokenizer(InstructTokenizerV7(mt.instruct_tokenizer.tokenizer), validator=MistralRequestValidatorV5(),
                            request_normalizer=InstructRequestNormalizerV7.normalizer())


def uses_prefix(conv):
    """whether a message sets `prefix`, which the V3 template does not read"""
    return any("prefix" in m for m in conv)


def requests():
    """every (conversation, tools) pair the golden file holds: the text-only conversations of mistral_ref, the tool conversations
    of mistral_tools_ref and v7_conversations()"""
    return [(c, []) for c in MR.conversations()] + MTR.tool_conversations() + v7_conversations()


def golden_counts():
    """(requests(), mistral_common's V3 count of each, its V7 count of each; -1 for a refusal), from the golden file, whose
    requests must be the generators'"""
    reqs = requests()
    g = np.load(GOLDEN)
    assert bytes(g["requests"]).decode("utf-8") == MR.conversations_json(reqs)
    return reqs, g["v3_counts"].tolist(), g["v7_counts"].tolist()


def _text(role, *texts):
    return {"role": role, "content": [{"type": "text", "text": t} for t in texts]}


def v7_conversations(seed=37, n=400):
    """n (conversation, tools) pairs in the gateway's form around what V7 does otherwise than V3: system messages at the start,
    between user turns, several in a row, after an assistant or tool message (refused) and alone; assistant turns of text and calls
    at once, or split over two messages, or an empty text merged with calls or text; tool results whose content is JSON in other
    spacing, not JSON, non-ASCII or empty, with call ids that end in "\\n"; conversations that end on an assistant message with
    "prefix": true (text, calls or both), and some with prefix on an earlier message (refused); tools with and without calls."""
    rng = random.Random(seed)
    pool = fuzzgen.fuzz_strings(seed, 200, max_atoms=8) + ["", " ", "Zürich ☀ 東京", "[SYSTEM_PROMPT]", "[/SYSTEM_PROMPT]",
                                                          "[TOOL_CONTENT]", "[TOOL_RESULTS]", "trailing   ", "\n\nafter breaks"]
    good_ids = [i for i in MTR.GOOD_IDS if i != "null"]

    def content():
        k = rng.random()
        if k < 0.35:
            return json.dumps(MTR._json_value(rng, pool), ensure_ascii=rng.random() < 0.5)
        if k < 0.5:
            return json.dumps(MTR._json_value(rng, pool), indent=rng.choice([None, 2]), separators=rng.choice([(",", ":"), (" , ", " : ")]))
        if k < 0.62:
            return ""
        return rng.choice(pool + ["東京 ☀ 21°C", "ok", "  {\"a\" : 1}  ", "[1, 2", "NaN", "-0", "1E5", "\"quoted\"", "null"])

    def calls(k):
        return [{"type": "tool_call", "tool_call": {"id": rng.choice(good_ids + ["null"]), "name": rng.choice(MTR.GOOD_NAMES),
                                                    "arguments": {rng.choice(MTR.TOOL_KEYS): MTR._json_value(rng, pool)
                                                                  for _ in range(rng.randint(0, 2))}}} for _ in range(k)]

    def results(cs):
        return [{"role": "tool", "content": [{"type": "tool_result", "tool_result": {
            "tool_call_id": c["tool_call"]["id"] if c["tool_call"]["id"] != "null" else rng.choice(good_ids),
            "content": content()}}]} for c in cs]

    def systems(k):
        return [_text("system", *[rng.choice(pool) for _ in range(rng.choice([1, 1, 2]))]) for _ in range(k)]

    out = []
    for _ in range(n):
        tools = [{"type": "unified", "name": rng.choice(MTR.GOOD_NAMES), "description": rng.choice(pool),
                  "parameters": {"json_schema": MTR._schema(rng, pool)}} for _ in range(rng.choice([0, 0, 1, 2]))]
        if rng.random() < 0.05:                   # system messages alone: no [INST], so the tools are not shown
            out.append((systems(rng.randint(1, 3)), tools))
            continue
        conv = systems(rng.choice([0, 0, 1, 1, 2, 3]))
        for _ in range(rng.randint(1, 3)):
            conv.append(_text("user", *[rng.choice(pool) for _ in range(rng.choice([1, 1, 2]))]))
            conv += systems(rng.choice([0, 0, 0, 1, 2]))          # between a user turn and the next assistant turn
            k = rng.random()
            if k < 0.2:
                conv.append(_text("assistant", rng.choice(pool) + "ok "))
                continue
            cs = calls(rng.choice([1, 1, 2]))
            if k < 0.5:                                           # calls only
                conv.append({"role": "assistant", "content": cs})
            elif k < 0.75:                                        # text and calls in one message
                conv.append({"role": "assistant", "content": [{"type": "text", "text": rng.choice(pool)}] + cs})
            elif k < 0.9:                                         # text, then the calls in a message of their own
                conv += [_text("assistant", rng.choice(pool) + " "), {"role": "assistant", "content": cs}]
            else:                                                 # an empty text merged with the calls
                conv += [_text("assistant", ""), {"role": "assistant", "content": cs}]
            conv += results(cs[:len(cs) - (1 if rng.random() < 0.05 else 0)])
            if rng.random() < 0.4:
                conv.append(_text("assistant", rng.choice(pool) + "done"))
            if rng.random() < 0.05:                               # after an assistant or tool message: refused
                conv += systems(1)
        k = rng.random()
        if k < 0.45:
            conv.append(_text("user", rng.choice(pool)))
            conv += systems(rng.choice([0, 0, 0, 1]))             # last: after the last [INST]
        elif k < 0.75 and conv[-1]["role"] != "assistant":        # the start of the reply
            if rng.random() < 0.7:
                parts = [{"type": "text", "text": rng.choice(pool) + rng.choice(["", "  ", "{"])}]
            else:
                parts = [{"type": "text", "text": rng.choice(pool)}] + calls(1) if rng.random() < 0.5 else calls(1)
            conv.append({"role": "assistant", "prefix": True, "content": parts})
        elif k < 0.8:                                             # an empty text merged with more text
            conv += [_text("assistant", ""), _text("assistant", rng.choice(pool) + "!"), {"role": "assistant", "prefix": True,
                                                                                         "content": [{"type": "text", "text": "So"}]}]
        if rng.random() < 0.04:                                   # prefix on a message that is not the last: refused
            j = [i for i, m in enumerate(conv[:-1]) if m["role"] == "assistant"]
            if j:
                conv[j[0]] = dict(conv[j[0]], prefix=True)
        out.append((conv, tools))
    return out


def mistral_count(tok, conv, tools):
    """len(encode_chat_completion(...).tokens) of a conversation in the gateway's message form and the request's tools, or -1 when
    mistral_common refuses it; an assistant message's `prefix` becomes AssistantMessage.prefix"""
    from mistral_common.exceptions import MistralCommonException
    from mistral_common.protocol.instruct.messages import AssistantMessage, SystemMessage, TextChunk, ToolMessage, UserMessage
    from mistral_common.protocol.instruct.request import ChatCompletionRequest
    from mistral_common.protocol.instruct.tool_calls import Function, FunctionCall, Tool, ToolCall
    kinds = {"system": SystemMessage, "user": UserMessage}
    try:
        if any(t["type"] != "unified" for t in tools):
            return -1                         # nothing for the model to see: the gateway refuses it
        mtools = [Tool(function=Function(name=t["name"], description=t["description"], parameters=t["parameters"]["json_schema"]))
                  for t in tools] or None
        msgs = []
        for m in conv:
            if m["role"] == "tool":
                r = [p["tool_result"] for p in m["content"] if p["type"] == "tool_result"][0]
                msgs.append(ToolMessage(tool_call_id=r["tool_call_id"], content=r["content"]))
                continue
            texts = [p["text"] for p in m["content"] if p["type"] == "text"]
            content = texts[0] if len(texts) == 1 else [TextChunk(text=t) for t in texts]
            if m["role"] != "assistant":
                msgs.append(kinds[m["role"]](content=content))
                continue
            calls = [ToolCall(id=c["id"], function=FunctionCall(name=c["name"], arguments=c["arguments"]))
                     for c in (p["tool_call"] for p in m["content"] if p["type"] == "tool_call")]
            msgs.append(AssistantMessage(content=content, tool_calls=calls or None, prefix=m.get("prefix", False)))
        return len(tok.encode_chat_completion(ChatCompletionRequest(messages=msgs, tools=mtools)).tokens)
    except (MistralCommonException, ValueError):     # (pydantic's ValidationError is a ValueError)
        return -1
