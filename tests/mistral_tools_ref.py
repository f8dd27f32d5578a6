"""The Mistral reference of the tool-use tests: mistral_common (1.11) when it imports, else the golden file that
tools/gen_mistral_data.py wrote from it (tests/golden/mistral_tools.npz).  Also the seeded tool conversations both use; the
vocabulary, the tokenizer loader and the text-only conversations are mistral_ref's."""
import json
import os
import random

import numpy as np

import fuzzgen
import mistral_ref as MR

GOLDEN = os.path.join(MR.ROOT, "tests", "golden", "mistral_tools.npz")


def tool_counts():
    """(tool_conversations(), mistral_common's count of each, -1 for a refusal): live when mistral_common imports, else the golden
    file, whose conversations must be the generator's"""
    convs = tool_conversations()
    mt = MR.live_tokenizer()
    if mt is not None:
        return convs, [mistral_count(mt, c, t) for c, t in convs]
    g = np.load(GOLDEN)
    assert bytes(g["conversations"]).decode("utf-8") == MR.conversations_json(convs)
    return convs, g["conversation_counts"].tolist()


def _json_value(rng, pool, depth=0):
    """a random JSON value: nested objects and lists, text from `pool`, integers, floats that print in every form of Python's repr"""
    kind = rng.choice(["str", "str", "int", "float", "bool", "null"] + (["obj", "list"] if depth < 3 else []))
    if kind == "str":
        return rng.choice(pool)
    if kind == "int":
        return rng.choice([0, 7, -3, 21, 1 << 40, -(1 << 62)])
    if kind == "float":
        return rng.choice([0.5, -2.25, 1e-07, 3.0, 1e16, 123456.789, 0.1, 2.5e-05])
    if kind == "bool":
        return rng.random() < 0.5
    if kind == "null":
        return None
    if kind == "list":
        return [_json_value(rng, pool, depth + 1) for _ in range(rng.randint(0, 3))]
    return {rng.choice(TOOL_KEYS): _json_value(rng, pool, depth + 1) for _ in range(rng.randint(0, 3))}


def _schema(rng, pool, depth=0):
    """a random valid JSON Schema (Draft 7) of tool parameters: nested objects, arrays, enums, bounds"""
    kind = rng.choice(["string", "integer", "number", "boolean", "enum"] + (["object", "object", "array"] if depth < 3 else []))
    if kind == "object":
        props = {rng.choice(TOOL_KEYS): _schema(rng, pool, depth + 1) for _ in range(rng.randint(1, 4))}
        s = {"type": "object", "properties": props, "required": rng.sample(sorted(props), rng.randint(0, len(props)))}
    elif kind == "array":
        s = {"type": "array", "items": _schema(rng, pool, depth + 1)}
    elif kind == "enum":
        s = {"type": "string", "enum": rng.sample(["celsius", "fahrenheit", "ºK", "東京", "[INST]"], 3)}
    elif kind == "number":
        s = {"type": "number", "minimum": rng.choice([0, 0.5, -1e-05])}
    else:
        s = {"type": kind}
    if rng.random() < 0.5:
        s["description"] = rng.choice(pool)
    return s


TOOL_KEYS = ["city", "unit", "query", "città", "名前", "[INST]", "</s>", "max_results", "filters", "options"]
# names mistral_common accepts (one trailing "\n" passes its re.match(r"^...$")), then ones it refuses
GOOD_NAMES = ["get_weather", "search-docs", "f", "lookup_2", "a" * 64, "Send_Email-v2", "name\n"]
BAD_NAMES = ["bad name", "[TOOL_CALLS]", "Zürich", "a" * 65, "", "x\n\n"]
GOOD_IDS = ["abc123XYZ", "000000000", "ZZZZzzzz9", "null", "q1w2e3r4t\n"]
BAD_IDS = ["abc123XY", "abc-23XYZ", "[INST]xyz", "ábc123XYZ", ""]


def tool_conversations(seed=23, n=480):
    """n (conversation, tools) pairs of tool use in the gateway's form (schemas/content/tool_call.v1, tool_result.v1,
    tools/tool_unified.v1): zero to three tools with nested parameter schemas; assistant turns of one or several calls, runs of
    tool results whose content is JSON, JSON with other spacing, not JSON or empty; non-ASCII and control-token spellings in names,
    arguments and results; system messages around tool turns.  Most are what mistral_common accepts; some break its rules of
    order, names, call ids or counts of results (and some give an inline_gts tool)."""
    rng = random.Random(seed)
    pool = fuzzgen.fuzz_strings(seed, 300, max_atoms=8) + ["", " ", "Zürich ☀ 東京", "[INST]", "[TOOL_CALLS]", "</s>",
                                                          "[/TOOL_RESULTS]", "[AVAILABLE_TOOLS]", "trailing   ", "tab\tand\nnewline \"q\""]
    pick = lambda good, bad, p_bad: rng.choice(bad) if rng.random() < p_bad else rng.choice(good)
    text = lambda role, t: {"role": role, "content": [{"type": "text", "text": t}]}

    def result_content():
        k = rng.random()
        if k < 0.45:
            return json.dumps(_json_value(rng, pool), ensure_ascii=rng.random() < 0.5)
        if k < 0.6:
            return json.dumps(_json_value(rng, pool), indent=rng.choice([None, 1]), separators=rng.choice([(",", ":"), (" , ", " : ")]))
        if k < 0.7:
            return ""
        return rng.choice(pool + ["{broken", "[1, 2", "NaN is not", "1.50", "  42  ", "\"quoted\"", "null", "1E5"])

    out = []
    for _ in range(n):
        bad = rng.random() < 0.25             # this conversation may break a rule of mistral_common's
        tools = []
        for _ in range(rng.choice([0, 1, 1, 2, 3])):
            if bad and rng.random() < 0.1:
                tools.append({"type": "inline_gts", "schema": {"json_schema": _schema(rng, pool)}})
            else:
                tools.append({"type": "unified", "name": pick(GOOD_NAMES, BAD_NAMES, 0.15 if bad else 0.0),
                              "description": rng.choice(pool), "parameters": {"json_schema": _schema(rng, pool)}})
        conv = []
        if rng.random() < 0.4:
            conv.append(text("system", rng.choice(pool)))
        conv.append(text("user", rng.choice(pool)))
        for _ in range(rng.randint(1, 3)):
            k = rng.random()
            if k < 0.7:                           # a tool turn: calls, then their results
                n_calls = rng.choice([1, 1, 2, 3])
                calls = [{"type": "tool_call", "tool_call": {"id": pick(GOOD_IDS, BAD_IDS, 0.1 if bad else 0.0),
                                                             "name": pick(GOOD_NAMES, BAD_NAMES, 0.1 if bad else 0.0),
                                                             "arguments": {rng.choice(TOOL_KEYS): _json_value(rng, pool)
                                                                           for _ in range(rng.randint(0, 3))}}}
                         for _ in range(n_calls)]
                conv.append({"role": "assistant", "content": calls})
                n_res = n_calls + (rng.choice([-1, 1]) if bad and rng.random() < 0.3 else 0)
                for c in calls[:max(n_res, 0)] + calls[:max(n_res - n_calls, 0)]:
                    rid = c["tool_call"]["id"] if c["tool_call"]["id"] != "null" else rng.choice(GOOD_IDS[:3])
                    conv.append({"role": "tool", "content": [{"type": "tool_result", "tool_result": {"tool_call_id": rid,
                                                                                                    "content": result_content()}}]})
                if rng.random() < 0.5:
                    conv.append(text("assistant", rng.choice(pool) + "ok "))
            else:
                conv.append(text("assistant", rng.choice(pool) + "ok "))
            if bad and rng.random() < 0.2:
                conv.append(text("system", rng.choice(pool)))    # after a tool message or an assistant message: refused
            conv.append(text("user", rng.choice(pool)))
            if rng.random() < 0.25:
                conv.append(text("system", rng.choice(pool)))    # between a user message and the next tool turn
        if rng.random() < 0.3:                    # end on the tool results (accepted) or on the calls (refused unless bad)
            conv = conv[:max(i for i, m in enumerate(conv) if m["role"] == "tool") + 1] if any(m["role"] == "tool" for m in conv) else conv
        if bad and rng.random() < 0.3:            # an order mistral_common refuses
            i = rng.randrange(len(conv))
            conv.insert(i, rng.choice([text("assistant", "x"), text("system", "s"),
                                       {"role": "tool", "content": [{"type": "tool_result", "tool_result": {"tool_call_id": "abc123XYZ", "content": "1"}}]}]))
        if bad and rng.random() < 0.2:            # an assistant turn of text and calls at once
            j = [i for i, m in enumerate(conv) if m["role"] == "assistant"]
            if j:
                conv[j[0]] = {"role": "assistant", "content": conv[j[0]]["content"] + [{"type": "text", "text": "both"}]}
        out.append((conv, tools))
    return out


def mistral_count(tok, conv, tools):
    """len(encode_chat_completion(...).tokens) of a conversation in the gateway's message form and the request's tools, or -1 when
    mistral_common refuses it"""
    from mistral_common.exceptions import MistralCommonException
    from mistral_common.protocol.instruct.messages import AssistantMessage, SystemMessage, TextChunk, ToolMessage, UserMessage
    from mistral_common.protocol.instruct.request import ChatCompletionRequest
    from mistral_common.protocol.instruct.tool_calls import Function, FunctionCall, Tool, ToolCall
    kinds = {"system": SystemMessage, "user": UserMessage, "assistant": AssistantMessage}
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
            calls = [ToolCall(id=c["id"], function=FunctionCall(name=c["name"], arguments=c["arguments"]))
                     for c in (p["tool_call"] for p in m["content"] if p["type"] == "tool_call")]
            msgs.append(kinds[m["role"]](content=content, tool_calls=calls) if calls else kinds[m["role"]](content=content))
        return len(tok.encode_chat_completion(ChatCompletionRequest(messages=msgs, tools=mtools)).tokens)
    except (MistralCommonException, ValueError):     # (pydantic's ValidationError is a ValueError)
        return -1
