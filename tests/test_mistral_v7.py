"""The "mistral-v7" chat template without a GPU: conversations counted as mistral_common's InstructTokenizerV7 counts them (its golden
counts, and live on fresh seeds when mistral_common imports), through the gateway service over the C oracle; the refusals; the V3
counts of the same requests, unchanged; the models that use V7."""
import pytest

import mistral_ref as MR
import mistral_tools_ref as MTR
import mistral_v7_ref as R
from cfbpe import plugin as P
from cfbpe import vocabs as V

CTX = P.SecurityContext.anonymous()
V3, V7 = P.CHAT_TEMPLATES["mistral-v3"], P.CHAT_TEMPLATES["mistral-v7"]
MODEL = "mistral::mistral-small-2501"


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


def _count(service, conv, tools, tpl):
    """the gateway's count, -1 for InvalidInput"""
    try:
        return service.count_chat_tokens(CTX, MODEL, conv, tpl, tools).input_tokens
    except P.InvalidInput:
        return -1


def _msg(role, t):
    return {"role": role, "content": [{"type": "text", "text": t}]}


def test_v7_counts_as_mistral_common(service):
    reqs, _, want = R.golden_counts()
    assert len(reqs) >= 1200 and sum(w >= 0 for w in want) >= 900 and sum(w < 0 for w in want) >= 150
    for (conv, tools), w in zip(reqs, want):
        assert _count(service, conv, tools, V7) == w, (conv, tools)


def test_v3_counts_of_the_same_requests_do_not_move(service):
    """the V3 template counts every request that sets no prefix as mistral_common's V3 does; on many of them V3 and V7 differ,
    and the gateway gives both"""
    reqs, want3, want7 = R.golden_counts()
    differ = 0
    for (conv, tools), w3, w7 in zip(reqs, want3, want7):
        if R.uses_prefix(conv):             # (the V3 template does not read prefix)
            continue
        assert _count(service, conv, tools, V3) == w3, (conv, tools)
        differ += w3 >= 0 and w7 >= 0 and w3 != w7
    assert differ >= 500


def test_the_golden_requests_cover_what_v7_changes():
    reqs, want3, want7 = R.golden_counts()
    ok = [(c, t) for (c, t), w in zip(reqs, want7) if w >= 0]
    roles = [[m["role"] for m in c] for c, _ in ok]
    results = [p["tool_result"]["content"] for c, _ in ok for m in c for p in m["content"] if p["type"] == "tool_result"]
    assert sum(r[0] == "system" for r in roles) >= 100                                       # at the start
    assert sum(any(a == "user" and b == "system" and "user" in r[i + 2:] for i, (a, b) in enumerate(zip(r, r[1:]))) for r in roles) >= 50
    assert sum(any(a == b == "system" for a, b in zip(r, r[1:])) for r in roles) >= 50       # several in a row
    assert sum(set(r) == {"system"} for r in roles) >= 10                                    # alone
    assert sum(c == "" for c in results) >= 50 and sum(not c.isascii() for c in results) >= 50
    assert sum(c[-1].get("prefix") is True for c, _ in ok) >= 100
    assert sum(bool(t) and any(p["type"] == "tool_call" for m in c for p in m["content"]) for c, t in ok) >= 100
    assert sum(bool(t) and not any(p["type"] == "tool_call" for m in c for p in m["content"]) for c, t in ok) >= 50
    assert sum(w3 < 0 <= w7 for w3, w7 in zip(want3, want7)) >= 100                          # text and calls at once ...


def test_v7_counts_live_on_fresh_seeds(service):
    tok = R.live_v7_tokenizer()
    if tok is None:
        pytest.skip("mistral_common is not installed")
    reqs = R.v7_conversations(seed=4049, n=300) + MTR.tool_conversations(seed=4051, n=200) + [(c, []) for c in MR.conversations(seed=4057, n=100)]
    for conv, tools in reqs:
        assert _count(service, conv, tools, V7) == R.mistral_count(tok, conv, tools), (conv, tools)


def weather_example():
    """(messages, tools) that V7 renders as
    <s>[SYSTEM_PROMPT]Be brief.[/SYSTEM_PROMPT][INST]Weather in Paris?[/INST][TOOL_CALLS][{"name": "get_weather", "arguments":
    {"city": "Paris"}, "id": "abc123XYZ"}]</s>[TOOL_RESULTS]abc123XYZ[TOOL_CONTENT]{"temp": 21}[/TOOL_RESULTS]21 C.</s>
    [AVAILABLE_TOOLS][...][/AVAILABLE_TOOLS][INST]And Rome?[/INST]"""
    tools = [{"type": "unified", "name": "get_weather", "description": "Weather of a city",
              "parameters": {"json_schema": {"type": "object", "properties": {"city": {"type": "string"}}, "required": ["city"]}}}]
    messages = [_msg("system", "Be brief."), _msg("user", "Weather in Paris?"),
                {"role": "assistant", "content": [{"type": "tool_call",
                                                   "tool_call": {"id": "abc123XYZ", "name": "get_weather", "arguments": {"city": "Paris"}}}]},
                {"role": "tool", "content": [{"type": "tool_result", "tool_result": {"tool_call_id": "abc123XYZ", "content": '{"temp":21}'}}]},
                _msg("assistant", "21 C."), _msg("user", "And Rome?")]
    return messages, tools


def test_weather_example(service):
    messages, tools = weather_example()
    texts, n_ctl = P.mistral_instruct_texts(messages, tools, 7)
    assert [t for t in texts if t] == [
        "Be brief.", "Weather in Paris?", '[{"name": "get_weather", "arguments": {"city": "Paris"}, "id": "abc123XYZ"}]',
        "abc123XYZ", '{"temp": 21}', "21 C.",
        '[{"type": "function", "function": {"name": "get_weather", "description": "Weather of a city", "parameters": '
        '{"type": "object", "properties": {"city": {"type": "string"}}, "required": ["city"]}}}]', "And Rome?"]
    # <s> [SYSTEM_PROMPT] [/SYSTEM_PROMPT] [INST] [/INST] [TOOL_CALLS] </s> [TOOL_RESULTS] [TOOL_CONTENT] [/TOOL_RESULTS] </s>
    # [AVAILABLE_TOOLS] [/AVAILABLE_TOOLS] [INST] [/INST]
    assert n_ctl == 15
    assert service.count_chat_tokens(CTX, MODEL, messages, V7, tools).input_tokens == 127
    assert service.count_chat_tokens(CTX, MODEL, messages, V3, tools).input_tokens == 133
    assert service.count_chat_tokens(CTX, MODEL, messages, V7).input_tokens == 68


def test_tool_results_and_prefix():
    """a result's content is the JSON it parses to written again, else as given, "" is "{}"; a trailing assistant message with
    prefix has no </s>; text and calls in one assistant turn.  Controls: <s> [INST] [/INST] [TOOL_CALLS] </s> [TOOL_RESULTS]
    [TOOL_CONTENT] [/TOOL_RESULTS]"""
    def result(content):
        conv = [_msg("user", "q"), {"role": "assistant", "content": [{"type": "tool_call", "tool_call": {"id": "null", "name": "f", "arguments": {}}}]},
                {"role": "tool", "content": [{"type": "tool_result", "tool_result": {"tool_call_id": "abc123XYZ", "content": content}}]}]
        texts, n_ctl = P.mistral_instruct_texts(conv, version=7)
        assert texts[:4] == ["q", "", '[{"name": "f", "arguments": {}}]', "abc123XYZ"] and n_ctl == 8
        return texts[4]
    assert result('{"a":1,\n "b" : [1.50, "\\u00e9"]}') == '{"a": 1, "b": [1.5, "é"]}'
    assert result("not JSON: Zürich") == "not JSON: Zürich"
    assert result("") == "{}"
    assert result('"quoted"') == '"quoted"'
    assert result(" 东京 ") == " 东京 "
    conv = [_msg("user", "q"), {"role": "assistant", "prefix": True, "content": [{"type": "text", "text": "Sure: "}]}]
    assert P.mistral_instruct_texts(conv, version=7) == (["q", "Sure:"], 3)        # <s> [INST] [/INST]
    call = {"type": "tool_call", "tool_call": {"id": "abc123XYZ", "name": "f", "arguments": {"x": 1}}}
    conv = [_msg("user", "q"), {"role": "assistant", "content": [{"type": "text", "text": "Let me look. "}, call]},
            {"role": "tool", "content": [{"type": "tool_result", "tool_result": {"tool_call_id": "abc123XYZ", "content": "1"}}]}]
    assert P.mistral_instruct_texts(conv, version=7) == (
        ["q", "Let me look.", '[{"name": "f", "arguments": {"x": 1}, "id": "abc123XYZ"}]', "abc123XYZ", "1"], 8)


REFUSALS = ["system_after_assistant", "system_after_tool", "prefix_not_last", "prefix_on_user", "prefix_not_bool", "assistant_last",
            "empty_assistant", "empty_prefix", "missing_result", "tool_after_user", "tool_alone", "call_id", "result_id", "name",
            "inline_gts", "no_message", "version"]


@pytest.mark.parametrize("case", REFUSALS)
def test_refusals(case):
    """each raises InvalidInput; where mistral_common has a form for the input, it refuses it too"""
    messages, tools = weather_example()
    version = 7
    if case == "system_after_assistant":
        messages.insert(5, _msg("system", "s"))
    elif case == "system_after_tool":
        messages.insert(4, _msg("system", "s"))
    elif case == "prefix_not_last":
        messages[4]["prefix"] = True
    elif case == "prefix_on_user":
        messages[5]["prefix"] = True
    elif case == "prefix_not_bool":
        messages.append(dict(_msg("assistant", "x"), prefix="yes"))
    elif case == "assistant_last":
        messages.append(_msg("assistant", "x"))
    elif case == "empty_assistant":
        messages[4] = _msg("assistant", "")
    elif case == "empty_prefix":
        messages.append(dict(_msg("assistant", ""), prefix=True))
    elif case == "missing_result":
        del messages[3]
    elif case == "tool_after_user":
        messages.insert(2, messages[3])
    elif case == "tool_alone":
        messages = [messages[3]]
    elif case == "call_id":
        messages[2]["content"][0]["tool_call"]["id"] = "call_abc123"
    elif case == "result_id":
        messages[3]["content"][0]["tool_result"]["tool_call_id"] = "null"
    elif case == "name":
        tools[0]["name"] = "get weather"
    elif case == "inline_gts":
        tools = [{"type": "inline_gts", "schema": {"json_schema": {"type": "object"}}}]
    elif case == "no_message":
        messages = []
    elif case == "version":
        version = 11
    with pytest.raises(P.InvalidInput):
        P.mistral_instruct_texts(messages, tools, version)
    tok = R.live_v7_tokenizer()
    if tok is not None and case not in ("prefix_on_user", "prefix_not_bool", "version"):
        assert R.mistral_count(tok, messages, tools) == -1


def test_templates_and_models():
    assert V3.instruct_version == 3 and V7 == P.ChatTemplate("mistral", instruct_version=7)
    assert P.ChatTemplate("mistral") == V3
    for model in ("mistral::mistral-large-2411", "mistral::pixtral-large-2411", "mistral::mistral-small-2501", "mistral::mistral-small-2503"):
        assert V.tokenizer_for_model(model) == V.ModelTokenizer("mistral_tekken", "mistral-v7", stand_in=True)
        assert V.for_model(model) == "mistral_tekken"
    for model in ("mistral::mistral-nemo", "mistral::pixtral-12b"):
        assert V.tokenizer_for_model(model) == V.ModelTokenizer("mistral_tekken", "mistral-v3")
    assert V.MODEL_VOCABS == {m: t.vocab for m, t in V.MODEL_TOKENIZERS.items()}
    assert all(t.chat_template in P.CHAT_TEMPLATES for t in V.MODEL_TOKENIZERS.values() if t.chat_template)
    with pytest.raises(V.VocabUnavailable):
        V.tokenizer_for_model("mistral::mistral-large-2407")
