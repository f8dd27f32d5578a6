"""The "mistral" chat template on tool use without a GPU: tool definitions, tool calls and tool results counted as mistral_common's
encode_chat_completion counts them (live when it imports, else its golden counts), through the gateway service over the C oracle."""
import pytest

import mistral_ref as MR
import mistral_tools_ref as MTR
from cfbpe import plugin as P

CTX = P.SecurityContext.anonymous()
TPL = P.CHAT_TEMPLATES["mistral-v3"]


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


def _msg(role, t):
    return {"role": role, "content": [{"type": "text", "text": t}]}


def weather_example():
    """(messages, tools) that encode_chat_completion renders as
    <s>[INST]Weather in Paris?[/INST][TOOL_CALLS][{"name": "get_weather", "arguments": {"city": "Paris"}, "id": "abc123XYZ"}]</s>
    [TOOL_RESULTS]{"content": {"temp": 21}, "call_id": "abc123XYZ"}[/TOOL_RESULTS]21 C.</s>
    [AVAILABLE_TOOLS][{"type": "function", "function": {...}}][/AVAILABLE_TOOLS][INST]Be brief.\n\nAnd Rome?[/INST]"""
    tools = [{"type": "unified", "name": "get_weather", "description": "Weather of a city",
              "parameters": {"json_schema": {"type": "object", "properties": {"city": {"type": "string"}}, "required": ["city"]}}}]
    messages = [_msg("system", "Be brief."), _msg("user", "Weather in Paris?"),
                {"role": "assistant", "content": [{"type": "tool_call",
                                                   "tool_call": {"id": "abc123XYZ", "name": "get_weather", "arguments": {"city": "Paris"}}}]},
                {"role": "tool", "content": [{"type": "tool_result", "tool_result": {"tool_call_id": "abc123XYZ", "content": '{"temp": 21}'}}]},
                _msg("assistant", "21 C."), _msg("user", "And Rome?")]
    return messages, tools


def test_tool_conversations_count_as_mistral_common(service):
    convs, want = MTR.tool_counts()
    assert len(convs) >= 400 and sum(w >= 0 for w in want) >= 300 and sum(w < 0 for w in want) >= 50
    for (conv, tools), w in zip(convs, want):
        if w < 0:                           # mistral_common refuses it (or the tools give the model nothing to read)
            with pytest.raises(P.InvalidInput):
                service.count_chat_tokens(CTX, "mistral::mistral-nemo", conv, TPL, tools)
        else:
            assert service.count_chat_tokens(CTX, "mistral::mistral-nemo", conv, TPL, tools).input_tokens == w, (conv, tools)


def test_weather_example(service):
    messages, tools = weather_example()
    texts, n_ctl = P.mistral_instruct_texts(messages, tools)
    assert texts == ["Weather in Paris?", '[{"name": "get_weather", "arguments": {"city": "Paris"}, "id": "abc123XYZ"}]',
                     '{"content": {"temp": 21}, "call_id": "abc123XYZ"}', "21 C.",
                     '[{"type": "function", "function": {"name": "get_weather", "description": "Weather of a city", "parameters": '
                     '{"type": "object", "properties": {"city": {"type": "string"}}, "required": ["city"]}}}]', "Be brief.\n\nAnd Rome?"]
    assert n_ctl == 12                      # <s> [INST] [/INST] [TOOL_CALLS] </s> [TOOL_RESULTS] [/TOOL_RESULTS] </s>
    assert service.count_chat_tokens(CTX, "mistral::mistral-nemo", messages, TPL, tools).input_tokens == 133
    # without tools: no [AVAILABLE_TOOLS] block (encode_chat_completion with tools=None or [] gives 74)
    assert service.count_chat_tokens(CTX, "mistral::mistral-nemo", messages, TPL, []).input_tokens == 74
    assert service.count_chat_tokens(CTX, "mistral::mistral-nemo", messages, TPL).input_tokens == 74


def test_tool_json_as_mistral_common_prints_it():
    """a result that parses as JSON is embedded as JSON in json.dumps's spacing, non-ASCII as is; one that does not is a string;
    an empty one is {}; a call id "null" is not printed"""
    def result(content):
        conv = [_msg("user", "q"), {"role": "assistant", "content": [{"type": "tool_call", "tool_call": {"id": "null", "name": "f", "arguments": {}}}]},
                {"role": "tool", "content": [{"type": "tool_result", "tool_result": {"tool_call_id": "abc123XYZ", "content": content}}]}]
        texts, n_ctl = P.mistral_instruct_texts(conv)
        assert texts[1] == '[{"name": "f", "arguments": {}}]' and n_ctl == 7
        return texts[2]
    assert result('{"a":1,\n "b" : [1.50, "\\u00e9"]}') == '{"content": {"a": 1, "b": [1.5, "é"]}, "call_id": "abc123XYZ"}'
    assert result("not JSON: Zürich") == '{"content": "not JSON: Zürich", "call_id": "abc123XYZ"}'
    assert result("") == '{"content": {}, "call_id": "abc123XYZ"}'
    assert result('"quoted"') == '{"content": "quoted", "call_id": "abc123XYZ"}'


@pytest.mark.parametrize("case", ["inline_gts", "reference", "name", "call_in_user", "result_in_assistant", "text_and_call",
                                  "two_results", "call_id", "result_id", "missing_result", "system_after_tool", "tool_after_user",
                                  "tool_alone", "arguments"])
def test_refusals(case):
    messages, tools = weather_example()
    call = messages[2]["content"][0]
    if case == "inline_gts":
        tools = [{"type": "inline_gts", "schema": {"json_schema": {"type": "object"}}}]
    elif case == "reference":
        tools = [{"type": "reference", "schema_id": "gts.x.tools.weather.v1~"}]
    elif case == "name":
        tools[0]["name"] = "get weather"
    elif case == "call_in_user":
        messages[1]["content"].append(call)
    elif case == "result_in_assistant":
        messages[4]["content"].append(messages[3]["content"][0])
    elif case == "text_and_call":
        messages[2]["content"].append({"type": "text", "text": "let me look"})
    elif case == "two_results":
        messages[3]["content"].append(messages[3]["content"][0])
    elif case == "call_id":
        call["tool_call"]["id"] = "call_abc123"
    elif case == "result_id":
        messages[3]["content"][0]["tool_result"]["tool_call_id"] = "null"
    elif case == "missing_result":
        del messages[3]
    elif case == "system_after_tool":
        messages.insert(4, _msg("system", "s"))
    elif case == "tool_after_user":
        messages.insert(2, messages[3])
    elif case == "tool_alone":
        messages = [messages[3]]
    elif case == "arguments":
        call["tool_call"]["arguments"] = '{"city": "Paris"}'
    with pytest.raises(P.InvalidInput):
        P.mistral_instruct_texts(messages, tools)


def test_other_kinds_refuse_tools_and_pass_over_tool_parts(service):
    messages, tools = weather_example()
    for name in ("openai-chatml", "llama3-instruct"):
        tpl = P.CHAT_TEMPLATES[name]
        with pytest.raises(P.InvalidInput):
            service.count_chat_tokens(CTX, "mistral::mistral-nemo", messages, tpl, tools)
        bare = [dict(m, content=[p for p in m["content"] if p["type"] == "text"]) for m in messages]
        assert service.count_chat_tokens(CTX, "mistral::mistral-nemo", messages, tpl, []).input_tokens == \
            service.count_chat_tokens(CTX, "mistral::mistral-nemo", bare, tpl).input_tokens
