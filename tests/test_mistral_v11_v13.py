"""The "mistral-v11" and "mistral-v13" chat templates without a GPU: conversations counted as mistral_common's InstructTokenizerV11
and InstructTokenizerV13 count them (their golden counts, and live on fresh seeds when mistral_common imports), through the gateway
service over the C oracle; the refusals; the V7 counts of the same requests, unchanged; the template names."""
import json

import pytest

import mistral_ref as MR
import mistral_tools_ref as MTR
import mistral_v7_ref as R7
import mistral_v11_v13_ref as R
from cfbpe import plugin as P
from cfbpe import vocabs as V

CTX = P.SecurityContext.anonymous()
TEMPLATES = {7: P.CHAT_TEMPLATES["mistral-v7"], 11: P.CHAT_TEMPLATES["mistral-v11"], 13: P.CHAT_TEMPLATES["mistral-v13"]}
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


@pytest.fixture(scope="module")
def live():
    """version -> mistral_common's tokenizer of that version, or None when mistral_common does not import"""
    return {11: R.live_tokenizer(11), 13: R.live_tokenizer(13)}


def _count(service, conv, tools, version):
    """the gateway's count, -1 for InvalidInput"""
    try:
        return service.count_chat_tokens(CTX, MODEL, conv, TEMPLATES[version], tools).input_tokens
    except P.InvalidInput:
        return -1


def _msg(role, t):
    return {"role": role, "content": [{"type": "text", "text": t}]}


@pytest.mark.parametrize("version", R.VERSIONS)
def test_counts_as_mistral_common(service, version):
    reqs, _, want11, want13 = R.golden_counts()
    want = want11 if version == 11 else want13
    assert len(reqs) >= 1700 and sum(w >= 0 for w in want) >= 900 and sum(w < 0 for w in want) >= 500
    for (conv, tools), w in zip(reqs, want):
        assert _count(service, conv, tools, version) == w, (conv, tools)


def test_v7_counts_of_the_same_requests_do_not_move(service):
    """the V7 counts of the V7 golden requests are the V7 golden file's, and the V7 template still gives mistral_common's V7
    count of every request; V7, V11 and V13 differ pairwise on hundreds of them"""
    reqs, want7, want11, want13 = R.golden_counts()
    _, _, old7 = R7.golden_counts()
    assert want7[:len(old7)] == old7
    for (conv, tools), w in zip(reqs, want7):
        assert _count(service, conv, tools, 7) == w, (conv, tools)
    for a, b in ((want7, want11), (want7, want13), (want11, want13)):
        assert sum(0 <= x != y >= 0 for x, y in zip(a, b)) >= 300


def _is_json(text):
    try:
        json.loads(text)
        return True
    except json.JSONDecodeError:
        return False


def test_the_golden_requests_cover_what_v11_and_v13_change():
    reqs, _, want11, want13 = R.golden_counts()
    for want in (want11, want13):
        ok = [(c, t) for (c, t), w in zip(reqs, want) if w >= 0]
        turns = [[p["tool_call"] for p in m["content"] if p["type"] == "tool_call"] for c, _ in ok for m in c if m["role"] == "assistant"]
        results = [p["tool_result"]["content"] for c, _ in ok for m in c for p in m["content"] if p["type"] == "tool_result"]
        assert sum(len(t) >= 2 for t in turns) >= 100 and sum(len(t) >= 3 for t in turns) >= 30      # several calls a turn
        users = [sum(m["role"] == "user" for m in c) for c, t in ok if t]
        assert sum(u == 1 for u in users) >= 40 and sum(u >= 2 for u in users) >= 100                 # tools, one or more user turns
        assert sum(r == "" for r in results) >= 30 and sum(not r.isascii() for r in results) >= 30
        assert sum(map(_is_json, results)) >= 200 and sum(bool(r) and not _is_json(r) for r in results) >= 100
        assert sum(c[-1].get("prefix") is True for c, _ in ok) >= 50
    calls11 = [c["id"] for (conv, _), w in zip(reqs, want11) if w >= 0 for m in conv for p in m["content"] if p["type"] == "tool_call"
               for c in [p["tool_call"]]]
    assert calls11.count("null") >= 30 and len(calls11) - calls11.count("null") >= 500                # with and without ids
    assert sum(w11 >= 0 > w13 for w11, w13 in zip(want11, want13)) >= 30                             # "null" ids: V13 refuses


@pytest.mark.parametrize("version", R.VERSIONS)
def test_counts_live_on_fresh_seeds(service, live, version):
    tok = live[version]
    if tok is None:
        pytest.skip("mistral_common is not installed")
    reqs = R.v13_conversations(seed=4099, n=300) + R7.v7_conversations(seed=4111, n=150) + MTR.tool_conversations(seed=4127, n=150) \
        + [(c, []) for c in MR.conversations(seed=4133, n=50)]
    for conv, tools in reqs:
        assert _count(service, conv, tools, version) == R.mistral_count(tok, conv, tools), (conv, tools)


def weather_example():
    """(messages, tools): the weather conversation of the V7 tests, with two calls in the assistant turn"""
    tools = [{"type": "unified", "name": "get_weather", "description": "Weather of a city",
              "parameters": {"json_schema": {"type": "object", "properties": {"city": {"type": "string"}}, "required": ["city"]}}}]
    call = lambda cid, city: {"type": "tool_call", "tool_call": {"id": cid, "name": "get_weather", "arguments": {"city": city}}}
    result = lambda cid, content: {"role": "tool", "content": [{"type": "tool_result", "tool_result": {"tool_call_id": cid, "content": content}}]}
    messages = [_msg("system", "Be brief."), _msg("user", "Weather in Paris and Rome?"),
                {"role": "assistant", "content": [call("abc123XYZ", "Paris"), call("def456UVW", "Rome")]},
                result("def456UVW", '{"temp":24}'), result("abc123XYZ", '{"temp":21}'),
                _msg("assistant", "21 C and 24 C."), _msg("user", "And Oslo?")]
    return messages, tools


TOOLS_JSON = ('[{"type": "function", "function": {"name": "get_weather", "description": "Weather of a city", "parameters": '
              '{"type": "object", "properties": {"city": {"type": "string"}}, "required": ["city"]}}}]')


def test_weather_example_v11(service, live):
    """<s>[SYSTEM_PROMPT]Be brief.[/SYSTEM_PROMPT][INST]Weather in Paris and Rome?[/INST]
    [TOOL_CALLS]get_weather[CALL_ID]abc123XYZ[ARGS]{"city": "Paris"}[TOOL_CALLS]get_weather[CALL_ID]def456UVW[ARGS]{"city": "Rome"}</s>
    [TOOL_RESULTS]def456UVW[TOOL_CONTENT]{"temp": 24}[/TOOL_RESULTS][TOOL_RESULTS]abc123XYZ[TOOL_CONTENT]{"temp": 21}[/TOOL_RESULTS]
    21 C and 24 C.</s>[AVAILABLE_TOOLS][...][/AVAILABLE_TOOLS][INST]And Oslo?[/INST]"""
    messages, tools = weather_example()
    texts, n_ctl = P.mistral_instruct_texts_v11(messages, tools, 11)
    assert [t for t in texts if t] == [
        "Be brief.", "Weather in Paris and Rome?", "get_weather", "abc123XYZ", '{"city": "Paris"}', "get_weather", "def456UVW",
        '{"city": "Rome"}', "def456UVW", '{"temp": 24}', "abc123XYZ", '{"temp": 21}', "21 C and 24 C.", TOOLS_JSON, "And Oslo?"]
    assert n_ctl == 1 + 2 + 2 + 2 * 3 + 1 + 2 * 3 + 1 + 2 + 2 == 23
    assert service.count_chat_tokens(CTX, MODEL, messages, TEMPLATES[11], tools).input_tokens == 155
    if live[11] is not None:
        assert R.mistral_count(live[11], messages, tools) == 155


def test_weather_example_v13(service, live):
    """<s>[SYSTEM_PROMPT]Be brief.[/SYSTEM_PROMPT][AVAILABLE_TOOLS][...][/AVAILABLE_TOOLS][INST]Weather in Paris and Rome?[/INST]
    [TOOL_CALLS]get_weather[ARGS]{"city": "Paris"}[TOOL_CALLS]get_weather[ARGS]{"city": "Rome"}</s>
    [TOOL_RESULTS]{"temp": 21}[/TOOL_RESULTS][TOOL_RESULTS]{"temp": 24}[/TOOL_RESULTS]21 C and 24 C.</s>[INST]And Oslo?[/INST]
    (the results in the order of the calls, which does not change the count)"""
    messages, tools = weather_example()
    texts, n_ctl = P.mistral_instruct_texts_v11(messages, tools, 13)
    assert [t for t in texts if t] == [
        "Be brief.", TOOLS_JSON, "Weather in Paris and Rome?", "get_weather", '{"city": "Paris"}', "get_weather", '{"city": "Rome"}',
        '{"temp": 24}', '{"temp": 21}', "21 C and 24 C.", "And Oslo?"]
    assert n_ctl == 1 + 2 + 2 + 2 + 2 * 2 + 1 + 2 * 2 + 1 + 2 == 19
    assert service.count_chat_tokens(CTX, MODEL, messages, TEMPLATES[13], tools).input_tokens == 129
    if live[13] is not None:
        assert R.mistral_count(live[13], messages, tools) == 129


def test_calls_without_ids_and_results_by_version():
    """V11 prints a call's id only when it is not "null"; V13 refuses a "null" id.  A result's content is the JSON it parses to
    written again, else as given, "" is "{}"; V13 prints no call id and no [TOOL_CONTENT]"""
    conv = [_msg("user", "q"), {"role": "assistant", "content": [{"type": "tool_call", "tool_call": {"id": "null", "name": "f", "arguments": {}}}]},
            _msg("user", "r")]
    assert P.mistral_instruct_texts_v11(conv, version=11) == (["q", "", "f", "{}", "r"], 8)   # <s> [INST] [/INST] [TOOL_CALLS] [ARGS] </s> [INST] [/INST]
    with pytest.raises(P.InvalidInput):
        P.mistral_instruct_texts_v11(conv, version=13)

    def result(content, version):
        conv = [_msg("user", "q"), {"role": "assistant", "content": [{"type": "tool_call", "tool_call": {"id": "abc123XYZ", "name": "f", "arguments": {"x": 1}}}]},
                {"role": "tool", "content": [{"type": "tool_result", "tool_result": {"tool_call_id": "abc123XYZ", "content": content}}]}]
        return P.mistral_instruct_texts_v11(conv, version=version)
    assert result('{"a":1,\n "b" : [1.50, "\\u00e9"]}', 11) == (["q", "", "f", "abc123XYZ", '{"x": 1}', "abc123XYZ", '{"a": 1, "b": [1.5, "é"]}'], 10)
    assert result('{"a":1,\n "b" : [1.50, "\\u00e9"]}', 13) == (["q", "", "f", '{"x": 1}', '{"a": 1, "b": [1.5, "é"]}'], 8)
    assert result("not JSON: Zürich", 13)[0][-1] == "not JSON: Zürich"
    assert result("", 13)[0][-1] == "{}"


REFUSALS = ["null_call_id", "duplicate_call_id", "duplicate_result", "unknown_result_id", "missing_result", "result_after_text",
            "result_after_first_message", "system_after_tool", "prefix_not_last", "assistant_last", "empty_assistant", "call_id",
            "result_id", "name", "no_message", "version"]


@pytest.mark.parametrize("version", R.VERSIONS)
@pytest.mark.parametrize("case", REFUSALS)
def test_refusals(case, version, live):
    """each raises InvalidInput; where mistral_common has a form for the input, it refuses it too"""
    messages, tools = weather_example()
    calls = messages[2]["content"]
    if case == "null_call_id":
        if version == 11:
            pytest.skip("V11 takes a call without an id (it prints none)")
        messages = messages[:2] + [{"role": "assistant", "content": [dict(calls[0], tool_call=dict(calls[0]["tool_call"], id="null"))]},
                                   _msg("user", "and?")]
    elif case == "duplicate_call_id":
        calls[1]["tool_call"]["id"] = "abc123XYZ"
        messages[3]["content"][0]["tool_result"]["tool_call_id"] = "abc123XYZ"
        del messages[4]
    elif case == "duplicate_result":
        messages[3]["content"][0]["tool_result"]["tool_call_id"] = "abc123XYZ"
    elif case == "unknown_result_id":
        messages[3]["content"][0]["tool_result"]["tool_call_id"] = "zzz999ZZZ"
    elif case == "missing_result":
        del messages[3]
    elif case == "result_after_text":
        messages.insert(6, messages[4])
    elif case == "result_after_first_message":
        messages = messages[2:5]
    elif case == "system_after_tool":
        messages.insert(4, _msg("system", "s"))
    elif case == "prefix_not_last":
        messages[5]["prefix"] = True
    elif case == "assistant_last":
        messages.append(_msg("assistant", "x"))
    elif case == "empty_assistant":
        messages[5] = _msg("assistant", "")
    elif case == "call_id":
        calls[0]["tool_call"]["id"] = "call_abc123"
    elif case == "result_id":
        messages[3]["content"][0]["tool_result"]["tool_call_id"] = "null"
    elif case == "name":
        tools[0]["name"] = "get weather"
    elif case == "no_message":
        messages = []
    with pytest.raises(P.InvalidInput):
        P.mistral_instruct_texts_v11(messages, tools, 15 if case == "version" else version)
    if live[version] is not None and case != "version":
        assert R.mistral_count(live[version], messages, tools) == -1


def test_templates_and_models():
    assert TEMPLATES[11] == P.ChatTemplate("mistral", instruct_version=11)
    assert TEMPLATES[13] == P.ChatTemplate("mistral", instruct_version=13)
    assert P.ChatTemplate("mistral") == P.CHAT_TEMPLATES["mistral-v3"]
    for version in (3, 7, 8, 12, 15):
        with pytest.raises(P.InvalidInput):
            P.mistral_instruct_texts_v11([_msg("user", "q")], version=version)
    for version in (11, 13):                # mistral_instruct_texts keeps to V3 and V7
        with pytest.raises(P.InvalidInput):
            P.mistral_instruct_texts([_msg("user", "q")], version=version)
    with pytest.raises(P.InvalidInput):     # the template refuses a version it does not count
        P.LlmGatewayTokenizerService(P.ClientHub(), []).count_chat_tokens(CTX, MODEL, [_msg("user", "q")], P.ChatTemplate("mistral", instruct_version=15))
    # no model maps to V11 or V13: no model's instruct version is known to the repository; the templates are used by name
    assert not any(t.chat_template in ("mistral-v11", "mistral-v13") for t in V.MODEL_TOKENIZERS.values())
