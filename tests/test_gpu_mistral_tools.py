"""The "mistral" chat template on tool use over the H100: the gateway service on GpuBpeTokenizerPlugin with the mistral_tekken
vocabulary counts every tool conversation as mistral_common's encode_chat_completion does (live when it imports, else its golden
counts), in one device call a request, and counts the text-only conversations without tools as before."""
import pytest

import mistral_ref as MR
import mistral_tools_ref as MTR

pytestmark = pytest.mark.gpu

MODEL = "mistral::mistral-nemo"


@pytest.fixture(scope="module")
def gpu():
    """(service, the plugin's count_tokens calls so far: the number of stretches of each)"""
    from cfbpe import plugin as P
    plug = P.GpuBpeTokenizerPlugin(device=0, vocab_names=("mistral_tekken",), max_batch_bytes=8 << 20, max_prompts=1 << 12)
    calls = []
    device_count = plug.count_tokens

    def count_tokens(ctx, req, *args, **kwargs):
        calls.append(len(req.offsets) - 1)
        return device_count(ctx, req, *args, **kwargs)
    plug.count_tokens = count_tokens
    hub = P.ClientHub()
    hub.register_scoped(P.TokenizerPluginClient, plug.instance.id, plug)
    yield P.LlmGatewayTokenizerService(hub, [plug.instance]), calls
    plug.close()


def _check(gpu, requests, want):
    from cfbpe import plugin as P
    svc, calls = gpu
    ctx, tpl = P.SecurityContext.anonymous(), P.CHAT_TEMPLATES["mistral-v3"]
    for (conv, tools), w in zip(requests, want):
        before = len(calls)
        if w < 0:
            with pytest.raises(P.InvalidInput):
                svc.count_chat_tokens(ctx, MODEL, conv, tpl, tools)
            assert len(calls) == before                     # refused before any device work
            continue
        assert svc.count_chat_tokens(ctx, MODEL, conv, tpl, tools).input_tokens == w, (conv, tools)
        texts, _ = P.mistral_instruct_texts(conv, tools)
        stretches = sum(1 for t in texts if t)
        assert calls[before:] == ([stretches] if stretches else [])   # every stretch of the request in ONE device call


def test_tool_conversations(gpu):
    convs, want = MTR.tool_counts()
    assert sum(w >= 0 for w in want) >= 300
    _check(gpu, convs, want)


def test_text_only_conversations_without_tools(gpu):
    convs = MR.conversations()
    mt = MR.live_tokenizer()
    if mt is not None:
        want = [MR.mistral_count(mt, c) for c in convs]
    else:
        g = MR.golden()
        assert bytes(g["conversations"]).decode("utf-8") == MR.conversations_json(convs)
        want = g["conversation_counts"].tolist()
    _check(gpu, [(c, None) for c in convs], want)
