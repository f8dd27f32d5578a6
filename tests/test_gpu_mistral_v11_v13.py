"""The "mistral-v11" and "mistral-v13" chat templates over the H100: the gateway service on GpuBpeTokenizerPlugin with the
mistral_tekken vocabulary counts every golden request as mistral_common's InstructTokenizerV11 and V13 do
(tests/golden/mistral_v11_v13.npz), in one device call a request, also from several threads at once."""
import pytest

import mistral_v11_v13_ref as R

pytestmark = pytest.mark.gpu

MODEL = "mistral::mistral-small-2503"


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


def _stretches(conv, tools, version):
    from cfbpe import plugin as P
    return sum(1 for t in P.mistral_instruct_texts_v11(conv, tools, version)[0] if t)


@pytest.mark.parametrize("version", R.VERSIONS)
def test_golden_requests(gpu, version):
    from cfbpe import plugin as P
    svc, calls = gpu
    reqs, _, want11, want13 = R.golden_counts()
    want = want11 if version == 11 else want13
    assert sum(w >= 0 for w in want) >= 900
    ctx, tpl = P.SecurityContext.anonymous(), P.CHAT_TEMPLATES["mistral-v%d" % version]
    for (conv, tools), w in zip(reqs, want):
        before = len(calls)
        if w < 0:
            with pytest.raises(P.InvalidInput):
                svc.count_chat_tokens(ctx, MODEL, conv, tpl, tools)
            assert len(calls) == before                     # refused before any device work
            continue
        assert svc.count_chat_tokens(ctx, MODEL, conv, tpl, tools).input_tokens == w, (conv, tools)
        n = _stretches(conv, tools, version)
        assert calls[before:] == ([n] if n else [])         # every stretch of the request in ONE device call


@pytest.mark.parametrize("version", R.VERSIONS)
def test_many_requests_one_device_call_each(gpu, version):
    """requests counted back to back from several threads: each still makes exactly one device call holding all its stretches"""
    from concurrent.futures import ThreadPoolExecutor
    from cfbpe import plugin as P
    svc, calls = gpu
    reqs, _, want11, want13 = R.golden_counts()
    ok = [(r, w) for r, w in zip(reqs, want11 if version == 11 else want13) if w >= 0]
    ctx, tpl = P.SecurityContext.anonymous(), P.CHAT_TEMPLATES["mistral-v%d" % version]
    before = len(calls)
    with ThreadPoolExecutor(8) as pool:
        got = list(pool.map(lambda rw: svc.count_chat_tokens(ctx, MODEL, rw[0][0], tpl, rw[0][1]).input_tokens, ok))
    assert got == [w for _, w in ok]
    stretches = sorted(_stretches(c, t, version) for (c, t), _ in ok)
    assert sorted(calls[before:]) == [s for s in stretches if s]
