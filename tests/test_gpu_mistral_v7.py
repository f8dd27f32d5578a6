"""The "mistral-v7" chat template over the H100: the gateway service on GpuBpeTokenizerPlugin with the mistral_tekken vocabulary
counts every golden request as mistral_common's InstructTokenizerV7 does (tests/golden/mistral_v7.npz), in one device call a
request, and the V3 template still gives mistral_common's V3 counts of the same requests."""
import pytest

import mistral_v7_ref as R

pytestmark = pytest.mark.gpu

MODEL = "mistral::pixtral-large-2411"


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


def _check(gpu, requests, want, name, version):
    from cfbpe import plugin as P
    svc, calls = gpu
    ctx, tpl = P.SecurityContext.anonymous(), P.CHAT_TEMPLATES[name]
    for (conv, tools), w in zip(requests, want):
        before = len(calls)
        if w < 0:
            with pytest.raises(P.InvalidInput):
                svc.count_chat_tokens(ctx, MODEL, conv, tpl, tools)
            assert len(calls) == before                     # refused before any device work
            continue
        assert svc.count_chat_tokens(ctx, MODEL, conv, tpl, tools).input_tokens == w, (conv, tools)
        texts, _ = P.mistral_instruct_texts(conv, tools, version)
        stretches = sum(1 for t in texts if t)
        assert calls[before:] == ([stretches] if stretches else [])   # every stretch of the request in ONE device call


def test_v7_golden_requests(gpu):
    reqs, _, want = R.golden_counts()
    assert sum(w >= 0 for w in want) >= 900
    _check(gpu, reqs, want, "mistral-v7", 7)


def test_v3_counts_of_the_same_requests(gpu):
    reqs, want3, want7 = R.golden_counts()
    keep = [i for i, (c, _) in enumerate(reqs) if not R.uses_prefix(c)]     # (the V3 template does not read prefix)
    assert sum(0 <= want3[i] != want7[i] >= 0 for i in keep) >= 500
    _check(gpu, [reqs[i] for i in keep], [want3[i] for i in keep], "mistral-v3", 3)


def test_many_v7_requests_one_device_call_each(gpu):
    """requests counted back to back from several threads: each still makes exactly one device call holding all its stretches"""
    from concurrent.futures import ThreadPoolExecutor
    from cfbpe import plugin as P
    svc, calls = gpu
    reqs, _, want = R.golden_counts()
    ok = [(r, w) for r, w in zip(reqs, want) if w >= 0]
    ctx, tpl = P.SecurityContext.anonymous(), P.CHAT_TEMPLATES["mistral-v7"]
    before = len(calls)
    with ThreadPoolExecutor(8) as pool:
        got = list(pool.map(lambda rw: svc.count_chat_tokens(ctx, MODEL, rw[0][0], tpl, rw[0][1]).input_tokens, ok))
    assert got == [w for _, w in ok]
    stretches = sorted(sum(1 for t in P.mistral_instruct_texts(c, t, 7)[0] if t) for (c, t), _ in ok)
    assert sorted(calls[before:]) == [s for s in stretches if s]
