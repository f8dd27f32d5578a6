"""Special-token encode at its table's limits and on prompts dense with matches on the H100 (cfbpe_encode_batch_special and
cfbpe_encode_batch_special_device, sync and async), against special_sets.reference: the sets of special_sets.py on the cl100k
and Tekken slots under three policies, eight vocabularies in one batch, a ~100 MB batch with more than 2^22 kept matches, and
EBADMSG at the last byte of the last prompt and in the first of 65 536 prompts."""
import base64
import random

import numpy as np
import pytest

import special_sets as SS
from conftest import COMBOS, pack

pytestmark = pytest.mark.gpu

NAMES = {0: "cl100k_base", 1: "o200k_base", 2: "llama3", 3: "tekken"}


def load(ctx, slot, pat):
    from cfbpe import vocabs as V
    rv = V.resolve(NAMES[pat], allow_stand_in=True)
    ctx.vocab_load(slot, rv.file_bytes, rv.spec.fmt, rv.pattern_id, rv.max_ranks)


@pytest.fixture(scope="module")
def ctx():
    from cfbpe import _native as N
    c = N.Context(0, 64 << 20, 1 << 20)
    for slot, (pat, _, _) in enumerate(SS.EIGHT):
        load(c, slot, pat)
    yield c
    c.close()


@pytest.fixture(scope="module")
def encoders(tekken_bytes):
    tiktoken = pytest.importorskip("tiktoken")
    from oracle import patterns as PT
    lines = tekken_bytes.splitlines()
    out = {}
    for pat, n in COMBOS:
        ranks = {base64.b64decode(l.split()[0]): i for i, l in enumerate(lines[:n])}
        out[pat] = SS.ordinary(tiktoken.Encoding("plain%d" % pat, pat_str=PT.PATTERNS[pat], mergeable_ranks=ranks, special_tokens={}))
    return out


@pytest.fixture(scope="module")
def sets():
    return {name: SS.special_set(name) for name in SS.SETS}


def call_device(ctx, data, offs, vid, modes, sync):
    """cfbpe_encode_batch_special_device on device copies of the batch: (ids, offsets, counts)"""
    import torch
    total, n = int(offs[-1]), len(offs) - 1
    d_bytes = torch.zeros(total + 64, dtype=torch.uint8, device="cuda")
    d_bytes[:total] = torch.from_numpy(data)
    d_offs = torch.from_numpy(offs.view(np.int64)).cuda()
    d_vid = None if vid is None else torch.from_numpy(np.ascontiguousarray(vid, np.uint8)).cuda()
    d_ids = torch.zeros(total + 1, dtype=torch.int32, device="cuda")
    d_oo = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    d_cc = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    ctx.encode_batch_special_device(n, d_bytes.data_ptr(), total, d_offs.data_ptr(), None if d_vid is None else d_vid.data_ptr(),
                                    d_ids.data_ptr(), total + 1, d_oo.data_ptr(), d_cc.data_ptr(), modes=modes, stream=s, sync=sync)
    if not sync:
        ctx.device_status(s)
    torch.cuda.synchronize()
    oo = d_oo.cpu().numpy().view(np.uint64)
    return d_ids[:int(oo[-1])].cpu().numpy().view(np.uint32), oo, d_cc.cpu().numpy().view(np.uint32)[:n]


def check_all_paths(ctx, prompts, vid, modes, tables, encs):
    """host call, device call sync and async against the reference (EBADMSG with the reference's prompt and index)"""
    from cfbpe import _native as N
    want = SS.reference(tables, modes, prompts, vid, encs)
    data, offs = pack(prompts)
    if want[0] == "bad":
        with pytest.raises(N.NativeError) as ei:
            ctx.encode_batch_special(data, offs, vid, modes)
        assert ei.value.code == N.EBADMSG and ei.value.bad == want[1:]
        with pytest.raises(N.NativeError) as ei:
            call_device(ctx, data, offs, vid, modes, True)
        assert ei.value.code == N.EBADMSG and ei.value.bad == want[1:]
        return want
    wc = np.array([len(w) for w in want[1]], np.uint32)
    wo = np.cumsum(np.concatenate([[0], wc])).astype(np.uint64)
    wi = np.array([i for w in want[1] for i in w], np.uint32)
    for how in ("host", "sync", "async"):
        ids, o, c = ctx.encode_batch_special(data, offs, vid, modes) if how == "host" else call_device(ctx, data, offs, vid, modes, how == "sync")
        assert np.array_equal(o, wo), how
        assert np.array_equal(ids, wi), how
        if how != "async":
            assert np.array_equal(c, wc), how
    return want


@pytest.mark.parametrize("policy", SS.POLICIES)
@pytest.mark.parametrize("name", SS.SETS)
def test_set_on_the_h100(ctx, encoders, sets, name, policy):
    """the set registered on the cl100k (slot 0) and Tekken (slot 3) slots, prompts alternating between them"""
    specials, texts = sets[name]
    ctx.vocab_set_specials(0, specials)
    ctx.vocab_set_specials(3, specials)
    try:
        T = SS.Table(specials)
        m = SS.policy_modes(policy, len(specials))
        modes = None if m is None else [m, None, None, m]
        tables = [T, None, None, T]
        encs = [encoders[0], None, None, encoders[3]]
        prompts = [t.encode() for t in texts]
        vid = np.array([3 * (i & 1) for i in range(len(prompts))], np.uint8)
        want = check_all_paths(ctx, prompts, vid, modes, tables, encs)
        if policy != "allow_all":
            assert want[0] == "bad"
            prompts, vid = SS.without_bad(tables, modes, prompts, vid)
            want = check_all_paths(ctx, prompts, vid, modes, tables, encs)
        assert want[0] == "ok"
        if policy == "allow_all":
            assert sum(len(k) for k in want[2]) > len(prompts)
    finally:
        ctx.vocab_set_specials(0, {})
        ctx.vocab_set_specials(3, {})


def test_eight_vocabularies_with_their_own_sets(ctx, encoders, sets):
    for slot, (_, name, _) in enumerate(SS.EIGHT):
        ctx.vocab_set_specials(slot, sets[name][0] if name else {})
    try:
        prompts, vid = SS.eight_vocab_batch(sets, 9, 6000)
        modes, tables = SS.eight_vocab_modes(sets)
        encs = [encoders[pat] for pat, _, _ in SS.EIGHT]
        assert check_all_paths(ctx, prompts, vid, modes, tables, encs)[0] == "bad"
        prompts, vid = SS.without_bad(tables, modes, prompts, vid)
        want = check_all_paths(ctx, prompts, vid, modes, tables, encs)
        assert {int(vid[i]) for i, ks in enumerate(want[2]) if ks} == {0, 1, 2, 3, 4, 7}
    finally:
        for slot in range(8):
            ctx.vocab_set_specials(slot, {})


def test_large_dense_batch(sets, oracle_vocabs):
    """~100 MB, more than 2^22 kept matches: tile_scan over millions of stretches, the splice and the offsets at full size.
    The batch repeats a pool of distinct prompts (dense ones and plain text) in a shuffled order; the reference cuts each
    distinct prompt once and the multi-threaded oracle encodes the distinct text stretches"""
    from cfbpe import _native as N
    from cfbpe import workload as W
    from oracle import oracle as O
    specials, texts = sets["dense"]
    T = SS.Table(specials)
    allow = SS.policy_modes("allow_all", len(specials))
    tdata, toffs, _, _ = W.make_config(3, 0.05)
    plain = [bytes(tdata[int(toffs[i]):int(toffs[i + 1])]) for i in range(len(toffs) - 1)]
    pool = [t.encode() for t in texts] + plain
    cuts = [SS.cut(T, allow, p)[1] for p in pool]
    # the distinct text stretches, encoded by the oracle in one batch
    stretches = {}
    for p, kept in zip(pool, cuts):
        at = 0
        for a, b, _ in kept + [(len(p), len(p), None)]:
            stretches.setdefault(p[at:a], len(stretches))
            at = b
    sl = list(stretches)
    sd, so = pack(sl)
    sids, soffs, _ = O.encode_batch([oracle_vocabs[0]], [0], sd, so, nthreads=8)
    enc = {s: sids[int(soffs[j]):int(soffs[j + 1])] for j, s in enumerate(sl)}
    item_ids = []
    for p, kept in zip(pool, cuts):
        parts, at = [], 0
        for a, b, k in kept:
            parts += [enc[p[at:a]], np.array([T.ids[k]], np.uint32)]
            at = b
        item_ids.append(np.concatenate(parts + [enc[p[at:]]]).astype(np.uint32))
    rng = random.Random(3)
    n_dense = len(texts)
    order, size, n_kept = [], 0, 0
    while size < 100 << 20:
        j = rng.randrange(n_dense) if rng.random() < 0.6 else n_dense + rng.randrange(len(plain))
        order.append(j)
        size += len(pool[j])
        n_kept += len(cuts[j])
    assert n_kept > 1 << 22, n_kept
    data, offs = pack([pool[j] for j in order])
    want = [item_ids[j] for j in order]
    wc = np.array([len(w) for w in want], np.uint32)
    c = N.Context(0, 112 << 20, len(order) + 2 * n_kept + 1024)
    try:
        load(c, 0, 0)
        c.vocab_set_specials(0, specials)
        ids, o, cnt = c.encode_batch_special(data, offs, None, [allow])
        assert np.array_equal(cnt, wc)
        assert np.array_equal(o, np.cumsum(np.concatenate([[0], wc])).astype(np.uint64))
        assert np.array_equal(ids, np.concatenate(want))
    finally:
        c.close()


def test_ebadmsg_at_the_batch_edges(ctx, sets):
    """the DISALLOWED special at the last byte of the last of 65 536 prompts, and in the first of them"""
    from cfbpe import _native as N
    specials, _ = sets["all_lengths"]
    ctx.vocab_set_specials(0, specials)
    try:
        rng = random.Random(65536)
        clean = [("".join(rng.choice("qwxy .,") for _ in range(rng.randint(0, 40)))).encode() for _ in range(65536)]
        assert list(specials)[0] == "@"
        at = 0                                        # the index of the one-byte special "@"
        for prompts, where in ((clean[:-1] + [clean[-1] + b"@"], 65535), ([b"@" + clean[0]] + clean[1:-1] + [clean[-1] + b"@"], 0)):
            data, offs = pack(prompts)
            for how in ("host", "device"):
                with pytest.raises(N.NativeError) as ei:
                    if how == "host":
                        ctx.encode_batch_special(data, offs)
                    else:
                        call_device(ctx, data, offs, None, None, True)
                assert ei.value.code == N.EBADMSG and ei.value.bad == (where, at), how
    finally:
        ctx.vocab_set_specials(0, {})
