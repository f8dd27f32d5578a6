#!/usr/bin/env python3
"""Device-resident time per call of encode with special tokens on the config-3 mix (a measurement aid, not a bench):
  (a) tiktoken's default policy (every special disallowed) on clean text -- scan + the ordinary path -- against
      cfbpe_encode_batch_device on the same bytes;
  (b) Llama-3-template-rendered prompts with about 5 allowed specials a prompt (cfbpe_encode_batch_special_device);
  (c) the same input as (b) end to end through the plugin trait's default (host cut + one encode_batch call);
  plus each kernel's time in one call of (b) (torch.profiler).  Seeded inputs only."""
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "cyberfabric-core_b200")):
    sys.path.insert(0, p)
import numpy as np
import torch
from cfbpe import plugin as P, workload as W

STEPS = int(os.environ.get("SPECIAL_TIMES_STEPS", "20"))
TPL = P.CHAT_TEMPLATES["llama3-instruct"]
SPECIALS = {t: 128000 + i for i, t in enumerate(TPL.special_tokens)}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def rendered(data, offs, seed):
    """each prompt as one Llama 3 turn and a generation prompt: 5 control tokens a prompt, its text as the message content"""
    rng = random.Random(seed)
    roles = ["system", "user", "assistant"]
    out = []
    for i in range(len(offs) - 1):
        t = bytes(data[int(offs[i]):int(offs[i + 1])]).decode("utf-8")
        out.append(TPL.bos + TPL.message_prefix.format(role=rng.choice(roles)) + t + TPL.message_suffix + TPL.generation_prompt)
    return P.pack_texts(out)


def timed(fn, steps):
    s = torch.cuda.current_stream()
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s); fn(); b.record(s)
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return round(float(np.median(ts)), 4), [round(min(ts), 4), round(max(ts), 4)]


def main():
    plug = P.GpuBpeTokenizerPlugin(device=0, vocab_names=("cl100k_base",), max_batch_bytes=160 << 20, max_prompts=1 << 20, allow_stand_in=True)
    c = plug.ctx
    c.vocab_set_specials(0, SPECIALS)
    plug._specials[0] = dict(SPECIALS)
    st = torch.cuda.current_stream().cuda_stream
    data, offs, _, _ = W.make_config(3, 1.0)
    rdata, roffs = rendered(data, offs, 3)
    res = {"gpu": gpu_info(), "steps": STEPS, "prompts": len(offs) - 1}

    def device_bufs(d, o):
        total, n = int(o[-1]), len(o) - 1
        db = torch.zeros(total + 64, dtype=torch.uint8, device="cuda"); db[:total] = torch.from_numpy(d)
        do = torch.from_numpy(o.view(np.int64)).cuda()
        return (n, db, total, do, torch.empty(total + 1, dtype=torch.int32, device="cuda"),
                torch.empty(n + 1, dtype=torch.int64, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda"))

    n, db, total, do, di, doo, dc = device_bufs(data, offs)
    plain = lambda: c.encode_batch_device(n, db.data_ptr(), total, do.data_ptr(), None, di.data_ptr(), total + 1, doo.data_ptr(), dc.data_ptr(), stream=st, sync=False)
    default = lambda: c.encode_batch_special_device(n, db.data_ptr(), total, do.data_ptr(), None, di.data_ptr(), total + 1, doo.data_ptr(), dc.data_ptr(),
                                                    modes=None, stream=st, sync=False)
    res["bytes_a"] = total
    res["a_encode_batch_device_ms"], res["a_encode_batch_device_range"] = timed(plain, STEPS)
    res["a_default_policy_ms"], res["a_default_policy_range"] = timed(default, STEPS)

    n2, db2, total2, do2, di2, doo2, dc2 = device_bufs(rdata, roffs)
    allow = np.ones(len(SPECIALS), np.uint8)
    special = lambda: c.encode_batch_special_device(n2, db2.data_ptr(), total2, do2.data_ptr(), None, di2.data_ptr(), total2 + 1, doo2.data_ptr(),
                                                    dc2.data_ptr(), modes=[allow], stream=st, sync=False)
    res["bytes_b"] = total2
    res["b_llama3_rendered_ms"], res["b_llama3_rendered_range"] = timed(special, STEPS)
    nt = c.encode_batch_special_device(n2, db2.data_ptr(), total2, do2.data_ptr(), None, di2.data_ptr(), total2 + 1, doo2.data_ptr(), dc2.data_ptr(),
                                       modes=[allow], stream=st)
    res["b_ids"] = int(nt)

    ctx = P.SecurityContext.anonymous()
    req = P.EncodeBatchRequest(P.VocabRef("cl100k_base"), rdata, roffs)
    ts = []
    for _ in range(3):
        t0 = time.perf_counter()
        want = P.TokenizerPluginClient.encode_batch_special(plug, ctx, req, SPECIALS, set(SPECIALS), set())
        ts.append((time.perf_counter() - t0) * 1e3)
    res["c_host_cut_e2e_ms"] = round(min(ts), 1)
    t0 = time.perf_counter()
    got = plug.encode_batch_special(ctx, req, SPECIALS, set(SPECIALS), set())
    res["b_plugin_e2e_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    assert np.array_equal(got.ids, want.ids) and np.array_equal(got.offsets, want.offsets)
    assert np.array_equal(di2[:nt].cpu().numpy().view(np.uint32), want.ids)

    from torch.profiler import ProfilerActivity, profile
    special()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        special()
        torch.cuda.synchronize()
    kt = {}
    for ev in prof.key_averages():
        name = ev.key
        short = name.split("(")[0].split("::")[-1].split("<")[0].replace("void ", "")
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if t:
            kt[short] = round(kt.get(short, 0) + t / 1e3, 4)
    res["b_kernel_ms"] = dict(sorted(kt.items(), key=lambda x: -x[1]))
    plug.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
