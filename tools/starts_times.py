#!/usr/bin/env python3
"""What token starts cost on the config-3 mix (a measurement aid, not a bench), alternating the two calls on the same bytes:
  (a) device-resident: the median of STEPS calls of cfbpe_encode_batch_device against cfbpe_encode_batch_starts_device;
  (b) each kernel's time in one call of each (torch.profiler, a run of its own);
  (c) the host call from pinned buffers, cfbpe_encode_batch against cfbpe_encode_batch_starts (pipelined).
Seeded inputs only; the outputs of both calls are compared."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "cyberfabric-core_b200")):
    sys.path.insert(0, p)
import numpy as np
import torch
from cfbpe import plugin as P, workload as W

STEPS = int(os.environ.get("STARTS_TIMES_STEPS", "20"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def timed_pair(fa, fb, steps):
    """alternate fa and fb; per-call device time (events), median and [min, max] of each"""
    s = torch.cuda.current_stream()
    for _ in range(3):
        fa(); fb()
    torch.cuda.synchronize()
    ta, tb = [], []
    for _ in range(steps):
        for fn, ts in ((fa, ta), (fb, tb)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s); fn(); b.record(s)
            b.synchronize()
            ts.append(a.elapsed_time(b))
    r = lambda ts: (round(float(np.median(ts)), 4), [round(min(ts), 4), round(max(ts), 4)])
    return r(ta), r(tb)


def kernel_times(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kt = {}
    for ev in prof.key_averages():
        short = ev.key.split("(")[0].split("::")[-1].split("<")[0].replace("void ", "")
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if t:
            kt[short] = round(kt.get(short, 0) + t / 1e3, 4)
    return dict(sorted(kt.items(), key=lambda x: -x[1]))


def main():
    plug = P.GpuBpeTokenizerPlugin(device=0, vocab_names=("cl100k_base",), max_batch_bytes=160 << 20, max_prompts=1 << 20, allow_stand_in=True)
    c = plug.ctx
    st = torch.cuda.current_stream().cuda_stream
    data, offs, _, _ = W.make_config(3, 1.0)
    total, n = int(offs[-1]), len(offs) - 1
    res = {"gpu": gpu_info(), "steps": STEPS, "prompts": n, "bytes": total}

    db = torch.zeros(total + 64, dtype=torch.uint8, device="cuda"); db[:total] = torch.from_numpy(data)
    do = torch.from_numpy(offs.view(np.int64)).cuda()
    di = torch.empty(total + 1, dtype=torch.int32, device="cuda")
    ds = torch.empty(total + 1, dtype=torch.int32, device="cuda")
    doo = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    dc = torch.empty(n, dtype=torch.int32, device="cuda")
    plain = lambda: c.encode_batch_device(n, db.data_ptr(), total, do.data_ptr(), None, di.data_ptr(), total + 1, doo.data_ptr(), dc.data_ptr(),
                                          stream=st, sync=False)
    starts = lambda: c.encode_batch_starts_device(n, db.data_ptr(), total, do.data_ptr(), None, di.data_ptr(), ds.data_ptr(), total + 1,
                                                  doo.data_ptr(), dc.data_ptr(), stream=st, sync=False)
    (res["a_device_ms"], res["a_device_range"]), (res["a_device_starts_ms"], res["a_device_starts_range"]) = timed_pair(plain, starts, STEPS)

    # host calls from pinned buffers (the pipelined path), alternating, outputs compared
    pin_data = c.pinned(total, np.uint8); pin_data.array[:] = data
    pin_offs = c.pinned(n + 1, np.uint64); pin_offs.array[:] = offs
    o_ids = c.pinned(total + 1, np.uint32); o_st = c.pinned(total + 1, np.uint32)
    o_off = c.pinned(n + 1, np.uint64); o_cnt = c.pinned(n, np.uint32)
    hp = lambda: c.encode_batch(pin_data.array, pin_offs.array, None, o_ids.array, o_off.array, o_cnt.array)
    hs = lambda: c.encode_batch_starts(pin_data.array, pin_offs.array, None, o_ids.array, o_st.array, o_off.array, o_cnt.array)
    for _ in range(2):
        hp(); hs()
    ta, tb = [], []
    for _ in range(STEPS):
        for fn, ts in ((hp, ta), (hs, tb)):
            t0 = time.perf_counter(); fn(); ts.append((time.perf_counter() - t0) * 1e3)
    res["c_host_ms"], res["c_host_range"] = round(float(np.median(ta)), 3), [round(min(ta), 3), round(max(ta), 3)]
    res["c_host_starts_ms"], res["c_host_starts_range"] = round(float(np.median(tb)), 3), [round(min(tb), 3), round(max(tb), 3)]
    ids_h, st_h, off_h, _ = hs()
    ids_h, st_h = ids_h.copy(), st_h.copy()
    ids_p = hp()[0].copy()
    assert np.array_equal(ids_h, ids_p)
    nt = len(ids_h)
    assert np.array_equal(di[:nt].cpu().numpy().view(np.uint32), ids_h)
    assert np.array_equal(ds[:nt].cpu().numpy().view(np.uint32), st_h)
    res["ids"] = nt
    res["b_kernel_ms_plain"] = kernel_times(plain)
    res["b_kernel_ms_starts"] = kernel_times(starts)
    for a in (pin_data, pin_offs, o_ids, o_st, o_off, o_cnt):
        a.free()
    plug.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
