#!/usr/bin/env python3
"""What truncation to a token budget costs (a measurement aid, not a bench), the calls alternating on the same bytes:
  (a) device-resident, config-3 mix, budget 512: the median of STEPS calls of cfbpe_truncate_batch_device, of the count-only
      cfbpe_encode_batch_device and of cfbpe_encode_batch_starts_device (the device part of today's route);
  (b) each kernel's time in one truncate call (torch.profiler, a run of its own);
  (c) the host call from pinned buffers: cfbpe_truncate_batch, cfbpe_count_batch and today's route -- cfbpe_encode_batch_starts,
      then the cut on the host (cfbpe.plugin.truncate_cuts, timed on its own: it is a Python loop);
  (d) a skewed batch: one 64 MiB prompt among small ones, budget 512 and half the big prompt's count (the most ids to sum),
      device-resident truncate against count, and the truncate kernels' times.
Seeded inputs only; the results of the truncate calls are checked against the cut from the starts."""
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
from cfbpe import _native as N, plugin as P, workload as W

STEPS = int(os.environ.get("TRUNCATE_TIMES_STEPS", "20"))
BUDGET = 512


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def timed(fns, steps):
    """alternate the calls; per-call device time (events): median and [min, max] of each"""
    s = torch.cuda.current_stream()
    for _ in range(3):
        for fn in fns:
            fn()
    torch.cuda.synchronize()
    ts = [[] for _ in fns]
    for _ in range(steps):
        for fn, t in zip(fns, ts):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s); fn(); b.record(s)
            b.synchronize()
            t.append(a.elapsed_time(b))
    return [(round(float(np.median(t)), 4), [round(min(t), 4), round(max(t), 4)]) for t in ts]


def host_timed(fns, steps):
    for _ in range(2):
        for fn in fns:
            fn()
    ts = [[] for _ in fns]
    for _ in range(steps):
        for fn, t in zip(fns, ts):
            t0 = time.perf_counter(); fn(); t.append((time.perf_counter() - t0) * 1e3)
    return [(round(float(np.median(t)), 3), [round(min(t), 3), round(max(t), 3)]) for t in ts]


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


class DeviceBatch:
    """a batch, its budgets and every output on the device; the three calls as closures"""

    def __init__(self, c, data, offs, budgets):
        self.c, self.n, self.total = c, len(offs) - 1, int(offs[-1])
        self.st = torch.cuda.current_stream().cuda_stream
        self.db = torch.zeros(self.total + 64, dtype=torch.uint8, device="cuda"); self.db[:self.total] = torch.from_numpy(data[:self.total])
        self.do = torch.from_numpy(offs.view(np.int64)).cuda()
        self.dbud = torch.from_numpy(budgets.view(np.int32)).cuda()
        self.di = torch.empty(self.total + 1, dtype=torch.int32, device="cuda")
        self.ds = torch.empty(self.total + 1, dtype=torch.int32, device="cuda")
        self.doo = torch.empty(self.n + 1, dtype=torch.int64, device="cuda")
        self.dc = torch.empty(self.n, dtype=torch.int32, device="cuda")
        self.dcut = torch.empty(self.n, dtype=torch.int32, device="cuda")
        self.dkept = torch.empty(self.n, dtype=torch.int32, device="cuda")

    def truncate(self, mode=N.TRUNCATE_HEAD):
        return lambda: self.c.truncate_batch_device(self.n, self.db.data_ptr(), self.total, self.do.data_ptr(), None, self.dbud.data_ptr(), mode,
                                                    self.dcut.data_ptr(), self.dkept.data_ptr(), self.dc.data_ptr(), self.st)

    def count(self):
        return lambda: self.c.encode_batch_device(self.n, self.db.data_ptr(), self.total, self.do.data_ptr(), None, None, 0, self.doo.data_ptr(),
                                                  self.dc.data_ptr(), stream=self.st, sync=False)

    def starts(self):
        return lambda: self.c.encode_batch_starts_device(self.n, self.db.data_ptr(), self.total, self.do.data_ptr(), None, self.di.data_ptr(),
                                                         self.ds.data_ptr(), self.total + 1, self.doo.data_ptr(), self.dc.data_ptr(),
                                                         stream=self.st, sync=False)

    def cuts(self):
        torch.cuda.synchronize()
        return self.dcut.cpu().numpy().view(np.uint32).copy(), self.dkept.cpu().numpy().view(np.uint32).copy()


def check(c, data, offs, budgets, got, mode=N.TRUNCATE_HEAD):
    _, st, off, _ = c.encode_batch_starts(data, offs)
    want = P.truncate_cuts(data, offs, off, st, budgets, mode == N.TRUNCATE_TAIL)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def skewed_batch(data, offs):
    """one 64 MiB prompt (config-3 text, cut at a character start) among the config-3 prompts of the next ~60 MB"""
    big = 64 << 20
    while data[big] & 0xC0 == 0x80:
        big -= 1
    p1 = int(np.searchsorted(offs, big + (60 << 20)))
    small = offs[int(np.searchsorted(offs, big)):p1]
    small = small - small[0]
    sdata = data[int(offs[int(np.searchsorted(offs, big))]):][:int(small[-1])]
    d = np.concatenate([data[:big], sdata])
    o = np.concatenate([[0], big + small]).astype(np.uint64)
    return d, o


def main():
    plug = P.GpuBpeTokenizerPlugin(device=0, vocab_names=("cl100k_base",), max_batch_bytes=160 << 20, max_prompts=1 << 20, allow_stand_in=True)
    c = plug.ctx
    data, offs, _, _ = W.make_config(3, 1.0)
    total, n = int(offs[-1]), len(offs) - 1
    counts = c.count_batch(data, offs).copy()
    budgets = np.full(n, BUDGET, dtype=np.uint32)
    res = {"gpu": gpu_info(), "steps": STEPS, "prompts": n, "bytes": total, "ids": int(counts.sum()), "budget": BUDGET,
           "prompts_cut": int((counts > BUDGET).sum())}

    # (a) device-resident
    dv = DeviceBatch(c, data, offs, budgets)
    (tr, tr_r), (cn, cn_r), (sr, sr_r) = timed([dv.truncate(), dv.count(), dv.starts()], STEPS)
    res.update(a_device_truncate_ms=tr, a_device_truncate_range=tr_r, a_device_count_ms=cn, a_device_count_range=cn_r,
               a_device_starts_ms=sr, a_device_starts_range=sr_r)
    dv.truncate()()
    got = dv.cuts()
    check(c, data, offs, budgets, got)
    # (b) the truncate call's kernels
    res["b_kernel_ms_truncate"] = kernel_times(dv.truncate())
    del dv

    # (c) host calls from pinned buffers, alternating
    pin_data = c.pinned(total, np.uint8); pin_data.array[:] = data
    pin_offs = c.pinned(n + 1, np.uint64); pin_offs.array[:] = offs
    o_ids = c.pinned(total + 1, np.uint32); o_st = c.pinned(total + 1, np.uint32)
    o_off = c.pinned(n + 1, np.uint64); o_cnt = c.pinned(n, np.uint32)
    o_cut = c.pinned(n, np.uint32); o_kept = c.pinned(n, np.uint32)
    ht = lambda: c.truncate_batch(pin_data.array, pin_offs.array, budgets, N.TRUNCATE_HEAD, None, o_cut.array, o_kept.array, o_cnt.array)
    hc = lambda: c.count_batch(pin_data.array, pin_offs.array, None, o_cnt.array)
    hs = lambda: c.encode_batch_starts(pin_data.array, pin_offs.array, None, o_ids.array, o_st.array, o_off.array, o_cnt.array)
    (tr, tr_r), (cn, cn_r), (sr, sr_r) = host_timed([ht, hc, hs], STEPS)
    res.update(c_host_truncate_ms=tr, c_host_truncate_range=tr_r, c_host_count_ms=cn, c_host_count_range=cn_r,
               c_host_starts_ms=sr, c_host_starts_range=sr_r)
    _, st, off, _ = hs()
    t0 = time.perf_counter()
    want = P.truncate_cuts(data, offs, off, st, budgets, False)
    res["c_host_cut_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    ht()
    assert np.array_equal(o_cut.array, want[0]) and np.array_equal(o_kept.array, want[1])
    for a in (pin_data, pin_offs, o_ids, o_st, o_off, o_cnt, o_cut, o_kept):
        a.free()

    # (d) the skewed batch
    sd, so = skewed_batch(data, offs)
    scounts = c.count_batch(sd, so).copy()
    res["d_skewed"] = {"prompts": len(so) - 1, "bytes": int(so[-1]), "big_prompt_bytes": int(so[1]), "big_prompt_ids": int(scounts[0])}
    for name, big_budget in (("budget_512", BUDGET), ("budget_half", int(scounts[0]) // 2)):
        sb = np.full(len(so) - 1, BUDGET, dtype=np.uint32)
        sb[0] = big_budget
        dv = DeviceBatch(c, sd, so, sb)
        (tr, tr_r), (cn, cn_r) = timed([dv.truncate(), dv.count()], STEPS)
        dv.truncate()()
        check(c, sd, so, sb, dv.cuts())
        res["d_skewed"][name] = {"truncate_ms": tr, "truncate_range": tr_r, "count_ms": cn, "count_range": cn_r,
                                 "kernel_ms": {k: v for k, v in kernel_times(dv.truncate()).items() if "truncate" in k}}
        del dv
    plug.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
