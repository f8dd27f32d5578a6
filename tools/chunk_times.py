#!/usr/bin/env python3
"""What chunking costs (a measurement aid, not a bench), the calls alternating on the same bytes: config-3 mix, chunks of 512
tokens with no overlap and with 64 tokens of overlap.
  (a) device-resident: the median of STEPS calls of cfbpe_chunk_batch_device (both overlaps), of the count-only
      cfbpe_encode_batch_device and of cfbpe_encode_batch_starts_device (the device part of today's route);
  (b) each kernel's time in one chunk call (torch.profiler, a run of its own);
  (c) the host call from pinned buffers: cfbpe_chunk_batch (both overlaps), cfbpe_truncate_batch (budget 512), cfbpe_count_batch and
      cfbpe_encode_batch_starts (today's route, before the host cuts anything).
Prints the card, its power limit and max SM clock.  Seeded inputs only; the chunks are checked against the ones cut on the host
from the starts (cfbpe.plugin.chunk_spans)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "cyberfabric-core_b200"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import numpy as np
import torch
from cfbpe import _native as N, plugin as P, workload as W
from truncate_times import DeviceBatch, gpu_info, host_timed, kernel_times, timed

STEPS = int(os.environ.get("CHUNK_TIMES_STEPS", "20"))
CHUNK, OVERLAPS = 512, (0, 64)


class DeviceChunks(DeviceBatch):
    """DeviceBatch with room for the chunks"""

    def __init__(self, c, data, offs):
        super().__init__(c, data, offs, np.zeros(len(offs) - 1, np.uint32))
        self.cap = N.Context.chunk_bound(offs, CHUNK, 0)
        self.dsp = torch.empty((self.cap, 2), dtype=torch.int32, device="cuda")
        self.dco = torch.empty(self.n + 1, dtype=torch.int64, device="cuda")

    def chunk(self, overlap):
        return lambda: self.c.chunk_batch_device(self.n, self.db.data_ptr(), self.total, self.do.data_ptr(), None, CHUNK, overlap,
                                                 self.dsp.data_ptr(), self.cap, self.dco.data_ptr(), self.dc.data_ptr(), self.st, False)

    def chunks(self):
        torch.cuda.synchronize()
        co = self.dco.cpu().numpy().view(np.uint64).copy()
        return self.dsp[:int(co[-1])].cpu().numpy().view(np.uint32).copy(), co


def main():
    plug = P.GpuBpeTokenizerPlugin(device=0, vocab_names=("cl100k_base",), max_batch_bytes=160 << 20, max_prompts=1 << 20, allow_stand_in=True)
    c = plug.ctx
    data, offs, _, _ = W.make_config(3, 1.0)
    total, n = int(offs[-1]), len(offs) - 1
    counts = c.count_batch(data, offs).copy()
    _, st, off, _ = c.encode_batch_starts(data, offs)
    want = {s: P.chunk_spans(data, offs, off, st, CHUNK, s) for s in OVERLAPS}
    res = {"gpu": gpu_info(), "steps": STEPS, "prompts": n, "bytes": total, "ids": int(counts.sum()), "chunk_tokens": CHUNK,
           "chunks": {str(s): int(want[s][1][-1]) for s in OVERLAPS}}

    # (a) device-resident
    dv = DeviceChunks(c, data, offs)
    r = timed([dv.chunk(0), dv.chunk(64), dv.count(), dv.starts()], STEPS)
    for name, (med, rng) in zip(("chunk_s0", "chunk_s64", "count", "starts"), r):
        res["a_device_%s_ms" % name], res["a_device_%s_range" % name] = med, rng
    for s in OVERLAPS:
        dv.chunk(s)()
        sp, co = dv.chunks()
        assert np.array_equal(sp, want[s][0]) and np.array_equal(co, want[s][1]), s
    # (b) the chunk call's kernels
    res["b_kernel_ms_chunk_s64"] = kernel_times(dv.chunk(64))
    del dv

    # (c) host calls from pinned buffers, alternating
    pin_data = c.pinned(total, np.uint8); pin_data.array[:] = data
    pin_offs = c.pinned(n + 1, np.uint64); pin_offs.array[:] = offs
    o_ids = c.pinned(total + 1, np.uint32); o_st = c.pinned(total + 1, np.uint32)
    o_off = c.pinned(n + 1, np.uint64); o_cnt = c.pinned(n, np.uint32)
    o_cut = c.pinned(n, np.uint32); o_kept = c.pinned(n, np.uint32)
    budgets = np.full(n, CHUNK, dtype=np.uint32)
    got = {}

    def hchunk(s):
        def f():
            got[s] = c.chunk_batch(pin_data.array, pin_offs.array, CHUNK, s, None, o_cnt.array)
        return f
    ht = lambda: c.truncate_batch(pin_data.array, pin_offs.array, budgets, N.TRUNCATE_HEAD, None, o_cut.array, o_kept.array, o_cnt.array)
    hc = lambda: c.count_batch(pin_data.array, pin_offs.array, None, o_cnt.array)
    hs = lambda: c.encode_batch_starts(pin_data.array, pin_offs.array, None, o_ids.array, o_st.array, o_off.array, o_cnt.array)
    r = host_timed([hchunk(0), hchunk(64), ht, hc, hs], STEPS)
    for name, (med, rng) in zip(("chunk_s0", "chunk_s64", "truncate", "count", "starts"), r):
        res["c_host_%s_ms" % name], res["c_host_%s_range" % name] = med, rng
    for s in OVERLAPS:
        assert np.array_equal(got[s][0], want[s][0]) and np.array_equal(got[s][1], want[s][1]), s
    for a in (pin_data, pin_offs, o_ids, o_st, o_off, o_cnt, o_cut, o_kept):
        a.free()
    plug.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
