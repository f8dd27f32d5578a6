#!/usr/bin/env python3
"""What unit starts cost on the config-3 mix (a measurement aid, not a bench): the bytes held in device memory, the median of
STEPS warmed calls of each of cfbpe_encode_batch_device, cfbpe_encode_batch_starts_device and cfbpe_encode_batch_char_starts_device
(code points, UTF-16 units), the four alternated call by call in one run, timed with CUDA events.  Prints the card's name and
power limit with the numbers.  Seeded inputs only; the unit starts are checked against the host reference once."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "cyberfabric-core_b200")):
    sys.path.insert(0, p)
import numpy as np
import torch
from cfbpe import _native as N, plugin as P, workload as W

STEPS = int(os.environ.get("CHAR_STARTS_TIMES_STEPS", "20"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def timed(fns, steps):
    """call the functions in turn, `steps` rounds after 3 warm-up rounds; per call device time (events): median, [min, max]"""
    s = torch.cuda.current_stream()
    for _ in range(3):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(steps):
        for k, fn in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s); fn(); b.record(s)
            b.synchronize()
            ts[k].append(a.elapsed_time(b))
    return {k: {"median_ms": round(float(np.median(v)), 4), "range_ms": [round(min(v), 4), round(max(v), 4)]} for k, v in ts.items()}


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
    dl = torch.empty(n, dtype=torch.int32, device="cuda")
    args = (n, db.data_ptr(), total, do.data_ptr(), None)
    char = lambda unit: (lambda: c.encode_batch_char_starts_device(*args, unit, di.data_ptr(), ds.data_ptr(), total + 1, doo.data_ptr(),
                                                                   dc.data_ptr(), dl.data_ptr(), stream=st, sync=False))
    fns = {
        "encode_batch_device": lambda: c.encode_batch_device(*args, di.data_ptr(), total + 1, doo.data_ptr(), dc.data_ptr(), stream=st, sync=False),
        "encode_batch_starts_device": lambda: c.encode_batch_starts_device(*args, di.data_ptr(), ds.data_ptr(), total + 1, doo.data_ptr(),
                                                                           dc.data_ptr(), stream=st, sync=False),
        "char_starts_device_codepoint": char(N.UNIT_CODEPOINT),
        "char_starts_device_utf16": char(N.UNIT_UTF16),
    }
    res["times"] = timed(fns, STEPS)
    base = res["times"]["encode_batch_starts_device"]["median_ms"]
    for k in ("char_starts_device_codepoint", "char_starts_device_utf16"):
        res["times"][k]["over_byte_starts_ms"] = round(res["times"][k]["median_ms"] - base, 4)

    # the device results of the last call (UTF-16) against the host reference over the byte starts
    c.device_status(st)
    nt = int(doo[n].item())
    ids = di[:nt].cpu().numpy().view(np.uint32).copy()
    got, lens = ds[:nt].cpu().numpy().view(np.uint32).copy(), dl.cpu().numpy().view(np.uint32).copy()
    _, bst, off, _ = c.encode_batch_starts(data, offs)
    want, want_lens = P.unit_starts(data, offs, off, bst, "utf16")
    assert np.array_equal(ids, c.encode_batch(data, offs)[0])
    assert np.array_equal(got, want) and np.array_equal(lens, want_lens)
    res["ids"] = nt
    plug.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
