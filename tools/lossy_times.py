#!/usr/bin/env python3
"""What encoding bytes that are not valid UTF-8 costs on the config-3 mix (a measurement aid, not a bench).  Timed with CUDA
events, the median of STEPS warmed calls, the calls of each pair alternated call by call in one run:
  device_clean     cfbpe_encode_batch_lossy_device against cfbpe_encode_batch_device on the same valid bytes in device memory
  device_strays_1  a stray byte (FF) in the middle of 1 % of the prompts: the lossy call on them against cfbpe_encode_batch_device
                   on the bytes CPython's decode("utf-8", "replace") makes of them
  device_strays_all  the same with a stray in every prompt
  host_clean, host_strays_1  the host calls from pinned buffers: cfbpe_encode_batch_lossy against cfbpe_encode_batch (valid bytes;
                   the repaired bytes)
Prints the card's name and power limit with the numbers; checks every lossy result against its strict counterpart once.
--rehearse builds the inputs and checks the repair counts on the host, without a GPU."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "cyberfabric-core_b200")):
    sys.path.insert(0, p)
import numpy as np
from cfbpe import workload as W

STEPS = int(os.environ.get("LOSSY_TIMES_STEPS", "20"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def with_strays(data, offs, every):
    """a stray FF near the middle of every `every`-th prompt: (bytes, offsets), and CPython's repair of them: (bytes, offsets)"""
    raw = data.tobytes()
    n = len(offs) - 1
    prompts = [raw[int(offs[i]):int(offs[i + 1])] for i in range(n)]
    for i in range(0, n, every):
        h = len(prompts[i]) // 2
        while 0 < h < len(prompts[i]) and prompts[i][h] & 0xC0 == 0x80:      # (at a character boundary: one U+FFFD a stray)
            h -= 1
        prompts[i] = prompts[i][:h] + b"\xff" + prompts[i][h:]

    def pack(ps):
        o = np.zeros(len(ps) + 1, dtype=np.uint64)
        o[1:] = np.cumsum([len(p) for p in ps], dtype=np.uint64)
        return np.frombuffer(b"".join(ps), dtype=np.uint8).copy(), o
    return pack(prompts), pack([p.decode("utf-8", "replace").encode("utf-8") for p in prompts])


def timed(fns, steps):
    """call the functions in turn, `steps` rounds after 3 warm-up rounds; per call device time (events): median, [min, max]"""
    import torch
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
    data, offs, _, _ = W.make_config(3, 1.0)
    total, n = int(offs[-1]), len(offs) - 1
    cases = {"clean": ((data, offs), (data, offs)), "strays_1": with_strays(data, offs, 100), "strays_all": with_strays(data, offs, 1)}
    res = {"steps": STEPS, "prompts": n, "bytes": {k: int(v[0][1][-1]) for k, v in cases.items()}}
    if "--rehearse" in sys.argv[1:]:
        for k, ((d, o), (rd, ro)) in cases.items():
            assert int(ro[-1]) - int(o[-1]) == {"clean": 0, "strays_1": 2 * ((n + 99) // 100), "strays_all": 2 * n}[k], k
        res["rehearsal"] = "inputs built, repaired sizes checked"
        print(json.dumps(res))
        return

    import torch
    from cfbpe import _native as N, plugin as P
    res["gpu"] = gpu_info()
    plug = P.GpuBpeTokenizerPlugin(device=0, vocab_names=("cl100k_base",), max_batch_bytes=160 << 20, max_prompts=1 << 20, allow_stand_in=True)
    c = plug.ctx
    st = torch.cuda.current_stream().cuda_stream
    cap = 160 << 20
    di = torch.empty(cap, dtype=torch.int32, device="cuda")
    doo = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    dc = torch.empty(n, dtype=torch.int32, device="cuda")
    dr = torch.empty(n, dtype=torch.int32, device="cuda")

    def on_device(d, o):
        t = int(o[-1])
        db = torch.zeros(t + 64, dtype=torch.uint8, device="cuda"); db[:t] = torch.from_numpy(d[:t])
        return db, torch.from_numpy(o.view(np.int64)).cuda(), t

    times = {}
    for k, ((d, o), (rd, ro)) in cases.items():
        raw, rep = on_device(d, o), on_device(rd, ro)
        lossy = lambda: c.encode_batch_lossy_device(n, raw[0].data_ptr(), raw[2], raw[1].data_ptr(), None, di.data_ptr(), cap, doo.data_ptr(),
                                                    dc.data_ptr(), dr.data_ptr(), stream=st, sync=False)
        strict = lambda: c.encode_batch_device(n, rep[0].data_ptr(), rep[2], rep[1].data_ptr(), None, di.data_ptr(), cap, doo.data_ptr(),
                                               dc.data_ptr(), stream=st, sync=False)
        t = timed({"lossy": lossy, "strict_on_repaired": strict}, STEPS)
        t["lossy"]["over_strict_ms"] = round(t["lossy"]["median_ms"] - t["strict_on_repaired"]["median_ms"], 4)
        times["device_" + k] = t
        lossy(); c.device_status(st)                          # the last lossy result against the strict call on the repaired bytes
        nt = int(doo[n].item())
        ids = di[:nt].cpu().numpy().view(np.uint32).copy()
        want_ids, want_off, _ = c.encode_batch(rd, ro)
        assert np.array_equal(ids, want_ids) and np.array_equal(doo.cpu().numpy().view(np.uint64), want_off), k
        assert int(dr.cpu().numpy().astype(np.int64).sum()) == (int(ro[-1]) - int(o[-1])) // 2, k
        del raw, rep
    for k in ("clean", "strays_1"):
        (d, o), (rd, ro) = cases[k]
        pins = []
        for arr in (d, o, rd, ro):
            p = c.pinned(arr.shape, arr.dtype); p.array[:] = arr; pins.append(p)
        oi, oo, oc, orp = c.pinned(cap, np.uint32), c.pinned(n + 1, np.uint64), c.pinned(n, np.uint32), c.pinned(n, np.uint32)
        fns = {"lossy": lambda: c.encode_batch_lossy(pins[0].array, pins[1].array, None, oi.array, oo.array, oc.array, orp.array),
               "strict_on_repaired": lambda: c.encode_batch(pins[2].array, pins[3].array, None, oi.array, oo.array, oc.array)}
        t = timed(fns, STEPS)
        t["lossy"]["over_strict_ms"] = round(t["lossy"]["median_ms"] - t["strict_on_repaired"]["median_ms"], 4)
        times["host_" + k] = t
        for p in pins + [oi, oo, oc, orp]:
            p.free()
    res["times"] = times
    plug.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
