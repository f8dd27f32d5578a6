#!/usr/bin/env python3
"""What an id base costs (a measurement aid, not a bench): cfbpe_encode_batch_device on the config-3 mix in device memory, on the
Tekken slot with base 0 (no rebase is launched) against the same slot with base 1000 (one read and one write of every id), the
calls alternated call by call, device time by CUDA events, the median of STEPS warmed calls.  Two pairs:
  one_vocab    d_vocab_ids = NULL: the rebase adds one constant
  per_prompt   every prompt names the slot in d_vocab_ids: the rebase finds each id's prompt in the offsets
The base is set between the timed calls (cfbpe_vocab_set_id_base takes the vocabularies exclusively; no device work).
Prints the card's name and power limit with the numbers, and checks once that the based ids are the unbased ones + 1000.
--out PATH writes the JSON line to PATH too.  --rehearse builds the inputs only."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "cyberfabric-core_b200")):
    sys.path.insert(0, p)
import numpy as np
from cfbpe import workload as W

STEPS = int(os.environ.get("ID_BASE_TIMES_STEPS", "20"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def main():
    data, offs, _, _ = W.make_config(3, 1.0)
    total, n = int(offs[-1]), len(offs) - 1
    res = {"steps": STEPS, "prompts": n, "bytes": total}
    if "--rehearse" in sys.argv[1:]:
        res["rehearsal"] = "inputs built"
        print(json.dumps(res))
        return
    import torch
    from cfbpe import _native as N
    tb = open(os.path.join(ROOT, "vocabs", "tekken_240911.tiktoken"), "rb").read()
    c = N.Context(0, max_batch_bytes=total + (1 << 20), max_prompts=n + 16)
    c.vocab_load(0, tb, N.FORMAT_TIKTOKEN, N.PATTERN_IDS["tekken"], 130072)
    dev = torch.device("cuda:0")
    d_bytes = torch.zeros(total + 64, dtype=torch.uint8, device=dev)
    d_bytes[:total] = torch.from_numpy(data).to(dev)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    d_ids = torch.empty(total + 1, dtype=torch.int32, device=dev)
    d_off = torch.empty(n + 1, dtype=torch.int64, device=dev)
    d_vid = torch.zeros(n, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    s = torch.cuda.current_stream()

    def call(per_prompt):
        return c.encode_batch_device(n, d_bytes.data_ptr(), total, d_offs.data_ptr(), d_vid.data_ptr() if per_prompt else None, d_ids.data_ptr(),
                                     total + 1, d_off.data_ptr(), None, stream, False)

    call(False); torch.cuda.synchronize()
    n_tok = int(d_off[-1].item())
    plain = d_ids[:n_tok].clone()
    res["ids"] = n_tok
    for mode, per_prompt in (("one_vocab", False), ("per_prompt", True)):
        ts = {"base0": [], "base1000": []}
        for r in range(STEPS + 3):         # 3 warm-up rounds; the base is set between the timed calls (it takes the vocabularies exclusively)
            for k, base in (("base0", 0), ("base1000", 1000)):
                c.vocab_set_id_base(0, base)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(s); call(per_prompt); b.record(s)
                b.synchronize()
                if r >= 3:
                    ts[k].append(a.elapsed_time(b))
        assert torch.equal(d_ids[:n_tok], plain + 1000), mode       # (the last call of a round is the based one)
        res[mode] = {k: {"median_ms": round(float(np.median(v)), 4), "range_ms": [round(min(v), 4), round(max(v), 4)]} for k, v in ts.items()}
        res[mode]["rebase_ms"] = round(res[mode]["base1000"]["median_ms"] - res[mode]["base0"]["median_ms"], 4)
    res["gpu"] = gpu_info()
    c.close()
    line = json.dumps(res)
    print(line)
    if "--out" in sys.argv[1:]:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
