#!/usr/bin/env python3
"""Per-kernel times against the DIVERSITY of the pieces (VERDICT r1, weak 10: the bench corpus is ~2 MB of text tiled to 134 MB, so
its distinct pieces are few and the hash probes hit L1 / L2 more than production text would).  Batches of the same size and prompt
lengths whose "words" are drawn from the vocabulary itself: the first D valid-UTF-8 tokens of the rank file, stripped, uniformly --
D = 1 000 ... all of them (about 10^5 distinct pieces).  The batches are cfbpe.workload.make_vocab_text's "diverse" kind: the words
joined by spaces, line breaks, punctuation and digit groups, with a share of separator-free runs.  JSON lines: D, per-kernel ms."""
import json, os, sys
os.environ.setdefault("CFBPE_ALLOW_STAND_IN", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "cyberfabric-core_b200")):
    sys.path.insert(0, p)
import numpy as np
import torch
from cfbpe import plugin as P, vocabs as V, workload as W, _native as N

rv = V.resolve("cl100k_base", allow_stand_in=True)
n_words = len(W.vocab_words(W.vocab_tokens(rv.file_bytes, rv.max_ranks)))
plug = P.GpuBpeTokenizerPlugin(0, ("cl100k_base",), 160 << 20, 1 << 17)
dev = torch.device("cuda:0")
n = 65536
for D in [int(a) for a in sys.argv[1:]] or [1000, 10000, n_words]:
    D = min(D, n_words)
    # prompts of 8..4096 bytes (like the bench batch), cut at character boundaries
    data, offs = W.make_vocab_text(rv.file_bytes, rv.max_ranks, 7, "diverse", n_prompts=n, distinct=D)
    total = len(data)
    d_bytes = torch.zeros(total + 256, dtype=torch.uint8, device=dev); d_bytes[:total] = torch.from_numpy(data.copy()).to(dev)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    d_ids = torch.empty(total + 1, dtype=torch.int32, device=dev)
    d_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    d_cnt = torch.empty(n, dtype=torch.int32, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    plug.ctx.profile_enable(True)
    acc = {k: 0.0 for k in N.KERNEL_NAMES}
    reps = 4
    for i in range(reps + 2):
        nt = plug.ctx.encode_batch_device(n, d_bytes.data_ptr(), total, d_offs.data_ptr(), None, d_ids.data_ptr(), d_ids.numel(), d_off.data_ptr(), d_cnt.data_ptr(), s, sync=True)
        pr = plug.ctx.profile_read()
        if i >= 2:
            for k in acc: acc[k] += pr["kernel_ms"][k] / reps
    plug.ctx.profile_enable(False)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        plug.ctx.encode_batch_device(n, d_bytes.data_ptr(), total, d_offs.data_ptr(), None, d_ids.data_ptr(), d_ids.numel(), d_off.data_ptr(), d_cnt.data_ptr(), s, sync=False)
    e1.record(); torch.cuda.synchronize(); plug.ctx.device_status(s)
    step = e0.elapsed_time(e1) / 5
    print(json.dumps({"distinct_words": D, "bytes": total, "tokens": nt, "miss_pieces": pr["n_miss_pieces"], "device_ms": round(step, 3), "GBps": round(total / step / 1e6, 2),
                      "kernel_ms": {k: round(v, 3) for k, v in acc.items() if v}}), flush=True)
