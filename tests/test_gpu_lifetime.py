"""A closed context gives back the device memory it took (csrc/cfbpe.cu: every buffer, stream and event of a context has an
owner that releases it): five rounds of create, use every group of buffers a context allocates on first use, close; this
process's device memory after every close equals its value after the first."""
import os

import numpy as np
import pytest

import fuzzgen
from conftest import pack

pytestmark = pytest.mark.gpu

GRANULARITY = 2 << 20          # the driver maps device memory in 2 MiB pages
ROUNDS = 5
MAX_BYTES = 4 << 20
SPECIALS = {"<|endoftext|>": 200000, "<|fim_prefix|>": 200001}


def nvml_processes(pynvml):
    """{(device index, pid): device bytes} of every process NVML lists (the GPUs are shared: a device-wide free-memory figure
    moves with other people's work, a process's own figure does not)"""
    out = {}
    for i in range(pynvml.nvmlDeviceGetCount()):
        for p in pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(i)):
            if p.usedGpuMemory is not None:
                out[(i, p.pid)] = p.usedGpuMemory
    return out


def own_entry(pynvml):
    """this process's key in nvml_processes: its pid, or, where NVML lists it under another PID (a container's PID namespace),
    the one entry that grows by a probe allocation and shrinks back when the probe is freed; None when there is none"""
    import torch
    torch.cuda.empty_cache()           # the probe must come from the driver, not from blocks torch keeps
    before = nvml_processes(pynvml)
    mine = [k for k in before if k[1] == os.getpid()]
    if len(mine) == 1:
        return mine[0]
    probe = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    grown = nvml_processes(pynvml)
    del probe
    torch.cuda.empty_cache()
    back = nvml_processes(pynvml)
    mine = [k for k in before if k in grown and k in back and 0 <= grown[k] - before[k] - (64 << 20) <= GRANULARITY
            and abs(back[k] - before[k]) <= GRANULARITY]
    return mine[0] if len(mine) == 1 else None


def use_every_group(c, tekken_bytes, data, offs, d_in, d_out):
    """every call that allocates lane buffers on first use, twice: consecutive calls take the context's two lanes in turn"""
    import torch
    from cfbpe import _native as N
    n, total = len(offs) - 1, int(offs[-1])
    c.vocab_load(0, tekken_bytes, N.FORMAT_TIKTOKEN, 0, 100256)
    c.vocab_set_specials(0, SPECIALS)
    allow = [np.ones(len(SPECIALS), np.uint8)]
    for _ in range(2):
        ids, _, _ = c.encode_batch(data, offs)                 # pipelined: CFBPE_PIPE_MIN_BYTES=1
        s_ids, _, _, _ = c.encode_batch_starts(data, offs)
        assert np.array_equal(s_ids, ids)
        c.truncate_batch(data, offs, 40)
        c.chunk_batch(data, offs, 64, 8)
        c.encode_batch_special(data, offs, modes=allow)
        nt = c.encode_batch_device(n, d_in[0].data_ptr(), total, d_in[1].data_ptr(), None, d_out[0].data_ptr(), total + 1,
                                   d_out[1].data_ptr(), d_out[2].data_ptr(), torch.cuda.current_stream().cuda_stream)
        assert nt == len(ids)
    c.profile_enable(True)                                     # a profiled call runs in one pass
    assert np.array_equal(c.encode_batch(data, offs)[0], ids)
    assert c.profile_read()["n_tokens"] == len(ids)
    c.profile_enable(False)


def test_closed_contexts_give_back_their_device_memory(tekken_bytes, monkeypatch):
    pynvml = pytest.importorskip("pynvml")
    import torch
    from cfbpe import _native as N
    monkeypatch.setenv("CFBPE_PIPE_MIN_BYTES", "1")
    monkeypatch.setenv("CFBPE_PIPE_CHUNK_BYTES", str(64 << 10))
    texts = fuzzgen.fuzz_strings(71, 8000, max_atoms=60)
    texts = [t + "<|endoftext|>" if i % 10 == 3 else t for i, t in enumerate(texts)]
    data, offs = pack([t.encode() for t in texts])
    n, total = len(offs) - 1, int(offs[-1])
    # the device-path call's buffers live across the rounds: the process's memory then moves only with the contexts
    d_in = (torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).cuda(), torch.from_numpy(offs.view(np.int64)).cuda())
    d_out = (torch.zeros(total + 1, dtype=torch.int32, device="cuda"), torch.zeros(n + 1, dtype=torch.int64, device="cuda"),
             torch.zeros(n, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    pynvml.nvmlInit()
    try:
        key = own_entry(pynvml)
        if key is None:
            pytest.skip("NVML lists no device memory this process can tell as its own")
        held, after = [], []
        for _ in range(ROUNDS):
            c = N.Context(0, MAX_BYTES, 1 << 18, n_workspaces=2)
            use_every_group(c, tekken_bytes, data, offs, d_in, d_out)
            held.append(nvml_processes(pynvml)[key])
            c.close()
            after.append(nvml_processes(pynvml)[key])
    finally:
        pynvml.nvmlShutdown()
    mib = ["%.1f MiB" % (m / 2 ** 20) for m in held + after]
    assert min(held) - after[0] > 32 * MAX_BYTES, mib      # the figure sees an open context: a lane holds ~33 bytes per byte of MAX_BYTES
    assert all(abs(m - after[0]) <= GRANULARITY for m in after), mib
