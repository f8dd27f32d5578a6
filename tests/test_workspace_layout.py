"""The workspace layout of csrc/pipeline.cuh (host code, on the CPU): a pipelined host call runs its sub-batches side by side in
one lane's buffers, so every sub-batch's slice must hold what a pass over its bytes touches without reaching into the next one,
and the lane's allocation must hold the last.  The sizes of a default lane are pinned: the per-lane device footprint."""
import os
import random
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))
import simlib  # noqa: E402

MAX_CHUNKS = 64


def _check_batch(offs, chunk, max_bytes, max_prompts, what):
    n = len(offs) - 1
    cut = simlib.plan_sub_batches(offs, chunk, MAX_CHUNKS)
    subs = []
    for k in range(len(cut) - 1):
        p0, p1 = cut[k], cut[k + 1]
        o0, length = int(offs[p0]), int(offs[p1] - offs[p0])
        lay = simlib.workspace_layout(o0, length, k, p0, max_bytes, max_prompts, MAX_CHUNKS)
        ext = lay["extent"]
        for name, cap in lay["caps"].items():
            assert cap == ext[name], (what, k, name, cap, ext[name])
        assert lay["bytes_at"] % 16 == 0, (what, k, lay["bytes_at"])
        subs.append((length, p1 - p0, lay))
    for k, (length, nk, lay) in enumerate(subs):
        ext = lay["extent"]
        last = k + 1 == len(subs)
        nxt = None if last else subs[k + 1][2]
        for name, (kind, _, start, alloc) in lay["buffers"].items():
            end = start + ext[kind]
            limit = alloc if last else nxt["buffers"][name][2]
            assert end <= limit, (what, k, len(subs), name, start, ext[kind], limit)
        bytes_end = lay["bytes_at"] + length
        assert bytes_end + (16 if last else 0) <= (lay["bytes_alloc"] if last else nxt["bytes_at"]), (what, k, "d_bytes")
        offs_end = lay["offsets_at"] + nk + 1
        assert offs_end <= (lay["offsets_alloc"] if last else nxt["offsets_at"]), (what, k, "offsets")
    assert cut[-1] == n


def test_sub_batch_slices_tile_the_lane_workspace():
    """for every sub-batch of plan_sub_batches and every buffer: the slice holds workspace_extent of its bytes and ends before
    the next slice starts, the last ends inside workspace_alloc, the caps the kernels check are the extents, and every sub-batch's
    bytes start on a 16-byte boundary; long, empty and tiny prompts, sub-batches of 1 byte to 12 MiB, max_bytes = the batch and more"""
    rng = random.Random(17)
    for trial in range(300):
        n = rng.choice([1, 2, 3, 17, 500, 5000])
        kind = rng.randint(0, 3)
        lens = [rng.choice([0, 1, 7, 4096]) if kind == 0 else rng.randint(0, 4096) if kind == 1 else rng.randint(0, 40) if kind == 2
                else rng.choice([0, 0, 3, 300000]) for _ in range(n)]
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
        total = int(offs[-1])
        chunk = rng.choice([1, 64, 1000, 12 << 10, 12 << 20])
        max_bytes = total if trial % 2 == 0 else total + rng.choice([1, 31, 4096, 12 << 20])
        max_prompts = n if trial % 3 else n + rng.randint(1, 1000)
        _check_batch(offs, chunk, max_bytes, max_prompts, (trial, n, kind, chunk, max_bytes))
    # the bench shape: 65 536 prompts of 8..4096 bytes in 12 MiB sub-batches, a lane of 256 MiB
    lens = np.random.default_rng(3).integers(8, 4097, size=65536)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    _check_batch(offs, 12 << 20, 256 << 20, 1 << 20, "bench")


def test_lane_allocation_sizes_are_pinned():
    """the element counts a lane of max_batch_bytes = 256 MiB, max_prompts = 2^20 allocates (64 sub-batches), worked out by
    hand from the sizes the lane has always had: the per-lane device footprint"""
    lay = simlib.workspace_layout(0, 0, 0, 0, 256 << 20, 1 << 20, MAX_CHUNKS)
    want = {
        "piece_bits": 8388868, "tok_bits": 8388868, "pstart_bits": 8388868,          # 2^23 words + 4 + 4 x 64
        "ids_by_pos": 268435457, "lscratch.rank": 268435457, "lscratch.aux0": 268435457, "lscratch.aux1": 268435457,
        "dense.by_piece": 268435457, "dense.extras": 268435457,                      # 2^28 + 1
        "long_list": 8388673,                                                        # 2^23 + 1 + 64
        "tile_counts": 32897, "tile_base": 32897,                                    # 2^15 tiles + 1 + 2 x 64
        "miss.list[0]": 20649073, "miss.list[1]": 38348114, "miss.list[2]": 134217920,   # 2^28 / (13 | 7 | 2) + 2 x 64 + 64
        "fix_list": 16777346,                                                        # 2^24 + 2 + 2 x 64
        "dense.tile_pieces": 131202, "dense.piece_base": 131202,                     # 2^17 + 2 + 2 x 64
        "block_prompt": 524418,                                                      # 2^19 + 2 + 2 x 64
    }
    got = {name: alloc for name, (_, _, _, alloc) in lay["buffers"].items()}
    assert got == want
    assert lay["bytes_alloc"] == 268436752            # 2^28 + 256 + 16 x 65
    assert lay["offsets_alloc"] == 1048641            # 2^20 + 1 + 64
