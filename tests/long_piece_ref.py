"""A reference BPE merge for pieces of MiB size (test infrastructure).

tiktoken's merge loop (and the oracle's encode_piece) rescan the whole piece for every merge: quadratic in the piece length,
billions of steps at 100 KB.  This is the same loop, kept in a doubly linked list of parts and a min-heap of pairs keyed by
(rank, start position), so a piece of n bytes costs O(n log n):
  * the whole piece, if it is a token, is that one token (tiktoken's shortcut);
  * otherwise the adjacent pair whose concatenation has the lowest rank merges, the leftmost one on equal ranks;
  * a merge changes only the pairs on either side of the new part: those two are pushed, the old entries go stale.
A heap entry names the start of its left part and its rank.  The rank is that of the pair's bytes, and a part's start never
changes while it lives, so an entry is current iff its left part is alive and the pair starting there still has that rank
(a merged pair covers more bytes: it cannot have the old rank again)."""
import base64
import heapq

NONE = -1
_SHIFT = 32          # heap key = rank << _SHIFT | start
K_LIST_MAX = 65535   # bpe_kernels.cuh: kListMax, the most parts bpe_long_kernel's list rounds take (16-bit link fields)


def ranks_of(rank_file: bytes, max_ranks: int = 0):
    """{token bytes: rank} of a rank file in the tiktoken format, its first max_ranks lines (0: all)"""
    lines = [l for l in rank_file.splitlines() if l.strip()]
    if max_ranks:
        lines = lines[:max_ranks]
    return {base64.b64decode(l.split()[0]): int(l.split()[1]) for l in lines}


def merge(ranks, piece: bytes):
    """the ranks of the tokens tiktoken's merge loop makes of `piece`; ranks: {token bytes: rank}"""
    n = len(piece)
    if n == 0:
        return []
    whole = ranks.get(piece)
    if whole is not None:
        return [whole]
    get = ranks.get
    nxt = list(range(1, n + 1))            # nxt[s]: start of the part after the part at s (n: none)
    prv = list(range(-1, n - 1))           # prv[s]: start of the part before it (-1: none)
    alive = [True] * n
    cur = [NONE] * n                       # cur[s]: rank of the pair (part at s, next part), NONE when there is none
    heap = []
    for s in range(n - 1):
        r = get(piece[s:s + 2])
        if r is not None:
            cur[s] = r
            heap.append((r << _SHIFT) | s)
    heapq.heapify(heap)
    mask = (1 << _SHIFT) - 1
    pop, push = heapq.heappop, heapq.heappush
    while heap:
        key = pop(heap)
        s = key & mask
        r = key >> _SHIFT
        if not alive[s] or cur[s] != r:
            continue
        t = nxt[s]
        e = nxt[t]
        alive[t] = False
        nxt[s] = e
        if e < n:
            prv[e] = s
            r2 = get(piece[s:nxt[e]])
            cur[s] = NONE if r2 is None else r2
            if r2 is not None:
                push(heap, (r2 << _SHIFT) | s)
        else:
            cur[s] = NONE
        p = prv[s]
        if p >= 0:
            r2 = get(piece[p:e])
            cur[p] = NONE if r2 is None else r2
            if r2 is not None:
                push(heap, (r2 << _SHIFT) | p)
    out = []
    s = 0
    while s < n:
        out.append(ranks[piece[s:nxt[s]]])
        s = nxt[s]
    return out


def first_difference(got, want):
    """None when the two id sequences are equal, else where they first differ and the ids there"""
    got, want = [int(v) for v in got], [int(v) for v in want]
    if got == want:
        return None
    i = next((k for k, (a, b) in enumerate(zip(got, want)) if a != b), min(len(got), len(want)))
    return "%d tokens, want %d; first difference at token %d: got %s, want %s" % (len(got), len(want), i, got[i:i + 4], want[i:i + 4])


def encode(ranks, pattern_id: int, prompt: bytes):
    """a whole prompt: the oracle's pre-tokenizer split, then merge() on every piece"""
    from oracle import oracle
    out, a = [], 0
    for e in oracle.split(pattern_id, prompt).tolist():
        out += merge(ranks, prompt[a:e])
        a = e
    return out


# ---- pieces that decide exactly how many parts bpe_long_kernel has when it could enter its list rounds.
# Filler 'q' never pairs.  'zz' has the lowest rank: the first batched round merges it and nothing else, leaving m parts.  The
# pairs left -- 'xy' at the last two parts, 'ab' at the first two, 'cd' in the middle, in that rank order -- are one merge each:
# while m > kListMax each costs a batched round of its own, and what is left when m <= kListMax goes to the list rounds.
# 'xyab' is never reached by the merge loop; a kernel whose 16-bit links wrap at m = 65536 makes the last part the first
# part's neighbour and merges the two into it.
BOUNDARY_TOKENS = [b"zz", b"xy", b"ab", b"cd", b"xyab"]
BOUNDARY_MERGES = {"first": b"ab", "mid": b"cd", "last": b"xy"}
# (parts after the first batched round, merges left, whether the list rounds run)
BOUNDARY_CASES = [
    (K_LIST_MAX - 1, ("first", "mid", "last"), True),
    (K_LIST_MAX, ("first", "mid", "last"), True),        # the last pair is parts 65 533 and 65 534
    (K_LIST_MAX + 1, ("first", "mid", "last"), True),    # one batched round ('xy'), then the list rounds at m = 65 535
    (K_LIST_MAX + 2, ("first", "mid", "last"), True),    # two batched rounds, then the list rounds merge 'cd'
    (K_LIST_MAX + 2, ("first", "last"), False),          # two batched rounds, then no pair is left
]


def boundary_rank_file() -> bytes:
    toks = [bytes([b]) for b in range(256)] + BOUNDARY_TOKENS
    return b"".join(base64.b64encode(t) + b" %d\n" % i for i, t in enumerate(toks))


def boundary_piece(m: int, merges) -> bytes:
    """a letter run of m + 1 bytes: m parts after 'zz' merges, then the merges named in `merges`"""
    head = BOUNDARY_MERGES["first"] if "first" in merges else b"qq"
    mid = BOUNDARY_MERGES["mid"] if "mid" in merges else b"qq"
    tail = BOUNDARY_MERGES["last"] if "last" in merges else b"qq"
    fill = m + 1 - 8
    a = fill // 2
    b = fill - a - 1
    return head + b"q" * a + mid + b"q" + b"zz" + b"q" * b + tail
