"""Vocabulary importers of the model-registry side (SURVEY.md section 8(f) item 3).

`hf_tokenizer_json_to_rank_file` turns a Hugging Face `tokenizer.json` of a byte-level BPE model (GPT-2 / Llama-3 / Qwen style)
into the `.tiktoken` rank file the device table builder reads (`csrc/vocab.cpp:parse_tiktoken`; format:
tiktoken/load.py:160-172: base64(token bytes), space, decimal rank, one per line).

The two formats describe the same merges differently -- HF lists the merges in order, tiktoken ranks every token's BYTES and
merges the adjacent pair whose concatenation ranks lowest -- and agree exactly when (a) the vocabulary holds all 256 single
bytes, (b) the ids of the mergeable tokens are base..base+n-1 (rank = id - base), and (c) the merge list, read in order, produces tokens of increasing id.
The importer checks all three and refuses a file it cannot convert exactly (a wrong count is worse than no count: the numbers
bill tenants).  Special / added tokens are returned separately: they are not part of the rank file (tiktoken keeps them apart too).
The base is 0 for GPT-2 / Llama-3 style files; Mistral's Tekken files put their 1000 control tokens first and number the
mergeable tokens from 1000 -- load such a rank file with that id base (cfbpe_vocab_set_id_base) to get the file's ids.
"""
from __future__ import annotations

import base64
import hashlib
import json
from typing import Dict, Optional, Tuple

from . import _native as N

# pattern strings as they appear in published tokenizer.json files (Split pre-tokenizers) -> pattern id of include/cfbpe.h
_KNOWN_PATTERNS = {
    r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+": N.PATTERN_LLAMA3,
    r"'(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}++|\p{N}{1,3}+| ?[^\s\p{L}\p{N}]++[\r\n]*+|\s++$|\s*[\r\n]|\s+(?!\S)|\s": N.PATTERN_CL100K,
}


class ImportError_(ValueError):
    """the file cannot be converted exactly"""


def bytes_to_unicode() -> Dict[int, str]:
    """GPT-2's printable stand-ins for the 256 byte values (the alphabet byte-level BPE vocabularies are written in)"""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(0xA1, 0xAC + 1)) + list(range(0xAE, 0xFF + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return {b: chr(c) for b, c in zip(bs, cs)}


def _find_pattern(node) -> Optional[str]:
    if isinstance(node, dict):
        if node.get("type") == "Split" and isinstance(node.get("pattern"), dict):
            return node["pattern"].get("Regex")
        for v in node.values():
            r = _find_pattern(v)
            if r:
                return r
    elif isinstance(node, list):
        for v in node:
            r = _find_pattern(v)
            if r:
                return r
    return None


def hf_tokenizer_json_to_rank_file(data: bytes) -> Tuple[bytes, dict]:
    """-> (rank file bytes, meta).  meta = {n_ranks, id_base, pattern_id or None, pattern, sha256 of the rank file, special_tokens}"""
    try:
        j = json.loads(data)
        model = j["model"]
    except (ValueError, KeyError, TypeError) as e:
        raise ImportError_("not a tokenizer.json: %s" % e) from None
    if model.get("type") != "BPE":
        raise ImportError_("model type %r is not BPE" % model.get("type"))
    vocab, merges = model.get("vocab"), model.get("merges")
    if not isinstance(vocab, dict) or not isinstance(merges, list):
        raise ImportError_("BPE model without vocab / merges")
    u2b = {c: b for b, c in bytes_to_unicode().items()}
    added = {t["content"]: int(t["id"]) for t in j.get("added_tokens", []) if isinstance(t, dict) and "content" in t}
    toks: Dict[int, bytes] = {}
    for s, i in vocab.items():
        if s in added:
            continue
        try:
            toks[int(i)] = bytes(u2b[ch] for ch in s)
        except KeyError:
            raise ImportError_("token %r is not written in the byte-level alphabet (not a byte-level BPE vocabulary)" % s) from None
    n = len(toks)
    base = min(toks) if toks else 0
    if sorted(toks) != list(range(base, base + n)):
        raise ImportError_("mergeable token ids are not %d..%d" % (base, base + n - 1))
    toks = {i - base: b for i, b in toks.items()}
    rank = {b: i for i, b in toks.items()}
    if len(rank) != n:
        raise ImportError_("two ids share the same bytes")
    if any(bytes([b]) not in rank for b in range(256)):
        raise ImportError_("the vocabulary does not hold all 256 single bytes")
    last = -1
    for m in merges:
        a, b = (m.split(" ", 1) if isinstance(m, str) else m)
        try:
            ab = bytes(u2b[ch] for ch in a) + bytes(u2b[ch] for ch in b)
        except KeyError:
            raise ImportError_("merge %r is not written in the byte-level alphabet" % (m,)) from None
        r = rank.get(ab)
        if r is None:
            raise ImportError_("merge %r produces a token that is not in the vocabulary" % (m,))
        if r <= last:
            raise ImportError_("merge order and token ids disagree at %r (id %d after id %d): rank-by-bytes would merge differently" % (m, r, last))
        last = r
    if len(merges) != n - 256:
        raise ImportError_("%d merges for %d multi-byte tokens: some tokens are not reachable by merges" % (len(merges), n - 256))
    out = b"".join(base64.b64encode(toks[i]) + b" " + str(i).encode() + b"\n" for i in range(n))
    pattern = _find_pattern(j.get("pre_tokenizer"))
    meta = {"n_ranks": n, "id_base": base, "pattern": pattern, "pattern_id": _KNOWN_PATTERNS.get(pattern), "sha256": hashlib.sha256(out).hexdigest(),
            "special_tokens": added}
    return out, meta


def tokenizer_descriptor(vocab_id: str, pattern_id: int, rank_file: bytes) -> dict:
    """the `tokenizer` object proposed for the model-registry `Model` entity (docs/model-registry-tokenizer-proposal.md)"""
    names = {v: k for k, v in N.PATTERN_IDS.items()}
    return {"vocab_id": vocab_id, "pattern_id": names[pattern_id], "sha256": hashlib.sha256(rank_file).hexdigest()}
