"""Python mirror of the ModKit plugin surface the tokenizer sits behind.

The Rust toolchain is absent from this image (SURVEY.md F7), so the host side above the C ABI
is written here with the names, argument meaning and error behaviour a ModKit plugin has
(INTEGRATION.md shows the Rust crates a maintainer would add).  Conventions mirrored, with
the reference file each one follows:

* plugin trait name ends in `PluginClient` (lint DE0503, dylint_lints/README.md:36); methods
  take the SecurityContext first and return Result<_, XError>
  (modules/system/tenant-resolver/tenant-resolver-sdk/src/plugin_api.rs:28-47);
* error enum with NoPluginAvailable / ServiceUnavailable(String) / Internal(String)
  (modules/system/tenant-resolver/tenant-resolver-sdk/src/error.rs:7-34);
* a plugin registers a GTS instance {id, vendor, priority, properties}
  (libs/modkit/src/gts/plugin.rs:12-17) and a client scoped by that instance id
  (libs/modkit/src/client_hub.rs:142-234); the gateway picks vendor match, lowest priority
  (libs/modkit/src/plugins/mod.rs:136-191) and resolves lazily, once;
* token counts feed Usage.input_tokens >= 0
  (modules/llm-gateway/llm-gateway-sdk/schemas/core/usage.v1.schema.json:8-12) and are the sum over a
  request's TextContent.text parts (schemas/content/text_content.v1.schema.json,
  schemas/core/message.v1.schema.json).

Prompt text is never logged (modules/llm-gateway/docs/DESIGN.md:120-124): only sizes and counts.
"""
from __future__ import annotations

import json
import re
import threading
import uuid
from dataclasses import dataclass, field
from typing import Tuple, Dict, List, Optional, Sequence

import numpy as np

from . import _native as N
from . import vocabs as V


# --------------------------------------------------------------------------- errors
class TokenizerError(Exception):
    """base of the SDK error enum (`TokenizerError` in the planned llm-gateway-sdk)"""


class NoPluginAvailable(TokenizerError):
    pass


class ServiceUnavailable(TokenizerError):
    pass


class Internal(TokenizerError):
    pass


class InvalidInput(TokenizerError):
    """bad offsets / malformed UTF-8 / oversize batch (maps to RFC 9457 Problem 400)"""


class VocabNotFound(TokenizerError):
    pass


def _map_native(e: N.NativeError) -> TokenizerError:
    if e.code in (N.EINVAL, N.EILSEQ, N.ENOSPC, N.EBADMSG):     # EBADMSG: the message names the disallowed special token
        return InvalidInput(str(e))
    if e.code == N.ENOENT:
        return VocabNotFound(str(e))
    if e.code in (N.ENODEV, N.ENOMEM):
        return ServiceUnavailable(str(e))
    return Internal(str(e))


# --------------------------------------------------------------------------- boundary types
@dataclass(frozen=True)
class SecurityContext:
    """libs/modkit-security/src/context.rs:23-39 (tenant identity carried on every plugin call)"""
    subject_id: uuid.UUID
    subject_tenant_id: uuid.UUID
    subject_type: Optional[str] = None
    token_scopes: Sequence[str] = ()

    @staticmethod
    def anonymous() -> "SecurityContext":
        z = uuid.UUID(int=0)
        return SecurityContext(z, z, "service", ("*",))


@dataclass(frozen=True)
class VocabRef:
    """names a loaded vocabulary: registry name ("cl100k_base") or canonical model id ("openai::gpt-4")"""
    name: str


@dataclass
class EncodeBatchRequest:
    vocab: VocabRef
    bytes: np.ndarray            # uint8, packed UTF-8 of all prompts
    offsets: np.ndarray          # uint64, n+1, offsets[0] == 0
    vocabs_per_prompt: Optional[Sequence[VocabRef]] = None   # multi-tenant batches: one vocab per prompt
    vocab_index: Optional[np.ndarray] = None   # uint8, n: with it, vocabs_per_prompt lists the DISTINCT vocabularies and
                                               # vocab_index[i] picks prompt i's (large batches: no per-prompt objects)
    with_starts: bool = False    # also return every token's byte offset within its prompt (EncodeBatchResponse.starts)
    starts_unit: str = "byte"    # with with_starts: "byte", or "codepoint" / "utf16" -- the starts in that unit and EncodeBatchResponse.lens
    errors: str = "strict"       # bytes that are not valid UTF-8: "strict" fails the call, "replace" encodes every prompt as
                                 # bytes.decode("utf-8", "replace") (EncodeBatchResponse.replaced; not with with_starts)


@dataclass
class EncodeBatchResponse:
    ids: np.ndarray              # uint32 dense id stream
    offsets: np.ndarray          # uint64, n+1
    counts: np.ndarray           # uint32, n
    starts: Optional[np.ndarray] = None   # uint32, one per id: offset of the token within its prompt in starts_unit (with_starts)
    lens: Optional[np.ndarray] = None     # uint32, one per prompt: its length in starts_unit (a "codepoint" / "utf16" request)
    replaced: Optional[np.ndarray] = None  # uint32, one per prompt: the U+FFFD its decode inserted (an errors="replace" request)


@dataclass
class TruncateBatchResponse:
    """where each prompt is cut to its token budget (TokenizerPluginClient.truncate_batch), one entry per prompt"""
    cut: np.ndarray              # uint32: byte position of the cut in the prompt; "head" keeps [0, cut), "tail" keeps [cut, len)
    kept: np.ndarray             # uint32: tokens of the prompt's encoding wholly inside the kept text
    counts: np.ndarray           # uint32: tokens of the whole prompt


TRUNCATE_KEEP = {"head": N.TRUNCATE_HEAD, "tail": N.TRUNCATE_TAIL}


def _truncate_mode(keep: str) -> int:
    if keep not in TRUNCATE_KEEP:
        raise InvalidInput("keep must be 'head' or 'tail', not %r" % (keep,))
    return TRUNCATE_KEEP[keep]


def _budgets(budgets, n: int) -> np.ndarray:
    try:
        return N.Context.budget_array(budgets, n)[:n]
    except N.NativeError as e:
        raise InvalidInput(str(e)) from e


def truncate_cuts(data: np.ndarray, offsets: np.ndarray, id_offsets: np.ndarray, starts: np.ndarray, budgets: np.ndarray,
                  tail: bool) -> Tuple[np.ndarray, np.ndarray]:
    """The truncation contract (include/cfbpe.h, cfbpe_truncate_batch) from every token's start: (cut, kept), uint32 per prompt.
    head: the first k = min(budget, c) tokens end at x; the cut is the character start at or before x.  tail: the last k tokens
    start at x; the cut is the character start at or after x (or the end).  kept: the tokens wholly inside the kept text."""
    n = len(offsets) - 1
    cut = np.zeros(n, dtype=np.uint32)
    kept = np.zeros(n, dtype=np.uint32)
    for i in range(n):
        o, ln = int(offsets[i]), int(offsets[i + 1]) - int(offsets[i])
        st = starts[int(id_offsets[i]):int(id_offsets[i + 1])].astype(np.int64)
        c = len(st)
        k = min(int(budgets[i]), c)
        j = c - k if tail else k
        x = int(st[j]) if j < c else ln                 # the first byte of token j (the end of token j - 1)
        if tail:
            while x < ln and data[o + x] & 0xC0 == 0x80:
                x += 1
            kept[i] = c - int(np.searchsorted(st, x, side="left"))
        else:
            while 0 < x < ln and data[o + x] & 0xC0 == 0x80:
                x -= 1
            ends = np.append(st[1:], ln) if c else st
            kept[i] = int(np.searchsorted(ends, x, side="right"))
        cut[i] = x
    return cut, kept


@dataclass
class ChunkBatchResponse:
    """every prompt cut into chunks of at most N tokens (TokenizerPluginClient.chunk_batch)"""
    spans: np.ndarray            # uint32 [chunks, 2]: (begin, end) of every chunk within its prompt, always character boundaries
    chunk_offsets: np.ndarray    # uint64 [n + 1]: prompt i's chunks are spans[chunk_offsets[i] .. chunk_offsets[i + 1]]
    counts: np.ndarray           # uint32: tokens of every whole prompt


def _chunk_args(chunk_tokens, overlap_tokens) -> Tuple[int, int]:
    ok = all(isinstance(v, (int, np.integer)) and not isinstance(v, bool) for v in (chunk_tokens, overlap_tokens))
    if not ok or not 1 <= int(chunk_tokens) <= 0xFFFFFFFF or not 0 <= int(overlap_tokens) < int(chunk_tokens):
        raise InvalidInput("chunk size must be an integer in 1 .. 2^32 - 1 and the overlap an integer in 0 .. chunk size - 1")
    return int(chunk_tokens), int(overlap_tokens)


def chunk_spans(data: np.ndarray, offsets: np.ndarray, id_offsets: np.ndarray, starts: np.ndarray, chunk_tokens: int,
                overlap_tokens: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """The chunking contract (include/cfbpe.h, cfbpe_chunk_batch) from every token's start: (spans uint32 [chunks, 2], chunk
    offsets uint64 [n + 1]).  Windows of N = chunk_tokens tokens start every N - overlap_tokens tokens until one reaches the last
    token; chunk k covers tokens [a, e) and its bytes are [F(a), F(e)), F(j) = the character start at or before token j's start,
    F(c) = the prompt's length."""
    n = len(offsets) - 1
    step = chunk_tokens - overlap_tokens
    spans, coffs = [], np.zeros(n + 1, dtype=np.uint64)
    for i in range(n):
        o, ln = int(offsets[i]), int(offsets[i + 1]) - int(offsets[i])
        st = starts[int(id_offsets[i]):int(id_offsets[i + 1])].astype(np.int64)
        c = len(st)

        def floor(j):
            if j >= c:
                return ln
            x = int(st[j])
            while 0 < x < ln and data[o + x] & 0xC0 == 0x80:
                x -= 1
            return x
        k = 0 if c == 0 else 1 if c <= chunk_tokens else 1 + (c - chunk_tokens + step - 1) // step
        for q in range(k):
            a = q * step
            spans.append((floor(a), floor(min(a + chunk_tokens, c))))
        coffs[i + 1] = coffs[i] + k
    return (np.array(spans, dtype=np.uint32).reshape(-1, 2), coffs)


STARTS_UNITS = {"byte": None, "codepoint": N.UNIT_CODEPOINT, "utf16": N.UNIT_UTF16}   # EncodeBatchRequest.starts_unit -> CFBPE_UNIT_*


def _starts_unit(unit: str) -> str:
    if unit not in STARTS_UNITS:
        raise InvalidInput("the offset unit must be 'byte', 'codepoint' or 'utf16', not %r" % (unit,))
    return unit


def unit_starts(data: np.ndarray, offsets: np.ndarray, id_offsets: np.ndarray, starts: np.ndarray, unit: str) -> Tuple[np.ndarray, np.ndarray]:
    """The unit-start contract (include/cfbpe.h, cfbpe_encode_batch_char_starts) from every token's byte start: (starts uint32, one
    per id; lens uint32, one per prompt) in `unit` ("byte", "codepoint" or "utf16").  A token's start is the number of units before
    the character that holds its first byte; a prompt's length is its units.  The prompts must be valid UTF-8."""
    n = len(offsets) - 1
    offs = np.asarray(offsets, dtype=np.int64)
    st = np.asarray(starts, dtype=np.int64)[:int(id_offsets[n])]
    if unit == "byte":
        return st.astype(np.uint32), np.diff(offs).astype(np.uint32)
    b = np.asarray(data[:int(offs[n])], dtype=np.uint8)
    lead = (b & 0xC0) != 0x80
    w = lead.astype(np.uint32)
    if unit == "utf16":
        w += (b >= 0xF0).astype(np.uint32)                     # a code point above the BMP is a surrogate pair
    cum = np.zeros(len(b) + 1, dtype=np.int64)
    np.cumsum(w, out=cum[1:])                                  # cum[x] = units of the characters that start before byte x
    char_start = np.maximum.accumulate(np.where(lead, np.arange(len(b), dtype=np.int64), 0)) if len(b) else np.zeros(0, np.int64)
    prompt = np.repeat(np.arange(n, dtype=np.int64), np.diff(np.asarray(id_offsets, dtype=np.int64)))
    pos = offs[prompt] + st                                    # each token's first byte in the batch
    out = cum[char_start[pos]] - cum[offs[prompt]] if len(pos) else np.zeros(0, np.int64)
    return out.astype(np.uint32), (cum[offs[1:]] - cum[offs[:-1]]).astype(np.uint32)


@dataclass
class CountTokensRequest:
    vocab: VocabRef
    bytes: np.ndarray
    offsets: np.ndarray
    vocabs_per_prompt: Optional[Sequence[VocabRef]] = None
    vocab_index: Optional[np.ndarray] = None
    errors: str = "strict"       # as EncodeBatchRequest.errors


UTF8_ERRORS = ("strict", "replace")


def _errors(req) -> str:
    """req.errors, checked: "replace" gives positions in the repaired text, not the caller's bytes, so it takes no starts"""
    e = getattr(req, "errors", "strict")
    if e not in UTF8_ERRORS:
        raise InvalidInput("errors must be 'strict' or 'replace', not %r" % (e,))
    if e == "replace" and getattr(req, "with_starts", False):
        raise InvalidInput("errors='replace' does not return starts: they would index the repaired text, not the request's bytes")
    return e


def repair_utf8(data: np.ndarray, offsets: np.ndarray):
    """every prompt as bytes.decode("utf-8", "replace").encode("utf-8") on the host: (bytes uint8, offsets uint64, replaced uint32
    -- the U+FFFD each decode inserted, one per maximal subpart of an ill-formed sequence)"""
    n = len(offsets) - 1
    raw = data.tobytes()
    parts, replaced = [], np.zeros(n, dtype=np.uint32)
    for i in range(n):
        p = raw[int(offsets[i]):int(offsets[i + 1])]
        try:
            parts.append(p.decode("utf-8").encode("utf-8"))
            continue
        except UnicodeDecodeError:
            pass
        text = p.decode("utf-8", "replace")
        replaced[i] = text.count("\ufffd") - p.count("\ufffd".encode("utf-8"))
        parts.append(text.encode("utf-8"))
    out_offs = np.zeros(n + 1, dtype=np.uint64)
    if n:
        out_offs[1:] = np.cumsum([len(x) for x in parts], dtype=np.uint64)
    return np.frombuffer(b"".join(parts) + b"\0", dtype=np.uint8)[:int(out_offs[-1])].copy(), out_offs, replaced


@dataclass
class DecodeBatchRequest:
    vocab: VocabRef
    ids: np.ndarray              # uint32, packed ids of all sequences
    offsets: np.ndarray          # uint64, n+1 (in ids)
    vocabs_per_prompt: Optional[Sequence[VocabRef]] = None
    vocab_index: Optional[np.ndarray] = None


@dataclass
class DecodeBatchResponse:
    bytes: np.ndarray            # uint8, the sequences' bytes back to back (tiktoken decode_bytes; not necessarily valid UTF-8)
    offsets: np.ndarray          # uint64, n+1


@dataclass
class Usage:
    """gts.x.llmgw.core.usage.v1~"""
    input_tokens: int
    output_tokens: int = 0


@dataclass(frozen=True)
class ChatTemplate:
    """How a provider frames a list of chat messages into the token stream it bills as `Usage.input_tokens`
    (SURVEY.md section 8(f) item 2: "chat-template overhead accounting").  Three kinds:

    "overhead"  a fixed number of framing tokens a message (OpenAI's ChatML accounting: every message is
                <|start|>{role/name}\n{content}<|end|>\n = `tokens_per_message` tokens beside role and content, a `name` costs
                `tokens_per_name` more, the reply is primed with `reply_priming` tokens);
    "rendered"  the conversation is rendered to text around control tokens (Llama 3, Mistral): `bos`, then per message
                `message_prefix.format(role=...)` + content + `message_suffix`, then `generation_prompt`; the strings in
                `special_tokens` count one token each, the text between them is tokenised as ordinary text;
    "mistral"   mistral_common's InstructTokenizer of `instruct_version` 3 (Tekken models: Mistral NeMo, Pixtral 12B), 7 (Mistral
                Large 2411, Pixtral Large 2411, Mistral Small 2501 and 2503), 11 or 13 on a conversation of text, tool calls and tool
                results, with the request's tools: mistral_instruct_texts (V3, V7) and mistral_instruct_texts_v11 (V11, V13) give
                the rules and the refusals.  Every message's text, the tools' JSON, each assistant turn's calls and each tool result
                are tokenised on their own, between control tokens ([AVAILABLE_TOOLS] before the last [INST] (V13: the first), [TOOL_CALLS], [TOOL_RESULTS]; V7 and later also
                [SYSTEM_PROMPT], [TOOL_CONTENT] (not V13); V11 and V13 also [ARGS], and V11 [CALL_ID]).
                The other kinds refuse tools; they pass over tool_call and tool_result parts.

    Message CONTENT is always ordinary text: a message that spells a control token gets the pieces of that spelling, never the
    control token (the gateway does not let user text forge framing)."""
    kind: str = "overhead"
    tokens_per_message: int = 3
    tokens_per_name: int = 1
    reply_priming: int = 3
    bos: str = ""
    message_prefix: str = ""
    message_suffix: str = ""
    generation_prompt: str = ""
    special_tokens: Tuple[str, ...] = ()
    instruct_version: int = 3           # "mistral": mistral_common's instruct tokenizer version, 3, 7, 11 or 13


# templates of the model families the stand-in vocabularies cover; a deployment lists its own next to the model's tokenizer
# (docs/model-registry-tokenizer-proposal.md)
CHAT_TEMPLATES = {
    # https://cookbook.openai.com "How to count tokens with tiktoken": gpt-3.5-turbo-0613 / gpt-4 and later
    "openai-chatml": ChatTemplate("overhead", tokens_per_message=3, tokens_per_name=1, reply_priming=3),
    # Meta Llama 3 instruct
    # Mistral's Tekken models (mistral_common InstructTokenizerV3): <s>, then [INST] user [/INST] and assistant </s>
    "mistral-v3": ChatTemplate("mistral"),
    # Mistral's V7 Tekken models (InstructTokenizerV7): system messages in place as [SYSTEM_PROMPT] text [/SYSTEM_PROMPT], tool
    # results as [TOOL_RESULTS] call id [TOOL_CONTENT] content [/TOOL_RESULTS]
    "mistral-v7": ChatTemplate("mistral", instruct_version=7),
    # InstructTokenizerV11: V7, with each tool call as [TOOL_CALLS] name [CALL_ID] id [ARGS] arguments
    "mistral-v11": ChatTemplate("mistral", instruct_version=11),
    # InstructTokenizerV13: V11 without call ids, tool results as [TOOL_RESULTS] content [/TOOL_RESULTS], tools before the first
    # user message
    "mistral-v13": ChatTemplate("mistral", instruct_version=13),
    "llama3-instruct": ChatTemplate("rendered", bos="<|begin_of_text|>",
                                    message_prefix="<|start_header_id|>{role}<|end_header_id|>\n\n", message_suffix="<|eot_id|>",
                                    generation_prompt="<|start_header_id|>assistant<|end_header_id|>\n\n",
                                    special_tokens=("<|begin_of_text|>", "<|start_header_id|>", "<|end_header_id|>", "<|eot_id|>")),
}


# the roles mistral_common's validator lets follow each role
MISTRAL_NEXT_ROLES = {"system": ("user", "assistant", "system"), "user": ("assistant", "system", "user"),
                      "assistant": ("assistant", "user", "tool"), "tool": ("assistant", "tool", "user")}
# its name and call-id rules, re.match(r"^...$"): "$" also matches before a final "\n", so one trailing "\n" passes
MISTRAL_NAME = re.compile(r"[a-zA-Z0-9_-]{1,64}\n?")
MISTRAL_CALL_ID = re.compile(r"[a-zA-Z0-9]{9}\n?")


def _mistral_json(value) -> str:
    """JSON as mistral_common writes it into the prompt: json.dumps(value, ensure_ascii=False)"""
    return json.dumps(value, ensure_ascii=False)


def _mistral_tool_content(content: str):
    """a tool result's content as mistral_common embeds it: the JSON value when the text parses as JSON, else the text; "" is {}"""
    if not content:
        return {}
    try:
        return json.loads(content)
    except json.JSONDecodeError:
        return content


def _mistral_normalized_content(content: str) -> str:
    """a tool result's content as mistral_common's V7 request normalizer leaves it: the JSON value it parses to, written again by
    _mistral_json, else the text as given; "" is "{}" """
    if not content:
        return "{}"
    try:
        return _mistral_json(json.loads(content))
    except json.JSONDecodeError:
        return content


def _mistral_tools(tools: Sequence[dict]) -> List[dict]:
    """the gateway's tools (schemas/tools/tool.v1) as mistral_common's Tool.model_dump() without `strict`"""
    out = []
    for t in tools:
        if t.get("type") != "unified":
            raise InvalidInput("the mistral template counts unified tools (name, description, parameters), not %r" % t.get("type"))
        name, description, params = t.get("name"), t.get("description"), t.get("parameters")
        schema = params.get("json_schema") if isinstance(params, dict) else None
        if not isinstance(name, str) or not isinstance(description, str) or not isinstance(schema, dict):
            raise InvalidInput("a unified tool has a string name and description and parameters {json_schema: object}")
        if not MISTRAL_NAME.fullmatch(name):
            raise InvalidInput("a tool name is 1 to 64 of a-z, A-Z, 0-9, '_' and '-'")
        out.append({"type": "function", "function": {"name": name, "description": description, "parameters": schema}})
    return out


def _mistral_message(m: dict, version: int = 3) -> Tuple[str, List[str], List[dict], Optional[Tuple[str, str]], bool]:
    """(role, text parts, tool calls, tool result (call id, content), prefix) of one gateway message; other parts (images ...)
    are not counted here.  A call is {"name", "arguments", "id"} as mistral_common prints it (no "id" for "null").  prefix is
    the `prefix` flag of an assistant message (Mistral's chat API: the reply continues this message), read under V7 and later."""
    role, parts = m.get("role"), m.get("content", [])
    if role not in MISTRAL_NEXT_ROLES:
        raise InvalidInput("the mistral template counts system, user, assistant and tool messages, not %r" % role)
    texts = [str(p["text"]) for p in parts if p.get("type") == "text"]
    text = "\n\n".join(texts)
    prefix = m.get("prefix", False) if version >= 7 else False
    if not isinstance(prefix, bool) or (prefix and role != "assistant"):
        raise InvalidInput("prefix is a boolean of an assistant message")
    calls, results = [], [p.get("tool_result") for p in parts if p.get("type") == "tool_result"]
    for p in parts:
        if p.get("type") != "tool_call":
            continue
        c = p.get("tool_call")
        if role != "assistant" or not isinstance(c, dict):
            raise InvalidInput("a tool_call part belongs to an assistant message")
        cid, name, args = c.get("id"), c.get("name"), c.get("arguments")
        if not isinstance(cid, str) or not isinstance(name, str) or not isinstance(args, dict):
            raise InvalidInput("a tool call has a string id and name and object arguments")
        if cid != "null" and not MISTRAL_CALL_ID.fullmatch(cid):
            raise InvalidInput("a tool call id is 9 of a-z, A-Z and 0-9")
        if cid == "null" and version == 13:
            raise InvalidInput("a tool call has an id under instruct V13")
        if not MISTRAL_NAME.fullmatch(name):
            raise InvalidInput("a tool call's name is 1 to 64 of a-z, A-Z, 0-9, '_' and '-'")
        calls.append({"name": name, "arguments": args, **({} if cid == "null" else {"id": cid})})
    if version == 3 and role == "assistant" and bool(text) == bool(calls):     # (V7: text, calls or both, once merged)
        raise InvalidInput("an assistant message holds text or tool calls, one of the two" if text else "an assistant message without text or tool calls")
    if (role == "tool") != bool(results):
        raise InvalidInput("a tool_result part belongs to a tool message" if results else "a tool message holds a tool_result part")
    result = None
    if role == "tool":
        r = results[0]
        if len(results) != 1 or text or not isinstance(r, dict) or not isinstance(r.get("content"), str) \
                or not isinstance(r.get("tool_call_id"), str):
            raise InvalidInput("a tool message holds one tool_result {tool_call_id: string, content: string} and no text")
        if not MISTRAL_CALL_ID.fullmatch(r["tool_call_id"]):
            raise InvalidInput("a tool result's tool_call_id is 9 of a-z, A-Z and 0-9")
        result = (r["tool_call_id"], r["content"])
    return role, texts, calls, result, prefix


def mistral_instruct_texts(messages: Sequence[dict], tools: Optional[Sequence[dict]] = None, version: int = 3) -> Tuple[List[str], int]:
    """A conversation as mistral_common 1.11's InstructTokenizerV3 (version 3) or InstructTokenizerV7 (version 7) encodes it
    (encode_chat_completion with its request validator in its default mode and its request normalizer): (the ordinary texts in
    order, the number of control tokens).  The token count is the control tokens plus the sum of the texts' token counts
    (Tekkenizer.encode(text, bos=False, eos=False), each text on its own).  JSON below is json.dumps(..., ensure_ascii=False):
    ", " and ": " between items, key order kept, non-ASCII as is.  Version 3:
      - a message's text is its text parts joined with "\n\n"; other parts (images ...) are not counted here;
      - an assistant message holds text or tool_call parts {id, name, arguments}; a tool message holds one tool_result part
        {tool_call_id, content};
      - system messages leave the sequence; the non-empty system texts, joined with "\n\n", are the system prompt;
      - consecutive user (or assistant) messages merge into one, their texts joined with "\n\n" and their tool calls listed in
        order (a system message between two messages of one role keeps them apart); tool messages stay one each;
      - when the first message left is not a user message, an empty user message goes first;
      - <s>; then per message: user -> [INST] text [/INST], where the LAST user message's text is the system prompt + "\n\n" +
        its text (when there is a system prompt), and [AVAILABLE_TOOLS] the tools [/AVAILABLE_TOOLS] go before that [INST]
        (when there are tools: a list of {"type": "function", "function": {"name", "description", "parameters"}});
        assistant -> its text without trailing spaces, or [TOOL_CALLS] the list of its calls {"name", "arguments", "id"}; then
        </s>; tool -> [TOOL_RESULTS] {"content": the result, "call_id": its id} [/TOOL_RESULTS], the result being the JSON value
        its content parses to, else the content as a string ("" is {}).
    What mistral_common refuses raises InvalidInput: no message; one message that is not a user or system message; an assistant
    message last; a system message after an assistant or tool message, a tool message after a system or user message; an
    assistant message without text and tool calls, or with both (also once merged); an assistant message while the tool calls of
    the one before it do not have exactly one tool message each (the first message is not checked); a tool name or tool-call name
    that is not 1-64 of [a-zA-Z0-9_-], a call id that is not 9 of [a-zA-Z0-9] (a call id may be "null": it is then not printed);
    a tool that is not a unified one.  A tool's parameters are taken as a valid JSON Schema (mistral_common checks them against
    Draft 7; this does not).

    Version 7 (MistralRequestValidatorV5, InstructRequestNormalizerV7) keeps the roles that may follow each role, the names, the
    call ids, the count of tool messages and the calls' JSON, and differs in this:
      - each system message stays where it is, as [SYSTEM_PROMPT] its text [/SYSTEM_PROMPT] (an empty one too); system messages
        in a row stay one each; nothing joins the user messages, and no empty user message goes first;
      - consecutive user (or assistant) messages merge into one whose text is all their text parts joined with "\n\n" (a message
        without text parts adds nothing);
      - an assistant message may hold text and tool calls: its turn is its text without trailing spaces, then [TOOL_CALLS] the
        list of its calls, then </s>; a turn with neither is refused (a message with neither passes when merged with one that
        has either);
      - tool -> [TOOL_RESULTS] call id [TOOL_CONTENT] content [/TOOL_RESULTS], the content being the JSON value it parses to
        written again, else the text as given ("" is "{}");
      - the last message may be an assistant message with "prefix": true, the start of the reply: its turn has no </s>.  prefix on
        any other message is refused;
      - the tools go before the last user message's [INST]; a conversation without a user message does not show them.

    Other versions are refused; mistral_instruct_texts_v11 gives versions 11 and 13."""
    if version not in (3, 7):
        raise InvalidInput("mistral_instruct_texts counts instruct versions 3 and 7 (11 and 13: mistral_instruct_texts_v11), "
                           "not %r" % (version,))
    return _mistral_texts(messages, tools, version)


def mistral_instruct_texts_v11(messages: Sequence[dict], tools: Optional[Sequence[dict]] = None, version: int = 11) -> Tuple[List[str], int]:
    """mistral_instruct_texts for mistral_common 1.11's InstructTokenizerV11 (version 11) or InstructTokenizerV13 (version 13),
    both with MistralRequestValidatorV13 (default mode) and InstructRequestNormalizerV13: (the ordinary texts in order, the
    number of control tokens).  They are version 7, except:
      - V11: each call of an assistant turn is [TOOL_CALLS] its name, then [CALL_ID] its id when the id is not "null", then
        [ARGS] its arguments' JSON (no list);
      - V13: as V11 without [CALL_ID] and its id, and a call's id is required ("null" is refused); a tool result is
        [TOOL_RESULTS] content [/TOOL_RESULTS] (no call id, no [TOOL_CONTENT]); the tools go before the FIRST user message;
      - both: the tool messages after an assistant message answer its calls by id: a result whose id is not among the ids of
        the calls of the assistant message before it, or answers one of them twice, is refused, and so are two calls of one
        message with one id; an assistant message while the calls of the one before it do not all have their result is refused
        (the first message is not checked).  The normalizer puts each run of results in the order of their calls, which does not
        change the count.
    Other versions are refused (3 and 7: mistral_instruct_texts)."""
    if version not in (11, 13):
        raise InvalidInput("mistral_instruct_texts_v11 counts instruct versions 11 and 13 (3 and 7: mistral_instruct_texts), "
                           "not %r" % (version,))
    return _mistral_texts(messages, tools, version)


def _mistral_texts(messages: Sequence[dict], tools: Optional[Sequence[dict]], version: int) -> Tuple[List[str], int]:
    """mistral_instruct_texts (version 3 or 7) and mistral_instruct_texts_v11 (version 11 or 13), on a version they take"""
    tool_defs = _mistral_tools(tools or ())
    if not messages:
        raise InvalidInput("a conversation for the mistral template has at least one message")
    msgs = [_mistral_message(m, version) for m in messages]
    roles = [m[0] for m in msgs]
    if any(m[4] for m in msgs[:-1]):
        raise InvalidInput("an assistant message with prefix is the last message")
    if len(roles) == 1 and roles[0] not in ("user", "system"):
        raise InvalidInput("a conversation of one message for the mistral template is a user or system message")
    if len(roles) > 1 and roles[-1] == "assistant" and not msgs[-1][4]:
        raise InvalidInput("a conversation for the mistral template ends with a user or tool message" +
                           (" or an assistant message with prefix" if version >= 7 else ""))
    for prev, role in zip(roles, roles[1:]):
        if role not in MISTRAL_NEXT_ROLES[prev]:
            raise InvalidInput("a message of role %r follows one of role %r" % (role, prev))
    if version >= 11:
        _check_mistral_call_ids(msgs)
    else:
        pending = 0                     # tool messages the last tool-calling assistant message still waits for
        for role, _, calls, _, _ in msgs[1:]:
            if role == "tool":
                pending -= 1
            elif role == "assistant":
                if pending:
                    raise InvalidInput("an assistant message follows tool calls without exactly one tool message each")
                pending = len(calls)
    if version >= 7:
        return _mistral_v7_texts(msgs, tool_defs, version)
    system = "\n\n".join(t for t in ("\n\n".join(parts) for role, parts, _, _, _ in msgs if role == "system") if t)
    turns: List[list] = []              # [role, text, calls, result] after merging
    prev = None
    for role, parts, calls, result, _ in msgs:
        text = "\n\n".join(parts)
        if role in ("user", "assistant") and role == prev:
            if not calls:               # (a message with tool calls has no text to merge)
                turns[-1][1] += "\n\n" + text
            turns[-1][2] += calls
            if turns[-1][1] and turns[-1][2]:
                raise InvalidInput("merged assistant messages hold both text and tool calls")
        elif role != "system":
            turns.append([role, text, list(calls), result])
        prev = role
    if not turns or turns[0][0] != "user":
        turns.insert(0, ["user", "", [], None])
    last_user = max(i for i, t in enumerate(turns) if t[0] == "user")
    texts, controls = [], 1             # <s>
    for i, (role, t, calls, result) in enumerate(turns):
        if role == "user":
            if i == last_user and tool_defs:
                texts.append(_mistral_json(tool_defs))
                controls += 2           # [AVAILABLE_TOOLS] [/AVAILABLE_TOOLS]
            texts.append(system + "\n\n" + t if i == last_user and system else t)
            controls += 2               # [INST] [/INST]
        elif role == "assistant":
            texts.append(_mistral_json(calls) if calls else t.rstrip(" "))
            controls += 2 if calls else 1   # ([TOOL_CALLS]) </s>
        else:
            call_id, content = result
            texts.append(_mistral_json({"content": _mistral_tool_content(content), "call_id": call_id}))
            controls += 2               # [TOOL_RESULTS] [/TOOL_RESULTS]
    return texts, controls


def _check_mistral_call_ids(msgs: Sequence[tuple]) -> None:
    """MistralRequestValidatorV13's check of tool results against the calls they answer (instruct V11 and V13), on messages
    _mistral_message read: the first message is not checked"""
    expected, answered = set(), set()   # the call ids of the last assistant message, the ones its tool messages answered
    for role, _, calls, result, _ in msgs[1:]:
        if role == "tool":
            if result[0] in answered:
                raise InvalidInput("two tool results answer the call %r" % result[0])
            if result[0] not in expected:
                raise InvalidInput("a tool result answers %r, not a call of the assistant message before it" % result[0])
            answered.add(result[0])
        elif role == "assistant":
            if len(answered) != len(expected):
                raise InvalidInput("an assistant message follows tool calls without a tool result each")
            expected, answered = set(), set()
            for c in calls:
                if c.get("id", "null") in expected:
                    raise InvalidInput("two tool calls of one assistant message have the id %r" % c.get("id", "null"))
                expected.add(c.get("id", "null"))


def _mistral_v7_texts(msgs: Sequence[tuple], tool_defs: List[dict], version: int) -> Tuple[List[str], int]:
    """mistral_instruct_texts under version 7, 11 or 13, on messages _mistral_message read and mistral_instruct_texts checked"""
    turns: List[list] = []              # [role, text parts, calls, result] after merging
    prev = None
    for role, parts, calls, result, _ in msgs:
        if role in ("user", "assistant") and role == prev:
            turns[-1][1] += parts
            turns[-1][2] += calls
        else:
            turns.append([role, list(parts), list(calls), result])
        prev = role
    users = [i for i, t in enumerate(turns) if t[0] == "user"]
    tools_at = (users[0] if version == 13 else users[-1]) if users else -1
    prefix = msgs[-1][4]
    texts, controls = [], 1             # <s>
    for i, (role, parts, calls, result) in enumerate(turns):
        text = "\n\n".join(parts)
        if role == "system":
            texts.append(text)
            controls += 2               # [SYSTEM_PROMPT] [/SYSTEM_PROMPT]
        elif role == "user":
            if i == tools_at and tool_defs:
                texts.append(_mistral_json(tool_defs))
                controls += 2           # [AVAILABLE_TOOLS] [/AVAILABLE_TOOLS]
            texts.append(text)
            controls += 2               # [INST] [/INST]
        elif role == "assistant":
            if not text and not calls:
                raise InvalidInput("an assistant message without text or tool calls (also once merged)")
            texts.append(text.rstrip(" "))
            if calls and version == 7:
                texts.append(_mistral_json(calls))
                controls += 1           # [TOOL_CALLS]
            for c in calls if version >= 11 else ():
                texts.append(c["name"])
                if version == 11 and "id" in c:
                    texts.append(c["id"])
                    controls += 1       # [CALL_ID]
                texts.append(_mistral_json(c["arguments"]))
                controls += 2           # [TOOL_CALLS] [ARGS]
            if not (prefix and i == len(turns) - 1):
                controls += 1           # </s>
        elif version == 13:
            texts.append(_mistral_normalized_content(result[1]))
            controls += 2               # [TOOL_RESULTS] [/TOOL_RESULTS]
        else:
            call_id, content = result
            texts += [call_id, _mistral_normalized_content(content)]
            controls += 3               # [TOOL_RESULTS] [TOOL_CONTENT] [/TOOL_RESULTS]
    return texts, controls


# --------------------------------------------------------------------------- plugin trait
class TokenizerPluginClient:
    """plugin API (scoped in ClientHub by GTS instance id)"""

    def encode_batch(self, ctx: SecurityContext, req: EncodeBatchRequest) -> EncodeBatchResponse:
        raise NotImplementedError

    def count_tokens(self, ctx: SecurityContext, req: CountTokensRequest) -> np.ndarray:
        raise NotImplementedError

    def decode_batch(self, ctx: SecurityContext, req: "DecodeBatchRequest") -> "DecodeBatchResponse":
        raise NotImplementedError

    def encode_batch_lossy(self, ctx: SecurityContext, req: EncodeBatchRequest) -> EncodeBatchResponse:
        """encode_batch of a request with errors="replace": every prompt encoded as bytes.decode("utf-8", "replace") would be, and
        EncodeBatchResponse.replaced.  This default works on any plugin: it repairs every prompt on the host (repair_utf8) and
        encodes the repaired batch strictly."""
        _errors(req)
        data, offs, replaced = repair_utf8(req.bytes, req.offsets)
        r = self.encode_batch(ctx, EncodeBatchRequest(req.vocab, data, offs, req.vocabs_per_prompt, req.vocab_index))
        return EncodeBatchResponse(r.ids, r.offsets, r.counts, replaced=replaced)

    def count_tokens_lossy(self, ctx: SecurityContext, req: CountTokensRequest) -> np.ndarray:
        """count_tokens of a request with errors="replace"; this default repairs on the host, as encode_batch_lossy"""
        _errors(req)
        data, offs, _ = repair_utf8(req.bytes, req.offsets)
        return self.count_tokens(ctx, CountTokensRequest(req.vocab, data, offs, req.vocabs_per_prompt, req.vocab_index))

    def encode_batch_special(self, ctx: SecurityContext, req: EncodeBatchRequest, special_tokens: dict, allowed: set,
                             disallowed: set) -> EncodeBatchResponse:
        """tiktoken's `Encoding.encode(text, allowed_special=allowed, disallowed_special=disallowed)` for every prompt of `req`.
        special_tokens: {"<|endoftext|>": 100257, ...}; allowed / disallowed: sets of token strings (allowed ones have an id).
        A prompt that holds a disallowed token raises InvalidInput.  This default works on any plugin: it cuts the texts on the
        host at every occurrence of an allowed token (leftmost first, the longest at a position), encodes the stretches between
        them with encode_batch -- all stretches of all prompts in ONE batch -- and puts the special ids back in."""
        import re
        n = len(req.offsets) - 1
        try:
            texts = [bytes(req.bytes[int(req.offsets[i]):int(req.offsets[i + 1])]).decode("utf-8") for i in range(n)]
        except UnicodeDecodeError as e:
            raise InvalidInput("a prompt holds malformed UTF-8") from e
        if disallowed:
            bad = re.compile("|".join(re.escape(t) for t in sorted(disallowed, key=len, reverse=True)))
            for t in texts:
                m = bad.search(t)
                if m:
                    raise InvalidInput("the text holds the special token %r, which is not allowed here" % m.group())
        cut = re.compile("|".join(re.escape(t) for t in sorted(allowed, key=len, reverse=True))) if allowed else None
        plan, stretches, refs = [], [], []    # per text: list of ("s", stretch index) | ("t", special id)
        per = req.vocabs_per_prompt
        if per is not None and req.vocab_index is not None:
            per = [per[int(k)] for k in req.vocab_index]
        for i, t in enumerate(texts):
            steps, pos = [], 0
            for m in (cut.finditer(t) if cut else ()):
                if m.start() > pos:
                    steps.append(("s", len(stretches))); stretches.append(t[pos:m.start()]); refs.append(None if per is None else per[i])
                steps.append(("t", int(special_tokens[m.group()])))
                pos = m.end()
            if pos < len(t):
                steps.append(("s", len(stretches))); stretches.append(t[pos:]); refs.append(None if per is None else per[i])
            plan.append(steps)
        enc = []
        if stretches:
            data, offs = pack_texts(stretches)
            r = self.encode_batch(ctx, EncodeBatchRequest(req.vocab, data, offs, None if per is None else refs))
            enc = [r.ids[int(r.offsets[i]):int(r.offsets[i + 1])] for i in range(len(stretches))]
        parts = []
        for steps in plan:
            p = [enc[i] if kind == "s" else np.array([i], dtype=np.uint32) for kind, i in steps]
            parts.append(np.concatenate(p).astype(np.uint32) if p else np.zeros(0, dtype=np.uint32))
        counts = np.array([len(p) for p in parts], dtype=np.uint32)
        offsets = np.zeros(n + 1, dtype=np.uint64)
        offsets[1:] = np.cumsum(counts, dtype=np.uint64)
        ids = np.concatenate(parts).astype(np.uint32) if parts else np.zeros(0, dtype=np.uint32)
        return EncodeBatchResponse(ids, offsets, counts)

    def truncate_batch(self, ctx: SecurityContext, req: EncodeBatchRequest, budgets, keep: str = "head") -> TruncateBatchResponse:
        """Cut every prompt of `req` to a token budget (an int, or one per prompt): keep its first ("head") or last ("tail")
        min(budget, count) tokens of the encoding of the whole prompt, cut at a character boundary -- include/cfbpe.h,
        cfbpe_truncate_batch.  This default works on any plugin: encode_batch with token starts, then the cut on the host."""
        tail = _truncate_mode(keep) == N.TRUNCATE_TAIL
        n = len(req.offsets) - 1
        bud = _budgets(budgets, n)
        r = self.encode_batch(ctx, EncodeBatchRequest(req.vocab, req.bytes, req.offsets, req.vocabs_per_prompt, req.vocab_index,
                                                      with_starts=True))
        if r.starts is None:
            raise ServiceUnavailable("the tokenizer plugin does not return token starts")
        cut, kept = truncate_cuts(req.bytes, req.offsets, r.offsets, r.starts, bud, tail)
        return TruncateBatchResponse(cut, kept, np.asarray(r.counts[:n], dtype=np.uint32))

    def encode_batch_unit_starts(self, ctx: SecurityContext, req: EncodeBatchRequest) -> EncodeBatchResponse:
        """encode_batch with every token's start in req.starts_unit and every prompt's length in it (EncodeBatchResponse.lens) --
        include/cfbpe.h, cfbpe_encode_batch_char_starts.  This default works on any plugin that returns byte starts: encode_batch
        with byte starts, then unit_starts on the host."""
        unit = _starts_unit(req.starts_unit)
        r = self.encode_batch(ctx, EncodeBatchRequest(req.vocab, req.bytes, req.offsets, req.vocabs_per_prompt, req.vocab_index,
                                                      with_starts=True))
        if r.starts is None:
            raise ServiceUnavailable("the tokenizer plugin does not return token starts")
        starts, lens = unit_starts(req.bytes, req.offsets, r.offsets, r.starts, unit)
        return EncodeBatchResponse(r.ids, r.offsets, r.counts, starts, lens)

    def chunk_batch(self, ctx: SecurityContext, req: EncodeBatchRequest, chunk_tokens: int, overlap_tokens: int = 0) -> ChunkBatchResponse:
        """Cut every prompt of `req` into chunks of at most chunk_tokens tokens that overlap by overlap_tokens, at character
        boundaries of the whole prompt's encoding -- include/cfbpe.h, cfbpe_chunk_batch.  This default works on any plugin:
        encode_batch with token starts, then the cuts on the host."""
        n_tok, overlap = _chunk_args(chunk_tokens, overlap_tokens)
        n = len(req.offsets) - 1
        r = self.encode_batch(ctx, EncodeBatchRequest(req.vocab, req.bytes, req.offsets, req.vocabs_per_prompt, req.vocab_index,
                                                      with_starts=True))
        if r.starts is None:
            raise ServiceUnavailable("the tokenizer plugin does not return token starts")
        spans, coffs = chunk_spans(req.bytes, req.offsets, r.offsets, r.starts, n_tok, overlap)
        return ChunkBatchResponse(spans, coffs, np.asarray(r.counts[:n], dtype=np.uint32))


GTS_PLUGIN_SCHEMA = "gts.x.core.modkit.plugin.v1~x.llmgw.tokenizer.plugin.v1~"


@dataclass
class PluginInstance:
    """BaseModkitPluginV1 content (libs/modkit/src/gts/plugin.rs:12-17)"""
    id: str
    vendor: str
    priority: int
    properties: dict = field(default_factory=dict)


class ClientHub:
    """type+scope keyed registry (libs/modkit/src/client_hub.rs:142-234), reduced to what the path needs"""

    def __init__(self):
        self._lock = threading.RLock()
        self._scoped: Dict[tuple, object] = {}

    def register_scoped(self, iface: type, scope: str, client: object) -> None:
        with self._lock:
            self._scoped[(iface, scope)] = client

    def get_scoped(self, iface: type, scope: str):
        with self._lock:
            try:
                return self._scoped[(iface, scope)]
            except KeyError:
                raise KeyError("ScopedNotFound(%s, %s)" % (iface.__name__, scope)) from None

    def try_get_scoped(self, iface: type, scope: str):
        with self._lock:
            return self._scoped.get((iface, scope))


def choose_plugin_instance(vendor: str, instances: Sequence[PluginInstance]) -> str:
    """vendor match, lowest priority wins, first wins ties (libs/modkit/src/plugins/mod.rs:136-191)"""
    best = None
    for inst in instances:
        if inst.vendor != vendor:
            continue
        if best is None or inst.priority < best.priority:
            best = inst
    if best is None:
        raise NoPluginAvailable("no tokenizer plugin for vendor %r" % vendor)
    return best.id


# --------------------------------------------------------------------------- the GPU plugin
class GpuBpeTokenizerPlugin(TokenizerPluginClient):
    """`gpu-bpe-tokenizer-plugin`: owns one device context; init = Module::init of the plugin
    (cuda context, vocab load -> device tables; multi-GPU broadcast is in cfbpe.dist)."""

    VENDOR = "cyberfabric"

    def __init__(self, device: int = 0, vocab_names: Sequence[str] = ("cl100k_base",), max_batch_bytes: int = 0,
                 max_prompts: int = 0, priority: int = 10, import_blobs: Optional[Dict[str, np.ndarray]] = None,
                 allow_stand_in: bool = False, devices: Optional[Sequence[int]] = None, n_workspaces: int = 1):
        """allow_stand_in: see cfbpe.vocabs.resolve -- benchmarks and tests only; a production plugin fails with VocabNotFound
        when a real rank file is missing instead of counting tokens with another vocabulary"""
        self.allow_stand_in = allow_stand_in
        self.max_batch_bytes = int(max_batch_bytes) if max_batch_bytes else 256 << 20     # cfbpe_create's defaults
        self.max_prompts = int(max_prompts) if max_prompts else 1 << 20
        try:
            self.ctx = N.Context(device, max_batch_bytes, max_prompts, devices=devices, n_workspaces=n_workspaces)
        except N.NativeError as e:
            raise _map_native(e) from e
        self._slot: Dict[str, int] = {}
        self._specials: Dict[int, dict] = {}      # slot -> the special tokens registered on it ({str: id}, in registration order)
        self.resolved: Dict[str, V.ResolvedVocab] = {}
        self._lock = threading.Lock()
        self.instance = PluginInstance(
            id=GTS_PLUGIN_SCHEMA + "cyberfabric.gpu_bpe.b200.v1", vendor=self.VENDOR, priority=priority,
            properties={"devices": list(devices) if devices else [device], "workspaces": n_workspaces, "vocabs": {}})
        for name in vocab_names:
            self.load_vocab(name, None if import_blobs is None else import_blobs.get(name))

    # -- vocab management (model-registry vocab loader side)
    def load_vocab(self, name: str, blob: Optional[np.ndarray] = None) -> int:
        with self._lock:
            if name in self._slot:
                return self._slot[name]
            slot = len(self._slot)
            if slot >= N.MAX_VOCABS:
                raise InvalidInput("too many vocabularies loaded")
            try:
                rv = V.resolve(name, self.allow_stand_in)
            except V.VocabUnavailable as e:
                raise VocabNotFound(str(e)) from e
            try:
                if blob is not None:
                    self.ctx.vocab_import(slot, blob)
                else:
                    self.ctx.vocab_load(slot, rv.file_bytes, rv.spec.fmt, rv.pattern_id, rv.max_ranks)
                if rv.spec.id_base:         # the model's own ids: control tokens first, the ordinary tokens after them
                    self.ctx.vocab_set_id_base(slot, rv.spec.id_base)
                    self.ctx.vocab_set_specials(slot, rv.control_tokens)
                    self._specials[slot] = dict(rv.control_tokens)
            except N.NativeError as e:
                raise _map_native(e) from e
            self._slot[name] = slot
            self.resolved[name] = rv
            # what a registry / operator sees about this instance: which file each vocabulary really is
            self.instance.properties["vocabs"][name] = {"slot": slot, "label": rv.label, "stand_in": rv.stand_in, "sha256": rv.sha256}
            return slot

    def export_vocab(self, name: str) -> np.ndarray:
        return self.ctx.vocab_export(self._slot[name])

    def _resolve_slot(self, ref: VocabRef) -> int:
        name = ref.name
        if name not in self._slot and name in V.MODEL_VOCABS:
            name = V.MODEL_VOCABS[name]
        if name not in self._slot:
            raise VocabNotFound("vocab %r is not loaded on this plugin" % ref.name)
        return self._slot[name]

    def _vocab_ids(self, req) -> Optional[np.ndarray]:
        n = len(req.offsets) - 1
        if req.vocabs_per_prompt is None:
            slot = self._resolve_slot(req.vocab)
            return None if slot == 0 else np.full(max(n, 1), slot, dtype=np.uint8)
        idx = getattr(req, "vocab_index", None)
        if idx is not None:         # a table of distinct vocabularies + one index per prompt
            if not isinstance(idx, np.ndarray) or idx.dtype != np.uint8 or idx.ndim != 1 or len(idx) != n:
                raise InvalidInput("vocab_index must be a uint8 array with one entry per prompt")
            lut = np.fromiter((self._resolve_slot(r) for r in req.vocabs_per_prompt), dtype=np.uint8, count=len(req.vocabs_per_prompt))
            if n and int(idx.max()) >= len(lut):
                raise InvalidInput("vocab_index names entry %d of %d vocabularies" % (int(idx.max()), len(lut)))
            return lut[idx] if n else np.zeros(1, dtype=np.uint8)
        if len(req.vocabs_per_prompt) != n:
            raise InvalidInput("vocabs_per_prompt must name one vocab per prompt")
        memo = {}
        out = np.empty(max(n, 1), dtype=np.uint8)
        for i, r in enumerate(req.vocabs_per_prompt):
            k = r.name
            v = memo.get(k)
            if v is None:
                v = memo[k] = self._resolve_slot(r)
            out[i] = v
        return out

    @staticmethod
    def _check_arrays(req):
        """what the C ABI cannot check (it takes no buffer lengths): dtypes, contiguity, and that the last offset stays
        inside the byte buffer -- otherwise the upload would read past the caller's array"""
        b, o = req.bytes, req.offsets
        if not isinstance(b, np.ndarray) or not isinstance(o, np.ndarray) or b.dtype != np.uint8 or o.dtype != np.uint64 or o.ndim != 1 or len(o) < 1:
            raise InvalidInput("bytes must be uint8 and offsets uint64 with n+1 entries")
        if not b.flags.c_contiguous or not o.flags.c_contiguous or b.ndim != 1:
            raise InvalidInput("bytes and offsets must be C-contiguous 1-D arrays")
        if int(o[0]) != 0 or int(o[-1]) > b.size:
            raise InvalidInput("offsets[0] must be 0 and offsets[n] (%d) must not exceed len(bytes) (%d)" % (int(o[-1]), b.size))

    # -- TokenizerPluginClient
    def encode_batch(self, ctx: SecurityContext, req: EncodeBatchRequest, out: Optional[EncodeBatchResponse] = None) -> EncodeBatchResponse:
        if _errors(req) == "replace":
            return self.encode_batch_lossy(ctx, req, out)
        self._check_arrays(req)
        vid = self._vocab_ids(req)
        unit = STARTS_UNITS[_starts_unit(req.starts_unit)]
        try:
            if req.with_starts and unit is not None:
                ids, starts, offs, counts, lens = self.ctx.encode_batch_char_starts(
                    req.bytes, req.offsets, unit, vid,
                    None if out is None else out.ids, None if out is None else out.starts,
                    None if out is None else out.offsets, None if out is None else out.counts, None if out is None else out.lens)
                return EncodeBatchResponse(ids, offs, counts, starts, lens)
            if req.with_starts:
                ids, starts, offs, counts = self.ctx.encode_batch_starts(
                    req.bytes, req.offsets, vid,
                    None if out is None else out.ids, None if out is None else out.starts,
                    None if out is None else out.offsets, None if out is None else out.counts)
                return EncodeBatchResponse(ids, offs, counts, starts)
            ids, offs, counts = self.ctx.encode_batch(
                req.bytes, req.offsets, vid,
                None if out is None else out.ids, None if out is None else out.offsets,
                None if out is None else out.counts)
        except N.NativeError as e:
            raise _map_native(e) from e
        return EncodeBatchResponse(ids, offs, counts)

    def encode_batch_unit_starts(self, ctx: SecurityContext, req: EncodeBatchRequest) -> EncodeBatchResponse:
        """the device path (cfbpe_encode_batch_char_starts): the unit starts are computed where the ids and byte starts are"""
        if req.starts_unit == "byte":
            return super().encode_batch_unit_starts(ctx, req)
        return self.encode_batch(ctx, EncodeBatchRequest(req.vocab, req.bytes, req.offsets, req.vocabs_per_prompt, req.vocab_index,
                                                         with_starts=True, starts_unit=req.starts_unit))

    def count_tokens(self, ctx: SecurityContext, req: CountTokensRequest, out_counts: Optional[np.ndarray] = None) -> np.ndarray:
        if _errors(req) == "replace":
            return self.count_tokens_lossy(ctx, req, out_counts)
        self._check_arrays(req)
        vid = self._vocab_ids(req)
        try:
            return self.ctx.count_batch(req.bytes, req.offsets, vid, out_counts)
        except N.NativeError as e:
            raise _map_native(e) from e

    def encode_batch_lossy(self, ctx: SecurityContext, req: EncodeBatchRequest, out: Optional[EncodeBatchResponse] = None) -> EncodeBatchResponse:
        """the device path (cfbpe_encode_batch_lossy): the bytes are checked, and repaired when they must be, on the device"""
        _errors(req)
        self._check_arrays(req)
        vid = self._vocab_ids(req)
        try:
            ids, offs, counts, replaced = self.ctx.encode_batch_lossy(
                req.bytes, req.offsets, vid, None if out is None else out.ids, None if out is None else out.offsets,
                None if out is None else out.counts, None if out is None else out.replaced)
        except N.NativeError as e:
            raise _map_native(e) from e
        return EncodeBatchResponse(ids, offs, counts, replaced=replaced)

    def count_tokens_lossy(self, ctx: SecurityContext, req: CountTokensRequest, out_counts: Optional[np.ndarray] = None) -> np.ndarray:
        """the device path (cfbpe_encode_batch_lossy without ids)"""
        _errors(req)
        self._check_arrays(req)
        vid = self._vocab_ids(req)
        try:
            return self.ctx.encode_batch_lossy(req.bytes, req.offsets, vid, out_counts=out_counts, counts_only=True)[2]
        except N.NativeError as e:
            raise _map_native(e) from e

    def decode_batch(self, ctx: SecurityContext, req: DecodeBatchRequest) -> DecodeBatchResponse:
        if req.ids.dtype != np.uint32 or req.offsets.dtype != np.uint64 or len(req.offsets) < 1:
            raise InvalidInput("ids must be uint32 and offsets uint64 with n+1 entries")
        if not req.ids.flags.c_contiguous or not req.offsets.flags.c_contiguous or int(req.offsets[-1]) > req.ids.size:
            raise InvalidInput("offsets[n] must not exceed len(ids); arrays must be C-contiguous")
        vid = self._vocab_ids(req)
        try:
            out, offs = self.ctx.decode_batch(req.ids, req.offsets, vid)
        except N.NativeError as e:
            raise _map_native(e) from e
        return DecodeBatchResponse(out, offs)

    def encode_batch_special(self, ctx: SecurityContext, req: EncodeBatchRequest, special_tokens: dict, allowed: set,
                             disallowed: set) -> EncodeBatchResponse:
        """the device path (cfbpe_encode_batch_special): the scan, the cut and the splice run as CUDA kernels.  The caller's
        special_tokens are registered on every slot the request uses when they differ from what the slot holds."""
        if not set(disallowed) <= set(special_tokens):      # a disallowed string that is no special token: only the host cut knows it
            return super().encode_batch_special(ctx, req, special_tokens, allowed, disallowed)
        self._check_arrays(req)
        vid = self._vocab_ids(req)
        n = len(req.offsets) - 1
        slots = [self._resolve_slot(req.vocab)] if vid is None else sorted(set(int(v) for v in vid[:n]))
        want = {str(k): int(v) for k, v in special_tokens.items()}
        modes = [None] * N.MAX_VOCABS
        m = np.array([N.SPECIAL_DISALLOW if t in disallowed else (N.SPECIAL_ALLOW if t in allowed else N.SPECIAL_ORDINARY) for t in want],
                     dtype=np.uint8)
        try:
            with self._lock:
                for slot in slots:
                    if list(self._specials.get(slot, {}).items()) != list(want.items()):      # (the order gives the mode indices)
                        self.ctx.vocab_set_specials(slot, want)
                        self._specials[slot] = dict(want)
                    modes[slot] = m
                ids, offs, counts = self.ctx.encode_batch_special(req.bytes, req.offsets, vid, modes)
        except N.NativeError as e:
            raise _map_native(e) from e
        return EncodeBatchResponse(ids, offs, counts)

    def truncate_batch(self, ctx: SecurityContext, req: EncodeBatchRequest, budgets, keep: str = "head") -> TruncateBatchResponse:
        """the device path (cfbpe_truncate_batch): the cut is computed where the ids are; only the cuts, kept counts and counts
        come back"""
        mode = _truncate_mode(keep)
        self._check_arrays(req)
        vid = self._vocab_ids(req)
        bud = _budgets(budgets, len(req.offsets) - 1)
        try:
            cut, kept, counts = self.ctx.truncate_batch(req.bytes, req.offsets, bud, mode, vid)
        except N.NativeError as e:
            raise _map_native(e) from e
        return TruncateBatchResponse(cut, kept, counts)

    def chunk_batch(self, ctx: SecurityContext, req: EncodeBatchRequest, chunk_tokens: int, overlap_tokens: int = 0) -> ChunkBatchResponse:
        """the device path (cfbpe_chunk_batch): the chunks are cut where the ids and starts are; only the spans, chunk offsets and
        counts come back"""
        n_tok, overlap = _chunk_args(chunk_tokens, overlap_tokens)
        self._check_arrays(req)
        vid = self._vocab_ids(req)
        try:
            spans, coffs, counts = self.ctx.chunk_batch(req.bytes, req.offsets, n_tok, overlap, vid)
        except N.NativeError as e:
            raise _map_native(e) from e
        return ChunkBatchResponse(spans, coffs, counts)

    def close(self):
        self.ctx.close()


# --------------------------------------------------------------------------- gateway side
def pack_texts(texts: Sequence[str]):
    """list[str] -> (uint8 packed bytes, uint64 offsets): the packed multi-tenant prompt buffer"""
    enc = [t.encode("utf-8") for t in texts]
    offs = np.zeros(len(enc) + 1, dtype=np.uint64)
    if enc:
        offs[1:] = np.cumsum([len(e) for e in enc], dtype=np.uint64)
    data = np.frombuffer(b"".join(enc), dtype=np.uint8) if enc else np.zeros(0, dtype=np.uint8)
    return data, offs


class LlmGatewayTokenizerService:
    """`llm-gateway::tokenizer` + `llm-gateway::usage::count_tokens`: the gateway-side domain service.
    Plugin resolution is lazy and cached (libs/modkit/src/plugins/mod.rs:44-78)."""

    def __init__(self, hub: ClientHub, instances: Sequence[PluginInstance], vendor: str = GpuBpeTokenizerPlugin.VENDOR):
        self._hub, self._instances, self._vendor = hub, list(instances), vendor
        self._resolved: Optional[str] = None
        self._lock = threading.Lock()

    def _plugin(self) -> TokenizerPluginClient:
        with self._lock:
            if self._resolved is None:
                self._resolved = choose_plugin_instance(self._vendor, self._instances)
        p = self._hub.try_get_scoped(TokenizerPluginClient, self._resolved)
        if p is None:
            raise ServiceUnavailable("tokenizer plugin %s is not registered yet" % self._resolved)
        return p

    def encode(self, ctx: SecurityContext, model: str, texts: Sequence[str]) -> List[np.ndarray]:
        data, offs = pack_texts(texts)
        r = self._plugin().encode_batch(ctx, EncodeBatchRequest(VocabRef(model), data, offs))
        return [r.ids[int(r.offsets[i]):int(r.offsets[i + 1])] for i in range(len(texts))]

    def encode_with_offsets(self, ctx: SecurityContext, model: str, texts: Sequence[str], unit: str = "byte") -> List[Tuple[np.ndarray, np.ndarray]]:
        """per text: (ids, spans), spans an (n, 2) uint64 array of each token's [start, end) range in `unit`:
          "byte"       indices into text.encode("utf-8");
          "codepoint"  indices into the str (tiktoken's decode_with_offsets gives these starts; Hugging Face tokenizers' `offsets`
                       are such spans);
          "utf16"      indices into the UTF-16 code units of the text, as JavaScript, Java and C# index their strings.
        In a character unit, a token's start is that of the character that holds its first byte: byte tokens of one character
        share a start, so some spans are empty, and the spans still slice the text back into exactly itself.  Cutting a text to a
        context window or into chunks of at most N tokens is a cut at a span boundary."""
        _starts_unit(unit)
        data, offs = pack_texts(texts)
        req = EncodeBatchRequest(VocabRef(model), data, offs, with_starts=True, starts_unit=unit)
        plug = self._plugin()
        r = plug.encode_batch(ctx, req) if unit == "byte" else plug.encode_batch_unit_starts(ctx, req)
        if r.starts is None:
            raise ServiceUnavailable("the tokenizer plugin does not return token starts")
        lens = np.diff(offs) if unit == "byte" else r.lens
        out = []
        for i in range(len(texts)):
            a, b = int(r.offsets[i]), int(r.offsets[i + 1])
            st = r.starts[a:b].astype(np.uint64)
            spans = np.empty((b - a, 2), dtype=np.uint64)
            spans[:, 0] = st
            spans[:-1, 1] = st[1:]
            if b > a:
                spans[-1, 1] = int(lens[i])
            out.append((r.ids[a:b], spans))
        return out

    def truncate(self, ctx: SecurityContext, model: str, texts: Sequence[str], max_tokens, keep: str = "head") -> List[Tuple[str, int, int]]:
        """Fit texts into a context window: per text, (the kept text, its tokens, the tokens of the whole text).  max_tokens: one
        budget for all texts or one per text; keep="head" keeps the first tokens (a long document, retrieved context), "tail" the
        last ones (a chat history).  The cut is at a token boundary of the whole text's encoding, moved to a character boundary
        so that the kept text is valid UTF-8 (its token count is then one to three less than the budget).  Encoding the kept text
        again may give other tokens: BPE is not prefix-stable."""
        data, offs = pack_texts(texts)
        r = self._plugin().truncate_batch(ctx, EncodeBatchRequest(VocabRef(model), data, offs), max_tokens, keep)
        tail = _truncate_mode(keep) == N.TRUNCATE_TAIL
        out = []
        for i in range(len(texts)):
            b = data[int(offs[i]):int(offs[i + 1])].tobytes()
            c = int(r.cut[i])
            out.append(((b[c:] if tail else b[:c]).decode("utf-8"), int(r.kept[i]), int(r.counts[i])))
        return out

    def chunk(self, ctx: SecurityContext, model: str, texts: Sequence[str], max_tokens: int, overlap: int = 0) -> List[List[str]]:
        """Split texts into chunks of at most max_tokens tokens that overlap by `overlap` tokens (a RAG splitter's chunk_size /
        chunk_overlap, or an embedding endpoint's long inputs): per text, its chunk strings.  The cuts are at token boundaries of
        the whole text's encoding, moved back to character boundaries, so every chunk is valid UTF-8; with no overlap the chunks
        join back into the text.  Encoding a chunk again may give other tokens: BPE is not prefix-stable."""
        data, offs = pack_texts(texts)
        r = self._plugin().chunk_batch(ctx, EncodeBatchRequest(VocabRef(model), data, offs), max_tokens, overlap)
        out = []
        for i in range(len(texts)):
            b = data[int(offs[i]):int(offs[i + 1])].tobytes()
            out.append([b[int(x):int(y)].decode("utf-8") for x, y in r.spans[int(r.chunk_offsets[i]):int(r.chunk_offsets[i + 1])]])
        return out

    def count_tokens(self, ctx: SecurityContext, model: str, messages: Sequence[dict]) -> Usage:
        """Usage.input_tokens of one chat request = sum of len(encode_ordinary(text)) over its
        TextContent parts (SURVEY.md 8 a4); the provider's framing on top of that: count_chat_tokens."""
        texts = [part["text"] for m in messages for part in m.get("content", []) if part.get("type") == "text"]
        if not texts:
            return Usage(0)
        data, offs = pack_texts(texts)
        counts = self._plugin().count_tokens(ctx, CountTokensRequest(VocabRef(model), data, offs))
        return Usage(int(counts.sum()))

    def count_chat_tokens(self, ctx: SecurityContext, model: str, messages: Sequence[dict], template: ChatTemplate,
                          tools: Optional[Sequence[dict]] = None) -> Usage:
        """`Usage.input_tokens` of one chat request as the provider counts it: content AND framing (ChatTemplate).
        messages: [{"role": "user", "name": optional, "content": [{"type": "text", "text": ...}, ...]}, ...]; parts that are
        not text (images ...) are priced elsewhere.  tools: the request's `tools` (schemas/tools/tool.v1), counted by the "mistral"
        kind only, which also counts tool_call and tool_result parts (mistral_instruct_texts, or mistral_instruct_texts_v11 for
        instruct versions 11 and 13);
        the other kinds refuse tools and pass over those parts.  Every stretch of text of the whole request, tool JSON included, goes to the device in ONE batch."""
        import re
        if tools and template.kind != "mistral":
            raise InvalidInput("the %r chat template does not count tools" % template.kind)
        texts: List[str] = []
        fixed = 0
        if template.kind == "overhead":
            for m in messages:
                fixed += template.tokens_per_message
                texts.append(str(m.get("role", "")))
                if m.get("name"):
                    fixed += template.tokens_per_name
                    texts.append(str(m["name"]))
                texts.extend(part["text"] for part in m.get("content", []) if part.get("type") == "text")
            fixed += template.reply_priming
        elif template.kind == "rendered":
            cut = re.compile("|".join(re.escape(t) for t in sorted(template.special_tokens, key=len, reverse=True))) if template.special_tokens else None

            def framing(text, into):          # control tokens count one each; the text between them is returned in pieces
                n, last = 0, 0
                for mt in (cut.finditer(text) if cut else ()):
                    into.append(text[last:mt.start()]); last = mt.end(); n += 1
                into.append(text[last:])
                return n
            # a stretch of ordinary text runs from one control token to the next: framing text and content are tokenised TOGETHER
            # (the pre-tokenizer may join the framing's trailing line breaks with the content's leading spaces)
            run: List[str] = [""]
            def feed_framing(text):
                nonlocal fixed
                pieces: List[str] = []
                fixed += framing(text, pieces)
                run[-1] += pieces[0]
                for p in pieces[1:]:
                    run.append(p)
            feed_framing(template.bos)
            for m in messages:
                feed_framing(template.message_prefix.format(role=m.get("role", "")))
                run[-1] += "".join(part["text"] for part in m.get("content", []) if part.get("type") == "text")
                feed_framing(template.message_suffix)
            feed_framing(template.generation_prompt)
            texts = [t for t in run if t]
        elif template.kind == "mistral":
            texts_of = mistral_instruct_texts_v11 if template.instruct_version in (11, 13) else mistral_instruct_texts
            texts, fixed = texts_of(messages, tools, template.instruct_version)
        else:
            raise InvalidInput("unknown chat template kind %r" % template.kind)
        texts = [t for t in texts if t]
        if not texts:
            return Usage(fixed)
        data, offs = pack_texts(texts)
        counts = self._plugin().count_tokens(ctx, CountTokensRequest(VocabRef(model), data, offs))
        return Usage(fixed + int(counts.sum()))

    def encode_with_special(self, ctx: SecurityContext, model: str, texts: Sequence[str], special_tokens: dict,
                            allowed_special=(), disallowed_special="all") -> List[np.ndarray]:
        """tiktoken's `Encoding.encode(text, allowed_special=..., disallowed_special=...)` (SURVEY.md section 8(f) item 2):
        the text is cut at every occurrence of an allowed special token (leftmost first), the stretches between them go
        through encode_ordinary -- all stretches of all texts in ONE plugin batch -- and the special ids are put back in.
        special_tokens: {"<|endoftext|>": 100257, ...}; allowed / disallowed: "all" or a set of token strings; a text
        that holds a disallowed special token raises InvalidInput (tiktoken raises ValueError).  Defaults as tiktoken's:
        nothing allowed, everything disallowed -- user text that spells a control token is refused, not turned into one.
        The work is the plugin's encode_batch_special: on the GPU plugin the scan, cut and splice run on the device; the trait's
        default cuts on the host."""
        allowed = set(special_tokens) if allowed_special == "all" else set(allowed_special)
        disallowed = (set(special_tokens) - allowed) if disallowed_special == "all" else set(disallowed_special)
        unknown = allowed - set(special_tokens)
        if unknown:
            raise InvalidInput("allowed special tokens without an id: %s" % sorted(unknown))
        data, offs = pack_texts(texts)
        r = self._plugin().encode_batch_special(ctx, EncodeBatchRequest(VocabRef(model), data, offs), special_tokens, allowed, disallowed)
        return [r.ids[int(r.offsets[i]):int(r.offsets[i + 1])] for i in range(len(texts))]

    def check_budget(self, ctx: SecurityContext, model: str, messages: Sequence[dict], remaining_tokens: int) -> bool:
        """pre-call estimate used by check_budget (modules/llm-gateway/docs/DESIGN.md:833-855)"""
        return self.count_tokens(ctx, model, messages).input_tokens <= remaining_tokens


# --------------------------------------------------------------------------- micro-batcher (SURVEY.md section 8(f) item 4)
class CountTokensMicroBatcher:
    """Coalesces concurrent count_tokens calls (one chat request each, a few KB) into GPU-sized batches.

    The gateway's request handlers call `count(ctx, model, texts)` from many threads (tokio tasks behind spawn_blocking in the
    Rust host); a single worker drains the queue, packs what is waiting -- up to max_batch_bytes, or whatever arrived within
    max_wait_s of the first item -- into ONE CountTokensRequest with one vocabulary per prompt, and hands every caller its own
    counts.  In ModKit terms this is a `stateful` lifecycle task (docs/modkit_unified_system/08_lifecycle_stateful_tasks.md:14-58):
    start() / stop() are its hooks.  A failed batch fails exactly the calls that were in it."""

    def __init__(self, plugin: TokenizerPluginClient, max_batch_bytes: int = 8 << 20, max_wait_s: float = 0.0005, max_queue: int = 65536,
                 max_batch_prompts: int = 1 << 16):
        import queue
        # a batch never exceeds what the plugin's device context accepts (otherwise one oversize batch fails every caller in it)
        lim_b = getattr(plugin, "max_batch_bytes", None)
        lim_p = getattr(plugin, "max_prompts", None)
        self._max_bytes = int(min(max_batch_bytes, lim_b)) if lim_b else int(max_batch_bytes)
        self._max_prompts = int(min(max_batch_prompts, lim_p)) if lim_p else int(max_batch_prompts)
        self._plugin, self._max_wait = plugin, float(max_wait_s)
        self._q = queue.Queue(maxsize=max_queue)
        self._worker: Optional[threading.Thread] = None
        self._stop = threading.Event()
        self._carry = None        # an item that did not fit the batch being packed: first of the next one
        self.batches = 0          # how many plugin calls were made (for tests / metrics)
        self.items = 0

    def start(self):
        if self._worker is None:
            self._stop.clear()
            self._worker = threading.Thread(target=self._run, name="count-tokens-batcher", daemon=True)
            self._worker.start()
        return self

    def stop(self):
        self._stop.set()
        if self._worker is not None:
            self._q.put(None)
            self._worker.join()
            self._worker = None

    def count(self, ctx: SecurityContext, model: str, texts: Sequence[str], timeout: Optional[float] = None) -> np.ndarray:
        """token counts of `texts` under `model`'s vocabulary; blocks until the batch this call rode in is done.
        What can be checked per request is checked HERE, before the request joins a batch with other tenants' requests:
        an unknown model or an oversize request fails this caller only."""
        import queue
        if self._worker is None:
            raise ServiceUnavailable("the micro-batcher is not running")
        enc = [t.encode("utf-8") for t in texts]
        size = sum(len(t) for t in enc)
        if size > self._max_bytes or len(enc) > self._max_prompts:
            raise InvalidInput("the request (%d bytes, %d texts) exceeds the batch limits (%d bytes, %d prompts)"
                               % (size, len(enc), self._max_bytes, self._max_prompts))
        resolve = getattr(self._plugin, "_resolve_slot", None)
        if resolve is not None:
            resolve(VocabRef(model))          # VocabNotFound for this caller alone
        item = {"ctx": ctx, "model": model, "texts": enc, "size": size, "done": threading.Event(), "out": None, "err": None}
        try:
            self._q.put(item, timeout=timeout)
        except queue.Full:
            raise ServiceUnavailable("the count_tokens queue is full") from None
        if not item["done"].wait(timeout):
            raise ServiceUnavailable("count_tokens timed out")
        if item["err"] is not None:
            raise item["err"]
        return item["out"]

    def _run(self):
        import queue, time
        while not self._stop.is_set():
            first = self._carry if self._carry is not None else self._q.get()
            self._carry = None
            if first is None:
                break
            batch, size, n = [first], first["size"], len(first["texts"])
            deadline = time.monotonic() + self._max_wait
            while size < self._max_bytes and n < self._max_prompts:
                try:
                    nxt = self._q.get(timeout=max(0.0, deadline - time.monotonic()))
                except queue.Empty:
                    break
                if nxt is None:
                    self._stop.set()
                    break
                if size + nxt["size"] > self._max_bytes or n + len(nxt["texts"]) > self._max_prompts:
                    self._carry = nxt          # does not fit: it opens the next batch
                    break
                batch.append(nxt)
                size += nxt["size"]
                n += len(nxt["texts"])
            self._flush(batch)
        if self._carry is not None:
            self._carry["err"] = ServiceUnavailable("the micro-batcher stopped"); self._carry["done"].set(); self._carry = None
        while True:               # fail what is still queued
            try:
                it = self._q.get_nowait()
            except queue.Empty:
                break
            if it is not None:
                it["err"] = ServiceUnavailable("the micro-batcher stopped"); it["done"].set()

    def _call(self, batch):
        """one plugin call for `batch`; fills out / raises"""
        pieces = [t for it in batch for t in it["texts"]]
        if not pieces:
            for it in batch:
                it["out"] = np.zeros(0, dtype=np.uint32)
            return
        offs = np.zeros(len(pieces) + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(t) for t in pieces])
        data = np.frombuffer(b"".join(pieces), dtype=np.uint8)
        vocabs = [VocabRef(it["model"]) for it in batch for _ in it["texts"]]
        # the call carries the first request's SecurityContext only as the transport identity: counting tokens reads no
        # tenant-scoped state, and every caller gets exactly its own prompts' counts back
        counts = self._plugin.count_tokens(batch[0]["ctx"], CountTokensRequest(vocabs[0], data, offs, vocabs_per_prompt=vocabs))
        k = 0
        for it in batch:
            n = len(it["texts"])
            it["out"] = np.array(counts[k:k + n], dtype=np.uint32)
            k += n

    def _flush(self, batch):
        """A failed batch is retried request by request, so a bad request (malformed UTF-8, a model whose vocabulary was
        unloaded meanwhile) fails its own caller and nobody else's -- requests of different tenants share batches."""
        try:
            self._call(batch)
            self.batches += 1
        except TokenizerError:
            for it in batch:
                try:
                    self._call([it])
                except Exception as e:    # noqa: BLE001
                    it["err"] = e
                self.batches += 1
        except Exception as e:    # noqa: BLE001 -- not an input problem: every caller of this batch gets the error
            for it in batch:
                it["err"] = e
            self.batches += 1
        self.items += len(batch)
        for it in batch:
            it["done"].set()
