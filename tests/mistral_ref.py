"""The Mistral reference of the Tekken tests: mistral_common (1.11) when it imports, else the golden file that
tools/gen_mistral_data.py wrote from it (tests/golden/mistral_tekken.npz).  Also the seeded conversations both use."""
import json
import os
import random

import numpy as np

import fuzzgen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "mistral_tekken.npz")
ID_BASE = 1000
N_RANKS = 130072


def live_tokenizer(name="tekken_240911.json"):
    """mistral_common's MistralTokenizer of one of its Tekken files, or None when mistral_common does not import"""
    try:
        import mistral_common
        from mistral_common.tokens.tokenizers.mistral import MistralTokenizer
    except ImportError:
        return None
    path = os.path.join(os.path.dirname(mistral_common.__file__), "data", name)
    return MistralTokenizer.from_file(path) if os.path.exists(path) else None


def golden():
    return np.load(GOLDEN)


def fuzz_texts():
    """mixed-script strings, and strings that spell the control tokens (ordinary text to Tekkenizer.encode)"""
    return fuzzgen.fuzz_strings(4711, 3000, max_atoms=40) + ["<s>[INST]Hi[/INST]Hello</s>", "[TOOL_CALLS] <unk><SPECIAL_999>", " [/INST] ", ""]


def conversations(seed=11, n=400):
    """n text-only conversations: every role order, merged runs, system messages anywhere, empty and space-padded texts, texts
    that spell control tokens; most end with a user message, some break mistral_common's rules of order"""
    rng = random.Random(seed)
    pool = fuzzgen.fuzz_strings(seed, 2 * n, max_atoms=10) + ["", " ", "  padded  ", "[INST]", "</s>", "\n\nafter breaks", "trailing   "]
    convs = []
    for _ in range(n):
        conv = []
        for _ in range(rng.randint(1, 7)):
            role = rng.choice(["system", "user", "user", "assistant", "assistant"])
            parts = [rng.choice(pool) for _ in range(rng.choice([1, 1, 1, 2, 3]))]
            if role == "assistant" and parts == [""]:
                parts = ["ok "]              # (an assistant message without text is refused by mistral_common and by the template)
            conv.append({"role": role, "content": [{"type": "text", "text": t} for t in parts]})
        roles = [m["role"] for m in conv if m["role"] != "system"]
        if roles and roles[-1] != "user":
            conv.append({"role": "user", "content": [{"type": "text", "text": rng.choice(pool)}]})
        if rng.random() < 0.3:
            conv.append({"role": "system", "content": [{"type": "text", "text": rng.choice(pool)}]})
        convs.append(conv)
    return convs


def mistral_count(tok, conv):
    """len(encode_chat_completion(...).tokens) of a conversation in the gateway's message form, or -1 when mistral_common refuses
    its structure"""
    from mistral_common.exceptions import InvalidMessageStructureException
    from mistral_common.protocol.instruct.messages import AssistantMessage, SystemMessage, TextChunk, UserMessage
    from mistral_common.protocol.instruct.request import ChatCompletionRequest
    kinds = {"system": SystemMessage, "user": UserMessage, "assistant": AssistantMessage}
    msgs = []
    for m in conv:
        texts = [p["text"] for p in m["content"] if p["type"] == "text"]
        content = texts[0] if len(texts) == 1 else [TextChunk(text=t) for t in texts]
        msgs.append(kinds[m["role"]](content=content))
    try:
        return len(tok.encode_chat_completion(ChatCompletionRequest(messages=msgs)).tokens)
    except InvalidMessageStructureException:
        return -1


def conversations_json(convs):
    return json.dumps(convs, ensure_ascii=False)
