"""Write the Mistral Tekken data files from mistral_common (run where mistral_common 1.11 is installed):

  vocabs/tekken_controls.json        the 1000 control tokens of tekken_240911.json in id order (<unk> 0, <s> 1, </s> 2, [INST] 3,
                                     ... [TOOL_CONTENT] 19, <SPECIAL_20> ... <SPECIAL_999>): the v3 JSON files do not list them,
                                     mistral_common's Tekkenizer supplies them
  tests/golden/mistral_tekken.npz    Tekkenizer.encode(s, bos=False, eos=False) of tests/mistral_ref.fuzz_texts(), and the token
                                     count of encode_chat_completion of every conversation of tests/mistral_ref.conversations()
                                     (the reference of the Tekken tests on a machine without mistral_common)
  tests/golden/mistral_tools.npz     the token count of encode_chat_completion of every tool conversation of
                                     tests/mistral_tools_ref.tool_conversations() with its tools (-1: mistral_common refuses it)

  python tools/gen_mistral_data.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mistral_ref  # noqa: E402
import mistral_tools_ref  # noqa: E402


def main():
    mt = mistral_ref.live_tokenizer()
    if mt is None:
        sys.exit("mistral_common is not installed")
    tek = mt.instruct_tokenizer.tokenizer
    controls = [tek.id_to_piece(i) for i in range(tek.num_special_tokens)]
    assert len(controls) == mistral_ref.ID_BASE and controls[:5] == ["<unk>", "<s>", "</s>", "[INST]", "[/INST]"]
    with open(os.path.join(ROOT, "vocabs", "tekken_controls.json"), "w", encoding="utf-8") as f:
        json.dump(controls, f, ensure_ascii=False, indent=0)
        f.write("\n")
    texts = mistral_ref.fuzz_texts()
    ids = [tek.encode(t, bos=False, eos=False) for t in texts]
    tb = [t.encode("utf-8") for t in texts]
    convs = mistral_ref.conversations()
    np.savez_compressed(
        mistral_ref.GOLDEN,
        text_bytes=np.frombuffer(b"".join(tb), dtype=np.uint8),
        text_offsets=np.concatenate([[0], np.cumsum([len(b) for b in tb])]).astype(np.uint64),
        ids=np.concatenate([np.asarray(x, dtype=np.uint32) for x in ids]),
        id_offsets=np.concatenate([[0], np.cumsum([len(x) for x in ids])]).astype(np.uint64),
        conversations=np.frombuffer(mistral_ref.conversations_json(convs).encode("utf-8"), dtype=np.uint8),
        conversation_counts=np.asarray([mistral_ref.mistral_count(mt, c) for c in convs], dtype=np.int64))
    tool_convs = mistral_tools_ref.tool_conversations()
    np.savez_compressed(
        mistral_tools_ref.GOLDEN,
        conversations=np.frombuffer(mistral_ref.conversations_json(tool_convs).encode("utf-8"), dtype=np.uint8),
        conversation_counts=np.asarray([mistral_tools_ref.mistral_count(mt, c, t) for c, t in tool_convs], dtype=np.int64))
    print("wrote vocabs/tekken_controls.json,", os.path.relpath(mistral_ref.GOLDEN, ROOT), "and", os.path.relpath(mistral_tools_ref.GOLDEN, ROOT))


if __name__ == "__main__":
    main()
