"""Write the Mistral instruct V7 golden file from mistral_common (run where mistral_common 1.11 is installed):

  tests/golden/mistral_v7.npz    every (conversation, tools) request of tests/mistral_v7_ref.requests() as JSON, and the token count
                                 of encode_chat_completion of each under InstructTokenizerV3 (v3_counts) and InstructTokenizerV7
                                 (v7_counts) of tekken_240911.json, -1 where mistral_common refuses it (the reference of the V7
                                 tests on a machine without mistral_common)

  python tools/gen_mistral_v7_data.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mistral_ref  # noqa: E402
import mistral_v7_ref  # noqa: E402


def main():
    v3, v7 = mistral_ref.live_tokenizer(), mistral_v7_ref.live_v7_tokenizer()
    if v3 is None or v7 is None:
        sys.exit("mistral_common is not installed")
    reqs = mistral_v7_ref.requests()
    np.savez_compressed(
        mistral_v7_ref.GOLDEN,
        requests=np.frombuffer(mistral_ref.conversations_json(reqs).encode("utf-8"), dtype=np.uint8),
        v3_counts=np.asarray([mistral_v7_ref.mistral_count(v3, c, t) for c, t in reqs], dtype=np.int64),
        v7_counts=np.asarray([mistral_v7_ref.mistral_count(v7, c, t) for c, t in reqs], dtype=np.int64))
    print("wrote", os.path.relpath(mistral_v7_ref.GOLDEN, ROOT))


if __name__ == "__main__":
    main()
