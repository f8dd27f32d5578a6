"""Write the Mistral instruct V11 / V13 golden file from mistral_common (run where mistral_common 1.11 is installed):

  tests/golden/mistral_v11_v13.npz   every (conversation, tools) request of tests/mistral_v11_v13_ref.requests() as JSON, and the
                                     token count of encode_chat_completion of each under InstructTokenizerV7 (v7_counts), V11
                                     (v11_counts) and V13 (v13_counts) of tekken_240911.json, -1 where mistral_common refuses it
                                     (the reference of the V11 / V13 tests on a machine without mistral_common).  V11 and V13 run
                                     on the stand-in tokenizer of mistral_v11_v13_ref.live_tokenizer.

  python tools/gen_mistral_v13_data.py

It prints how many requests each version accepts, and on how many accepted by both the counts of two versions differ.
"""
import itertools
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mistral_ref  # noqa: E402
import mistral_v7_ref  # noqa: E402
import mistral_v11_v13_ref  # noqa: E402


def main():
    toks = {7: mistral_v7_ref.live_v7_tokenizer(), 11: mistral_v11_v13_ref.live_tokenizer(11), 13: mistral_v11_v13_ref.live_tokenizer(13)}
    if any(t is None for t in toks.values()):
        sys.exit("mistral_common is not installed")
    reqs = mistral_v11_v13_ref.requests()
    counts = {v: [mistral_v11_v13_ref.mistral_count(t, c, tools) for c, tools in reqs] for v, t in toks.items()}
    np.savez_compressed(
        mistral_v11_v13_ref.GOLDEN,
        requests=np.frombuffer(mistral_ref.conversations_json(reqs).encode("utf-8"), dtype=np.uint8),
        **{"v%d_counts" % v: np.asarray(n, dtype=np.int64) for v, n in counts.items()})
    print("wrote", os.path.relpath(mistral_v11_v13_ref.GOLDEN, ROOT), "with", len(reqs), "requests")
    for v, n in counts.items():
        print("V%d accepts %d" % (v, sum(w >= 0 for w in n)))
    for a, b in itertools.combinations(counts, 2):
        print("V%d and V%d differ on %d" % (a, b, sum(0 <= x != y >= 0 for x, y in zip(counts[a], counts[b]))))


if __name__ == "__main__":
    main()
