import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "cyberfabric-core_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "simt")):
    if p not in sys.path:
        sys.path.insert(0, p)

os.environ.setdefault("CFBPE_ALLOW_STAND_IN", "1")   # tests run on the stand-in vocabularies (the real OpenAI / Meta rank files are not on the box)
TEKKEN_PATH = os.path.join(ROOT, "vocabs", "tekken_240911.tiktoken")
# (pattern id, vocab size) of each benchmark slot; see cfbpe/vocabs.py
COMBOS = [(0, 100256), (1, 150000), (2, 128000), (3, 130072)]


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session")
def tekken_bytes():
    with open(TEKKEN_PATH, "rb") as f:
        return f.read()


@pytest.fixture(scope="session")
def oracle_vocabs(tekken_bytes):
    """pattern id -> OracleVocab of that slot's size"""
    from oracle import oracle
    return {pat: oracle.OracleVocab(tekken_bytes, n) for pat, n in COMBOS}


@pytest.fixture(scope="session")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "encode_golden.npz"))


def golden_cases(golden):
    tb, to = golden["text_bytes"], golden["text_offsets"]
    return [bytes(tb[int(to[i]):int(to[i + 1])]) for i in range(len(to) - 1)]


def pack(prompts):
    offs = np.zeros(len(prompts) + 1, dtype=np.uint64)
    if prompts:
        offs[1:] = np.cumsum([len(p) for p in prompts], dtype=np.uint64)
    data = np.frombuffer(b"".join(prompts), dtype=np.uint8).copy() if prompts else np.zeros(0, np.uint8)
    return data, offs
