"""Vocabulary registry: the "model-registry vocab loader" side of the path (SURVEY.md 8 a5).

The reference's `Model` entity has no tokenizer field (modules/model-registry/docs/PRD.md:196-209);
the mapping canonical model id `{provider_slug}::{provider_model_id}` (PRD.md:197) -> VocabSpec
lives here until the registry grows one.

Real OpenAI / Meta rank files are NOT on this box (no network; SURVEY.md F8).  A VocabSpec
therefore resolves in this order:
  1. a real rank file found in $CFBPE_VOCAB_DIR or vocabs/ whose sha256 matches the published one;
  2. ONLY when the caller opts in (allow_stand_in=True / CFBPE_ALLOW_STAND_IN=1: benchmarks and tests): the committed
     Mistral Tekken rank file truncated to the same vocabulary size, used with the requested pattern -- labelled
     `stand_in=True` so that every benchmark line and the plugin instance's properties say so.  Otherwise: VocabUnavailable.

The "tekken" vocabulary speaks raw ranks 0..n-1 of the rank file (the stand-in slot every benchmark and test uses as such).
"mistral_tekken" is the same ranks as mistral_common numbers them for Mistral's Tekken models: its 1000 control tokens first
(<unk> 0, <s> 1, </s> 2, [INST] 3, [/INST] 4, ...; vocabs/tekken_controls.json) and the ordinary token of rank r at id 1000 + r
(the plugin loads it with cfbpe_vocab_set_id_base(1000) and registers the control tokens as its special tokens).  Mistral NeMo's
tekken_240718 and Pixtral's tekken_240911 hold the same first 130072 ranks, so both models use the committed 240911 file.
Mistral's instruct-V7 models (Large 2411, Pixtral Large 2411, Small 2501 and 2503) map to "mistral_tekken" too, as a stand-in:
their own tekken.json files are not here (MODEL_TOKENIZERS labels them stand_in=True).  A model's chat template sits in its
MODEL_TOKENIZERS entry, beside its vocabulary, so the gateway never infers it from the model's name.  No model maps to the
instruct V11 or V13 templates: the repository holds no source for any model's instruct version, so they are used by name.
"""
import hashlib
import json
import os
from dataclasses import dataclass

from . import _native as N

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
VOCAB_DIR = os.path.join(_ROOT, "vocabs")
TEKKEN_FILE = os.path.join(VOCAB_DIR, "tekken_240911.tiktoken")
TEKKEN_CONTROLS_FILE = os.path.join(VOCAB_DIR, "tekken_controls.json")

# published sha256 of the OpenAI files (tiktoken_ext/openai_public.py)
KNOWN_SHA256 = {
    "cl100k_base.tiktoken": "223921b76ee99bde995b7ff738513eef100fb51d18c93597a113bcffe865b2a7",
    "o200k_base.tiktoken": "446a9538cb6c348e3516120d7c08b09f57c36495e2acfffe59a5bf8b0cfb1a2d",
}


@dataclass(frozen=True)
class VocabSpec:
    name: str
    pattern: str          # cl100k | o200k | llama3 | tekken
    n_ranks: int          # vocabulary size of the real thing
    real_file: str = ""   # file name of the real rank file, if one exists publicly
    fmt: int = N.FORMAT_TIKTOKEN
    id_base: int = 0      # id of the ordinary token of rank 0 (cfbpe_vocab_set_id_base)
    controls: str = ""    # file under vocabs/ that lists the control tokens in id order (ids 0 .. id_base - 1), if any


SPECS = {
    "cl100k_base": VocabSpec("cl100k_base", "cl100k", 100256, "cl100k_base.tiktoken"),
    "o200k_base": VocabSpec("o200k_base", "o200k", 199998, "o200k_base.tiktoken"),
    "llama3": VocabSpec("llama3", "llama3", 128000, "llama3.tiktoken"),
    "tekken": VocabSpec("tekken", "tekken", 130072, "tekken_240911.tiktoken"),
    "mistral_tekken": VocabSpec("mistral_tekken", "tekken", 130072, "tekken_240911.tiktoken", id_base=1000, controls="tekken_controls.json"),
}

@dataclass(frozen=True)
class ModelTokenizer:
    """How the gateway counts one model's requests: the vocabulary (SPECS) and the chat template (plugin.CHAT_TEMPLATES; "" when
    none is registered for the model) that frames its conversations.  stand_in: the vocabulary is not the model's own tokenizer
    file but stands in for it, so its counts are the stand-in's and may differ from the provider's."""
    vocab: str
    chat_template: str = ""
    stand_in: bool = False


# canonical model id -> its tokenizer (provider_slug::provider_model_id, modules/model-registry/docs/PRD.md:197)
MODEL_TOKENIZERS = {
    "openai::gpt-4": ModelTokenizer("cl100k_base"), "openai::gpt-3.5-turbo": ModelTokenizer("cl100k_base"),
    "openai::text-embedding-3-small": ModelTokenizer("cl100k_base"),
    "openai::gpt-4o": ModelTokenizer("o200k_base"), "openai::gpt-4o-mini": ModelTokenizer("o200k_base"), "openai::o1": ModelTokenizer("o200k_base"),
    "meta::llama-3-8b-instruct": ModelTokenizer("llama3"), "meta::llama-3.1-70b-instruct": ModelTokenizer("llama3"),
    # instruct V3: their own tekken files hold the committed file's first 130072 ranks
    "mistral::mistral-nemo": ModelTokenizer("mistral_tekken", "mistral-v3"),
    "mistral::pixtral-12b": ModelTokenizer("mistral_tekken", "mistral-v3"),
    # instruct V7: STAND-IN -- their own tekken.json files are not in this repository; tekken_240911 and its control tokens stand
    # in for them (the V7 rules are checked against mistral_common on tekken_240911, not on these models' files)
    "mistral::mistral-large-2411": ModelTokenizer("mistral_tekken", "mistral-v7", stand_in=True),
    "mistral::pixtral-large-2411": ModelTokenizer("mistral_tekken", "mistral-v7", stand_in=True),
    "mistral::mistral-small-2501": ModelTokenizer("mistral_tekken", "mistral-v7", stand_in=True),
    "mistral::mistral-small-2503": ModelTokenizer("mistral_tekken", "mistral-v7", stand_in=True),
}
# canonical model id -> vocab
MODEL_VOCABS = {model: t.vocab for model, t in MODEL_TOKENIZERS.items()}


@dataclass
class ResolvedVocab:
    spec: VocabSpec
    file_bytes: bytes
    max_ranks: int
    stand_in: bool
    label: str
    sha256: str

    @property
    def pattern_id(self):
        return N.PATTERN_IDS[self.spec.pattern]

    @property
    def control_tokens(self) -> dict:
        """{token string: id} of the vocabulary's control tokens (empty for a vocabulary without them)"""
        return control_tokens(self.spec)


def control_tokens(spec: VocabSpec) -> dict:
    if not spec.controls:
        return {}
    with open(os.path.join(VOCAB_DIR, spec.controls), encoding="utf-8") as f:
        toks = json.load(f)
    if len(toks) != spec.id_base:
        raise ValueError("%s lists %d control tokens for id base %d" % (spec.controls, len(toks), spec.id_base))
    return {t: i for i, t in enumerate(toks)}


def _read(path):
    with open(path, "rb") as f:
        return f.read()


class VocabUnavailable(LookupError):
    """the vocabulary is unknown, or its real rank file is not on this host and stand-ins were not asked for"""


def resolve(name: str, allow_stand_in: bool = False) -> ResolvedVocab:
    """allow_stand_in: serve a vocabulary whose real rank file is absent from the truncated Tekken file (benchmarks and
    tests only -- its token counts are NOT the real model's).  Off by default: a gateway must not bill from a stand-in."""
    if name not in SPECS:
        raise VocabUnavailable("unknown vocabulary %r" % name)
    spec = SPECS[name]
    if name in ("tekken", "mistral_tekken"):
        data = _read(TEKKEN_FILE)
        return ResolvedVocab(spec, data, spec.n_ranks, False, "tekken_240911[:130072]" + (" + 1000" if spec.id_base else ""),
                             hashlib.sha256(data).hexdigest())
    for d in filter(None, [os.environ.get("CFBPE_VOCAB_DIR"), VOCAB_DIR]):
        p = os.path.join(d, spec.real_file)
        if os.path.exists(p):
            data = _read(p)
            sha = hashlib.sha256(data).hexdigest()
            want = KNOWN_SHA256.get(spec.real_file)
            if want and sha != want:
                raise ValueError("%s: sha256 %s does not match the published %s" % (p, sha, want))
            return ResolvedVocab(spec, data, 0, False, spec.real_file, sha)
    if not (allow_stand_in or os.environ.get("CFBPE_ALLOW_STAND_IN") == "1"):
        raise VocabUnavailable("%s: %s is not in $CFBPE_VOCAB_DIR or %s (stand-ins are opt-in: allow_stand_in=True)"
                               % (name, spec.real_file, VOCAB_DIR))
    data = _read(TEKKEN_FILE)
    n = min(spec.n_ranks, 150000)
    return ResolvedVocab(spec, data, n, True, "STAND-IN tekken_240911[:%d] + %s pattern" % (n, spec.pattern),
                         hashlib.sha256(data).hexdigest())


def for_model(canonical_id: str) -> str:
    """vocab name for a model-registry canonical id; VocabUnavailable if the model is unknown"""
    return tokenizer_for_model(canonical_id).vocab


def tokenizer_for_model(canonical_id: str) -> ModelTokenizer:
    """vocabulary, chat template and stand-in flag of a model-registry canonical id; VocabUnavailable if the model is unknown"""
    try:
        return MODEL_TOKENIZERS[canonical_id]
    except KeyError:
        raise VocabUnavailable("no vocabulary is registered for model %r" % canonical_id) from None
