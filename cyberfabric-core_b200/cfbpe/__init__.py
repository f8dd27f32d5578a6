"""cfbpe -- host side of the H100-native batched BPE tokenizer (cyberfabric-core llm-gateway path).

`_native`   ctypes binding of libcfbpe.so (the C ABI in include/cfbpe.h)
`plugin`    Python mirror of the ModKit plugin surface (TokenizerPluginClient, usage meter)
`vocabs`    vocabulary registry / model-registry vocab loader
`workload`  synthetic prompt batches of BASELINE.json's configs
`dist`      one-process-per-GPU sharding, NCCL vocab broadcast and count gather
"""
from . import _native  # noqa: F401
from ._native import Context, NativeError  # noqa: F401
