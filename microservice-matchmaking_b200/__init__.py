"""H100-native opponent-search engine — host side above the C ABI (include/mm_engine.h).

The directory name follows the reference repository; import it with
``importlib.import_module("microservice-matchmaking_b200")`` (the hyphen rules out
a plain ``import`` statement).  Nothing here computes: the search tick runs in
hand-written sm_90a CUDA inside csrc/libmm_engine.so, and the package fails loudly
(ImportError / RuntimeError) when that library or a CUDA device is missing.
"""
from . import abi, synth  # noqa: F401
from .engine import Engine, EngineError, library_path, load_library  # noqa: F401
