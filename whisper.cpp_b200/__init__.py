"""whisper.cpp_b200 -- CUDA-native Whisper inference engine for the H100 (sm_90a), behind the whisper.h C ABI.

The product is `libwhisper_b200.so` (CUDA + C++, built in-tree by `make -C whisper.cpp_b200`).  This package only
holds the host-side Python mirror of the reference interface (`api.py`) and the synthetic-model tooling (`synth.py`).
The directory name contains a dot, so load it by path:

    import importlib.util, os
    spec = importlib.util.spec_from_file_location("whisper_cpp_b200", os.path.join(repo, "whisper.cpp_b200", "__init__.py"),
                                                  submodule_search_locations=[os.path.join(repo, "whisper.cpp_b200")])
"""
from .api import WhisperB200, bind_whisper_api, FullParams, ContextParams, TokenData, LIB_PATH  # noqa: F401
from . import synth  # noqa: F401
