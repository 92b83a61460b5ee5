"""flash_vstream_b200 — H100-native (sm_90a) implementation of Flash-VStream's streaming hot path:
ViT-L/14 frame encoding + Flash-Memory consolidation, behind the reference's own Python surface.

    flash_vstream_b200.compress_functions   <->  flash_vstream.model.compress_functions
    flash_vstream_b200.vstream_arch         <->  flash_vstream.model.vstream_arch (hot-path half)
    flash_vstream_b200.clip_encoder         <->  flash_vstream.model.multimodal_encoder.clip_encoder
    flash_vstream_b200.ops                  tensor-level wrappers over the C ABI (include/fvs_b200.h)
    flash_vstream_b200.StreamPool           many streams on one GPU, stepped together (multistream.py)
    flash_vstream_b200.CLIPFramePreprocessor, .Qwen2VLFramePreprocessor, .Qwen2VLVideoFetcher
                                            decoded uint8 frames -> tower pixels on the GPU (preprocess.py)
    flash_vstream_b200.StreamCheckpoint     a live stream's state on the host / on disk: suspend, resume, move (checkpoint.py)
    flash_vstream_b200.install()            rebinds the reference's modules to these implementations

All arithmetic happens in libfvs_b200.so (hand-written CUDA for sm_90a).  There is no CPU fallback: importing the
package is cheap, but any op raises if the library or a CUDA device is missing.
"""
from . import _lib  # noqa: F401

__version__ = "0.1.0"


def install():
    from .install import install as _install
    return _install()


def native_library_path():
    return str(_lib.lib_path())


def __getattr__(name):      # StreamPool imports torch: loaded on first use, so that importing the package stays cheap
    if name == "StreamPool":
        from .multistream import StreamPool
        return StreamPool
    if name in ("CLIPFramePreprocessor", "Qwen2VLFramePreprocessor", "Qwen2VLVideoFetcher"):
        from . import preprocess
        return getattr(preprocess, name)
    if name == "StreamCheckpoint":
        from .checkpoint import StreamCheckpoint
        return StreamCheckpoint
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
