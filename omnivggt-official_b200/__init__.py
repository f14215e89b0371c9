"""H100-native OmniVGGT hot path (aggregator + DPT heads) behind the reference's OmniVGGT() API.

    from omnivggt_official_b200 import OmniVGGT      # drop-in for omnivggt.models.omnivggt.OmniVGGT

The compute path is the sm_90a CUDA library ``libovg.so`` (csrc/, C ABI in include/ovg.h); PyTorch is used for
device memory, streams, the frozen DINOv2 patchifier and the (tiny) camera head only.
"""
__all__ = ["OmniVGGT", "load_library"]


def load_library():
    from omnivggt_official_b200 import _lib
    return _lib.load()


def __getattr__(name):
    if name == "OmniVGGT":
        from omnivggt_official_b200.model import OmniVGGT
        return OmniVGGT
    raise AttributeError(name)
