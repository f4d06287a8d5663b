"""miniengineao_b200 -- H100-native multi-scale SSAO pipeline behind the MiniEngineAO
AmbientOcclusion component surface.  The compute path is libmeao.so (hand-written sm_90a CUDA,
C ABI in include/meao.h); this package is the thin Python host that mirrors the reference
component and its parameters.  There is no CPU fallback."""
from .ambient_occlusion import AmbientOcclusion, Camera  # noqa: F401
from ._native import MeaoError  # noqa: F401

__all__ = ["AmbientOcclusion", "Camera", "MeaoError", "ambient_occlusion_op", "ambient_occlusion_batch_op"]

# package name -> torch_ops function (the package already has a module named ambient_occlusion)
_TORCH_OPS = {"ambient_occlusion_op": "ambient_occlusion", "ambient_occlusion_batch_op": "ambient_occlusion_batch"}


def __getattr__(name):
    """ambient_occlusion_op / ambient_occlusion_batch_op: torch_ops.ambient_occlusion / ambient_occlusion_batch, the torch.library
    operators, imported (and registered) on first use so that importing the package does not import torch."""
    if name in _TORCH_OPS:
        from . import torch_ops
        for n, f in _TORCH_OPS.items():
            globals()[n] = getattr(torch_ops, f)
        return globals()[name]
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
