"""`torch.ops.rotation.rotate` on sm_90a, plus the autograd wrapper.

Same operator surface as the reference's JIT-built extension
(/root/reference/paroquant/kernels/cuda/__init__.py:52-65, rotation.cu:128-135): importing this
package registers

    rotation::rotate(Tensor x, Tensor idx_ij, Tensor theta, Tensor? scales=None,
                     int group_size=128) -> Tensor

for the CUDA dispatch key (and a fake/meta implementation for torch.compile), so call sites such
as `torch.ops.rotation.rotate(x, pairs, theta, channel_scales)` work unchanged.  The kernel is
ahead-of-time compiled into libparo_b200.so; there is no JIT step and no CPU implementation.
"""
from __future__ import annotations

import torch

from ... import _cabi

_cabi.lib()  # fail at import time, loudly, if the library was not built

_SCHEMA = "(Tensor x, Tensor idx_ij, Tensor theta, Tensor? scales=None, int group_size=128) -> Tensor"

try:
    torch.library.define("rotation::rotate", _SCHEMA)
except RuntimeError as e:  # pragma: no cover - another provider (the reference build) registered it first
    raise ImportError(
        "torch.ops.rotation.rotate is already registered in this process (is the reference "
        "paroquant.kernels.cuda imported too?); only one provider can own the op") from e


@torch.library.impl("rotation::rotate", "CUDA")
def _rotate_cuda(x, idx_ij, theta, scales=None, group_size=128):
    return _cabi.rotate(x, idx_ij, theta, scales, group_size)


@torch.library.register_fake("rotation::rotate")
def _rotate_fake(x, idx_ij, theta, scales=None, group_size=128):
    return torch.empty_like(x)


from .autograd import RotateTensorFunc, scaled_pairwise_rotation  # noqa: E402

__all__ = ["scaled_pairwise_rotation", "RotateTensorFunc"]
