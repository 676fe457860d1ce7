"""`RotateQuantizedLinear` -- module surface of the HF transformers backend.

Mirror of /root/reference/paroquant/inference/backends/transformers/modules.py:16-71: flat
buffers whose names are the checkpoint keys (`theta`, `pairs`, `channel_scales`, `qweight`,
`qzeros`, `scales`, `bias`), so `load_state_dict` / `from_pretrained` fill them directly.  The
reference's forward is rotate -> AutoAWQ GEMM (two kernels, fp16 only); here the first forward
prepacks the buffers once and every forward is ONE fused sm_90a launch, fp16 or bf16.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from ....linear import ParoLinearKernel


class RotateQuantizedLinear(nn.Module):
    def __init__(self, in_features: int, out_features: int, bias: bool = False, group_size: int = 128,
                 bits: int = 4, krot: int = 8):
        super().__init__()
        if bits != 4:
            raise ValueError(f"Unsupported bits={bits}. Supported: [4]")
        self.in_features, self.out_features = in_features, out_features
        self.w_bit, self.group_size = bits, group_size
        pack, n_groups = 32 // bits, in_features // group_size
        self.register_buffer("theta", torch.zeros(krot, in_features // 2, dtype=torch.float16))
        self.register_buffer("pairs", torch.zeros(krot, in_features, dtype=torch.int16))
        self.register_buffer("channel_scales", torch.ones(1, in_features, dtype=torch.float16))
        self.register_buffer("qweight", torch.zeros(in_features, out_features // pack, dtype=torch.int32))
        self.register_buffer("qzeros", torch.zeros(n_groups, out_features // pack, dtype=torch.int32))
        self.register_buffer("scales", torch.zeros(n_groups, out_features, dtype=torch.float16))
        if bias:
            self.register_buffer("bias", torch.zeros(out_features, dtype=torch.float16))
        else:
            self.bias = None
        self._kernel: ParoLinearKernel | None = None
        self._kernel_key = None

    def prepack(self, dtype: torch.dtype) -> ParoLinearKernel:
        """Build (or rebuild after a device / dtype / weight change) the fused-kernel layout."""
        key = (dtype, self.qweight.device, self.qweight._version, self.theta._version, self.pairs._version,
               self.channel_scales._version, self.qzeros._version, self.scales._version)
        if self._kernel is None or self._kernel_key != key:
            self._kernel = ParoLinearKernel.from_tensors(
                self.qweight, self.qzeros, self.scales, self.theta, self.pairs, self.channel_scales,
                [self.out_features], group_size=self.group_size, dtype=dtype)
            self._kernel_key = key
        return self._kernel

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if x.dtype not in (torch.float16, torch.bfloat16):
            raise RuntimeError(f"Expected float16 or bfloat16 input, got {x.dtype}")
        y = self.prepack(x.dtype)(x, self.bias)
        return y.reshape(*x.shape[:-1], self.out_features)
