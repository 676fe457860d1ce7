"""Autograd wrapper around `torch.ops.rotation.rotate`.

Surface of /root/reference/paroquant/kernels/cuda/autograd.py:6-65 (`RotateTensorFunc`,
`scaled_pairwise_rotation`) used by the offline optimiser and the checkpoint converter.
Forward is the sm_90a kernel.  Backward is ONE launch (`paro_rotate_backward`,
csrc/paro_rotate.cu) where the reference walks the rotations in Python (per rotation two rotate
launches, five gathers and a reduction).  It uses the identities

    y_i =  c a + s b,   y_j = -s a + c b
    dy_i/dtheta = y_j,  dy_j/dtheta = -y_i          =>  dL/dtheta = sum_rows (G_i y_j - G_j y_i)

on the stage OUTPUT (t) and its gradient (g), then un-rotates both with -theta (a Givens
rotation is orthogonal, so the same update back-propagates g), rounding t and g to x.dtype after
every rotation exactly where the per-rotation launches stored them; the row sums run in fp32.

Deviation from the reference, on purpose: grad_theta here is the gradient (checked against autograd through a dense
formulation, tests/test_gpu_rotate.py, tests/test_oracle.py).  The reference evaluates
`(ga*b - gb*a)*cos - (ga*a + gb*b)*sin` (autograd.py:50-52) -- the right expression for the OUTPUT-space gradient and the
INPUT values of a pair -- after it has un-rotated g as well (autograd.py:38), which makes it return
`cos * dL/dtheta - sin * sum_rows(g . t)`.  Setting `REFERENCE_THETA_EXPRESSION = True` (or PARO_ROTATE_BACKWARD=reference in the
environment) makes the same launch return that value instead, for runs that must reproduce the reference's optimiser
trajectories; `oracle.np_rotate_backward(..., reference_formula=True)` restates it.  grad_x and grad_scale are the reference's.
"""
from __future__ import annotations

import torch

import os

from ... import _cabi

REFERENCE_THETA_EXPRESSION = os.environ.get("PARO_ROTATE_BACKWARD", "") == "reference"


class RotateTensorFunc(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, idx_ij, theta, scale=None, group_size=128):
        y = torch.ops.rotation.rotate(x, idx_ij, theta, scale, group_size)
        ctx.group_size = group_size
        ctx.has_scale = scale is not None
        ctx.save_for_backward(x, idx_ij, theta, y, *((scale,) if scale is not None else ()))
        return y

    @staticmethod
    def backward(ctx, grad_out):
        x, idx_ij, theta, y = ctx.saved_tensors[:4]
        scale = ctx.saved_tensors[4] if ctx.has_scale else None
        K = idx_ij.shape[1]
        flat_scale = None if scale is None else scale.reshape(-1)
        gx, gth, gsc = _cabi.rotate_backward(y.reshape(-1, K), grad_out.reshape(-1, K).to(y.dtype), x.reshape(-1, K), idx_ij, theta,
                                             flat_scale, ctx.group_size, reference_formula=REFERENCE_THETA_EXPRESSION)
        grad_x = gx.view_as(x)
        grad_theta = gth.to(theta.dtype)
        grad_scale = None if scale is None else gsc.to(scale.dtype).view_as(scale)
        return grad_x, None, grad_theta, grad_scale, None


def scaled_pairwise_rotation(x, idx_ij, theta, scales=None, group_size=128):
    return RotateTensorFunc.apply(x, idx_ij, theta, scales, group_size)
