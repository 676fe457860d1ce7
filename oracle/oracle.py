"""CPU oracle for the ParoQuant hot path.  TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this module.  Nothing under ``paroquant_b200/`` does.

Two independent restatements of the same algorithm live here and are checked against each other
(tests/test_oracle.py) and against outputs of the unmodified reference kernels captured on an H100
(tests/golden/ref_gpu_*.npz, made by tools/gen_ref_golden.py):

  * ``c_*``   -- thin ctypes wrappers over oracle/paro_oracle.c (scalar loops, ``fmaf``)
  * ``np_*``  -- vectorised numpy, with an error-free emulation of the fp32 FMA

Reference lines each function follows (paths relative to /root/reference):
  awq_pack / awq_unpack   paroquant/cli/convert.py:19,149-155 ; inference/backends/mlx/load.py:15-24
  dequant                 inference/backends/mlx/load.py:46-54 (+ one rounding to T, SURVEY.md A.3)
  rotate                  kernels/cuda/rotation.cu:10-43,62-95 ; rotation.cuh:16-75,91-173
  linear                  inference/backends/vllm/plugin.py:281-311 ; transformers/modules.py:57-71

Documented deviation: sin/cos are correctly rounded here, MUFU approximations on the GPU
(see the header of paro_oracle.c).

dtype is one of "float32", "float16", "bfloat16".  Half types are carried as numpy uint16 bit
patterns for bfloat16 and numpy float16 for float16 at the API surface; helpers convert.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB_PATH = _HERE / "_build" / "libparo_oracle.so"
_DT = {"float32": 0, "float16": 1, "bfloat16": 2}
AWQ_ORDER = np.array([0, 2, 4, 6, 1, 3, 5, 7])       # convert.py:19
AWQ_INV = np.array([0, 4, 1, 5, 2, 6, 3, 7])         # mlx/load.py:18


# ------------------------------------------------------------------ build / load of the C oracle

def build_c_oracle(force: bool = False) -> Path:
    src = _HERE / "paro_oracle.c"
    if force or not _LIB_PATH.exists() or _LIB_PATH.stat().st_mtime < src.stat().st_mtime:
        _LIB_PATH.parent.mkdir(exist_ok=True)
        # -ffp-contract=off: every rounding in the oracle is written out explicitly
        subprocess.check_call(
            ["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
             "-o", str(_LIB_PATH), str(src), "-lm"])
    return _LIB_PATH


_lib = None


def _c():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(str(build_c_oracle()))
        for name in ("paro_oracle_rotate", "paro_oracle_linear"):
            getattr(_lib, name).restype = ctypes.c_int
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


# ------------------------------------------------------------------ dtype helpers (numpy side)

def f32_to_bf16_bits(x: np.ndarray) -> np.ndarray:
    """Round-to-nearest-even fp32 -> bf16 bit patterns (uint16)."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    r = ((u.astype(np.uint64) + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(nan, ((u >> 16) | 0x40).astype(np.uint16), r)


def bf16_bits_to_f32(b: np.ndarray) -> np.ndarray:
    return (np.ascontiguousarray(b, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def round_to(x: np.ndarray, dtype: str) -> np.ndarray:
    """fp32 array -> fp32 array holding values representable in `dtype` (one RNE rounding)."""
    x = np.asarray(x, dtype=np.float32)
    if dtype == "float32":
        return x
    if dtype == "float16":
        with np.errstate(over="ignore"):
            return x.astype(np.float16).astype(np.float32)
    return bf16_bits_to_f32(f32_to_bf16_bits(x))


def to_bits(x_f32: np.ndarray, dtype: str) -> np.ndarray:
    """fp32 values (already representable) -> storage array for the C oracle."""
    if dtype == "float32":
        return np.ascontiguousarray(x_f32, dtype=np.float32)
    if dtype == "float16":
        return np.ascontiguousarray(np.asarray(x_f32, np.float32).astype(np.float16)).view(np.uint16)
    return f32_to_bf16_bits(x_f32)


def from_bits(b: np.ndarray, dtype: str) -> np.ndarray:
    if dtype == "float32":
        return np.asarray(b, dtype=np.float32)
    if dtype == "float16":
        return np.ascontiguousarray(b, dtype=np.uint16).view(np.float16).astype(np.float32)
    return bf16_bits_to_f32(b)


def _ftz(x: np.ndarray) -> np.ndarray:
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return np.where((u & 0x7F800000) == 0, u & 0x80000000, u).astype(np.uint32).view(np.float32)


def _fma32(a: np.ndarray, b: np.ndarray, c: np.ndarray) -> np.ndarray:
    """Correctly rounded fp32 fma(a, b, c) = RN32(a*b + c) from float64 pieces.

    a*b is exact in float64 (24+24 significant bits).  t = fl64(a*b + c) can be inexact, and
    rounding t to fp32 could then double-round; TwoSum recovers the lost part e and breaks the
    (only possible) failure case, a tie at the fp32 rounding step.
    """
    s = a.astype(np.float64) * b.astype(np.float64)
    p = c.astype(np.float64)
    t = s + p
    bb = t - s
    e = (s - (t - bb)) + (p - bb)                     # exact error of the float64 add
    with np.errstate(over="ignore"):
        r = t.astype(np.float32)
    d = t - r.astype(np.float64)                      # exact: r is within one fp32 ulp of t
    up = np.nextafter(r, np.float32(np.inf))
    dn = np.nextafter(r, np.float32(-np.inf))
    tie_up = (d > 0) & (np.abs(d) == (up.astype(np.float64) - r.astype(np.float64)) / 2)
    tie_dn = (d < 0) & (np.abs(d) == (r.astype(np.float64) - dn.astype(np.float64)) / 2)
    fix = np.isfinite(r) & (e != 0)
    r = np.where(fix & tie_up & (e > 0), up, r)
    r = np.where(fix & tie_dn & (e < 0), dn, r)
    return r.astype(np.float32)


# ------------------------------------------------------------------ AWQ pack / unpack

def np_awq_pack(values: np.ndarray) -> np.ndarray:
    """convert.py:149-155.  values [R, C] in 0..15 -> int32 [R, C/8]."""
    v = np.asarray(values).astype(np.uint32)
    r = v.reshape(v.shape[0], -1, 8)[:, :, AWQ_ORDER]
    out = np.zeros(r.shape[:2], dtype=np.uint32)
    for i in range(8):
        out |= (r[:, :, i] & 0xF) << np.uint32(4 * i)
    return out.view(np.int32)


def np_awq_unpack(packed: np.ndarray) -> np.ndarray:
    """mlx/load.py:21-24.  int32 [R, C/8] -> uint8 [R, C]."""
    p = np.ascontiguousarray(packed).view(np.uint32).astype(np.int64)
    raw = ((p[:, :, None] >> np.arange(0, 32, 4, dtype=np.int64)) & 0xF).astype(np.uint8)
    return raw[:, :, AWQ_INV].reshape(p.shape[0], -1)


def c_awq_pack(values: np.ndarray) -> np.ndarray:
    v = np.ascontiguousarray(values, dtype=np.uint8)
    out = np.empty((v.shape[0], v.shape[1] // 8), dtype=np.int32)
    _c().paro_oracle_awq_pack(_p(v), ctypes.c_int64(v.shape[0]), ctypes.c_int64(v.shape[1]), _p(out))
    return out


def c_awq_unpack(packed: np.ndarray) -> np.ndarray:
    p = np.ascontiguousarray(packed, dtype=np.int32)
    out = np.empty((p.shape[0], p.shape[1] * 8), dtype=np.uint8)
    _c().paro_oracle_awq_unpack(_p(p), ctypes.c_int64(p.shape[0]), ctypes.c_int64(p.shape[1]), _p(out))
    return out


# ------------------------------------------------------------------ dequant

def np_dequant(qweight, qzeros, scales_f32, group: int, dtype: str) -> np.ndarray:
    """W[k, n] = T((q - z) * s_T) as fp32.  scales_f32: fp32 values (fp16 on disk)."""
    q = np_awq_unpack(qweight).astype(np.float32)
    z = np_awq_unpack(qzeros).astype(np.float32)
    s = round_to(np.asarray(scales_f32, np.float32), dtype)     # vLLM holds scales in T (A.3)
    d = q - np.repeat(z, group, axis=0)
    return round_to(d * np.repeat(s, group, axis=0), dtype)


def c_dequant(qweight, qzeros, scales_f32, group: int, dtype: str) -> np.ndarray:
    qw = np.ascontiguousarray(qweight, dtype=np.int32)
    qz = np.ascontiguousarray(qzeros, dtype=np.int32)
    K, N = qw.shape[0], qw.shape[1] * 8
    s = to_bits(round_to(scales_f32, dtype), dtype)
    W = np.empty((K, N), dtype=np.float32)
    _c().paro_oracle_dequant(_p(qw), _p(qz), _p(s), ctypes.c_int64(K), ctypes.c_int64(N),
                             ctypes.c_int(group), ctypes.c_int(_DT[dtype]), _p(W))
    return W


# ------------------------------------------------------------------ rotation

def _prep_rot(x_f32, pairs, theta_f32, scales_f32, dtype):
    x = round_to(np.asarray(x_f32, np.float32), dtype)
    x2 = np.ascontiguousarray(x.reshape(-1, x.shape[-1]))
    th = round_to(np.asarray(theta_f32, np.float32), dtype)          # rotation.cu:75
    sc = None if scales_f32 is None else round_to(np.asarray(scales_f32, np.float32).reshape(-1), dtype)
    idx = np.ascontiguousarray(pairs, dtype=np.int16)
    return x, x2, th, sc, idx


def c_rotate(x_f32, pairs, theta_f32, scales_f32=None, group: int = 128, dtype: str = "bfloat16"):
    """rotate(x, idx_ij, theta, scales, group_size) -- rotation.cu:128-131 schema.  Returns fp32
    values representable in dtype, same shape as x."""
    x, x2, th, sc, idx = _prep_rot(x_f32, pairs, theta_f32, scales_f32, dtype)
    M, K = x2.shape
    xb, tb = to_bits(x2, dtype), to_bits(th, dtype)
    sb = None if sc is None else to_bits(sc, dtype)
    out = np.empty_like(xb)
    rc = _c().paro_oracle_rotate(_p(xb), _p(out), _p(idx), _p(tb), _p(sb), ctypes.c_int64(M),
                                 ctypes.c_int64(K), ctypes.c_int(idx.shape[0]), ctypes.c_int(group),
                                 ctypes.c_int(_DT[dtype]))
    if rc:
        raise RuntimeError(f"paro_oracle_rotate failed rc={rc}")
    return from_bits(out, dtype).reshape(x.shape)


def np_rotate(x_f32, pairs, theta_f32, scales_f32=None, group: int = 128, dtype: str = "bfloat16", sincos=None):
    """sincos: optional (c, s), fp32 [krot, K/2], used in place of the correctly rounded cos / sin of T(theta) -- e.g. the
    GPU's own __sincosf values, which makes this an exact restatement of the CUDA rotation (tests/gpu_reference.py:
    kernel_sincos).  Everything else, every rounding point included, is unchanged."""
    x, x2, th, sc, idx = _prep_rot(x_f32, pairs, theta_f32, scales_f32, dtype)
    M, K = x2.shape
    krot = idx.shape[0]
    ng = K // group
    if sc is not None:
        v = _ftz(_ftz(x2) * _ftz(sc)[None, :]) if dtype == "float32" else round_to(x2 * sc[None, :], dtype)
    else:
        v = x2.copy()
    v = v.reshape(M, ng, group)
    off = np.arange(ng)[:, None]
    for r in range(krot):
        p = idx[r].astype(np.int64).reshape(ng, group)
        pi, pj = p[:, 0::2], p[:, 1::2]                          # [ng, G/2]
        if sincos is None:
            t = th[r].astype(np.float64).reshape(ng, group // 2)
            s_ = np.sin(t).astype(np.float32)[None]
            c_ = np.cos(t).astype(np.float32)[None]
        else:
            c_ = np.asarray(sincos[0][r], np.float32).reshape(1, ng, group // 2)
            s_ = np.asarray(sincos[1][r], np.float32).reshape(1, ng, group // 2)
        a = _ftz(v[:, off, pi])
        b = _ftz(v[:, off, pj])
        s_b, c_b = np.broadcast_to(s_, a.shape), np.broadcast_to(c_, a.shape)
        yi = _ftz(_fma32(c_b, a, _ftz(s_b * b)))
        yj = _ftz(_fma32(c_b, b, _ftz(s_b * -a)))
        v[:, off, pi] = round_to(yi, dtype)
        v[:, off, pj] = round_to(yj, dtype)
    return v.reshape(x.shape)


def np_rotate_backward(x_f32, pairs, theta_f32, y_f32, grad_out_f32, scales_f32=None, group: int = 128, reference_formula: bool = False):
    """RotateTensorFunc.backward in float64, structured like kernels/cuda/autograd.py:20-61: walk the rotations last to first,
    un-rotate t and g with -theta, form dtheta from the un-rotated values; grad_x = g * scale, grad_scale = sum_rows(x * g)
    (autograd.py:54-56).  No per-rotation rounding: the mathematical gradient the per-dtype kernels are compared with.

    dtheta: with (a, b) / (ga, gb) the un-rotated values / gradients of a pair, the gradient is the 2-D cross product
        dL/dtheta = sum_rows (ga*b - gb*a)                       (rotation invariant: equals sum_rows (G_i y_j - G_j y_i))
    which is what this function and the CUDA backward return (checked against autograd of a dense formulation, tests/test_oracle.py).
    The reference evaluates  (ga*b - gb*a) * cos - (ga*a + gb*b) * sin  (autograd.py:50-52) -- the right expression for the
    OUTPUT-space gradient G and the INPUT values (a, b), but it is applied after g has been un-rotated too (autograd.py:38), so it
    returns  cos * dL/dtheta - sin * sum_rows(g . t):  `reference_formula=True` reproduces that value for comparison.
    Returns (grad_x, grad_theta [krot, K/2], grad_scale [K] or None)."""
    idx = np.ascontiguousarray(pairs, dtype=np.int16)
    krot, K = idx.shape
    ng = K // group
    x = np.asarray(x_f32, np.float64).reshape(-1, K)
    t = np.asarray(y_f32, np.float64).reshape(-1, K).reshape(-1, ng, group).copy()
    g = np.asarray(grad_out_f32, np.float64).reshape(-1, K).reshape(-1, ng, group).copy()
    th = np.asarray(theta_f32, np.float64)
    grad_theta = np.zeros((krot, K // 2), np.float64)
    off = np.arange(ng)[:, None]
    for r in range(krot - 1, -1, -1):
        p = idx[r].astype(np.int64).reshape(ng, group)
        pi, pj = p[:, 0::2], p[:, 1::2]
        ang = th[r].reshape(ng, group // 2)
        c_, s_ = np.cos(ang)[None], np.sin(ang)[None]
        for v in (t, g):                                           # rotate(., idx, -theta): [[c, -s], [s, c]]
            a, b = v[:, off, pi].copy(), v[:, off, pj].copy()
            v[:, off, pi] = c_ * a - s_ * b
            v[:, off, pj] = s_ * a + c_ * b
        a, b, ga, gb = t[:, off, pi], t[:, off, pj], g[:, off, pi], g[:, off, pj]
        cross = (ga * b - gb * a).sum(0)
        grad_theta[r] = ((cross * c_[0] - (ga * a + gb * b).sum(0) * s_[0]) if reference_formula else cross).reshape(-1)
    gflat = g.reshape(-1, K)
    if scales_f32 is None:
        return gflat.reshape(np.shape(x_f32)), grad_theta, None
    sc = np.asarray(scales_f32, np.float64).reshape(-1)
    return (gflat * sc[None, :]).reshape(np.shape(x_f32)), grad_theta, (x * gflat).sum(0)


# ------------------------------------------------------------------ GEMM / linear

def np_gemm(xrot_f32, W_f32, bias_f32=None, dtype: str = "bfloat16", return_acc: bool = False):
    a = np.asarray(xrot_f32, np.float32)
    acc = a.reshape(-1, a.shape[-1]).astype(np.float64) @ np.asarray(W_f32).astype(np.float64)
    y = round_to(acc.astype(np.float32), dtype)
    if bias_f32 is not None:
        y = round_to(y + round_to(np.asarray(bias_f32, np.float32), dtype)[None, :], dtype)
    y = y.reshape(*a.shape[:-1], W_f32.shape[1])
    return (y, acc) if return_acc else y


def c_gemm(xrot_f32, W_f32, bias_f32=None, dtype: str = "bfloat16"):
    a = np.asarray(xrot_f32, np.float32)
    a2 = np.ascontiguousarray(a.reshape(-1, a.shape[-1]))
    W = np.ascontiguousarray(W_f32, dtype=np.float32)
    M, K = a2.shape
    N = W.shape[1]
    ab = to_bits(a2, dtype)
    bb = None if bias_f32 is None else to_bits(round_to(bias_f32, dtype), dtype)
    y = np.empty((M, N), dtype=ab.dtype)
    _c().paro_oracle_gemm(_p(ab), _p(W), _p(bb), ctypes.c_int64(M), ctypes.c_int64(N), ctypes.c_int64(K),
                          ctypes.c_int(_DT[dtype]), _p(y), None)
    return from_bits(y, dtype).reshape(*a.shape[:-1], N)


def linear(x_f32, layer: dict, dtype: str = "bfloat16", impl: str = "c", W_cache: dict | None = None):
    """The whole hot path for one (possibly merged) linear, as ParoQuantLinearMethod.apply does it
    (plugin.py:281-311): per partition rotate -> dequant GEMM, concatenate, add bias.

    layer: dict with qweight [K, N/8] i32, qzeros [K/G, N/8] i32, scales [K/G, N] f32-valued,
    theta [P, R, K/2], pairs [P, R, K] i16, channel_scales [P, 1, K], part_sizes [P], group,
    optional bias [N].
    """
    rot = c_rotate if impl == "c" else np_rotate
    deq = c_dequant if impl == "c" else np_dequant
    gemm = c_gemm if impl == "c" else np_gemm
    group = int(layer["group"])
    key = (id(layer["qweight"]), dtype, impl)
    if W_cache is not None and key in W_cache:
        W = W_cache[key]
    else:
        W = deq(layer["qweight"], layer["qzeros"], layer["scales"], group, dtype)
        if W_cache is not None:
            W_cache[key] = W
    outs, n0 = [], 0
    for p, n in enumerate(layer["part_sizes"]):
        xr = rot(x_f32, layer["pairs"][p], layer["theta"][p], layer["channel_scales"][p], group, dtype)
        outs.append(gemm(xr, W[:, n0:n0 + n], None, dtype))
        n0 += n
    y = np.concatenate(outs, axis=-1)
    if layer.get("bias") is not None:
        y = round_to(y + round_to(layer["bias"], dtype), dtype)
    return y


# ------------------------------------------------------------------ element-wise neighbours of the linear (chains)
# The reference leaves these to vLLM (call sites of ParoQuantLinearMethod.apply, plugin.py:281-311): they are restated
# from vLLM 0.22's kernels -- csrc/activation_kernels.cu (silu_and_mul: T(x / (1 + exp(-x))) * y in T) and
# csrc/layernorm_kernels.cu (fused_add_rms_norm: z = T(x + residual), variance of z in fp32, T(T(z * rstd) * w)).

def silu_and_mul(gate_up_f32, dtype: str = "bfloat16"):
    """[.., 2K] -> [.., K]: T(T(silu(gate)) * up)."""
    a = np.asarray(gate_up_f32, np.float32)
    K = a.shape[-1] // 2
    g, u = a[..., :K], a[..., K:]
    with np.errstate(over="ignore"):
        act = round_to(g / (np.float32(1.0) + np.exp(-g)).astype(np.float32), dtype)
    return round_to(act * u, dtype)


def add_residual(y_f32, residual_f32, dtype: str = "bfloat16"):
    """h = T(y + residual) -- the new residual stream of fused_add_rms_norm."""
    return round_to(np.asarray(y_f32, np.float32) + np.asarray(residual_f32, np.float32), dtype)


def rms_norm(h_f32, weight_f32, eps: float, dtype: str = "bfloat16"):
    """T(T(h * rsqrt(mean(h^2) + eps)) * w), statistics in fp32."""
    h = np.asarray(h_f32, np.float32)
    var = (h.astype(np.float64) ** 2).mean(axis=-1, keepdims=True)
    rstd = (1.0 / np.sqrt(var + eps)).astype(np.float32)
    return round_to(round_to(h * rstd, dtype) * round_to(weight_f32, dtype), dtype)


def rel_err(a, b) -> float:
    """Normwise relative error ||a - b|| / ||b|| in float64 (the parity metric, SURVEY.md 8d)."""
    a = np.asarray(a, np.float64).ravel()
    b = np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))
