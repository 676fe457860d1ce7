"""fp64 restatement of the MoE router's semantics (include/paro_b200.h: paro_moe_route); a helper module: pytest does not
collect it.  The reference has no routing code of its own (its MLX backend leaves it to mlx-lm); this restates softmax -> top-k ->
optional renormalise as Qwen3-MoE (norm_topk_prob) and Mixtral route, with the gate a T-typed linear as the serving stacks run it.
tests/test_moe_route_plan.py pins it against a torch formulation and on ties; tests/test_gpu_moe_route.py holds the kernel to it."""
from __future__ import annotations

import numpy as np

from oracle.oracle import round_to


def np_moe_route(x_f32, w_f32, top_k: int, renormalize: bool = True, dtype: str = "bfloat16", logits=None):
    """x [T, H] and router weight w [E, H] (values of `dtype`) -> (ids [T, k] int32, weights [T, k] float64, logits [T, E] float32).

      logit[t, e] = T(sum_h x[t, h] * w[e, h])          the sum in float64, one rounding to T
      p[t, :]     = softmax(logit[t, :])                float64, max subtracted first
      slots       = the top_k experts by descending logit; equal logits -> lower expert id first; slot 0 is the largest
      weights     = p[t, id_s], divided by their sum over the slots (in slot order) when renormalize

    `logits` [T, E], when given, replaces the first line (values of `dtype`): routing of logits computed elsewhere."""
    if logits is None:
        logits = round_to(np.asarray(x_f32, np.float64) @ np.asarray(w_f32, np.float64).T, dtype)
    logits = np.asarray(logits, np.float32)
    l64 = logits.astype(np.float64)
    ex = np.exp(l64 - l64.max(axis=-1, keepdims=True))
    p = ex / ex.sum(axis=-1, keepdims=True)
    ids = np.argsort(-l64, axis=-1, kind="stable")[:, :top_k]          # stable: equal logits keep ascending ids
    wts = np.take_along_axis(p, ids, axis=-1)
    if renormalize:
        den = np.zeros(wts.shape[0])
        for s in range(top_k):
            den = den + wts[:, s]
        wts = wts / den[:, None]
    return ids.astype(np.int32), wts, logits
