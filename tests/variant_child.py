"""Runs the case list of one forced launch variant in a fresh process and prints a JSON summary on stdout (started by
tests/test_gpu_variants.py; pytest does not collect this file).

    python tests/variant_child.py <variant>

The planner knobs (PARO_DECODE_C, PARO_NO_CLUSTER, PARO_DECODE_STREAM, PARO_DECODE_PREROT_M, PARO_SMALL_M_MAX, ...) are read
once per process, so every variant needs its own.  The caller sets them and PARO_DECODE_VERBOSE=1: the library logs every
launch plan on stderr, and a `[case] <name>` line on stderr before each case ties those lines to the case.  Every single
linear is checked element-wise (gpu_reference.check_linear) and for run-to-run bit reproducibility, a selection-weight linear
(tests/selection_layers.py) for equality with its exact products; a decoder-tail chain is
checked stage by stage against the single-linear entry point plus plain torch element-wise ops, normwise < 1e-3.
"""
from __future__ import annotations

import json
import sys
import traceback
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))


def lin(K, parts, Ms, group=128, dt="bfloat16", bias=False, krot=8, kind="linear"):
    return {"kind": kind, "K": K, "parts": parts, "Ms": Ms, "group": group, "dt": dt, "bias": bias, "krot": krot}


def sel(K, parts, Ms, **kw):
    return lin(K, parts, Ms, kind="selection", **kw)


def tail(hidden, inter, Ms):
    return {"kind": "tail", "hidden": hidden, "inter": inter, "Ms": Ms}


_CLUSTER_CASES = [lin(1024, [256, 128], (1, 3, 4, 9, 16), bias=True), lin(2048, [384, 128], (1, 4, 16), group=64, dt="float16", krot=9),
                  sel(1024, [256, 128], (1, 5, 16), bias=True)]

CASES = {
    # the only decode branch that stores straight to y; bias and partial last blocks included (K <= 4096: one CTA holds K)
    "decode_c1": [lin(1024, [256, 128], (1, 4, 5, 16), bias=True), lin(640, [48, 16, 32], (3, 16), group=64, dt="float16"),
                  lin(4096, [4096], (1, 16)), lin(2048, [384], (2, 9), krot=3),
                  sel(640, [48, 16, 32], (1, 4, 16), group=64, dt="float16", krot=3)],
    "decode_c2": _CLUSTER_CASES,
    "decode_c4": _CLUSTER_CASES,
    "decode_c8": _CLUSTER_CASES,
    # decode has no plan for c = 3 / 16: single linears fall back to the stream kernel with 3 / 16 K slices
    "stream_c3": [lin(1024, [256, 128], (1, 4, 16), bias=True), lin(2048, [384], (1, 9), group=64, dt="float16", krot=7),
                  lin(4096, [4096, 1024, 1024], (1, 16)), tail(2048, 4096, (1, 16)),
                  sel(1024, [256, 128], (1, 9), group=64, dt="float16", krot=7, bias=True)],
    "stream_c16": [lin(2048, [384], (1, 4, 16), bias=True), lin(4096, [4096, 1024, 1024], (1, 9), dt="float16", krot=16),
                   tail(2048, 4096, (1, 16)), sel(2048, [384], (1, 16), krot=16)],
    "no_cluster": [lin(1024, [256, 128], (1, 16), bias=True), lin(4096, [4096], (1, 5)), lin(14336, [4096], (1, 4)),
                   sel(1024, [256, 128], (1, 5, 16), bias=True)],
    "stream_only": [lin(1024, [256, 128], (1, 5, 16), bias=True), lin(4096, [4096, 1024, 1024], (1, 16)), lin(4096, [14336, 14336], (1,)),
                    lin(14336, [4096], (1, 16)), lin(11008, [4096], (4,)),
                    sel(1024, [256, 128], (1, 5, 16), group=64, dt="float16", krot=9)],
    "prerot_never": [lin(1024, [256, 128], (5, 9, 16), bias=True), lin(2048, [384], (16,), group=64, krot=3), lin(14336, [4096], (4, 16)),
                     sel(1024, [256, 128], (5, 16), krot=3)],
    "prerot_from2": [lin(1024, [256, 128], (1, 2, 3, 4), bias=True), lin(2048, [384], (2, 4), krot=9), sel(1024, [256, 128], (2, 3, 4), krot=9)],
    "gemm_only": [lin(1024, [256, 128], (1, 7, 16), bias=True), lin(4096, [4096], (1, 16)), lin(640, [48, 16, 32], (3,), group=64, dt="float16"),
                  sel(640, [48, 16, 32], (1, 16), group=64, dt="float16", bias=True)],
    "shallow_ring": [lin(1024, [256, 128], (1, 4, 8, 16), bias=True), lin(4096, [4096], (1, 8)),
                     lin(1024, [256, 128], (1, 8, 16), bias=True, kind="chain1"), lin(4096, [4096], (1, 8), kind="chain1"),
                     sel(1024, [256, 128], (1, 8, 16), bias=True)],
}


def _name(c, M):
    if c["kind"] == "tail":
        return f"tail h{c['hidden']} i{c['inter']} M{M}"
    return (f"{c['kind']} {c['K']}x{c['parts']} g{c['group']} {c['dt']} krot{c['krot']}{' bias' if c['bias'] else ''} M{M}")


def _run_linear(c, M, note):
    import torch

    from gpu_reference import check_linear
    from paroquant_b200 import _cabi, chain
    from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer
    from paroquant_b200.linear import ParoLinearKernel

    T = getattr(torch, c["dt"])
    if c["kind"] == "selection":
        return _run_selection(c, M, note, T)
    L = make_synthetic_layer(c["K"], c["parts"], group_size=c["group"], krot=c["krot"], seed=c["K"] + M, device="cuda", bias=c["bias"])
    k = ParoLinearKernel.from_buffers(L, T, check_pairs=False)
    bias = None if L.bias is None else L.bias.to(T)
    x = make_synthetic_activations(M, c["K"], seed=M, device="cuda", dtype=T)
    if c["kind"] == "chain1":
        def run():
            y = torch.empty(M, sum(c["parts"]), dtype=T, device="cuda")
            chain.ParoChain([chain.ChainStep(k, x=x, y=y, bias=bias)], M)()
            return y
    else:
        def run():
            return k(x, bias)
    y = run()
    note["launches"] = _cabi.last_launch_count()
    torch.cuda.synchronize()
    note["ratio"] = check_linear(k, L, x, y, bias, what=note["name"])
    assert torch.equal(run(), y), "not bit-reproducible run to run"


def _run_selection(c, M, note, T):
    """Selection weights (tests/selection_layers.py): every output element equal to its exact product."""
    import torch

    from gpu_reference import assert_same_values, exact_rotated
    from paroquant_b200 import _cabi
    from paroquant_b200.checkpoint import make_synthetic_activations
    from paroquant_b200.linear import ParoLinearKernel
    from selection_layers import cover, selection_layer

    launches = set()
    for shift in cover(c["K"], sum(c["parts"])):
        S = selection_layer(c["K"], c["parts"], group=c["group"], krot=c["krot"], seed=c["K"] + M, shift=shift, bias=c["bias"])
        L = S.L.to("cuda")
        k = ParoLinearKernel.from_buffers(L, T, check_pairs=False)
        bias = None if L.bias is None else L.bias.to(T)
        x = make_synthetic_activations(M, c["K"], seed=M + shift, device="cuda", dtype=T)
        y = torch.full((M, sum(c["parts"])), float("nan"), dtype=T, device="cuda")
        k.forward_into(x, y, bias)
        launches.add(_cabi.last_launch_count())
        ref = S.apply(exact_rotated(L, x), T)
        if bias is not None:
            ref = (ref.float() + bias.float()).to(T)
        assert_same_values(y, ref, f"{note['name']} shift {shift}")
    assert len(launches) == 1, launches
    note["launches"] = launches.pop()
    note["exact"] = True


def _run_tail(c, M, note):
    import torch

    from paroquant_b200 import chain
    from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer
    from paroquant_b200.linear import ParoLinearKernel

    T, h, i = torch.bfloat16, c["hidden"], c["inter"]
    Ls = {"o": make_synthetic_layer(h, [h], seed=21, device="cuda"), "gate_up": make_synthetic_layer(h, [i, i], seed=22, device="cuda"),
          "down": make_synthetic_layer(i, [h], seed=23, device="cuda"), "qkv": make_synthetic_layer(h, [h, h // 4, h // 4], seed=24, device="cuda")}
    ks = {n: ParoLinearKernel.from_buffers(L, T, check_pairs=False) for n, L in Ls.items()}
    g = torch.Generator().manual_seed(25)
    attn = make_synthetic_activations(M, h, seed=26, dtype=T).cuda()
    resid = make_synthetic_activations(M, h, seed=27, dtype=T).cuda()
    w1 = (1.0 + 0.1 * torch.randn(h, generator=g)).to(T).cuda()
    w2 = (1.0 + 0.1 * torch.randn(h, generator=g)).to(T).cuda()
    ch, bufs = chain.decoder_tail(ks["o"], ks["gate_up"], ks["down"], ks["qkv"], attn_out=attn, residual=resid,
                                  post_attn_norm=w1, next_input_norm=w2, eps=1e-5)
    ch()
    torch.cuda.synchronize()

    def rms(v, w):
        vf = v.float()
        return (vf * torch.rsqrt(vf.pow(2).mean(-1, keepdim=True) + 1e-5)).to(T) * w

    def silu_mul(v):
        gg = v[..., :i].float()
        return (gg / (1.0 + torch.exp(-gg))).to(T) * v[..., i:]

    def err(a, b):
        return float((a.double() - b.double()).norm() / b.double().norm())

    stages = {
        "residual_mid": (ks["o"](attn).float() + resid.float()).to(T),
        "mlp_act": ks["gate_up"](rms(bufs["residual_mid"], w1)),
        "residual_out": (ks["down"](silu_mul(bufs["mlp_act"])).float() + bufs["residual_mid"].float()).to(T),
        "qkv": ks["qkv"](rms(bufs["residual_out"], w2)),
    }
    note["stage_err"] = {n: err(bufs[n], ref) for n, ref in stages.items()}
    for n, e in note["stage_err"].items():
        assert e < 1e-3, f"stage {n}: normwise error {e}"


def main(variant: str) -> int:
    import torch

    results = []
    for c in CASES[variant]:
        for M in c["Ms"]:
            note = {"name": _name(c, M), "kind": c["kind"], "M": M, "K": c.get("K", c.get("hidden")), "ok": False}
            print(f"[case] {note['name']}", file=sys.stderr, flush=True)
            try:
                (_run_tail if c["kind"] == "tail" else _run_linear)(c, M, note)
                note["ok"] = True
            except (AssertionError, RuntimeError) as e:
                note["error"] = f"{type(e).__name__}: {e}"
                traceback.print_exc()
                torch.cuda.synchronize()   # a launch error surfaces here and ends the run with a non-zero exit
            sys.stderr.flush()
            results.append(note)
    print(json.dumps({"variant": variant, "cases": results}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
