"""Same inputs, our kernels against the UNMODIFIED reference pipeline (its rotate kernel + vLLM Marlin).

The reference outputs are stored in tests/golden/ref_pipeline_samples.npz (tools/ref_gpu.py samples, run on an H100):
for every seed-defined case the output's shape and a seeded sample of its elements (flat indices + raw bits).  The
layer and the activations are regenerated here from the same seeds, our output is computed at full size and compared
at the sampled elements: bit-exact for the rotation, relative error < 1e-3 for the fused linear."""
import json

import numpy as np
import pytest
import torch

from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

_Z = np.load(GOLDEN / "ref_pipeline_samples.npz")
CASES = json.loads(str(_Z["spec"]))
_TD = {"float32": torch.float32, "float16": torch.float16, "bfloat16": torch.bfloat16}


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_against_reference_kernels(case):
    import paroquant_b200.kernels.cuda  # noqa: F401
    from paroquant_b200.linear import ParoLinearKernel

    dt = _TD[case["dtype"]]
    L = make_synthetic_layer(case["K"], case["parts"], seed=case["seed"]).to("cuda")
    x = make_synthetic_activations(case["M"], case["K"], seed=case["xseed"], dtype=dt).cuda()
    name = case["name"]
    idx = torch.from_numpy(_Z[name + "_idx"].astype(np.int64))
    ref = torch.from_numpy(np.ascontiguousarray(_Z[name + "_val"]))
    ref = ref if dt == torch.float32 else ref.view(torch.int16).view(dt)
    if case["kind"] == "rotate":
        out = torch.ops.rotation.rotate(x, L.pairs[0], L.theta[0], L.channel_scales[0]).cpu()
        assert list(out.shape) == _Z[name + "_shape"].tolist()
        got = out.reshape(-1)[idx]
        assert torch.equal(got, ref), f"{(got != ref).float().mean().item():.4%} differ"   # bit exact
    else:
        y = ParoLinearKernel.from_buffers(L, dt, check_pairs=False, max_m=case["M"])(x).cpu()
        assert list(y.shape) == _Z[name + "_shape"].tolist()
        got = y.reshape(-1)[idx].float()
        err = ((got - ref.float()).norm() / ref.float().norm()).item()
        assert err < 1e-3, err
