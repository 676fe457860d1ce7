"""One process, two devices: every kernel that asks for more than 48 KB of dynamic shared memory opts in on each device it
launches on, not once per process.  A MoE block with its device router (decode_step: router + MoE decode kernels; prefill_step:
router + grouped GEMMs) runs on cuda:0 and then on cuda:1 and must give the same routing, h and y bit for bit."""
import pytest
import torch

from paroquant_b200.checkpoint import make_synthetic_activations
from paroquant_b200.experts import ParoExperts, ParoRouter
from test_gpu_moe import _blocks

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")]


def _run(dev, blocks, router_w, x, k):
    out = []
    with torch.cuda.device(dev):
        ex = ParoExperts(blocks, torch.bfloat16, device=dev)
        router = ParoRouter(router_w, k, True, dtype=torch.bfloat16, device=dev)
        for make, T in ((ex.decode_step, 16), (ex.prefill_step, 40)):
            st = make(T, k, router=router)
            st.x.copy_(x[:T])
            st.step()
            out += [st.topk_ids.cpu(), st.topk_weights.cpu(), st.h.cpu(), st.y.cpu()]
    return out


def test_moe_steps_with_router_on_a_second_device():
    if len({torch.cuda.get_device_properties(i).multi_processor_count for i in (0, 1)}) > 1:
        pytest.skip("the two devices plan for different SM counts, so their summation orders may differ")
    E, H, I, k = 16, 2048, 768, 4
    blocks = _blocks(E, H, I)
    router_w = torch.randn(E, H, generator=torch.Generator().manual_seed(3)) * (2.0 / H ** 0.5)
    x = make_synthetic_activations(40, H, seed=11)
    first = _run("cuda:0", blocks, router_w, x, k)
    second = _run("cuda:1", blocks, router_w, x, k)
    names = ["decode ids", "decode weights", "decode h", "decode y", "prefill ids", "prefill weights", "prefill h", "prefill y"]
    for name, a, b in zip(names, first, second):
        assert torch.equal(a, b), f"{name} on cuda:1 differs from cuda:0"
