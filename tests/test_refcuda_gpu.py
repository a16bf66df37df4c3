"""GPU parity against the reference's OWN CUDA kernels (ms_deform_im2col_cuda.cuh).

The reference outputs were recorded once by tests/golden/make_golden_refcuda.py (which runs those kernels, compiled by
oracle/Makefile `ref`) and are stored in tests/golden/refcuda_samples.npz: for every case and every output tensor, the
values at a fixed, seeded sample of positions (the full tensors of the larger cases are hundreds of MB), plus the
largest |grad_value| that scales its tolerance.  The inputs are regenerated here from the same seeds."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refcuda_samples.npz")
SAMPLES = 1024
OUTPUTS = ("out", "grad_value", "grad_loc", "grad_attn")

CASES = {
    "c1_enc": (1, 8, 32, [(60, 80), (30, 40), (15, 20), (8, 10)], 4, None),
    "c2_dec_n2": (2, 8, 32, [(100, 167), (50, 84), (25, 42), (13, 21)], 4, 300),
    "d36_l8": (1, 8, 36, [(17, 30), (9, 15), (5, 8), (3, 4)] * 2, 4, 311),
    "ref_test_shape": (2, 2, 4, [(8, 8), (4, 4), (2, 2)], 2, 3),
}


def case_inputs(name, dev):
    """value, shapes, loc, attn, grad_out of one case, generated on the host from a seed that depends on the name"""
    N, M, D, hw, P, Lq = CASES[name]
    g = torch.Generator().manual_seed(len(name))
    shapes = torch.as_tensor(hw, dtype=torch.long)
    S = int((shapes[:, 0] * shapes[:, 1]).sum())
    Lq = S if Lq is None else Lq
    L = len(hw)
    value = torch.randn(N, S, M, D, generator=g).to(dev)
    loc = (torch.rand(N, Lq, M, L, P, 2, generator=g) * 1.2 - 0.1).to(dev)
    attn = torch.softmax(torch.randn(N, Lq, M, L * P, generator=g), -1).view(N, Lq, M, L, P).to(dev)
    gout = torch.randn(N, Lq, M * D, generator=g).to(dev)
    return value, shapes.to(dev), loc, attn, gout


def sample_index(numel, salt):
    """the fixed positions compared for a tensor of `numel` elements: all of them when there are few"""
    if numel <= SAMPLES:
        return torch.arange(numel)
    g = torch.Generator().manual_seed(1000 + salt)
    return torch.randint(0, numel, (SAMPLES,), generator=g)


def sampled(tensors):
    return {k: t.reshape(-1)[sample_index(t.numel(), i).to(t.device)].cpu()
            for i, (k, t) in enumerate(zip(OUTPUTS, tensors))}


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: torch.from_numpy(z[k]) for k in z.files}


@pytest.mark.parametrize("name", sorted(CASES))
def test_matches_reference_cuda_kernels(golden, cuda_device, name):
    from trackformer_b200 import ext
    msda = ext.load()
    value, shapes, loc, attn, gout = case_inputs(name, cuda_device)
    out = msda.ms_deform_attn_forward(value, shapes, loc, attn, 64)
    gv, gl, ga = msda.ms_deform_attn_backward(value, shapes, loc, attn, gout, 64)
    got = sampled((out, gv, gl, ga))
    ref = {k: golden[f"{name}/{k}"] for k in OUTPUTS}
    scale = max(1.0, float(golden[f"{name}/grad_value_absmax"]))
    torch.testing.assert_close(got["out"], ref["out"], rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(got["grad_value"], ref["grad_value"], rtol=1e-4, atol=1e-4 * scale)
    torch.testing.assert_close(got["grad_attn"], ref["grad_attn"], rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(got["grad_loc"], ref["grad_loc"], rtol=5e-4, atol=5e-3)
