"""Records tests/golden/refcuda_samples.npz: the reference's own CUDA kernels (oracle/_ref/libmsda_refcuda.so, built by
``make -f oracle/Makefile ref`` from the reference sources) on the cases of tests/test_refcuda_gpu.py.

Needs a GPU and the built oracle/_ref library:  python tests/golden/make_golden_refcuda.py [OUT.npz]"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from oracle import refcuda  # noqa: E402
import test_refcuda_gpu as t  # noqa: E402


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else t.GOLDEN
    assert refcuda.available(), "oracle/_ref/libmsda_refcuda.so is not built"
    dev = torch.device("cuda:0")
    rec = {}
    for name in sorted(t.CASES):
        value, shapes, loc, attn, gout = t.case_inputs(name, dev)
        out = refcuda.forward(value, shapes, loc, attn)
        gv, gl, ga = refcuda.backward(value, shapes, loc, attn, gout)
        for k, v in t.sampled((out, gv, gl, ga)).items():
            rec[f"{name}/{k}"] = v.numpy().astype(np.float32)
        rec[f"{name}/grad_value_absmax"] = np.float32(gv.abs().max().item())
    np.savez_compressed(out_path, **rec)
    print("wrote", out_path, "on", torch.cuda.get_device_name(0))


if __name__ == "__main__":
    main()
