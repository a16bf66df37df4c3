"""trackformer_b200 -- H100-native (sm_90a) implementation of TrackFormer's per-frame hot path:
the Deformable-DETR encoder-decoder centred on the multi-scale deformable attention operator.

Layout
  csrc/            hand-written CUDA kernels + the C ABI (include/msda_b200.h) + pybind glue
  ext.py           loader for the in-tree extension (fails loudly when it is missing -- no CPU fallback)
  msda_function.py / msda_module.py   mirrors of the reference's MSDeformAttnFunction / MSDeformAttn

The package never imports anything from ``oracle/`` (test infrastructure).
"""
__version__ = "0.1.0"
