"""ORACLE / BASELINE -- TEST INFRASTRUCTURE ONLY (build container).

Stages the reference's Python model package and configs from /root/reference into the git-ignored
``baseline/_ref/`` so that they travel to the GPU box with the snapshot (the reference tree itself does not exist
there).  Nothing is copied into the repository's history; the product never imports it.  Used by
tools/ref_gpu_bench.py for (a) the zero-edit drop-in run -- the reference's own ``MSDeformAttn`` / ``DeformableDETR``
classes on this repo's ``MultiScaleDeformableAttention`` extension -- and (b) the "reference on the same GPU" arm
-- the same classes on the reference's own CUDA kernels (oracle/_ref).
"""
from __future__ import annotations

import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
DST = os.path.join(ROOT, "baseline", "_ref")


def stage(verbose: bool = False) -> bool:
    src_pkg = os.path.join(REF, "src", "trackformer")
    if not os.path.isdir(src_pkg):
        return False
    dst_pkg = os.path.join(DST, "src", "trackformer")
    for sub in ("models", "util"):
        shutil.copytree(os.path.join(src_pkg, sub), os.path.join(dst_pkg, sub), dirs_exist_ok=True,
                        ignore=shutil.ignore_patterns("__pycache__", "*.pyc", "build", "*.so"))
    shutil.copy2(os.path.join(src_pkg, "__init__.py"), os.path.join(dst_pkg, "__init__.py"))
    os.makedirs(os.path.join(DST, "cfgs"), exist_ok=True)
    for name in os.listdir(os.path.join(REF, "cfgs")):
        if name.endswith(".yaml"):
            shutil.copy2(os.path.join(REF, "cfgs", name), os.path.join(DST, "cfgs", name))
    if verbose:
        print("[stage_reference] ->", DST)
    return True


if __name__ == "__main__":
    print(stage(verbose=True))
