#!/usr/bin/env python
"""Tracker segmentation-mask fixtures recorded FROM THE REFERENCE (build container only).

Runs the unmodified reference `Tracker` (src/trackformer/models/tracker.py) with the reference's `DeformablePostProcess`
and `PostProcessSegm` on CPU and stores, next to the summary of tests/golden/make_golden_tracker.py, the per-frame
label maps of the results' masks ([F, H, W], track id or -1):

  * tracker_masks_<case>.npz for every case of tracker_fixtures.CASES: the scripted detector with the masks of
    tests/track_mask_fixtures.py (seeded elliptical logit fields, saturated pairs that tie exactly, stale masks
    through steps_termination=2 in `reid_embedding`).

The existing tracker_<case>.npz files are not touched.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE)))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
sys.path.insert(0, HERE)


def main():
    from make_golden_model import import_reference
    import_reference()
    from trackformer.models.tracker import Tracker
    from trackformer.models.deformable_detr import DeformablePostProcess
    from trackformer.models.detr_segmentation import PostProcessSegm
    import track_mask_fixtures as tmf
    import tracker_fixtures as tf
    for case in tf.CASES:
        out = tmf.run_case(Tracker, DeformablePostProcess(), PostProcessSegm(), case)
        np.savez_compressed(os.path.join(HERE, f"tracker_masks_{case}.npz"), **out)
        lab = out["labels"]
        print(f"masks {case}: {len(out['rows'])} result rows, labelled pixels per frame "
              f"{(lab >= 0).sum((1, 2)).tolist()}")


if __name__ == "__main__":
    main()
