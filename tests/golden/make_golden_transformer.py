#!/usr/bin/env python
"""Vanilla-transformer golden fixtures recorded FROM THE REFERENCE (build container only).

Runs the unmodified reference ``Transformer`` (src/trackformer/models/transformer.py) on CPU in fp32,
driven by the shared runner of tests/transformer_fixtures.py, for the post-norm (train.yaml) and pre-norm layers, and
stores tests/golden/transformer_{post,pre}.npz with the outputs, the gradients of a seeded weighted sum and the
state_dict key names and shapes of the six-layer model.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import transformer_fixtures as tf
    sys.path.insert(0, HERE)
    from make_golden_model import import_reference
    import_reference()                                  # stubs visdom and the compiled extension
    from trackformer.models.transformer import Transformer
    for mode, pre_norm in (("post", False), ("pre", True)):
        res = tf.run_transformer(Transformer, pre_norm)
        res["state_dict_shapes"] = np.asarray(json.dumps(tf.state_dict_shapes(Transformer, pre_norm)))
        path = os.path.join(HERE, f"transformer_{mode}.npz")
        np.savez(path, **res)
        print(f"{mode:5s} -> {os.path.relpath(path)} ({os.path.getsize(path) / 1024:.0f} KiB)", flush=True)


if __name__ == "__main__":
    main()
