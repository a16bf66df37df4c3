"""MultiSequenceTracker on the H100: the batched decision kernel against single launches, and whole sequences through
the batched CUDA-graph detector against a DeviceTracker over GraphedDetector on each sequence alone."""
import numpy as np
import pytest
import torch

import multi_tracker_fixtures as mtf
import tracker_fixtures as tf
from test_tracker_gpu import _build, _probe_threshold

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


@pytest.mark.parametrize("n", [1, 3, 8, 16])
def test_batched_kernel_equals_single_launches(dev, n):
    """n scripted sequences of every case, each with its case's thresholds, the odd ones joining two steps late: one batched launch
    per step vs a DeviceTracker (one launch per sequence and frame) on each.  The post-processing kernel is row-wise,
    so both kernels see the same bits and must write the same bits: result rows, and the next state, queries and
    counters after every sequence's last frame."""
    from trackformer_b200.deformable_detr import DeformablePostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.multi_tracker import MultiSequenceTracker
    specs = mtf.sequence_specs(n, noise=False)
    dets = [make().to(dev) for _, make, _, _ in specs]
    tr = MultiSequenceTracker(mtf.Mux(dets).to(dev), {"bbox": DeformablePostProcess()}, tf.BASE_CFG, max_batch=n)
    its = {s: mtf.blobs(det, s, frames, public, dev) for s, ((_, _, frames, public), det) in enumerate(zip(specs, dets))}
    for step in range(tf.N_FRAMES + 2):
        batch = {}
        for s, it in its.items():
            if s % 2 and step < 2:
                continue
            if s not in tr._seqs:
                tr.start(s, specs[s][0])
            blob = next(it, None)
            if blob is not None:
                batch[s] = blob
        tr.step(batch)
    for s, (cfg, make, frames, public) in enumerate(specs):
        det = make().to(dev)
        ref = DeviceTracker(det, {"bbox": DeformablePostProcess()}, cfg, False)
        for blob in mtf.blobs(det, s, frames, public, dev):
            ref.step(blob)
        got = tr.sequence(s)
        a, b = tf.summarise(ref), tf.summarise(got)
        for key in a:
            np.testing.assert_array_equal(a[key], b[key], err_msg=f"sequence {s}: {key}")
        assert (got._n_active, got._n_inactive, got._n_query) == (ref._n_active, ref._n_inactive, ref._n_query)
        n_rows = ref._n_active + ref._n_inactive
        sa, sb = ref._bufs["state"][ref._cur], got._bufs["state"][got._cur]
        assert torch.equal(sa["header"], sb["header"])
        for name in sa:
            if name != "header":
                assert torch.equal(sa[name][:n_rows], sb[name][:n_rows]), (s, name)
        for name in ("q_boxes", "q_embeds"):
            assert torch.equal(ref._bufs[name][:ref._n_query], got._bufs[name][:got._n_query]), (s, name)


@pytest.mark.parametrize("multi_frame", [False, True])
def test_multi_tracker_equals_device_tracker_per_sequence(dev, multi_frame):
    """the small real model under CUDA-graph replay: three sequences of different seeds stepped together, the third
    joining two frames late (so a batch mixes images with and without a previous frame).  Each sequence equals a
    DeviceTracker over GraphedDetector on it alone: ids, frames, obj_ind, num_reids, active / inactive ids exactly,
    boxes and scores to the tolerance of the graph-replay test -- unless a decision of the single run sits closer to its
    threshold than the batch-size noise, which the recorded first frames measure (those are always compared).  Captures: one per distinct (B, kb, prev) key."""
    from trackformer_b200.deformable_detr import DeformablePostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.multi_tracker import MultiSequenceTracker
    import model_fixtures as mf
    build, size = _build(dev), (128, 160)
    thr = _probe_threshold(build, dev, multi_frame, size)
    cfg = dict(tf.BASE_CFG)
    cfg.update(detection_obj_score_thresh=thr, track_obj_score_thresh=thr * 0.97, reid_score_thresh=thr * 0.99,
               inactive_patience=3, reid_sim_threshold=2.0, detection_nms_thresh=0.7, track_nms_thresh=0.7)
    model, _ = build(True, multi_frame)
    mf.canonical_weights_(model, 0)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if "class_embed" in name and name.endswith("bias"):
                p[0] += 6.0
    model.to(dev)
    model.tracking()
    seeds, late, n_frames = (5, 7, 9), {2: 2}, 6

    def blob(frame):
        return {"img": frame[None].to(dev), "orig_size": torch.tensor([[size[0] * 4, size[1] * 4]])}

    class RowLog(DeformablePostProcess):                   # every frame's packed rows, all images of the call
        def __init__(self):
            super().__init__()
            self.log = []

        def packed(self, outputs, target_sizes):
            rows = super().packed(outputs, target_sizes)
            self.log.append(rows.cpu().numpy().copy())
            return rows

    det = GraphedDetector(model, bucket=16)
    multi_log = RowLog()
    tr = MultiSequenceTracker(det, {"bbox": multi_log}, cfg, max_batch=3)
    frames = {i: tf.model_frames(size, n_frames, seed) for i, seed in enumerate(seeds)}
    keys = set()
    with torch.no_grad():
        for step in range(n_frames + 2):
            batch = {}
            for i in frames:
                t = step - late.get(i, 0)
                if t == 0:
                    tr.start(i)
                if 0 <= t < n_frames:
                    batch[i] = blob(frames[i][t])
            captures = det.captures
            kb = det._padded_count(max(tr.sequence(i)._n_query for i in batch))
            prev = any(tr.sequence(i)._prev_features[0] is not None for i in batch)
            key = (len(batch), kb, prev and det.uses_prev)
            tr.step(batch)
            assert det.captures - captures == (key not in keys)      # a new prev_valid pattern is no new graph
            keys.add(key)
    nq = model.num_queries
    firsts = {0: multi_log.log[0][0, -nq:], 1: multi_log.log[0][1, -nq:], 2: multi_log.log[2][2, -nq:]}
    total = 0
    for i, seed in enumerate(seeds):
        post = RowLog()
        ref = DeviceTracker(GraphedDetector(model, bucket=16), {"bbox": post}, cfg, False)
        with torch.no_grad():
            for frame in frames[i]:
                ref.step(blob(frame))
        a, b = tf.summarise(ref), tf.summarise(tr.sequence(i))
        total += len(a["rows"])
        # each sequence's first frame (no track queries) through the batch-B graph vs the batch-1 graph
        np.testing.assert_array_equal(post.log[0][0, :, 1], firsts[i][:, 1])
        np.testing.assert_allclose(post.log[0][0], firsts[i], rtol=1e-4, atol=1e-3)
        # the batch-B forward sums in another order than batch 1 (cuBLAS / cuDNN pick other kernels): ids can only be
        # required to agree when no decision of the single-sequence run sits within that noise of its threshold
        scores = np.concatenate([r[0][r[0][:, 1] == 0, 0] for r in post.log])
        margin = min(float(np.abs(scores - cfg[t]).min())
                     for t in ("detection_obj_score_thresh", "track_obj_score_thresh", "reid_score_thresh"))
        noise = float(np.abs(post.log[0][0, :, 0] - firsts[i][:, 0]).max())
        print(f"sequence {i}: {len(a['rows'])} result rows; first-frame score difference batch {len(firsts)} vs 1: "
              f"{noise:.1e}; closest decision {margin:.1e} from its threshold")
        np.testing.assert_array_equal(a["frame_index"], b["frame_index"])
        if margin > 10 * noise:
            for key in ("num_reids", "track_num", "active_ids", "inactive_ids", "inactive_counts"):
                np.testing.assert_array_equal(a[key], b[key], err_msg=f"sequence {i}: {key}")
            np.testing.assert_array_equal(a["rows"][:, :3], b["rows"][:, :3])
            np.testing.assert_allclose(a["rows"][:, 3:], b["rows"][:, 3:], rtol=1e-4, atol=1e-3)
    assert total > 0
