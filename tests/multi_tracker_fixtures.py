"""Shared pieces of the MultiSequenceTracker tests.

`Mux` is a batched detector over per-sequence scripted detectors (tracker_fixtures.ScriptedDetector, or the noise
detector of test_track_step_cpu): each image carries its sequence's number in its pixels, and image b's answer is
that sequence's detector's answer, laid out as `GraphedDetector.batched` lays it out (its K_b track-query rows at the
end of the kb padded slots, then the object queries).  So a MultiSequenceTracker over a Mux and one tracker per
sequence over that sequence's own detector see the same detections, and any difference is the bookkeeping's.
"""

import numpy as np
import torch

import host_twin
import tracker_fixtures as tf

NQ, HIDDEN, CLASSES = 20, 32, 20


class Mux(torch.nn.Module):
    num_queries, hidden_dim, overflow_boxes = NQ, HIDDEN, True

    def __init__(self, detectors, bucket=4):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))
        self.dets, self.bucket = detectors, bucket

    def batched(self, samples, targets, prev_features):
        ids = samples[:, 0, 0, 0].long().tolist()
        ks = [0 if t is None else int(t["track_query_boxes"].shape[0]) for t in targets]
        kb = -(-max(ks) // self.bucket) * self.bucket
        dev = self.p.device
        logits = torch.full((len(ids), kb + NQ, CLASSES), -30.0, device=dev)
        boxes = torch.full((len(ids), kb + NQ, 4), 0.5, device=dev)
        embeds = torch.zeros(len(ids), kb + NQ, HIDDEN, device=dev)
        for b, (i, t, k) in enumerate(zip(ids, targets, ks)):
            out = self.dets[i](None, None if t is None else [t], None)[0]
            c = out["pred_logits"].shape[-1]
            logits[b, kb - k:, :c] = out["pred_logits"][0]
            boxes[b, kb - k:] = out["pred_boxes"][0]
            embeds[b, kb - k:] = out["hs_embed"][0]
        return {"pred_logits": logits, "pred_boxes": boxes, "hs_embed": embeds}, None, ks, kb


def sequence_specs(n, n_frames=tf.N_FRAMES, noise=True):
    """n sequences: scripted scenes of every case and (with `noise`; host tensors only) random-noise scenes, each with
    its own thresholds, length and seed.  Returns [(cfg, make_detector, n_frames, public_from_detector)]."""
    from test_track_step_cpu import _RandomDetector
    specs = []
    cases = list(tf.CASES)
    for s in range(n):
        if noise and s % 3 == 2:
            rng = np.random.RandomState(s)
            cfg = dict(tf.BASE_CFG)
            cfg.update(public_detections=[False, "center_distance", "min_iou_0_5"][(s // 3) % 3],
                       detection_obj_score_thresh=float(rng.uniform(0.5, 0.8)),
                       track_obj_score_thresh=float(rng.uniform(0.4, 0.7)), reid_score_thresh=float(rng.uniform(0.4, 0.8)),
                       detection_nms_thresh=float(rng.choice([0.0, 0.3, 0.6])),
                       track_nms_thresh=float(rng.choice([0.0, 0.4, 0.7])), steps_termination=int(rng.randint(1, 3)),
                       inactive_patience=int(rng.randint(1, 6)), reid_greedy_matching=bool(s % 2),
                       reid_sim_threshold=float(rng.choice([0.0, 3.0, 6.0])), reid_sim_only=s % 5 == 4)
            specs.append((cfg, lambda s=s: _RandomDetector(s, num_queries=NQ, hidden=HIDDEN), n_frames - s % 4, True))
        else:
            case = cases[s % len(cases)]
            scene = tf.Scene(seed=s)
            specs.append((tf.tracker_cfg(case), lambda scene=scene: tf.ScriptedDetector(scene), n_frames - s % 5, False))
    return specs


def blobs(det, seq_id, n_frames, scene_public, device="cpu"):
    """the frames of one sequence: the image carries the sequence number; 'dets' is read after the forward"""
    for t in range(n_frames):
        class Blob(dict):
            def __getitem__(self, key):
                if key == "dets" and scene_public:
                    return det.public
                return dict.__getitem__(self, key)
        dets = (torch.from_numpy(det.scene.public_dets(t))[None] if not scene_public else None)
        yield Blob(img=torch.full((1, 3, 8, 8), float(seq_id), device=device), orig_size=torch.tensor([[480, 640]]),
                   dets=dets)


def build_host(tmp, name):
    return host_twin.build(name, tmp)


def output_spans(a):
    """(address, bytes) of everything one step may write -- both state buffers (the routine also updates the
    incoming state's anchors), the next-frame queries, the integer scratch and the header + result rows"""
    cap, hid = a.capacity, a.hidden
    spans = []
    for st in (a.inp, a.out):
        spans += [(st.header, 32), (st.ids, 4 * cap), (st.pos, 16 * cap), (st.anchor, 16 * cap), (st.score, 4 * cap),
                  (st.obj_ind, 4 * cap), (st.count_inactive, 4 * cap), (st.count_termination, 4 * cap),
                  (st.bank, 4 * cap * hid)]
    spans += [(a.q_boxes, 16 * cap), (a.q_embeds, 4 * cap * hid), (a.iscratch, 64 * cap),
              (a.result, 4 * (8 + 8 * (a.n_query + a.nq)))]
    return spans
