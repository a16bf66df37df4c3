"""Segmentation masks for the scripted tracking scene of tests/tracker_fixtures.py, shared by the mask-fixture recorder
(tests/golden/make_golden_track_masks.py, which drives the reference Tracker) and the mask tests (which drive ours).

`MaskedScriptedDetector` is tracker_fixtures.ScriptedDetector plus `pred_masks` (stride-4 logits, MOTS tracking): every
row the scripted detector answers for an object gets a seeded elliptical logit field around that object's box, clutter
rows sit near -6, and designated (object, frame) pairs have an amplitude >= 40, so where two of them overlap the
sigmoids saturate to exactly 1.0 and tie.  Its boxes, logits and embeddings are the scripted detector's, unchanged.
`blobs` adds the padded input size "size" that the mask post-processing upsamples to.
"""
import numpy as np
import torch

import tracker_fixtures as tf

MASK_HW = (27, 37)                  # pred_masks grid of the scripted detector
MASK_SIZE = (118, 157)              # blob["size"]: the bilinear target (non-integer scales on both axes)


class MaskedScriptedDetector(tf.ScriptedDetector):
    def __init__(self, scene, **kwargs):
        super().__init__(scene, **kwargs)
        n_t = tf.N_FRAMES + 8
        mrng = np.random.RandomState(7)
        self.amp = mrng.uniform(3.0, 9.0, (n_t, scene.n)).astype(np.float32)
        self.stretch = mrng.uniform(1.0, 1.4, (n_t, scene.n, 2)).astype(np.float32)
        for t in range(n_t):
            for j in range(scene.n):
                if t % 4 == 1 or (j + t) % 5 == 0:
                    self.amp[t, j] = 40.0 + 10.0 * mrng.rand()
        self.clutter_masks = (-6.0 + 0.5 * mrng.standard_normal((n_t, self.num_queries) + MASK_HW)).astype(np.float32)

    def forward(self, img, targets=None, prev_features=None):
        sc, t = self.scene, self.frame
        res = super().forward(img, targets, prev_features)
        out = res[0]
        logits = out["pred_logits"][0].detach().cpu().numpy()
        followed = []
        if targets is not None:
            hs = targets[0]["track_query_hs_embeds"].detach().float().cpu().numpy()
            followed = list((hs @ sc.emb.T).argmax(1))
        k, nq = len(followed), self.num_queries
        masks = np.full((k + nq,) + MASK_HW, -6.0, np.float32)
        masks[k:] = self.clutter_masks[t]
        # the rows ScriptedDetector.forward answers: every track query, and the object-query row of each visible
        # object that is not tracked now (or that is tracked and duplicated this frame)
        for row, j in enumerate(followed):
            masks[row] = self.mask_field(j, t, sc.box(j, t))
        tracked_now = {j for row, j in enumerate(followed) if logits[row, 0] > 0 and logits[row, 3] < 0}
        for j in range(sc.n):
            if not sc.alive(j, t) or sc.occluded(j, t):
                continue
            if j not in tracked_now or (j, t) in sc.dup:
                masks[k + self.slot_of[t, j]] = self.mask_field(j, t, sc.box(j, t))
        out["pred_masks"] = torch.from_numpy(masks)[None].to(self.anchor.device)
        return res

    def mask_field(self, j, t, box):
        """amp * (1 - elliptical distance from the box centre), at least -6, on the MASK_HW grid (fp32)"""
        h, w = MASK_HW
        ys = ((np.arange(h, dtype=np.float32) + np.float32(0.5)) / np.float32(h))[:, None]
        xs = ((np.arange(w, dtype=np.float32) + np.float32(0.5)) / np.float32(w))[None, :]
        rx = np.float32(max(box[2], 0.02)) * self.stretch[t, j, 0] / np.float32(2)
        ry = np.float32(max(box[3], 0.02)) * self.stretch[t, j, 1] / np.float32(2)
        d = ((xs - box[0]) / rx) ** 2 + ((ys - box[1]) / ry) ** 2
        return np.maximum(self.amp[t, j] * (np.float32(1) - d), np.float32(-6)).astype(np.float32)


def blobs(scene, n_frames=tf.N_FRAMES):
    for blob in tf.blobs(scene, n_frames):
        blob["size"] = torch.tensor([list(MASK_SIZE)])
        yield blob


def label_maps(tracker, n_frames, size):
    """[F, H, W] int16: per frame the id of the result whose mask holds the pixel, -1 for none; masks are disjoint"""
    out = np.full((n_frames,) + tuple(size), -1, np.int16)
    for tid, frames in tracker.results.items():
        for f, r in frames.items():
            m = np.asarray(r["mask"])
            assert m.dtype == bool and m.shape == tuple(size), (m.dtype, m.shape)
            assert (out[f][m] == -1).all(), f"masks of frame {f} overlap"
            out[f][m] = tid
    return out


def run_case(tracker_cls, post, segm, case, device="cpu", seed=0):
    """tracker_fixtures.run_case with scripted masks and the `segm` post-processor; adds the per-frame label maps"""
    scene = tf.Scene(seed=seed)
    det = MaskedScriptedDetector(scene, overflow_boxes=tf.CASES[case]["overflow"]).to(device)
    tracker = tracker_cls(det, {"bbox": post, "segm": segm}, tf.tracker_cfg(case), False)
    tracker.reset()
    per_frame = []
    for blob in blobs(scene):
        tracker.step(blob)
        per_frame.append([t.id for t in tracker.tracks] + [-1] + [t.id for t in tracker.inactive_tracks])
    out = tf.summarise(tracker, det)
    width = max(len(p) for p in per_frame)
    out["per_frame_ids"] = np.asarray([p + [-2] * (width - len(p)) for p in per_frame], np.int64)
    out["labels"] = label_maps(tracker, tf.N_FRAMES, (tf.IMG_H, tf.IMG_W))
    return out


def run_model_sequence(build, tracker_cls, post, segm, cfg_overrides, size=(128, 160), n_frames=5, device="cpu",
                       out_lay_scale=1.0, wrap=None):
    """tracker_fixtures.run_model_sequence with the segmentation model (mask_head.out_lay scaled by `out_lay_scale`),
    the `segm` post-processor and blob["size"]; `wrap(model)` may put e.g. a GraphedDetector in between.  Adds the
    per-frame label maps."""
    import model_fixtures as mf
    model, _ = build(True, False, masks=True)
    mf.canonical_weights_(model, 0)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if "class_embed" in name and name.endswith("bias"):
                p[0] += 6.0
        model.mask_head.out_lay.weight.mul_(out_lay_scale)
        model.mask_head.out_lay.bias.mul_(out_lay_scale)
    model.to(device)
    model.tracking()
    cfg = dict(tf.BASE_CFG)
    cfg.update(cfg_overrides)
    tracker = tracker_cls(model if wrap is None else wrap(model), {"bbox": post, "segm": segm}, cfg, False)
    tracker.reset()
    orig = (size[0] * 4, size[1] * 4)
    with torch.no_grad():
        for frame in tf.model_frames(size, n_frames):
            tracker.step({"img": frame[None], "orig_size": torch.tensor([list(orig)]), "dets": torch.zeros(1, 0, 4),
                          "size": torch.tensor([list(size)])})
    out = tf.summarise(tracker)
    out["labels"] = label_maps(tracker, n_frames, orig)
    return out
