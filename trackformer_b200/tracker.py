"""Online multi-object tracker driven by track queries.

Host-side mirror of src/trackformer/models/tracker.py:16-581 (`Tracker`, `Track`): same constructor, `reset`, `step(blob)`,
`get_results`, the same `tracker_cfg` keys (cfgs/track.yaml:27-50) and the same decisions frame by frame -- score
thresholds for keeping / re-identifying / starting tracks (tracker.py:337-373, 425-436), both NMS passes (388-406,
494-515), public-detection gating (122-164), ReID by embedding distance or greedy centre distance (166-264), the
`reid_sim_only` mode (547-548) and the result dictionary (533-545).

What is different is where the state lives.  The reference keeps one Python `Track` object per target whose fields are
device tensors, and reads them back one `.cpu()` at a time (several host synchronisations per track per frame).  Here
the per-target state is a struct of arrays:

  * output embeddings (the only state the detector consumes) stay in ONE device tensor, `_hs[slot]`, gathered into the
    next frame's track queries with one index_select and updated with one index_copy per frame;
  * boxes, scores, counters and ids live in host arrays (fp32 / int64, the very values the detector produced);
  * a frame costs ONE device->host copy: the packed rows {score, label, x0, y0, x1, y1} written by the fused
    post-processing kernel (csrc/track_post.cu) -- plus one more (the distance matrix) only when ReID has candidates.

All decisions are then taken on those host arrays in fp32, in the reference's order, so track ids, `obj_ind`,
`num_reids` and the frame sets of the results are identical and boxes / scores are the detector's values bit for bit.

Segmentation masks (MOTS, on when `obj_detector_post` has a "segm" entry; tracker.py:311-321, 333-373, 419-466,
509-538).  The reference runs the mask head on every query row, upsamples every row to the image size, copies all of
it to the host and then uses the few rows that end the frame as active tracks.  Here a track takes a new mask exactly
where it takes a new embedding (`hs_writes`), so after the decisions the mask head runs on those rows only
(`mask_logits` of a segmentation model, or `GraphedDetector.mask_logits`), and `resolve_track_masks`
(csrc/track_masks.cu on the GPU) resolves the overlaps of all active tracks at the original resolution into one label
map -- the frame's only extra read-back.  A track that keeps its previous mask reads it from the previous label map,
which stays on the device.  `results[id][frame]["mask"]` is the reference's bool array [H, W], or with
`mask_rle=True` its COCO RLE dict (`mots.encode`'s format, what the MOTS20 result file holds), made from the device label
map by csrc/mask_rle.cu so that only the strings are read back (`mots.decode` gives the array); `Track.mask` is the
frame's resolved bool mask for active tracks and None for inactive ones (the reference keeps an inactive track's last
mask, which nothing reads: a track that comes back always takes a new one).

Attention maps (`generate_attention_maps=True`, tracker.py:37-60, 335-481, 539-541; vanilla DETR models only, as in the
reference).  The detector's `generate_attention_maps` switch makes its forward return `out["attention_maps"]`
[1, Q, h, w], the last decoder layer's cross-attention weights averaged over heads.  A track takes a new map exactly
where it takes a new embedding (`hs_writes`), else keeps the one it had; after the decisions the maps of the result
rows are gathered on the device and read back in one copy.  `results[id][frame]["attention_map"]` is that float32
[h, w] array; `Track.attention_map` is the frame's map (a host tensor) for active tracks and None for inactive ones,
like `Track.mask`.
"""
from collections import deque

import numpy as np
import torch
import torch.nn.functional as F
from scipy.optimize import linear_sum_assignment

from .graphed_detector import GraphedDetector
from .mots import label_map_rle
from .segmentation import resolve_track_masks

__all__ = ["Tracker", "Track", "nms_keep", "pairwise_iou"]


# ------------------------------------------------------------------------------------------------ fp32 box helpers
def _to_cxcywh(xyxy: np.ndarray) -> np.ndarray:
    """util/box_ops.py:18-22 in fp32."""
    x0, y0, x1, y1 = (xyxy[..., k] for k in range(4))
    return np.stack([(x0 + x1) / np.float32(2), (y0 + y1) / np.float32(2), x1 - x0, y1 - y0], axis=-1).astype(np.float32)


def _clip(xyxy: np.ndarray, height, width) -> np.ndarray:
    """torchvision.ops.boxes.clip_boxes_to_image for size (height, width)."""
    out = xyxy.copy()
    out[..., 0::2] = np.clip(out[..., 0::2], np.float32(0), np.float32(width))
    out[..., 1::2] = np.clip(out[..., 1::2], np.float32(0), np.float32(height))
    return out


def pairwise_iou(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """torchvision.ops.box_iou in fp32: [len(a), len(b)]."""
    a, b = a.astype(np.float32, copy=False), b.astype(np.float32, copy=False)
    area_a = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    area_b = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    lt = np.maximum(a[:, None, :2], b[None, :, :2])
    rb = np.minimum(a[:, None, 2:], b[None, :, 2:])
    wh = np.clip(rb - lt, np.float32(0), None)
    inter = wh[..., 0] * wh[..., 1]
    return inter / (area_a[:, None] + area_b[None, :] - inter)


def nms_keep(boxes: np.ndarray, scores: np.ndarray, threshold: float) -> np.ndarray:
    """Boolean keep mask of greedy NMS, torchvision.ops.nms semantics: visit boxes by descending score (stable, so equal
    scores -- e.g. the +inf given to established tracks, tracker.py:503 -- keep their list order) and suppress every later
    box whose IoU with a kept one EXCEEDS `threshold`; arithmetic in fp32 like the torchvision kernels."""
    n = len(boxes)
    keep = np.zeros(n, dtype=bool)
    if n == 0:
        return keep
    boxes = boxes.astype(np.float32, copy=False)
    order = np.argsort(-scores.astype(np.float32, copy=False), kind="stable")
    area = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1])
    dead = np.zeros(n, dtype=bool)
    thr = np.float32(threshold)
    for pos, i in enumerate(order):
        if dead[i]:
            continue
        keep[i] = True
        rest = order[pos + 1:]
        rest = rest[~dead[rest]]
        if len(rest) == 0:
            continue
        w = np.clip(np.minimum(boxes[i, 2], boxes[rest, 2]) - np.maximum(boxes[i, 0], boxes[rest, 0]), np.float32(0), None)
        h = np.clip(np.minimum(boxes[i, 3], boxes[rest, 3]) - np.maximum(boxes[i, 1], boxes[rest, 1]), np.float32(0), None)
        inter = w * h
        with np.errstate(invalid="ignore", divide="ignore"):
            iou = inter / (area[i] + area[rest] - inter)
        dead[rest[iou > thr]] = True
    return keep


# ---------------------------------------------------------------------------------------------------- track views
class Track:
    """Read-only view of one target with the reference's field names (tracker.py:555-581).  `pos`, `score` and `obj_ind`
    are host values; `hs_embed` is a one-element list holding the device embedding."""

    def __init__(self, tracker, slot):
        s = tracker._state
        self.id = int(s.ids[slot])
        self.pos = torch.from_numpy(s.pos[slot].copy())
        self.last_pos = deque([torch.from_numpy(s.anchor[slot].copy())])
        self.score = torch.tensor(s.score[slot])
        self.count_inactive = int(s.count_inactive[slot])
        self.count_termination = int(s.count_termination[slot])
        self.obj_ind = torch.tensor([int(s.obj_ind[slot])])
        self.hs_embed = [tracker._embedding_of(slot)]
        self.gt_id = None
        self.mask = tracker._mask_of(slot)
        self.attention_map = tracker._attention_map_of(slot)

    def has_positive_area(self) -> bool:
        return bool(self.pos[2] > self.pos[0] and self.pos[3] > self.pos[1])


class _State:
    """Host half of the struct of arrays; grows by doubling."""

    def __init__(self, capacity=64):
        self.capacity = capacity
        self.pos = np.zeros((capacity, 4), np.float32)
        self.anchor = np.zeros((capacity, 4), np.float32)      # = last_pos[-1] of the reference's Track
        self.score = np.zeros(capacity, np.float32)
        self.obj_ind = np.zeros(capacity, np.int64)
        self.ids = np.full(capacity, -1, np.int64)
        self.count_inactive = np.zeros(capacity, np.int64)
        self.count_termination = np.zeros(capacity, np.int64)

    def grow(self):
        for name in ("pos", "anchor", "score", "obj_ind", "ids", "count_inactive", "count_termination"):
            old = getattr(self, name)
            new = np.zeros((2 * self.capacity,) + old.shape[1:], old.dtype)
            if name == "ids":
                new[:] = -1
            new[:self.capacity] = old
            setattr(self, name, new)
        self.capacity *= 2


class Tracker:
    """Drop-in for trackformer.models.tracker.Tracker (same arguments, tracker.py:19-20)."""

    def __init__(self, obj_detector, obj_detector_post, tracker_cfg, generate_attention_maps=False, logger=None,
                 verbose=False, frame_ingest=None, mask_rle=False):
        self.obj_detector = obj_detector
        self.frame_ingest = frame_ingest      # FrameIngest for blobs that carry a raw "frame"; made on first use if None
        self.obj_detector_post = obj_detector_post
        self.detection_obj_score_thresh = tracker_cfg["detection_obj_score_thresh"]
        self.track_obj_score_thresh = tracker_cfg["track_obj_score_thresh"]
        self.detection_nms_thresh = tracker_cfg["detection_nms_thresh"]
        self.track_nms_thresh = tracker_cfg["track_nms_thresh"]
        self.public_detections = tracker_cfg["public_detections"]
        self.inactive_patience = float(tracker_cfg["inactive_patience"])
        self.reid_sim_threshold = tracker_cfg["reid_sim_threshold"]
        self.reid_sim_only = tracker_cfg["reid_sim_only"]
        self.reid_score_thresh = tracker_cfg["reid_score_thresh"]
        self.reid_greedy_matching = tracker_cfg["reid_greedy_matching"]
        self.prev_frame_dist = tracker_cfg["prev_frame_dist"]
        self.steps_termination = tracker_cfg["steps_termination"]
        if generate_attention_maps:
            # the reference asserts the same (tracker.py:38): only a vanilla decoder has a multihead_attn to read
            layers = getattr(getattr(getattr(obj_detector, "transformer", None), "decoder", None), "layers", None)
            if not layers or not hasattr(layers[-1], "multihead_attn"):
                raise ValueError("Generation of attention maps not possible for deformable DETR.")
        if hasattr(obj_detector, "generate_attention_maps"):
            # the detector's switch follows the tracker that drives it: one built without maps turns it back off
            obj_detector.generate_attention_maps = bool(generate_attention_maps)
        self.masks = "segm" in obj_detector_post
        self.mask_rle = bool(mask_rle)        # results' "mask": COCO RLE dicts (mots.label_map_rle) instead of bool arrays
        self.generate_attention_maps = bool(generate_attention_maps)
        self._logger = logger if logger is not None else (lambda *log_strs: None)
        self._verbose = verbose
        self._pinned = None
        self.reset()

    # ------------------------------------------------------------------------------------------------ accessors
    @property
    def num_object_queries(self):
        return self.obj_detector.num_queries

    @property
    def device(self):
        return next(self.obj_detector.parameters()).device

    @property
    def tracks(self):
        return [Track(self, s) for s in self._active]

    @property
    def inactive_tracks(self):
        return [Track(self, s) for s in self._inactive]

    def get_results(self):
        return self.results

    def reset(self, hard=True):
        """tracker.py:71-80"""
        self._label = None                    # [H, W] int32 device label map of the last frame's masks
        self._maps = {}                       # track id -> float32 [h, w] attention map, for the last frame's results
        self._state = _State()
        self._hs = None                       # [capacity, hidden] device embeddings, allocated at the first detection
        self._active, self._inactive = [], []
        self._free = list(range(self._state.capacity - 1, -1, -1))
        self._prev_features = deque([None], maxlen=self.prev_frame_dist)
        if hard:
            self.track_num = 0
            self.results = {}
            self.frame_index = 0
            self.num_reids = 0

    # ------------------------------------------------------------------------------------------------- internals
    def _embedding_of(self, slot):
        return self._hs[slot] if self._hs is not None else None

    def _attention_map_of(self, slot):
        if slot not in self._active:
            return None
        m = self._maps.get(int(self._state.ids[slot]))
        return None if m is None else torch.from_numpy(m)

    def _attention_maps(self, det_out, src_rows, ids):
        """This frame's maps of the result tracks (ids, in order): `src_rows[t]` is the query row whose map track t
        takes, -1 to keep its previous one.  The new rows are gathered on the device and read back in one copy."""
        maps = det_out[0]["attention_maps"][0]
        fresh = [k for k, r in enumerate(src_rows) if r >= 0]
        host = None
        if fresh:
            rows = torch.as_tensor([int(src_rows[k]) for k in fresh], dtype=torch.long).to(maps.device)
            host = maps.index_select(0, rows).float().cpu().numpy()
        return self._book_maps(src_rows, ids, host)

    def _book_maps(self, src_rows, ids, host):
        """Keep this frame's maps: `host` [n, h, w] holds the new maps of the tracks with `src_rows[t] >= 0`, in order;
        the other tracks keep theirs.  Returns the maps in `ids` order (None for a track that never had one)."""
        new, j = {}, 0
        for k, tid in enumerate(ids):
            tid = int(tid)
            if src_rows[k] >= 0:
                new[tid] = host[j]
                j += 1
            elif tid in self._maps:
                new[tid] = self._maps[tid]
        self._maps = new
        return [new.get(int(tid)) for tid in ids]

    def _mask_of(self, slot):
        if self._label is None or slot not in self._active:
            return None
        return self._label == int(self._state.ids[slot])

    def _with_image(self, blob):
        """The blob `step` works on.  A blob with "img" is returned as it is.  One with "frame" -- the raw uint8
        [H, W, 3] RGB video frame, host or device -- gets "img", "size" and "orig_size" from the frame ingest
        (frame_ingest.py: the reference's validation transform on the GPU, bit for bit); its other entries, e.g. the
        public detections "dets" in original-image pixels, keep their meaning."""
        if "frame" not in blob:
            return blob
        if "img" in blob:
            raise ValueError('Tracker.step: the blob has both "img" and "frame"; give the pre-processed image or the '
                             'raw uint8 frame, not both')
        if self.frame_ingest is None:
            from .frame_ingest import FrameIngest
            self.frame_ingest = FrameIngest(self.device)
        out = {k: v for k, v in blob.items() if k != "frame"}
        out.update(self.frame_ingest(blob["frame"]))
        return out

    def _detect(self, img, target, prev_features):
        """The detector call; with masks on, a segmentation model runs without its mask head (`detect`)."""
        if self.masks and callable(getattr(self.obj_detector, "mask_logits", None)):
            return self.obj_detector.detect(img, target, prev_features)
        return self.obj_detector(img, target, prev_features)

    def _mask_rows(self, det_out, rows):
        """[len(rows), h, w] mask logits of the query rows `rows` of this frame's detector call."""
        det = self.obj_detector
        if isinstance(det, GraphedDetector):
            return det.mask_logits(rows)[0]
        if callable(getattr(det, "mask_logits", None)):
            _, _, features, memory, hs = det_out
            return det.mask_logits(features, memory, hs, rows)[0]
        masks = det_out[0]["pred_masks"][0]           # any reference-shaped detector: the full head's output
        return masks.index_select(0, torch.as_tensor(rows, dtype=torch.long, device=masks.device))

    def _mask_job(self, src_rows, ids, blob, orig):
        """What resolving this frame's masks takes, for the active tracks `ids` (list order) with `src_rows[t]` the query
        row whose mask track t takes (-1: it keeps its previous one): `(rows, src, prev, size)` -- the sorted query rows
        the mask head must compute, each track's index into them (-1 when stale), the previous label map when a track
        is stale (else None) and the padded input size.  None when no track is active."""
        if not len(ids):
            return None
        stale = any(r < 0 for r in src_rows)
        if stale and (self._label is None or tuple(self._label.shape) != tuple(orig)):
            # the reference fails here too (torch.stack of masks of different sizes, tracker.py:510)
            raise ValueError(f"orig_size changed to {tuple(orig)} while tracks keep their masks of size "
                             f"{None if self._label is None else tuple(self._label.shape)}")
        rows = sorted({int(r) for r in src_rows if r >= 0})
        index = {r: i for i, r in enumerate(rows)}
        src = [index[int(r)] if r >= 0 else -1 for r in src_rows]
        size = [int(v) for v in blob["size"].reshape(-1, 2)[0].tolist()]
        return rows, src, (self._label if stale else None), size

    def _resolve_masks(self, det_out, src_rows, ids, blob, orig):
        """Masks of the active tracks (ids, in list order) of this frame: `src_rows[t]` is the query row whose mask
        track t takes, -1 to keep its previous one.  Returns the results' masks in `ids` order: bool arrays [H, W] from
        the host label map (the one read-back), or with `mask_rle` the COCO RLEs made from the device label map."""
        job = self._mask_job(src_rows, ids, blob, orig)
        if job is None:
            self._label = None
            return []
        rows, src, prev, size = job
        if rows:
            logits = self._mask_rows(det_out, rows)
        else:
            logits = torch.zeros(0, 1, 1, device=self._label.device)
        self._label = resolve_track_masks(logits, src, [int(i) for i in ids], prev, size, size, orig)
        if self.mask_rle:
            return label_map_rle(self._label, ids)
        host = self._label.cpu().numpy()
        return [host == i for i in ids]

    def _take_slot(self):
        if not self._free:
            old = self._state.capacity
            self._state.grow()
            self._free = list(range(2 * old - 1, old - 1, -1))
            if self._hs is not None:
                self._hs = torch.cat([self._hs, torch.zeros_like(self._hs)], 0)
        return self._free.pop()

    def _alive(self, slot) -> bool:
        """has_positive_area and still within the patience window (tracker.py:171-174, 270-273)"""
        p = self._state.pos[slot]
        return bool(p[2] > p[0] and p[3] > p[1]) and self._state.count_inactive[slot] <= self.inactive_patience

    def _prune_inactive(self, released):
        kept = [s for s in self._inactive if self._alive(s)]
        released.extend(s for s in self._inactive if s not in kept)
        self._inactive = kept

    def _deactivate(self, slots):
        """tracker.py:86-91: back to the position at the start of the step, then onto the inactive list"""
        gone = set(slots)
        self._active = [s for s in self._active if s not in gone]
        for s in slots:
            self._state.pos[s] = self._state.anchor[s]
        self._inactive += list(slots)

    def _packed_rows(self, outputs, orig_size):
        """One [Q, 6] host array {score, label, x0, y0, x1, y1} for the (single) image of this step."""
        post = self.obj_detector_post["bbox"]
        if hasattr(post, "packed"):
            rows = post.packed(outputs, orig_size)[0]
        else:                                   # any reference-shaped post-processor
            res = post(outputs, orig_size)[0]
            rows = torch.cat([res["scores"][:, None], res["labels"][:, None].float(), res["boxes"]], 1)
        if rows.is_cuda:
            if self._pinned is None or self._pinned.shape[0] < rows.shape[0]:
                self._pinned = torch.empty(max(1024, rows.shape[0]), 6, dtype=torch.float32).pin_memory()
            host = self._pinned[:rows.shape[0]]
            host.copy_(rows, non_blocking=True)
            torch.cuda.current_stream(rows.device).synchronize()
            return host.numpy().copy()
        return rows.detach().float().numpy().copy()

    # ------------------------------------------------------------------------------------- public detections gating
    def public_detections_mask(self, new_boxes, public_boxes):
        """tracker.py:122-164 on host arrays."""
        n = len(new_boxes)
        if not self.public_detections:
            return np.ones(n, dtype=bool)
        mask = np.zeros(n, dtype=bool)
        if not len(public_boxes) or not n:
            return mask
        public_boxes = np.asarray(public_boxes, dtype=np.float32).reshape(-1, 4)
        if self.public_detections == "center_distance":
            size = ((new_boxes[:, 2] - new_boxes[:, 0]) * (new_boxes[:, 3] - new_boxes[:, 1])).astype(np.float32)
            d = _to_cxcywh(new_boxes)[:, None, :2] - _to_cxcywh(public_boxes)[None, :, :2]
            d = (d ** 2).sum(axis=2)
            for j in range(len(public_boxes)):
                i = d[:, j].argmin()
                if d[i, j] < size[i]:
                    d[i, :] = 1e18
                    mask[i] = True
        elif self.public_detections == "min_iou_0_5":
            iou = pairwise_iou(new_boxes, public_boxes)
            for j in range(len(public_boxes)):
                i = iou[:, j].argmax()
                if iou[i, j] >= 0.5:
                    iou[i, :] = 0
                    mask[i] = True
        else:
            raise NotImplementedError
        return mask

    # ------------------------------------------------------------------------------------------------------ ReID
    def reid(self, new_boxes, new_scores, new_query_idx, hs_embeds, hs_writes, released):
        """tracker.py:166-264.  Returns the mask of detections NOT consumed by a re-identified track."""
        st = self._state
        self._prune_inactive(released)
        n = len(new_boxes)
        free_mask = np.ones(n, dtype=bool)
        if not self._inactive or not n:
            return free_mask
        if self.reid_greedy_matching:
            det = _to_cxcywh(new_boxes)
            old = _to_cxcywh(st.pos[self._inactive])
            dist = old[:, None, :2] - det[None, :, :2]
            dist = (dist ** 2).sum(axis=2)
            track_size, item_size = old[:, 2] * old[:, 3], det[:, 2] * det[:, 3]
            invalid = (dist > track_size[:, None]) + (dist > item_size[None, :])
            dist = dist + invalid * 1e18
            work = dist                         # the reference's greedy pass edits the matrix it later thresholds
            rows, cols = [], []
            for i in range(work.shape[0]):
                j = work[i].argmin()
                if work[i][j] < 1e16:
                    work[:, j] = 1e18
                    work[i, j] = 0.0
                    rows.append(i)
                    cols.append(j)
        else:
            # L2 distance of the last output embeddings, F.pairwise_distance semantics (eps inside the norm)
            old = self._hs.index_select(0, torch.as_tensor(self._inactive, device=self._hs.device))
            new = hs_embeds.index_select(0, torch.as_tensor(new_query_idx, device=hs_embeds.device))
            c = old.shape[1]
            dist = F.pairwise_distance(old[:, None, :].expand(-1, n, -1).reshape(-1, c),
                                       new[None, :, :].expand(len(self._inactive), -1, -1).reshape(-1, c))
            dist = dist.view(len(self._inactive), n).cpu().numpy()
            rows, cols = linear_sum_assignment(dist)
        revived = []
        for r, c in zip(rows, cols):
            if dist[r, c] <= self.reid_sim_threshold:
                slot = self._inactive[r]
                self._logger(f"REID: track.id={st.ids[slot]} - count_inactive={st.count_inactive[slot]} - "
                             f"to_inactive_frame={self.frame_index - st.count_inactive[slot]}")
                st.count_inactive[slot] = 0
                st.pos[slot] = new_boxes[c]
                st.anchor[slot] = new_boxes[c]
                st.score[slot] = new_scores[c]
                hs_writes[slot] = int(new_query_idx[c])
                free_mask[c] = False
                revived.append(slot)
                self._active.append(slot)
                self.num_reids += 1
        self._inactive = [s for s in self._inactive if s not in revived]
        return free_mask

    # ------------------------------------------------------------------------------------------------------ step
    @torch.no_grad()
    def step(self, blob):
        """One frame (tracker.py:266-548).  `blob` holds the pre-processed "img" (with "orig_size", and "size" when
        masks are on) or the raw uint8 "frame" (`_with_image`)."""
        blob = self._with_image(blob)
        st = self._state
        released = []                            # slots freed during this step; recycled only afterwards
        hs_writes = {}                           # slot -> query index whose embedding the slot takes this frame
        self._prune_inactive(released)
        self._logger(f"FRAME: {self.frame_index + 1}")
        if self._inactive:
            self._logger(f"INACTIVE TRACK IDS: {[int(st.ids[s]) for s in self._inactive]}")
        for s in self._active:
            st.anchor[s] = st.pos[s]

        dev = self.device
        img = blob["img"].to(dev)
        orig_size = blob["orig_size"]
        height, width = (int(v) for v in orig_size[0].tolist())
        orig_size = orig_size.to(dev)

        order = self._active + self._inactive
        n_prev = len(order)
        target = None
        if n_prev:
            q_boxes = _to_cxcywh(st.pos[order]) / np.array([width, height, width, height], dtype=np.float32)
            target = [{
                "track_query_boxes": torch.from_numpy(q_boxes).to(dev),
                "image_id": torch.tensor([1]).to(dev),
                "track_query_hs_embeds": self._hs.index_select(0, torch.as_tensor(order, device=dev)),
            }]

        det_out = self._detect(img, target, self._prev_features[0])
        outputs, _, features, _, _ = det_out
        hs_embeds = outputs["hs_embed"][0]
        rows = self._packed_rows(outputs, orig_size)
        scores, labels = rows[:, 0], rows[:, 1]
        boxes = rows[:, 2:6] if self.obj_detector.overflow_boxes else _clip(rows[:, 2:6], height, width)
        nq = self.num_object_queries
        n_total = rows.shape[0]
        if self._hs is None:
            self._hs = torch.zeros(st.capacity, hs_embeds.shape[1], dtype=hs_embeds.dtype, device=hs_embeds.device)

        # ---- established tracks and re-identification queries (tracker.py:329-406)
        if n_prev:
            t_scores, t_boxes, t_person = scores[:-nq], boxes[:-nq], labels[:-nq] == 0
            keep = np.logical_and(t_scores > self.track_obj_score_thresh, t_person)
            to_inactive = []
            for i, s in enumerate(self._active):
                if keep[i]:
                    st.score[s], st.pos[s] = t_scores[i], t_boxes[i]
                    hs_writes[s] = i
                    st.count_termination[s] = 0
                else:
                    st.count_termination[s] += 1
                    if st.count_termination[s] >= self.steps_termination:
                        to_inactive.append(s)
            keep = np.logical_and(t_scores > self.reid_score_thresh, t_person)
            from_inactive = []
            for i, s in enumerate(self._inactive, start=len(self._active)):
                if keep[i]:
                    st.score[s], st.pos[s] = t_scores[i], t_boxes[i]
                    hs_writes[s] = i
                    from_inactive.append(s)
            if to_inactive:
                self._logger(f"NEW INACTIVE TRACK IDS (track_obj_score_thresh={self.track_obj_score_thresh}): "
                             f"{[int(st.ids[s]) for s in to_inactive]}")
            self.num_reids += len(from_inactive)
            self._inactive = [s for s in self._inactive if s not in from_inactive]
            self._active += from_inactive
            self._deactivate(to_inactive)

            if self.track_nms_thresh and self._active:
                ok = nms_keep(st.pos[self._active], st.score[self._active], self.track_nms_thresh)
                dropped = [s for s, k in zip(self._active, ok) if not k]
                if dropped:
                    self._logger(f"REMOVE TRACK IDS (track_nms_thresh={self.track_nms_thresh}): "
                                 f"{[int(st.ids[s]) for s in dropped]}")
                self._active = [s for s, k in zip(self._active, ok) if k]
                released += dropped

        # ---- new detections (tracker.py:408-492)
        first_obj = n_total - nq
        d_keep = np.logical_and(scores[-nq:] > self.detection_obj_score_thresh, labels[-nq:] == 0)
        d_idx = np.nonzero(d_keep)[0]
        d_boxes, d_scores = boxes[-nq:][d_idx], scores[-nq:][d_idx]
        public = blob["dets"][0] if "dets" in blob else []
        if torch.is_tensor(public):
            public = public.detach().cpu().numpy()
        sel = self.public_detections_mask(d_boxes, public)
        d_idx, d_boxes, d_scores = d_idx[sel], d_boxes[sel], d_scores[sel]
        sel = self.reid(d_boxes, d_scores, d_idx + first_obj, hs_embeds, hs_writes, released)
        d_idx, d_boxes, d_scores = d_idx[sel], d_boxes[sel], d_scores[sel]

        new_slots = []
        for i in range(len(d_idx)):
            s = self._take_slot()
            st = self._state                     # _take_slot may have re-allocated the arrays
            st.ids[s] = self.track_num + i
            st.pos[s] = st.anchor[s] = d_boxes[i]
            st.score[s] = d_scores[i]
            st.obj_ind[s] = d_idx[i]
            st.count_inactive[s] = st.count_termination[s] = 0
            hs_writes[s] = int(d_idx[i] + first_obj)
            new_slots.append(s)
        self._active += new_slots
        self.track_num += len(new_slots)
        if new_slots:
            self._logger(f"INIT TRACK IDS (detection_obj_score_thresh={self.detection_obj_score_thresh}): "
                         f"{[int(st.ids[s]) for s in new_slots]}")

        if self.detection_nms_thresh and self._active:
            fresh = set(new_slots)
            nms_scores = np.array([st.score[s] if s in fresh else np.inf for s in self._active], dtype=np.float32)
            ok = nms_keep(st.pos[self._active], nms_scores, self.detection_nms_thresh)
            dropped = [s for s, k in zip(self._active, ok) if not k]
            if dropped:
                self._logger(f"REMOVE TRACK IDS (detection_nms_thresh={self.detection_nms_thresh}): "
                             f"{[int(st.ids[s]) for s in dropped]}")
            self._active = [s for s, k in zip(self._active, ok) if k]
            released += dropped

        # ---- masks (tracker.py:509-521) and results (tracker.py:533-548)
        self._result_rows = np.asarray([hs_writes.get(s, -1) for s in self._active], np.int64)
        masks = maps = None
        if self.masks:
            masks = self._resolve_masks(det_out, self._result_rows, st.ids[self._active], blob, (height, width))
        if self.generate_attention_maps:
            maps = self._attention_maps(det_out, self._result_rows, st.ids[self._active])
        for k, s in enumerate(self._active):
            box = st.pos[s] if self.obj_detector.overflow_boxes else _clip(st.pos[s], height, width)
            entry = {"bbox": box.copy(), "score": np.array(st.score[s]), "obj_ind": int(st.obj_ind[s])}
            if masks is not None:
                entry["mask"] = masks[k]
            if maps is not None and maps[k] is not None:
                entry["attention_map"] = maps[k].copy()
            self.results.setdefault(int(st.ids[s]), {})[self.frame_index] = entry
        for s in self._inactive:
            st.count_inactive[s] += 1
        self.frame_index += 1
        self._prev_features.append(features)
        if self.reid_sim_only:
            self._deactivate(list(self._active))

        # ---- one scatter of this frame's embeddings into the bank, then recycle the freed slots
        live = set(self._active) | set(self._inactive)
        writes = [(s, q) for s, q in hs_writes.items() if s in live]
        if writes:
            slots = torch.as_tensor([s for s, _ in writes], device=hs_embeds.device)
            qidx = torch.as_tensor([q for _, q in writes], device=hs_embeds.device)
            self._hs.index_copy_(0, slots, hs_embeds.index_select(0, qidx))
        for s in released:
            st.ids[s] = -1
        self._free.extend(released)
