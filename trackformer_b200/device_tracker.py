"""Online tracker whose per-frame decisions are taken on the device (SURVEY section 8, row f3).

`DeviceTracker` has the constructor, `reset`, `step(blob)`, `get_results`, `tracks` / `inactive_tracks` of
`trackformer_b200.tracker.Tracker` (and therefore of src/trackformer/models/tracker.py:16-581) and produces the same
track ids, `obj_ind`, `num_reids`, frame sets, boxes and scores.  What differs is where the bookkeeping runs:

  * `Tracker` copies the frame's packed detections to the host and takes every decision in numpy;
  * `DeviceTracker` keeps the whole per-target state (ids, boxes, counters, embeddings) in device arrays and runs
    csrc/track_step.cu -- ONE launch per frame that applies the score thresholds, both NMS passes, public-detection
    gating, ReID (greedy centre distance, or embedding distance + Hungarian matching) and writes the frame's result
    rows, the new state and the NEXT frame's track queries (boxes + embeddings) in place.  The host reads back one
    small buffer per frame (the result rows + five counters: that read is also how it learns the number of track
    queries the next forward takes) and never uploads anything but the image and, if used, the public detections.

CUDA only: on CPU tensors `step` raises (use `Tracker`, whose bookkeeping is host code by design).

Segmentation masks work as in `Tracker`: word 7 of each result row is the query row whose embedding -- and so whose
mask -- the track took this frame (-1: it keeps its previous mask), so the mask head runs on those rows after the
read-back and the same resolution kernel writes the frame's label map (and, with `mask_rle=True`, csrc/mask_rle.cu the
results' COCO RLEs from it).  Attention maps (`generate_attention_maps=True`) take the same rows: after the read-back
the maps of those rows are gathered on the device and read back in one copy; with the switch off nothing is added.

Differences a user can see: the debug logger receives the FRAME and INIT TRACK IDS lines only (the per-decision lines
of tracker.py:375-379, 399-402, 232-235 would need the decisions on the host); `tracks` / `inactive_tracks` between
frames cost one extra download of the state; tracks + object queries are limited to 2048 rows per frame.
"""
import ctypes
from collections import deque

import numpy as np
import torch

from .tracker import Track, Tracker, _State

__all__ = ["DeviceTracker"]

_MAX_ROWS = 2048                      # csrc/track_step_core.h kMaxRows
_STATE_FIELDS = (("ids", torch.int32, 1), ("pos", torch.float32, 4), ("anchor", torch.float32, 4),
                 ("score", torch.float32, 1), ("obj_ind", torch.int32, 1), ("count_inactive", torch.int32, 1),
                 ("count_termination", torch.int32, 1))


class _StateC(ctypes.Structure):
    """TfbTrackState (include/tfb200_fused.h)"""
    _fields_ = [(n, ctypes.c_void_p) for n in ("header", "ids", "pos", "anchor", "score", "obj_ind", "count_inactive",
                                                "count_termination", "bank")]


class _ArgsC(ctypes.Structure):
    """TfbTrackStepArgs (include/tfb200_fused.h)"""
    _fields_ = ([(n, ctypes.c_void_p) for n in ("rows", "hs_embeds", "public_dets")]
                + [("inp", _StateC), ("out", _StateC)]
                + [(n, ctypes.c_void_p) for n in ("q_boxes", "q_embeds", "result", "iscratch", "fscratch", "dscratch")]
                + [(n, ctypes.c_double) for n in ("inactive_patience", "reid_sim_threshold")]
                + [(n, ctypes.c_float) for n in ("detection_obj_score_thresh", "track_obj_score_thresh",
                                                 "reid_score_thresh", "detection_nms_thresh", "track_nms_thresh")]
                + [(n, ctypes.c_int32) for n in ("capacity", "hidden", "nq", "n_query", "n_public", "img_h", "img_w",
                                                 "overflow_boxes", "public_mode", "reid_greedy_matching", "reid_sim_only",
                                                 "steps_termination", "detection_nms_on", "track_nms_on")])


_PUBLIC_MODES = {False: 0, None: 0, "center_distance": 1, "min_iou_0_5": 2}
_lib = None


def _library():
    global _lib
    if _lib is None:
        from . import ext
        ext.load()                                   # raises with the build command when the native code is missing
        _lib = ctypes.CDLL(ext.library_path())
        _lib.tfb200_track_step_f32.argtypes = [ctypes.POINTER(_ArgsC), ctypes.c_void_p]
        _lib.tfb200_track_step_f32.restype = ctypes.c_int
    return _lib


class DeviceTracker(Tracker):
    """Drop-in for trackformer.models.tracker.Tracker with the frame-by-frame decisions on the GPU."""

    def reset(self, hard=True):
        """tracker.py:71-80"""
        self._bufs = None
        self._label = None
        self._maps = {}
        self._cur = 0                                 # index of the state buffer holding the current state
        self._n_active = self._n_inactive = self._n_query = 0
        self._host_view = None
        self._prev_features = deque([None], maxlen=self.prev_frame_dist)
        self._state, self._hs, self._active, self._inactive, self._free = _State(1), None, [], [], []
        if hard:
            self.track_num = 0
            self.results = {}
            self.frame_index = 0
            self.num_reids = 0
        if self.public_detections not in _PUBLIC_MODES:
            raise NotImplementedError(self.public_detections)

    # ------------------------------------------------------------------------------------------------- buffers
    def _allocate(self, capacity, hidden, width, dev):
        def state():
            s = {"header": torch.zeros(8, dtype=torch.int32, device=dev),
                 "bank": torch.zeros(capacity, hidden, dtype=torch.float32, device=dev)}
            for name, dtype, cols in _STATE_FIELDS:
                s[name] = torch.zeros((capacity, cols) if cols > 1 else (capacity,), dtype=dtype, device=dev)
            return s
        bufs = {
            "capacity": capacity, "hidden": hidden, "width": width, "state": [state(), state()],
            "q_boxes": torch.zeros(capacity, 4, dtype=torch.float32, device=dev),
            "q_embeds": torch.zeros(capacity, hidden, dtype=torch.float32, device=dev),
            "result": torch.zeros(8 + 8 * capacity, dtype=torch.int32, device=dev),
            "iscratch": torch.zeros(16 * capacity, dtype=torch.int32, device=dev),
            "fscratch": torch.zeros(8 * capacity + capacity * width, dtype=torch.float32, device=dev),
            "dscratch": torch.zeros(4 * capacity, dtype=torch.float64, device=dev),
            "host": torch.zeros(8 + 8 * capacity, dtype=torch.int32),
            "image_id": torch.tensor([1], device=dev),
        }
        if dev.type == "cuda":
            bufs["host"] = bufs["host"].pin_memory()
        return bufs

    def _ensure(self, hidden, nq, n_public, dev):
        need = self._n_active + self._n_inactive + nq
        width = max(nq, n_public, 1)
        b = self._bufs
        if b is not None and b["capacity"] >= need and b["width"] >= width and b["hidden"] == hidden:
            return
        if need > _MAX_ROWS:
            raise RuntimeError(f"DeviceTracker: {need} tracks + object queries exceed the kernel's {_MAX_ROWS} rows")
        capacity = 256 if b is None else b["capacity"]
        while capacity < need:
            capacity *= 2
        capacity = min(capacity, _MAX_ROWS)
        new = self._allocate(capacity, hidden, max(width, 256 if b is None else b["width"]), dev)
        if b is not None:                              # carry the live state and the pending queries over
            n = self._n_active + self._n_inactive
            old, cur = b["state"][self._cur], new["state"][0]
            for key in cur:
                cur[key][:n if key != "header" else 8].copy_(old[key][:n if key != "header" else 8])
            new["q_boxes"][:self._n_query].copy_(b["q_boxes"][:self._n_query])
            new["q_embeds"][:self._n_query].copy_(b["q_embeds"][:self._n_query])
        else:                                          # a soft reset keeps the id / ReID counters (tracker.py:76-80)
            new["state"][0]["header"].copy_(torch.tensor([0, 0, self.track_num, self.num_reids, 0, 0, 0, 0],
                                                         dtype=torch.int32))
        self._bufs, self._cur = new, 0

    # -------------------------------------------------------------------------------------------------- launch
    def _launch(self, args, tensors):
        """One launch of csrc/track_step.cu on the current stream.  No host path: CPU tensors are an error."""
        if not all(t.is_cuda for t in tensors):
            raise RuntimeError("DeviceTracker runs its bookkeeping in a CUDA kernel and needs CUDA tensors; "
                               "trackformer_b200.tracker.Tracker is the host-side tracker")
        rc = _library().tfb200_track_step_f32(ctypes.byref(args), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc != 0:
            raise RuntimeError(f"tfb200_track_step_f32 failed (code {rc})")

    def _device_rows(self, outputs, orig_size):
        post = self.obj_detector_post["bbox"]
        if hasattr(post, "packed"):
            return post.packed(outputs, orig_size)[0]
        res = post(outputs, orig_size)[0]                # any reference-shaped post-processor
        return torch.cat([res["scores"][:, None], res["labels"][:, None].float(), res["boxes"]], 1)

    # ---------------------------------------------------------------------------------------------------- step
    @torch.no_grad()
    def step(self, blob):
        """One frame (tracker.py:266-548); `blob` as for `Tracker.step`: "img" or the raw uint8 "frame"."""
        blob = self._with_image(blob)
        self._logger(f"FRAME: {self.frame_index + 1}")
        dev = self.device
        img = blob["img"].to(dev)
        orig_size = blob["orig_size"]
        height, width = (int(v) for v in orig_size[0].tolist())
        orig_size = orig_size.to(dev)

        n_query = self._n_query
        target = None
        if n_query:
            b = self._bufs
            target = [{"track_query_boxes": b["q_boxes"][:n_query], "image_id": b["image_id"],
                       "track_query_hs_embeds": b["q_embeds"][:n_query]}]
        det_out = self._detect(img, target, self._prev_features[0])
        outputs, _, features, _, _ = det_out
        hs_embeds = outputs["hs_embed"][0].float().contiguous()
        rows = self._device_rows(outputs, orig_size).float().contiguous()
        nq = self.num_object_queries
        assert rows.shape[0] == n_query + nq, (rows.shape, n_query, nq)

        public = self._public(blob, dev)
        n_public = 0 if public is None else int(public.shape[0])
        self._ensure(hs_embeds.shape[1], nq, n_public, dev)
        b = self._bufs
        a = self._args(rows.data_ptr(), hs_embeds.data_ptr(), public, b["result"].data_ptr(), nq, height, width)
        tensors = [rows, hs_embeds, b["result"]] + ([public] if n_public else [])
        self._launch(a, tensors)

        # ---- the one read-back of the frame: header + result rows (at most n_query + nq of them)
        words = 8 + 8 * (n_query + nq)
        host = b["host"][:words]
        host.copy_(b["result"][:words], non_blocking=True)
        if host.is_pinned():
            torch.cuda.current_stream(dev).synchronize()
        self._take_results(host.numpy(), det_out, blob, height, width)
        self._prev_features.append(features)

    def _public(self, blob, dev):
        """This frame's public detections [n, 4] on the device (None when the tracker does not use them)."""
        if not self.public_detections:
            return None
        public = blob["dets"][0] if "dets" in blob else []
        return torch.as_tensor(np.asarray(public.cpu() if torch.is_tensor(public) else public, dtype=np.float32)
                               .reshape(-1, 4)).to(dev)

    def _args(self, rows, hs_embeds, public, result, nq, height, width):
        """The kernel's arguments for this frame (after `_ensure`): `rows` / `hs_embeds` / `result` device addresses."""
        b = self._bufs
        n_public = 0 if public is None else int(public.shape[0])
        src, dst = b["state"][self._cur], b["state"][1 - self._cur]
        a = _ArgsC()
        a.rows, a.hs_embeds = rows, hs_embeds
        a.public_dets = public.data_ptr() if n_public else None
        for c_state, t_state in ((a.inp, src), (a.out, dst)):
            for name in t_state:
                setattr(c_state, name, t_state[name].data_ptr())
        for name in ("q_boxes", "q_embeds", "iscratch", "fscratch", "dscratch"):
            setattr(a, name, b[name].data_ptr())
        a.result = result
        a.inactive_patience, a.reid_sim_threshold = float(self.inactive_patience), float(self.reid_sim_threshold)
        a.detection_obj_score_thresh = float(self.detection_obj_score_thresh)
        a.track_obj_score_thresh = float(self.track_obj_score_thresh)
        a.reid_score_thresh = float(self.reid_score_thresh)
        a.detection_nms_thresh = float(self.detection_nms_thresh or 0.0)
        a.track_nms_thresh = float(self.track_nms_thresh or 0.0)
        a.capacity, a.hidden, a.nq, a.n_query, a.n_public = b["capacity"], b["hidden"], nq, self._n_query, n_public
        a.img_h, a.img_w = height, width
        a.overflow_boxes = int(bool(self.obj_detector.overflow_boxes))
        a.public_mode = _PUBLIC_MODES[self.public_detections]
        a.reid_greedy_matching, a.reid_sim_only = int(bool(self.reid_greedy_matching)), int(bool(self.reid_sim_only))
        a.steps_termination = int(self.steps_termination)
        a.detection_nms_on, a.track_nms_on = int(bool(self.detection_nms_thresh)), int(bool(self.track_nms_thresh))
        return a

    @staticmethod
    def _result_body(out):
        """The result rows [n, 8] int32 of a frame's read-back words `out` (header + result rows): word 0 the track id,
        word 7 the query row the track took this frame (-1: none).  Raises on an error the kernel reported."""
        error, n_results = int(out[5]), int(out[6])
        if error:
            raise RuntimeError(f"track_step kernel reported error {error} (1: query count / state mismatch, 2: capacity)")
        return out[8:8 + 8 * n_results].reshape(n_results, 8)

    def _take_results(self, out, det_out, blob, height, width, masks=None, maps=None):
        """Book the frame from its read-back words `out` (header + result rows) and advance to the next frame.  The
        results' `masks` / attention `maps` (in result order) are made here from `det_out` unless the caller hands
        them in (MultiSequenceTracker makes them for all its sequences at once)."""
        body = self._result_body(out)
        n_active, n_inactive, track_num, num_reids, n_next = (int(v) for v in out[:5])
        n_results = len(body)
        fbody = body.view(np.float32)
        self._result_rows = body[:, 7].astype(np.int64)
        if self.masks and masks is None:
            masks = self._resolve_masks(det_out, self._result_rows, body[:, 0], blob, (height, width))
        if self.generate_attention_maps and maps is None:
            maps = self._attention_maps(det_out, self._result_rows, body[:, 0])
        for k in range(n_results):
            entry = {"bbox": fbody[k, 3:7].copy(), "score": np.array(fbody[k, 2]), "obj_ind": int(body[k, 1])}
            if masks is not None:
                entry["mask"] = masks[k]
            if maps is not None and maps[k] is not None:
                entry["attention_map"] = maps[k].copy()
            self.results.setdefault(int(body[k, 0]), {})[self.frame_index] = entry
        if track_num > self.track_num:
            self._logger(f"INIT TRACK IDS (detection_obj_score_thresh={self.detection_obj_score_thresh}): "
                         f"{list(range(self.track_num, track_num))}")
        self.track_num, self.num_reids = track_num, num_reids
        self._n_active, self._n_inactive, self._n_query = n_active, n_inactive, n_next
        self._cur = 1 - self._cur
        self._host_view = None
        self.frame_index += 1

    # ------------------------------------------------------------------------------------- host views (on demand)
    def _download(self):
        """Copy the device state into the host struct of arrays the `Track` views read (one synchronisation; only
        used when somebody looks at `tracks` / `inactive_tracks` between frames)."""
        if self._host_view is not None:
            return
        n = self._n_active + self._n_inactive
        st = _State(max(n, 1))
        if n:
            cur = self._bufs["state"][self._cur]
            for name, _, _ in _STATE_FIELDS:
                getattr(st, name)[:n] = cur[name][:n].cpu().numpy()
            self._hs = cur["bank"]
        self._state = st
        self._active = list(range(self._n_active))
        self._inactive = list(range(self._n_active, n))
        self._host_view = True

    @property
    def tracks(self):
        self._download()
        return [Track(self, s) for s in self._active]

    @property
    def inactive_tracks(self):
        self._download()
        return [Track(self, s) for s in self._inactive]
