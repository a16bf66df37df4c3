"""Several independent sequences tracked at once: one batched detector call and one decision launch per step for all.

`MultiSequenceTracker` keeps, per sequence key, exactly the state of a `DeviceTracker` (device state buffers, id / ReID
counters, `frame_index`, the `prev_frame_dist` window of previous-frame features, `results`) and steps every sequence
it is handed together:

  * frames are ingested per sequence (`"img"` blobs as they are, raw uint8 `"frame"` blobs through `FrameIngest`);
  * the images are grouped by input size -- images of different sizes are never padded together, since padding would
    change the border sampling of the deformable model against a batch-1 run -- and each group is ONE
    `GraphedDetector.batched` call (one CUDA graph replay at batch B), one post-processing launch and ONE launch of
    csrc/track_step.cu's batched kernel, whose CTA b takes sequence b's decisions on its real rows in place;
  * the result rows of every sequence of the step land in one device buffer, are read back in ONE copy into pinned
    memory and the host synchronises ONCE per step.

Each sequence's results are those of a `DeviceTracker` over `GraphedDetector` on that sequence alone, up to the
floating-point effects of running the detector at batch B.  `track_sequences` keeps up to `max_batch` sequences
running and hands a finished sequence's slot to the next waiting one.

Not batched (rejected in the constructor): segmentation masks (an `obj_detector_post` with "segm") and
`generate_attention_maps=True`; `Tracker` and `DeviceTracker` keep both.
"""
import ctypes

import numpy as np
import torch

from . import device_tracker
from .device_tracker import DeviceTracker, _ArgsC, _MAX_ROWS
from .graphed_detector import GraphedDetector

__all__ = ["MultiSequenceTracker", "track_sequences"]

MAX_BATCH = 16                           # csrc/track_step.cu kMaxBatch
_WORDS = 8 + 8 * _MAX_ROWS               # header + result rows of one sequence, at most


def _library():
    lib = device_tracker._library()
    if not hasattr(lib, "_batched_ready"):
        lib.tfb200_track_step_batched_f32.argtypes = [ctypes.POINTER(_ArgsC), ctypes.c_int, ctypes.c_void_p]
        lib.tfb200_track_step_batched_f32.restype = ctypes.c_int
        lib._batched_ready = True
    return lib


class MultiSequenceTracker:
    """`DeviceTracker`'s arguments plus `max_batch` (<= 16, the number of sequences that can be running at once).

    `start(key)` begins a sequence (a hard reset if the key runs already), `step({key: blob, ...})` advances the
    sequences named, `get_results(key)` / `finish(key)` return a sequence's results (`finish` also frees its slot).
    `start(key, tracker_cfg)` gives that sequence its own thresholds; sequences with different settings share a step.
    `obj_detector` is a `GraphedDetector` or a model, which is then wrapped in one."""

    def __init__(self, obj_detector, obj_detector_post, tracker_cfg, generate_attention_maps=False, logger=None,
                 verbose=False, frame_ingest=None, mask_rle=False, max_batch=8):
        if not 1 <= int(max_batch) <= MAX_BATCH:
            raise ValueError(f"max_batch must be in 1..{MAX_BATCH}, got {max_batch}")
        if "segm" in obj_detector_post:
            raise ValueError("MultiSequenceTracker does not batch segmentation masks; use DeviceTracker or Tracker")
        if generate_attention_maps:
            raise ValueError("MultiSequenceTracker does not batch attention maps; use DeviceTracker or Tracker")
        if not callable(getattr(obj_detector, "batched", None)):
            obj_detector = GraphedDetector(obj_detector)
        self.obj_detector = obj_detector
        self.obj_detector_post = obj_detector_post
        self.tracker_cfg = dict(tracker_cfg)
        self.max_batch = int(max_batch)
        self.frame_ingest = frame_ingest
        self._logger, self._verbose, self._mask_rle = logger, verbose, mask_rle
        self._seqs = {}
        self._result = self._host = None

    @property
    def device(self):
        return next(self.obj_detector.parameters()).device

    # -------------------------------------------------------------------------------------------------- sequences
    def start(self, key, tracker_cfg=None):
        if key not in self._seqs and len(self._seqs) >= self.max_batch:
            raise RuntimeError(f"MultiSequenceTracker: {self.max_batch} sequences are running; finish one first")
        if self.frame_ingest is None and self.device.type == "cuda":       # one ingest (and its buffers) for all
            from .frame_ingest import FrameIngest
            self.frame_ingest = FrameIngest(self.device)
        self._seqs[key] = DeviceTracker(self.obj_detector, self.obj_detector_post,
                                        self.tracker_cfg if tracker_cfg is None else tracker_cfg, False, self._logger,
                                        self._verbose, self.frame_ingest, self._mask_rle)

    def sequence(self, key):
        """The `DeviceTracker` holding sequence `key`'s state (`tracks`, `inactive_tracks`, `frame_index`, ...)."""
        return self._seqs[key]

    def get_results(self, key):
        return self._seqs[key].results

    def finish(self, key):
        return self._seqs.pop(key).results

    # ------------------------------------------------------------------------------------------------------ step
    def _launch(self, args, n, tensors):
        """One launch of the batched decision kernel over `n` sequences.  No host path: CPU tensors are an error."""
        if not all(t.is_cuda for t in tensors):
            raise RuntimeError("MultiSequenceTracker runs its bookkeeping in a CUDA kernel and needs CUDA tensors; "
                               "trackformer_b200.tracker.Tracker is the host-side tracker")
        rc = _library().tfb200_track_step_batched_f32(args, n, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc != 0:
            raise RuntimeError(f"tfb200_track_step_batched_f32 failed (code {rc})")

    def _rows(self, out, orig_size):
        post = self.obj_detector_post["bbox"]
        if hasattr(post, "packed"):
            return post.packed(out, orig_size)
        return torch.stack([torch.cat([r["scores"][:, None], r["labels"][:, None].float(), r["boxes"]], 1)
                            for r in post(out, orig_size)])

    @torch.no_grad()
    def step(self, blobs):
        """One frame of every sequence named in `blobs` ({key: blob}; blobs as `DeviceTracker.step` takes them)."""
        missing = [k for k in blobs if k not in self._seqs]
        if missing:
            raise KeyError(f"MultiSequenceTracker.step: sequences {missing} were not started")
        if not blobs:
            return
        dev = self.device
        nq = self.obj_detector.num_queries
        if self._result is None:
            self._result = torch.zeros(self.max_batch * _WORDS, dtype=torch.int32, device=dev)
            self._host = torch.zeros(self.max_batch * _WORDS, dtype=torch.int32)
            if dev.type == "cuda":
                self._host = self._host.pin_memory()
        stride = 8 + 8 * (max(self._seqs[k]._n_query for k in blobs) + nq)

        groups = {}                                          # input size -> [(key, blob)]
        for key, blob in blobs.items():
            seq = self._seqs[key]
            blob = seq._with_image(blob)
            if "frame" in blobs[key]:                        # the ingest buffer is reused by the next frame of its shape
                blob["img"] = blob["img"].clone()
            groups.setdefault(tuple(blob["img"].shape[-2:]), []).append((key, blob))

        order, keep = [], []
        for members in groups.values():
            seqs = [self._seqs[k] for k, _ in members]
            for seq in seqs:
                seq._logger(f"FRAME: {seq.frame_index + 1}")
            imgs = torch.cat([b["img"] for _, b in members]).to(dev)
            targets = [{"track_query_boxes": s._bufs["q_boxes"][:s._n_query],
                        "track_query_hs_embeds": s._bufs["q_embeds"][:s._n_query]} if s._n_query else None
                       for s in seqs]
            out, features, ks, kb = self.obj_detector.batched(imgs, targets, [s._prev_features[0] for s in seqs])
            orig = torch.cat([b["orig_size"] for _, b in members])
            sizes = [tuple(int(v) for v in o) for o in orig.tolist()]
            rows = self._rows(out, orig.to(dev)).float().contiguous()
            hs = out["hs_embed"].float().contiguous()
            hidden, per_image = hs.shape[-1], kb + nq
            args = (_ArgsC * len(members))()
            tensors = [rows, hs, self._result]
            for i, ((key, blob), seq) in enumerate(zip(members, seqs)):
                assert ks[i] == seq._n_query, (ks[i], seq._n_query)
                public = seq._public(blob, dev)
                seq._ensure(hidden, nq, 0 if public is None else int(public.shape[0]), dev)
                first = i * per_image + kb - ks[i]           # the image's real rows: [kb - K_b, kb + nq) of its block
                args[i] = seq._args(rows.data_ptr() + first * 6 * rows.element_size(),
                                    hs.data_ptr() + first * hidden * hs.element_size(), public,
                                    self._result.data_ptr() + len(order) * stride * 4, nq, *sizes[i])
                if public is not None and len(public):
                    tensors.append(public)
                order.append((key, blob, sizes[i]))
                seq._prev_features.append((features, i))
            self._launch(args, len(members), tensors)
            keep.append((rows, hs, args))                    # alive until the kernel has read them

        # ---- the one read-back of the step: every sequence's header + result rows
        words = len(order) * stride
        host = self._host[:words]
        host.copy_(self._result[:words], non_blocking=True)
        if host.is_pinned():
            torch.cuda.current_stream(dev).synchronize()
        out = host.numpy()
        for p, (key, blob, (height, width)) in enumerate(order):
            self._seqs[key]._take_results(out[p * stride:(p + 1) * stride], None, blob, height, width)


def track_sequences(tracker, sequences):
    """Track every sequence of `sequences` ({name: iterable of blobs}) with `tracker` (a `MultiSequenceTracker`),
    keeping up to `tracker.max_batch` of them running; when one ends, the next waiting one takes its slot.
    Returns {name: results}."""
    waiting = iter(sequences.items())
    running, results = {}, {}
    while True:
        batch = {}
        for name in list(running):
            blob = next(running[name], None)
            if blob is None:
                results[name] = tracker.finish(name)
                del running[name]
            else:
                batch[name] = blob
        while len(running) < tracker.max_batch:
            entry = next(waiting, None)
            if entry is None:
                break
            name, blobs = entry
            tracker.start(name)
            running[name] = iter(blobs)
            blob = next(running[name], None)
            if blob is None:
                results[name] = tracker.finish(name)
                del running[name]
            else:
                batch[name] = blob
        if not batch:
            return results
        tracker.step(batch)
