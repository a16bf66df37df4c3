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

Segmentation masks (MOTS: an `obj_detector_post` with "segm") and attention maps (`generate_attention_maps=True`,
vanilla decoders) are batched too.  After the one read-back, word 7 of every result row names the query row whose mask
and map its track takes, and then:

  * per input-size group, ONE `batched_mask_logits` call runs the ragged mask head over the rows every sequence's
    tracks took (the head stays eager);
  * ONE launch of csrc/track_masks.cu resolves the label maps of every sequence, each against its own previous label
    map for the tracks that keep their masks;
  * with `mask_rle=True`, ONE call of csrc/mask_rle.cu's batched entry encodes every sequence's results (two
    device-to-host copies); with bool masks all label maps leave the device in one copy;
  * attention maps: one gather per group, copied to the host before the same synchronise.

So a step synchronises the host at most three times whatever the number of sequences (result rows, then the RLE
header and strings; twice with bool masks or maps alone), where stepping the sequences one by one costs up to three
per sequence.  The detector must have `batched_mask_logits` for masks (a `GraphedDetector` over a segmentation model,
or such a model, which is then wrapped) and a vanilla decoder for maps, as `Tracker` requires.
"""
import ctypes

import numpy as np
import torch

from . import device_tracker
from .device_tracker import DeviceTracker, _ArgsC, _MAX_ROWS
from .graphed_detector import GraphedDetector
from .mots import label_maps_rle
from .segmentation import resolve_track_masks_many

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
        if not callable(getattr(obj_detector, "batched", None)):
            obj_detector = GraphedDetector(obj_detector)
        self.masks = "segm" in obj_detector_post
        if self.masks and not (callable(getattr(obj_detector, "batched_mask_logits", None))
                               and getattr(obj_detector, "has_mask_head", True)):
            raise ValueError("MultiSequenceTracker does not batch segmentation masks; use DeviceTracker or Tracker")
        self.generate_attention_maps = bool(generate_attention_maps)
        if self.generate_attention_maps:
            layers = getattr(getattr(getattr(obj_detector, "transformer", None), "decoder", None), "layers", None)
            if not layers or not hasattr(layers[-1], "multihead_attn"):     # Tracker's check: a vanilla decoder
                raise ValueError("MultiSequenceTracker does not batch attention maps; use DeviceTracker or Tracker")
        if hasattr(obj_detector, "generate_attention_maps"):
            obj_detector.generate_attention_maps = self.generate_attention_maps
        self.obj_detector = obj_detector
        self.obj_detector_post = obj_detector_post
        self.tracker_cfg = dict(tracker_cfg)
        self.max_batch = int(max_batch)
        self.frame_ingest = frame_ingest
        self._logger, self._verbose, self._mask_rle = logger, verbose, mask_rle
        self._seqs = {}
        self._result = self._host = None
        self._pinned = {}                                    # name -> pinned host buffer, grown on demand

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
                                        self.tracker_cfg if tracker_cfg is None else tracker_cfg,
                                        self.generate_attention_maps, self._logger, self._verbose, self.frame_ingest,
                                        self._mask_rle)

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

        order, keep, calls = [], [], []
        for members in groups.values():
            seqs = [self._seqs[k] for k, _ in members]
            for seq in seqs:
                seq._logger(f"FRAME: {seq.frame_index + 1}")
            imgs = torch.cat([b["img"] for _, b in members]).to(dev, non_blocking=True)
            targets = [{"track_query_boxes": s._bufs["q_boxes"][:s._n_query],
                        "track_query_hs_embeds": s._bufs["q_embeds"][:s._n_query]} if s._n_query else None
                       for s in seqs]
            out, features, ks, kb = self.obj_detector.batched(imgs, targets, [s._prev_features[0] for s in seqs])
            orig = torch.cat([b["orig_size"] for _, b in members])
            sizes = [tuple(int(v) for v in o) for o in orig.tolist()]
            rows = self._rows(out, orig.to(dev, non_blocking=True)).float().contiguous()
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
            calls.append((getattr(self.obj_detector, "last_batched", None), out.get("attention_maps"), ks, kb,
                          range(len(order) - len(members), len(order))))

        # ---- the one read-back of the step: every sequence's header + result rows
        words = len(order) * stride
        host = self._host[:words]
        host.copy_(self._result[:words], non_blocking=True)
        if host.is_pinned():
            torch.cuda.current_stream(dev).synchronize()
        out = host.numpy()
        views = [out[p * stride:(p + 1) * stride] for p in range(len(order))]
        bodies = [DeviceTracker._result_body(v) for v in views]
        masks = self._resolve_all(order, bodies, calls) if self.masks else [None] * len(order)
        maps = self._gather_maps(order, bodies, calls) if self.generate_attention_maps else None
        synced = False
        if self.masks:
            masks, synced = self._mask_results(order, bodies, masks)
        if maps is not None:
            if not synced:                                   # no mask read-back waited for the copies above
                self._synchronize(dev)
            maps = [book() for book in maps]
        for p, (key, blob, (height, width)) in enumerate(order):
            self._seqs[key]._take_results(views[p], None, blob, height, width, masks[p],
                                          None if maps is None else maps[p])

    # ------------------------------------------------------------------------------------- masks and maps, batched
    @staticmethod
    def _synchronize(dev):
        if dev.type == "cuda":
            torch.cuda.current_stream(dev).synchronize()

    def _pinned_buffer(self, name, numel, dtype, dev):
        """A host buffer of `numel` elements (pinned when the step runs on CUDA), reused across steps."""
        buf = self._pinned.get(name)
        if buf is None or buf.numel() < numel or buf.dtype != dtype:
            buf = torch.empty(max(numel, 1), dtype=dtype)
            if dev.type == "cuda":
                buf = buf.pin_memory()
            self._pinned[name] = buf
        return buf[:numel]

    def _resolve_all(self, order, bodies, calls):
        """Every sequence's label map of this step: one ragged mask-head call per group, then one resolution launch.
        Sets each sequence's `_label`; returns, per sequence, the label map (None when it has no active track)."""
        jobs = [None] * len(order)
        for p, (key, blob, orig) in enumerate(order):
            body = bodies[p]
            jobs[p] = self._seqs[key]._mask_job(body[:, 7].astype(np.int64), body[:, 0], blob, orig)
        logits = [None] * len(order)
        for call, _, _, _, members in calls:
            sizes = [0 if jobs[p] is None else len(jobs[p][0]) for p in members]
            rows = [r for p in members if jobs[p] is not None for r in jobs[p][0]]
            if not rows:
                continue
            head = self.obj_detector.batched_mask_logits(rows, sizes, call)
            o = 0
            for p, n in zip(members, sizes):
                if n:
                    logits[p] = head[o:o + n]
                o += n
        work = []
        for p, (key, blob, orig) in enumerate(order):
            if jobs[p] is None:
                continue
            rows, src, prev, size = jobs[p]
            lg = logits[p] if logits[p] is not None else torch.zeros(0, 1, 1, device=prev.device)
            work.append((p, (lg, src, [int(i) for i in bodies[p][:, 0]], prev, size, size, orig)))
        labels = resolve_track_masks_many([job for _, job in work])
        out = [None] * len(order)
        for (p, _), label in zip(work, labels):
            out[p] = label
        for p, (key, _, _) in enumerate(order):
            self._seqs[key]._label = out[p]
        return out

    def _mask_results(self, order, bodies, labels):
        """The results' masks of every sequence from its label map: RLEs from one batched encoder call, or bool arrays
        from one copy of all label maps.  Also returns whether that read-back synchronised the host."""
        live = [p for p, lab in enumerate(labels) if lab is not None]
        out = [[] for _ in order]
        if not live:
            return out, False
        dev = labels[live[0]].device
        if self._mask_rle:
            rles = label_maps_rle([labels[p] for p in live], [bodies[p][:, 0] for p in live])
            for p, r in zip(live, rles):
                out[p] = r
            return out, dev.type == "cuda"
        flat = torch.cat([labels[p].reshape(-1) for p in live])
        host = self._pinned_buffer("labels", flat.numel(), torch.int32, dev)
        host.copy_(flat, non_blocking=True)
        self._synchronize(dev)
        host = host.numpy()
        o = 0
        for p in live:
            n = labels[p].numel()
            lab = host[o:o + n].reshape(labels[p].shape)
            out[p] = [lab == i for i in bodies[p][:, 0]]
            o += n
        return out, dev.type == "cuda"

    def _gather_maps(self, order, bodies, calls):
        """Issue one gather per group of the maps the tracks took and its copy to the host (no synchronise).  Returns
        per sequence a callable that books its maps once the copies have landed."""
        result = [None] * len(order)
        for _, maps, ks, kb, members in calls:
            flat = maps.flatten(0, 1)                        # [B * (kb + nq), h, w]: the padded rows of every image
            per_image = maps.shape[1]
            index, spans = [], []
            for i, p in enumerate(members):
                fresh = [int(r) for r in bodies[p][:, 7] if r >= 0]
                spans.append((p, len(index), len(fresh)))
                index += [i * per_image + kb - ks[i] + r for r in fresh]
            host = None
            if index:
                index = torch.as_tensor(index, dtype=torch.long).to(flat.device, non_blocking=True)
                picked = flat.index_select(0, index).float()
                host = self._pinned_buffer(f"maps{members.start}", picked.numel(), torch.float32,
                                           flat.device).view(picked.shape)
                host.copy_(picked, non_blocking=True)
            for p, o, n in spans:
                seq = self._seqs[order[p][0]]
                body = bodies[p]

                def book(seq=seq, body=body, host=host, o=o, n=n):
                    return seq._book_maps(body[:, 7].astype(np.int64), body[:, 0],
                                          None if not n else host[o:o + n].numpy().copy())   # buffer is reused
                result[p] = book
        return result


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
