"""CUDA-graph replay of the tracking-mode detector forward (SURVEY section 8, row f3).

Online tracking of one sequence is batch-1 and latency-bound (`batched`, below, steps several sequences together):
the reference issues ~2000 small kernels per frame from Python (src/trackformer/models/tracker.py:306 ->
DeformableDETR.forward) and the number of track queries changes from frame to
frame, so nothing about a frame's launch sequence is reusable as it stands.  `GraphedDetector` makes it reusable:

  * the track queries of a frame are padded up to a multiple of `bucket` with filler queries that the real queries
    cannot attend to (`track_query_padding` -> key-padding mask of the decoder's query self-attention,
    deformable_transformer.py); every other decoder op is row-wise, so the real rows come out as in the unpadded
    model and the filler rows are dropped before anything is returned;
  * for every (image shape, padded track-query count, previous-frame-features yes/no) one CUDA graph of the whole
    forward is captured on first use and replayed afterwards; inputs are copied into the graph's static buffers.

It has the call signature, attributes and return value of the model it wraps -- `Tracker(GraphedDetector(model), ...)`
-- except that `aux_outputs` are not returned (the tracker reads them only for verbose logging).

For segmentation models (those with `detect` / `mask_logits`, segmentation.py) the graph holds `detect`, the forward
without the mask head, so `pred_masks` is not returned either; `mask_logits(rows)` runs the head eagerly on the rows
the tracker asks for, from the static buffers of the last call.
`use_graphs=False` keeps the padding but runs the model eagerly (used by the CPU tests of the padding logic).

With the vanilla model's `generate_attention_maps` switch on, the switch is part of the plan key: the captured graph
computes the maps as one more static output, and `out["attention_maps"]` drops the filler rows like the other outputs
(`batched` returns them padded, like its other outputs).  `batched_mask_logits` is `mask_logits` for a `batched` call:
the ragged mask head over a different set of rows per image.
"""
import torch

from .util import NestedTensor

__all__ = ["GraphedDetector"]


class _Plan:
    graph = None
    prev = None


class GraphedDetector:
    def __init__(self, model, bucket: int = 32, use_graphs: bool = True, warmup: int = 2):
        if bucket < 1:
            raise ValueError("bucket must be >= 1")
        self.model = model
        self.bucket = int(bucket)
        self.use_graphs = use_graphs
        self.warmup = warmup
        self.multi_frame = bool(getattr(model, "multi_frame_attention", False))
        # models that read prev_features (deformable_detr.py `_project_levels`): multi-frame attention and/or merged
        # frame features -- both must see the caller's previous-frame maps, and both keep what we return across frames
        self.uses_prev = self.multi_frame or bool(getattr(model, "merge_frame_features", False))
        self.has_mask_head = callable(getattr(model, "mask_logits", None))
        self._plans = {}
        self._last = None
        self.last_batched = None                     # (plan, K_b) of the last `batched` call, for batched_mask_logits
        self.replays = 0
        self.captures = 0

    # ---- the attributes the tracker reads from its detector (tracker.py:38,45,69,323)
    @property
    def num_queries(self):
        return self.model.num_queries

    @property
    def hidden_dim(self):
        return self.model.hidden_dim

    @property
    def overflow_boxes(self):
        return self.model.overflow_boxes

    @property
    def transformer(self):
        return self.model.transformer

    @property
    def generate_attention_maps(self):
        return bool(getattr(self.model, "generate_attention_maps", False))

    @generate_attention_maps.setter
    def generate_attention_maps(self, on):
        self.model.generate_attention_maps = bool(on)

    def parameters(self):
        return self.model.parameters()

    def tracking(self):
        self.model.tracking()
        return self

    # ------------------------------------------------------------------------------------------------------------
    def _padded_count(self, k: int) -> int:
        return 0 if k == 0 else -(-k // self.bucket) * self.bucket

    def _run(self, plan):
        targets = None
        if plan.kb:
            targets = [{"track_query_boxes": plan.boxes, "track_query_hs_embeds": plan.hs,
                        "track_query_padding": plan.padding, "image_id": plan.image_id}]
        forward = self.model.detect if self.has_mask_head else self.model
        with torch.no_grad():
            out, _, plan.features, plan.memory, plan.hs_all = forward(plan.img, targets, plan.prev)
        plan.logits, plan.out_boxes, plan.hs_embed = out["pred_logits"], out["pred_boxes"], out["hs_embed"]
        plan.attention_maps = out.get("attention_maps")

    def _build(self, key, img, kb, prev_features):
        dev = img.device
        plan = _Plan()
        plan.kb = kb
        plan.img = img.clone()
        if kb:
            plan.hs = torch.zeros(kb, self.hidden_dim, device=dev)
            plan.boxes = torch.full((kb, 4), 0.5, device=dev)
            plan.padding = torch.ones(kb, dtype=torch.bool, device=dev)
            plan.slot_index = torch.arange(kb, device=dev)
            plan.image_id = torch.tensor([1], device=dev)
        if prev_features is not None:
            plan.prev = []
            for f in prev_features:
                mask = f.mask.clone()
                if getattr(f.mask, "_no_padding", False):
                    mask._no_padding = True
                plan.prev.append(NestedTensor(f.tensors.clone(), mask))
        if self.use_graphs:
            if not img.is_cuda:
                raise RuntimeError("GraphedDetector(use_graphs=True) needs CUDA tensors")
            if hasattr(self.model.backbone[0], "prepare"):
                self.model.backbone[0].prepare()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):                    # cuDNN autotuning, memoised grids / encodings
                for _ in range(self.warmup):
                    self._run(plan)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            plan.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(plan.graph):
                self._run(plan)
            self.captures += 1
        self._plans[key] = plan
        return plan

    def __call__(self, samples, targets=None, prev_features=None):
        self._last = None
        if isinstance(samples, NestedTensor) or not torch.is_tensor(samples) or samples.ndim != 4 or samples.shape[0] != 1:
            return self.model(samples, targets, prev_features)        # padded batches: outside the graphed domain
        k = 0
        if targets is not None and "track_query_boxes" in targets[0]:
            k = int(targets[0]["track_query_boxes"].shape[0])
        kb = self._padded_count(k)
        use_prev = self.uses_prev and prev_features is not None
        key = (tuple(samples.shape), samples.dtype, kb, use_prev, self.generate_attention_maps)
        plan = self._plans.get(key)
        if plan is None:
            plan = self._build(key, samples, kb, prev_features if use_prev else None)
        plan.img.copy_(samples, non_blocking=True)
        if kb:
            plan.hs[:k].copy_(targets[0]["track_query_hs_embeds"], non_blocking=True)
            plan.boxes[:k].copy_(targets[0]["track_query_boxes"], non_blocking=True)
            torch.ge(plan.slot_index, k, out=plan.padding)
        if use_prev:
            for dst, src in zip(plan.prev, prev_features):
                if dst.tensors is not src.tensors:
                    dst.tensors.copy_(src.tensors, non_blocking=True)
        if plan.graph is not None:
            plan.graph.replay()
            self.replays += 1
        else:
            self._run(plan)

        nq = self.num_queries
        self._last = (plan, k)

        def real_rows(x, dim):
            """drop the filler rows kb-k ... : [track queries (k) | object queries (nq)]"""
            if kb == k:
                return x
            return torch.cat([x.narrow(dim, 0, k), x.narrow(dim, kb, nq)], dim)

        out = {"pred_logits": real_rows(plan.logits, 1), "pred_boxes": real_rows(plan.out_boxes, 1),
               "hs_embed": real_rows(plan.hs_embed, 1)}
        if plan.attention_maps is not None:
            out["attention_maps"] = real_rows(plan.attention_maps, 1)
        features = plan.features
        if self.uses_prev and plan.graph is not None:
            # the static feature maps are overwritten by the next replay, but the tracker hands them back as
            # prev_features (possibly several frames later, prev_frame_dist > 1): give it its own copy
            features = []
            for f in plan.features:
                mask = f.mask
                features.append(NestedTensor(f.tensors.clone(), mask))
        # NB: for models that never read prev_features the returned `features` / `memory` (and, when no filler rows had
        # to be dropped, the output rows) are views of the graph's static buffers: valid until the next call.
        return out, targets, features, plan.memory, real_rows(plan.hs_all, 2)

    def _build_batched(self, samples, kb, prev_features):
        dev, bsz = samples.device, samples.shape[0]
        plan = _Plan()
        plan.kb = kb
        plan.img = samples.clone()
        if kb:
            plan.hs = torch.zeros(bsz, kb, self.hidden_dim, device=dev)
            plan.boxes = torch.full((bsz, kb, 4), 0.5, device=dev)
            plan.padding = torch.ones(bsz, kb, dtype=torch.bool, device=dev)
            plan.slot_index = torch.arange(kb, device=dev)
            plan.first = torch.zeros(bsz, 1, dtype=torch.int64, device=dev)
            plan.image_id = torch.tensor([1], device=dev)
        if prev_features is not None:
            plan.prev_valid = torch.zeros(bsz, dtype=torch.bool, device=dev)
            src, i = next(p for p in prev_features if p is not None)
            plan.prev = []
            for f in src:
                mask = f.mask[i:i + 1].expand(bsz, -1, -1).clone()
                if getattr(f.mask, "_no_padding", False):
                    mask._no_padding = True
                plan.prev.append(NestedTensor(f.tensors[i:i + 1].repeat(bsz, 1, 1, 1), mask))
        plan.graph = None
        if self.use_graphs:
            if not samples.is_cuda:
                raise RuntimeError("GraphedDetector(use_graphs=True) needs CUDA tensors")
            if hasattr(self.model.backbone[0], "prepare"):
                self.model.backbone[0].prepare()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(self.warmup):
                    self._run_batched(plan)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            plan.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(plan.graph):
                self._run_batched(plan)
            self.captures += 1
        return plan

    def _run_batched(self, plan):
        targets = None
        if plan.kb:
            targets = [{"track_query_boxes": plan.boxes[b], "track_query_hs_embeds": plan.hs[b],
                        "track_query_padding": plan.padding[b], "image_id": plan.image_id}
                       for b in range(plan.img.shape[0])]
        forward = self.model.detect if self.has_mask_head else self.model
        prev_valid = None if plan.prev is None else plan.prev_valid
        with torch.no_grad():
            out, _, features, plan.memory, plan.hs_all = forward(plan.img, targets, plan.prev, prev_valid)
        plan.features = features[-3:]                    # what a later call takes as prev_features
        plan.all_features = features                     # the mask head also reads the stride-4 level
        plan.logits, plan.out_boxes, plan.hs_embed = out["pred_logits"], out["pred_boxes"], out["hs_embed"]
        plan.attention_maps = out.get("attention_maps")

    def batched(self, samples, targets=None, prev_features=None):
        """One forward of B images that each carry their own track queries -- B independent sequences stepped together.

        ``samples`` [B, 3, H, W] (one input size: images of different sizes would be padded, which changes the border
        sampling of a batch-1 run).  ``targets[b]`` holds image b's ``track_query_boxes`` [K_b, 4] and
        ``track_query_hs_embeds`` [K_b, C] (or is None: K_b = 0).  ``prev_features[b]`` is ``(features, i)`` -- image i
        of a ``features`` list this method returned earlier -- or None where the image has no previous frame; the
        model then reads the image's own features, as a batch-1 call with ``prev_features=None`` does.

        All images are padded to ``kb`` = the bucket of max K_b track queries.  Image b's K_b track queries take the
        LAST K_b of its kb slots, so its real rows ``[kb - K_b, kb + nq)`` (track queries, then object queries) are
        contiguous and a consumer reads them in place with a row offset.  One CUDA graph is captured per (B, H, W,
        dtype, kb, previous-frame features yes/no); which images have a previous frame is a static input of it.

        Returns ``(out, features, ks, kb)``: ``out`` with the padded ``pred_logits`` / ``pred_boxes`` / ``hs_embed``
        [B, kb + nq, .] -- and ``attention_maps`` [B, kb + nq, h, w] with the vanilla model's switch on -- (views of
        the graph's buffers: valid until the next call), the levels ``features`` a later call takes as
        ``prev_features`` (its own copy), and the host ints K_b.  ``last_batched`` then names this call for
        ``batched_mask_logits``."""
        if not torch.is_tensor(samples) or samples.ndim != 4:
            raise ValueError("GraphedDetector.batched takes one [B, 3, H, W] tensor of same-sized images")
        bsz = samples.shape[0]
        targets = [None] * bsz if targets is None else list(targets)
        prev_features = [None] * bsz if prev_features is None else list(prev_features)
        if len(targets) != bsz or len(prev_features) != bsz:
            raise ValueError("GraphedDetector.batched: one target and one prev_features entry per image")
        ks = [0 if t is None else int(t["track_query_boxes"].shape[0]) for t in targets]
        kb = self._padded_count(max(ks))
        use_prev = self.uses_prev and any(p is not None for p in prev_features)
        key = ("batched", tuple(samples.shape), samples.dtype, kb, use_prev, self.generate_attention_maps)
        plan = self._plans.get(key)
        if plan is None:
            plan = self._plans[key] = self._build_batched(samples, kb, prev_features if use_prev else None)
        self._last = None
        plan.img.copy_(samples, non_blocking=True)
        if kb:
            for b, (t, k) in enumerate(zip(targets, ks)):
                if k:
                    plan.hs[b, kb - k:].copy_(t["track_query_hs_embeds"], non_blocking=True)
                    plan.boxes[b, kb - k:].copy_(t["track_query_boxes"], non_blocking=True)
            plan.first.copy_(torch.tensor([[kb - k] for k in ks]), non_blocking=True)
            torch.lt(plan.slot_index, plan.first, out=plan.padding)
        if use_prev:
            valid = [p is not None for p in prev_features]
            plan.prev_valid.copy_(torch.tensor(valid), non_blocking=True)
            src = {id(p[0]) for p in prev_features if p is not None}
            whole = (all(valid) and len(src) == 1 and all(p[1] == b for b, p in enumerate(prev_features))
                     and prev_features[0][0][0].tensors.shape[0] == bsz)
            if whole:                                     # the batch of the last step, in the same order
                for dst, f in zip(plan.prev, prev_features[0][0]):
                    dst.tensors.copy_(f.tensors, non_blocking=True)
            else:
                for b, p in enumerate(prev_features):
                    if p is not None:
                        for dst, f in zip(plan.prev, p[0]):
                            dst.tensors[b].copy_(f.tensors[p[1]], non_blocking=True)
        if plan.graph is not None:
            plan.graph.replay()
            self.replays += 1
        else:
            self._run_batched(plan)
        self.last_batched = (plan, ks)
        features = plan.features
        if self.uses_prev and plan.graph is not None:
            features = [NestedTensor(f.tensors.clone(), f.mask) for f in plan.features]
        out = {"pred_logits": plan.logits, "pred_boxes": plan.out_boxes, "hs_embed": plan.hs_embed}
        if plan.attention_maps is not None:
            out["attention_maps"] = plan.attention_maps
        return out, features, ks, kb

    def batched_mask_logits(self, src_rows, sizes, call=None):
        """Mask logits ``[sum(sizes), H/4, W/4]`` of rows of a ``batched`` call, computed eagerly by the ragged mask
        head from that call's static feature / memory / decoder buffers (valid until the next call with the same
        plan key).  Image b contributes ``sizes[b]`` rows; ``src_rows`` holds them image after image as REAL row
        indices of the image (``[track queries (K_b) | object queries]``, what the decision kernel reports), which
        sit at padded row ``kb - K_b + r``.  ``call`` is the ``last_batched`` value right after that call (default:
        the last call).  Images may contribute no rows."""
        if not self.has_mask_head:
            raise RuntimeError("GraphedDetector.batched_mask_logits: the wrapped model has no mask head")
        if call is None:
            call = getattr(self, "last_batched", None)
            if call is None:
                raise RuntimeError("GraphedDetector.batched_mask_logits: no batched call to take the rows from")
        plan, ks = call
        sizes = [int(n) for n in sizes]
        if len(sizes) != len(ks):
            raise ValueError(f"GraphedDetector.batched_mask_logits: {len(sizes)} sizes for a batch of {len(ks)}")
        rows = torch.as_tensor(src_rows, dtype=torch.long).reshape(-1).cpu()
        if rows.numel() != sum(sizes):
            raise ValueError("GraphedDetector.batched_mask_logits: len(src_rows) != sum(sizes)")
        shift = torch.repeat_interleave(torch.tensor([plan.kb - k for k in ks], dtype=torch.long),
                                        torch.tensor(sizes, dtype=torch.long))
        padded = (rows + shift).to(plan.img.device, non_blocking=True)
        with torch.no_grad():
            return self.model.mask_logits(plan.all_features, plan.memory, plan.hs_all, rows=(padded, sizes))

    def detect(self, samples, targets=None, prev_features=None):
        """The call itself: for segmentation models the graph already holds the forward without the mask head."""
        return self(samples, targets, prev_features)

    def mask_logits(self, rows):
        """Mask logits ``[1, len(rows), H/4, W/4]`` of the real query rows ``rows`` of the last call ([track queries |
        object queries], as returned), computed eagerly from the static feature / memory / decoder buffers.  Valid
        until the next call."""
        if not self.has_mask_head:
            raise RuntimeError("GraphedDetector.mask_logits: the wrapped model has no mask head")
        if self._last is None:
            raise RuntimeError("GraphedDetector.mask_logits: no graphed call to take the rows from")
        plan, k = self._last
        padded = [int(r) if r < k else int(r) - k + plan.kb for r in rows]      # skip the filler rows k ... kb-1
        with torch.no_grad():
            return self.model.mask_logits(plan.features, plan.memory, plan.hs_all, padded)
