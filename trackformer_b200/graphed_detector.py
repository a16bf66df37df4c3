"""CUDA-graph replay of the tracking-mode detector forward (SURVEY section 8, row f3).

Online tracking is batch-1 and latency-bound: the reference issues ~2000 small kernels per frame from Python
(src/trackformer/models/tracker.py:306 -> DeformableDETR.forward) and the number of track queries changes from frame to
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
computes the maps as one more static output, and `out["attention_maps"]` drops the filler rows like the other outputs.
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
