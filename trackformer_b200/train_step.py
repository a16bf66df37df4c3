"""One training step of the detection hot path, replayed from CUDA graphs.

This is the GPU-side counterpart of the six hot lines of the reference's training loop
(src/trackformer/engine.py:126-151):

    outputs = model(samples, targets); loss_dict = criterion(outputs, targets); losses = sum(w_k * loss_k)
    optimizer.zero_grad(); losses.backward(); clip_grad_norm_(params, max_norm); optimizer.step()

plus the gradient all-reduce the reference gets from DistributedDataParallel (src/train.py:86-89).

Why graphs: an eager PyTorch step of this model issues ~5000 small kernels and is host-bound (the launch
overhead exceeds the kernels' own run time).  The model forward and its
backward are static-shape, sync-free programs, so they are captured once (``torch.cuda.CUDAGraph``) and
replayed -- two graph launches instead of thousands of kernel launches.  The backward graph also contains the
accumulation into the gradient buffer, so nothing per-parameter runs eagerly.  Between the two sits what cannot be captured: the Hungarian matching (scipy on the host, like the
reference, matcher.py:104,127 -- the index bookkeeping must stay bit-exact) and the loss, which is small.

Tracking: for a ``DETRTrackingBase`` model in training mode whose targets carry ``prev_image`` / ``prev_target``, a step
is the reference's tracking step (detr_tracking.py forward + criterion + backward), decomposed so that the heavy parts
replay from graphs as well -- see ``_tracking_route`` for how a step's route is chosen and ``_track_step`` for the
pieces.

Multi-GPU: one process per GPU.  Gradients live in ONE flat fp32 buffer (every ``param.grad`` is a view into
it), so the data-parallel exchange is a single NCCL all-reduce of 162 MB over NVLink/NVSwitch after the backward
graph, followed by clip + fused AdamW.  (DDP's bucketed overlap would hide ~0.4 ms of a ~20 ms step; a single
flat all-reduce keeps the backward capturable and costs one launch.)
"""
from __future__ import annotations

import os
from typing import List, Optional

import torch
import torch.distributed as dist
from torch import nn


class _DetectorCore(nn.Module):
    """Tensor-in / tensors-out view of the detector for graph capture: frames -> (logits[K,B,Q,C], boxes[K,B,Q,4]), and
    for a two-stage model the encoder head's (logits [B,S,C], boxes [B,S,4]) after them.

    With ``masks`` (segmentation models) the detector runs without its mask head and the mask branch's inputs
    follow the two heads: ``(logits, boxes, queries, memory, src, pad, fpn0, fpn1, fpn2)`` (``DETRSegmBase.mask_inputs``);
    the step runs the head itself on the matched rows only."""

    def __init__(self, model, masks: bool = False):
        super().__init__()
        self.model = model
        self.masks = masks

    def forward(self, frames):
        if self.masks:
            out, _, features, memory, hs = self.model.detect(frames, None, None)
            return self._heads(out) + self._mask_inputs(features, memory, hs)
        out, _, _, _, _ = self.model(frames, None, None)
        return self._heads(out)

    def _mask_inputs(self, features, memory, hs):
        q, memory, src, pad, fpns = self.model.mask_inputs(features, memory, hs)
        return (q, memory, src, pad, *fpns)

    def detector(self, frames, targets=None, prev_features=None):
        """The detector's own forward (``DeformableDETR.forward``) of a tracking model: previous frames, and current
        frames with precomputed track-query targets -- not ``DETRTrackingBase.forward``, which would rewrite them."""
        from .detr_tracking import DETRTrackingBase
        return super(DETRTrackingBase, self.model).forward(frames, targets, prev_features)

    def track(self, frames, targets, prev_features):
        out, _, features, memory, hs = self.detector(frames, targets, prev_features)
        if self.masks:
            return self._heads(out) + self._mask_inputs(features, memory, hs)
        return self._heads(out)

    def _heads(self, out):
        stacked = getattr(self.model, "stacked_heads", None)
        if stacked is not None and stacked[0].shape[0] == len(out["aux_outputs"]) + 1:
            heads = tuple(stacked)                   # the very tensors the dictionary entries are slices of
        else:
            heads = (torch.stack([a["pred_logits"] for a in out["aux_outputs"]] + [out["pred_logits"]]),
                     torch.stack([a["pred_boxes"] for a in out["aux_outputs"]] + [out["pred_boxes"]]))
        enc = out.get("enc_outputs")
        if enc is not None:
            heads += (enc["pred_logits"], enc["pred_boxes"])
        return heads


class TrainStep:
    """``loss = step(frames, targets)`` -- forward, criterion, backward, [all-reduce], clip, optimizer."""

    def __init__(self, model, criterion, optimizer_factory=None, max_norm: float = 0.1,
                 use_graphs: bool = True, example_frames: Optional[torch.Tensor] = None,
                 example_targets: Optional[list] = None, flat_adamw: Optional[dict] = None, track_bucket: int = 32,
                 masks: bool = False):
        """``optimizer_factory(params)`` builds any torch optimizer; ``flat_adamw={'groups': [...], 'betas':..., 'eps':...}``
        (groups as for torch.optim.AdamW, e.g. flat_adamw.reference_param_groups(model)) instead lays the PARAMETERS out
        flat as well and updates them with the one-pass clip + AdamW kernel.  ``track_bucket``: tracking steps pad their
        track queries up to a multiple of it, and one pair of current-frame graphs is captured per padded count.

        ``masks=True`` trains a segmentation model (``DETRSegmBase``, with ``freeze_detr`` or without) with a criterion
        whose losses are ``labels`` / ``boxes`` / ``cardinality`` / ``masks``: the graphs end at the mask head's inputs,
        and between them the mask head runs eagerly on the last layer's matched query rows only (see ``_mask_loss``)."""
        if track_bucket < 1:
            raise ValueError("track_bucket must be >= 1")
        self.track_bucket = int(track_bucket)
        self._prev_plans, self._track_plans = {}, {}
        self.track_captures = 0
        segm = hasattr(model, "mask_head") or "masks" in getattr(criterion, "losses", ())
        if masks and getattr(model, "two_stage", False):
            raise NotImplementedError("TrainStep(masks=True) does not train two-stage segmentation models (its mask "
                                      "step does not carry the encoder outputs); run the model and SetCriterion eagerly")
        if segm and not masks:
            raise NotImplementedError("TrainStep trains segmentation models only with masks=True (without it their "
                                      "mask losses would be dropped); or run the model and SetCriterion eagerly")
        if masks and not (hasattr(model, "mask_head") and hasattr(model, "mask_inputs")
                          and set(getattr(criterion, "losses", ())) == {"labels", "boxes", "cardinality", "masks"}):
            raise ValueError("masks=True needs a segmentation model and a criterion with the losses labels, boxes, "
                             "cardinality and masks")
        self.masks = bool(masks)
        self.model = model
        self.criterion = criterion
        self.max_norm = max_norm
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        prepare = getattr(getattr(model, "backbone", [None])[0], "prepare", None)
        if prepare is not None:
            prepare()                                   # final parameter memory formats before gradient views exist
        self.params: List[nn.Parameter] = [p for p in model.parameters() if p.requires_grad]
        self.core = _DetectorCore(model, self.masks)
        # The loss normaliser (world-averaged box count, detr.py:397-401) is a device scalar in a static buffer, refreshed
        # every step by ONE scalar all-reduce that every rank issues on every path -- so ranks may take different
        # paths (full-step graph / two graphs / eager) in the same step and still run the same collective sequence.
        self.s_num_boxes = None
        self.g_fwd = self.g_bwd = self.g_full = None
        # input prefetch (see prefetch()): staging buffer + copy stream, created on first use
        self._staged = self._staging = self._copy_stream = self._staged_ready = self._staging_free = None
        # gradient hand-over instead of per-parameter accumulation (see _backward_into_flat)
        self.gather_grads = os.environ.get("TFB200_GATHER_GRADS", "1") != "0"

        # flat layout: groups (if any) are contiguous and start on a 16-byte boundary
        groups = None
        names = {id(p): n for n, p in model.named_parameters()}
        is_bb = lambda p: names.get(id(p), "").startswith("backbone.")                       # noqa: E731
        if flat_adamw is not None:
            assert optimizer_factory is None, "give either optimizer_factory or flat_adamw"
            groups = [dict(g, params=list(g["params"])) for g in flat_adamw["groups"]]
            # groups made of backbone parameters go last: the flat buffers then read [transformer | backbone], the
            # order in which the backward finishes them (see _phases)
            groups.sort(key=lambda g: bool(g["params"]) and all(is_bb(p) for p in g["params"]))
            ordered = [p for g in groups for p in g["params"]]
            assert len({id(p) for p in ordered}) == len(ordered) == len(self.params) and \
                {id(p) for p in ordered} == {id(p) for p in self.params}, "groups must partition the trainable parameters"
            self.params = ordered
        else:
            self.params.sort(key=is_bb)                                                      # stable: model order kept
        # every tensor starts on a 256-byte boundary: library GEMM / convolution kernels and the vectorised elementwise
        # kernels need 16-byte aligned operands, and a densely packed buffer would misalign everything behind the first
        # odd-sized bias (the padding -- < 64 floats per tensor -- stays zero in gradients, parameters and moments)
        align = 64
        offsets, ranges, ofs = [], [], 0
        for g in (groups or [{"params": self.params}]):
            begin = ofs = -(-ofs // align) * align
            for p in g["params"]:
                ofs = -(-ofs // align) * align
                offsets.append(ofs)
                ofs += p.numel()
            ranges.append((begin, ofs))
        total = -(-ofs // align) * align
        dev = self.params[0].device
        self._offsets = offsets
        # Backward in three pieces when several ranks run (see _phases): [0, i_bb) everything but the backbone,
        # [i_l4, end) layer4, [i_bb, i_l4) layer2-3 -- each a contiguous slice of the flat gradient
        i_bb = next((i for i, p in enumerate(self.params) if is_bb(p)), len(self.params))
        i_l4 = next((i for i, p in enumerate(self.params) if is_bb(p) and ".layer4." in names[id(p)]), len(self.params))
        trunk = getattr(getattr(model, "backbone", [None])[0], "body", None)
        contiguous_tail = all(is_bb(p) for p in self.params[i_bb:]) and \
            all(".layer4." in names[id(p)] for p in self.params[i_l4:])
        # (not for mask models: their single flat all-reduce follows the eager mask branch, same order on every rank)
        self.phased = (self.world > 1 and not self.masks and os.environ.get("TFB200_OVERLAP_AR", "1") != "0"
                       and trunk is not None
                       and hasattr(trunk, "cut") and 0 < i_bb < i_l4 < len(self.params) and contiguous_tail)
        self._trunk, self._i_bb, self._i_l4 = trunk, i_bb, i_l4
        off_bb = offsets[i_bb] if i_bb < len(offsets) else total
        off_l4 = offsets[i_l4] if i_l4 < len(offsets) else total
        self._ranges3 = ((0, off_bb), (off_l4, total), (off_bb, off_l4))
        self._comm_stream = None

        def flat_view(buf, p, o):
            chunk = buf[o:o + p.numel()]
            if p.dim() == 4 and not p.is_contiguous() and p.is_contiguous(memory_format=torch.channels_last):
                co, ci, kh, kw = p.shape                # NHWC filter: the view gets the same strides
                return chunk.view(co, kh, kw, ci).permute(0, 3, 1, 2)
            return chunk.view_as(p)

        # flat gradient buffer: param.grad are views -> one zero-fill, one all-reduce, one norm
        self.flat_grad = torch.zeros(total, dtype=torch.float32, device=dev)
        for p, o in zip(self.params, offsets):
            p.grad = flat_view(self.flat_grad, p, o)
        self._views = [p.grad for p in self.params]
        head = ("mask_head.", "bbox_attention.")
        self._mask_params = [p for p in self.params if names.get(id(p), "").startswith(head)]
        self._mask_views = [p.grad for p in self._mask_params]
        self.flat_param = None
        self.flat_optimizer = None
        if groups is not None:
            from .flat_adamw import FlatAdamW
            self.flat_param = torch.zeros(total, dtype=torch.float32, device=dev)
            with torch.no_grad():
                for p, o in zip(self.params, offsets):
                    view = flat_view(self.flat_param, p, o)
                    view.copy_(p)
                    p.data = view                        # the parameter now lives in the flat buffer
            self.flat_optimizer = FlatAdamW(groups, ranges, self.flat_param, self.flat_grad,
                                            flat_adamw.get("betas", (0.9, 0.999)), flat_adamw.get("eps", 1e-8))
        self.optimizer = optimizer_factory(self.params) if optimizer_factory is not None else None
        if use_graphs:
            assert example_frames is not None and example_frames.is_cuda
            if self.masks:
                self._capture_masks(example_frames)
            else:
                self._capture(example_frames)
            if example_targets is not None and getattr(criterion, "device_matcher", False) and not self.masks:
                self._capture_full(example_targets)

    # ------------------------------------------------------------------------------------------
    def _capture(self, example: torch.Tensor) -> None:
        """Two graphs sharing one memory pool: (1) the model forward, (2) zero-fill of the flat gradient +
        the whole model backward INCLUDING the accumulation into the flat gradient views -- so a replay leaves the
        finished gradient in ``flat_grad`` with no per-parameter eager work."""
        self.static_frames = example.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                      # warm-up off the capture path: cuDNN autotuning, memos
            for _ in range(3):
                heads = self.core(self.static_frames)
                torch.autograd.backward(heads, [torch.zeros_like(h) for h in heads])
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        pool = self._pool = torch.cuda.graph_pool_handle()
        self.g_fwd = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_fwd, pool=pool):
            self.s_heads = self.core(self.static_frames)
        self.s_gheads = [torch.zeros_like(h) for h in self.s_heads]     # cotangents, encoder heads last (two-stage)
        self.g_bwd = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_bwd, pool=pool):
            self.flat_grad.zero_()
            torch.autograd.backward(self.s_heads, self.s_gheads)
        self.flat_grad.zero_()

    def _capture_masks(self, example: torch.Tensor) -> None:
        """``_capture`` for a segmentation model: the forward graph ends at the heads and the mask branch's inputs, the
        backward graph takes a cotangent for each of them that requires grad (none with ``freeze_detr``: no graph)."""
        self.static_frames = example.clone()
        self._pool = torch.cuda.graph_pool_handle()
        self.g_fwd, self.s_outs, self.g_bwd, self.s_grads = self._warm_up_and_capture(
            lambda: self.core(self.static_frames), backward=True, count=False)

    def _capture_full(self, example_targets: list) -> None:
        """ONE graph for forward + matching cost + device Hungarian matching + loss + backward, usable whenever the
        ground truth has the captured per-image box counts (boxes / labels are copied into static buffers).  Other
        box counts take the two-graph path with the loss in between."""
        self.full_sizes = tuple(len(t["labels"]) for t in example_targets)
        if min(self.full_sizes) == 0:                      # (no collective before this point: ranks may differ here)
            return
        self.s_targets = [{"boxes": t["boxes"].clone(), "labels": t["labels"].clone()} for t in example_targets]
        dev = self.static_frames.device
        # local count for the warm-up / capture passes; __call__ overwrites it with the world average every step
        self.s_num_boxes = torch.tensor(float(max(sum(self.full_sizes), 1)), device=dev)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                                            # memos, lazy inits
            for _ in range(2):
                if self.phased:
                    self._phase_a(self.static_frames, self.s_targets, self.s_num_boxes)
                    self._phase_b()
                    self._phase_c()
                else:
                    self._heads_loss(self.core(self.static_frames), self.s_targets, self.s_num_boxes).backward()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        if self.phased:
            # three graphs: the gradient slice each one finishes is all-reduced while the next one replays
            with torch.cuda.graph(g, pool=self._pool):
                self.s_loss = self._phase_a(self.static_frames, self.s_targets, self.s_num_boxes)
            self.g_pb, self.g_pc = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.g_pb, pool=self._pool):
                self._phase_b()
            with torch.cuda.graph(self.g_pc, pool=self._pool):
                self._phase_c()
        else:
            with torch.cuda.graph(g, pool=self._pool):
                loss = self._heads_loss(self.core(self.static_frames), self.s_targets, self.s_num_boxes)
                self._backward_into_flat(loss)
                self.s_loss = loss.detach()
        self.g_full = g
        self.flat_grad.zero_()

    # ------------------------------------------------------------------------------------------ phased backward
    # With several ranks the backward runs in three pieces so that the NCCL all-reduce of a finished slice of the flat
    # gradient overlaps the rest of the backward (what DistributedDataParallel's buckets give the reference,
    # src/train.py:86-89):   A  forward + loss + backward of everything but the backbone   -> slice [transformer]
    #                        B  backward of layer4                                           -> slice [layer4]
    #                        C  backward of layer3 + layer2                                  -> slice [layer2-3]
    # The trunk hands the transformer (and layer4) DETACHED copies of its stage outputs (backbone.py `cut`), so each
    # piece is an ordinary autograd.grad call whose cotangents come from the previous piece.  Same values as the
    # monolithic backward (the chain rule, evaluated in the same order).
    def _gather(self, first: int, params, grads) -> None:
        views = self._views[first:first + len(params)]
        dst = [v for v, g in zip(views, grads) if g is not None]
        src = [g for g in grads if g is not None]
        if dst:
            torch._foreach_copy_(dst, src)
        for v, g in zip(views, grads):
            if g is None:
                v.zero_()

    def _phase_a(self, frames, targets, num_boxes):
        rec = {}

        def cut(tag, t):
            if not t.requires_grad:
                return t
            leaf = t.detach().requires_grad_(True)
            rec[tag] = (t, leaf)
            return leaf
        self._trunk.cut = cut
        try:
            heads = self.core(frames)
        finally:
            self._trunk.cut = None
        loss = self._heads_loss(heads, targets, num_boxes)
        head = self.params[:self._i_bb]
        tags = list(rec)
        grads = torch.autograd.grad(loss, head + [rec[t][1] for t in tags], allow_unused=True)
        self._gather(0, head, grads[:len(head)])
        self._cut_out = {t: rec[t][0] for t in tags}
        self._cut_leaf = {t: rec[t][1] for t in tags}
        self._cut_grad = dict(zip(tags, grads[len(head):]))
        return loss.detach()

    def _phase_b(self) -> None:
        tail = self.params[self._i_l4:]
        x4, g4 = self._cut_out.get("layer4/tap"), self._cut_grad.get("layer4/tap")
        nxt = self._cut_leaf.get("layer3/next")
        self._g_next = None
        if x4 is None or g4 is None:
            self._gather(self._i_l4, tail, [None] * len(tail))
            return
        grads = torch.autograd.grad([x4], tail + ([nxt] if nxt is not None else []), grad_outputs=[g4], allow_unused=True)
        self._gather(self._i_l4, tail, grads[:len(tail)])
        if nxt is not None:
            self._g_next = grads[len(tail)]

    def _phase_c(self) -> None:
        mid = self.params[self._i_bb:self._i_l4]
        outs, cots = [], []
        x3 = self._cut_out.get("layer3/tap", self._cut_out.get("layer3/next"))
        g3 = self._cut_grad.get("layer3/tap")
        if self._g_next is not None:
            g3 = self._g_next if g3 is None else g3 + self._g_next
        if x3 is not None and g3 is not None:
            outs.append(x3)
            cots.append(g3)
        x2, g2 = self._cut_out.get("layer2/tap"), self._cut_grad.get("layer2/tap")
        if x2 is not None and g2 is not None:
            outs.append(x2)
            cots.append(g2)
        if not outs:
            self._gather(self._i_bb, mid, [None] * len(mid))
            return
        self._gather(self._i_bb, mid, torch.autograd.grad(outs, mid, grad_outputs=cots, allow_unused=True))

    def _all_reduce_slice(self, which: int):
        """start the all-reduce of one of the three gradient slices on the communication stream"""
        a, b = self._ranges3[which]
        if b <= a:
            return None
        view = self.flat_grad[a:b]
        if view.is_cuda:
            if self._comm_stream is None:
                self._comm_stream = torch.cuda.Stream()
            self._comm_stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self._comm_stream):
                return dist.all_reduce(view, async_op=True)
        return dist.all_reduce(view, async_op=True)

    def _backward_into_flat(self, loss: torch.Tensor) -> None:
        """``loss.backward()`` leaving the gradient in ``flat_grad``.

        Accumulating into the flat views costs one small add launch per parameter (~300 per step, each reading the view
        it was just zero-filled into).  Instead the views are detached for the duration of the backward, so autograd
        simply hands each parameter its finished gradient tensor, and ONE multi-tensor copy gathers them into the flat
        buffer; parameters that received no gradient get their slice zeroed.  Same values (a + 0 = a)."""
        if not self.gather_grads:
            self.flat_grad.zero_()
            loss.backward()
            return
        views = [p.grad for p in self.params]
        for p in self.params:
            p.grad = None
        try:
            loss.backward()
            got = [p.grad for p in self.params]
        finally:
            for p, v in zip(self.params, views):
                p.grad = v
        dst = [v for v, g in zip(views, got) if g is not None]
        src = [g for g in got if g is not None]
        if dst:
            torch._foreach_copy_(dst, src)
        for v, g in zip(views, got):
            if g is None:
                v.zero_()

    def _heads_loss(self, heads, targets, num_boxes=None):
        """``_loss`` of the detector's ``heads`` (see ``_DetectorCore``): two-stage encoder heads included"""
        return self._loss(heads[0], heads[1], targets, num_boxes, enc=tuple(heads[2:4]) if len(heads) > 2 else None)

    def _loss(self, logits, boxes, targets, num_boxes=None, track_queries=False, with_dict=False, enc=None):
        """Weighted total of the criterion's entries (engine.py:139-140: sum(loss_dict[k] * weight_dict[k]));
        ``with_dict``: -> (total, loss dictionary); ``enc``: a two-stage model's encoder (logits, boxes)."""
        if track_queries:
            loss_dict = self.criterion.forward_stacked(logits, boxes, targets, num_boxes, track_queries=True)
        elif enc is not None:
            loss_dict = self.criterion.forward_stacked(logits, boxes, targets, num_boxes, enc_outputs=enc)
        else:
            loss_dict = self.criterion.forward_stacked(logits, boxes, targets, num_boxes)
        total = self._total(loss_dict)
        return (total, loss_dict) if with_dict else total

    def _total(self, loss_dict):
        wd = self.criterion.weight_dict
        stacked = getattr(loss_dict, "stacked", None)
        names = ("loss_ce", "loss_bbox", "loss_giou")
        if stacked is not None and all(k in loss_dict for k in names) and \
                not any(k in wd and not any(k == n or k.startswith(n + "_") for n in names) for k in loss_dict):
            # the same sum over the per-layer loss vectors: stack, one multiply with the [3, K] weight table, one sum
            k = stacked[0].shape[0]
            key = (k, stacked[0].device)
            if getattr(self, "_loss_w_key", None) != key:
                rows = [[float(wd.get(f"{n}_{i}", 0.0)) for i in range(k - 1)] + [float(wd.get(n, 0.0))] for n in names]
                self._loss_w = torch.tensor(rows, dtype=stacked[0].dtype, device=stacked[0].device)
                self._loss_w_key = key
            total = (torch.stack(stacked) * self._loss_w).sum()
            enc = [loss_dict[k] * wd[k] for k in loss_dict if k.endswith("_enc") and k in wd]     # two-stage encoder
            return total + sum(enc) if enc else total
        return sum(loss_dict[k] * wd[k] for k in loss_dict if k in wd)

    # ------------------------------------------------------------------------------------------ masks
    def _mask_loss(self, outs, targets, num_boxes, track_queries):
        """The whole weighted loss of a segmentation step from the detector's outputs ``outs`` (see ``_DetectorCore``).

        The box, class and cardinality terms come from ``forward_stacked`` as for the box-only models; the mask head
        then runs on the last layer's matched query rows only (``LossDict.matched``), image after image, and their
        compact logits ``[P, h, w]`` are scored pair by pair.  The reference runs the head on every query and reads the
        matched rows (detr.py:330-357): the rows are independent (own attention softmax, own GroupNorm sample, no
        dropout), so the losses and gradients are the same and unmatched rows -- filler track queries included --
        get zero gradient either way.  No host synchronisation: the per-image counts come from the targets."""
        from .criterion import mask_losses
        logits, boxes, q, memory, src, pad, *fpns = outs
        box_loss, loss_dict = self._loss(logits, boxes, targets, num_boxes, track_queries, with_dict=True)
        if num_boxes is None:
            num_boxes = self.criterion._num_boxes(targets, logits.device)
        _, rows, tgt = loss_dict.matched
        if sum(loss_dict.matched_sizes) == 0:           # no pair: both mask losses are 0 (detr.py:330-357)
            return box_loss
        pred =self.model.mask_logits_from(q, memory, src, pad, fpns, rows=(rows, loss_dict.matched_sizes))
        found = mask_losses(pred[None], torch.arange(pred.shape[0], device=pred.device), tgt, targets, num_boxes)
        wd = self.criterion.weight_dict
        return box_loss + found["loss_mask"] * wd["loss_mask"] + found["loss_dice"] * wd["loss_dice"]

    def _mask_backward(self, loss) -> None:
        """``_backward_into_flat`` of a segmentation step (eager paths)."""
        if loss.requires_grad:
            self._backward_into_flat(loss)
        else:                                   # frozen detector and no matched row: nothing trains
            self.flat_grad.zero_()

    def _mask_step_replayed(self, outs, grads, g_bwd, targets, num_boxes, track_queries):
        """A segmentation step between its graphs (``outs`` just replayed): loss, mask branch and ONE autograd.grad
        into the cotangent buffers ``grads`` and the mask head's parameters, then the backward graph (which zero-fills
        ``flat_grad``) and only after it the mask head's gradients into their slices of ``flat_grad``."""
        leaves = [o.detach().requires_grad_(True) if g is not None else o.detach() for o, g in zip(outs, grads)]
        loss = self._mask_loss(leaves, targets, num_boxes, track_queries)
        inputs = [x for x, g in zip(leaves, grads) if g is not None]
        wrt = inputs + self._mask_params
        got = torch.autograd.grad(loss, wrt, allow_unused=True) if loss.requires_grad and wrt else [None] * len(wrt)
        for dst, g in zip([g for g in grads if g is not None], got[:len(inputs)]):
            if g is None:
                dst.zero_()
            else:
                dst.copy_(g)
        if g_bwd is not None:
            g_bwd.replay()
        else:
            self.flat_grad.zero_()
        head = got[len(inputs):]
        dst = [v for v, g in zip(self._mask_views, head) if g is not None]
        if dst:
            torch._foreach_copy_(dst, [g for g in head if g is not None])
        return loss

    # ------------------------------------------------------------------------------------------ tracking
    def _tracking_route(self, targets) -> str:
        """How ``step(frames, targets)`` runs, decided by the model, the criterion and the targets:

        ``"detect"``  the detection step: the model is not a tracking model in training mode, or the targets carry no
                      ``prev_image`` (the tracking model then trains detection, as its own forward would);
        ``"eager"``   the reference composition -- model(frames, targets) + ``criterion.forward`` + backward into the flat
                      gradient -- for what the decomposed step does not cover: a previous-previous frame
                      (``prev_prev_image``), backpropagation through the previous frame, and criteria other than the
                      box-only ones (``labels`` / ``boxes`` / ``cardinality``, either classifier);
        ``"track"``   everything else: the decomposed step of ``_track_step``."""
        from .detr_tracking import DETRTrackingBase
        model, crit = self.model, self.criterion
        if (not isinstance(model, DETRTrackingBase) or not model.training or model._tracking or not targets
                or "prev_image" not in targets[0]):
            return "detect"
        losses = {"labels", "boxes", "cardinality"} | ({"masks"} if getattr(self, "masks", False) else set())
        if ("prev_prev_image" in targets[0] or model._backprop_prev_frame
                or set(crit.losses) != losses
                or not hasattr(crit.matcher, "match_layers_forced")):
            return "eager"
        return "track"

    def _tracking_eager(self, frames, targets, num_boxes):
        out, targets_out, _, _, _ = self.model(frames, targets)
        loss_dict = self.criterion(out, targets_out, num_boxes)
        wd = self.criterion.weight_dict
        loss = sum(loss_dict[k] * wd[k] for k in loss_dict if k in wd)
        self._backward_into_flat(loss)
        return loss

    def _graphs(self) -> bool:
        return self.g_fwd is not None

    def _warm_up_and_capture(self, run, backward: bool, count: bool = True):
        """Capture ``run`` (and, with ``backward``, the zero-fill + backward of its outputs) into graphs of the step's
        pool.  The warm-up passes draw nothing from the CPU generator; its state is restored regardless, so that the
        track-query decisions of a step do not depend on whether it captured.  Outputs that do not require grad get no
        cotangent buffer (None in ``grads``); when none does, there is no backward graph."""
        with torch.random.fork_rng(devices=[]):
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    outs = run()
                    diff = [o for o in outs if o.requires_grad]
                    if backward and diff:
                        torch.autograd.backward(diff, [torch.zeros_like(o) for o in diff])
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            g_fwd = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g_fwd, pool=self._pool):
                outs = run()
            g_bwd = grads = None
            if backward:
                grads = [torch.zeros_like(o) if o.requires_grad else None for o in outs]
                diff = [(o, g) for o, g in zip(outs, grads) if g is not None]
                if diff:
                    g_bwd = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g_bwd, pool=self._pool):
                        self.flat_grad.zero_()
                        torch.autograd.backward([o for o, _ in diff], [g for _, g in diff])
                self.flat_grad.zero_()
        if count:
            self.track_captures += 1
        return g_fwd, outs, g_bwd, grads

    def _previous_frame(self, targets):
        """Step 1: the previous frames through the detector under no_grad (training mode, as the reference runs them),
        replayed from one graph per image shape.  -> (logits, boxes, hs_embed of the last layer, backbone features)."""
        images = [t["prev_image"] for t in targets]
        if not self._graphs() or len({tuple(im.shape) for im in images}) != 1:
            with torch.no_grad():
                out, _, features, _, _ = self.core.detector(images)
            return out["pred_logits"], out["pred_boxes"], out["hs_embed"], features, None
        frames = torch.stack(images)
        key = (tuple(frames.shape), frames.dtype)
        plan = self._prev_plans.get(key)
        if plan is None:
            plan = {"frames": frames.clone()}

            def run():
                with torch.no_grad():
                    out, _, features, _, _ = self.core.detector(plan["frames"])
                plan["features"] = features
                return out["pred_logits"], out["pred_boxes"], out["hs_embed"]
            plan["graph"], plan["outs"], _, _ = self._warm_up_and_capture(run, backward=False)
            self._prev_plans[key] = plan
        plan["frames"].copy_(frames)
        plan["graph"].replay()
        return (*plan["outs"], plan["features"], key)

    def _previous_matching(self, logits, boxes, prev_targets):
        """Step 2: the previous frame's last layer against its boxes, unforced -- what the model's own matcher computes
        (detr_tracking.py) -- on the device, with the pairs read back once for the bookkeeping."""
        matcher = self.model._matcher
        sizes = [len(t["boxes"]) for t in prev_targets]
        found = None
        if logits.is_cuda and self.criterion.device_matcher and min(sizes) > 0:
            found = matcher.match_layers_device(logits[None], boxes[None], prev_targets)
        if found is None:
            return matcher({"pred_logits": logits, "pred_boxes": boxes}, prev_targets)
        src, tgt, status = found
        host = torch.cat([src[0], tgt[0], status.long()]).cpu()
        if int(host[-1]) != 0:
            raise RuntimeError(f"device Hungarian matching failed (status {int(host[-1])})")
        n = sum(sizes)
        src_h, tgt_h = host[:n], host[n:2 * n]
        out, ofs = [], 0
        for size in sizes:
            out.append((src_h[ofs:ofs + size].clone(), tgt_h[ofs:ofs + size] - ofs))
            ofs += size
        return out

    def _track_step(self, frames, targets, num_boxes):
        """The reference's tracking step (DETRTrackingBase.forward(samples, targets) + criterion + backward), in pieces:

          1. previous frames, no_grad, from a graph per image shape (``_previous_frame``);
          2. their matching on the device (``_previous_matching``);
          3. the model's own ``add_track_queries_to_targets``, unchanged: the same decisions and the same CPU-generator
             draws as the eager model -- the only host reads of the step (boxes, matched pairs, track ids) are here;
          4. the current frame with the K track queries padded to a multiple of ``track_bucket`` (filler rows hidden
             from the real queries by ``track_query_padding``), replayed from a forward and a backward graph per padded
             count, with the forced device matching and the row-masked fused loss in between (``_track_current``).

        Without graphs (``use_graphs=False``, or on the CPU) the same pieces run eagerly.

        Memory: every captured current-frame bucket keeps its own forward activations alive in the shared pool (its
        backward graph consumes them at replay), so each bucket costs about one forward's saved activations, plus one
        previous-frame graph per image shape; the backward graphs' temporaries are shared.  A coarser ``track_bucket``
        means fewer buckets."""
        prev_targets = [t["prev_target"] for t in targets]
        logits, boxes, hs, features, prev_key = self._previous_frame(targets)
        prev_indices = self._previous_matching(logits, boxes, prev_targets)
        self.model.add_track_queries_to_targets(targets, prev_indices, {"pred_boxes": boxes, "hs_embed": hs})
        uses_prev = bool(getattr(self.model, "multi_frame_attention", False) or
                         getattr(self.model, "merge_frame_features", False))
        return self._track_current(frames, targets, num_boxes, features if uses_prev else None,
                                   prev_key if uses_prev else None)

    def _track_current(self, frames, targets, num_boxes, prev_features, prev_key):
        """Step 4 of ``_track_step``: no host synchronisation from here to the end of the step."""
        n_track = {int(t["track_query_boxes"].shape[0]) for t in targets}
        if len(n_track) != 1:
            raise ValueError("every image of a tracking batch needs the same number of track queries")
        k = n_track.pop()
        kb = 0 if k == 0 else -(-k // self.track_bucket) * self.track_bucket
        padded = self.track_bucket > 1 and kb > 0
        bs, dev = frames.shape[0], frames.device
        dim = self.model.hidden_dim
        # graphs read the previous frame's features from its graph's static buffers: none when that frame ran eagerly
        graphed = self._graphs() and (prev_features is None or prev_key is not None)
        key = (tuple(frames.shape), frames.dtype, kb, prev_key)
        plan = self._track_plans.get(key) if graphed else None
        new = plan is None
        if new:
            plan = {"frames": frames.clone() if graphed else frames, "hs": torch.zeros(bs, kb, dim, device=dev),
                    "boxes": torch.full((bs, kb, 4), 0.5, device=dev),
                    "padding": torch.zeros(bs, kb, dtype=torch.bool, device=dev), "slot": torch.arange(kb, device=dev)}
            if graphed:
                self._track_plans[key] = plan
        elif plan["frames"] is not frames:
            plan["frames"].copy_(frames, non_blocking=True)
        track_targets = None
        if kb:
            plan["hs"][:, :k].copy_(torch.stack([t["track_query_hs_embeds"] for t in targets]))
            plan["boxes"][:, :k].copy_(torch.stack([t["track_query_boxes"] for t in targets]))
            plan["padding"].copy_((plan["slot"] >= k).expand(bs, kb))
            track_targets = [{"track_query_hs_embeds": plan["hs"][b], "track_query_boxes": plan["boxes"][b]}
                             for b in range(bs)]
            if padded:
                for b, tt in enumerate(track_targets):
                    tt["track_query_padding"] = plan["padding"][b]
        loss_targets = [dict(t, track_query_padding=plan["padding"][b]) if padded else t for b, t in enumerate(targets)]

        def run():
            return self.core.track(plan["frames"], track_targets, prev_features)

        if not graphed:
            if self.masks:
                loss = self._mask_loss(run(), loss_targets, num_boxes, True)
                self._mask_backward(loss)
                return loss
            logits, boxes = run()
            loss = self._loss(logits, boxes, loss_targets, num_boxes, track_queries=True)
            self._backward_into_flat(loss)
            return loss
        if new:
            plan["g_fwd"], plan["outs"], plan["g_bwd"], plan["grads"] = self._warm_up_and_capture(run, backward=True)
        plan["g_fwd"].replay()
        if self.masks:
            return self._mask_step_replayed(plan["outs"], plan["grads"], plan["g_bwd"], loss_targets, num_boxes, True)
        logits, boxes = (o.detach().requires_grad_(True) for o in plan["outs"])
        loss = self._loss(logits, boxes, loss_targets, num_boxes, track_queries=True)
        for dst, g in zip(plan["grads"], torch.autograd.grad(loss, (logits, boxes))):
            dst.copy_(g)
        plan["g_bwd"].replay()
        return loss

    def _normaliser(self, targets, device):
        if self.s_num_boxes is None:
            self.s_num_boxes = torch.ones((), device=device)
        if hasattr(self.criterion, "num_boxes_device"):
            return self.criterion.num_boxes_device(targets, device, out=self.s_num_boxes)
        return None

    def prefetch(self, frames: torch.Tensor) -> None:
        """Start moving the NEXT step's frames (pinned host memory) to the device on a side stream, so that the copy
        runs under the step that is executing; the next ``step(None, targets)`` consumes them.  The data loader's job in
        a training loop (the reference moves each batch synchronously at the top of the iteration, engine.py:126-128)."""
        dev = self.flat_grad.device
        if dev.type != "cuda":
            self._staged = frames
            return
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(dev)
            self._staged_ready, self._staging_free = torch.cuda.Event(), torch.cuda.Event()
            self._staging_free.record(torch.cuda.current_stream(dev))
        if self._staging is None or self._staging.shape != frames.shape or self._staging.dtype != frames.dtype:
            self._staging = torch.empty(frames.shape, dtype=frames.dtype, device=dev)
        cs = self._copy_stream
        cs.wait_event(self._staging_free)               # the previous step has finished reading the staging buffer
        with torch.cuda.stream(cs):
            self._staging.copy_(frames, non_blocking=True)
        self._staged_ready.record(cs)
        self._staged = self._staging

    def _release_staging(self, dev):
        if self._staging_free is not None:
            self._staging_free.record(torch.cuda.current_stream(dev))

    def __call__(self, frames: Optional[torch.Tensor], targets: list) -> torch.Tensor:
        dev = self.flat_grad.device
        staged = frames is None
        if staged:
            if self._staged is None:
                raise ValueError("step(None, targets) needs frames handed over with prefetch() first")
            frames, self._staged = self._staged, None
            if dev.type == "cuda":
                torch.cuda.current_stream(dev).wait_event(self._staged_ready)
        route = self._tracking_route(targets)
        full = (route == "detect" and self.g_full is not None
                and tuple(len(t["labels"]) for t in targets) == self.full_sizes)
        # one scalar all-reduce per step on EVERY path, before anything else (same collective order on all ranks)
        num_boxes = self._normaliser(targets, dev) if (self.world > 1 or full or route == "track"
                                                       or self.masks) else None
        pending = None
        if route != "detect":
            loss = (self._track_step if route == "track" else self._tracking_eager)(frames, targets, num_boxes)
        elif full:
            if frames is not self.static_frames:
                self.static_frames.copy_(frames, non_blocking=True)     # device or pinned-host source
            if staged and dev.type == "cuda":
                self._release_staging(dev)
                staged = False
            for st, t in zip(self.s_targets, targets):
                if t["boxes"] is not st["boxes"]:
                    st["boxes"].copy_(t["boxes"], non_blocking=True)
                    st["labels"].copy_(t["labels"], non_blocking=True)
            self.g_full.replay()
            loss = self.s_loss
            if self.phased:
                pending = [self._all_reduce_slice(0)]
                self.g_pb.replay()
                pending.append(self._all_reduce_slice(1))
                self.g_pc.replay()
                pending.append(self._all_reduce_slice(2))
        elif self.phased and self.g_fwd is None:
            loss = self._phase_a(frames, targets, num_boxes)
            pending = [self._all_reduce_slice(0)]
            self._phase_b()
            pending.append(self._all_reduce_slice(1))
            self._phase_c()
            pending.append(self._all_reduce_slice(2))
        elif self.masks:
            if self.g_fwd is not None:
                if frames is not self.static_frames:
                    self.static_frames.copy_(frames, non_blocking=True)
                if staged and dev.type == "cuda":
                    self._release_staging(dev)
                    staged = False
                self.g_fwd.replay()
                loss = self._mask_step_replayed(self.s_outs, self.s_grads, self.g_bwd, targets, num_boxes, False)
            else:
                loss = self._mask_loss(self.core(frames), targets, num_boxes, False)
                self._mask_backward(loss)
        elif self.g_fwd is not None:
            if frames is not self.static_frames:
                self.static_frames.copy_(frames, non_blocking=True)     # device or pinned-host source
            if staged and dev.type == "cuda":
                self._release_staging(dev)
                staged = False
            self.g_fwd.replay()
            heads = [h.detach().requires_grad_(True) for h in self.s_heads]
            loss = self._heads_loss(heads, targets, num_boxes)
            for dst, g in zip(self.s_gheads, torch.autograd.grad(loss, heads)):
                dst.copy_(g)
            self.g_bwd.replay()
        else:
            loss = self._heads_loss(self.core(frames), targets, num_boxes)
            self._backward_into_flat(loss)
        if self.world > 1:
            if self.phased:
                # every path issues the SAME three collectives in the same order (ranks may take different paths)
                if pending is None:
                    pending = [self._all_reduce_slice(i) for i in range(3)]
                for work in pending:
                    if work is not None:
                        work.wait()
            else:
                dist.all_reduce(self.flat_grad)
            self.flat_grad.div_(self.world)
        if self.optimizer is not None:
            if self.max_norm > 0:
                # clip_grad_norm_ over a flat buffer: one norm, one scale, no host sync
                norm = torch.linalg.vector_norm(self.flat_grad)
                self.flat_grad.mul_(torch.clamp(self.max_norm / (norm + 1e-6), max=1.0))
            self.optimizer.step()
        elif self.flat_optimizer is not None:
            norm = torch.linalg.vector_norm(self.flat_grad) if self.max_norm > 0 else None
            self.flat_optimizer.step(norm, self.max_norm)
        if staged and dev.type == "cuda":                # eager paths read the staging buffer directly: free it now
            self._release_staging(dev)
        return loss.detach()
