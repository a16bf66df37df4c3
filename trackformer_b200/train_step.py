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
    """Tensor-in / tensors-out view of the detector for graph capture: frames -> (logits[K,B,Q,C], boxes[K,B,Q,4])."""

    def __init__(self, model):
        super().__init__()
        self.model = model

    def forward(self, frames):
        out, _, _, _, _ = self.model(frames, None, None)
        stacked = getattr(self.model, "stacked_heads", None)
        if stacked is not None and stacked[0].shape[0] == len(out["aux_outputs"]) + 1:
            return stacked                           # the very tensors the dictionary entries are slices of
        logits = torch.stack([a["pred_logits"] for a in out["aux_outputs"]] + [out["pred_logits"]])
        boxes = torch.stack([a["pred_boxes"] for a in out["aux_outputs"]] + [out["pred_boxes"]])
        return logits, boxes


class TrainStep:
    """``loss = step(frames, targets)`` -- forward, criterion, backward, [all-reduce], clip, optimizer."""

    def __init__(self, model, criterion, optimizer_factory=None, max_norm: float = 0.1,
                 use_graphs: bool = True, example_frames: Optional[torch.Tensor] = None,
                 example_targets: Optional[list] = None, flat_adamw: Optional[dict] = None):
        """``optimizer_factory(params)`` builds any torch optimizer; ``flat_adamw={'groups': [...], 'betas':..., 'eps':...}``
        (groups as for torch.optim.AdamW, e.g. flat_adamw.reference_param_groups(model)) instead lays the PARAMETERS out
        flat as well and updates them with the one-pass clip + AdamW kernel."""
        if hasattr(model, "mask_head") or "masks" in getattr(criterion, "losses", ()):
            raise NotImplementedError("TrainStep does not train segmentation models (their mask losses would be "
                                      "dropped); run the model and SetCriterion eagerly instead")
        self.model = model
        self.criterion = criterion
        self.max_norm = max_norm
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        prepare = getattr(getattr(model, "backbone", [None])[0], "prepare", None)
        if prepare is not None:
            prepare()                                   # final parameter memory formats before gradient views exist
        self.params: List[nn.Parameter] = [p for p in model.parameters() if p.requires_grad]
        self.core = _DetectorCore(model)
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
        self.phased = (self.world > 1 and os.environ.get("TFB200_OVERLAP_AR", "1") != "0" and trunk is not None
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
            self._capture(example_frames)
            if example_targets is not None and getattr(criterion, "device_matcher", False):
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
                lg, bx = self.core(self.static_frames)
                torch.autograd.backward((lg, bx), (torch.zeros_like(lg), torch.zeros_like(bx)))
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        pool = self._pool = torch.cuda.graph_pool_handle()
        self.g_fwd = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_fwd, pool=pool):
            self.s_logits, self.s_boxes = self.core(self.static_frames)
        self.s_glogits = torch.zeros_like(self.s_logits)
        self.s_gboxes = torch.zeros_like(self.s_boxes)
        self.g_bwd = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_bwd, pool=pool):
            self.flat_grad.zero_()
            torch.autograd.backward((self.s_logits, self.s_boxes), (self.s_glogits, self.s_gboxes))
        self.flat_grad.zero_()

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
                    lg, bx = self.core(self.static_frames)
                    self._loss(lg, bx, self.s_targets, self.s_num_boxes).backward()
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
                lg, bx = self.core(self.static_frames)
                loss = self._loss(lg, bx, self.s_targets, self.s_num_boxes)
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
            logits, boxes = self.core(frames)
        finally:
            self._trunk.cut = None
        loss = self._loss(logits, boxes, targets, num_boxes)
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

    def _loss(self, logits, boxes, targets, num_boxes=None):
        """Weighted total of the criterion's entries (engine.py:139-140: sum(loss_dict[k] * weight_dict[k]))."""
        loss_dict = self.criterion.forward_stacked(logits, boxes, targets, num_boxes)
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
            return (torch.stack(stacked) * self._loss_w).sum()
        return sum(loss_dict[k] * wd[k] for k in loss_dict if k in wd)

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
        full = self.g_full is not None and tuple(len(t["labels"]) for t in targets) == self.full_sizes
        # one scalar all-reduce per step on EVERY path, before anything else (same collective order on all ranks)
        num_boxes = self._normaliser(targets, dev) if (self.world > 1 or full) else None
        pending = None
        if full:
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
        elif self.g_fwd is not None:
            if frames is not self.static_frames:
                self.static_frames.copy_(frames, non_blocking=True)     # device or pinned-host source
            if staged and dev.type == "cuda":
                self._release_staging(dev)
                staged = False
            self.g_fwd.replay()
            logits = self.s_logits.detach().requires_grad_(True)
            boxes = self.s_boxes.detach().requires_grad_(True)
            loss = self._loss(logits, boxes, targets, num_boxes)
            g_logits, g_boxes = torch.autograd.grad(loss, (logits, boxes))
            self.s_glogits.copy_(g_logits)
            self.s_gboxes.copy_(g_boxes)
            self.g_bwd.replay()
        else:
            logits, boxes = self.core(frames)
            loss = self._loss(logits, boxes, targets, num_boxes)
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
