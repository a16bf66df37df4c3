"""uint8 video frames straight into the detector: the reference's validation transform on the GPU, bit for bit.

The reference's sequence datasets (src/trackformer/datasets/tracking/mot17_sequence.py:68-81) turn every frame into the
detector's input on one CPU thread: `RandomResize([val_width], max_size)` (datasets/coco.py:304-307 ->
datasets/transforms.py:115-145, Pillow's bilinear resize of the 8-bit image), `ToTensor` and
`Normalize([0.485, 0.456, 0.406], [0.229, 0.224, 0.225])`.  `FrameIngest` takes the `H x W x 3` uint8 RGB frame itself --
host or device memory -- and produces the same `img`, `size` and `orig_size` with one launch of csrc/frame_ingest.cu.

The result is not close to the reference's, it is equal: Pillow resamples 8-bit images in integers (weights quantised to
22 fractional bits, the intermediate image rounded to bytes between the horizontal and the vertical pass), and the byte
to float step is a 3 x 256 table built here with the reference's own torch ops.  The per-axis coefficient tables are
built on the host in double precision exactly as Pillow builds them, cached per (input length, output length) and
uploaded once.

No CPU path: the constructor raises on a non-CUDA device.
"""
import math

import numpy as np
import torch

from .util import NestedTensor

__all__ = ["FrameIngest", "val_size", "resample_table", "normalise_table", "check_frame"]

PRECISION_BITS = 22
IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
_LAYOUT = "expected one uint8 RGB frame of shape [H, W, 3] (interleaved channels last; numpy array or torch tensor)"


def val_size(height, width, val_width=800, max_size=1333):
    """(h, w) the validation transform resizes a `height x width` frame to (`get_size_with_aspect_ratio`,
    datasets/transforms.py:118-136): shorter side to `val_width` unless that pushes the longer side beyond `max_size`,
    in which case the shorter side becomes `int(round(max_size * short / long))`; the longer side is truncated, not
    rounded; a frame whose shorter side already has the target length is returned unchanged."""
    h, w, size = int(height), int(width), int(val_width)
    if h <= 0 or w <= 0 or size <= 0 or (max_size is not None and max_size <= 0):
        raise ValueError(f"val_size: sizes must be positive, got {height} x {width}, val_width={val_width}, "
                         f"max_size={max_size}")
    if max_size is not None:
        short, long = float(min(w, h)), float(max(w, h))
        if long / short * size > max_size:
            size = int(round(max_size * short / long))
    if (w <= h and w == size) or (h <= w and h == size):
        return h, w
    if w < h:
        return int(size * h / w), size
    return size, int(size * w / h)


def resample_table(in_size, out_size):
    """Pillow's bilinear coefficients for one axis (`precompute_coeffs` + `normalize_coeffs_8bpc`) as an int32 array
    [out_size, 2 + ksize]: per output index {lo, cnt, k_0 .. k_{ksize-1}}; the output is
    clamp((2^21 + sum_{j < cnt} pixel[lo + j] * k_j) >> 22, 0, 255).  All arithmetic in double, in Pillow's order."""
    n, m = int(in_size), int(out_size)
    if n <= 0 or m <= 0:
        raise ValueError(f"resample_table: lengths must be positive, got {in_size} -> {out_size}")
    scale = n / m
    fs = max(scale, 1.0)
    support = 1.0 * fs                                   # bilinear: a triangle of half-width 1, widened when reducing
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / fs
    center = (np.arange(m, dtype=np.float64) + 0.5) * scale
    lo = np.maximum((center - support + 0.5).astype(np.int64), 0)          # C's (int): truncation
    cnt = np.minimum((center + support + 0.5).astype(np.int64), n) - lo
    j = np.arange(ksize, dtype=np.int64)[None, :]
    a = np.abs((j + lo[:, None] - center[:, None] + 0.5) * ss)
    wgt = np.where((a < 1.0) & (j < cnt[:, None]), 1.0 - a, 0.0)
    total = np.zeros(m, np.float64)
    for col in range(ksize):                             # Pillow accumulates the sum tap by tap
        total = total + wgt[:, col]
    wgt = np.where(total[:, None] != 0.0, wgt / np.where(total == 0.0, 1.0, total)[:, None], wgt)
    table = np.empty((m, 2 + ksize), np.int32)
    table[:, 0], table[:, 1] = lo, cnt
    table[:, 2:] = (0.5 + wgt * float(1 << PRECISION_BITS)).astype(np.int64)   # weights are >= 0: truncation rounds
    return table


def normalise_table(mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """[3, 256] fp32: entry [c][u] is what `to_tensor` + `normalize(mean, std)` make of byte u in channel c, computed
    with the same torch ops (`float().div(255)`, `sub(mean).div(std)`), so a look-up reproduces them bit for bit."""
    mean = torch.as_tensor(mean, dtype=torch.float32).reshape(-1)
    std = torch.as_tensor(std, dtype=torch.float32).reshape(-1)
    if mean.numel() != 3 or std.numel() != 3:
        raise ValueError("FrameIngest: mean and std need three values (R, G, B)")
    if bool((std == 0).any()):
        raise ValueError("FrameIngest: std must not contain zeros")
    u = torch.arange(256, dtype=torch.uint8)[None, :].expand(3, 256)
    return u.float().div(255).sub_(mean[:, None]).div_(std[:, None]).contiguous()


def check_frame(frame):
    """Validate one frame and return (kind, H, W), kind in {"numpy", "cpu", "cuda"}; ValueError names the layout."""
    if isinstance(frame, np.ndarray):
        kind, dtype_ok = "numpy", frame.dtype == np.uint8
    elif torch.is_tensor(frame):
        kind, dtype_ok = ("cuda" if frame.is_cuda else "cpu"), frame.dtype == torch.uint8
    else:
        raise ValueError(f"FrameIngest: got {type(frame).__name__}; {_LAYOUT}")
    shape = tuple(frame.shape)
    if not dtype_ok:
        raise ValueError(f"FrameIngest: got dtype {frame.dtype}; {_LAYOUT}")
    if len(shape) != 3 or shape[2] != 3 or shape[0] < 1 or shape[1] < 1:
        raise ValueError(f"FrameIngest: got shape {shape}; {_LAYOUT}")
    if kind == "cuda" and (frame.stride(2) != 1 or frame.stride(1) != 3 or frame.stride(0) < 3 * shape[1]):
        raise ValueError(f"FrameIngest: got a CUDA tensor with strides {tuple(frame.stride())}; {_LAYOUT}, "
                         f"pixels contiguous within a row (only the row stride is free)")
    return kind, shape[0], shape[1]


class _Buffers:
    """What one input shape needs, allocated at its first frame and reused afterwards."""

    def __init__(self, H, W, h, w, device):
        self.staging = torch.empty(H, W, 3, dtype=torch.uint8).pin_memory()
        self.frame = torch.empty(H, W, 3, dtype=torch.uint8, device=device)
        self.img = torch.empty(1, 3, h, w, dtype=torch.float32, device=device)
        self.size = torch.tensor([[h, w]])
        self.orig_size = torch.tensor([[H, W]])
        self.uploaded = torch.cuda.Event()
        self.pending = False


class FrameIngest:
    """`FrameIngest(device)(frame)` -> `{"img": [1, 3, h, w] fp32 on the device, "size": [[h, w]], "orig_size":
    [[H, W]]}`: the keys and shapes of the reference's sequence blobs, with `(h, w) = val_size(H, W, val_width,
    max_size)`.

    `frame` is one `[H, W, 3]` uint8 RGB image: a numpy array or CPU tensor (copied through a pinned staging buffer the
    object owns, asynchronously on the current stream) or a CUDA tensor (read in place; its rows may be strided).
    Everything is enqueued on the current stream and nothing synchronises with the host, except that re-filling the
    staging buffer waits for the previous upload from it.

    Buffers are kept per input shape and reused, so a steady sequence allocates nothing after its first frame.  The
    returned `img` is therefore only VALID UNTIL THE NEXT CALL WITH THE SAME INPUT SHAPE (`GraphedDetector` copies it
    into its static buffer at once; clone it to keep it).  `batch` returns fresh tensors.
    """

    def __init__(self, device, val_width=800, max_size=1333, mean=IMAGENET_MEAN, std=IMAGENET_STD):
        val_size(1, 1, val_width, max_size)               # validates the two settings
        lut = normalise_table(mean, std)
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError(f"FrameIngest runs in a CUDA kernel and has no CPU path (device {device}); the reference's "
                               f"host transform is datasets/transforms.py")
        from . import ext
        self._ext = ext.load()                            # raises with the build command when the native code is missing
        self.device = device if device.index is not None else torch.device("cuda", torch.cuda.current_device())
        self.val_width, self.max_size = int(val_width), (None if max_size is None else int(max_size))
        self._lut = lut.to(self.device)
        self._tables = {}                                 # (in, out) -> (device table, largest cnt) or (None, 0)
        self._buffers = {}                                # (H, W) -> _Buffers

    # ------------------------------------------------------------------------------------------------- internals
    def _table(self, n, m):
        if n == m:                                        # Pillow skips a pass that keeps the length
            return None, 0
        entry = self._tables.get((n, m))
        if entry is None:
            table = resample_table(n, m)
            entry = (torch.from_numpy(table).to(self.device), int(table[:, 1].max()))
            self._tables[(n, m)] = entry
        return entry

    def _buffers_for(self, H, W):
        buf = self._buffers.get((H, W))
        if buf is None:
            buf = _Buffers(H, W, *val_size(H, W, self.val_width, self.max_size), self.device)
            self._buffers[(H, W)] = buf
        return buf

    def _run(self, frame, dst):
        """Enqueue upload (if needed) and kernel for one validated frame; dst is a [3, h, w] view on the device."""
        kind, H, W = check_frame(frame)
        buf = self._buffers_for(H, W)
        if kind == "cuda":
            if frame.device != self.device:
                raise ValueError(f"FrameIngest: frame on {frame.device}, ingest on {self.device}")
            src = frame
        else:
            if buf.pending:
                buf.uploaded.synchronize()                # the previous upload still reads the staging buffer
            if kind == "numpy":
                np.copyto(buf.staging.numpy(), frame)
            else:
                buf.staging.copy_(frame)
            buf.frame.copy_(buf.staging, non_blocking=True)
            buf.uploaded.record(torch.cuda.current_stream(self.device))
            buf.pending = True
            src = buf.frame
        h, w = int(dst.shape[1]), int(dst.shape[2])
        xtab, xcnt = self._table(W, w)
        ytab, ycnt = self._table(H, h)
        self._ext.frame_ingest(src, xtab, xcnt, ytab, ycnt, self._lut, dst)
        return buf

    # ---------------------------------------------------------------------------------------------------- public
    def __call__(self, frame):
        with torch.cuda.device(self.device):
            buf = self._buffers_for(*check_frame(frame)[1:])
            self._run(frame, buf.img[0])
        return {"img": buf.img, "size": buf.size, "orig_size": buf.orig_size}

    def batch(self, frames):
        """Frames of any sizes -> `(NestedTensor, sizes [B, 2], orig_sizes [B, 2])`: one zero-padded
        `[B, 3, Hmax, Wmax]` batch with its `True = padding` mask, equal to `nested_tensor_from_tensor_list` over the
        single-frame results.  The slab is zeroed once and the kernel writes every image into its corner of it."""
        frames = list(frames)
        if not frames:
            raise ValueError("FrameIngest.batch: no frames")
        orig = [check_frame(f)[1:] for f in frames]
        sizes = [val_size(H, W, self.val_width, self.max_size) for H, W in orig]
        hmax, wmax = max(s[0] for s in sizes), max(s[1] for s in sizes)
        with torch.cuda.device(self.device):
            slab = torch.zeros(len(frames), 3, hmax, wmax, dtype=torch.float32, device=self.device)
            mask = torch.ones(len(frames), hmax, wmax, dtype=torch.bool, device=self.device)
            for i, (frame, (h, w)) in enumerate(zip(frames, sizes)):
                self._run(frame, slab[i, :, :h, :w])
                mask[i, :h, :w] = False
        return NestedTensor(slab, mask), torch.tensor(sizes), torch.tensor(orig)
