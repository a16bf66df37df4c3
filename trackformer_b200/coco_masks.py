"""COCO polygon segmentations as masks on the GPU (csrc/coco_poly.cu), equal bit for bit to pycocotools 2.0.

`convert_coco_poly_to_mask` is the reference's datasets/coco.py function of that name, which decodes every training
sample's instance masks with pycocotools on the host; here one packed upload, one read-back of sizes and one mask
launch.  `poly_runs` is what `coco_eval.GroundTruth(..., device=)` uses for polygon ground truth.

Semantics (pycocotools' `frPyObjects`, `rleFrPoly`, `rleFrBbox` and `merge`):
- A list segmentation whose first part has 4 numbers is a list of [x, y, w, h] boxes, each rasterised as the polygon
  (x, y), (x, y + h), (x + w, y + h), (x + w, y) with x + w and y + h in double; every part must then have 4 numbers.
  A first part of more than 4 numbers makes every part a polygon of len(part) // 2 vertices (a later 4-number part is a
  2-vertex polygon).  A first part of fewer than 4 numbers, or no part, is a ValueError.
- Each part is walked on pycocotools' 5x grid: vertex (int)(5 c + .5), truncated toward zero; the y-boundary toggles
  of its boundary points; a pixel is set when an odd number of the part's toggles lie at or before its column-major
  index.  The parts of one annotation are merged by union.
- Compressed RLE dicts (`convert_coco_poly_to_mask` only) are decoded on the device; a dict whose counts is a list is
  a ValueError, as the reference's function fails on it.

Limits, each a ValueError naming the annotation: a non-finite coordinate; |5 c + .5| >= 2^31 (the grid value would
overflow a C int); more than 2^31 - 1 boundary points in one call (boundary points of a part: the sum over its edges
of max(|dx|, |dy|) + 1 on the 5x grid; toggles never outnumber them); an image of 2^31 pixels or more.

Memory: the count call takes about 8 B per vertex (its workspace and the toggle offsets); the runs call 16 B per
toggle plus CUB's segmented-sort buffers, and 8 B per toggle of run capacity.  An edge crosses each pixel column
once at most, so a part has at most (its vertices) x w toggles.  At 1080 x 1920 a full-frame rectangle has 30,004
boundary points and 3,840 toggles; the worst 80-vertex full-frame polygon, zig-zagging between the left and right
sides, has 768,080 boundary points and 153,600 toggles: about 2.5 MB of keys and values and 1.2 MB of run capacity
besides the sort buffers.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

__all__ = ["convert_coco_poly_to_mask", "pack_polygons", "poly_runs", "check_sizes"]

SIZES = 5                        # TFB200_POLY_SIZES (include/tfb200_fused.h)
_ST, _BAD_FINITE, _BAD_RANGE = 2, 3, 4
_INT32_MAX = 2 ** 31 - 1
_ALIGN = 256


def pack_polygons(segmentations, hw, names) -> dict:
    """Host packing of list segmentations (one pass): xy [V][2] fp64, part_off [P + 1] int64, part_ann [P] int32,
    ann_part [A + 1] int64, ann_hw [A][2] int32.  `hw` [A][2] the image sizes, `names` what an error message calls
    each annotation.  Raises ValueError for segmentations pycocotools rejects."""
    flat, part_len, n_parts = [], [], []
    for seg, (h, w), name in zip(segmentations, hw, names):
        if int(h) * int(w) >= 2 ** 31:
            raise ValueError(f"coco_poly: {name}: its image is over 2^31 pixels")
        if not isinstance(seg, (list, tuple)) or len(seg) == 0 or not hasattr(seg[0], "__len__") or len(seg[0]) < 4:
            raise ValueError(f"coco_poly: {name}: a list segmentation needs a first part of at least 4 numbers")
        if len(seg[0]) == 4:                               # frBbox: [x, y, w, h] boxes
            for p in seg:
                if len(p) != 4:
                    raise ValueError(f"coco_poly: {name}: a box-list segmentation has a part of {len(p)} numbers")
                x, y, bw, bh = (float(v) for v in p)
                xe, ye = x + bw, y + bh
                flat.extend((x, y, x, ye, xe, ye, xe, y))
                part_len.append(4)
        else:                                              # frPoly: len(p) // 2 vertices per part
            for p in seg:
                k = len(p) // 2
                flat.extend(p[:2 * k])
                part_len.append(k)
        n_parts.append(len(seg))
    try:
        xy = np.asarray(flat, np.float64).reshape(-1, 2)
    except (TypeError, ValueError) as e:
        raise ValueError(f"coco_poly: a polygon coordinate is not a number ({e})") from None
    if len(xy) >= _INT32_MAX:
        raise ValueError(f"coco_poly: {len(xy)} vertices in one call, over 2^31 - 2")
    n_parts = np.asarray(n_parts, np.int64)
    return dict(xy=xy, part_off=np.concatenate(([0], np.cumsum(part_len, dtype=np.int64))),
                part_ann=np.repeat(np.arange(len(n_parts), dtype=np.int32), n_parts),
                ann_part=np.concatenate(([0], np.cumsum(n_parts))).astype(np.int64),
                ann_hw=np.asarray(hw, np.int32).reshape(-1, 2))


def geometry(z):
    """(n_parts, n_ann, n_edges) of a packing."""
    return len(z["part_ann"]), len(z["ann_hw"]), len(z["xy"])


def check_sizes(sizes, ann_points, names):
    """Raises the ValueError of a count call's sizes [5]; `ann_points()` returns its per-annotation point counts."""
    st = int(sizes[_ST])
    if st & 1:
        raise ValueError(f"coco_poly: {names[int(sizes[_BAD_FINITE])]} has a non-finite coordinate")
    if st & 2:
        raise ValueError(f"coco_poly: {names[int(sizes[_BAD_RANGE])]} has a coordinate c with |5 c + .5| >= 2^31, "
                         f"which overflows pycocotools' int grid")
    if st & 4:
        a = int(np.argmax(np.cumsum(np.asarray(ann_points(), np.int64)) > _INT32_MAX))
        raise ValueError(f"coco_poly: {names[a]} takes the boundary points of one call over 2^31 - 1")


_lib = None


def _library():
    global _lib
    if _lib is None:
        from . import ext
        ext.load()                                   # raises with the build command when the native code is missing
        lib = ctypes.CDLL(ext.library_path())
        vp, i32, i64, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_size_t
        geo = [vp] * 5 + [i32, i32, i64]
        lib.tfb200_coco_poly_count_workspace_bytes.argtypes = [i32, i32, i64]
        lib.tfb200_coco_poly_count_workspace_bytes.restype = sz
        lib.tfb200_coco_poly_count.argtypes = geo + [vp, sz, vp, vp, vp, vp]
        lib.tfb200_coco_poly_count.restype = i32
        lib.tfb200_coco_poly_runs_workspace_bytes.argtypes = [i32, i32, i64]
        lib.tfb200_coco_poly_runs_workspace_bytes.restype = sz
        lib.tfb200_coco_poly_runs.argtypes = geo + [vp, i64, vp, sz, vp, vp, vp]
        lib.tfb200_coco_poly_runs.restype = i32
        lib.tfb200_coco_rle_runs.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, vp, vp]
        lib.tfb200_coco_rle_runs.restype = i32
        lib.tfb200_coco_masks_u8.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp, vp, vp]
        lib.tfb200_coco_masks_u8.restype = i32
        _lib = lib
    return _lib


def _upload(arrays, device):
    """One host-to-device copy of several numpy arrays: a dict of device tensors viewing one buffer."""
    offs, at = {}, 0
    for k, a in arrays.items():
        offs[k] = at
        at += (a.nbytes + _ALIGN - 1) // _ALIGN * _ALIGN
    buf = np.zeros(max(at, _ALIGN), np.uint8)
    for k, a in arrays.items():
        buf[offs[k]:offs[k] + a.nbytes] = np.ascontiguousarray(a).reshape(-1).view(np.uint8)
    dev = torch.from_numpy(buf).pin_memory().to(device, non_blocking=True)
    return {k: dev[offs[k]:offs[k] + a.nbytes].view(torch.from_numpy(np.empty(0, a.dtype)).dtype)
            for k, a in arrays.items()}


def _check(rc, name):
    if rc != 0:
        raise RuntimeError(f"{name} failed (code {rc})")


def _count(lib, g, z, stream):
    P, A, E = geometry(z)
    dev = g["xy"].device
    ws_bytes = lib.tfb200_coco_poly_count_workspace_bytes(P, A, E)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    toggle_off = torch.empty(E + 1, dtype=torch.int32, device=dev)
    ann_points = torch.empty(max(A, 1), dtype=torch.int64, device=dev)
    _check(lib.tfb200_coco_poly_count(*_geo_ptrs(g), P, A, E, ws.data_ptr(), ws_bytes, toggle_off.data_ptr(),
                                      ann_points.data_ptr(), g["sizes"].data_ptr(), stream), "tfb200_coco_poly_count")
    return toggle_off, ann_points


def _runs(lib, g, z, toggle_off, n_toggles, stream):
    P, A, E = geometry(z)
    dev = g["xy"].device
    ws_bytes = lib.tfb200_coco_poly_runs_workspace_bytes(P, A, n_toggles)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    run_off = torch.empty(A + 1, dtype=torch.int64, device=dev)
    runs = torch.empty((max(n_toggles, 1), 2), dtype=torch.int32, device=dev)
    _check(lib.tfb200_coco_poly_runs(*_geo_ptrs(g), P, A, E, toggle_off.data_ptr(), n_toggles, ws.data_ptr(),
                                     ws_bytes, run_off.data_ptr(), runs.data_ptr(), stream), "tfb200_coco_poly_runs")
    return run_off, runs


def _geo_ptrs(g):
    return [g[k].data_ptr() for k in ("xy", "part_off", "part_ann", "ann_part", "ann_hw")]


def poly_runs(segmentations, hw, names, device):
    """The union runs of every list segmentation on `device`, read back: (run_off [A + 1] int64, runs [R][2] int64
    column-major start, length), annotation a's runs at run_off[a] .. run_off[a + 1].  One upload, one read-back of
    sizes, one of run_off and one of the runs."""
    z = pack_polygons(segmentations, hw, names)
    device = torch.device(device)
    g = _upload({**z, "sizes": np.zeros(SIZES, np.int64)}, device)
    lib = _library()
    stream = torch.cuda.current_stream(device).cuda_stream
    toggle_off, ann_points = _count(lib, g, z, stream)
    sizes = g["sizes"].cpu().numpy()
    check_sizes(sizes, lambda: ann_points.cpu().numpy(), names)
    run_off, runs = _runs(lib, g, z, toggle_off, int(sizes[1]), stream)
    run_off = run_off.cpu().numpy()
    return run_off, runs[:int(run_off[-1])].cpu().numpy().view(np.uint32).astype(np.int64)


def convert_coco_poly_to_mask(segmentations, height, width, device=None):
    """The reference's `convert_coco_poly_to_mask` on the GPU: uint8 [N, height, width] on `device` (default: the
    current CUDA device), mask i the union of segmentation i's parts.  Entries are list segmentations (polygons or
    [x, y, w, h] boxes) or compressed-RLE dicts of size [height, width]."""
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    H, W, N = int(height), int(width), len(segmentations)
    if H * W >= 2 ** 31:
        raise ValueError(f"convert_coco_poly_to_mask: {H}x{W} is over 2^31 pixels")
    if N == 0:
        return torch.zeros((0, H, W), dtype=torch.uint8, device=dev)
    polys, poly_names, strings, src = [], [], [], np.zeros(N, np.int32)
    for i, s in enumerate(segmentations):
        if isinstance(s, dict):
            counts = s.get("counts")
            if not isinstance(counts, (str, bytes)):
                raise ValueError(f"coco_poly: segmentation {i}: an RLE dict needs compressed (string) counts")
            if [int(v) for v in s.get("size", ())] != [H, W]:
                raise ValueError(f"coco_poly: segmentation {i}: its RLE is {s.get('size')}, the image {H}x{W}")
            src[i] = -1 - len(strings)
            strings.append(counts.encode() if isinstance(counts, str) else bytes(counts))
        else:
            src[i] = len(polys)
            polys.append(s)
            poly_names.append(f"segmentation {i}")
    z = pack_polygons(polys, [(H, W)] * len(polys), poly_names)
    str_len = np.asarray([len(c) for c in strings], np.int64)
    arrays = {**z, "src": src, "chars": np.frombuffer(b"".join(strings) or b"\0", np.uint8),
              "str_off": np.concatenate(([0], np.cumsum(str_len))).astype(np.int64),
              "cap_off": np.concatenate(([0], np.cumsum(str_len // 2))).astype(np.int64),
              "sizes": np.asarray([0, 0, 0, 0, 0, len(strings)], np.int64)}
    g = _upload(arrays, dev)
    lib = _library()
    stream = torch.cuda.current_stream(dev).cuda_stream
    dummy = g["sizes"]
    rle_bounds = torch.empty((max(len(strings), 1), 2), dtype=torch.int64, device=dev)
    rle_runs = torch.empty((max(int(arrays["cap_off"][-1]), 1), 2), dtype=torch.int32, device=dev)
    if polys:
        toggle_off, ann_points = _count(lib, g, z, stream)
    if strings:
        _check(lib.tfb200_coco_rle_runs(g["chars"].data_ptr(), g["str_off"].data_ptr(), g["cap_off"].data_ptr(),
                                        len(strings), H, W, rle_bounds.data_ptr(), rle_runs.data_ptr(),
                                        dummy[SIZES:].data_ptr(), stream), "tfb200_coco_rle_runs")
    sizes = g["sizes"].cpu().numpy()                       # the one read-back
    if int(sizes[SIZES]) < len(strings):
        raise ValueError(f"coco_poly: segmentation {int(np.flatnonzero(src == -1 - int(sizes[SIZES]))[0])}: "
                         f"a malformed RLE counts string")
    run_off, runs = dummy, dummy
    if polys:
        check_sizes(sizes, lambda: ann_points.cpu().numpy(), poly_names)
        run_off, runs = _runs(lib, g, z, toggle_off, int(sizes[1]), stream)
    out = torch.empty((N, H, W), dtype=torch.uint8, device=dev)
    _check(lib.tfb200_coco_masks_u8(g["src"].data_ptr(), N, H, W, run_off.data_ptr(), runs.data_ptr(),
                                    rle_bounds.data_ptr(), rle_runs.data_ptr(), out.data_ptr(), stream),
           "tfb200_coco_masks_u8")
    return out
