"""MOTS results as COCO run-length encodings, and the MOTS20 result file.

A mask's RLE is the dictionary pycocotools ``mask.encode(np.asfortranarray(mask))`` returns, ``{"size": [H, W],
"counts": bytes}``: the run lengths of the mask read in column-major order, starting with a (possibly empty) run of
zeros, written as pycocotools' ``rleToString`` characters.  ``encode`` / ``decode`` restate that format in numpy, so
pycocotools is not needed; ``label_map_rle`` makes the RLEs of every track of a tracker label map at once
(``label_maps_rle`` of several maps), on the GPU (csrc/mask_rle.cu) for CUDA maps, so only the strings leave the
device; ``write_results`` writes the file ``MOTS20Sequence.write_results`` (datasets/tracking/mots20_sequence.py:72-91) writes, from bool masks or from RLEs.
"""
import csv
import os

import numpy as np
import torch

__all__ = ["encode", "decode", "decode_counts", "label_map_rle", "label_maps_rle", "write_results"]

_MAX_CHARS = 13                 # characters of any int64 count difference


def _counts(flat_f: np.ndarray) -> np.ndarray:
    """run lengths of a column-major flattened bool mask, zero run first"""
    n = flat_f.size
    b = np.flatnonzero(np.diff(flat_f.view(np.int8), prepend=np.int8(0)))
    return np.diff(np.concatenate(([0], b, [n]))).astype(np.int64)


def _string(cnts: np.ndarray) -> bytes:
    """pycocotools rleToString"""
    x = cnts.copy()
    x[3:] -= cnts[1:-2]
    out = np.empty((len(x), _MAX_CHARS), np.uint8)
    emit = np.empty((len(x), _MAX_CHARS), bool)
    alive = np.ones(len(x), bool)
    for k in range(_MAX_CHARS):
        c = x & 0x1F
        x = x >> 5
        more = np.where(c & 0x10, x != -1, x != 0)
        emit[:, k] = alive
        out[:, k] = (c | np.where(more, 0x20, 0)) + 48
        alive &= more
        if not alive.any():
            break
    return out[:, :k + 1][emit[:, :k + 1]].tobytes()


def encode(mask) -> dict:
    """COCO RLE of a 2-D bool / 0-1 mask [H, W]: what pycocotools ``mask.encode(np.asfortranarray(mask))`` returns."""
    m = np.asarray(mask)
    if m.ndim != 2:
        raise ValueError(f"encode: a 2-D mask is required, got shape {m.shape}")
    flat = np.ascontiguousarray(m.T).reshape(-1) != 0
    return {"size": [int(m.shape[0]), int(m.shape[1])], "counts": _string(_counts(flat))}


def decode(rle: dict) -> np.ndarray:
    """bool mask [H, W] of a COCO RLE (``encode``'s inverse; pycocotools ``rleFrString`` + ``decode``)."""
    h, w = (int(v) for v in rle["size"])
    cnts = decode_counts(rle["counts"])
    if (cnts < 0).any() or cnts.sum() != h * w:
        raise ValueError(f"decode: the runs do not cover a {h}x{w} mask")
    vals = (np.arange(len(cnts)) % 2).astype(bool)
    return np.repeat(vals, cnts).reshape(w, h).T.copy()


def decode_counts(s) -> np.ndarray:
    """int64 run lengths of a compressed RLE counts string (pycocotools ``rleFrString``), zero run first."""
    c = np.frombuffer(s.encode() if isinstance(s, str) else bytes(s), np.uint8).astype(np.int64) - 48
    if c.size == 0 or c[-1] & 0x20:
        raise ValueError("decode: truncated counts string")
    last = (c & 0x20) == 0                               # the last character of each value
    starts = np.concatenate(([0], np.flatnonzero(last)[:-1] + 1))
    k = np.arange(c.size) - np.repeat(starts, np.diff(np.concatenate((starts, [c.size]))))
    x = np.add.reduceat((c & 0x1F) << (5 * k), starts)
    ends = np.flatnonzero(last)
    x = np.where(c[ends] & 0x10, x | (-1 << (5 * (k[ends] + 1))), x)
    cnts = x.copy()
    for first in (3, 4):                                 # cnts[i] = x[i] + cnts[i - 2] for i > 2
        if len(x) > first:
            cnts[first::2] = cnts[first - 2] + np.cumsum(x[first::2])
    return cnts


def label_map_rle(label, ids) -> list:
    """RLEs of the masks ``label == ids[t]`` of a label map [H, W], in ``ids`` order (ids >= 0; other label values are
    background).  A CUDA int32 map is encoded by csrc/mask_rle.cu, and only the strings are copied to the host;
    anything else goes through ``encode``."""
    return label_maps_rle([label], [ids])[0]


def label_maps_rle(labels, ids_per_map) -> list:
    """``label_map_rle`` of several label maps at once (e.g. one per sequence of a multi-sequence step; sizes may
    differ): returns one list of RLEs per map.  When every map is a CUDA int32 tensor on one device, all of them are
    encoded by ONE call of csrc/mask_rle.cu's batched entry (up to 16 maps per call) with two device-to-host copies,
    the string offsets and the strings; otherwise each map goes through ``encode``."""
    labels, ids_per_map = list(labels), [np.asarray(i, dtype=np.int64).reshape(-1) for i in ids_per_map]
    if len(labels) != len(ids_per_map):
        raise ValueError("label_maps_rle: one ids list per label map")
    if any(len(i) and int(i.min()) < 0 for i in ids_per_map):
        raise ValueError("label_map_rle: ids must be >= 0")
    if not labels:
        return []
    first = labels[0]
    if all(torch.is_tensor(lab) and lab.is_cuda and lab.dtype == torch.int32 and lab.device == first.device
           for lab in labels):
        from . import ext
        packed = torch.from_numpy(np.concatenate(ids_per_map).astype(np.int32)).to(first.device, non_blocking=True)
        views, o = [], 0
        for i in ids_per_map:
            views.append(packed[o:o + len(i)])
            o += len(i)
        out = []
        for c in range(0, len(labels), 16):
            strings = ext.load().mask_rle_batched(labels[c:c + 16], views[c:c + 16])
            out += [[{"size": [int(v) for v in lab.shape], "counts": s} for s in per]
                    for lab, per in zip(labels[c:c + 16], strings)]
        return out
    return [_label_map_rle_host(lab, ids) for lab, ids in zip(labels, ids_per_map)]


def _label_map_rle_host(label, ids) -> list:
    lab = label.cpu().numpy() if torch.is_tensor(label) else np.asarray(label)
    ids = [int(i) for i in ids]
    if lab.ndim != 2:
        raise ValueError(f"label_map_rle: a 2-D label map is required, got shape {lab.shape}")
    flat = np.ascontiguousarray(lab.T).reshape(-1)
    size = [int(lab.shape[0]), int(lab.shape[1])]
    return [{"size": size, "counts": _string(_counts(flat == i))} for i in ids]


def write_results(results: dict, output_dir: str, seq_name: str) -> str:
    """``<output_dir>/<seq_name>.txt`` as ``MOTS20Sequence.write_results`` writes it: one space-separated csv row
    ``frame + 1, id + 1, 2, H, W, counts`` per result, in the dictionaries' order.  A result's "mask" is a bool array
    (encoded here) or an RLE dict (written as it is).  Returns the file's path."""
    os.makedirs(output_dir, exist_ok=True)
    path = os.path.join(output_dir, f"{seq_name}.txt")
    with open(path, "w", newline="") as f:
        writer = csv.writer(f, delimiter=" ")
        for i, track in results.items():
            for frame, data in track.items():
                rle = data["mask"] if isinstance(data["mask"], dict) else encode(data["mask"])
                counts = rle["counts"]
                writer.writerow([frame + 1, i + 1, 2, int(rle["size"][0]), int(rle["size"][1]),
                                 counts.decode("UTF-8") if isinstance(counts, bytes) else counts])
    return path
