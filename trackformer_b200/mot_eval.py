"""MOTChallenge CLEAR-MOT and identity metrics on the GPU, in place of the reference's motmetrics-based
`get_mot_accum` / `evaluate_mot_accums` (src/trackformer/util/track_utils.py:354-417), for many sequences at once.

`get_mot_accum(results, seq_loader)` packs one sequence into a picklable `MotAccumulator` of numpy arrays (so
accumulators can be all-gathered across ranks as engine.py does): per-frame offsets into object and hypothesis rows,
dense GT / track ids, float32 x, y, w, h boxes.  `evaluate_mot_accums(accums, names)` uploads every sequence in one
copy, runs csrc/mot_eval.cu (valid pairs of every frame, the frame-by-frame matching of motmetrics'
`MOTAccumulator.update` with one CTA per sequence, and the identity matching), reads the per-sequence counters back
once, and returns motmetrics' `(summary, str_summary)`: a DataFrame with motmetrics' metric names per sequence plus
OVERALL, and its rendering with the MOTChallenge column names.

The metrics are those of motmetrics 1.2.0 as the reference calls it (`MOTAccumulator(auto_id=True)`, IoU distances
with max_iou=0.5, `motchallenge_metrics`), without the extended TRANSFER / ASCEND / MIGRATE counts.  Where a frame's
optimal assignment is not unique (equal sums of distances), the kernel's choice may differ from motmetrics' `lap`
solver.  CUDA only: there is no host fallback.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass

import numpy as np
import torch

__all__ = ["MotAccumulator", "get_mot_accum", "evaluate_mot_accums", "evaluate_counters", "summarize",
           "MAX_CLEAR_COMPONENT", "MAX_ID_COMPONENT"]

MAX_CLEAR_COMPONENT = 64     # objects / hypotheses of one residual component of a frame (csrc/mot_eval_core.h)
MAX_ID_COMPONENT = (8192, 65536)   # smaller, larger side (GT ids or track ids) of one identity component

COLUMNS = ["idf1", "idp", "idr", "recall", "precision", "num_unique_objects", "mostly_tracked", "partially_tracked",
           "mostly_lost", "num_false_positives", "num_misses", "num_switches", "num_fragmentations", "mota", "motp"]
NAMEMAP = {"idf1": "IDF1", "idp": "IDP", "idr": "IDR", "recall": "Rcll", "precision": "Prcn",
           "num_unique_objects": "GT", "mostly_tracked": "MT", "partially_tracked": "PT", "mostly_lost": "ML",
           "num_false_positives": "FP", "num_misses": "FN", "num_switches": "IDs", "num_fragmentations": "FM",
           "mota": "MOTA", "motp": "MOTP"}
_RATIOS = ("idf1", "idp", "idr", "recall", "precision", "mota")

# out slots of tfb200_mot_eval_f32 (include/tfb200_fused.h)
(_STATUS, _PAIRS, _MATCH, _SWITCH, _MISS, _FP, _FRAG, _MT, _PT, _ML, _IDTP, _CROWS, _CCOLS, _IROWS, _ICOLS,
 _SUMD) = range(16)
_ERRORS = {2: "a frame has more objects or hypotheses than the sizes given",
           4: f"a frame's residual assignment has a component over {MAX_CLEAR_COMPONENT} objects or hypotheses",
           8: f"the identity matching has a component over {MAX_ID_COMPONENT[0]} x {MAX_ID_COMPONENT[1]} ids"}


@dataclass
class MotAccumulator:
    """One sequence, packed.  Frame f holds object rows frame_obj[f]:frame_obj[f + 1] and hypothesis rows
    frame_hyp[f]:frame_hyp[f + 1], in the order motmetrics sees them (the frame's `gt` dict order; the order in which
    `results` lists its tracks)."""
    frame_obj: np.ndarray        # int64 [F + 1]
    obj_id: np.ndarray           # int32 [n_obj], index into gt_ids
    obj_box: np.ndarray          # float32 [n_obj, 4] x, y, w, h
    frame_hyp: np.ndarray        # int64 [F + 1]
    hyp_id: np.ndarray           # int32 [n_hyp], index into track_ids
    hyp_box: np.ndarray          # float32 [n_hyp, 4]
    gt_ids: np.ndarray           # the GT ids, as given
    track_ids: np.ndarray        # the track ids, as given

    @property
    def num_frames(self):
        return len(self.frame_obj) - 1


def _xywh(b):
    b = np.asarray(b, dtype=np.float32).reshape(-1, 4)
    return np.stack((b[:, 0], b[:, 1], b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]), axis=1)   # float32 w, h


def get_mot_accum(results, seq_loader):
    """The reference's signature: `results` {track_id: {frame: {"bbox": x1, y1, x2, y2, ...}}}, `seq_loader` yields
    frames whose "gt" is {gt_id: x1, y1, x2, y2} (an array, or a [1, 4] tensor as the DataLoader collates it).  Result
    frames beyond the loader's length are ignored."""
    n_obj, gt_keys, gt_boxes = [], [], []
    for frame_data in seq_loader:
        gt = frame_data["gt"] or {}
        n_obj.append(len(gt))
        gt_keys.extend(int(k) for k in gt.keys())
        gt_boxes.extend(np.asarray(b, dtype=np.float32).reshape(-1)[:4] for b in gt.values())
    F = len(n_obj)
    gt_ids, obj_id = np.unique(np.asarray(gt_keys, dtype=np.int64), return_inverse=True)
    frames, tracks, boxes = [], [], []
    for t, track in enumerate(results.values()):
        for f, data in track.items():
            if 0 <= int(f) < F:
                frames.append(int(f))
                tracks.append(t)
                boxes.append(np.asarray(data["bbox"], dtype=np.float32).reshape(-1)[:4])
    frames, tracks = np.asarray(frames, dtype=np.int64), np.asarray(tracks, dtype=np.int64)
    order = np.lexsort((tracks, frames))
    frame_hyp = np.zeros(F + 1, dtype=np.int64)
    frame_hyp[1:] = np.cumsum(np.bincount(frames, minlength=F))
    frame_obj = np.zeros(F + 1, dtype=np.int64)
    frame_obj[1:] = np.cumsum(n_obj)
    return MotAccumulator(
        frame_obj=frame_obj, obj_id=obj_id.astype(np.int32).reshape(-1),
        obj_box=_xywh(np.stack(gt_boxes) if gt_boxes else np.zeros((0, 4), np.float32)),
        frame_hyp=frame_hyp, hyp_id=tracks[order].astype(np.int32),
        hyp_box=_xywh(np.stack(boxes)[order] if boxes else np.zeros((0, 4), np.float32)),
        gt_ids=gt_ids, track_ids=np.asarray(list(results.keys())))


_lib = None


def _library():
    global _lib
    if _lib is None:
        from . import ext
        ext.load()                                   # raises with the build command when the native code is missing
        _lib = ctypes.CDLL(ext.library_path())
        vp, i32, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
        _lib.tfb200_mot_eval_workspace_bytes.argtypes = [i32, i32, i64, i64, i64, i32, i32, i64]
        _lib.tfb200_mot_eval_workspace_bytes.restype = ctypes.c_size_t
        _lib.tfb200_mot_eval_f32.argtypes = ([vp] * 7 + [i32, i32, i64, i64, i64, i32, i32, i64, vp, ctypes.c_size_t,
                                                         vp, vp])
        _lib.tfb200_mot_eval_f32.restype = ctypes.c_int
    return _lib


def _pack(accums):
    """Every sequence in one byte buffer (arrays 256-byte aligned) + the sizes of the C entry."""
    S = len(accums)
    F = [a.num_frames for a in accums]
    G = [len(a.gt_ids) for a in accums]
    H = [len(a.track_ids) for a in accums]
    seq = np.zeros((S, 8), dtype=np.int64)
    seq[:, 1] = np.cumsum(F)
    seq[1:, 0] = seq[:-1, 1]
    seq[1:, 2] = np.cumsum(G)[:-1]
    seq[:, 3] = G
    seq[1:, 4] = np.cumsum(H)[:-1]
    seq[:, 5] = H
    cells = np.asarray(G, dtype=np.int64) * np.asarray(H, dtype=np.int64)
    seq[1:, 6] = np.cumsum(cells)[:-1]
    n_obj = np.cumsum([0] + [len(a.obj_id) for a in accums])
    n_hyp = np.cumsum([0] + [len(a.hyp_id) for a in accums])
    frame_obj = np.concatenate([[0]] + [a.frame_obj[1:] + n_obj[s] for s, a in enumerate(accums)])
    frame_hyp = np.concatenate([[0]] + [a.frame_hyp[1:] + n_hyp[s] for s, a in enumerate(accums)])
    co, ch = np.diff(frame_obj), np.diff(frame_hyp)
    arrays = [seq, frame_obj.astype(np.int32), frame_hyp.astype(np.int32),
              np.concatenate([a.obj_id for a in accums]).astype(np.int32),
              np.concatenate([a.obj_box for a in accums]).astype(np.float32),
              np.concatenate([a.hyp_id for a in accums]).astype(np.int32),
              np.concatenate([a.hyp_box for a in accums]).astype(np.float32)]
    offsets, at = [], 0
    for x in arrays:
        offsets.append(at)
        at += -(-max(x.nbytes, 1) // 256) * 256
    buf = np.zeros(at, dtype=np.uint8)
    for x, o in zip(arrays, offsets):
        buf[o:o + x.nbytes] = x.reshape(-1).view(np.uint8)
    sizes = dict(S=S, F=int(sum(F)), n_gt=int(sum(G)), n_trk=int(sum(H)), tp_cells=int(cells.sum()),
                 max_obj=int(co.max(initial=0)), max_hyp=int(ch.max(initial=0)),
                 products=int((co * ch).sum()), n_obj=int(n_obj[-1]), n_hyp=int(n_hyp[-1]))
    return buf, offsets, sizes


def _run(buf_dev, offsets, z, pair_cap, stream):
    lib = _library()
    ws_bytes = lib.tfb200_mot_eval_workspace_bytes(z["S"], z["F"], z["n_gt"], z["n_trk"], z["tp_cells"],
                                                   z["max_obj"], z["max_hyp"], pair_cap)
    if ws_bytes == 0:
        raise ValueError(f"mot_eval: sizes out of range: {z}")
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=buf_dev.device)
    out = torch.empty(z["S"] * 16, dtype=torch.int64, device=buf_dev.device)
    ptrs = [buf_dev.data_ptr() + o for o in offsets]
    rc = lib.tfb200_mot_eval_f32(*ptrs, z["S"], z["F"], z["n_gt"], z["n_trk"], z["tp_cells"], z["max_obj"],
                                 z["max_hyp"], pair_cap, ws.data_ptr(), ws_bytes, out.data_ptr(), stream)
    if rc != 0:
        raise RuntimeError(f"tfb200_mot_eval_f32 failed (code {rc})")
    return out.view(z["S"], 16).cpu().numpy()                 # the one read-back (synchronises)


def evaluate_counters(accums, device=None):
    """The kernel's per-sequence counters: int64 [S, 16] (include/tfb200_fused.h, tfb200_mot_eval_f32's out) plus the
    packed sizes.  Raises when a sequence exceeds a stated limit."""
    if not torch.cuda.is_available():
        raise RuntimeError("mot_eval needs a CUDA device: the evaluation runs on the GPU and has no host fallback")
    if not accums:
        raise ValueError("mot_eval: no accumulators")
    device = torch.device(device if device is not None else "cuda")
    buf, offsets, z = _pack(accums)
    with torch.cuda.device(device):
        buf_dev = torch.from_numpy(buf).to(device)              # the one upload
        stream = torch.cuda.current_stream(device).cuda_stream
        pair_cap = min(z["products"], 2 * (z["n_obj"] + z["n_hyp"]))
        out = _run(buf_dev, offsets, z, pair_cap, stream)
        if (out[:, _STATUS] & 1).any():                         # more valid pairs than guessed: size them exactly
            out = _run(buf_dev, offsets, z, int(out[:, _PAIRS].sum()), stream)
    for bit, what in _ERRORS.items():
        bad = np.nonzero(out[:, _STATUS] & bit)[0]
        if len(bad):
            raise RuntimeError(f"mot_eval: {what} (sequences {bad.tolist()}; largest residual component "
                               f"{out[:, _CROWS].max()} x {out[:, _CCOLS].max()}, largest identity component "
                               f"{out[:, _IROWS].max()} x {out[:, _ICOLS].max()})")
    return out, z


def _metrics(c):
    with np.errstate(divide="ignore", invalid="ignore"):
        n_obj, n_pred = np.float64(c["num_objects"]), np.float64(c["num_predictions"])
        det = np.float64(c["matches"] + c["switches"])
        idtp = np.float64(c["idtp"])
        return {"idf1": 2 * idtp / (n_obj + n_pred), "idp": idtp / n_pred, "idr": idtp / n_obj,
                "recall": det / n_obj, "precision": det / (det + c["fp"]),
                "num_unique_objects": c["gt"], "mostly_tracked": c["mt"], "partially_tracked": c["pt"],
                "mostly_lost": c["ml"], "num_false_positives": c["fp"], "num_misses": c["misses"],
                "num_switches": c["switches"], "num_fragmentations": c["fm"],
                "mota": 1.0 - (c["misses"] + c["switches"] + c["fp"]) / n_obj, "motp": c["sum_d"] / det}


def evaluate_mot_accums(accums, names, generate_overall=True):
    """(summary, str_summary) as the reference's evaluate_mot_accums returns them: `summary[metric][name]` for
    motmetrics' motchallenge metric names, with an OVERALL row (counts summed over sequences, ratios recomputed from
    the sums) when `generate_overall`."""
    names = list(names)
    if len(names) != len(accums):
        raise ValueError("mot_eval: one name per accumulator")
    return summarize(accums, names, evaluate_counters(list(accums))[0], generate_overall)


def summarize(accums, names, out, generate_overall=True):
    """`evaluate_mot_accums`' result from the kernel's counters `out` [S, 16]."""
    import pandas as pd

    names = list(names)
    rows = []
    for a, o in zip(accums, out):
        rows.append({"num_objects": len(a.obj_id), "num_predictions": len(a.hyp_id), "matches": int(o[_MATCH]),
                     "switches": int(o[_SWITCH]), "misses": int(o[_MISS]), "fp": int(o[_FP]), "fm": int(o[_FRAG]),
                     "gt": len(a.gt_ids), "mt": int(o[_MT]), "pt": int(o[_PT]), "ml": int(o[_ML]),
                     "idtp": int(o[_IDTP]), "sum_d": float(o[_SUMD:_SUMD + 1].view(np.float64)[0])})
    index = names
    if generate_overall:
        rows.append({k: sum(r[k] for r in rows) for k in rows[0]})
        index = names + ["OVERALL"]
    summary = pd.DataFrame([_metrics(r) for r in rows], index=index, columns=COLUMNS)
    for col in COLUMNS:
        summary[col] = summary[col].astype(np.float64 if col in _RATIOS or col == "motp" else np.int64)
    formatters = {NAMEMAP[c]: ("{:.1%}".format if c in _RATIOS else "{:.3f}".format if c == "motp" else "{:d}".format)
                  for c in COLUMNS}
    str_summary = summary.rename(columns=NAMEMAP).to_string(formatters=formatters)
    return summary, str_summary
