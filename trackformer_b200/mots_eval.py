"""MOTS metrics on the GPU -- sMOTSA, MOTSA, MOTSP (Voigtlaender et al., CVPR 2019) with the CLEAR-MOT and identity
counts of `mot_eval` -- from the masks' COCO RLE strings, for many sequences in one pass.

`get_mots_accum(results, gt, num_frames)` packs one sequence into a picklable `MotsAccumulator` of numpy arrays (so
accumulators can be all-gathered across ranks as engine.py does with `MotAccumulator`): per-frame mask offsets, dense
ids, sizes, string offsets and one byte buffer of every counts string.  It decodes nothing.
`evaluate_mots_accums(accums, names)` uploads every sequence in one copy, runs csrc/mots_eval.cu (the strings decoded
into foreground intervals on the device, each frame side sorted by interval start, exact integer intersections,
the ignore rule, then mot_eval_core.h's frame-by-frame and identity matching), reads the per-sequence counters back
once, and returns `(summary, str_summary)` as `mot_eval.evaluate_mot_accums` does.

The definition:
- GT rows of class 2 are objects, class 10 rows are ignore regions, other classes are dropped.  Result rows of class 2
  (or without a class, as the tracker returns them) are hypotheses, others are dropped.  Frames at or beyond
  `num_frames` are ignored.
- A (GT, hypothesis) pair is a candidate iff inter > 0 and 2 inter >= union (pixel counts), with d = 1 - inter / union
  in fp64.  A hypothesis with no candidate whose pixels lie more than half in the union of the frame's ignore regions
  is removed before anything is counted: it is neither a false positive nor a prediction.
- Matching, switches, MT / PT / ML, FM and IDTP are `mot_eval`'s (motmetrics 1.2.0's rules) on those pairs; objects
  of a frame in the file's row order (a GT path) or the dict's id order (a GT dict), hypotheses in the order
  `results` lists its tracks.
- TP = matches + switches, TP~ = TP - sum of d; MOTSA = (TP - FP - IDS) / GT detections, sMOTSA = (TP~ - FP - IDS) / GT
  detections, MOTSP = TP~ / TP.  OVERALL sums the counts and recomputes the ratios.
- Masks of one side of a frame must not overlap (GT and ignore regions together; hypotheses); each mask must have
  the sequence's size and a well-formed string whose runs cover it.  Any of these raises `ValueError` naming the
  sequence and its first offending frame (0-based); a duplicate (frame, id) in a file raises in `mots.read_rows`.

Masks on one side do not overlap, so apart from exact IoU = 0.5 ties the counts that define sMOTSA, MOTSA, MOTSP and
IDF1 do not depend on the matcher.  MT / PT / ML and FM follow motmetrics' boundary conventions; parity with the
official MOTS20 evaluation tool is not claimed and not tested.  CUDA only: there is no host fallback.
"""
from __future__ import annotations

import ctypes
import os
from dataclasses import dataclass

import numpy as np
import torch

from . import mots
from .mot_eval import _CROWS, _CCOLS, _FP, _FRAG, _ICOLS, _IDTP, _IROWS, _MATCH, _MISS, _ML, _MT, _PT, _STATUS, \
    _SUMD, _SWITCH, MAX_CLEAR_COMPONENT, MAX_ID_COMPONENT
from .mot_eval import _ERRORS as _MOT_ERRORS

__all__ = ["MotsAccumulator", "get_mots_accum", "evaluate_mots_accums", "evaluate_counters", "summarize",
           "MAX_PIXELS"]

MAX_PIXELS = 1 << 28            # H x W of a sequence's masks (csrc/mots_eval_core.h)
GT_CLASS, IGNORE_CLASS = 2, 10

COLUMNS = ["smotsa", "motsa", "motsp", "idf1", "idp", "idr", "recall", "precision", "num_unique_objects",
           "mostly_tracked", "partially_tracked", "mostly_lost", "num_detections", "num_false_positives",
           "num_misses", "num_switches", "num_fragmentations", "num_ignored"]
NAMEMAP = {"smotsa": "sMOTSA", "motsa": "MOTSA", "motsp": "MOTSP", "idf1": "IDF1", "idp": "IDP", "idr": "IDR",
           "recall": "Rcll", "precision": "Prcn", "num_unique_objects": "GT", "mostly_tracked": "MT",
           "partially_tracked": "PT", "mostly_lost": "ML", "num_detections": "TP", "num_false_positives": "FP",
           "num_misses": "FN", "num_switches": "IDs", "num_fragmentations": "FM", "num_ignored": "Ign"}
_RATIOS = ("smotsa", "motsa", "motsp", "idf1", "idp", "idr", "recall", "precision")

# slots after mot_eval's 16 per sequence (include/tfb200_fused.h, tfb200_mots_eval)
_XSLOTS = 11
_XSTATUS, _XGTDETS, _XKEPT, _XREMOVED, _XINTERVALS, _XINTERSECTING, _XFIRST = range(7)
_XERRORS = {1: "GT masks (or ignore regions) overlap", 2: "result masks overlap",
            4: "a mask's size differs from the sequence's", 8: "a malformed RLE string or runs that do not cover H x W",
            16: "more intervals than the interval capacity"}


@dataclass
class MotsAccumulator:
    """One sequence, packed.  Frame f holds mask rows frame_mask[3f] .. (GT objects), frame_mask[3f + 1] .. (ignore
    regions), frame_mask[3f + 2] .. frame_mask[3f + 3] (hypotheses); mask k's counts string is
    chars[str_off[k]:str_off[k + 1]]."""
    frame_mask: np.ndarray       # int64 [3 F + 1]
    mask_id: np.ndarray          # int32 [n]: index into gt_ids (objects), track_ids (hypotheses), 0 (ignore)
    mask_size: np.ndarray        # int32 [n, 2] H, W
    str_off: np.ndarray          # int64 [n + 1]
    chars: np.ndarray            # uint8 [str_off[-1]]
    size: tuple                  # the sequence's H, W
    gt_ids: np.ndarray           # the GT ids, as given
    track_ids: np.ndarray        # the track ids, as given

    @property
    def num_frames(self):
        return (len(self.frame_mask) - 1) // 3

    def side_counts(self):
        """[F, 3] masks per frame: objects, ignore regions, hypotheses"""
        return np.diff(self.frame_mask).reshape(-1, 3)


def _rle(mask):
    """(H, W, counts bytes) of an RLE dict or a bool array (encoded with mots.encode: a numpy pass over the pixels)"""
    if not isinstance(mask, dict):
        mask = mots.encode(mask.cpu().numpy() if torch.is_tensor(mask) else mask)
    c = mask["counts"]
    return int(mask["size"][0]), int(mask["size"][1]), c.encode() if isinstance(c, str) else bytes(c)


def get_mots_accum(results, gt, num_frames):
    """`results` {track_id: {frame: {"mask": RLE dict or bool [H, W], "class_id" (optional)}}} (0-based frames),
    `gt` the `mots.load_results` form of a GT file or the file's path, `num_frames` the sequence length.  Packs the
    strings as they are; bool masks are encoded here with `mots.encode` (a host pass over every pixel: pass
    `Tracker(..., mask_rle=True)` results to avoid it).

    The order of a frame's objects decides motmetrics' tie-breaking where two pairs have exactly equal d (IoU = 0.5
    ties): with a path they are in the file's row order; with a dict, in the dict's id order (for `load_results`, the
    order in which ids first appear in the file), which can differ from the file's order within a frame.  Hypotheses
    are in the order `results` lists its tracks."""
    F = int(num_frames)
    if isinstance(gt, (str, os.PathLike)):
        gt_rows = [(f - 1, i - 1, c, rle) for f, i, c, rle in mots.read_rows(os.fspath(gt))]
    else:
        gt_rows = [(int(f), i, d.get("class_id", GT_CLASS), d["mask"]) for i, tr in gt.items() for f, d in tr.items()]
    gt_rows = [r for r in gt_rows if 0 <= r[0] < F and r[2] in (GT_CLASS, IGNORE_CLASS)]
    gt_ids = np.unique(np.asarray([r[1] for r in gt_rows if r[2] == GT_CLASS], dtype=np.int64))
    track_ids = list(results.keys())
    hyp_rows = [(int(f), t, d["mask"]) for t, tr in enumerate(results.values()) for f, d in tr.items()
                if 0 <= int(f) < F and d.get("class_id", GT_CLASS) == GT_CLASS]
    # rows: (frame, side, order) -> stable sort keeps the source order within a frame side
    rows = [(f, 0 if c == GT_CLASS else 1, int(np.searchsorted(gt_ids, i)) if c == GT_CLASS else 0, m)
            for f, i, c, m in gt_rows]
    rows += [(f, 2, t, m) for f, t, m in hyp_rows]
    order = sorted(range(len(rows)), key=lambda k: (rows[k][0], rows[k][1]))
    enc = [_rle(rows[k][3]) for k in order]
    frame_side = np.zeros(3 * F, dtype=np.int64)
    if rows:
        np.add.at(frame_side, [3 * rows[k][0] + rows[k][1] for k in order], 1)
    strings = [e[2] for e in enc]
    str_off = np.zeros(len(strings) + 1, dtype=np.int64)
    str_off[1:] = np.cumsum([len(s) for s in strings])
    sizes = np.asarray([e[:2] for e in enc], dtype=np.int64).reshape(-1, 2)
    first_gt = [e[:2] for k, e in zip(order, enc) if rows[k][1] != 2]
    size = tuple(first_gt[0]) if first_gt else tuple(sizes[0]) if len(sizes) else (0, 0)
    if size[0] * size[1] >= MAX_PIXELS or (sizes >= 2 ** 31).any():
        raise ValueError(f"get_mots_accum: masks of {size[0]} x {size[1]} pixels: H x W must be < 2^28")
    return MotsAccumulator(
        frame_mask=np.concatenate(([0], np.cumsum(frame_side))).astype(np.int64),
        mask_id=np.asarray([rows[k][2] for k in order], dtype=np.int32),
        mask_size=sizes.astype(np.int32), str_off=str_off,
        chars=np.frombuffer(b"".join(strings), dtype=np.uint8).copy(), size=(int(size[0]), int(size[1])),
        gt_ids=gt_ids, track_ids=np.asarray(track_ids))


_lib = None


def _library():
    global _lib
    if _lib is None:
        from . import ext
        ext.load()                                   # raises with the build command when the native code is missing
        _lib = ctypes.CDLL(ext.library_path())
        vp, i32, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
        _lib.tfb200_mots_eval_workspace_bytes.argtypes = [i32, i32, i32, i64, i64, i64, i32, i32, i64, i64, i64]
        _lib.tfb200_mots_eval_workspace_bytes.restype = ctypes.c_size_t
        _lib.tfb200_mots_eval.argtypes = ([vp] * 9 + [i32, i32, i32, i64, i64, i64, i32, i32, i64, i64, i64, vp,
                                                      ctypes.c_size_t, vp, vp])
        _lib.tfb200_mots_eval.restype = ctypes.c_int
    return _lib


def _pack(accums):
    """Every sequence in one byte buffer (arrays 256-byte aligned, the strings last) + the sizes of the C entry."""
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
    n_mask = np.cumsum([0] + [len(a.mask_id) for a in accums])
    n_chr = np.cumsum([0] + [len(a.chars) for a in accums])
    frame_mask = np.concatenate([[0]] + [a.frame_mask[1:] + n_mask[s] for s, a in enumerate(accums)])
    sides = np.concatenate([a.side_counts() for a in accums]).reshape(-1, 3)
    no, nh = sides[:, 0], sides[:, 2]
    frame_cell = np.concatenate(([0], np.cumsum((no + 1) * nh)))
    frame_obj = np.concatenate(([0], np.cumsum(no)))
    frames = np.repeat(np.arange(sum(F)), sides.sum(1))
    gt_rows = np.concatenate([np.arange(b, b + n) for b, n in zip(frame_mask[0:-1:3], no)]) if len(no) else []
    mask_id = np.concatenate([a.mask_id for a in accums]).astype(np.int32)
    mask = np.stack([frames, mask_id, *np.concatenate([a.mask_size for a in accums]).reshape(-1, 2).T], 1) \
        if len(mask_id) else np.zeros((0, 4))
    str_off = np.concatenate([[0]] + [a.str_off[1:] + n_chr[s] for s, a in enumerate(accums)])
    lens = np.diff(str_off)
    arrays = [seq, np.asarray([a.size for a in accums], np.int32), frame_mask.astype(np.int32), frame_cell,
              frame_obj.astype(np.int32), mask_id[np.asarray(gt_rows, dtype=np.int64)], mask.astype(np.int32),
              str_off.astype(np.int64), np.concatenate([a.chars for a in accums])]
    offsets, at = [], 0
    for x in arrays:
        offsets.append(at)
        at += -(-max(x.nbytes, 1) // 256) * 256
    buf = np.zeros(at, dtype=np.uint8)
    for x, o in zip(arrays, offsets):
        buf[o:o + x.nbytes] = x.reshape(-1).view(np.uint8)
    n_obj = int(no.sum())
    products = int((no * nh).sum())
    sizes = dict(S=S, F=int(sum(F)), n_masks=int(n_mask[-1]), n_gt=int(sum(G)), n_trk=int(sum(H)),
                 tp_cells=int(cells.sum()), max_obj=int(no.max(initial=0)), max_hyp=int(nh.max(initial=0)),
                 pair_cap=min(products, 2 * n_obj), interval_cap=int((lens // 2).sum()),
                 cells=int(frame_cell[-1]))
    if sizes["n_masks"] >= 2 ** 31 or sizes["interval_cap"] >= 2 ** 31 or sizes["F"] >= 2 ** 29:
        raise ValueError(f"mots_eval: more than 2^31 masks or string characters / 2 in one call: {sizes}")
    return buf, offsets, sizes


def _entry_args(z):
    return (z["S"], z["F"], z["n_masks"], z["n_gt"], z["n_trk"], z["tp_cells"], z["max_obj"], z["max_hyp"],
            z["pair_cap"], z["interval_cap"], z["cells"])


def evaluate_counters(accums, device=None, names=None):
    """The kernel's per-sequence counters: int64 [S, 16 + 11] (include/tfb200_fused.h, tfb200_mots_eval's out) plus
    the packed sizes.  Raises `ValueError` for invalid masks, `RuntimeError` when a sequence exceeds a stated limit."""
    if not torch.cuda.is_available():
        raise RuntimeError("mots_eval needs a CUDA device: the evaluation runs on the GPU and has no host fallback")
    if not accums:
        raise ValueError("mots_eval: no accumulators")
    device = torch.device(device if device is not None else "cuda")
    buf, offsets, z = _pack(accums)
    lib = _library()
    with torch.cuda.device(device):
        buf_dev = torch.from_numpy(buf).to(device)              # the one upload
        stream = torch.cuda.current_stream(device).cuda_stream
        ws_bytes = lib.tfb200_mots_eval_workspace_bytes(*_entry_args(z))
        if ws_bytes == 0:
            raise ValueError(f"mots_eval: sizes out of range: {z}")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        out = torch.empty(z["S"] * (16 + _XSLOTS), dtype=torch.int64, device=device)
        rc = lib.tfb200_mots_eval(*[buf_dev.data_ptr() + o for o in offsets], *_entry_args(z), ws.data_ptr(),
                                  ws_bytes, out.data_ptr(), stream)
        if rc != 0:
            raise RuntimeError(f"tfb200_mots_eval failed (code {rc})")
        out = out.cpu().numpy()                                 # the one read-back (synchronises)
    return check_counters(out, z, names), z


def check_counters(flat, z, names=None):
    """[S, 16 + 11] counters from the entry's flat out; raises for a set status bit."""
    S = z["S"]
    out = np.concatenate([flat[:S * 16].reshape(S, 16), flat[S * 16:].reshape(S, _XSLOTS)], 1)
    names = list(names) if names is not None else [str(s) for s in range(S)]
    x = out[:, 16:]
    for b, what in enumerate(_XERRORS.values()):
        bad = np.nonzero(x[:, _XSTATUS] & (1 << b))[0]
        if len(bad):
            s = int(bad[0])
            raise ValueError(f"mots_eval: sequence {names[s]}: frame {int(x[s, _XFIRST + b])}: {what}"
                             if b < 4 else f"mots_eval: {what}")
    for bit, what in _MOT_ERRORS.items():
        bad = np.nonzero(out[:, _STATUS] & bit)[0]
        if len(bad):
            raise RuntimeError(f"mots_eval: {what} (sequences {[names[s] for s in bad]}; largest residual component "
                               f"{out[:, _CROWS].max()} x {out[:, _CCOLS].max()}, largest identity component "
                               f"{out[:, _IROWS].max()} x {out[:, _ICOLS].max()})")
    if (out[:, _STATUS] & 1).any():                             # cannot happen for masks that pass the checks above
        raise RuntimeError("mots_eval: more valid pairs than two per GT mask")
    return out


def _metrics(c):
    with np.errstate(divide="ignore", invalid="ignore"):
        gt_dets, n_pred = np.float64(c["gt_dets"]), np.float64(c["kept"])
        tp = np.float64(c["matches"] + c["switches"])
        tp_soft = tp - c["sum_d"]
        idtp = np.float64(c["idtp"])
        return {"smotsa": (tp_soft - c["fp"] - c["switches"]) / gt_dets,
                "motsa": (tp - c["fp"] - c["switches"]) / gt_dets, "motsp": tp_soft / tp,
                "idf1": 2 * idtp / (gt_dets + n_pred), "idp": idtp / n_pred, "idr": idtp / gt_dets,
                "recall": tp / gt_dets, "precision": tp / (tp + c["fp"]),
                "num_unique_objects": c["gt"], "mostly_tracked": c["mt"], "partially_tracked": c["pt"],
                "mostly_lost": c["ml"], "num_detections": c["matches"] + c["switches"],
                "num_false_positives": c["fp"], "num_misses": c["misses"], "num_switches": c["switches"],
                "num_fragmentations": c["fm"], "num_ignored": c["removed"]}


def evaluate_mots_accums(accums, names, generate_overall=True):
    """(summary, str_summary) as `mot_eval.evaluate_mot_accums` returns them: `summary[metric][name]` for the MOTS
    metric names of COLUMNS, with an OVERALL row (counts summed over sequences, ratios recomputed from the sums) when
    `generate_overall`."""
    names = list(names)
    if len(names) != len(accums):
        raise ValueError("mots_eval: one name per accumulator")
    return summarize(accums, names, evaluate_counters(list(accums), names=names)[0], generate_overall)


def summarize(accums, names, out, generate_overall=True):
    """`evaluate_mots_accums`' result from the counters `out` [S, 16 + 11]."""
    import pandas as pd

    names = list(names)
    rows = []
    for a, o in zip(accums, out):
        x = o[16:]
        rows.append({"gt_dets": int(x[_XGTDETS]), "kept": int(x[_XKEPT]), "removed": int(x[_XREMOVED]),
                     "matches": int(o[_MATCH]), "switches": int(o[_SWITCH]), "misses": int(o[_MISS]),
                     "fp": int(o[_FP]), "fm": int(o[_FRAG]), "mt": int(o[_MT]), "pt": int(o[_PT]), "ml": int(o[_ML]),
                     "gt": len(a.gt_ids), "idtp": int(o[_IDTP]),
                     "sum_d": float(o[_SUMD:_SUMD + 1].view(np.float64)[0])})
    index = names
    if generate_overall:
        rows.append({k: sum(r[k] for r in rows) for k in rows[0]})
        index = names + ["OVERALL"]
    summary = pd.DataFrame([_metrics(r) for r in rows], index=index, columns=COLUMNS)
    for col in COLUMNS:
        summary[col] = summary[col].astype(np.float64 if col in _RATIOS else np.int64)
    formatters = {NAMEMAP[c]: ("{:.1%}".format if c in _RATIOS and c != "motsp" else "{:.3f}".format
                               if c == "motsp" else "{:d}".format) for c in COLUMNS}
    str_summary = summary.rename(columns=NAMEMAP).to_string(formatters=formatters)
    return summary, str_summary
