"""DeviceTracker's decision routine on the CPU suite.

csrc/track_step_core.h is written once and compiled twice: by nvcc into the one-CTA kernel DeviceTracker launches, and
-- here -- by g++ with one "thread" (tests/host_build/track_step_host.cpp).  Substituting that build for the kernel
launch lets the reference-recorded sequences of tests/golden/tracker_*.npz (every branch of Tracker.step: births,
deaths, both NMS passes, both ReID modes, both public-detection modes, reid_sim_only) run through the device algorithm
without a GPU.  The CUDA build of the same source is compared with the same fixtures in tests/test_tracker_gpu.py.
The product class itself refuses CPU tensors (last test)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import host_twin
from test_tracker_cpu import check_against_gold
import tracker_fixtures as tf
from trackformer_b200.deformable_detr import DeformablePostProcess
from trackformer_b200.device_tracker import DeviceTracker, _ArgsC
from trackformer_b200.tracker import Tracker

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")


@pytest.fixture(scope="module")
def host_tracker(tmp_path_factory):
    lib = host_twin.build("track_step_host", tmp_path_factory.mktemp("track_step"))
    lib.tfb200_track_step_host.argtypes = [ctypes.POINTER(_ArgsC)]
    lib.tfb200_track_step_host.restype = ctypes.c_int

    class HostBuildTracker(DeviceTracker):
        def _launch(self, args, tensors):
            assert not any(t.is_cuda for t in tensors)
            assert lib.tfb200_track_step_host(ctypes.byref(args)) == 0
    return HostBuildTracker


def test_args_struct_matches_the_header():
    """sizeof(TfbTrackStepArgs) as the C compiler sees it == the ctypes mirror"""
    src = '#include <stdio.h>\n#include "include/tfb200_fused.h"\nint main(){printf("%zu", sizeof(TfbTrackStepArgs));}'
    exe = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"tfb200_sizeof_{os.getpid()}")
    subprocess.run(["gcc", "-x", "c", "-", "-I", os.path.dirname(HERE), "-o", exe], input=src.encode(), check=True,
                   cwd=os.path.dirname(HERE))
    try:
        assert int(subprocess.check_output([exe])) == ctypes.sizeof(_ArgsC)
    finally:
        os.remove(exe)


@pytest.mark.parametrize("case", list(tf.CASES))
def test_device_routine_matches_reference(host_tracker, case):
    out = tf.run_case(host_tracker, DeformablePostProcess(), case)
    check_against_gold(out, case)


@pytest.mark.parametrize("case", list(tf.CASES))
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_device_routine_equals_host_tracker_on_other_scenes(host_tracker, case, seed):
    """scenes the fixtures do not hold: the host tracker (itself pinned to the reference) is the yardstick"""
    a = tf.run_case(Tracker, DeformablePostProcess(), case, seed=seed)
    b = tf.run_case(host_tracker, DeformablePostProcess(), case, seed=seed)
    for key in a:
        if key == "rows":
            np.testing.assert_array_equal(a[key][:, :3], b[key][:, :3], err_msg=key)
            np.testing.assert_allclose(a[key][:, 3:], b[key][:, 3:], rtol=1e-6, atol=1e-4)
        else:
            np.testing.assert_array_equal(a[key], b[key], err_msg=f"{case}/{seed}: {key}")


@pytest.mark.parametrize("name,multi_frame", [("model_sequence", False), ("model_sequence_multi_frame", True)])
def test_device_routine_over_the_real_detector(host_tracker, name, multi_frame, monkeypatch):
    from oracle.torch_ref import msda_core_torch
    import trackformer_b200.msda_module as mm
    from test_model_parity_cpu import build

    class _OracleFn:
        @staticmethod
        def apply(value, shapes, loc, attn, step):
            return msda_core_torch(value, shapes, loc, attn)
    monkeypatch.setattr(mm, "MSDeformAttnFunction", _OracleFn)
    gold = np.load(os.path.join(GOLD, f"tracker_{name}.npz"))
    cfg = {k: float(v) for k, v in zip(gold["cfg_keys"], gold["cfg_values"])}
    cfg["prev_frame_dist"] = int(cfg["prev_frame_dist"])
    out = tf.run_model_sequence(build, host_tracker, DeformablePostProcess(), cfg, multi_frame=multi_frame)
    for key in ("num_reids", "track_num", "frame_index", "active_ids", "inactive_ids", "inactive_counts"):
        np.testing.assert_array_equal(out[key], gold[key], err_msg=key)
    assert out["rows"].shape == gold["rows"].shape
    np.testing.assert_array_equal(out["rows"][:, :3], gold["rows"][:, :3])
    np.testing.assert_allclose(out["rows"][:, 3:], gold["rows"][:, 3:], rtol=1e-3, atol=1e-3)


def test_many_tracks_grow_the_buffers(host_tracker):
    from test_tracker_cpu import test_many_tracks_grow_the_bank  # noqa: F401  (same scripted detector, 150 targets)

    class Many(torch.nn.Module):
        num_queries, overflow_boxes = 150, True

        def __init__(self):
            super().__init__()
            self.p = torch.nn.Parameter(torch.zeros(1))

        def forward(self, img, targets=None, prev_features=None):
            k = 0 if targets is None else len(targets[0]["track_query_boxes"])
            g = torch.Generator().manual_seed(3)
            centres = torch.rand(150, 2, generator=g) * 0.8 + 0.1
            boxes = torch.cat([centres, torch.full((150, 2), 0.01)], 1)
            logits = torch.full((k + 150, 4), -5.0)
            logits[:, 0] = 2.0
            embeds = torch.arange(k + 150, dtype=torch.float32)[:, None].expand(-1, 8).contiguous()
            if k:
                boxes = torch.cat([targets[0]["track_query_boxes"], boxes], 0)
                logits[k:, 0] = -2.0
                embeds[:k] = targets[0]["track_query_hs_embeds"]
            return {"pred_logits": logits[None], "pred_boxes": boxes[None], "hs_embed": embeds[None]}, None, None, None, None

    tr = host_tracker(Many(), {"bbox": DeformablePostProcess()}, tf.tracker_cfg("default"), False)
    blob = {"img": torch.zeros(1, 3, 8, 8), "orig_size": torch.tensor([[1000, 1000]]), "dets": torch.zeros(1, 0, 4)}
    for _ in range(3):
        tr.step(blob)
    assert tr._bufs["capacity"] == 512                       # 256 at the first frame, 150 tracks + 150 queries later
    assert len(tr.tracks) == 150 and tr.track_num == 150
    assert sorted(t.id for t in tr.tracks) == list(range(150))
    for t in tr.tracks:
        assert float(t.hs_embed[-1][0]) == float(t.obj_ind.item())


def test_soft_reset_keeps_the_id_counter(host_tracker):
    scene = tf.Scene()
    det = tf.ScriptedDetector(scene)
    tr = host_tracker(det, {"bbox": DeformablePostProcess()}, tf.tracker_cfg("default"), False)
    blobs = list(tf.blobs(scene))
    tr.step(blobs[0])
    first = tr.track_num
    assert first > 0
    tr.reset(hard=False)
    det.frame = 0
    tr.step(blobs[0])
    assert tr.track_num == 2 * first and min(t.id for t in tr.tracks) == first and tr.frame_index == 2


def test_product_class_refuses_cpu_tensors():
    scene = tf.Scene()
    tr = DeviceTracker(tf.ScriptedDetector(scene), {"bbox": DeformablePostProcess()}, tf.tracker_cfg("default"), False)
    with pytest.raises(RuntimeError, match="CUDA"):
        tr.step(next(iter(tf.blobs(scene))))


class _RandomDetector(torch.nn.Module):
    """Noise detector: every frame answers k track queries + nq object queries with seeded random boxes, logits and
    embeddings (track queries mostly keep their box).  Two trackers that take the same decisions see the same outputs."""
    overflow_boxes = True

    def __init__(self, seed, num_queries=24, hidden=16):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))
        self.seed, self.num_queries, self.hidden_dim, self.frame = seed, num_queries, hidden, 0

    def forward(self, img, targets=None, prev_features=None):
        g = torch.Generator().manual_seed(self.seed * 1000 + self.frame)
        self.frame += 1
        k = 0 if targets is None else len(targets[0]["track_query_boxes"])
        nq = self.num_queries
        centres = torch.rand(k + nq, 2, generator=g) * 0.8 + 0.1
        sizes = torch.rand(k + nq, 2, generator=g) * 0.25 + 0.02
        boxes = torch.cat([centres, sizes], 1)
        logits = torch.randn(k + nq, 3, generator=g) * 1.5
        logits[:, 0] += 0.3
        embeds = torch.randn(k + nq, self.hidden_dim, generator=g)
        if k:
            keep = torch.rand(k, generator=g) < 0.8
            boxes[:k][keep] = targets[0]["track_query_boxes"][keep] + 0.01 * torch.randn(int(keep.sum()), 4, generator=g)
            embeds[:k] = targets[0]["track_query_hs_embeds"] + 0.3 * embeds[:k]
            logits[:k, 0] += 0.8
        boxes[:, 2:].clamp_(min=0.0)
        # public detections of this frame: jittered copies of some object-query boxes plus a few random ones
        cx, cy, w, h = (boxes[k:] + 0.01 * torch.randn(nq, 4, generator=g)).unbind(1)
        pub = torch.stack([(cx - w / 2) * 640, (cy - h / 2) * 480, (cx + w / 2) * 640, (cy + h / 2) * 480], 1)
        pub = pub[torch.rand(nq, generator=g) < 0.5]
        xy = torch.rand(3, 2, generator=g) * 400
        self.public = torch.cat([pub, torch.cat([xy, xy + 60], 1)], 0)[None]
        return {"pred_logits": logits[None], "pred_boxes": boxes[None], "hs_embed": embeds[None]}, None, None, None, None


@pytest.mark.parametrize("seed", range(30))
def test_device_routine_equals_host_tracker_on_random_scenes(host_tracker, seed):
    rng = np.random.RandomState(seed)
    cfg = dict(tf.BASE_CFG)
    cfg.update(
        public_detections=[False, "center_distance", "min_iou_0_5"][seed % 3],
        detection_obj_score_thresh=float(rng.uniform(0.5, 0.8)), track_obj_score_thresh=float(rng.uniform(0.4, 0.7)),
        reid_score_thresh=float(rng.uniform(0.4, 0.8)), detection_nms_thresh=float(rng.choice([0.0, 0.3, 0.6])),
        track_nms_thresh=float(rng.choice([0.0, 0.4, 0.7])), steps_termination=int(rng.randint(1, 3)),
        inactive_patience=int(rng.randint(1, 6)), reid_greedy_matching=bool(seed % 2),
        reid_sim_threshold=float(rng.choice([0.0, 3.0, 6.0])), reid_sim_only=seed % 5 == 4)
    outs = []
    for cls in (Tracker, host_tracker):
        det = _RandomDetector(seed)
        tr = cls(det, {"bbox": DeformablePostProcess()}, cfg, False)

        class Blob(dict):                               # 'dets' is read after the forward: hand out that frame's boxes
            def __getitem__(self, key):
                return det.public if key == "dets" else dict.__getitem__(self, key)
        for t in range(14):
            tr.step(Blob(img=torch.zeros(1, 3, 8, 8), orig_size=torch.tensor([[480, 640]]), dets=None))
        outs.append(tf.summarise(tr))
    a, b = outs
    assert a["track_num"] > 5
    for key in a:
        if key == "rows":
            np.testing.assert_array_equal(a[key][:, :3], b[key][:, :3], err_msg=key)
            np.testing.assert_allclose(a[key][:, 3:], b[key][:, 3:], rtol=1e-6, atol=1e-4)
        else:
            np.testing.assert_array_equal(a[key], b[key], err_msg=f"seed {seed}: {key}")


def test_error_paths_of_the_step_routine(host_tracker):
    """a state / query-count mismatch is reported through the header (error 1), too many rows through error 2 -- and the
    Python side refuses to grow beyond the routine's 2048 rows"""
    scene = tf.Scene()
    det = tf.ScriptedDetector(scene)
    tr = host_tracker(det, {"bbox": DeformablePostProcess()}, tf.tracker_cfg("default"), False)
    blobs = list(tf.blobs(scene))
    tr.step(blobs[0])
    assert tr._n_query > 0
    tr._n_query -= 1                                    # the detector will answer one track query too few
    with pytest.raises((RuntimeError, AssertionError), match="error 1|shape|\\("):
        tr.step(blobs[1])

    class Huge(torch.nn.Module):
        num_queries, overflow_boxes = 2100, True

        def __init__(self):
            super().__init__()
            self.p = torch.nn.Parameter(torch.zeros(1))

        def forward(self, img, targets=None, prev_features=None):
            q = self.num_queries
            return {"pred_logits": torch.full((1, q, 2), -5.0), "pred_boxes": torch.full((1, q, 4), 0.5),
                    "hs_embed": torch.zeros(1, q, 4)}, None, None, None, None
    big = host_tracker(Huge(), {"bbox": DeformablePostProcess()}, tf.tracker_cfg("default"), False)
    with pytest.raises(RuntimeError, match="2048"):
        big.step({"img": torch.zeros(1, 3, 8, 8), "orig_size": torch.tensor([[100, 100]]), "dets": torch.zeros(1, 0, 4)})


def test_public_detections_without_a_dets_entry(host_tracker):
    """blob without 'dets' while public detections are required: nothing may start (tracker.py:437-446 with no boxes)"""
    scene = tf.Scene()
    cfg = tf.tracker_cfg("public_center")
    outs = []
    for cls in (Tracker, host_tracker):
        det = tf.ScriptedDetector(scene, overflow_boxes=False)
        tr = cls(det, {"bbox": DeformablePostProcess()}, cfg, False)
        for blob in list(tf.blobs(scene))[:3]:
            blob.pop("dets")
            tr.step(blob)
        outs.append((tr.track_num, len(tr.results)))
    assert outs[0] == outs[1] == (0, 0)


def test_device_routine_under_the_padded_detector(host_tracker, monkeypatch):
    """GraphedDetector's filler-padded program (eager on CPU) fed by the routine's own next-frame queries: same ids and
    values as the host tracker over the same padded detector"""
    from oracle.torch_ref import msda_core_torch
    import trackformer_b200.msda_module as mm
    from test_model_parity_cpu import build
    from trackformer_b200.graphed_detector import GraphedDetector

    class _OracleFn:
        @staticmethod
        def apply(value, shapes, loc, attn, step):
            return msda_core_torch(value, shapes, loc, attn)
    monkeypatch.setattr(mm, "MSDeformAttnFunction", _OracleFn)
    gold = np.load(os.path.join(GOLD, "tracker_model_sequence.npz"))
    cfg = {k: float(v) for k, v in zip(gold["cfg_keys"], gold["cfg_values"])}
    cfg["prev_frame_dist"] = int(cfg["prev_frame_dist"])
    outs = []
    for base in (Tracker, host_tracker):
        class Padded(base):
            def __init__(self, model, post, cfg_, attn):
                super().__init__(GraphedDetector(model, bucket=8, use_graphs=False), post, cfg_, attn)
        outs.append(tf.run_model_sequence(build, Padded, DeformablePostProcess(), cfg))
    a, b = outs
    assert len(a["rows"]) > 0
    for key in ("num_reids", "track_num", "frame_index", "active_ids", "inactive_ids", "inactive_counts"):
        np.testing.assert_array_equal(a[key], b[key], err_msg=key)
    np.testing.assert_array_equal(a["rows"][:, :3], b["rows"][:, :3])
    np.testing.assert_allclose(a["rows"][:, 3:], b["rows"][:, 3:], rtol=1e-6, atol=1e-6)
