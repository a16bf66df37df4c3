"""Frame ingest on the GPU (csrc/frame_ingest.cu through FrameIngest): equal -- torch.equal, no tolerance -- to the images
recorded from the reference's validation transform and to the host restatement of tests/test_frame_ingest_cpu.py at
production shapes; every input kind, buffer reuse, padded batches, and Tracker / DeviceTracker fed raw uint8 frames."""
import numpy as np
import pytest
import torch

import track_mask_fixtures as tmf
import tracker_fixtures as tf
from test_frame_ingest_cpu import GOLD, NAMES, restated_img, synthetic_frame

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


@pytest.mark.parametrize("name", NAMES)
def test_equals_reference_transform(dev, name):
    from trackformer_b200.frame_ingest import FrameIngest
    val_width, max_size = (int(v) for v in GOLD[f"{name}_settings"])
    out = FrameIngest(dev, val_width, max_size)(GOLD[f"{name}_frame"])
    assert out["img"].is_cuda and out["img"].dtype == torch.float32
    assert torch.equal(out["img"].cpu()[0], torch.from_numpy(GOLD[f"{name}_img"]))
    assert out["size"].tolist() == [GOLD[f"{name}_size"].tolist()]
    assert out["orig_size"].tolist() == [GOLD[f"{name}_orig_size"].tolist()]


@pytest.mark.parametrize("shape,val_width,max_size", [
    ((1080, 1920), 800, 1333),            # -> 750 x 1333, ksize 5
    ((480, 640), 800, 1333),              # -> 800 x 1066, enlargement, ksize 3
    ((800, 1333), 800, 1333),             # both passes skipped
    ((1080, 1920), 200, 1333),            # -> 200 x 355, ksize 13
    ((1600, 333), 20, 1333),              # -> 96 x 20, ksize 35: a tile's footprint needs more than 48 KB of shared memory
    ((4000, 200), 3, 1333),               # -> 60 x 3, ksize 135: the footprint of 16 rows does not fit, tiles get 8
])
def test_equals_restatement_at_production_shapes(dev, shape, val_width, max_size):
    from trackformer_b200.frame_ingest import FrameIngest
    frame = synthetic_frame(*shape, seed=11)
    got = FrameIngest(dev, val_width, max_size)(frame)["img"].cpu()
    assert torch.equal(got, restated_img(frame, val_width, max_size))


def test_input_kinds_and_buffer_reuse(dev):
    from trackformer_b200.frame_ingest import FrameIngest
    ingest = FrameIngest(dev, 120, 200)
    a, b = synthetic_frame(216, 384, seed=1), synthetic_frame(150, 130, seed=2)
    want_a, want_b = restated_img(a, 120, 200), restated_img(b, 120, 200)
    wide = torch.zeros(216, 400, 3, dtype=torch.uint8, device=dev)
    wide[:, :384] = torch.from_numpy(a).to(dev)
    kinds = {"numpy": a, "numpy_strided": np.ascontiguousarray(a[:, ::-1])[:, ::-1], "cpu": torch.from_numpy(a.copy()),
             "pinned": torch.from_numpy(a.copy()).pin_memory(), "cuda": torch.from_numpy(a).to(dev),
             "cuda_row_strided": wide[:, :384]}
    assert not kinds["cuda_row_strided"].is_contiguous()
    for kind, frame in kinds.items():
        assert torch.equal(ingest(frame)["img"].cpu(), want_a), kind

    # steady state: a known shape allocates nothing, and another shape in between corrupts neither result
    out_b = ingest(b)["img"]
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(dev)
    first = ingest(a)["img"]
    again = ingest(b)["img"]
    second = ingest(kinds["cuda"])["img"]
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(dev) == before
    assert first.data_ptr() == second.data_ptr() and again.data_ptr() == out_b.data_ptr()
    assert torch.equal(second.cpu(), want_a) and torch.equal(again.cpu(), want_b)

    with pytest.raises(ValueError, match=r"\[H, W, 3\]"):
        ingest(torch.from_numpy(a).to(dev).permute(2, 0, 1))
    with pytest.raises(ValueError, match=r"\[H, W, 3\]"):
        ingest(torch.from_numpy(a).to(dev)[:, ::2])


def test_extension_rejects_wrong_arguments(dev):
    from trackformer_b200 import ext
    from trackformer_b200.frame_ingest import normalise_table, resample_table
    m = ext.load()
    src = torch.zeros(10, 20, 3, dtype=torch.uint8, device=dev)
    lut = normalise_table().to(dev)
    dst = torch.empty(3, 10, 20, device=dev)
    m.frame_ingest(src, None, 0, None, 0, lut, dst)
    with pytest.raises(RuntimeError, match="uint8 CUDA"):
        m.frame_ingest(src.cpu(), None, 0, None, 0, lut, dst)
    with pytest.raises(RuntimeError, match="uint8 CUDA"):
        m.frame_ingest(src.float(), None, 0, None, 0, lut, dst)
    with pytest.raises(RuntimeError, match="table is required"):
        m.frame_ingest(src, None, 0, None, 0, lut, torch.empty(3, 10, 16, device=dev))
    with pytest.raises(RuntimeError, match="lut"):
        m.frame_ingest(src, None, 0, None, 0, lut[:, :128].contiguous(), dst)
    with pytest.raises(RuntimeError, match="last dimension"):
        m.frame_ingest(src, None, 0, None, 0, lut, torch.empty(3, 10, 40, device=dev)[:, :, ::2])
    xt = torch.from_numpy(resample_table(20, 16)).to(dev)
    with pytest.raises(RuntimeError, match="xtab"):
        m.frame_ingest(src, xt[:8].contiguous(), 3, None, 0, lut, torch.empty(3, 10, 16, device=dev))
    with pytest.raises(RuntimeError, match="code -2"):          # cnt beyond ksize
        m.frame_ingest(src, xt, 99, None, 0, lut, torch.empty(3, 10, 16, device=dev))


def test_batch_equals_nested_tensor_of_single_results(dev):
    from trackformer_b200.frame_ingest import FrameIngest
    from trackformer_b200.util import nested_tensor_from_tensor_list
    ingest = FrameIngest(dev, 120, 200)
    frames = [synthetic_frame(216, 384, seed=1), torch.from_numpy(synthetic_frame(300, 170, seed=2)).to(dev),
              synthetic_frame(60, 80, seed=3), synthetic_frame(216, 384, seed=4)]
    singles, sizes, origs = [], [], []
    for f in frames:
        out = ingest(f)
        singles.append(out["img"][0].clone())
        sizes.append(out["size"][0].tolist())
        origs.append(out["orig_size"][0].tolist())
    want = nested_tensor_from_tensor_list(singles)
    got, got_sizes, got_origs = ingest.batch(frames)
    assert len({tuple(s) for s in sizes}) == 3
    assert torch.equal(got.tensors, want.tensors) and torch.equal(got.mask, want.mask)
    assert got_sizes.tolist() == sizes and got_origs.tolist() == origs


# --------------------------------------------------------------------------------------------- under the trackers
def uint8_video(size, n_frames, seed=5):
    """a slowly changing synthetic uint8 video [n, H, W, 3]"""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, size + (3,)).astype(np.float32)
    drift = rng.standard_normal(size + (3,)).astype(np.float32)
    return [np.clip(base + 6.0 * t * drift, 0, 255).astype(np.uint8) for t in range(n_frames)]


@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("tracker", ["Tracker", "DeviceTracker"])
def test_trackers_from_uint8_frames_equal_preprocessed(dev, tracker, masks):
    """blob["frame"] against blob["img"] made by the host restatement: same ids, boxes, scores and masks, and the
    ingest's images replay the graphs the detector already holds for that shape"""
    import model_fixtures as mf
    from trackformer_b200.deformable_detr import DeformablePostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.frame_ingest import FrameIngest, val_size
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.model_factory import build_model, default_args
    from trackformer_b200.segmentation import PostProcessSegm
    from trackformer_b200.tracker import Tracker

    orig, settings, n_frames = (230, 300), (128, 214), 5
    video = uint8_video(orig, n_frames)
    size = val_size(*orig, *settings)
    assert size != orig
    torch.manual_seed(0)
    model, _, _ = build_model(default_args(True, False, device=str(dev), **({"masks": True} if masks else {})))
    mf.canonical_weights_(model, 0)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if "class_embed" in name and name.endswith("bias"):
                p[0] += 6.0
        if masks:
            model.mask_head.out_lay.weight.mul_(8.0)
            model.mask_head.out_lay.bias.mul_(8.0)
    model.to(dev)
    model.tracking()
    cfg = dict(tf.BASE_CFG)
    cfg.update(detection_obj_score_thresh=0.3, track_obj_score_thresh=0.3, reid_score_thresh=0.3, inactive_patience=3,
               reid_sim_threshold=2.0, detection_nms_thresh=0.7, track_nms_thresh=0.7, steps_termination=2)
    posts = {"bbox": DeformablePostProcess()}
    if masks:
        posts["segm"] = PostProcessSegm()
    cls = {"Tracker": Tracker, "DeviceTracker": DeviceTracker}[tracker]

    det = GraphedDetector(model, bucket=16)                # one detector for both runs: the same graphs replay

    def run(make_blob, **kwargs):
        tr = cls(det, posts, cfg, False, **kwargs)
        tr.reset()
        with torch.no_grad():
            for t in range(n_frames):
                tr.step(make_blob(t))
        out = tf.summarise(tr)
        if masks:
            out["labels"] = tmf.label_maps(tr, n_frames, orig)
        return out

    dets = torch.zeros(1, 0, 4)
    want = run(lambda t: {"img": restated_img(video[t], *settings), "orig_size": torch.tensor([list(orig)]),
                          "size": torch.tensor([list(size)]), "dets": dets})
    captures = det.captures
    got = run(lambda t: {"frame": video[t], "dets": dets}, frame_ingest=FrameIngest(dev, *settings))
    assert len(want["rows"]) > 0
    for key in want:
        np.testing.assert_array_equal(got[key], want[key], err_msg=key)
    if masks:
        assert (want["labels"] >= 0).any()
    assert 0 < captures < n_frames and det.captures == captures      # the ingest's images replay the existing graphs


def test_default_ingest_is_created_on_first_use(dev):
    """a tracker built without an ingest makes the default one (800 / 1333) when it first sees a "frame\""""
    from trackformer_b200.deformable_detr import DeformablePostProcess
    from trackformer_b200.frame_ingest import FrameIngest
    from trackformer_b200.tracker import Tracker

    class Recording(tf.ScriptedDetector):
        def forward(self, img, targets=None, prev_features=None):
            self.seen = img
            return super().forward(img, targets, prev_features)
    det = Recording(tf.Scene(seed=0), overflow_boxes=False).to(dev)
    tr = Tracker(det, {"bbox": DeformablePostProcess()}, tf.tracker_cfg("default"), False)
    tr.reset()
    frame = synthetic_frame(tf.IMG_H, tf.IMG_W, seed=9)
    tr.step({"frame": frame, "dets": torch.zeros(1, 0, 4)})
    assert isinstance(tr.frame_ingest, FrameIngest) and tr.frame_index == 1
    assert torch.equal(det.seen.cpu(), restated_img(frame))
