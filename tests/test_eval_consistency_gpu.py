"""The relations of tests/test_eval_consistency_cpu.py -- COCO box AP = mask AP on rectangles, MOT = MOTS on
rectangles, the MOTS ignore rule against dense masks, and every evaluator's invariances -- through the public CUDA
entry points: `CocoEvaluator`, `evaluate_mot_accums` / `evaluate_mots_accums` (and their counters), and
`PanopticEvaluator` / `pq_compute`.  Also at full size: a 1080 x 1920 MOTS scene and COCO masks at 800 x 1333."""
import numpy as np
import pytest
import torch

import eval_consistency_fixtures as ef
import test_eval_consistency_cpu as rel
from trackformer_b200 import coco_eval as ce
from trackformer_b200 import mot_eval, mots_eval

pytestmark = pytest.mark.gpu


class CudaBackend:
    def coco(self, dataset, updates, iou_type):
        ev = ce.CocoEvaluator(dataset, (iou_type,))
        for u in updates:
            ev.update({i: {k: v.to("cuda") for k, v in p.items()} for i, p in u.items()})
        ev.synchronize_between_processes()
        ev.accumulate()
        ev.summarize()
        e = ev.coco_eval[iou_type]
        return e.eval["precision"], e.eval["recall"], e.eval["scores"], e.stats

    def mot(self, accums, names):
        out, _ = mot_eval.evaluate_counters(accums)
        summary, _ = mot_eval.evaluate_mot_accums(accums, names)
        return out, summary

    def mots(self, accums, names):
        out, _ = mots_eval.evaluate_counters(accums, names=names)
        summary, _ = mots_eval.evaluate_mots_accums(accums, names)
        return out, summary

    pq_device = "cuda"

    def pq_lib(self):
        return None

    def pq_map(self, m):
        return torch.from_numpy(m).to("cuda")


@pytest.fixture
def backend(cuda_device):
    return CudaBackend()


@pytest.mark.parametrize("seed", range(2))
def test_coco_bbox_equals_segm(backend, seed):
    rel.check_coco_bbox_equals_segm(backend, *ef.coco_scene(seed))


def test_coco_bbox_equals_segm_800x1333(backend):
    ds, up = ef.coco_scene(5, images=((800, 1333, 80), (800, 1333, 260), (64, 96, 32), (64, 64, 32)))
    box = rel.check_coco_bbox_equals_segm(backend, ds, up)
    rel.same(box, backend.coco(ds, [ef.coco_permute(up, np.random.default_rng(5))], "segm"))


@pytest.mark.parametrize("iou_type", ["bbox", "segm"])
def test_coco_invariances(backend, iou_type):
    rel.check_coco_invariances(backend, *ef.coco_scene(11), iou_type, 11)


@pytest.mark.parametrize("iou_type", ["bbox", "segm"])
def test_coco_translation(backend, iou_type):
    ds, up = ef.coco_scene(12, images=((200, 200, 16), (488, 488, 120), (64, 64, 32), (72, 72, 32)), pad=4)
    rel.check_coco_translation(backend, ds, up, iou_type, 12)


@pytest.mark.parametrize("seed", range(2))
def test_mot_equals_mots(backend, seed):
    rel.check_mot_equals_mots(backend, ef.track_scenes(10 * seed))


def test_mot_equals_mots_1080x1920(backend):
    scenes = ef.track_scenes(20)
    scenes["full"] = ef.track_scene(21, n_frames=6, size=(1080, 1920), cell=(120, 120), p_obj=0.8)
    rel.check_mot_equals_mots(backend, scenes)


def test_track_invariances(backend):
    rel.check_track_invariances(backend, ef.track_scenes(40), 40)


@pytest.mark.parametrize("seed", range(2))
def test_mot_invariances_overlapping_boxes(backend, seed):
    rel.check_mot_invariances_overlapping(backend, seed)


@pytest.mark.parametrize("seed", range(2))
def test_mots_ignore_rule_against_dense_masks(backend, seed):
    rel.check_mots_ignore_rule(backend, ef.track_scene(50 + seed, n_frames=10, ignore=True))


def test_mots_ignore_rule_1080x1920(backend):
    rel.check_mots_ignore_rule(backend, ef.track_scene(60, n_frames=4, size=(1080, 1920), cell=(120, 120),
                                                       ignore=True))


@pytest.mark.parametrize("seed", range(2))
def test_pq_invariances(backend, tmp_path, seed):
    rel.check_pq_invariances(backend, ef.pq_scene(seed), tmp_path, seed)


def test_pq_compute_batching(backend, tmp_path):
    rel.check_pq_compute_batching(backend, ef.pq_scene(7, n_images=6), tmp_path)
