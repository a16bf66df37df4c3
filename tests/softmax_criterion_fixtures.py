"""Inputs of the softmax set-criterion fixture (tests/golden/softmax_criterion.npz).

The vanilla-DETR criterion (cfgs/train.yaml: ``focal_loss: false``, weighted cross-entropy over C = classes + 1 logits,
"no object" last, ``eos_coef`` 0.1) with the tracking targets of train_tracking.yaml.  The inputs come from the same
seeded generator as the focal fixture (tests/set_criterion_fixtures.py) -- trained rows, background rows confident on
the last column (here: "no object"), boxes in every overlap relation, pinned and false-positive track queries -- at the
vanilla model's 100 object queries:

  coco   C + 1 = 92, 20 track rows (3 and 2 false positives) before 100 object rows, 30 and 45 boxes
  mot    C + 1 = 21, 30 track rows (4 and 6 false positives) before 100 object rows, 40 and 55 boxes

tests/golden/make_golden_softmax_criterion.py records the reference's own SetCriterion on them, with
``track_query_false_positive_eos_weight`` on ("fp1") and off ("fp0").
"""
import set_criterion_fixtures as scf

K = scf.K
COST_CLASS, COST_BBOX, COST_GIOU = 1.0, 5.0, 2.0          # cfgs/train.yaml
EOS_COEF = 0.1
N_OBJ = 100

CASES = {
    "coco": dict(seed=40, C=92, sizes=(30, 45), n_track=20, n_fp=(3, 2)),
    "mot": dict(seed=41, C=21, sizes=(40, 55), n_track=30, n_fp=(4, 6)),
}
FP_WEIGHT = {"fp1": True, "fp0": False}


def make_case(name):
    """-> dict(logits [K,B,Q,C+1] f32, boxes [K,B,Q,4] f32, targets [B] (CPU), weights [3,K] f64, meta), drawn by
    set_criterion_fixtures.make_case with this module's case table and query count"""
    saved = scf.CASES, scf.N_OBJ
    scf.CASES, scf.N_OBJ = CASES, N_OBJ
    try:
        return scf.make_case(name)
    finally:
        scf.CASES, scf.N_OBJ = saved


checksum = scf.checksum
grad_logits_rows = scf.grad_logits_rows
stacked_indices = scf.stacked_indices
