"""CPU: oracle/evaluation.py, the numpy restatement of the frame-mAP of test.py / train.py::validate, against the
reference's own run_evaluation: the per-class APs recorded in tests/golden/eval_cases.npz (bit for bit on every
tie-free case, within the tie bracket on the others), a fresh seeded case run through the reference checkout when it is
present, and the pairwise-summation model against np.sum."""
import os
import sys

import numpy as np
import pytest

from oracle import evaluation as oev
from oracle import refload

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "eval_cases.npz")


def load():
    z = np.load(GOLDEN)
    cats = [{"id": int(i), "name": str(n)} for i, n in zip(z["cat_ids"], z["cat_names"])]
    return z, cats, [str(c) for c in z["cases"]]


def case_text(z, name):
    """The CSV lines test.py writes for the case: detections from every clip's rows, then the ground truth."""
    det, count = z[name + "_det"], z[name + "_count"]
    keys = list(zip([str(v) for v in z[name + "_video"]], [int(f) for f in z[name + "_fid"]]))
    ld = [int(v) for v in z[name + "_label_dict"]]
    clips = [[(det[b, k, :4], int(det[b, k, 5]), det[b, k, 4]) for k in range(int(count[b]))] for b in range(len(keys))]
    gkeys = list(zip([str(v) for v in z[name + "_gt_video"]], [int(f) for f in z[name + "_gt_fid"]]))
    excl = list(zip([str(v) for v in z[name + "_excl_video"]], [int(f) for f in z[name + "_excl_fid"]]))
    return (oev.gt_lines(gkeys, z[name + "_gt_boxes"], z[name + "_gt_labels"]), oev.detection_lines(clips, keys, ld), excl)


def bits(a):
    a = np.asarray(a, dtype=np.float64)
    return np.where(np.isnan(a), np.int64(-1), a.view(np.int64))


def test_golden_cases_cover_the_issue_list():
    z, cats, names = load()
    assert {"distinct", "ties", "edge", "many"} <= set(names)
    assert bool(z["distinct_tie_free"]) and bool(z["edge_tie_free"]) and bool(z["many_tie_free"])
    assert not bool(z["ties_tie_free"])
    assert len(cats) == 60 and max(c["id"] for c in cats) == 80


@pytest.mark.parametrize("name", ["distinct", "ties", "ties_fine", "edge", "many"])
def test_oracle_matches_the_reference(name):
    z, cats, _ = load()
    gt, det, excl = case_text(z, name)
    ev = oev.run(cats, gt, det, excl)
    ap, ref = ev.per_class_ap(), z[name + "_ref_ap"]
    lo, hi = ev.ap_bounds()
    assert np.array_equal(np.isnan(ap), np.isnan(ref))
    ok = ~np.isnan(ref)
    assert np.all(lo[ok] <= ref[ok]) and np.all(ref[ok] <= hi[ok])
    if bool(z[name + "_tie_free"]):
        assert np.array_equal(bits(ap), bits(ref))
        m = oev.metrics(cats, ap)
        assert m["PascalBoxes_Precision/mAP@0.5IOU"] == z[name + "_ref_map"]
        assert len(m) == 61


def test_pairwise_sum_model_equals_np_sum():
    """Adversarial arrays: magnitudes over 16 decades, both signs, every length class of the model (< 8, <= 128,
    split once, split many times)."""
    rs = np.random.RandomState(7)
    for n in list(range(0, 20)) + [127, 128, 129, 135, 136, 255, 256, 257, 1000, 1023, 4097, 20011]:
        for _ in range(3):
            a = rs.standard_normal(n) * 10.0 ** rs.randint(-8, 8, n)
            assert oev.pairwise_sum(a) == float(np.sum(a)), n
    a = np.array([1e16, 1.0, -1e16] * 50 + [3.0] * 7)
    assert oev.pairwise_sum(a) == float(np.sum(a))


def test_csv_round_is_the_round_trip():
    for v, s in ((np.float32(0.99995), "0.9999"), (np.float32(0.123456), "0.1235"), (1e-45, "1e-45"), (2.5e-5, "2.5e-05")):
        assert oev.csv_round(v) == float(format(float(v), ".4")) == float(s)


@pytest.mark.skipif(not refload.available(), reason="needs the reference checkout")
def test_oracle_matches_a_fresh_reference_run():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_eval_golden as g
    gap = g.reference()
    cats, _ = gap.read_labelmap(open(g.LABELMAP))
    ld = sorted(c["id"] for c in cats)
    rs = np.random.RandomState(99)
    case = g.random_case(rs, 30, 8, len(ld), ld, g.unique_scores(rs, 2000))
    det = g.det_text(case, ld)
    gt = oev.gt_lines(case.gt_keys, case.gt_boxes, case.gt_labels)
    import contextlib
    import io
    with contextlib.redirect_stdout(io.StringIO()):
        m = gap.run_evaluation(open(g.LABELMAP), g.text(gt, "gt.csv"), g.text(det, "det.csv"), None)
    ours = oev.metrics(cats, oev.run(cats, gt, det).per_class_ap())
    assert list(m) == list(ours)
    for k in m:
        assert bits(m[k]) == bits(ours[k]), k
