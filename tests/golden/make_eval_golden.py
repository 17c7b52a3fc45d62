"""Generates tests/golden/eval_cases.npz by running the reference's own get_ava_performance.run_evaluation (imported
unmodified from the reference checkout) on the CSV text test.py:129-139 and :210-218 would write for seeded detector
outputs and ground truth.  Only runnable where the reference checkout exists; the fixture it writes is committed.

    python tests/golden/make_eval_golden.py

numpy 2 removed the np.float / np.NAN aliases the evaluator uses (and np.bool in some releases); the missing ones are set
here to float, nan and bool before the import.  The CSV files are io.StringIO objects (with the .name read_csv logs).

Shared: cat_ids / cat_names (read_labelmap of the AVA v2.1 label map), cases.  Per case <name>: _det float32
[clips, cap, 8] and _count int32 [clips] (step_detect_f32's output of every clip), _video / _fid (the clip keys), _batches
(clips per add_detections call), _label_dict (detector class -> label id), _gt_video / _gt_fid / _gt_boxes float64 [n, 4]
/ _gt_labels (ground-truth rows), _excl_video / _excl_fid, _ref_ap float64 [80] (the reference's per-category APs at
their class index, NaN elsewhere), _ref_map, _tie_free (True when no group of equal scores of a class mixes TPs and FPs:
the oracle's bounds coincide, so every tie order gives the reference's result).
"""
import contextlib
import io
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import evaluation as oev  # noqa: E402
from oracle import refload  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "eval_cases.npz")
LABELMAP = os.path.join(refload.REF, "external", "ActivityNet", "Evaluation", "ava",
                        "ava_action_list_v2.1_for_activitynet_2018.pbtxt.txt")
F = np.float32


def reference():
    for name, value in (("bool", bool), ("float", float), ("NAN", np.nan)):
        if not hasattr(np, name):      # numpy 2 has np.bool again (np.bool_); replacing it breaks numpy.ma
            setattr(np, name, value)
    if refload.REF not in sys.path:
        sys.path.insert(0, refload.REF)
    import logging
    logging.disable(logging.CRITICAL)
    from external.ActivityNet.Evaluation import get_ava_performance as gap
    return gap


def text(lines, name):
    f = io.StringIO("".join(lines))
    f.name = name
    return f


class Case:
    def __init__(self, cap):
        self.cap, self.clips, self.keys, self.batches = cap, [], [], []
        self.gt_keys, self.gt_boxes, self.gt_labels, self.excl = [], [], [], []

    def batch(self, clips):
        """clips: [(key, rows)] with rows [(x1, y1, x2, y2, score, class index)]"""
        for key, rows in clips:
            d = np.zeros((self.cap, 8), F)
            for k, r in enumerate(rows):
                d[k, :6] = r
                d[k, 6] = k
            self.clips.append((d, len(rows)))
            self.keys.append(key)
        self.batches.append(len(clips))

    def gt(self, key, box, label):
        self.gt_keys.append(key)
        self.gt_boxes.append(box)
        self.gt_labels.append(label)


def det_text(case, label_dict):
    clips = [[(d[k, :4], int(d[k, 5]), d[k, 4]) for k in range(n)] for d, n in case.clips]
    return oev.detection_lines(clips, case.keys, label_dict)


def random_case(rs, n_frames, per_batch, ncls, label_dict, score_fn, rows_per_frame=(5, 40), cap=64, gt_per_frame=(1, 6)):
    case = Case(cap)
    frames = [("vid%02d" % (i // 10), 900 + i) for i in range(n_frames)]
    clips = []
    for key in frames:
        ng = rs.randint(gt_per_frame[0], gt_per_frame[1] + 1)
        gts = []
        for _ in range(ng):
            x1, y1 = rs.uniform(0, 0.6, 2)
            w, h = rs.uniform(0.1, 0.4, 2)
            b = np.array([x1, y1, x1 + w, y1 + h])
            lab = label_dict[rs.randint(0, ncls)]
            case.gt(key, b, lab)
            gts.append((b, lab))
        rows = []
        for _ in range(rs.randint(*rows_per_frame)):
            b, lab = gts[rs.randint(0, len(gts))]
            cl = label_dict.index(lab) if rs.rand() < 0.7 else rs.randint(0, ncls)
            jb = b + rs.normal(0, 0.04, 4)
            rows.append((F(jb[0]), F(jb[1]), F(jb[2]), F(jb[3]), score_fn(), cl))
        clips.append((key, rows))
    for i in range(0, len(clips), per_batch):
        case.batch(clips[i:i + per_batch])
    return case


def unique_scores(rs, n):
    """n scores, distinct after the 4-digit rounding: 1000..9999 over 10^4 and over 10^5."""
    pool = np.concatenate([np.arange(1000, 10000) / 1e4, np.arange(1000, 10000) / 1e5])
    vals = iter(F(v) for v in rs.permutation(pool)[:n])
    return lambda: next(vals)


def edge_case(rs, label_dict, ncls):
    case = Case(64)
    lab = label_dict
    A, Bk, Ck, Dk, Ek, Xk = ("e0", 901), ("e0", 902), ("e1", 903), ("e1", 904), ("e2", 905), ("e2", 906)
    score = unique_scores(rs, 400)
    # A: IoU exactly 0.5, two identical ground truths (argmax ties), degenerate ground truths (NaN IoU, zero area) first
    case.gt(A, [0.0, 0.0, 1.0, 1.0], lab[0])
    case.gt(A, [0.2, 0.2, 0.6, 0.6], lab[1])
    case.gt(A, [0.2, 0.2, 0.6, 0.6], lab[1])
    case.gt(A, [np.nan, 0.1, 0.3, 0.3], lab[2])    # a NaN coordinate: every IoU with it is NaN
    case.gt(A, [0.1, 0.2, 0.3, 0.2], lab[2])       # zero area
    case.gt(A, [0.1, 0.1, 0.3, 0.3], lab[2])
    case.gt(A, [0.3, 0.3, 0.5, 0.5], lab[5])       # a non-whitelisted label below: dropped
    rows_a = [(F(0.0), F(0.0), F(0.5), F(1.0), score(), 0),          # IoU 0.5
              (F(0.2), F(0.2), F(0.6), F(0.6), score(), 1), (F(0.2), F(0.2), F(0.6), F(0.6), score(), 1),
              (F(0.21), F(0.2), F(0.6), F(0.6), score(), 1),
              (F(0.1), F(0.1), F(0.3), F(0.3), score(), 2),          # NaN against the degenerate box: FP
              (F(0.5), F(0.5), F(0.4), F(0.9), score(), 3),          # x1 > x2: invalid
              (F(0.5), F(0.5), F(0.9), F(0.5), score(), 3),          # y1 == y2: invalid
              (F(0.1), F(0.1), F(0.2), F(0.2), score(), ncls),       # non-whitelisted label id
              (F(0.1), F(0.1), F(0.2), F(0.2), score(), ncls + 1)]
    # B: excluded; C: detections only; D: ground truth only; E: split across two batches; X: tiny and decade-crossing values
    case.gt(Bk, [0.1, 0.1, 0.5, 0.5], lab[0])
    case.gt(Dk, [0.1, 0.1, 0.5, 0.5], lab[0])
    case.gt(Dk, [0.1, 0.1, 0.5, 0.5], lab[7])       # class 7: ground truth, no detection anywhere
    case.gt(Ek, [0.1, 0.1, 0.5, 0.5], lab[4])
    case.gt(Ek, [0.5, 0.5, 0.9, 0.9], lab[4])
    case.gt(Xk, [1e-30, 2e-40, 0.99995, 0.5], lab[6])
    case.gt(Xk, [9.9995e-3, 0.0, 0.99995, 0.99995], lab[6])
    case.excl.append(Bk)
    rows_b = [(F(0.1), F(0.1), F(0.5), F(0.5), score(), 0)]
    rows_c = [(F(0.1), F(0.1), F(0.5), F(0.5), score(), 0), (F(0.2), F(0.1), F(0.5), F(0.5), score(), 4)]
    rows_e1 = [(F(0.1), F(0.1), F(0.5), F(0.5), score(), 4), (F(0.5), F(0.5), F(0.9), F(0.95), score(), 4)]
    rows_e2 = [(F(0.5), F(0.5), F(0.9), F(0.9), score(), 4), (F(0.11), F(0.1), F(0.5), F(0.5), score(), 4)]
    rows_x = [(F(1e-30), F(2e-40), F(0.99995), F(0.5), F(0.99995), 6),
              (F(9.9995e-3), F(1e-45), F(0.99995), F(0.99995), F(9.9995e-3), 6),
              (F(9.99949e-3), F(0.0), F(0.999951), F(0.99995), F(0.5), 6),
              (F(0.2), F(0.2), F(0.3), F(0.3), F(1.00005e-3), 6)]
    case.batch([(A, rows_a), (Bk, rows_b), (Ek, rows_e1), (Ck, rows_c)])
    case.batch([(Xk, rows_x), (Dk, []), (Ek, rows_e2)])
    return case


def many_case(rs, label_dict):
    """More than 10,000 rows of one class in one image (distinct scores: no tie at the cut)."""
    n = 10400
    case = Case(n)
    key = ("big", 902)
    case.gt(key, [0.1, 0.1, 0.5, 0.5], label_dict[3])
    case.gt(key, [0.4, 0.4, 0.8, 0.8], label_dict[3])
    score = unique_scores(rs, n + 50)
    rows = []
    for _ in range(n):
        j = rs.normal(0, 0.05, 4)
        rows.append((F(0.1 + j[0]), F(0.1 + j[1]), F(0.5 + j[2]), F(0.5 + j[3]), score(), 3))
    case.gt(("big", 903), [0.1, 0.1, 0.5, 0.5], label_dict[3])
    case.batch([(key, rows)])
    case.batch([(("big", 903), [r[:4] + (score(), 3) for r in rows[:50]])])
    return case


def main():
    gap = reference()
    cats, _ = gap.read_labelmap(open(LABELMAP))
    ids = [c["id"] for c in cats]
    label_dict = sorted(ids)
    ncls = len(label_dict)
    missing = [i for i in range(1, 81) if i not in ids]
    rs = np.random.RandomState(2024)
    cases = {
        "distinct": random_case(rs, 60, 8, ncls, label_dict, unique_scores(rs, 3000)),
        "ties": random_case(rs, 60, 8, ncls, label_dict, lambda: F(rs.choice([0.25, 0.5, 0.75]))),
        "ties_fine": random_case(rs, 40, 8, 5, label_dict, lambda: F(0.3 + rs.randint(0, 3) * 1e-5)),
        "edge": edge_case(rs, label_dict + missing[:2], ncls),
        "many": many_case(rs, label_dict),
    }
    out = {"cat_ids": np.array(ids), "cat_names": np.array([c["name"] for c in cats]), "cases": np.array(list(cases))}
    for name, case in cases.items():
        ld = label_dict + missing[:2] if name == "edge" else label_dict
        dlines = det_text(case, ld)
        glines = oev.gt_lines(case.gt_keys, case.gt_boxes, case.gt_labels)
        elines = ["%s,%04d\n" % k for k in case.excl]
        with contextlib.redirect_stdout(io.StringIO()):     # run_evaluation pprints the metrics
            m = gap.run_evaluation(open(LABELMAP), text(glines, "gt.csv"), text(dlines, "det.csv"),
                                   text(elines, "excl.csv") if elines else None)
        index = {c["id"]: c["name"] for c in cats}
        ref = np.array([m["PascalBoxes_PerformanceByCategory/AP@0.5IOU/%s" % index[i + 1]] if i + 1 in index else np.nan
                        for i in range(max(ids))])
        ev = oev.run(cats, glines, dlines, case.excl)
        lo, hi = ev.ap_bounds()
        ap = ev.per_class_ap()
        tie_free = bool(np.array_equal(lo, hi, equal_nan=True))
        assert np.all((lo <= ref) | np.isnan(ref)) and np.all((ref <= hi) | np.isnan(ref)), name
        if tie_free:
            assert np.array_equal(ap, ref, equal_nan=True), (name, ap, ref)
        print("%-10s rows %6d, gt %4d, tie-free %s, mAP %.6f" % (name, len(dlines), len(glines), tie_free,
                                                                 m["PascalBoxes_Precision/mAP@0.5IOU"]))
        out[name + "_det"] = np.stack([d for d, _ in case.clips])
        out[name + "_count"] = np.array([n for _, n in case.clips], np.int32)
        out[name + "_video"] = np.array([k[0] for k in case.keys])
        out[name + "_fid"] = np.array([k[1] for k in case.keys])
        out[name + "_batches"] = np.array(case.batches)
        out[name + "_label_dict"] = np.array(ld)
        out[name + "_gt_video"] = np.array([k[0] for k in case.gt_keys])
        out[name + "_gt_fid"] = np.array([k[1] for k in case.gt_keys])
        out[name + "_gt_boxes"] = np.array(case.gt_boxes, np.float64)
        out[name + "_gt_labels"] = np.array(case.gt_labels)
        out[name + "_excl_video"] = np.array([k[0] for k in case.excl] or [""])[:len(case.excl)]
        out[name + "_excl_fid"] = np.array([k[1] for k in case.excl], np.int64)
        out[name + "_ref_ap"] = ref
        out[name + "_ref_map"] = np.float64(m["PascalBoxes_Precision/mAP@0.5IOU"])
        out[name + "_tie_free"] = np.bool_(tie_free)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
