"""Generates tests/golden/cls_stage_cases.npz for the classification pre-training stage (train_cls.py).  Only runnable where
the reference checkout exists; the fixture it writes is committed.

    python tests/golden/make_cls_stage_golden.py

Sample selection (train_cls.py:260-297): the reference's own `select_proposals` (utils/utils.py:342-423) and
`flatten_tubes` (utils/tube_utils.py:214), imported unmodified through oracle/refload, on anchors made as ava_cls.py:350-357
makes them (float64: each ground truth or a box near it, plus boxes away from every ground truth, tiled over T frames and
scaled to 400 x 400).  The row building of train_cls.py:271-291 is restated in `reference_rows`.  A seed is kept only when
oracle/select_cls.py's train_cls_select gives the same rows and generator states (that rejects seeds decided by an argsort tie).
Per case <name>: _nums, _ngt, _targets (float32 [sum G, chunks, 4 + C]), _props (float64 [sum n, T, 4]), _np_key / _np_pos
/ _py_state before and _after, _tubes / _targets_out (the flat outputs).

Validation (train_cls.py:433-554): seeded class-only scores and proposals, the CSV text train_cls.py:537-543 writes for them
and the ground truth of :456-466, evaluated by the reference's own get_ava_performance.run_evaluation with exclusions.  Per
case <name>: _prob float32 [R, C], _tubes float32 [R, T, 5] (flatten_tubes with the frame index), _nums [clips], _batches
(clips per validation batch), _video / _fid (clip keys), _gt_video / _gt_fid / _gt_boxes / _gt_labels, _excl_video /
_excl_fid, _width / _height / _conf, _rows (CSV rows written), _ref_ap float64 [80], _ref_map, and _ap_lo / _ap_hi
(oracle/evaluation.py's bracket of the tie contract: equal per class when no group of equal scores mixes TPs and FPs).
Shared: cat_ids / cat_names, label_dict (detector class -> label id, train_cls.py:43-53).
"""
import contextlib
import io
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_eval_golden import LABELMAP, reference as eval_reference, text  # noqa: E402
from oracle import evaluation as oev  # noqa: E402
from oracle import refload  # noqa: E402
from oracle import select_cls as osel  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cls_stage_cases.npz")
F = np.float32
C, T, WIDTH, HEIGHT = 60, 9, 400, 400      # scripts/train_cls.sh: 60 classes, T=9; ava_cls.py:21


def iou1(a, b):
    w = min(a[2], b[2]) - max(a[0], b[0])
    h = min(a[3], b[3]) - max(a[1], b[1])
    inter = max(w, 0.0) * max(h, 0.0)
    return inter / ((a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - inter)


def near(rs, box, lo):
    """A box with IoU > lo with `box` (normalised)."""
    while True:
        c = box + rs.uniform(-0.03, 0.03, 4) * np.array([box[2] - box[0], box[3] - box[1]] * 2)
        if c[2] > c[0] and c[3] > c[1] and iou1(c, box) > lo:
            return c


def away(rs, gts):
    """A box with IoU < 0.2 against every ground truth (sample_anchors' negatives)."""
    while True:
        x1, y1 = rs.uniform(0, 0.8, 2)
        w, h = rs.uniform(0.05, 0.3, 2)
        c = np.array([x1, y1, min(x1 + w, 1.0), min(y1 + h, 1.0)])
        if all(iou1(c, g) < 0.2 for g in gts):
            return c


def make_clip(rs, n_gt, chunks=1, extra_pos=0, negatives=3, gt_itself=False):
    """(targets [n_gt, chunks, 4 + C] float32, anchor tubes [n, T, 4] float64) as ava_cls.py:329-357 makes them."""
    gts = []
    for _ in range(n_gt):
        x1, y1 = rs.uniform(0, 0.6, 2)
        w, h = rs.uniform(0.15, 0.4, 2)
        gts.append(np.array([x1, y1, x1 + w, y1 + h]))
    tg = np.zeros((n_gt, chunks, 4 + C), F)
    for k in range(chunks):
        tg[:, k, :4] = np.array(gts, F) + (rs.uniform(-0.01, 0.01, (n_gt, 4)).astype(F) if k else 0)
    tg[:, :, 4:] = rs.uniform(0, 1, (n_gt, chunks, C)) > 0.9
    tg[:, :, :4] = np.minimum(np.maximum(tg[:, :, :4], 0.0), 1.0) * F(WIDTH)      # scale_tubes_abs on float32
    anchors = []
    for g in gts:
        anchors.append(g.copy() if gt_itself else near(rs, g, 0.75))
        anchors += [near(rs, g, 0.8) for _ in range(extra_pos)]
        anchors += [away(rs, gts) for _ in range(negatives)]
    a = np.tile(np.stack(anchors)[:, None], (1, T, 1))
    a = np.minimum(np.maximum(a, 0.0), 1.0)
    for i in range(4):
        a[:, :, i] *= float(WIDTH if i % 2 == 0 else HEIGHT)
    return tg, a


def reference_rows(ref, targets, tubes):
    """train_cls.py:260-297 with the reference's select_proposals and flatten_tubes; the row building restated."""
    max_chunks = 1
    selected_tubes, target_tubes = [], []
    for b in range(len(targets)):
        cur = tubes[b]
        pos, neg, _ = ref.utils.select_proposals(targets[b][:, int(max_chunks / 2)].reshape(targets[b].shape[0], 1, -1),
                                                 cur[:, int(cur.shape[1] / 2)].reshape(cur.shape[0], 1, -1), None,
                                                 0.75, 5, 'uniform', 3)
        st = np.zeros((len(pos) + len(neg), cur.shape[1], 4), F)
        tt = np.zeros((len(pos) + len(neg), 1, 6 + C), F)
        for row, (ii, jj) in enumerate(pos):
            st[row] = cur[jj]
            tt[row, :, :4] = targets[b][ii, 0, :4]
            tt[row, :, 6:] = targets[b][ii, 0, 4:]
            tt[row, :, 4] = 1
        for row, (ii, jj) in enumerate(neg, start=len(pos)):
            st[row] = cur[jj]
            tt[row, :, 4] = 1
        selected_tubes.append(st)
        target_tubes.append(np.concatenate([tt, tt, tt], axis=1))
    flat_targets, _ = ref.tube_utils.flatten_tubes(target_tubes, batch_idx=False)
    flat_tubes, _ = ref.tube_utils.flatten_tubes(selected_tubes, batch_idx=True)
    return np.asarray(flat_tubes, F), np.asarray(flat_targets, F)


def find_selection(ref, name, ngt, seed0, want=None, **kw):
    for seed in range(seed0, seed0 + 200):
        rs = np.random.RandomState(seed)
        clips = [make_clip(rs, g, **(kw.get("per_clip", [{}] * len(ngt))[b])) for b, g in enumerate(ngt)]
        targets, tubes = [c[0] for c in clips], [c[1] for c in clips]
        np.random.seed(seed + 7); random.seed(seed + 11)
        before = (np.random.get_state(), random.getstate())
        out = reference_rows(ref, targets, tubes)
        after = (np.random.get_state(), random.getstate())
        np.random.set_state(before[0]); random.setstate(before[1])
        mine = osel.train_cls_select(targets, [t.copy() for t in tubes], C)
        same = all(np.array_equal(x, y) for x, y in zip(out, mine))
        if not same or random.getstate() != after[1] or not np.array_equal(np.random.get_state()[1], after[0][1]) \
                or np.random.get_state()[2] != after[0][2]:
            print("  %s: seed %d rejected" % (name, seed))
            continue
        if want is not None and not want(targets, out, before, after):
            continue
        return targets, tubes, out, before, after
    raise RuntimeError("no seed found for " + name)


def positives_above(targets, out, before, after):
    """Some clip has more positives than ground truths: candidates above 0.75 were drawn as extra positives."""
    flat_t, flat_g = out
    clip = (flat_t[:, 0, 0] // T).astype(int)
    pos = flat_g[:, 1, :4].any(1)
    return any(pos[clip == b].sum() > t.shape[0] for b, t in enumerate(targets))


def selection_cases(ref):
    cases = [
        ("b1_one_gt", [1], None, {}),
        ("b4", [2, 4, 1, 3], None, {}),
        ("shuffle_cut", [8, 6], lambda t, o, a, b: a[1] != b[1], {}),
        ("extra_positives", [2, 3], positives_above, {"per_clip": [{"extra_pos": 3}, {"extra_pos": 2}]}),
        ("no_free_negatives", [2, 3], None, {"per_clip": [{"negatives": 0, "gt_itself": True}, {}]}),
        ("chunks3_b4", [1, 5, 2, 7], None, {"per_clip": [{"chunks": 3}] * 4}),
    ]
    rec = {"sel_cases": np.array([c[0] for c in cases])}
    for k, (name, ngt, want, kw) in enumerate(cases):
        targets, tubes, out, before, after = find_selection(ref, name, ngt, 100 * k, want, **kw)
        rec[name + "_nums"] = np.array([t.shape[0] for t in tubes]); rec[name + "_ngt"] = np.array(ngt)
        rec[name + "_targets"] = np.concatenate(targets); rec[name + "_props"] = np.concatenate(tubes)
        rec[name + "_tubes"], rec[name + "_targets_out"] = out
        for tag, (np_state, py_state) in (("", before), ("_after", after)):
            rec[name + "_np_key" + tag] = np_state[1]; rec[name + "_np_pos" + tag] = np.array(np_state[2])
            rec[name + "_py_state" + tag] = np.array(py_state[1], dtype=np.int64)
        print("%-18s rows %d" % (name, out[0].shape[0]))
    return rec


def cls_detection_lines(prob, flat_tubes, nums, keys, label_dict, conf, width, height):
    """train_cls.py:507-543 on numpy arrays: one CSV row per (clip, class, proposal) with score > conf."""
    out, start = [], 0
    for b, n in enumerate(nums):
        p, tb = prob[start:start + n], flat_tubes[start:start + n][:, flat_tubes.shape[1] // 2, 1:]
        start += n
        for cl in range(prob.shape[1]):
            scores = p[:, cl]
            mask = scores > F(conf)
            if not mask.any():
                continue
            boxes = tb[mask].copy()
            boxes[:, ::2] /= width
            boxes[:, 1::2] /= height
            for s, bx in zip(scores[mask], boxes):
                out.append('{0},{1:04},{2:.4},{3:.4},{4:.4},{5:.4},{6},{7:.4}\n'.format(
                    keys[b][0], keys[b][1], bx[0], bx[1], bx[2], bx[3], label_dict[cl], s))
    return out


def validation_case(rs, n_frames, batch, label_dict, width, height, distinct):
    keys = [("val%02d" % (i // 20), 902 + i) for i in range(n_frames)]
    gt_keys, gt_boxes, gt_labels, nums, tubes = [], [], [], [], []
    for key in keys:
        ng = rs.randint(1, 5)
        gts = []
        for _ in range(ng):
            x1, y1 = rs.uniform(0, 0.6, 2)
            w, h = rs.uniform(0.15, 0.4, 2)
            g = np.array([x1, y1, x1 + w, y1 + h])
            gts.append(g)
            for lab in rs.choice(label_dict, rs.randint(1, 3), replace=False):
                gt_keys.append(key); gt_boxes.append(g); gt_labels.append(int(lab))
        anchors = []
        for g in gts:                       # ava_cls.py in val mode: each ground truth, then its negatives
            anchors.append(g)
            anchors += [away(rs, gts) for _ in range(rs.randint(0, 4))]
        a = np.minimum(np.maximum(np.tile(np.stack(anchors)[:, None], (1, T, 1)), 0.0), 1.0)
        for i in range(4):
            a[:, :, i] *= float(width if i % 2 == 0 else height)
        nums.append(a.shape[0])
        tubes.append(a.astype(F))
    R = sum(nums)
    flat = np.zeros((R, T, 5), F)
    start = 0
    for b, t in enumerate(tubes):           # flatten_tubes(batch_idx=True) inside each validation batch
        flat[start:start + t.shape[0], :, 0] = np.arange(T) + (b % batch) * T
        flat[start:start + t.shape[0], :, 1:] = t
        start += t.shape[0]
    if distinct:                            # scores distinct after the 4-digit rounding: 10% above conf
        pool = np.concatenate([np.arange(1001, 10000) / 1e4, np.arange(1001, 10000) / 1e5]).astype(F)
        prob = (rs.uniform(0, 0.0099, (R, C))).astype(F)
        hit = rs.uniform(0, 1, (R, C)) < 0.1
        prob[hit] = rs.permutation(pool)[:int(hit.sum())]
    else:                                   # sigmoid-like scores, some exactly at conf_thresh
        prob = (rs.uniform(0, 1, (R, C)) ** 4).astype(F)
        prob[rs.uniform(0, 1, (R, C)) < 0.01] = F(0.01)
        for b in range(0, len(nums), 37):   # a few clips with no score above conf_thresh
            s = sum(nums[:b])
            prob[s:s + nums[b]] = F(0.005)
    excl = keys[3:n_frames:50]
    return keys, gt_keys, gt_boxes, gt_labels, nums, flat, prob, excl


def validation_cases(rec):
    gap = eval_reference()
    cats, _ = gap.read_labelmap(open(LABELMAP))
    ids = sorted(c["id"] for c in cats)
    label_dict = ids                                   # train_cls.py:43-53 with the 60-class whitelist
    rec["cat_ids"] = np.array([c["id"] for c in cats]); rec["cat_names"] = np.array([c["name"] for c in cats])
    rec["label_dict"] = np.array(label_dict)
    rs = np.random.RandomState(2025)
    cases = [("val_ties", 240, 8, 400, 300, False), ("val_distinct", 40, 4, 400, 400, True)]
    rec["val_cases"] = np.array([c[0] for c in cases])
    conf = 0.01
    for name, n_frames, batch, width, height, distinct in cases:
        keys, gkeys, gboxes, glabels, nums, flat, prob, excl = validation_case(rs, n_frames, batch, label_dict, width, height,
                                                                               distinct)
        dlines = cls_detection_lines(prob, flat, nums, keys, label_dict, conf, width, height)
        glines = oev.gt_lines(gkeys, gboxes, glabels)
        elines = ["%s,%04d\n" % k for k in excl]
        with contextlib.redirect_stdout(io.StringIO()):
            m = gap.run_evaluation(open(LABELMAP), text(glines, "gt.csv"), text(dlines, "det.csv"), text(elines, "excl.csv"))
        index = {c["id"]: c["name"] for c in cats}
        ref = np.array([m["PascalBoxes_PerformanceByCategory/AP@0.5IOU/%s" % index[i + 1]] if i + 1 in index else np.nan
                        for i in range(max(ids))])
        lo, hi = oev.run(cats, glines, dlines, excl).ap_bounds()
        assert np.all((lo <= ref) | np.isnan(ref)) and np.all((ref <= hi) | np.isnan(ref)), name
        exact = int(np.sum((lo == hi) & ~np.isnan(ref)))
        print("%-14s rows %6d, gt %4d, classes tie-free %d of %d, mAP %.6f" % (
            name, len(dlines), len(glines), exact, int((~np.isnan(ref)).sum()), m["PascalBoxes_Precision/mAP@0.5IOU"]))
        rec[name + "_prob"], rec[name + "_tubes"], rec[name + "_nums"] = prob, flat, np.array(nums)
        rec[name + "_batches"] = np.array([min(batch, n_frames - i) for i in range(0, n_frames, batch)])
        rec[name + "_video"] = np.array([k[0] for k in keys]); rec[name + "_fid"] = np.array([k[1] for k in keys])
        rec[name + "_gt_video"] = np.array([k[0] for k in gkeys]); rec[name + "_gt_fid"] = np.array([k[1] for k in gkeys])
        rec[name + "_gt_boxes"] = np.array(gboxes, np.float64); rec[name + "_gt_labels"] = np.array(glabels)
        rec[name + "_excl_video"] = np.array([k[0] for k in excl]); rec[name + "_excl_fid"] = np.array([k[1] for k in excl])
        rec[name + "_width"], rec[name + "_height"], rec[name + "_conf"] = np.int64(width), np.int64(height), np.float64(conf)
        rec[name + "_rows"] = np.int64(len(dlines))
        rec[name + "_ref_ap"], rec[name + "_ref_map"] = ref, np.float64(m["PascalBoxes_Precision/mAP@0.5IOU"])
        rec[name + "_ap_lo"], rec[name + "_ap_hi"] = lo, hi


def main():
    assert refload.available(), "reference checkout not present"
    ref = refload.load()
    rec = {"numpy_version": np.array(np.__version__)}
    rec.update(selection_cases(ref))
    validation_cases(rec)
    np.savez_compressed(OUT, **rec)
    print("wrote %s (%.2f MB)" % (OUT, os.path.getsize(OUT) / 1e6))


if __name__ == "__main__":
    main()
