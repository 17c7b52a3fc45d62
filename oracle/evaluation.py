"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the frame-mAP of test.py:110-226 / train.py::validate: the CSV rows
those drivers write, read back as get_ava_performance.read_csv reads them, and run_evaluation's PascalDetectionEvaluator
(object_detection_evaluation.py, per_image_evaluation.py, np_box_ops.iou, metrics.py) at IoU 0.5.

Steps, each as the reference performs it:
1. CSV rounding: every box coordinate and score is written with '{:.4}' and parsed with float(); rows of label ids
   outside the label map are dropped; the image key is make_image_key(video, int(fid)); boxes are kept as [y1, x1, y2, x2].
2. Exclusions: excluded keys are dropped from both files.  Rows of one key merge in row order.
3. Per image, in the order of each key's first detection row: invalid boxes (y1 >= y2 or x1 >= x2) dropped; per class
   the scores > -10, sorted descending, the first 10,000; np_box_ops.iou in float64; greedy matching (the first maximum
   of each IoU row, a NaN counting as the maximum, TP when >= 0.5 and the ground truth is not taken yet).
4. Ground-truth instances counted per class (label id - 1) over max(id) classes.
5. Per class: the per-image (score, TP) arrays concatenated in image order, sorted descending; precision, recall, the
   precision made non-increasing, the sum over recall changes; AP 0.0 with ground truth and no detection, NaN without
   ground truth; mAP = np.nanmean over the classes.

Tie contract, which the device (step_b200.evaluation, eval.cu) follows too: every descending sort is a stable ascending
argsort reversed (equal scores: the later element first).  numpy's default argsort orders equal values its own way
(differently on AVX-512 CPUs), so:
- the result is the reference's bit for bit whenever no group of equal scores of one class mixes TPs and FPs (within one
  image and class the multiset of (score, TP) pairs does not depend on the order of equal scores, except for a tie at
  the 10,000-row cut);
- otherwise the reference's AP of the class lies in [ap_bounds lo, hi]: FPs first in every mixed group, TPs first.
The pairwise summation of np.sum is `pairwise_sum` (numpy 2's order), which the device reproduces.

Pinned by tests/golden/eval_cases.npz (metrics of the reference's own run_evaluation, tests/golden/make_eval_golden.py).
"""
import csv
from collections import OrderedDict

import numpy as np

MAX_PER_IMAGE_CLASS = 10000   # np_box_list_ops.non_max_suppression's max_output_size
IOU = 0.5


def csv_round(v):
    """'{:.4}' then float(): what a CSV field of the drivers parses back to."""
    return float(format(float(v), ".4"))


def make_image_key(video, ts):
    return "%s,%04d" % (video, int(ts))


# ---- the CSV text the drivers write ----
def detection_lines(clips, keys, label_dict):
    """test.py:210-218: clips = postprocess.to_lists(...) (per clip [(box[4], class index, score)]), keys = (video, fid)
    per clip."""
    out = []
    for (video, fid), rows in zip(keys, clips):
        for box, cl, s in rows:
            out.append('{0},{1:04},{2:.4},{3:.4},{4:.4},{5:.4},{6},{7:.4}\n'.format(video, fid, box[0], box[1], box[2], box[3],
                                                                                      label_dict[cl], s))
    return out


def gt_lines(keys, boxes, labels):
    """test.py:129-139: one row per (box, label); keys = (video, fid) per row."""
    return ['{0},{1:04},{2:.4},{3:.4},{4:.4},{5:.4},{6}\n'.format(v, f, b[0], b[1], b[2], b[3], int(l))
            for (v, f), b, l in zip(keys, boxes, labels)]


def read_csv(lines, whitelist):
    """get_ava_performance.read_csv over text lines: key -> [y1, x1, y2, x2] rows, label ids, scores (1.0 without)."""
    boxes, labels, scores = OrderedDict(), OrderedDict(), OrderedDict()
    for row in csv.reader(lines):
        key = make_image_key(row[0], row[1])
        x1, y1, x2, y2 = [float(n) for n in row[2:6]]
        action = int(row[6])
        if whitelist and action not in whitelist:
            continue
        score = float(row[7]) if len(row) == 8 else 1.0
        boxes.setdefault(key, []).append([y1, x1, y2, x2])
        labels.setdefault(key, []).append(action)
        scores.setdefault(key, []).append(score)
    return boxes, labels, scores


# ---- the evaluator ----
def desc(x):
    """np.argsort(x)[::-1] under the tie contract."""
    return np.argsort(x, kind="stable")[::-1]


def iou(b1, b2):
    """np_box_ops.iou, float64, its operations in its order."""
    y_min1, x_min1, y_max1, x_max1 = np.split(b1, 4, axis=1)
    y_min2, x_min2, y_max2, x_max2 = np.split(b2, 4, axis=1)
    min_ymax = np.minimum(y_max1, np.transpose(y_max2))
    max_ymin = np.maximum(y_min1, np.transpose(y_min2))
    ih = np.maximum(np.zeros(max_ymin.shape), min_ymax - max_ymin)
    min_xmax = np.minimum(x_max1, np.transpose(x_max2))
    max_xmin = np.maximum(x_min1, np.transpose(x_min2))
    iw = np.maximum(np.zeros(max_xmin.shape), min_xmax - max_xmin)
    inter = ih * iw
    a1 = (b1[:, 2] - b1[:, 0]) * (b1[:, 3] - b1[:, 1])
    a2 = (b2[:, 2] - b2[:, 0]) * (b2[:, 3] - b2[:, 1])
    with np.errstate(invalid="ignore", divide="ignore"):
        return inter / (np.expand_dims(a1, 1) + np.expand_dims(a2, 0) - inter)


def per_image(boxes, scores, labels, gt_boxes, gt_labels):
    """compute_object_detection_metrics: {class index: (scores, TP flags)} of one image (labels 0-based)."""
    valid = np.logical_and(boxes[:, 0] < boxes[:, 2], boxes[:, 1] < boxes[:, 3])
    boxes, scores, labels = boxes[valid], scores[valid], labels[valid]
    out = {}
    for c in np.unique(labels):
        sel = labels == c
        b, s = boxes[sel], scores[sel]
        keep = np.greater(s, -10.0)
        b, s = b[keep], s[keep]
        if s.size == 0:
            continue
        order = desc(s)[:MAX_PER_IMAGE_CLASS]
        b, s = b[order], s[order]
        g = gt_boxes[gt_labels == c]
        tp = np.zeros(s.size, dtype=bool)
        if g.size:
            ov = iou(b, g)
            best = np.argmax(ov, axis=1)
            taken = np.zeros(g.shape[0], dtype=bool)
            for i in range(s.size):
                j = best[i]
                if ov[i, j] >= IOU and not taken[j]:
                    tp[i] = taken[j] = True
        out[int(c)] = (s, tp)
    return out


def pairwise_sum(a):
    """np.sum of a contiguous float64 array in numpy's order: from 0.0; n < 8 in order; n <= 128 eight partial sums
    ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the remainder in order; above, the halves split at n//2 - (n//2) % 8."""
    def pw(lo, n):
        if n < 8:
            r = 0.0
            for i in range(lo, lo + n):
                r += a[i]
            return r
        if n <= 128:
            r = [float(a[lo + j]) for j in range(8)]
            i = 8
            while i < n - n % 8:
                for j in range(8):
                    r[j] += a[lo + i + j]
                i += 8
            res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
            for k in range(i, n):
                res += a[lo + k]
            return res
        n2 = n // 2
        n2 -= n2 % 8
        return pw(lo, n2) + pw(lo + n2, n - n2)
    a = [float(v) for v in np.asarray(a, dtype=np.float64)]
    return 0.0 + pw(0, len(a))


def average_precision(tp_sorted, num_gt):
    """compute_precision_recall + compute_average_precision of TP flags already in the class order."""
    if tp_sorted.size == 0:
        return 0.0
    t = tp_sorted.astype(int)
    cum_tp, cum_fp = np.cumsum(t), np.cumsum(1 - t)
    precision = cum_tp.astype(float) / (cum_tp + cum_fp)
    recall = cum_tp.astype(float) / num_gt
    recall = np.concatenate([[0], recall, [1]])
    precision = np.concatenate([[0], precision, [0]])
    precision = np.maximum.accumulate(precision[::-1])[::-1]
    idx = np.where(recall[1:] != recall[:-1])[0] + 1
    return np.sum((recall[idx] - recall[idx - 1]) * precision[idx])


class Evaluation:
    """run_evaluation over parsed rows: per-class scores / TP flags, ground-truth counts, and the APs."""

    def __init__(self, categories, gt, det, excluded=()):
        self.n_classes = max(c["id"] for c in categories)
        excluded = set(excluded)
        gboxes, glabels, _ = gt
        self.num_gt = np.zeros(self.n_classes, dtype=int)
        gt_img = {}
        for key in gboxes:
            if key in excluded:
                continue
            b = np.array(gboxes[key], dtype=float)
            l = np.array(glabels[key], dtype=int) - 1
            gt_img[key] = (b, l)
            for c in range(self.n_classes):
                self.num_gt[c] += np.sum(l == c)
        dboxes, dlabels, dscores = det
        self.scores = [[] for _ in range(self.n_classes)]
        self.tps = [[] for _ in range(self.n_classes)]
        empty = (np.zeros((0, 4)), np.zeros(0, dtype=int))
        for key in dboxes:
            if key in excluded:
                continue
            gb, gl = gt_img.get(key, empty)
            res = per_image(np.array(dboxes[key], dtype=float), np.array(dscores[key], dtype=float),
                            np.array(dlabels[key], dtype=int) - 1, gb, gl)
            for c, (s, tp) in res.items():
                if 0 <= c < self.n_classes:
                    self.scores[c].append(s)
                    self.tps[c].append(tp)

    def _ap(self, order_fn):
        ap = np.full(self.n_classes, np.nan)
        for c in range(self.n_classes):
            if self.num_gt[c] == 0:
                continue
            if not self.scores[c]:
                ap[c] = 0.0
                continue
            s, tp = np.concatenate(self.scores[c]), np.concatenate(self.tps[c])
            ap[c] = average_precision(tp[order_fn(s, tp)], self.num_gt[c])
        return ap

    def per_class_ap(self):
        return self._ap(lambda s, tp: desc(s))

    def ap_bounds(self):
        """(lo, hi): every mixed tie group of a class with its FPs first, with its TPs first."""
        lo = self._ap(lambda s, tp: np.lexsort((tp.astype(int), -s)))
        hi = self._ap(lambda s, tp: np.lexsort((-tp.astype(int), -s)))
        return lo, hi


def run(categories, gt_text, det_text, exclusions=()):
    """Evaluation of CSV text lines (gt_text, det_text) as run_evaluation reads them; exclusions = (video, fid) pairs."""
    whitelist = set(c["id"] for c in categories)
    excluded = {make_image_key(v, f) for v, f in exclusions}
    return Evaluation(categories, read_csv(gt_text, whitelist), read_csv(det_text, whitelist), excluded)


def metrics(categories, per_class):
    """PascalDetectionEvaluator.evaluate's dict."""
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        out = {"PascalBoxes_Precision/mAP@0.5IOU": np.nanmean(per_class)}
    index = {c["id"]: c for c in categories}
    for idx in range(per_class.size):
        if idx + 1 in index:
            out["PascalBoxes_PerformanceByCategory/AP@0.5IOU/%s" % index[idx + 1]["name"]] = per_class[idx]
    return out
