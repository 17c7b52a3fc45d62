"""`FrameAP` -- frame-mAP on the device: what test.py:110-226 and train.py::validate compute by writing the detections and
the ground truth to CSV files and calling utils/eval_utils.ava_evaluation (get_ava_performance.run_evaluation, the AVA
Pascal evaluator at IoU 0.5), without writing or parsing the files.

    ev = FrameAP(categories, label_dict, exclusions)        # one per refinement step
    for each batch:
        ev.add_ground_truth(keys, boxes, labels)             # the rows test.py:129-139 writes to testing_gt.csv
        ev.add_detections(detector.run(prob, loc), keys)     # the rows test.py:210-218 writes, one key per clip
    metrics = ev.evaluate()                                  # run_evaluation's metrics dict

`add_detections` launches one kernel (step_eval_append, eval.cu) per 64 clips and does not synchronise: the rows are
rounded as the CSV round trip rounds them ('{:.4}' then float()) and appended to a device store.  The store grows when
the next call's worst case (clips x detector capacity) might not fit; only then does the call wait, for the row counter
of the previous call.  `evaluate` uploads the ground truth, runs step_eval_run and reads back the per-class APs.

Ties: every descending sort of the evaluator is a stable ascending argsort reversed, as in select.py.  The result is the
reference's bit for bit unless a group of equal scores of one class mixes true and false positives; then the reference's
AP of that class lies between the AP with the true positives of every such group first and the one with them last
(README.md).
"""
import ctypes

import numpy as np
import torch

from . import _lib as L

INT32_MAX = 2 ** 31 - 1
# the structs' names before they were read from the header
EvalRows, EvalAppendParams, EvalParams = L.step_eval_rows, L.step_eval_append_params, L.step_eval_params


def image_key(key):
    """get_ava_performance.make_image_key: (video_name, timestamp) -> "video_name,%04d"; a "video_name,timestamp"
    string is read the same way."""
    if isinstance(key, str):
        video, _, ts = key.rpartition(",")
        return "%s,%04d" % (video, int(ts))
    video, ts = key
    return "%s,%04d" % (video, int(ts))


def csv_round(v):
    """The value a '{:.4}'-formatted CSV field parses back to."""
    return float(format(float(v), ".4"))


def _ptr(t):
    return t.data_ptr() if t is not None else None


class FrameAP:
    """Frame-mAP of one detection set (one refinement step) against the ground truth, as run_evaluation computes it.

    categories: read_labelmap's list of {"id", "name"} (label ids, 1-based; the largest id is the class count).
    label_dict: detector class index -> label id (args.label_dict); rows of a label id outside `categories` are dropped.
    exclusions: image keys dropped from the ground truth and the detections (ava_val_excluded_timestamps).
    device: where the detections live (default: the current CUDA device)."""

    def __init__(self, categories, label_dict, exclusions=(), device=None):
        self.categories = [{"id": int(c["id"]), "name": c["name"]} for c in categories]
        if not self.categories:
            raise ValueError("FrameAP: no categories")
        ids = [c["id"] for c in self.categories]
        if min(ids) < 1:
            raise ValueError("FrameAP: category ids must be 1-based (got %d)" % min(ids))
        self.n_classes = max(ids)
        if self.n_classes > L.EVAL_MAX_CLASSES:
            raise ValueError("FrameAP: largest category id %d exceeds %d" % (self.n_classes, L.EVAL_MAX_CLASSES))
        self.whitelist = set(ids)
        if isinstance(label_dict, dict):
            table = [int(label_dict.get(c, 0)) for c in range(max(label_dict) + 1)] if label_dict else []
        else:
            table = [int(v) for v in label_dict]
        if not table:
            raise ValueError("FrameAP: empty label_dict")
        self.class_of = [v - 1 if v in self.whitelist else -1 for v in table]
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if self.device.type != "cuda":
            raise RuntimeError("FrameAP: the evaluator runs on a CUDA device, got %s" % self.device)
        self._class_of = torch.tensor(self.class_of, dtype=torch.int32, device=self.device)
        self.excluded = {image_key(k) for k in exclusions}
        self.per_class_ap = None
        self.reset()

    def reset(self):
        """Forget every ground-truth and detection row."""
        dev = self.device
        self._ids = {}
        self._gt = []
        self._counters = torch.zeros(2, dtype=torch.int32, device=dev)
        self._img_first = torch.full((L.EVAL_MAX_IMAGES,), INT32_MAX, dtype=torch.int32, device=dev)
        self._cap = 0
        self._box = self._score = self._scode = self._img = self._cls = None
        self._host_counters = torch.zeros(2, dtype=torch.int32).pin_memory()
        self._event = None
        self._kept = 0            # rows kept, exact as of the last counter read
        self._kept_bound = 0      # rows kept, an upper bound including the calls since
        self._read_bound = 0      # rows read (kept or not), an upper bound

    # ---- the row store ----
    def _rows(self):
        return L.step_eval_rows(capacity=self._cap, counters=_ptr(self._counters), img_first=_ptr(self._img_first),
                                box=_ptr(self._box), score=_ptr(self._score), scode=_ptr(self._scode), img=_ptr(self._img),
                                cls=_ptr(self._cls))

    def _refresh(self):
        """Exact counters from the copy the last add_detections queued (waits for it only if it has not landed)."""
        if self._event is not None:
            if not self._event.query():
                self._event.synchronize()
            self._kept = self._kept_bound = int(self._host_counters[0])
            self._read_bound = int(self._host_counters[1])

    def reserve(self, rows):
        """Make room for `rows` detection rows in all, so that no later add_detections has to grow the store."""
        rows = int(rows)
        if rows > L.EVAL_MAX_ROWS:
            raise ValueError("FrameAP: %d rows exceed the %d the store holds" % (rows, L.EVAL_MAX_ROWS))
        if rows <= self._cap:
            return
        self._refresh()
        dev, n = self.device, self._kept
        box = torch.empty((rows, 4), dtype=torch.float64, device=dev)
        score = torch.empty((rows,), dtype=torch.float64, device=dev)
        ints = [torch.empty((rows,), dtype=torch.int32, device=dev) for _ in range(3)]
        if n:
            box[:n].copy_(self._box[:n])
            score[:n].copy_(self._score[:n])
            for new, old in zip(ints, (self._scode, self._img, self._cls)):
                new[:n].copy_(old[:n])
        self._box, self._score, (self._scode, self._img, self._cls) = box, score, ints
        self._cap = rows

    def _make_room(self, worst):
        if self._kept_bound + worst <= self._cap and self._read_bound + worst <= L.EVAL_MAX_ROWS:
            return
        self._refresh()
        if self._read_bound + worst > L.EVAL_MAX_ROWS:
            raise ValueError("FrameAP: %d + %d detection rows exceed the %d rows an evaluation reads"
                             % (self._read_bound, worst, L.EVAL_MAX_ROWS))
        if self._kept_bound + worst > self._cap:
            self.reserve(min(L.EVAL_MAX_ROWS, max(2 * self._cap, self._kept_bound + worst, 1 << 20)))

    def _image_id(self, key):
        k = image_key(key)
        if k in self.excluded:
            return -1
        i = self._ids.get(k)
        if i is None:
            i = self._ids[k] = len(self._ids)
        return i

    # ---- input ----
    def add_ground_truth(self, keys, boxes, labels):
        """Ground-truth rows as the GT CSV carries them: one image key per row, boxes [n, 4] (x1, y1, x2, y2, normalised)
        and label ids.  Rows of one key merge in the order they are given, across calls too."""
        boxes = np.asarray(boxes).reshape(-1, 4)
        labels = np.asarray(labels).reshape(-1)
        if len(keys) != boxes.shape[0] or labels.shape[0] != boxes.shape[0]:
            raise ValueError("FrameAP: %d keys, %d boxes and %d labels" % (len(keys), boxes.shape[0], labels.shape[0]))
        rows = []
        for key, box, lab in zip(keys, boxes, labels):
            lab = int(lab)
            if lab not in self.whitelist:
                continue
            i = self._image_id(key)
            if i < 0:
                continue
            x1, y1, x2, y2 = (csv_round(v) for v in box)
            rows.append((i, lab - 1, y1, x1, y2, x2))
        if rows:
            self._gt.append(np.array(rows, dtype=np.float64))

    def add_detections(self, det, keys):
        """det: a Detector.run / detect result (det [B, cap, 8], count [B] on the device); keys: one image key per clip.
        Launches only, unless the store has to grow."""
        d, cnt = det["det"], det["count"]
        B = len(keys)
        L.need_cuda(d, cnt)
        if d.dtype != torch.float32 or d.dim() != 3 or d.shape[2] != 8 or not d.is_contiguous() or d.shape[0] < B:
            raise ValueError("FrameAP: det must be a contiguous float32 [B >= %d, cap, 8] tensor, got %s %s"
                             % (B, d.dtype, tuple(d.shape)))
        if cnt.dtype != torch.int32 or cnt.dim() != 1 or cnt.shape[0] < B or not cnt.is_contiguous():
            raise ValueError("FrameAP: count must be a contiguous int32 [B >= %d] tensor, got %s %s" % (B, cnt.dtype, tuple(cnt.shape)))
        if "tubes_nums" in det and len(det["tubes_nums"]) != B:
            raise ValueError("FrameAP: %d keys for %d clips" % (B, len(det["tubes_nums"])))
        if d.device != self.device or cnt.device != self.device:
            raise RuntimeError("FrameAP: detections on %s, evaluator on %s" % (d.device, self.device))
        if B == 0:
            return
        cap = d.shape[1]
        ids = [self._image_id(k) for k in keys]
        self._make_room(B * cap)
        with torch.cuda.device(self.device):
            stream = L.stream()
            for b0 in range(0, B, L.EVAL_MAX_CLIPS):
                nb = min(L.EVAL_MAX_CLIPS, B - b0)
                p = L.step_eval_append_params(det=d.data_ptr() + b0 * cap * 8 * 4, count=cnt.data_ptr() + b0 * 4, B=nb,
                                              cap=cap, ncls=len(self.class_of), class_of=self._class_of.data_ptr(),
                                              rows=self._rows())
                p.img[:nb] = ids[b0:b0 + nb]
                L.check(L.lib().step_eval_append(ctypes.byref(p), stream))
            self._host_counters.copy_(self._counters, non_blocking=True)
            if self._event is None:
                self._event = torch.cuda.Event()
            self._event.record()
        self._kept_bound += B * cap
        self._read_bound += B * cap

    # ---- result ----
    def _ground_truth(self, n_images):
        g = np.concatenate(self._gt) if self._gt else np.zeros((0, 6))
        img, cls = g[:, 0].astype(np.int64), g[:, 1].astype(np.int64)
        order = np.lexsort((cls, img))                  # by image, then class; row order within (lexsort is stable)
        img, cls, box = img[order], cls[order], np.ascontiguousarray(g[order, 2:6])
        off = np.searchsorted(img, np.arange(n_images + 1)).astype(np.int32)
        num_gt = np.bincount(cls, minlength=self.n_classes).astype(np.int32)
        return box, cls.astype(np.int32), off, num_gt

    def evaluate(self):
        """The metrics dict of run_evaluation: 'PascalBoxes_Precision/mAP@0.5IOU' and one
        'PascalBoxes_PerformanceByCategory/AP@0.5IOU/<name>' per category.  The 80 (n_classes) per-class APs, NaN for a
        class without ground truth, are left in `self.per_class_ap`."""
        dev = self.device
        n_kept, _ = (int(v) for v in self._counters.cpu())
        if n_kept > self._cap:
            raise RuntimeError("FrameAP: %d rows kept in a store of %d" % (n_kept, self._cap))
        n_images = len(self._ids)
        box, cls, off, num_gt = self._ground_truth(n_images)
        max_gt = int(np.diff(off).max()) if n_images else 0
        t = {k: torch.from_numpy(v).to(dev) for k, v in
             (("box", box), ("cls", cls), ("off", off), ("num_gt", num_gt))}
        ws_bytes = L.lib().step_eval_workspace_bytes(n_kept, self.n_classes, box.shape[0])
        p = L.step_eval_params(rows=self._rows(), n_rows=n_kept, n_classes=self.n_classes, n_images=n_images,
                               n_gt=box.shape[0], max_gt_per_image=max_gt, gt_box=_ptr(t["box"]) if box.shape[0] else None,
                               gt_cls=_ptr(t["cls"]) if box.shape[0] else None, gt_img_off=_ptr(t["off"]),
                               num_gt=_ptr(t["num_gt"]), workspace_bytes=ws_bytes)
        ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
        ap = torch.empty((self.n_classes,), dtype=torch.float64, device=dev)
        p.workspace, p.ap = ws.data_ptr(), ap.data_ptr()
        with torch.cuda.device(dev):
            L.check(L.lib().step_eval_run(ctypes.byref(p), L.stream()))   # checks every field before its first launch
            ap_host = ap.cpu().numpy()
        self.per_class_ap = ap_host
        return metrics_dict(self.categories, ap_host)


def metrics_dict(categories, per_class_ap):
    """PascalDetectionEvaluator.evaluate's dict from the per-class APs (mAP: np.nanmean over every class)."""
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)   # every class without ground truth: nanmean is NaN
        mean_ap = np.nanmean(per_class_ap)
    out = {"PascalBoxes_Precision/mAP@0.5IOU": mean_ap}
    index = {c["id"]: c for c in categories}
    for idx in range(per_class_ap.size):
        if idx + 1 in index:
            out["PascalBoxes_PerformanceByCategory/AP@0.5IOU/%s" % index[idx + 1]["name"]] = per_class_ap[idx]
    return out
