"""Detection post-processing on the device: the per-clip x per-class loop of the reference drivers
(test.py:156-218, demo.py:140-174 -- B*60*max_iter tiny CPU NMS calls per batch) as TWO launches of libstep_b200
(`step_detect_f32`), with no torch arithmetic, no gather tensors and no synchronisation: CUDA-graph capturable.

For every (clip, class): keep tubes whose centre-frame score > conf_thresh, clamp their centre-frame box
with valid_tubes (the drivers call it with its 400x400 defaults, test.py:191), run greedy NMS
(cpu/nms_cpu.cpp semantics, bit-exact), normalise by (width, height), then per clip either every survivor in
file order or the top-k scores in the order of the reference's tuple sort (test.py:205-208).

demo.py then merges the overlapping detections across classes (demo.py:176-198): `Merger` does that on the device in
three more launches (`step_detect_merge_f32`), and `merged_results` / `result_lines` turn one read-back of its result
into the reference's `merged_result` dicts and results.txt lines (demo.py:200-217).
"""
import numpy as np
import torch

from . import _lib as L

_plan_cache = {}


def _plan(tubes_nums, device):
    """clip_offsets [B+1] int32 on the device (one small H2D per distinct batch shape, cached)."""
    key = (tuple(int(n) for n in tubes_nums), str(device))
    p = _plan_cache.get(key)
    if p is None:
        offs = np.concatenate([[0], np.cumsum(np.asarray(tubes_nums, np.int64))]).astype(np.int32)
        p = torch.from_numpy(offs).to(device)
        _plan_cache[key] = p
    return p


class Detector:
    """Pre-allocated outputs for one batch shape, so `run` only launches (what StepRunner captures)."""

    def __init__(self, tubes_nums, num_classes, device, conf_thresh, nms_thresh, width, height, topk=0,
                 valid_size=(400, 400), ge=True):
        self.nums = [int(n) for n in tubes_nums]
        self.B, self.R, self.ncls = len(self.nums), int(sum(self.nums)), int(num_classes)
        self.max_n = max(self.nums) if self.nums else 0
        if self.max_n > L.lib().step_nms_segmented_max_rows():
            raise RuntimeError("detect: %d tubes in one clip exceed the %d-row per-(clip, class) NMS problem"
                               % (self.max_n, L.lib().step_nms_segmented_max_rows()))
        self.conf, self.thr, self.topk, self.ge = float(conf_thresh), float(nms_thresh), int(topk or 0), bool(ge)
        self.w, self.h, self.valid = float(width), float(height), (float(valid_size[0]), float(valid_size[1]))
        self.cap = max(1, min(self.topk, self.max_n * self.ncls) if self.topk > 0 else self.max_n * self.ncls)
        self.offs = _plan(self.nums, device)
        n_cand = max(1, self.R * self.ncls)
        self.keep = torch.zeros((n_cand,), dtype=torch.uint8, device=device)
        self.score = torch.zeros((n_cand,), dtype=torch.float32, device=device)
        self.box = torch.zeros((n_cand, 4), dtype=torch.float32, device=device)
        self.det = torch.zeros((max(self.B, 1), self.cap, 8), dtype=torch.float32, device=device)
        self.count = torch.zeros((max(self.B, 1),), dtype=torch.int32, device=device)

    def run(self, pred_prob, pred_loc):
        """pred_prob [R,T,cls] (any strides, e.g. the expand view `inference` returns) | [R,cls]; pred_loc [R,T,4]."""
        L.need_cuda(pred_prob, pred_loc)
        prob = pred_prob[:, pred_prob.shape[1] // 2] if pred_prob.dim() == 3 else pred_prob   # test.py:158-159
        if prob.dtype != torch.float32 or prob.stride(1) != 1:
            prob = prob.float().contiguous()
        if pred_loc.dtype != torch.float32 or not pred_loc.is_contiguous():
            pred_loc = pred_loc.float().contiguous()
        if prob.shape[0] != self.R or prob.shape[1] != self.ncls:
            raise RuntimeError("detect: expected %d x %d scores, got %s" % (self.R, self.ncls, tuple(prob.shape)))
        T = pred_loc.shape[1]
        mid = pred_loc[:, T // 2]                                                                # test.py:160-161 (view)
        if self.R and self.B:
            with torch.cuda.device(prob.device):
                L.check(L.lib().step_detect_f32(L.ptr(prob), prob.stride(0), L.c_void_p(mid.data_ptr()), pred_loc.stride(0),
                                                L.ptr(self.offs), self.B, self.R, self.max_n, self.ncls, self.conf, self.thr,
                                                1 if self.ge else 0, self.valid[0], self.valid[1], self.w, self.h, self.topk,
                                                self.cap, L.ptr(self.keep), L.ptr(self.score), L.ptr(self.box),
                                                L.ptr(self.det), L.ptr(self.count), L.stream(prob.device)))
        return {"det": self.det, "count": self.count, "keep": self.keep, "score": self.score, "box": self.box,
                "tubes_nums": self.nums}


class ClsDetector:
    """The class-only detections of the classification pre-training stage's validation (train_cls.py:505-543) in one
    launch of `step_detect_scores_f32`: for every clip, class and proposal (the reference's file order), the proposal's
    score when it is > conf_thresh, with its centre-frame box divided by (width, height) in float32.  No valid_tubes clamp,
    no NMS, no top-k.  The result has Detector.run's layout, so FrameAP.add_detections takes it; `run` only launches
    (no allocation for float32 inputs, no synchronisation), so it can be captured in a CUDA graph."""

    def __init__(self, tubes_nums, num_classes, device, conf_thresh, width, height):
        self.nums = [int(n) for n in tubes_nums]
        self.B, self.R, self.ncls = len(self.nums), int(sum(self.nums)), int(num_classes)
        self.max_n = max(self.nums) if self.nums else 0
        self.conf, self.w, self.h = float(conf_thresh), float(width), float(height)
        self.cap = max(1, self.max_n * self.ncls)       # every row of a clip fits: nothing is cut
        self.offs = _plan(self.nums, device)
        self.det = torch.zeros((max(self.B, 1), self.cap, 8), dtype=torch.float32, device=device)
        self.count = torch.zeros((max(self.B, 1),), dtype=torch.int32, device=device)

    def run(self, global_prob, flat_tubes):
        """global_prob [R, cls] (the class-only head's output; any row stride), flat_tubes [R, T, 5] (frame index first)."""
        L.need_cuda(global_prob, flat_tubes)
        prob = global_prob
        if prob.dtype != torch.float32 or prob.dim() != 2 or prob.stride(1) != 1:
            prob = prob.float().reshape(prob.shape[0], -1).contiguous()
        if flat_tubes.dtype != torch.float32 or not flat_tubes.is_contiguous():
            flat_tubes = flat_tubes.float().contiguous()
        if prob.shape[0] != self.R or prob.shape[1] != self.ncls:
            raise RuntimeError("detect_scores: expected %d x %d scores, got %s" % (self.R, self.ncls, tuple(global_prob.shape)))
        if flat_tubes.dim() != 3 or flat_tubes.shape[0] != self.R or flat_tubes.shape[2] != 5:
            raise RuntimeError("detect_scores: expected [%d, T, 5] tubes, got %s" % (self.R, tuple(flat_tubes.shape)))
        T = flat_tubes.shape[1]
        box = flat_tubes.data_ptr() + ((T // 2) * 5 + 1) * 4                        # flat_tubes[:, T // 2, 1:5]
        if self.R and self.B:
            with torch.cuda.device(prob.device):
                L.check(L.lib().step_detect_scores_f32(L.ptr(prob), prob.stride(0), L.c_void_p(box), flat_tubes.stride(0),
                                                       L.ptr(self.offs), self.B, self.R, self.max_n, self.ncls, self.conf,
                                                       self.w, self.h, self.cap, L.ptr(self.det), L.ptr(self.count),
                                                       L.stream(prob.device)))
        return {"det": self.det, "count": self.count, "tubes_nums": self.nums}


def detect(pred_prob, pred_loc, tubes_nums, conf_thresh, nms_thresh, width, height, topk=0, valid_size=(400, 400)):
    """pred_prob [R,T,cls] | [R,cls], pred_loc [R,T,4] (history[i] of `inference`), all on the device.
    Returns device tensors, no synchronisation:
      det [B, cap, 8] = (x1, y1, x2, y2 normalised, score, class, tube-in-clip, 0) and count [B] -- the kept detections
      of every clip in the reference's order (file order, or best score first when topk > 0);
      keep / score / box over the R*cls candidate rows (clip-major, class, tube)."""
    ncls = pred_prob.shape[-1]
    d = Detector(tubes_nums, ncls, pred_prob.device, conf_thresh, nms_thresh, width, height, topk, valid_size)
    return d.run(pred_prob, pred_loc)


def to_lists(det, n_clips=None):
    """Materialise (one D2H of the compact result) as per-clip lists of (box[4], cls, score), reference order."""
    cnt = det["count"].cpu().numpy()
    rows = det["det"].cpu().numpy()
    out = []
    for b in range(len(det["tubes_nums"]) if n_clips is None else n_clips):
        out.append([(rows[b, k, :4].copy(), int(rows[b, k, 5]), float(rows[b, k, 4])) for k in range(int(cnt[b]))])
    return out


class Merger:
    """The cross-class merge of demo.py:176-198 on a Detector's rows, with pre-allocated outputs, so `run` only launches
    (what StepRunner captures).  Per clip, a row not yet taken leads a group and takes every later row not yet taken whose
    compute_box_iou with it is > global_thresh (float32); each group's box is its members' np.mean.  run(det) returns
      mbox [B, cap, 4]   the merged boxes in the order of the reference's dict;
      pairs [B, cap, 2]  int32 (det row, key index) in the order results.txt lists them;
      count [B, 2]       int32 (keys, pairs) of each clip."""

    def __init__(self, detector, global_thresh):
        self.detector = detector
        self.B, self.cap, self.thr = detector.B, detector.cap, float(global_thresh)
        if self.cap > L.lib().step_detect_merge_max_rows():
            raise RuntimeError("merge: %d rows per clip exceed the %d-row merge" % (self.cap, L.lib().step_detect_merge_max_rows()))
        dev, nb = detector.det.device, max(self.B, 1)
        self.mbox = torch.zeros((nb, self.cap, 4), dtype=torch.float32, device=dev)
        self.pairs = torch.zeros((nb, self.cap, 2), dtype=torch.int32, device=dev)
        self.count = torch.zeros((nb, 2), dtype=torch.int32, device=dev)
        self.ws = torch.empty((L.lib().step_detect_merge_workspace_bytes(self.B, self.cap),), dtype=torch.uint8, device=dev)
        # host mirrors of the outputs and of the detector's rows: the materialisers read them back with one synchronisation
        self.host = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
                     for t in (self.mbox, self.pairs, self.count, detector.det)]

    def run(self, det):
        """det: the dict Detector.run returned (its det / count are read in place)."""
        d, c = det["det"], det["count"]
        if d.data_ptr() != self.detector.det.data_ptr() or c.data_ptr() != self.detector.count.data_ptr():
            raise RuntimeError("merge: det is not the result of this Merger's Detector")
        if self.B:
            with torch.cuda.device(d.device):
                L.check(L.lib().step_detect_merge_f32(L.ptr(d), L.ptr(c), self.B, self.cap, self.thr, L.ptr(self.mbox),
                                                      L.ptr(self.pairs), L.ptr(self.count), L.ptr(self.ws), self.ws.numel(),
                                                      L.stream(d.device)))
        return {"mbox": self.mbox, "pairs": self.pairs, "count": self.count, "host": self.host, "tubes_nums": det["tubes_nums"]}


def merged_results(merged, det, label_dict):
    """Per clip, demo.py:177-198's `merged_result`: {mean box string: [(label, score), ...]} with the reference's keys,
    lists and dict order (np.float32 scores), as overlay_image takes it.  One read-back of the merge and the detector's
    rows (one synchronisation).  merged: Merger.run's result; det: the Detector.run result it was run on."""
    host = merged["host"]
    for h, t in zip(host, (merged["mbox"], merged["pairs"], merged["count"], det["det"])):
        h.copy_(t, non_blocking=True)
    torch.cuda.current_stream(merged["mbox"].device).synchronize()
    mbox, pairs, count, rows = (h.numpy() for h in host)
    out = []
    for b in range(len(merged["tubes_nums"])):
        n_keys, n_pairs = int(count[b, 0]), int(count[b, 1])
        keys = [",".join(mbox[b, k].astype(str).tolist()) for k in range(n_keys)]     # demo.py:197
        result = {k: [] for k in keys}
        for r, k in pairs[b, :n_pairs].tolist():
            result[keys[k]].append((label_dict[int(rows[b, r, 5])], rows[b, r, 4]))
        out.append(result)
    return out


def result_lines(results, infos):
    """demo.py:209-217: the results.txt lines (newline included) of the clips of one batch, from merged_results' dicts
    and the loader's infos (video_name, fid)."""
    lines = []
    for result, info in zip(results, infos):
        for key in result:
            box = np.asarray(key.split(","), dtype=np.float32)
            for l, s in result[key]:
                lines.append("{0},{1:04},{2:.4},{3:.4},{4:.4},{5:.4},{6},{7:.4}\n".format(
                    info["video_name"], info["fid"], box[0], box[1], box[2], box[3], l, s))
    return lines
