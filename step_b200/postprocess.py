"""Detection post-processing on the device: the per-clip x per-class loop of the reference drivers
(test.py:156-218, demo.py:121-198 -- B*60*max_iter tiny CPU NMS calls per batch) as TWO launches of libstep_b200
(`step_detect_f32`), with no torch arithmetic, no gather tensors and no synchronisation: CUDA-graph capturable.

For every (clip, class): keep tubes whose centre-frame score > conf_thresh, clamp their centre-frame box
with valid_tubes (the drivers call it with its 400x400 defaults, test.py:191), run greedy NMS
(cpu/nms_cpu.cpp semantics, bit-exact), normalise by (width, height), then per clip either every survivor in
file order or the top-k scores in the order of the reference's tuple sort (test.py:205-208).
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
