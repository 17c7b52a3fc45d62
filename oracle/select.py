"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the training-sample selection of train.py:291-310: for every refinement
step, `train_select` (utils/utils.py:135-340, with `select_proposals` at :342-423) followed by the two `flatten_tubes` calls.

It draws from numpy's global RandomState (`np.random.choice`) and Python's `random` (`random.shuffle`) itself, in the
reference's order, so it leaves both generators where the reference leaves them.  Two parity contracts, which the device
(step_b200.select) follows too:
- ties: every `np.argsort(x)[::-1]` is a stable ascending argsort reversed (equal values: the larger index first).  numpy's
  default quicksort orders equal values in an implementation-defined way, so the two agree whenever the reference is well
  defined (no tie at a decision point);
- softmax weights: `float32(exp(float64(x)))`, the correctly rounded exponential.  numpy's float32 `exp` is not correctly
  rounded on its AVX-512 path; a draw differs only when a uniform lands between the two weights' cdf boundaries.

Pinned by tests/golden/select_cases.npz (outputs of the reference's own train_select, tests/golden/make_select_golden.py).
"""
import random

import numpy as np

from .tubes import extrapolate_tubes, flatten_tubes, valid_tubes

F = np.float32
SAMPLINGS = ("uniform", "random", "softmax")


def check_inputs(cfg, targets, tubes):
    """The cases in which the reference fails (np.max of an empty axis, np.stack of an empty list, pdb.set_trace()),
    raised as ValueError before any work."""
    if len(targets) != len(tubes) or len(targets) == 0:
        raise ValueError("select: %d target lists for %d proposal lists" % (len(targets), len(tubes)))
    for b, (g, t) in enumerate(zip(targets, tubes)):
        if np.asarray(g).shape[0] == 0:
            raise ValueError("select: clip %d has no ground truth" % b)
        if np.asarray(t).shape[0] == 0:
            raise ValueError("select: clip %d has no proposals" % b)
    if 0 < cfg.topk < cfg.num_classes:
        raise ValueError("select: 0 < topk=%d < num_classes=%d keeps int(topk / num_classes) * 2 == 0 candidates per "
                         "class" % (cfg.topk, cfg.num_classes))
    if cfg.selection_sampling not in SAMPLINGS:
        raise ValueError("select: selection_sampling %r is not one of %s" % (cfg.selection_sampling, SAMPLINGS))


def _desc(x):
    """np.argsort(x)[::-1] under the tie contract."""
    return np.argsort(x, kind="stable")[::-1]


def _box_iou(g, a):
    """compute_box_iou (tube_utils.py:269-308) of two boxes held as numpy scalars, whose types it keeps: an operation
    between two float32 values rounds to float32, one with a float64 (float64 proposals) to float64."""
    x1 = a[0] if a[0] > g[0] else g[0]
    y1 = a[1] if a[1] > g[1] else g[1]
    x2 = a[2] if a[2] < g[2] else g[2]
    y2 = a[3] if a[3] < g[3] else g[3]
    w, h = np.maximum(x2 - x1, 0.0), np.maximum(y2 - y1, 0.0)
    inter = w * h if (w > 0 and h > 0) else 0.0
    return F(inter / ((g[2] - g[0]) * (g[3] - g[1]) + (a[2] - a[0]) * (a[3] - a[1]) - inter))


def tube_iou(gt, anchors):
    """compute_tube_iou (tube_utils.py:310-351) at one frame: gt [G, 4] float32, anchors [N, 4]; 0 where either box sums
    to 0."""
    out = np.zeros((gt.shape[0], anchors.shape[0]), dtype=F)
    for i in range(gt.shape[0]):
        for j in range(anchors.shape[0]):
            if np.sum(gt[i]) and np.sum(anchors[j]):
                out[i, j] = _box_iou(list(gt[i]), list(anchors[j]))
    return out


def neg_weights(scores, sampling):
    if sampling == "uniform":
        s = scores + F(1e-6)
        return s / np.sum(s)
    if sampling == "random":
        return np.ones((len(scores),)) / len(scores)
    e = np.exp(scores.astype(np.float64)).astype(F)
    return e / np.sum(e)


def select_proposals(gt, anchors, scores, cls_thresh, max_pos_num, sampling, neg_ratio):
    """utils.py:342-423 at one frame: gt [G, 4] float32, anchors [N, 4], scores [N] float32 or None.
    Returns (positive pairs, negative pairs, ious [G, N])."""
    ious = tube_iou(gt, anchors)
    if scores is None:
        scores = np.max(ious, axis=0)
    pos, occupied = [], set()
    temp = ious.copy()
    for _ in range(ious.shape[0]):            # each ground truth in turn takes its best unoccupied candidate
        g = int(np.argmax(np.max(temp, axis=1)))
        free = [int(j) for j in _desc(ious[g]) if int(j) not in occupied]
        if free:
            occupied.add(free[0])
            pos.append((g, free[0]))
            temp[g, :] = -1
    if len(pos) > max_pos_num:
        random.shuffle(pos)
        pos = pos[:max_pos_num]
    cls_thresh = F(cls_thresh)
    hit = [int(j) for j in np.where(np.sum(ious > cls_thresh, axis=0))[0] if int(j) not in occupied]
    if hit and len(pos) < max_pos_num:
        size = min(len(hit), max_pos_num - len(pos))
        for k in np.random.choice(len(hit), size, p=np.ones((len(hit),)) / len(hit), replace=False):
            j = hit[k]
            occupied.add(j)
            pos.append((int(np.argmax(ious[:, j])), j))
    occupied.update(hit)
    neg = []
    free = [j for j in range(anchors.shape[0]) if j not in occupied]
    if free:
        size = min(len(pos) * neg_ratio, len(free))
        if size > 0:
            w = neg_weights(scores[free], sampling)
            for k in np.random.choice(len(free), size, p=w, replace=False):
                neg.append((int(np.argmax(ious[:, free[k]])), free[k]))
    return pos, neg, ious


def step_candidates(cfg, hist, b0, n):
    """utils.py:168-243 for one clip of a step > 1: (tubes [Nc, L, 4], scores [Nc], first, last) from the history rows
    [b0, b0 + n)."""
    W, H = cfg.image_size[0], cfg.image_size[1]
    p = np.asarray(hist["pred_prob"], dtype=F)[b0:b0 + n]
    if p.ndim == 2:
        p = p[:, None, :]
    s = p[:, 0].copy()
    for t in range(1, p.shape[1]):          # torch.mean over frames: a sequential float32 sum over L, then / L
        s = s + p[:, t]
    s = s / F(p.shape[1])
    K = int(cfg.topk / cfg.num_classes) * 2 if cfg.topk > 0 else n
    entries = []
    for c in range(cfg.num_classes):
        ids = _desc(s[:, c])[:K]
        entries += [(s[t, c], c, j, int(t)) for j, t in enumerate(ids)]
    entries.sort(key=lambda e: e[0])         # Python's stable sort by score, then reversed
    entries = entries[::-1]
    seen, order = set(), []
    for e in entries:
        if e[3] not in seen:
            seen.add(e[3])
            order.append(e)
    if cfg.topk > 0:
        order = order[:cfg.topk]
    rows = [b0 + e[3] for e in order]
    scores = np.asarray([e[0] for e in order], dtype=F)
    tubes = valid_tubes(np.asarray(hist["pred_loc"], dtype=F)[rows], W, H)
    first = last = None
    if cfg.temporal_mode == "predict":
        first = valid_tubes(np.asarray(hist["pred_first_loc"], dtype=F)[rows], W, H)
        last = valid_tubes(np.asarray(hist["pred_last_loc"], dtype=F)[rows], W, H)
    return tubes, scores, first, last


def train_select(step, hist, targets, tubes, cfg):
    """utils.py:135-340: per-clip lists (selected tubes [R_b, L, 4], targets [R_b, 3, 6 + C])."""
    chunks = cfg.NUM_CHUNKS[step]
    max_chunks = cfg.NUM_CHUNKS[cfg.max_iter]
    T_start = int((max_chunks - chunks) / 2) * cfg.T
    T_length = chunks * cfg.T
    mid = int(max_chunks / 2)
    C = cfg.num_classes
    b0 = 0
    sel_tubes, sel_targets = [], []
    for b in range(len(targets)):
        tg = np.asarray(targets[b])
        if step == 1:
            cand, scores, first, last = np.asarray(tubes[b]), None, None, None
        else:
            n = hist["tubes_nums"][b]
            cand, scores, first, last = step_candidates(cfg, hist, b0, n)
            b0 += n
        pos, neg, ious = select_proposals(tg[:, mid, :4].astype(F), cand[:, cand.shape[1] // 2], scores,
                                          cfg.cls_thresh[step - 1], cfg.max_pos_num, cfg.selection_sampling,
                                          cfg.neg_ratio)
        pairs = pos + neg
        R = len(pairs)
        out = np.zeros((R, cand.shape[1], 4), dtype=F)
        centre = np.zeros((R, 6 + C), dtype=F)
        for r, (g, j) in enumerate(pairs):
            out[r] = cand[j]
            if r < len(pos) or ious[g, j] >= F(cfg.reg_thresh[step - 1]):
                centre[r, :4] = tg[g, mid, :4]
                centre[r, 6:] = tg[g, mid, 4:]
                centre[r, 5] = 1
                centre[r, 4] = 1 if r < len(pos) else 0
        if step - 1 in cfg.NUM_CHUNKS and chunks == cfg.NUM_CHUNKS[step - 1] + 2:
            js = np.array([j for _, j in pairs], dtype=np.int64)
            if cfg.temporal_mode == "predict":
                out = np.concatenate([first[js], out, last[js]], axis=1)
            elif cfg.temporal_mode == "extrapolate":
                out = extrapolate_tubes(out, cfg.T)
            else:
                m = out[:, :1].copy()
                for t in range(1, out.shape[1]):
                    m = m + out[:, t:t + 1]
                m = np.tile(m / F(out.shape[1]), (1, cfg.T, 1))
                out = np.concatenate((m, out, m), axis=1)
        nb = np.zeros((2, R, 6 + C), dtype=F)
        if cfg.temporal_mode == "predict" and step < cfg.max_iter and cfg.NUM_CHUNKS[step + 1] == chunks + 2:
            for k, ci in enumerate((int((T_start - cfg.T) / cfg.T), int((T_start + T_length) / cfg.T))):
                for r, (g, _) in enumerate(pos):
                    nb[k, r, :4] = tg[g, ci, :4]
                    if nb[k, r, :4].sum() > 0:
                        nb[k, r, 5] = 1
                    nb[k, r, 6:] = tg[g, ci, 4:]
        sel_tubes.append(out)
        sel_targets.append(np.stack([nb[0], centre, nb[1]], axis=1))
    return sel_tubes, sel_targets


def _flat(parts, batch_idx):
    if sum(p.shape[0] for p in parts) == 0:   # every clip empty: zero rows (the reference's np.concatenate raises)
        _, L, d = parts[0].shape
        return np.zeros((0, L, d + (1 if batch_idx else 0)), dtype=F)
    return flatten_tubes(parts, batch_idx=batch_idx)[0].astype(F)


def select_samples(cfg, history, targets, tubes):
    """train.py:291-310 for every step: ([R_i, L_i, 5] flat tubes, [R_i, 3, 6 + C] flat targets) per step.
    history: step_b200.inference's list with its tensors as numpy arrays (pred_prob [R, L, C] or [R, C])."""
    check_inputs(cfg, targets, tubes)
    step_tubes, step_targets = [], []
    for i in range(1, cfg.max_iter + 1):
        st, sg = train_select(i, history[i - 2] if i > 1 else None, targets, tubes, cfg)
        step_tubes.append(_flat(st, True))
        step_targets.append(_flat(sg, False))
    return step_tubes, step_targets
