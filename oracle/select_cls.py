"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the sample selection of the classification pre-training stage,
train_cls.py:260-297: per clip `select_proposals` (oracle/select.py, utils/utils.py:342-423) on chunk 0 of the targets
(the stage's max_chunks is 1) and the proposals' centre frame, the stage's rows, then the two `flatten_tubes` calls.

It draws from numpy's global RandomState and Python's `random` through oracle/select.py's `select_proposals`, so it
shares that module's tie contract and leaves both generators where the reference leaves them.  Pinned by
tests/golden/cls_stage_cases.npz (the reference's own select_proposals and flatten_tubes,
tests/golden/make_cls_stage_golden.py).
"""
import numpy as np

from .select import _flat, select_proposals

F = np.float32


def train_cls_select(targets, tubes, num_classes, cls_thresh=0.75, max_pos_num=5, sampling="uniform", neg_ratio=3):
    """A positive carries its ground truth's box, classification flag 1 and labels; a negative classification flag 1
    only; the regression flag stays 0, and the one target row is repeated three times.  The defaults are train_cls.py's
    literals.  Returns (flat tubes [R, T, 5], flat targets [R, 3, 6 + C])."""
    if len(targets) != len(tubes) or len(targets) == 0:
        raise ValueError("select: %d target lists for %d proposal lists" % (len(targets), len(tubes)))
    for b, (g, t) in enumerate(zip(targets, tubes)):
        if np.asarray(g).shape[0] == 0:
            raise ValueError("select: clip %d has no ground truth" % b)
        if np.asarray(t).shape[0] == 0:
            raise ValueError("select: clip %d has no proposals" % b)
    sel_tubes, sel_targets = [], []
    for b in range(len(targets)):
        tg, cand = np.asarray(targets[b]), np.asarray(tubes[b])
        pos, neg, _ = select_proposals(tg[:, 0, :4].astype(F), cand[:, cand.shape[1] // 2], None, cls_thresh, max_pos_num,
                                       sampling, neg_ratio)
        out = np.zeros((len(pos) + len(neg), cand.shape[1], 4), dtype=F)
        row = np.zeros((len(pos) + len(neg), 6 + num_classes), dtype=F)
        for r, (g, j) in enumerate(pos + neg):
            out[r] = cand[j]
            row[r, 4] = 1
            if r < len(pos):
                row[r, :4] = tg[g, 0, :4]
                row[r, 6:] = tg[g, 0, 4:]
        sel_tubes.append(out)
        sel_targets.append(np.repeat(row[:, None], 3, axis=1))
    return _flat(sel_tubes, True), _flat(sel_targets, False)
