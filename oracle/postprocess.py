"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the detection post-processing loop of the reference's
test.py:156-218 (per clip, per class: score > conf -> valid_tubes(400x400 default) -> nms -> normalise)."""
import numpy as np

from . import ops, tubes


def detections(prob, boxes, tubes_nums, conf_thresh, nms_thresh, width, height, topk=0, with_tube=False):
    """prob [R,cls], boxes [R,4] (centre frame).  Returns per clip a list of (box[4] normalised, cls, score) in the order
    test.py:204-208 writes them: file order (class, then kept tube ascending) when topk <= 0; otherwise a stable ascending
    sort on the score, reversed (tied scores in reverse file order), cut at topk.  with_tube: (box, cls, score, tube in
    clip)."""
    out, start = [], 0
    for n in tubes_nums:
        p, b = prob[start:start + n], boxes[start:start + n]
        start += n
        dets = []
        for c in range(prob.shape[1]):
            s = p[:, c]
            m = s > conf_thresh                                   # test.py:183 scores.gt(conf_thresh)
            if not m.any():
                continue
            bb = tubes.valid_tubes(b[m].reshape(-1, 1, 4)).reshape(-1, 4)   # test.py:191 (default 400x400)
            keep = ops.nms(bb, s[m], nms_thresh)                  # test.py:192
            tube = np.nonzero(m)[0]
            for k in keep:
                box = bb[k].copy()
                box[0::2] /= width; box[1::2] /= height           # test.py:197-198
                dets.append((box, c, float(s[m][k])) + ((int(tube[k]),) if with_tube else ()))
        if topk and topk > 0:
            dets.sort(key=lambda d: d[2])
            dets = dets[::-1][:topk]
        out.append(dets)
    return out
