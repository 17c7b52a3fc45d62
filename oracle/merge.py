"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the cross-class merge of the reference's demo.py:176-198: a greedy
merge of the detections of one clip whose compute_box_iou (utils/tube_utils.py:269-308) with an earlier group's leader
is > global_thresh, each group's box being the np.mean of its members' boxes, collected in a dict keyed by the mean's
string."""
import numpy as np

F32 = np.float32


def box_iou(a, b):
    """compute_box_iou of two float32 boxes (x1, y1, x2, y2): every operation rounded to float32, no "+1" in the areas,
    no intersection unless both sides are positive; a zero union gives NaN."""
    iw = max(F32(min(a[2], b[2]) - max(a[0], b[0])), F32(0))
    ih = max(F32(min(a[3], b[3]) - max(a[1], b[1])), F32(0))
    inter = F32(iw * ih) if (iw > 0 and ih > 0) else F32(0)
    union = F32(F32(F32(a[2] - a[0]) * F32(a[3] - a[1])) + F32(F32(b[2] - b[0]) * F32(b[3] - b[1])))
    union = F32(union - inter)
    with np.errstate(invalid="ignore", divide="ignore"):
        return F32(inter / union)


def demo_merge(dets, label_dict, global_thresh):
    """dets: one clip's detections in demo.py's scores_list order, (box[4] float32 normalised, class, score) as
    oracle.postprocess.detections returns them.  Returns demo.py's `merged_result`: {mean box string: [(label, score)]}
    with np.float32 scores.  The threshold is compared in float32 (numpy 2 keeps a Python float operand weak)."""
    thr = F32(global_thresh)
    boxes = [np.asarray(d[0], F32) for d in dets]
    taken = [False] * len(dets)
    result = {}
    for i in range(len(dets)):
        if taken[i]:
            continue
        members = [i]
        for j in range(i + 1, len(dets)):
            if not taken[j] and box_iou(boxes[i], boxes[j]) > thr:
                taken[j] = True
                members.append(j)
        total = (F32(0) + boxes[members[0]]).astype(F32)   # np.mean(axis=0) of a (n, 4) array: 0 + b0 + b1 + ... in
        for j in members[1:]:                                # row order (the identity +0.0 first: -0.0 sums to +0.0)
            total = (total + boxes[j]).astype(F32)
        mean = (total / F32(len(members))).astype(F32)
        key = ",".join(str(F32(v)) for v in mean)    # shortest round-trip repr: equal strings <=> equal floats
        result[key] = [(label_dict[int(dets[j][1])], F32(dets[j][2])) for j in members]
    return result
