"""Generates tests/golden/merge_cases.npz: demo.py's per-clip loop (demo.py:130-217: per-class NMS, the cross-class merge
and the results.txt lines) run by the UNMODIFIED reference on synthetic histories.  Only runnable where the reference
tree exists; the fixture it writes is committed.

    python tests/golden/make_merge_golden.py

Per case <name>: the inputs (_prob [R, C] and _loc [R, 4], the centre frame demo.py:124-127 slices; _nums; _cfg = conf,
nms, topk, width, height, global_thresh, valid), the rows the merge reads (_rows [M, 7] = clip, class, score, box, in
scores_list order), the merged dicts (_keys, _key_clip; _items [I, 4] = clip, key index in the clip, label, score, in
dict order) and the results.txt text (_text)."""
import io
import os
import sys
import textwrap
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refload  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
R = refload.load()
F32 = np.float32
LABELS = [1, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 17, 20, 22, 24, 26, 27, 28, 29, 30, 34, 36, 37, 38, 41, 43, 45,
          46, 47, 48, 49, 51, 52, 54, 56, 57, 58, 59, 60, 61, 62, 63, 64, 65, 66, 67, 68, 69, 70, 72, 73, 74, 76, 77, 78, 79, 80]


def _reference_demo_loop_source():
    """The per-clip loop of the reference's demo.py (`tubes_count = 0` through the results.txt writes, demo.py:130-217),
    read from the file where it lies and dedented -- executed, never stored."""
    lines = open(os.path.join(refload.REF, "demo.py")).read().split("\n")
    start = next(i for i, l in enumerate(lines) if l.strip() == "tubes_count = 0")
    end = next(i for i in range(start, len(lines)) if lines[i].strip().startswith("torch.cuda.synchronize()"))
    return textwrap.dedent("\n".join(lines[start:end]))


def run_reference_demo_loop(prob, loc, nums, conf, nms_thresh, topk, width, height, global_thresh, valid=True):
    """Executes the loop on one batch; returns per clip (scores_list rows, merged_result) and the results.txt text."""
    fout = io.StringIO()
    captured = []
    env = {}

    def overlay_image(src, dst, pred_boxes, id2class):   # demo.py:204-207: capture instead of drawing
        rows = [(c, s) + tuple(float(v) for v in env["all_boxes"][c][j]) for s, c, j in env["scores_list"]]
        captured.append((rows, {k: list(v) for k, v in pred_boxes.items()}))

    fake_os = SimpleNamespace(path=SimpleNamespace(isdir=lambda p: True, join=os.path.join), makedirs=lambda p: None)
    env.update({
        "pred_prob": torch.from_numpy(prob.copy()), "pred_tubes": torch.from_numpy(loc.copy()), "tubes_nums": list(nums),
        "infos": [{"video_name": "vid%d" % (b % 2), "fid": 7 + 3 * b} for b in range(len(nums))],
        "args": SimpleNamespace(num_classes=prob.shape[1], nms_thresh=nms_thresh, evaluate_topk=topk, topk=topk,
                                label_dict=LABELS, save_root="/nonexistent", data_root="/nonexistent", id2class={}),
        "conf_thresh": conf, "global_thresh": global_thresh, "width": width, "height": height, "im_format": "frame%04d.jpg",
        "np": np, "torch": torch, "os": fake_os, "print": lambda *a, **k: None, "fout": fout,
        "valid_tubes": R.tube_utils.valid_tubes if valid else (lambda t: t), "nms": R.roi_layers.nms,
        "compute_box_iou": R.tube_utils.compute_box_iou, "overlay_image": overlay_image})
    exec(compile(_reference_demo_loop_source(), "reference demo.py:130-217", "exec"), env)
    return captured, fout.getvalue()


out = {}


def case(name, prob, loc, nums, conf, nms_thresh, topk, width=400, height=400, global_thresh=0.8, valid=True):
    prob, loc = np.asarray(prob, F32), np.asarray(loc, F32)
    captured, text = run_reference_demo_loop(prob, loc, nums, conf, nms_thresh, topk, width, height, global_thresh, valid)
    rows, keys, key_clip, items = [], [], [], []
    for b, (r, merged) in enumerate(captured):
        rows += [(b,) + row for row in r]
        for k, key in enumerate(merged):
            keys.append(key)
            key_clip.append(b)
            items += [(b, k, label, s) for label, s in merged[key]]
    out[name + "_prob"], out[name + "_loc"], out[name + "_nums"] = prob, loc, np.asarray(nums, np.int64)
    out[name + "_cfg"] = np.asarray([conf, nms_thresh, topk, width, height, global_thresh, valid], np.float64)
    out[name + "_rows"] = np.asarray(rows, F32).reshape(-1, 7)
    out[name + "_keys"] = np.asarray(keys, dtype=str)
    out[name + "_key_clip"] = np.asarray(key_clip, np.int64)
    out[name + "_items"] = np.asarray(items, F32).reshape(-1, 4)
    out[name + "_text"] = np.asarray(text)
    print(name, "rows per clip", [sum(1 for r in rows if r[0] == b) for b in range(len(nums))],
          "keys per clip", [key_clip.count(b) for b in range(len(nums))], "lines", text.count("\n"))
    return captured


def people(rs, B, n, P, jitter):
    """n tubes per clip around P people: centre-frame boxes [B*n, 4] in a 400x400 frame."""
    loc = []
    for _ in range(B):
        xy = rs.uniform(0, 260, (P, 2))
        wh = rs.uniform(60, 140, (P, 2))
        who = rs.randint(0, P, n)
        box = np.concatenate([xy[who], xy[who] + wh[who]], 1) + rs.normal(0, jitter, (n, 4))
        loc.append(box)
    return np.concatenate(loc).astype(F32)


def iou_pair(target, x, y):
    """Two integer pixel boxes at (x, y) whose normalised compute_box_iou is exactly `target` (float32)."""
    ref = R.tube_utils.compute_box_iou
    for h in range(40, 150):
        for w1 in range(40, 150):
            for w2 in range(int(0.7 * w1), w1):
                a, b = (x, y, x + w1, y + h), (x, y, x + w2, y + h)
                if ref(np.asarray(a, F32) / F32(400), np.asarray(b, F32) / F32(400))[0, 0] == target:
                    return a, b
    raise RuntimeError("no pair")


def main():
    rs = np.random.RandomState(17)
    C = 60
    # demo-like: B = 4, 34 tubes, 60 classes, conf 0.4 (demo.py:54), nms 0.4 (config.py default), no top-k
    loc = people(rs, 4, 34, 4, 3.0)
    prob = rs.uniform(0, 1, (4 * 34, C)).astype(F32) ** 3
    case("demo", prob, loc, [34] * 4, 0.4, 0.4, -1)
    # dense: conf 0.01, with and without top-k 300
    loc = people(rs, 2, 34, 3, 4.0)
    prob = rs.uniform(0, 1, (2 * 34, C)).astype(F32)
    case("dense", prob, loc, [34] * 2, 0.01, 0.4, -1)
    case("dense_topk", prob, loc, [34] * 2, 0.01, 0.4, 300)
    # one group of 34 x 60 = 2040 members (nms 0.95 keeps every jittered tube in every class), whose np.mean differs from
    # a pairwise sum in float32
    for _ in range(100):
        base = rs.uniform(60, 120, 2)
        loc = np.concatenate([base, base + 150])[None] + rs.uniform(-2, 2, (34, 4))
        loc = loc.astype(F32)
        prob = rs.uniform(0.5, 1, (34, C)).astype(F32)
        cap = case("big_group", prob, loc, [34], 0.4, 0.95, -1)
        boxes = np.asarray([r[2:] for r in cap[0][0]], F32)
        pairwise = np.asarray([np.sum(np.ascontiguousarray(boxes[:, c])) for c in range(4)], F32) / F32(len(boxes))
        if len(cap[0][1]) == 1 and not np.array_equal(boxes.mean(0), pairwise):
            break
    else:
        raise RuntimeError("no case with a sequential / pairwise difference")
    # edges: an empty clip; IoU exactly float32(0.8) (kept apart) and the next float32 above it (merged); one row; tubes
    # with no score above conf
    t8 = F32(0.8)
    a, b = iou_pair(t8, 10, 20)
    a2, b2 = iou_pair(np.nextafter(t8, F32(1)), 210, 220)
    far = (10, 300, 90, 390)
    loc = np.asarray([a, b, far, a2, b2,
                      (5, 5, 100, 100), (200, 200, 300, 300),
                      (5, 5, 100, 100), (200, 200, 300, 300)], F32)
    prob = np.zeros((9, 6), F32)
    prob[0, 0], prob[1, 1], prob[2, 2], prob[3, 3], prob[4, 4] = 0.9, 0.8, 0.7, 0.6, 0.5
    prob[5, 3] = 0.55                     # the clip's one row
    prob[7:, :] = 0.3                     # nothing above conf
    case("edges", prob, loc, [0, 5, 2, 2], 0.4, 0.4, -1)
    # identical zero-area boxes of two classes (only reachable past valid_tubes, which widens degenerate boxes): their IoU
    # is NaN, so they form two groups with one mean -- a repeated key, which keeps the first position and the last list
    loc = np.asarray([(50, 60, 50, 90), (10, 10, 120, 150), (200, 200, 260, 300)], F32)
    prob = np.zeros((3, 4), F32)
    prob[0, 0], prob[0, 2], prob[1, 1], prob[2, 3], prob[1, 3] = 0.9, 0.7, 0.8, 0.6, 0.65
    case("zero_area", prob, loc, [3], 0.4, 0.4, -1, valid=False)
    np.savez_compressed(os.path.join(OUT, "merge_cases.npz"), **out)


if __name__ == "__main__":
    main()
