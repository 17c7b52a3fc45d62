"""Time the classification pre-training stage's sample selection and validation (train_cls.py) on one GPU:

    python tools/cls_stage_bench.py [--reps N] [--frames F] [--host-frames H] [--out FILE.jsonl]

1. Selection at scripts/train_cls.sh's B = 4 (T = 9, 60 classes; per clip 1-6 ground truths, each with a box near it and
   3 boxes away from every ground truth, float64, as ava_cls.py makes them): step_b200.select_cls_samples, CUDA events
   around the whole call including its one read-back, against the host loop of train_cls.py:260-297 on the same inputs
   (oracle/select_cls.py's train_cls_select, which has the reference's loops, plus the upload of its two arrays), host wall
   time.  Warmed up; medians of N calls.
2. Validation on F synthetic frames in batches of 8 clips (1-4 ground truths per frame, each ground truth and 0-3 boxes
   away from it as proposals, class scores u^4 for uniform u): per batch ClsDetector.run + FrameAP.add_detections (CUDA
   events), then FrameAP.evaluate() (host wall time, it ends in a read-back).  Against the host restatement of
   train_cls.py:505-554 on the first H frames: the scores and boxes copied to the host, the CSV text of :537-543 and
   oracle/evaluation.py's numpy restatement of ava_evaluation on that text (the reference's evaluator has the same loops).
Prints the card's name, power limit and maximum SM clock with the results.
Correctness is covered by tests/test_gpu_cls_stage.py."""
import argparse
import io
import json
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from _bench import card  # noqa: E402
import step_b200  # noqa: E402
from make_cls_stage_golden import away, cls_detection_lines, make_clip  # noqa: E402
from oracle import evaluation as oev  # noqa: E402
from oracle import select_cls as osel  # noqa: E402
from step_b200.postprocess import ClsDetector  # noqa: E402

C, T, W, BATCH = 60, 9, 400, 8


def med(v, nd=4):
    return round(statistics.median(v), nd)


def selection(reps, B=4):
    rs = np.random.RandomState(5)
    clips = [make_clip(rs, rs.randint(1, 7)) for _ in range(B)]
    targets, tubes = [c[0] for c in clips], [c[1] for c in clips]
    np.random.seed(1)
    random.seed(2)
    for _ in range(10):
        step_b200.select_cls_samples(targets, tubes, C)
        t, g = osel.train_cls_select(targets, tubes, C)
        torch.from_numpy(t).cuda(), torch.from_numpy(g).cuda()
    torch.cuda.synchronize()
    dev, host = [], []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        t, _ = step_b200.select_cls_samples(targets, tubes, C)
        b.record()
        b.synchronize()
        dev.append(a.elapsed_time(b))
        t0 = time.perf_counter()
        ht, hg = osel.train_cls_select(targets, tubes, C)
        ht, hg = torch.from_numpy(ht).cuda(), torch.from_numpy(hg).cuda()
        torch.cuda.synchronize()
        host.append((time.perf_counter() - t0) * 1e3)
    return {"what": "select_cls_samples vs host loop", "B": B, "reps": reps, "gt_per_clip": [int(x.shape[0]) for x in targets],
            "proposals_per_clip": [int(x.shape[0]) for x in tubes], "rows": int(t.shape[0]),
            "device_call_ms_median": med(dev), "device_call_ms_p10_p90": [round(float(np.percentile(dev, q)), 4) for q in (10, 90)],
            "host_loop_ms_median": med(host, 3)}


def validation_set(frames, seed=7):
    rs = np.random.RandomState(seed)
    keys, gkeys, gboxes, glabels, nums, boxes = [], [], [], [], [], []
    label_ids = list(range(1, C + 1))
    for i in range(frames):
        key = ("bench%04d" % (i // 900), 902 + i % 900)
        keys.append(key)
        gts = []
        for _ in range(rs.randint(1, 5)):
            x1, y1 = rs.uniform(0, 0.6, 2)
            w, h = rs.uniform(0.15, 0.4, 2)
            g = np.array([x1, y1, x1 + w, y1 + h])
            gts.append(g)
            gkeys.append(key); gboxes.append(g); glabels.append(label_ids[rs.randint(0, C)])
        anchors = []
        for g in gts:
            anchors.append(g)
            anchors += [away(rs, gts) for _ in range(rs.randint(0, 4))]
        nums.append(len(anchors))
        boxes.append(np.stack(anchors) * W)
    return keys, gkeys, np.array(gboxes), np.array(glabels), nums, np.concatenate(boxes).astype(np.float32)


def flat_batch(boxes, nums):
    out = np.zeros((boxes.shape[0], T, 5), np.float32)
    start = 0
    for b, n in enumerate(nums):
        out[start:start + n, :, 0] = np.arange(T) + b * T
        out[start:start + n, :, 1:] = boxes[start:start + n, None]
        start += n
    return out


def validation(frames, host_frames):
    cats = [{"id": i, "name": "c%d" % i} for i in range(1, C + 1)]
    label_dict = list(range(1, C + 1))
    keys, gkeys, gboxes, glabels, nums, boxes = validation_set(frames)
    gen = torch.Generator(device="cuda").manual_seed(3)
    batches, start = [], 0
    for c0 in range(0, frames, BATCH):
        n = nums[c0:c0 + BATCH]
        R = sum(n)
        prob = torch.rand((R, C), generator=gen, device="cuda") ** 4
        tubes = torch.from_numpy(flat_batch(boxes[start:start + R], n)).cuda()
        batches.append((c0, n, prob, tubes, ClsDetector(n, C, "cuda:0", 0.01, W, W)))
        start += R

    def device_pass():
        ev = step_b200.FrameAP(cats, label_dict, device="cuda:0")
        ev.add_ground_truth(gkeys, gboxes, glabels)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for c0, n, prob, tubes, det in batches:
            ev.add_detections(det.run(prob, tubes), keys[c0:c0 + len(n)])
        b.record()
        b.synchronize()
        t0 = time.perf_counter()
        m = ev.evaluate()
        return a.elapsed_time(b), (time.perf_counter() - t0) * 1e3, int(ev._counters[0]), m["PascalBoxes_Precision/mAP@0.5IOU"]
    device_pass()                                   # warm-up: every shape and the store's growth
    runs = [device_pass() for _ in range(3)]
    add_ms, eval_ms = med([r[0] for r in runs], 2), med([r[1] for r in runs], 2)
    rows, mean_ap = runs[0][2], runs[0][3]

    # host restatement on the first host_frames frames
    sub = [b for b in batches if b[0] < host_frames]
    hf = sum(len(b[1]) for b in sub)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    text = io.StringIO()
    for c0, n, prob, tubes, _ in sub:
        lines = cls_detection_lines(prob.cpu().numpy(), tubes.cpu().numpy(), n, keys[c0:c0 + len(n)], label_dict, 0.01, W, W)
        text.writelines(lines)
    t1 = time.perf_counter()
    first = set(keys[:hf])
    gsel = [i for i, k in enumerate(gkeys) if k in first]
    glines = oev.gt_lines([gkeys[i] for i in gsel], gboxes[gsel], glabels[gsel])
    dlines = text.getvalue().splitlines(keepends=True)
    t2 = time.perf_counter()
    oev.run(cats, glines, dlines).per_class_ap()
    t3 = time.perf_counter()
    return {"what": "validation: ClsDetector.run + add_detections per batch, evaluate()", "frames": frames, "batch": BATCH,
            "detection_rows": rows, "rows_per_frame": round(rows / frames, 1), "mAP": round(float(mean_ap), 6),
            "device_detect_and_append_ms_total": add_ms, "device_detect_and_append_us_per_batch": round(1e3 * add_ms / len(batches), 2),
            "device_evaluate_ms": eval_ms,
            "host_subset_frames": hf, "host_subset_rows": len(dlines),
            "host_csv_ms_per_frame": round((t1 - t0) * 1e3 / hf, 3),
            "host_oracle_evaluation_ms_per_frame": round((t3 - t2) * 1e3 / hf, 3),
            "device_ms_per_frame": round((add_ms + eval_ms) / frames, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--frames", type=int, default=57600)
    ap.add_argument("--host-frames", type=int, default=400)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "cls_stage_bench needs a GPU"
    lines = [card(0), selection(a.reps), validation(a.frames, a.host_frames)]
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write("".join(json.dumps(ln) + "\n" for ln in lines))


if __name__ == "__main__":
    main()
