"""Time the device frame-mAP (step_b200.FrameAP) on a validation-sized synthetic set, on one GPU:

    python tools/eval_bench.py [--frames N] [--rows R] [--oracle-frames M] [--out FILE.jsonl]

Workload: N = 57,600 frames (the AVA v2.1 validation keyframes) in 8-clip batches, R = 300 detection rows per frame
(an assumption: STEP's real count is unmeasured), 1-6 ground-truth rows per frame, the AVA v2.1 label map (60 of 80 ids).
Rows are drawn on the device in the layout of step_detect_f32's output (det [8, R, 8], count [8]).
1. add_detections: CUDA events around each call (launches only; the store is reserved first), median over the batches.
2. evaluate(): CUDA events around the device work of step_eval_run alone, and host wall time of the whole call (ground
   truth upload and the read-back included).
3. Peak device memory of the run (torch.cuda.max_memory_allocated).
4. oracle/evaluation.py on the first M = 2,000 frames: single-threaded host wall time of one call, the CSV text parsing
   included (a stand-in for the reference's run_evaluation, which has the same loops).
Prints the card's name, power limit and maximum SM clock with the results.
Correctness is covered by tests/test_gpu_eval.py."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from _bench import card  # noqa: E402
import step_b200  # noqa: E402
from oracle import evaluation as oev  # noqa: E402

# the AVA v2.1 label map's ids (ava_action_list_v2.1_for_activitynet_2018), names replaced by their ids
AVA_IDS = [1, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 17, 20, 22, 24, 26, 27, 28, 29, 30, 34, 36, 37, 38, 41, 43, 45,
           46, 47, 48, 49, 51, 52, 54, 56, 57, 58, 59, 60, 61, 62, 63, 64, 65, 66, 67, 68, 69, 70, 72, 73, 74, 76, 77, 78, 79, 80]


def make_batch(g, B, R, C, gt_boxes):
    """det rows around the batch's ground truth: x1, y1, x2, y2 normalised, score, class, tube, 0."""
    dev = gt_boxes.device
    pick = torch.randint(0, gt_boxes.shape[1], (B, R), generator=g, device=dev)
    base = torch.gather(gt_boxes, 1, pick[..., None].expand(B, R, 4))
    det = torch.zeros((B, R, 8), dtype=torch.float32, device=dev)
    det[..., :4] = base + 0.04 * torch.randn((B, R, 4), generator=g, device=dev)
    det[..., 4] = torch.rand((B, R), generator=g, device=dev)
    det[..., 5] = torch.randint(0, C, (B, R), generator=g, device=dev).float()
    return det


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=57600)
    ap.add_argument("--rows", type=int, default=300)
    ap.add_argument("--oracle-frames", type=int, default=2000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    B, R, C = 8, a.rows, len(AVA_IDS)
    cats = [{"id": i, "name": str(i)} for i in AVA_IDS]
    rs = np.random.RandomState(0)
    g = torch.Generator(device=dev)
    g.manual_seed(0)
    ev = step_b200.FrameAP(cats, AVA_IDS, device=dev)
    ev.reserve(a.frames * R)
    count = torch.full((B,), R, dtype=torch.int32, device=dev)
    gt_all, times, det_lines, gt_lines = [], [], [], []
    torch.cuda.reset_peak_memory_stats()
    for f0 in range(0, a.frames, B):
        keys = [("v%04d" % ((f0 + b) // 900), 902 + (f0 + b) % 900) for b in range(B)]
        ng = rs.randint(1, 7, B)
        xy = rs.uniform(0, 0.6, (B, 6, 2))
        boxes = np.concatenate([xy, xy + rs.uniform(0.1, 0.4, (B, 6, 2))], 2)
        labels = rs.choice(AVA_IDS, (B, 6))
        gk, gb, gl = [], [], []
        for b in range(B):
            gk += [keys[b]] * ng[b]
            gb.append(boxes[b, :ng[b]])
            gl.append(labels[b, :ng[b]])
        gb, gl = np.concatenate(gb), np.concatenate(gl)
        ev.add_ground_truth(gk, gb, gl)
        det = make_batch(g, B, R, C, torch.from_numpy(boxes.astype(np.float32)).to(dev))
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        ev.add_detections({"det": det, "count": count}, keys)
        e.record()
        times.append((s, e))
        if f0 < a.oracle_frames:
            d = det.cpu().numpy()
            clips = [[(d[b, k, :4], int(d[b, k, 5]), d[b, k, 4]) for k in range(R)] for b in range(B)]
            det_lines += oev.detection_lines(clips, keys, AVA_IDS)
            gt_lines += oev.gt_lines(gk, gb, gl)
    torch.cuda.synchronize()
    add_ms = [s.elapsed_time(e) for s, e in times]
    # evaluate(): device time of step_eval_run from the launch stream, wall time of the call
    from step_b200 import _lib
    orig = _lib.lib().step_eval_run
    ev_times = []

    def timed(p, stream):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        rc = orig(p, stream)
        e.record()
        ev_times.append((s, e))
        return rc
    lib = _lib.lib()
    lib.step_eval_run = timed
    walls = []
    try:
        for _ in range(3):
            t0 = time.perf_counter()
            m = ev.evaluate()
            walls.append((time.perf_counter() - t0) * 1e3)
    finally:
        lib.step_eval_run = orig
    torch.cuda.synchronize()
    eval_ms = [s.elapsed_time(e) for s, e in ev_times]
    peak = torch.cuda.max_memory_allocated() / 2 ** 20
    t0 = time.perf_counter()
    om = oev.run(cats, gt_lines, det_lines)
    om.per_class_ap()
    oracle_s = time.perf_counter() - t0
    lines = [card(0),
             {"what": "add_detections", "frames": a.frames, "rows_per_frame": R, "clips_per_batch": B,
              "batches": len(add_ms), "device_ms_median": round(statistics.median(add_ms), 4),
              "device_ms_p10_p90": [round(float(np.percentile(add_ms, 10)), 4), round(float(np.percentile(add_ms, 90)), 4)]},
             {"what": "evaluate", "rows": int(ev._counters[0].item()), "images": len(ev._ids),
              "device_ms": [round(t, 3) for t in eval_ms], "wall_ms": [round(t, 2) for t in walls],
              "mAP": float(m["PascalBoxes_Precision/mAP@0.5IOU"]), "peak_mem_mib": round(peak, 1)},
             {"what": "oracle_host", "frames": a.oracle_frames, "rows": len(det_lines), "wall_s": round(oracle_s, 2)}]
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        with open(a.out, "a") as f:
            f.write("".join(json.dumps(ln) + "\n" for ln in lines))


if __name__ == "__main__":
    main()
