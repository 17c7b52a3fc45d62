"""Time demo.py's detection post-processing and cross-class merge (demo.py:130-198) on the device against the host loop, on
one GPU:

    python tools/demo_bench.py [--reps N] [--host-reps M] [--out FILE.jsonl]

Workload: demo.py's shape on the shipped configuration (scripts/train_step.sh: T=3, 3 steps, NUM_CHUNKS {1:1, 2:1, 3:3},
context on): B = 8 clips of 36 frames at 400x400, 34 proposals per clip, synthetic nets, merge threshold 0.8
(demo.py:55), no top-k (evaluate_topk's default).  Two cases: demo.py's conf 0.4 and a dense conf 0.01, nms 0.4.
1. The merge alone (Merger.run on the last step's detections): CUDA events around each launch sequence, median of N.
2. Inside the captured step: graph replays of StepRunner without detection, with detect=dict(...) and with
   detect=dict(..., merge=0.8), run alternately N times each; medians of CUDA events around each replay.  Their
   differences are the detection and the merge inside the step.
3. The host side of the device path: merged_results (one read-back and the dicts), host wall time, median of N.
4. The host loop demo.py:130-198 over the same history after .cpu(): oracle.postprocess.detections with the library's
   nms on CPU tensors (what demo.py calls under compat.patch) and oracle.merge.demo_merge, single-threaded; host wall
   time, median of M.
Prints the card's name, power limit and maximum SM clock with the results.
Correctness is covered by tests/test_gpu_merge.py."""
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

import step_b200  # noqa: E402
from _bench import card  # noqa: E402
from oracle import merge as om  # noqa: E402
from oracle import postprocess as opp  # noqa: E402
from step_b200 import roi_layers, synth  # noqa: E402
from step_b200.postprocess import Merger, merged_results  # noqa: E402

B, T_IN, HW, N = 8, 36, 400, 34
LABELS = list(range(1, 61))


def events(fn, reps):
    out = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        out.append((s, e))
    torch.cuda.synchronize()
    return [s.elapsed_time(e) for s, e in out]


def med(xs, nd=4):
    return round(statistics.median(xs), nd)


def host_loop(prob, loc, nums, conf, nms_thresh):
    """demo.py:130-198 through the numpy restatement, with the library's nms on CPU tensors."""
    dets = opp.detections(prob, loc, nums, conf, nms_thresh, float(HW), float(HW))
    return [om.demo_merge(d, LABELS, 0.8) for d in dets]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--host-reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    cfg = synth.make_cfg(fp16=True, image_size=(HW, HW), **synth.WORKLOADS["shipped"].cfg)
    nets = synth.device_nets(cfg, [synth.head_state_dict(100 + i, cfg) for i in range(cfg.max_iter)], context=True)
    tubes = synth.make_proposals(B, N, cfg.T, HW, HW)
    x = synth.make_clips(B, T_IN, HW, HW).to(dev)
    last = cfg.max_iter - 1
    # the library's nms on CPU tensors, as demo.py calls it under compat.patch
    opp.ops.nms = lambda b, s, t: roi_layers.nms(torch.from_numpy(np.ascontiguousarray(b)),
                                                 torch.from_numpy(np.ascontiguousarray(s)), t).numpy()
    plain = step_b200.StepRunner(cfg, nets, B, T_IN, HW, HW, tubes, context=True)
    lines = [card(0)]
    for name, conf in (("demo", 0.4), ("dense", 0.01)):
        det_kw = dict(conf_thresh=conf, nms_thresh=0.4, topk=0)
        detect = step_b200.StepRunner(cfg, nets, B, T_IN, HW, HW, tubes, context=True, detect=det_kw)
        merge = step_b200.StepRunner(cfg, nets, B, T_IN, HW, HW, tubes, context=True, detect=dict(det_kw, merge=0.8))
        runners = {"step": plain, "step_detect": detect, "step_detect_merge": merge}
        for r in runners.values():
            r.x.copy_(x)
            r()
        torch.cuda.synchronize()
        times = {k: [] for k in runners}
        for _ in range(a.reps):
            for k, r in runners.items():
                times[k] += events(r, 1)
        d = merge.detections[last]
        merger = Merger(merge.detectors[last], 0.8)
        merger.run(d)
        merge_ms = events(lambda: merger.run(d), a.reps)
        walls = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            res = merged_results(merge.merged[last], d, LABELS)
            walls.append((time.perf_counter() - t0) * 1e3)
        counts = merge.merged[last]["count"].cpu().numpy()
        # the host loop over the same history
        h = merge.history[last]
        prob = h["pred_prob"][:, h["pred_prob"].shape[1] // 2].float().cpu().numpy()
        loc = h["pred_loc"][:, h["pred_loc"].shape[1] // 2].float().cpu().numpy()
        host = []
        for _ in range(a.host_reps):
            t0 = time.perf_counter()
            ref = host_loop(prob, loc, [N] * B, conf, 0.4)
            host.append((time.perf_counter() - t0) * 1e3)
        same = [list(r) for r in ref] == [list(r) for r in res]
        rows = [int(v) for v in d["count"].cpu().numpy()]
        lines.append({"what": "demo_merge", "case": name, "B": B, "T_in": T_IN, "HW": HW, "tubes_per_clip": N,
                      "conf_thresh": conf, "nms_thresh": 0.4, "global_thresh": 0.8, "rows_per_clip": rows,
                      "keys_per_clip": [int(v) for v in counts[:, 0]],
                      "merge_device_ms_median": med(merge_ms),
                      "replay_ms_median": {k: med(v, 3) for k, v in times.items()},
                      "detect_in_step_ms": round(med(times["step_detect"], 3) - med(times["step"], 3), 3),
                      "detect_merge_in_step_ms": round(med(times["step_detect_merge"], 3) - med(times["step"], 3), 3),
                      "merged_results_host_ms_median": med(walls, 3),
                      "host_loop_130_198_ms_median": med(host, 1), "host_keys_equal_device": same})
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        with open(a.out, "a") as f:
            f.write("".join(json.dumps(ln) + "\n" for ln in lines))


if __name__ == "__main__":
    main()
