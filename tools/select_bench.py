"""Time the training-sample selection (step_b200.select_samples) at the shipped configuration (scripts/train_step.sh: T=3,
NUM_CHUNKS {1:1, 2:1, 3:3}, max_iter 3, predict mode, topk 300, 60 classes, 34 proposals and 3 ground truths per clip,
softmax sampling), on one GPU:

    python tools/select_bench.py [--reps N] [--iters K] [--out FILE.jsonl]

1. select_samples on a history from step_b200.inference (synthetic nets and ContextNet, 400x400 clips of 36 frames) for
   B=2 and B=8: CUDA events around the whole call, which includes its one read-back; warmed up, median of N calls.
2. oracle/select.py, the numpy restatement, on the same history after .cpu(): host wall time of one single-threaded call
   (time.perf_counter; a stand-in for the reference's train_select, which has the same loops), median of N calls.
3. The shipped ROIPool training iteration at B=2 (inference pre-pass + selection + train_step without an update), with
   the host selection (history copied to the host, oracle/select.py, upload) and with the device selection, run
   alternately K times each; medians of the wall time per iteration.
Prints the card's name, power limit and maximum SM clock with the results.
Correctness is covered by tests/test_gpu_select.py."""
import argparse
import json
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import step_b200  # noqa: E402
from _bench import card  # noqa: E402
from oracle import select as osel  # noqa: E402
from step_b200 import synth, training  # noqa: E402

W = synth.WORKLOADS["shipped"].HW


def inputs(cfg, B, n=34, G=3, seed=4):
    rs = np.random.RandomState(seed)
    targets, tubes = [], []
    for _ in range(B):
        x1, y1 = rs.uniform(0, 0.5 * W, (2, G, 1))
        w, h = rs.uniform(0.2 * W, 0.45 * W, (2, G, 1))
        box = np.concatenate([x1, y1, x1 + w, y1 + h], 1)
        tg = np.zeros((G, 3, 4 + cfg.num_classes), np.float32)
        tg[:, :, :4] = box[:, None] + rs.uniform(-4, 4, (G, 3, 4))
        tg[:, :, 4:] = rs.uniform(0, 1, (G, 3, cfg.num_classes)) > 0.9
        targets.append(tg)
        src = box[rs.randint(0, G, n)] + rs.normal(0, 0.1 * W, (n, 4))
        src[:, 2:] = np.maximum(src[:, 2:], src[:, :2] + 8)
        tubes.append(np.tile(src[:, None], (1, cfg.T, 1)))
    return targets, tubes


def prepass(cfg, nets, x, tubes):
    with torch.no_grad():
        cf = nets["base_net"](x)
        ctx = nets["context_net"](cf)
        hist, _ = step_b200.inference(cfg, cf, ctx, nets, cfg.max_iter - 1, tubes, want_trajectory=False)
    return hist


def host_select(cfg, hist, targets, tubes):
    hh = [{k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in h.items()} for h in hist]
    st, sg = osel.select_samples(cfg, hh, targets, tubes)
    return [torch.from_numpy(t).cuda() for t in st], [torch.from_numpy(g).cuda() for g in sg]


def selection(cfg, nets, B, reps):
    targets, tubes = inputs(cfg, B)
    x = synth.make_clips(B, 36, W, W, seed=11).cuda()
    hist = prepass(cfg, nets, x, tubes)
    np.random.seed(1)
    random.seed(2)
    for _ in range(10):
        step_b200.select_samples(cfg, hist, targets, tubes)
    dev = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step_b200.select_samples(cfg, hist, targets, tubes)
        b.record()
        b.synchronize()
        dev.append(a.elapsed_time(b))
    hh = [{k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in h.items()} for h in hist]
    cpu = []
    for _ in range(reps):
        t0 = time.perf_counter()
        osel.select_samples(cfg, hh, targets, tubes)
        cpu.append((time.perf_counter() - t0) * 1e3)
    return {"what": "selection", "B": B, "reps": reps, "device_call_ms_median": round(statistics.median(dev), 4),
            "device_call_ms_p10_p90": [round(float(np.percentile(dev, 10)), 4), round(float(np.percentile(dev, 90)), 4)],
            "host_oracle_wall_ms_median": round(statistics.median(cpu), 3),
            "rows_per_step": [int(t.shape[0]) for t in step_b200.select_samples(cfg, hist, targets, tubes)[0]]}


def iteration(cfg, nets, iters):
    B = 2
    targets, tubes = inputs(cfg, B)
    x = synth.make_clips(B, 36, W, W, seed=11).cuda()

    def one(device_select):
        hist = prepass(cfg, nets, x, tubes)
        if device_select:
            st, sg = step_b200.select_samples(cfg, hist, targets, tubes)
        else:
            st, sg = host_select(cfg, hist, targets, tubes)
        training.train_step(cfg, nets, x, st, sg)
    for _ in range(3):
        one(True)
        one(False)
    times = {"host": [], "device": []}
    for _ in range(iters):
        for k in ("host", "device"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            one(k == "device")
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
    return {"what": "training iteration (pre-pass + selection + train_step, ROIPool, no update)", "B": B, "iters": iters,
            "host_selection_ms_median": round(statistics.median(times["host"]), 2),
            "device_selection_ms_median": round(statistics.median(times["device"]), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "select_bench needs a GPU"
    cfg, nets = synth.make_workload("shipped", pool_mode="pool")[:2]
    cfg.__dict__.update(cls_thresh=[0.2, 0.35, 0.5], reg_thresh=[0.2, 0.35, 0.5], topk=300, max_pos_num=5,
                        selection_sampling="softmax", neg_ratio=2)
    lines = [card(0)] + [selection(cfg, nets, B, a.reps) for B in (2, 8)] + [iteration(cfg, nets, a.iters)]
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write("".join(json.dumps(ln) + "\n" for ln in lines))


if __name__ == "__main__":
    main()
