"""What the heads' training-mode dropout costs in the shipped training step (scripts/train_step.sh: --dropout 0.3).

    python tools/dropout_bench.py [--rounds K] [--out FILE]

Builds the step of `tools/train_bench.py --shipped 2` (2 clips of 36 x 400 x 400, 34 tubes per clip, 3 temporal steps,
ContextNet on) for three configurations -- fp32 with ROIAlign, fp32 with ROIPool, fp16 with ROIAlign --, puts the heads in
.train() (nn.Dropout(0.3)) and times train_step(..., dropout=True) against dropout=False, alternated in one process, K
rounds each after one warm-up of each (wall time around a device synchronise).  One more dropout=True step runs under
torch.profiler, and the device time of the dropout kernels (the draws' forward copies and context means, and the masked
backward siblings) is summed from its trace.  Prints one JSON line per configuration, with the card's name, power
limit and maximum SM clock.  Correctness is covered by tests/test_gpu_dropout.py."""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from _bench import card  # noqa: E402
from step_b200 import synth, training  # noqa: E402


def build(fp16, pool_mode):
    cfg, nets, x, st, sg = synth.make_workload("shipped", fp16, pool_mode, dropout=0.3)
    for i in range(cfg.max_iter):
        nets["det_net%d" % i].train()
    return cfg, nets, x, st, sg


def is_dropout_kernel(name):
    # the new kernels, and the DROP = true instantiations of the backward kernels they share with the undropped path
    siblings = ("mean_mid_bwd_kernel", "f32_accum_f16_kernel", "f32_accum_f32_kernel", "ctx_grad_reduce_kernel")
    return "dropout" in name or (any(k in name for k in siblings) and "true>" in name)


def measure(fp16, pool_mode, rounds):
    cfg, nets, x, st, sg = build(fp16, pool_mode)
    loss_scale = 1024.0 if fp16 else 1.0

    def step(drop):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        training.train_step(cfg, nets, x, st, sg, loss_scale=loss_scale, dropout=drop)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3
    step(True), step(False)
    times = {True: [], False: []}
    for _ in range(rounds):
        for drop in (True, False):
            times[drop].append(step(drop))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(True)
    kern = {}
    for e in prof.key_averages():
        if is_dropout_kernel(e.key):
            kern[e.key.split("(")[0]] = round(e.device_time_total / 1e3, 3)
    on, off = statistics.median(times[True]), statistics.median(times[False])
    w = synth.WORKLOADS["shipped"]
    return {"config": "shipped", "B": w.B, "tubes_per_clip": w.N, "precision": "fp16" if fp16 else "fp32", "pool_mode": pool_mode,
            "rounds": rounds, "step_ms_dropout": round(on, 1), "step_ms_no_dropout": round(off, 1),
            "step_ms_dropout_all": [round(t, 1) for t in times[True]], "step_ms_no_dropout_all": [round(t, 1) for t in times[False]],
            "dropout_kernels_device_ms": round(sum(kern.values()), 3), "dropout_kernels": kern}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--out")
    a = ap.parse_args()
    gpu = card(0)
    lines = []
    for fp16, pool_mode in ((False, "align"), (False, "pool"), (True, "align")):
        rec = measure(fp16, pool_mode, a.rounds)
        rec.update(gpu, torch=torch.__version__)
        print(json.dumps(rec), flush=True)
        lines.append(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
