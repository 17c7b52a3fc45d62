"""What training through torch.autograd costs against train_step, at the shipped step (scripts/train_step.sh).

    python tools/autograd_bench.py [--rounds K] [--out FILE]

Builds the `shipped` workload (2 clips of 36 x 400 x 400, 34 tubes per clip, 3 temporal steps, ContextNet on, heads with
nn.Dropout(0.3) in training mode), fp32, once with ROIAlign and once with ROIPool, and times in one process, alternated
over K rounds after one warm-up of each (wall time around a device synchronise):
  * autograd: the restatement of train.py:263-347 in tests/test_gpu_autograd.py (the modules' forwards, the driver's torch
    ops, loss_back.backward()), parameter gradients zeroed before each;
  * train_step(..., loss_scale=1.0, dropout=True).
Neither runs an optimizer.  Peak memory is torch.cuda.max_memory_allocated over one step of each.  One more autograd
step runs under torch.profiler, and the device time of the NCHW ROIAlign / ROIPool backward kernels (the ones the
driver's contiguous conv_feat slices reach; the field keeps the name it had when they scattered with atomics) is summed
from its trace, beside that of train_step's channels-last ROI backward in a profiled train_step.  Prints one JSON line per pool mode with the card's name, power
limit and maximum SM clock, and writes them to FILE (default profiles/h100_<power limit>_autograd_bench.jsonl)."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

from _bench import card  # noqa: E402
from step_b200 import synth, training  # noqa: E402
from test_gpu_autograd import train_py_iteration  # noqa: E402


def kernel_ms(prof, names):
    return round(sum(e.device_time_total for e in prof.key_averages() if any(n in e.key for n in names)) / 1e3, 3)


def measure(pool_mode, rounds):
    cfg, nets, x, st, sg = synth.make_workload("shipped", False, pool_mode, dropout=0.3)
    for net in nets.values():
        net.train()
    params = [p for net in nets.values() for p in net.parameters() if p.requires_grad]

    def autograd_step():
        for p in params:
            p.grad = None
        train_py_iteration(cfg, nets, x, st, sg)

    def train_step():
        training.train_step(cfg, nets, x, st, sg, loss_scale=1.0, dropout=True)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    runs = {"autograd": autograd_step, "train_step": train_step}
    peak = {}
    for k, fn in runs.items():
        torch.cuda.reset_peak_memory_stats()
        timed(fn)
        peak[k] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    times = {k: [] for k in runs}
    for _ in range(rounds):
        for k, fn in runs.items():
            times[k].append(timed(fn))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        autograd_step()
        torch.cuda.synchronize()
    nchw = kernel_ms(prof, ("roi_align_bwd_nchw", "roi_pool_bwd_nchw"))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        train_step()
        torch.cuda.synchronize()
    nhwc = kernel_ms(prof, ("roi_align_bwd", "roi_pool_bwd"))
    w = synth.WORKLOADS["shipped"]
    med = {k: round(statistics.median(v), 1) for k, v in times.items()}
    return {"config": "shipped", "B": w.B, "tubes_per_clip": w.N, "precision": "fp32", "pool_mode": pool_mode, "dropout": 0.3,
            "rounds": rounds, "step_ms_autograd": med["autograd"], "step_ms_train_step": med["train_step"],
            "step_ms_autograd_all": [round(t, 1) for t in times["autograd"]],
            "step_ms_train_step_all": [round(t, 1) for t in times["train_step"]],
            "peak_gib_autograd": peak["autograd"], "peak_gib_train_step": peak["train_step"],
            "roi_bwd_nchw_atomic_device_ms": nchw, "roi_bwd_train_step_device_ms": nhwc}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    gpu = card(0)
    out = a.out
    if out is None:
        try:
            limit = "%dw" % round(float(gpu["power_limit"].split()[0]))
        except ValueError:
            limit = "unknown"
        out = os.path.join(ROOT, "profiles", "h100_%s_autograd_bench.jsonl" % limit)
    lines = []
    for pool_mode in ("align", "pool"):
        rec = measure(pool_mode, a.rounds)
        rec.update(gpu, torch=torch.__version__)
        print(json.dumps(rec), flush=True)
        lines.append(json.dumps(rec))
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
