"""What normalising with batch statistics (freeze_stats=False) costs in the training step.

    python tools/bn_stats_bench.py [--rounds K] [--out FILE]

Builds the step of `tools/train_bench.py --shipped 2 --pool` (2 clips of 36 x 400 x 400, 34 tubes per clip, 3 temporal
steps, ContextNet on) on fp16 (loss scale 1024) and fp32 (loss scale 1.0), each twice from the same weights: with
freeze_stats=True (running statistics, the nets in eval mode as the other tools run them) and with freeze_stats=False (the
nets in train(): every BatchNorm normalises with batch statistics and updates its running statistics).  In one process,
after one warm-up step of each, K rounds alternate the two: one timed train_step (wall time around a device synchronise,
no parameter update) and one with training.TIMING on for the device time of the backward's BatchNorm phase (`bn_bwd`:
step_bn_bwd_*; `act_bwd` with frozen statistics).  Then one step of each under torch.profiler gives the device time of the
forward's step_bn_stats_* and step_bn_apply_* kernels, and one more the peak memory.  The bytes those kernels must move
(z read by the statistics; z read and y written by the apply; dy, y and z read twice and dz written by the backward) are
counted from every batch-statistics convolution of the step and set against the HBM floor (3.35 TB/s, the H100 SXM data
sheet).  Prints one JSON line per precision, with the card's name, power limit and maximum SM clock.
Correctness is covered by tests/test_gpu_bn_stats.py."""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from _bench import card  # noqa: E402
from step_b200 import engine as E, synth, training  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def build(fp16, freeze_stats):
    cfg, nets, x, st, sg = synth.make_workload("shipped", fp16, "pool", freeze_stats=freeze_stats)
    if not freeze_stats:
        for k, n in nets.items():
            if k != "roi_net":
                n.train()
    return dict(cfg=cfg, nets=nets, x=x, st=st, sg=sg)


def counted_bytes(fn):
    """Runs fn() with engine._conv_batch_stats wrapped; returns the bytes of z the batch-statistics convolutions produced
    (elements x storage size), the unit the traffic model multiplies."""
    orig, box = E._conv_batch_stats, [0]

    def wrapped(x, w, shift, outs, *a, **kw):
        o = outs[0]
        box[0] += o.N * o.T * o.H * o.W * sum(t.C for t in outs) * o.buf.element_size()
        return orig(x, w, shift, outs, *a, **kw)
    E._conv_batch_stats = wrapped
    try:
        fn()
    finally:
        E._conv_batch_stats = orig
    return box[0]


def kernel_ms(fn, names):
    """Device time (ms) of the kernels whose names contain one of `names`, over one call of fn, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    for ev in prof.key_averages():
        for n in names:
            if n in ev.key:
                out[n] += ev.device_time_total / 1e3
    return out


def measure(fp16, rounds):
    runs = {fs: build(fp16, fs) for fs in (True, False)}
    loss_scale = 1024.0 if fp16 else 1.0

    def call(fs):
        r = runs[fs]
        return training.train_step(r["cfg"], r["nets"], r["x"], r["st"], r["sg"], loss_scale=loss_scale)

    def step(fs, phases=False):
        training.TIMING = {} if phases else None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        call(fs)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        ph = training.timing_summary() if phases else None
        training.TIMING = None
        return ms, ph
    for fs in (True, False):
        step(fs)
    times = {True: [], False: []}
    bn_phase = {True: [], False: []}
    for _ in range(rounds):
        for fs in (True, False):
            times[fs].append(step(fs)[0])
            ph = step(fs, phases=True)[1]
            bn_phase[fs].append(ph.get("bn_bwd", 0.0) + ph.get("act_bwd", 0.0))
    k = kernel_ms(lambda: call(False), ("bn_stats_partial", "bn_stats_final", "bn_apply", "bn_bwd_partial", "bn_bwd_reduce",
                                        "bn_bwd_dz"))
    z_bytes = counted_bytes(lambda: call(False))
    peak = {}
    for fs in (True, False):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        call(fs)
        torch.cuda.synchronize()
        peak[fs] = torch.cuda.max_memory_allocated() / 2 ** 20
    fwd_ms = k["bn_stats_partial"] + k["bn_stats_final"] + k["bn_apply"]
    bwd_ms = k["bn_bwd_partial"] + k["bn_bwd_reduce"] + k["bn_bwd_dz"]
    fwd_bytes, bwd_bytes = 3 * z_bytes, 7 * z_bytes
    med = {fs: statistics.median(times[fs]) for fs in (True, False)}
    w = synth.WORKLOADS["shipped"]
    return {"config": "shipped", "B": w.B, "tubes_per_clip": w.N, "precision": "fp16" if fp16 else "fp32",
            "pool_mode": "pool", "rounds": rounds,
            "step_ms_running_stats": round(med[True], 1), "step_ms_batch_stats": round(med[False], 1),
            "step_ms_running_stats_all": [round(t, 1) for t in times[True]],
            "step_ms_batch_stats_all": [round(t, 1) for t in times[False]],
            "bn_bwd_phase_ms_running_stats": round(statistics.median(bn_phase[True]), 2),
            "bn_bwd_phase_ms_batch_stats": round(statistics.median(bn_phase[False]), 2),
            "kernel_ms": {n: round(v, 3) for n, v in k.items()},
            "fwd_bn_kernel_ms": round(fwd_ms, 3), "bwd_bn_kernel_ms": round(bwd_ms, 3),
            "z_mb": round(z_bytes / 2 ** 20, 1), "fwd_bn_mb": round(fwd_bytes / 2 ** 20, 1), "bwd_bn_mb": round(bwd_bytes / 2 ** 20, 1),
            "fwd_bn_hbm_floor_ms": round(fwd_bytes / HBM_BYTES_PER_S * 1e3, 3),
            "bwd_bn_hbm_floor_ms": round(bwd_bytes / HBM_BYTES_PER_S * 1e3, 3),
            "fwd_bn_share_of_hbm_floor": round(fwd_bytes / HBM_BYTES_PER_S * 1e3 / fwd_ms, 3) if fwd_ms else None,
            "bwd_bn_share_of_hbm_floor": round(bwd_bytes / HBM_BYTES_PER_S * 1e3 / bwd_ms, 3) if bwd_ms else None,
            "peak_mb_running_stats": round(peak[True], 1), "peak_mb_batch_stats": round(peak[False], 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bn_stats_bench: needs a CUDA device")
    gpu = card(0)
    lines = []
    for fp16 in (True, False):
        rec = measure(fp16, a.rounds)
        rec.update(gpu, torch=torch.__version__)
        print(json.dumps(rec), flush=True)
        lines.append(json.dumps(rec))
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
