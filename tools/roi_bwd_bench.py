"""What the deterministic ROI backward costs: its five entries on their own, the driver iteration that reaches the NCHW
entries, and train_step, which reaches the channels-last ones.

    python tools/roi_bwd_bench.py [--rounds K] [--out FILE]

  * kernels: device time (CUDA events around each call, 3 warm-up calls, median of 20) of step_roi_align_bwd_nchw_f32,
    step_roi_pool_bwd_nchw_f32, step_roi_align_bwd_nhwc, step_roi_align_bwd_slice_nhwc and step_roi_pool_bwd_slice_nhwc on
    the operands of tests/golden/make_roi_bwd_golden.py's cases: the shipped step (2 clips x 9 frames of 25 x 25 x 832,
    612 rows of its 9-frame step, ROINet('align')'s adaptive sampling, fp32 and fp16 grad_out) and the classification
    stage (4 clips, 720 rows);
  * driver: tests/test_gpu_autograd.py's train_py_iteration at the shipped step, fp32, ROIAlign and ROIPool (wall time
    around a device synchronise, median over K rounds after one warm-up);
  * train_step at the shipped step, fp32 and fp16, ROIAlign, with the device time of its ROIAlign backward launches summed
    from a torch.profiler trace of one more step.
Prints one JSON line per measurement with the card's name, power limit and maximum SM clock, and writes them to FILE
(default profiles/h100_<power limit>_roi_bwd_bench.jsonl)."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]
import torch  # noqa: E402

import make_roi_bwd_golden as G  # noqa: E402
from _bench import card  # noqa: E402
from step_b200 import _lib as L  # noqa: E402
from step_b200 import synth, training  # noqa: E402
from test_gpu_autograd import train_py_iteration  # noqa: E402


def device_ms(fn, warm=3, n=20):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return round(statistics.median(ts), 4)


def kernel_records(name):
    c = next(c for c in G.CASES if c["name"] == name)
    rois, go, gin, feat = G.operands(c)
    r, K, H, W, C, R = G._cu(rois), c["K"], c["H"], c["W"], c["C"], c["R"]
    lib, s = L.lib(), L.stream()
    out = {}
    for tag, dt in (("f32", torch.float32), ("f16", torch.float16)):
        g = G._cu(go).to(dt)
        gi = G._cu(gin)
        out["align_bwd_nhwc_" + tag] = device_ms(lambda: L.check(lib.step_roi_align_bwd_nhwc(
            L.ptr(g), L.dt(g), C, L.ptr(r), R, G.SCALE, 7, 7, K, H, W, C, 0, L.ptr(gi), C, s)))
        out["align_bwd_slice_nhwc_" + tag] = device_ms(lambda: L.check(lib.step_roi_align_bwd_slice_nhwc(
            L.ptr(g), L.dt(g), C, L.ptr(r), R, G.SCALE, 7, 7, K, H, W, C, 0, c["roi_T"], c["feat_T"], c["t_start"], L.ptr(gi), C,
            None, 0, s)))
        am = G.pool_argmax(c, rois, feat)
        out["pool_bwd_slice_nhwc_" + tag] = device_ms(lambda: L.check(lib.step_roi_pool_bwd_slice_nhwc(
            L.ptr(g), L.dt(g), C, L.ptr(am), L.ptr(r), R, 7, 7, K, H, W, C, c["roi_T"], c["feat_T"], c["t_start"], L.ptr(gi), C,
            s)))
    # the reference layout, on the same rows (frame indices of the slice, read as frames of a [frames, C, H, W] map)
    frames = (K // c["feat_T"]) * c["roi_T"]
    g = G._cu(go[..., :C]).permute(0, 3, 1, 2).contiguous()
    gi = torch.empty((frames, C, H, W), device="cuda")
    out["align_bwd_nchw_f32"] = device_ms(lambda: L.check(lib.step_roi_align_bwd_nchw_f32(
        L.ptr(g), L.ptr(r), R, G.SCALE, 7, 7, frames, C, H, W, 0, L.ptr(gi), s)))
    fe = torch.randn(frames, C, H, W, generator=torch.Generator().manual_seed(0)).cuda()
    pout = torch.empty((R, C, 7, 7), device="cuda")
    am = torch.empty((R, C, 7, 7), dtype=torch.int32, device="cuda")
    L.check(lib.step_roi_pool_fwd_nchw_f32(L.ptr(fe), frames, C, H, W, L.ptr(r), R, G.SCALE, 7, 7, L.ptr(pout), L.ptr(am), s))
    out["pool_bwd_nchw_f32"] = device_ms(lambda: L.check(lib.step_roi_pool_bwd_nchw_f32(
        L.ptr(g), L.ptr(am), L.ptr(r), R, 7, 7, frames, C, H, W, L.ptr(gi), s)))
    return {"what": "kernels", "case": name, "rows": R, "frames": frames, "H": H, "W": W, "C": C, "device_ms": out}


def wall_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def step_record(what, pool_mode, fp16, rounds):
    cfg, nets, x, st, sg = synth.make_workload("shipped", fp16, pool_mode, dropout=0.3)
    for net in nets.values():
        net.train()
    params = [p for net in nets.values() for p in net.parameters() if p.requires_grad]

    def driver():
        for p in params:
            p.grad = None
        train_py_iteration(cfg, nets, x, st, sg)

    def step():
        training.train_step(cfg, nets, x, st, sg, loss_scale=1.0 if not fp16 else 1024.0, dropout=True)

    fn = driver if what == "driver" else step
    wall_ms(fn)
    times = [wall_ms(fn) for _ in range(rounds)]
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    roi = sum(e.device_time_total for e in prof.key_averages() if "roi_align_bwd" in e.key or "roi_pool_bwd" in e.key) / 1e3
    return {"what": what, "config": "shipped", "precision": "fp16" if fp16 else "fp32", "pool_mode": pool_mode,
            "rounds": rounds, "step_ms": round(statistics.median(times), 1), "step_ms_all": [round(t, 1) for t in times],
            "roi_bwd_device_ms": round(roi, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    gpu = card(0)
    out = a.out
    if out is None:
        try:
            limit = "%dw" % round(float(gpu["power_limit"].split()[0]))
        except ValueError:
            limit = "unknown"
        out = os.path.join(ROOT, "profiles", "h100_%s_roi_bwd_bench.jsonl" % limit)
    recs = [kernel_records("shipped_step9"), kernel_records("cls_step9"),
            step_record("driver", "align", False, a.rounds), step_record("driver", "pool", False, a.rounds),
            step_record("train_step", "align", False, a.rounds), step_record("train_step", "align", True, a.rounds)]
    lines = []
    for rec in recs:
        rec.update(gpu, torch=torch.__version__)
        print(json.dumps(rec), flush=True)
        lines.append(json.dumps(rec))
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
