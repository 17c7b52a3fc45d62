"""What training BatchNorm's affine parameters (freeze_affine=False) costs in the training step.

    python tools/bn_affine_bench.py [--rounds K] [--out FILE]

Builds the step of `tools/train_bench.py --shipped 2 --pool` (2 clips of 36 x 400 x 400, 34 tubes per clip, 3 temporal
steps, ContextNet on) and of `--cls 4 --pool` (the first training stage: 4 clips, one class-only head), on fp16 (loss scale
1024) and fp32 (loss scale 1.0), each twice from the same weights: once with freeze_affine=True and once with False.  In one
process, after one warm-up step of each, K rounds alternate the two: per round one timed train_step (wall time around a
device synchronise, no parameter update) and one with training.TIMING on, from which the device time of the `act_bwd`
phase (step_act_bwd_*, or step_act_bn_bwd_* where gamma / beta train) is read.  Prints one JSON line per configuration
and precision, with the card's name and power limit.  Correctness is covered by tests/test_gpu_bn_affine.py."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import step_b200  # noqa: E402
from step_b200 import synth, training  # noqa: E402

T_IN, HW = 36, 400


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, limit = [s.strip() for s in q.stdout.strip().split(",")] if q.returncode == 0 else (torch.cuda.get_device_name(0), "unknown")
    return name, limit


def build(stage, fp16, freeze_affine):
    cls = stage == "cls"
    if cls:
        B, N = 4, 20
        cfg = synth.make_cfg(fp16=fp16, T=9, max_iter=1, NUM_CHUNKS={1: 1}, no_context=False, image_size=(HW, HW),
                             freeze_affine=freeze_affine)
    else:
        B, N = 2, 34
        cfg = synth.make_cfg(fp16=fp16, T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False, image_size=(HW, HW),
                             freeze_affine=freeze_affine)
    nets = {"base_net": step_b200.BaseNet(cfg), "roi_net": step_b200.ROINet("pool", 7), "context_net": step_b200.ContextNet(cfg)}
    nets["base_net"].load_state_dict(synth.base_net_state_dict())
    nets["context_net"].load_state_dict(synth.context_net_state_dict())
    if cls:
        h = step_b200.TwoBranchNet(cfg, cls_only=True)
        h.load_state_dict(synth.cls_head_state_dict(100, cfg))
        nets["det_net0"] = h
    else:
        for i in range(3):
            h = step_b200.TwoBranchNet(cfg)
            h.load_state_dict(synth.head_state_dict(100 + i, cfg))
            nets["det_net%d" % i] = h
    for k in nets:
        nets[k] = nets[k].cuda().eval()
        if hasattr(nets[k], "set_device"):
            nets[k].set_device("cuda:0")
    x = synth.make_clips(B, T_IN, HW, HW).cuda()
    if cls:
        ft, fg = synth.make_cls_case(cfg, B, N, HW, HW)
        st, sg = [ft], [fg]
    else:
        st, sg = synth.make_train_case(cfg, B, N, HW, HW)
    n_bn = sum(p.requires_grad for n in nets.values() for k, p in n.named_parameters() if "batch3d" in k)
    return dict(cfg=cfg, nets=nets, x=x, st=[t.cuda() for t in st], sg=[t.cuda() for t in sg], B=B, N=N, n_bn=n_bn)


def measure(stage, fp16, rounds):
    runs = {fa: build(stage, fp16, fa) for fa in (True, False)}
    loss_scale = 1024.0 if fp16 else 1.0

    def step(fa, phases=False):
        r = runs[fa]
        training.TIMING = {} if phases else None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = training.train_step(r["cfg"], r["nets"], r["x"], r["st"], r["sg"], loss_scale=loss_scale)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        act = training.timing_summary().get("act_bwd") if phases else None
        training.TIMING = None
        return ms, act, len(out["grads"])
    n_grads = {fa: step(fa)[2] for fa in (True, False)}
    times = {True: [], False: []}
    act = {True: [], False: []}
    for _ in range(rounds):
        for fa in (True, False):
            times[fa].append(step(fa)[0])
            act[fa].append(step(fa, phases=True)[1])
    med = {fa: statistics.median(times[fa]) for fa in (True, False)}
    amed = {fa: statistics.median(act[fa]) for fa in (True, False)}
    return {"config": stage, "B": runs[True]["B"], "tubes_per_clip": runs[True]["N"], "precision": "fp16" if fp16 else "fp32",
            "pool_mode": "pool", "rounds": rounds, "bn_tensors_trained": runs[False]["n_bn"],
            "grads_frozen_affine": n_grads[True], "grads_trained_affine": n_grads[False],
            "step_ms_frozen_affine": round(med[True], 1), "step_ms_trained_affine": round(med[False], 1),
            "step_ms_frozen_affine_all": [round(t, 1) for t in times[True]],
            "step_ms_trained_affine_all": [round(t, 1) for t in times[False]],
            "act_bwd_ms_frozen_affine": round(amed[True], 2), "act_bwd_ms_trained_affine": round(amed[False], 2),
            "act_bwd_ms_frozen_affine_all": act[True], "act_bwd_ms_trained_affine_all": act[False],
            "act_bwd_ratio": round(amed[False] / amed[True], 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bn_affine_bench: needs a CUDA device")
    name, limit = card()
    lines = []
    for stage in ("shipped", "cls"):
        for fp16 in (True, False):
            rec = measure(stage, fp16, a.rounds)
            rec.update(gpu=name, power_limit=limit, torch=torch.__version__)
            print(json.dumps(rec), flush=True)
            lines.append(json.dumps(rec))
            torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
