"""What training BatchNorm's affine parameters (freeze_affine=False) costs in the training step.

    python tools/bn_affine_bench.py [--rounds K] [--out FILE]

Builds the step of `tools/train_bench.py --shipped 2 --pool` (2 clips of 36 x 400 x 400, 34 tubes per clip, 3 temporal
steps, ContextNet on) and of `--cls 4 --pool` (the first training stage: 4 clips, one class-only head), on fp16 (loss scale
1024) and fp32 (loss scale 1.0), each twice from the same weights: once with freeze_affine=True and once with False.  In one
process, after one warm-up step of each, K rounds alternate the two: per round one timed train_step (wall time around a
device synchronise, no parameter update) and one with training.TIMING on, from which the device time of the `act_bwd`
phase (step_act_bwd_*, or step_act_bn_bwd_* where gamma / beta train) is read.  Prints one JSON line per configuration
and precision, with the card's name, power limit and maximum SM clock.
Correctness is covered by tests/test_gpu_bn_affine.py."""
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


def build(stage, fp16, freeze_affine):
    cfg, nets, x, st, sg = synth.make_workload(stage, fp16, "pool", freeze_affine=freeze_affine)
    n_bn = sum(p.requires_grad for n in nets.values() for k, p in n.named_parameters() if "batch3d" in k)
    return dict(cfg=cfg, nets=nets, x=x, st=st, sg=sg, n_bn=n_bn)


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
    w = synth.WORKLOADS[stage]
    return {"config": stage, "B": w.B, "tubes_per_clip": w.N, "precision": "fp16" if fp16 else "fp32",
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
    gpu = card(0)
    lines = []
    for stage in ("shipped", "cls"):
        for fp16 in (True, False):
            rec = measure(stage, fp16, a.rounds)
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
