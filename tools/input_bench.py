"""Time the input transform on the device (step_b200.transforms.BaseTransform, kernel step_frames_to_clip_u8) and what it
changes for the captured step.

    python tools/input_bench.py [--launches N] [--rounds R] [--steps S] [--out FILE.jsonl]

1. The kernel alone, median of N individually event-timed launches at two shapes: C4 (8 clips x 32 frames of 360x640 ->
   224x224, bench.py's workload) and the shipped training batch (2 x 36 frames of 360x640 -> 400x400).  Bytes are counted
   from shapes: every source byte read once, the fp32 clip written once; the floor is those bytes at the data sheet's
   3.35 TB/s.
2. StepRunner at C4 (graph on, bench.py's detection post-processing) fed pinned uint8 360x640 frames (transform=...) against
   the same runner fed pinned fp32 224x224 clips, in alternating runs of S steps each (each run ends in a synchronise);
   clips/s per run, medians reported, and the host-to-device bytes per batch of both.
Prints the card's name, power limit and maximum SM clock with the results.
Correctness is covered by tests/test_gpu_transform.py."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from _bench import card  # noqa: E402
import bench  # noqa: E402
import step_b200  # noqa: E402
from step_b200 import synth  # noqa: E402
from step_b200.transforms import BaseTransform, frame_entry, frame_table  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
SHAPES = {"c4": dict(B=8, T=32, H0=360, W0=640, HW=224), "shipped": dict(B=2, T=36, H0=360, W0=640, HW=400)}


def frames(B, T, H0, W0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (B, T, 3, H0, W0), dtype=torch.uint8, generator=g)


def kernel_time(name, s, launches, dev):
    tr = BaseTransform((s["HW"], s["HW"]), scale=2)
    src = frames(s["B"], s["T"], s["H0"], s["W0"]).to(dev)
    table = frame_table([frame_entry(src[b], s["HW"]) for b in range(s["B"])], dev)
    out = torch.empty((s["B"], s["T"], 3, s["HW"], s["HW"]), dtype=torch.float32, device=dev)
    for _ in range(10):
        tr.launch(table, s["B"], s["T"], out)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(launches)]
    for a, b in ev:
        a.record()
        tr.launch(table, s["B"], s["T"], out)
        b.record()
    torch.cuda.synchronize()
    ms = statistics.median(a.elapsed_time(b) for a, b in ev)
    n_in = s["B"] * s["T"] * 3 * s["H0"] * s["W0"]
    n_out = s["B"] * s["T"] * 3 * s["HW"] * s["HW"] * 4
    floor_ms = (n_in + n_out) / HBM_BYTES_PER_S * 1e3
    return {"shape": name, **s, "launches": launches, "kernel_ms_median": round(ms, 4), "bytes_in": n_in,
            "bytes_out": n_out, "GB_per_s": round((n_in + n_out) / ms / 1e6, 1), "floor_ms": round(floor_ms, 4),
            "x_floor": round(ms / floor_ms, 2)}


def runner_rates(rounds, steps, dev):
    W = bench.WORKLOAD
    B, T_in, HW = W["B"], W["T_in"], W["HW"]
    cfg = synth.make_cfg(fp16=True, T=T_in // 4, max_iter=W["max_iter"], NUM_CHUNKS={1: 1, 2: 1, 3: 1}, image_size=(HW, HW))
    nets = bench.build_nets(cfg, dev)
    tubes = synth.make_proposals(B, W["N"], cfg.T, HW, HW)
    tr = BaseTransform((HW, HW), scale=2)
    u8 = frames(B, T_in, 360, 640, seed=1).pin_memory()
    f32 = tr.apply(u8).cpu().pin_memory()
    arms = {"uint8_360x640": (step_b200.StepRunner(cfg, nets, B, T_in, HW, HW, tubes, detect=bench.DETECT, transform=tr,
                                                   source_hw=(360, 640)), u8),
            "fp32_224x224": (step_b200.StepRunner(cfg, nets, B, T_in, HW, HW, tubes, detect=bench.DETECT), f32)}
    rates = {k: [] for k in arms}
    with torch.no_grad():
        for k, (r, x) in arms.items():
            for _ in range(3):
                r(x)
        torch.cuda.synchronize()
        for _ in range(rounds):
            for k, (r, x) in arms.items():
                t0 = time.perf_counter()
                for _ in range(steps):
                    r(x)
                torch.cuda.synchronize()
                rates[k].append(B * steps / (time.perf_counter() - t0))
    return {"B": B, "T_in": T_in, "rounds": rounds, "steps_per_round": steps,
            "clips_per_s_median": {k: round(statistics.median(v), 1) for k, v in rates.items()},
            "clips_per_s_runs": {k: [round(x, 1) for x in v] for k, v in rates.items()},
            "h2d_bytes_per_batch": {k: x.numel() * x.element_size() for k, (_, x) in arms.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "input_bench needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lines = [card(0)]
    lines += [kernel_time(k, s, a.launches, dev) for k, s in SHAPES.items()]
    lines.append(runner_rates(a.rounds, a.steps, dev))
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("".join(json.dumps(ln) + "\n" for ln in lines))


if __name__ == "__main__":
    main()
