"""Time the training augmentation (step_b200.transforms.TubeAugmentation): its kernel on the device, and its host stage.

    python tools/augment_bench.py [--rounds R] [--launches N] [--out FILE.jsonl]     # device: needs a GPU
    python tools/augment_bench.py --host [--clips N] [--out FILE.jsonl]             # host stage, one core

1. Device: at the shipped training shape (2 clips x 36 frames of 360x640 -> 400x400, scale 2), the augmenting kernel
   (step_frames_to_clip_aug_u8, every flag on, one fixed seeded recipe per clip) and the BaseTransform kernel
   (step_frames_to_clip_u8) in alternating rounds of N event-timed launches each; medians over all launches.  Bytes are
   counted from shapes: the source bytes the kernel taps read once (the crop rect's, for the augmenting kernel), the erase
   noise once, the fp32 clip written once; the floor is those bytes at the data sheet's 3.35 TB/s.  Prints the card's name,
   power limit and maximum SM clock with the results.
2. Host (--host, CPU time of one core, not device time): the host stage's time per 36-frame 360x640 clip, and, where the
   reference checkout exists (oracle/refload.py), the reference's TubeAugmentation on the same clips, tubes and seeds
   with cv2 on one thread.
Correctness is covered by tests/test_gpu_augment.py."""
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
from step_b200.transforms import BaseTransform, TubeAugmentation, frame_entry, frame_table  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
B, T, H0, W0, HW = 2, 36, 360, 640, 400
ALL = dict(do_flip=True, do_crop=True, do_photometric=True, do_erase=True)


def clip_bgr(seed):
    return np.random.RandomState(seed).randint(0, 256, (T, H0, W0, 3)).astype(np.uint8)


def tubes(seed, N=3, K=3):
    rs = np.random.RandomState(seed)
    x1, y1 = rs.uniform(0.05, 0.5, (2, N, 1))
    w, h = rs.uniform(0.25, 0.45, (2, N, 1))
    boxes = np.stack([x1, y1, x1 + w, y1 + h], -1).repeat(K, 1)
    return np.concatenate([boxes, np.ones((N, K, 2))], -1).astype(np.float32)


def recipes(tr, seed=7):
    """One recipe per clip with every op on (the first seeded draws whose gates are all on and whose crop keeps at
    least half the frame), so the timed program is the longest one."""
    out, s = [], seed
    while len(out) < B:
        np.random.seed(s)
        tr(np.empty((T, H0, W0, 3), np.uint8), tubes(s), None)
        r = tr.last_recipe
        if all(v is not None for v in (r.brightness, r.contrast, r.saturation, r.hue)) and r.erase and \
                r.crop[2] * r.crop[3] * 2 >= H0 * W0:
            out.append(r)
        s += 1
    return out


def device(rounds, launches):
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    aug = TubeAugmentation((HW, HW), scale=2, **ALL)
    base = BaseTransform((HW, HW), scale=2)
    recs = recipes(aug)
    g = torch.Generator().manual_seed(0)
    src = torch.randint(0, 256, (B, T, 3, H0, W0), dtype=torch.uint8, generator=g).to(dev)
    table = frame_table([frame_entry(src[b], HW) for b in range(B)], dev)
    out = torch.empty((B, T, 3, HW, HW), dtype=torch.float32, device=dev)
    # the augmenting launch's device tables, built once through apply's packing
    aug_out = aug.apply([(src[b], recs[b]) for b in range(B)])
    packed = {}
    orig = aug.launch

    def capture(table_, params, erase, noise, B_, T_, out_):
        packed.update(table=table_, params=params, erase=erase, noise=noise)
        return orig(table_, params, erase, noise, B_, T_, out_)
    aug.launch = capture
    aug.apply([(src[b], recs[b]) for b in range(B)])
    aug.launch = orig
    arms = {"base_transform": lambda: base.launch(table, B, T, out),
            "tube_augmentation": lambda: aug.launch(packed["table"], packed["params"], packed["erase"],
                                                    packed["noise"], B, T, aug_out)}
    for f in arms.values():
        for _ in range(10):
            f()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(launches)]
            for a, b in ev:
                a.record()
                f()
                b.record()
            torch.cuda.synchronize()
            times[k] += [a.elapsed_time(b) for a, b in ev]
    n_out = B * T * 3 * HW * HW * 4
    n_noise = sum(r.noise.size * 4 for r in recs)
    bytes_ = {"base_transform": (B * T * 3 * H0 * W0, n_out),
              "tube_augmentation": (sum(T * 3 * r.crop[2] * r.crop[3] for r in recs) + n_noise, n_out)}
    lines = []
    for k, v in times.items():
        ms = statistics.median(v)
        n_in, n_o = bytes_[k]
        floor_ms = (n_in + n_o) / HBM_BYTES_PER_S * 1e3
        lines.append({"kernel": k, "B": B, "T": T, "H0": H0, "W0": W0, "HW": HW, "rounds": rounds,
                      "launches_per_round": launches, "kernel_ms_median": round(ms, 4),
                      "kernel_ms_p10_p90": [round(float(np.percentile(v, 10)), 4), round(float(np.percentile(v, 90)), 4)],
                      "bytes_in": n_in, "bytes_out": n_o, "GB_per_s": round((n_in + n_o) / ms / 1e6, 1),
                      "floor_ms": round(floor_ms, 4), "x_floor": round(ms / floor_ms, 2)})
    lines.append({"recipes": [repr(r) for r in recs]})
    return lines


def host(clips):
    """CPU seconds per clip on one core (cv2 limited to one thread; the host stage does no pixel work)."""
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    ours = TubeAugmentation((HW, HW), scale=2, **ALL)
    data = [(clip_bgr(i), tubes(i)) for i in range(clips)]
    res = {"what": "host CPU time per 36-frame 360x640 clip, one core, not device time", "clips": clips}

    def run(tr):
        t = []
        for i, (f, tb) in enumerate(data):
            np.random.seed(100 + i)
            t0 = time.process_time()
            tr(f, tb.copy(), None)
            t.append(time.process_time() - t0)
        return t
    t = run(ours)
    res["host_stage_s_median"] = statistics.median(t)
    res["host_stage_s_range"] = [min(t), max(t)]
    from oracle import refload
    if refload.available():
        import cv2
        cv2.setNumThreads(1)
        sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
        import make_augment_golden
        ref = make_augment_golden.load_augmentations().TubeAugmentation((HW, HW), scale=2, **ALL)
        t = run(ref)
        res["reference_s_median"] = statistics.median(t)
        res["reference_s_range"] = [min(t), max(t)]
        res["cv2"] = cv2.__version__
    import platform
    res["cpu"] = platform.processor() or platform.machine()
    return [res]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--host", action="store_true")
    ap.add_argument("--clips", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=40)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.host:
        lines = host(a.clips)
    else:
        assert torch.cuda.is_available(), "augment_bench needs a GPU (or --host)"
        lines = [card(0)] + device(a.rounds, a.launches)
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write("".join(json.dumps(ln) + "\n" for ln in lines))


if __name__ == "__main__":
    main()
