"""What synchronising the heads' batch statistics across ranks costs (train_step, freeze_stats=False, world_size > 1).

    python tools/bn_sync_bench.py [--rounds K] [--out FILE]

One GPU: the price of splitting each reduction around an exchange, before any exchange.  The BatchNorm shapes (M pixels,
C channels) are those of every batch-statistics convolution of the `tools/bn_stats_bench.py` step (the shipped
configuration, 2 clips of 36 x 400 x 400, 34 tubes per clip).  For each precision, K rounds alternate the fused entries
(step_bn_stats_* and step_bn_bwd_*) and the split entries at one rank (step_bn_stats_local_* + step_bn_stats_merge and
step_bn_bwd_sums_* + step_bn_bwd_merge_dz_*) over every shape, each timed with CUDA events over 20 passes; the medians are
reported.

Two or more GPUs: the shipped fp16 step on each of two ranks over NCCL (each rank one clip), freeze_stats True and False
alternated, with CUDA events around every exchange of the heads (engine.all_gather_rows) timed separately.  With a single
GPU that part prints "not measured: needs 2 GPUs".  Every line carries the card's name, power limit and maximum SM clock.
Correctness is covered by tests/test_gpu_bn_sync.py."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch  # noqa: E402

from _bench import card  # noqa: E402
from step_b200 import _lib as L, engine as E, synth, training  # noqa: E402

PASSES = 20


def bn_shapes():
    """(M, C) of every BatchNorm output of one shipped batch-statistics step (fp16; the shapes do not depend on precision)."""
    cfg, nets, x, st, sg = synth.make_workload("shipped", True, "pool", freeze_stats=False)
    for k, n in nets.items():
        if k != "roi_net":
            n.train()
    orig, shapes = E._conv_batch_stats, []

    def wrapped(x_, w, shift, outs, *a, **kw):
        shapes.extend((o.N * o.T * o.H * o.W, o.C) for o in outs)
        return orig(x_, w, shift, outs, *a, **kw)
    E._conv_batch_stats = wrapped
    try:
        training.train_step(cfg, nets, x, st, sg, loss_scale=1024.0)
    finally:
        E._conv_batch_stats = orig
    torch.cuda.synchronize()
    return shapes


class Shape:
    """Operands and workspaces of one (M, C) for both variants."""

    def __init__(self, f16, M, C):
        dt = torch.float16 if f16 else torch.float32
        self.f16, self.M, self.C = f16, M, C
        self.z = torch.randn((M, C), device="cuda").to(dt)
        self.dy = (torch.randn((M, C), device="cuda") * 1e-2).to(dt)
        self.y = torch.rand((M, C), device="cuda").to(dt)
        self.dz = torch.empty_like(self.z)
        self.gamma, self.beta = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
        self.rm, self.rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
        self.st = torch.empty((4, C), device="cuda")
        self.trip, self.sums = torch.empty((1, 3, C), device="cuda"), torch.empty((1, 2, C), device="cuda")
        self.dg, self.db = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
        lib = L.lib()
        self.nb = max(lib.step_bn_stats_workspace_bytes(M, C), lib.step_bn_bwd_workspace_bytes(M, C))
        self.ws = torch.empty((self.nb // 4,), device="cuda")

    def fused(self):
        lib, s, f = L.lib(), self, self.f16
        st = s.st
        L.check((lib.step_bn_stats_f16 if f else lib.step_bn_stats_f32)(
            L.ptr(s.z), s.C, s.M, s.C, L.ptr(s.gamma), L.ptr(s.beta), 1e-5, 0.1, L.ptr(s.rm), L.ptr(s.rv), L.ptr(st[0]), L.ptr(st[1]),
            L.ptr(st[2]), L.ptr(st[3]), L.ptr(s.ws), s.nb, L.stream()))
        L.check((lib.step_bn_bwd_f16 if f else lib.step_bn_bwd_f32)(
            L.ptr(s.dy), s.C, L.ptr(s.y), s.C, L.ptr(s.z), s.C, s.M, s.C, L.ptr(st[0]), L.ptr(st[1]), L.ptr(s.gamma), 1, 1.0,
            L.ptr(s.dz), s.C, L.ptr(s.dg), L.ptr(s.db), L.ptr(s.ws), s.nb, L.stream()))

    def split(self):
        lib, s, f = L.lib(), self, self.f16
        st = s.st
        L.check((lib.step_bn_stats_local_f16 if f else lib.step_bn_stats_local_f32)(
            L.ptr(s.z), s.C, s.M, s.C, L.ptr(s.trip), s.C, L.ptr(s.ws), s.nb, L.stream()))
        L.check(lib.step_bn_stats_merge(L.ptr(s.trip), 1, s.C, s.M, s.C, L.ptr(s.gamma), L.ptr(s.beta), 1e-5, 0.1, L.ptr(s.rm),
                                        L.ptr(s.rv), L.ptr(st[0]), L.ptr(st[1]), L.ptr(st[2]), L.ptr(st[3]), L.stream()))
        L.check((lib.step_bn_bwd_sums_f16 if f else lib.step_bn_bwd_sums_f32)(
            L.ptr(s.dy), s.C, L.ptr(s.y), s.C, L.ptr(s.z), s.C, s.M, s.C, L.ptr(st[0]), L.ptr(st[1]), 1, 1.0, L.ptr(s.sums), s.C,
            L.ptr(s.dg), L.ptr(s.db), L.ptr(s.ws), s.nb, L.stream()))
        L.check((lib.step_bn_bwd_merge_dz_f16 if f else lib.step_bn_bwd_merge_dz_f32)(
            L.ptr(s.sums), 1, s.C, s.M, L.ptr(s.dy), s.C, L.ptr(s.y), s.C, L.ptr(s.z), s.C, s.M, s.C, L.ptr(st[0]), L.ptr(st[1]),
            L.ptr(s.gamma), 1, L.ptr(s.dz), s.C, L.ptr(s.ws), s.nb, L.stream()))


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(PASSES):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / PASSES


def measure_split(shapes, rounds):
    out = []
    for f16 in (True, False):
        ops = [Shape(f16, M, C) for M, C in shapes]
        run = {"fused": lambda: [o.fused() for o in ops], "split": lambda: [o.split() for o in ops]}
        for fn in run.values():
            fn()
        times = {k: [] for k in run}
        for _ in range(rounds):
            for k, fn in run.items():
                times[k].append(timed(fn))
        med = {k: statistics.median(v) for k, v in times.items()}
        out.append({"part": "split_at_one_rank", "precision": "fp16" if f16 else "fp32", "bn_outputs": len(shapes),
                    "rounds": rounds, "passes": PASSES, "fused_ms": round(med["fused"], 3), "split_ms": round(med["split"], 3),
                    "split_over_fused": round(med["split"] / med["fused"], 3),
                    "fused_ms_all": [round(t, 3) for t in times["fused"]], "split_ms_all": [round(t, 3) for t in times["split"]]})
        del ops
        torch.cuda.empty_cache()
    return out


def dist_worker(out_path, rounds):
    """One rank of the two-GPU measurement (under torch.distributed.run)."""
    import torch.distributed as dist
    rank = int(os.environ["RANK"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    runs = {}
    for fs in (True, False):
        cfg, nets, x, st, sg = synth.make_workload("shipped", True, "pool", B=1, device=str(dev), freeze_stats=fs)
        if not fs:
            for k, n in nets.items():
                if k != "roi_net":
                    n.train()
        runs[fs] = (cfg, nets, x, st, sg)
    orig, events = E.all_gather_rows, []

    def timed_gather(t, group):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = orig(t, group)
        b.record()
        events.append((a, b))
        return out
    E.all_gather_rows = timed_gather

    def step(fs):
        events.clear()
        torch.cuda.synchronize()
        dist.barrier()
        t0 = time.perf_counter()
        training.train_step(*runs[fs], loss_scale=1024.0, world_size=2)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        return ms, sum(a.elapsed_time(b) for a, b in events), len(events)
    for fs in (True, False):
        step(fs)
    res = {True: [], False: []}
    for _ in range(rounds):
        for fs in (True, False):
            res[fs].append(step(fs))
    if rank == 0:
        med = {fs: statistics.median(t for t, _, _ in v) for fs, v in res.items()}
        rec = {"part": "step_world_size_2_nccl", "precision": "fp16", "clips_per_rank": 1, "rounds": rounds,
               "step_ms_running_stats": round(med[True], 1), "step_ms_batch_stats_synced": round(med[False], 1),
               "exchange_ms": round(statistics.median(e for _, e, _ in res[False]), 2), "exchanges": res[False][0][2],
               "step_ms_batch_stats_synced_all": [round(t, 1) for t, _, _ in res[False]]}
        with open(out_path, "w") as f:
            json.dump(rec, f)
    dist.barrier()
    dist.destroy_process_group()


def measure_two_gpus(rounds):
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "rank0.json")
        cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node=2", os.path.abspath(__file__),
               "--dist-worker", out, "--rounds", str(rounds)]
        subprocess.run(cmd, check=True, cwd=ROOT, timeout=1800)
        with open(out) as f:
            return json.load(f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out")
    ap.add_argument("--dist-worker")
    a = ap.parse_args()
    if a.dist_worker:
        return dist_worker(a.dist_worker, a.rounds)
    if not torch.cuda.is_available():
        raise SystemExit("bn_sync_bench: needs a CUDA device")
    gpu = card(0)
    recs = measure_split(bn_shapes(), a.rounds)
    if torch.cuda.device_count() >= 2:
        recs.append(measure_two_gpus(a.rounds))
    else:
        recs.append({"part": "step_world_size_2_nccl", "result": "not measured: needs 2 GPUs"})
    lines = []
    for rec in recs:
        rec.update(gpu, torch=torch.__version__)
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
