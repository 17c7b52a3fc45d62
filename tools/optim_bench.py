"""Time one parameter update of the shipped configuration (scripts/train_step.sh: train.py:125-126 trains with Adam over the
159 parameter groups of utils/solver.py:get_params): the non-finite check and the Adam update of step_b200.optim.Adam over
the 159 trainable tensors (44,422,936 parameters: trunk 7,518,272, ContextNet 4,754,432, 3 x 10,716,744 per head) with
seeded random gradients, alternated with torch.optim.Adam(fused=True) and (foreach=True) on identical tensors.

    python tools/optim_bench.py [--iters N] [--train-step]

--train-step also times one shipped train_step (2 clips of 36x400x400, 34 tubes per clip) with optimizer=Adam against
lr=None (no update).  Correctness is covered by tests/test_gpu_optim.py."""
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
from step_b200 import _lib as L, optim, synth, training  # noqa: E402

GROUPS = os.path.join(ROOT, "tests", "golden", "shipped_param_groups.npz")
HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
UPDATE_BYTES_PER_PARAM = 28        # Adam reads p, g, m, v and writes p, m, v (fp32)
CHECK_BYTES_PER_PARAM = 4          # the check reads g


def groups_of(nets):
    """The reference's get_params groups for the shipped configuration (tests/golden/shipped_param_groups.npz)."""
    g = np.load(GROUPS)
    named = {k: dict(n.named_parameters()) for k, n in nets.items()}
    return [{"params": [named[str(m)][str(n)]], "lr": float(lr), "weight_decay": float(wd)}
            for m, n, lr, wd in zip(g["module"], g["name"], g["lr"], g["weight_decay"])]


def bench_update(iters):
    nets = synth.make_workload("shipped")[1]
    ref_groups = groups_of(nets)
    n_params = sum(g["params"][0].numel() for g in ref_groups)
    gen = torch.Generator(device="cuda").manual_seed(0)
    grads = [torch.randn(g["params"][0].shape, generator=gen, device="cuda") * 1e-3 for g in ref_groups]

    def make(ctor, **kw):
        groups = [dict(g, params=[g["params"][0].detach().clone()]) for g in ref_groups]
        for g, gr in zip(groups, grads):
            g["params"][0].grad = gr.clone()
        return ctor(groups, lr=7.5e-4, **kw)
    impls = {"step_b200": make(optim.Adam), "torch_fused": make(torch.optim.Adam, fused=True),
             "torch_foreach": make(torch.optim.Adam, foreach=True)}
    wall = {k: [] for k in impls}
    dev_ms = {k: [] for k in impls}
    for it in range(10 + iters):
        for name, opt in impls.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e0.record()
            opt.step()
            e1.record()
            torch.cuda.synchronize()
            if it >= 10:
                wall[name].append((time.perf_counter() - t0) * 1e3)
                dev_ms[name].append(e0.elapsed_time(e1))
    # the two launches alone (check + update) from the table the last step uploaded
    opt = impls["step_b200"]
    tables = opt._tables[torch.device("cuda", 0)]
    n = len(ref_groups)
    lib = L.lib()
    table = L.c_void_p(tables.table.data_ptr())
    kern = []
    for it in range(10 + iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        L.check(lib.step_multi_tensor_nonfinite_f32(table, n, L.ptr(tables.blocks), tables.n_blocks, L.ptr(tables.flag), L.stream()))
        L.check(lib.step_multi_tensor_adam_f32(table, n, L.ptr(tables.blocks), tables.n_blocks, L.stream()))
        e1.record()
        torch.cuda.synchronize()
        if it >= 10:
            kern.append(e0.elapsed_time(e1))
    alg_bytes = n_params * (UPDATE_BYTES_PER_PARAM + CHECK_BYTES_PER_PARAM)
    med = statistics.median
    out = {"tensors": n, "parameters": n_params, "iters": iters,
           "algorithmic_GB": {"update": round(n_params * UPDATE_BYTES_PER_PARAM / 1e9, 3),
                              "check": round(n_params * CHECK_BYTES_PER_PARAM / 1e9, 3)},
           "datasheet_floor_ms": round(alg_bytes / HBM_BYTES_PER_S * 1e3, 3),
           "step_b200_kernels_ms": round(med(kern), 3),
           "step_b200_kernels_TB_per_s": round(alg_bytes / (med(kern) * 1e-3) / 1e12, 2),
           "share_of_3.35TB_per_s": round(alg_bytes / HBM_BYTES_PER_S / (med(kern) * 1e-3), 3)}
    for name in impls:
        out[name] = {"step_wall_ms_median": round(med(wall[name]), 3), "step_wall_ms_min": round(min(wall[name]), 3),
                     "step_events_ms_median": round(med(dev_ms[name]), 3)}
    return out


def bench_train_step(reps=3):
    cfg, nets, *batch = synth.make_workload("shipped")
    opt = optim.Adam(groups_of(nets))
    times = {"optimizer_adam": [], "lr_none": []}
    for it in range(1 + reps):
        for name, kw in (("optimizer_adam", dict(optimizer=opt)), ("lr_none", dict(lr=None))):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            training.train_step(cfg, nets, *batch, **kw)
            torch.cuda.synchronize()
            if it > 0:
                times[name].append((time.perf_counter() - t0) * 1e3)
    w = synth.WORKLOADS["shipped"]
    return {"train_step_ms": {k: [round(v, 1) for v in vs] for k, vs in times.items()},
            "B": w.B, "tubes_per_clip": w.N, "clip": "%dx%dx%d" % (w.T_in, w.HW, w.HW)}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--train-step", action="store_true")
    a = ap.parse_args()
    print(json.dumps(card(0)), flush=True)
    print(json.dumps(bench_update(a.iters)), flush=True)
    if a.train_step:
        print(json.dumps(bench_train_step()), flush=True)
