"""3x3x3 stride-1 max pools of the step (branch_3 of every Mixed block, i3dpt.py:149-152) one by one: us and DRAM GB/s on
the compulsory bytes (input once + output once).  Inputs rotate over enough buffers to exceed the 50 MB L2; the result is
compared bit for bit with torch's max_pool3d on the zero-padded input."""
import json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from _bench import card
from step_b200 import engine as E
from step_b200.engine import Act

SHAPES = [("mixed_3b", 8, 16, 28, 28, 192), ("mixed_3c", 8, 16, 28, 28, 256), ("mixed_4b", 8, 8, 14, 14, 480),
          ("mixed_4c", 8, 8, 14, 14, 512), ("mixed_4f", 8, 8, 14, 14, 528), ("head_5b/5c", 88, 8, 7, 7, 832)]
PEAK = 3350.0   # GB/s, HBM3 of the H100 SXM data sheet (700 W)


def timed(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


print(json.dumps(card(0)), flush=True)
for name, N, T, H, W, C in SHAPES:
    nbytes = N * T * H * W * C * 2
    nbuf = max(2, int(400e6 // (2 * nbytes)) + 1)
    xs = [Act(torch.randn(N, T, H, W, C, device="cuda").half()) for _ in range(nbuf)]
    ys = [Act(torch.empty(N, T, H, W, C, device="cuda", dtype=torch.float16)) for _ in range(nbuf)]
    state = {"i": 0}

    def go():
        i = state["i"] = (state["i"] + 1) % nbuf
        E.maxpool(xs[i], (3, 3, 3), (1, 1, 1), out=ys[i])
    us = timed(go)
    E.maxpool(xs[0], (3, 3, 3), (1, 1, 1), out=ys[0])
    torch.cuda.synchronize()
    ref = torch.nn.functional.max_pool3d(torch.nn.functional.pad(xs[0].buf[:1].permute(0, 4, 1, 2, 3).float(), (1, 1, 1, 1, 1, 1)), 3, 1)
    ok = torch.equal(ref.permute(0, 2, 3, 4, 1).half(), ys[0].buf[:1])
    print("%-12s [%d,%d,%d,%d,%d] %6.1f MB  %6.1f us %5.0f GB/s (%.2f of %d)   equals torch %s"
          % (name, N, T, H, W, C, 2 * nbytes / 1e6, us, 2 * nbytes / us / 1e3, 2 * nbytes / us / 1e3 / PEAK, PEAK, ok), flush=True)
