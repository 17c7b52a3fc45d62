"""Time individual conv layers of the C4 workload through the C ABI (CUDA events, 20 reps after 3 warm-ups).
Knobs via env: STEP_B200_AMODE."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from step_b200 import _lib as L, engine as E
from step_b200.engine import Act

LAYERS = {
    # name: (N, T, H, W, Cin, Cout, k, pad, residual)
    "stem_s2d":   (8, 16, 112, 112, 32, 64, (4, 4, 4), (1, 1, 1), False),
    "conv2c":     (8, 16, 56, 56, 64, 192, (3, 3, 3), None, False),
    "3b_b2b":     (8, 16, 28, 28, 16, 32, (3, 3, 3), None, False),
    "3c_b2b":     (8, 16, 28, 28, 32, 96, (3, 3, 3), None, False),
    "4e_b2b":     (8, 8, 14, 14, 32, 64, (3, 3, 3), None, False),
    "4f_b2b":     (8, 8, 14, 14, 32, 128, (3, 3, 3), None, False),
    "5b_b2b":     (88, 8, 7, 7, 32, 128, (3, 3, 3), None, False),
    "3b_b1b":     (8, 16, 28, 28, 96, 128, (3, 3, 3), None, False),
    "3c_b1b":     (8, 16, 28, 28, 128, 192, (3, 3, 3), None, False),
    "4c_b1b":     (8, 8, 14, 14, 112, 224, (3, 3, 3), None, False),
    "4e_b1b":     (8, 8, 14, 14, 144, 288, (3, 3, 3), None, False),
    "5c_b2b":     (88, 8, 7, 7, 48, 128, (3, 3, 3), None, False),
    "4f_b1b":     (8, 8, 14, 14, 160, 320, (3, 3, 3), None, False),
    "5b_b1b":     (88, 8, 7, 7, 160, 320, (3, 3, 3), None, False),
    "5c_b1b":     (88, 8, 7, 7, 192, 384, (3, 3, 3), None, False),
    "loc_1088":   (704, 1, 7, 7, 1088, 1024, (1, 1, 1), None, False),
    "loc_3x3":    (704, 1, 7, 7, 256, 256, (1, 3, 3), None, False),
    "loc_res":    (704, 1, 7, 7, 256, 1024, (1, 1, 1), None, True),
    "loc_nores":  (704, 1, 7, 7, 256, 1024, (1, 1, 1), None, False),
    "loc_1024":   (704, 1, 7, 7, 1024, 256, (1, 1, 1), None, False),
    "5b_fused":   (88, 8, 7, 7, 832, 448, (1, 1, 1), None, False),
    "4b_fused":   (8, 8, 14, 14, 480, 304, (1, 1, 1), None, False),
    "conv2b":     (8, 16, 56, 56, 64, 64, (1, 1, 1), None, False),
    "3b_fused":   (8, 16, 28, 28, 192, 176, (1, 1, 1), None, False),
    "3c_fused":   (8, 16, 28, 28, 256, 288, (1, 1, 1), None, False),
    "3c_b3":      (8, 16, 28, 28, 256, 64, (1, 1, 1), None, False),
    "4c_fused":   (8, 8, 14, 14, 512, 296, (1, 1, 1), None, False),
    "5c_fused":   (88, 8, 7, 7, 832, 624, (1, 1, 1), None, False),
    "5b_b3":      (88, 8, 7, 7, 832, 128, (1, 1, 1), None, False),
    "4b_b1b":     (8, 8, 14, 14, 96, 208, (3, 3, 3), None, False),
    "4d_b1b":     (8, 8, 14, 14, 128, 256, (3, 3, 3), None, False),
}
names = sys.argv[1:] or list(LAYERS)
torch.manual_seed(0)
for name in names:
    N, T, H, W, Cin, Cout, k, pad, res = LAYERS[name]
    x = Act(torch.randn(N, T, H, W, Cin, device="cuda").half())
    w = (torch.randn(Cout, k[0] * k[1] * k[2], Cin, device="cuda") / (Cin * k[0] * k[1] * k[2]) ** 0.5).half()
    out = Act(torch.empty(N, T, H, W, Cout, device="cuda", dtype=torch.float16))
    r = Act(torch.randn(N, T, H, W, Cout, device="cuda").half()) if res else None
    sc = torch.ones(Cout, device="cuda"); sh = torch.zeros(Cout, device="cuda")
    am = int(os.environ['CB_AMODE']) if os.environ.get('CB_AMODE') and k != (1, 1, 1) else None
    f = lambda: E.conv(x, w, sc, sh, out, k, (1, 1, 1), pad, True, r, a_mode=am)
    for _ in range(3): f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    e0.record()
    for _ in range(reps): f()
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / reps * 1e3
    gf = 2.0 * N * T * H * W * Cin * Cout * k[0] * k[1] * k[2] / 1e9
    # spot check against torch on a sample of output pixels (tool only: the parity tests live in tests/)
    err = -1.0
    if os.environ.get("CB_CHECK", "1") == "1":
        import torch.nn.functional as F
        n_s = min(N, 2)
        xs = x.buf[:n_s].float().permute(0, 4, 1, 2, 3)
        ws = w.float().view(Cout, k[0], k[1], k[2], Cin).permute(0, 4, 1, 2, 3)
        pd = pad if pad is not None else tuple(E.same_pad(kk, 1)[0] for kk in k)
        hi = tuple(kk - 1 - q for kk, q in zip(k, pd))
        xp = F.pad(xs, (pd[2], hi[2], pd[1], hi[1], pd[0], hi[0]))
        ref = F.conv3d(xp, ws).permute(0, 2, 3, 4, 1)
        if res:
            ref = ref + r.buf[:n_s].float()
        ref = torch.relu(ref)
        err = float((out.buf[:n_s].float() - ref).abs().max() / ref.abs().max())
    print("%-10s %8.1f us  %7.1f TFLOP/s  %4.1f%% of 989 (H100 SXM data sheet; algorithmic %.1f GFLOP)  rel_err %.1e" % (name, us, gf / us * 1e3, gf / us * 1e3 / 9.89, gf, err))
