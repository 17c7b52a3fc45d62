"""Per-layer times of every convolution of the C4 step (STEP inference, batch 8, T = 32, 224 x 224, 11 proposals,
max_iter = 3), through the same entry points the pipeline uses (CUDA events, 20 reps after 3 warm-ups).

    python tools/conv_bench.py [--check] [name ...]
    python tools/conv_bench.py --ksweep

For each layer: launches per step, the kernel that runs it, algorithmic and executed (zero-padded) GMAC per launch,
the conv_umma tile (BK, BN, number of N tiles), time per launch and TFLOP/s on the algorithmic FLOPs.  The last line
sums time x count over the step.  The tile columns mirror pick_bk / pick_tile in step_b200/csrc/conv_umma.cu and read
the instantiated tiles from its STEP_CONV_TILES list.  A tool, not the benchmark (bench.py).

--ksweep times a 1x1x1 conv at the head shape (M = 34,496, Cout = 256: BK 64 / BN 256, 270 tiles) for Cin = 256 ... 2048
and fits the time of one wave of tiles against K: the intercept is the part of a tile's time outside the K loop."""
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from _bench import card  # noqa: E402
from step_b200 import _lib as L, engine as E  # noqa: E402
from step_b200.engine import Act  # noqa: E402

TRUNK_56, TRUNK_28, TRUNK_14 = (8, 16, 56, 56), (8, 16, 28, 28), (8, 8, 14, 14)
HEAD, LOCAL = (88, 8, 7, 7), (704, 1, 7, 7)     # 8 clips x 11 tubes, T' = 8; the local branch runs on frames
LAYERS = [
    # name, count per step, (N, T, H, W), Cin, Cout, k     (fused 1x1 = the Mixed block's three 1x1 branches in one GEMM)
    ("stem_s2d",   1, (8, 16, 112, 112), 24, 64, (4, 4, 4)),    # the 24 live channels of the 32-channel s2d row
    ("conv2b",     1, TRUNK_56, 64, 64, (1, 1, 1)),
    ("conv2c",     1, TRUNK_56, 64, 192, (3, 3, 3)),
    ("3b_fused",   1, TRUNK_28, 192, 176, (1, 1, 1)),
    ("3b_b1b",     1, TRUNK_28, 96, 128, (3, 3, 3)),
    ("3b_b2b",     1, TRUNK_28, 16, 32, (3, 3, 3)),
    ("3b_b3",      1, TRUNK_28, 192, 32, (1, 1, 1)),
    ("3c_fused",   1, TRUNK_28, 256, 288, (1, 1, 1)),
    ("3c_b1b",     1, TRUNK_28, 128, 192, (3, 3, 3)),
    ("3c_b2b",     1, TRUNK_28, 32, 96, (3, 3, 3)),
    ("3c_b3",      1, TRUNK_28, 256, 64, (1, 1, 1)),
    ("4b_fused",   1, TRUNK_14, 480, 304, (1, 1, 1)),
    ("4b_b1b",     1, TRUNK_14, 96, 208, (3, 3, 3)),
    ("4b_b2b",     1, TRUNK_14, 16, 48, (3, 3, 3)),
    ("4b_b3",      1, TRUNK_14, 480, 64, (1, 1, 1)),
    ("4c_fused",   1, TRUNK_14, 512, 296, (1, 1, 1)),
    ("4c_b1b",     1, TRUNK_14, 112, 224, (3, 3, 3)),
    ("4c_b2b",     1, TRUNK_14, 24, 64, (3, 3, 3)),
    ("4c_b3",      1, TRUNK_14, 512, 64, (1, 1, 1)),
    ("4d_fused",   1, TRUNK_14, 512, 280, (1, 1, 1)),
    ("4d_b1b",     1, TRUNK_14, 128, 256, (3, 3, 3)),
    ("4d_b2b",     1, TRUNK_14, 24, 64, (3, 3, 3)),
    ("4d_b3",      1, TRUNK_14, 512, 64, (1, 1, 1)),
    ("4e_fused",   1, TRUNK_14, 512, 288, (1, 1, 1)),
    ("4e_b1b",     1, TRUNK_14, 144, 288, (3, 3, 3)),
    ("4e_b2b",     1, TRUNK_14, 32, 64, (3, 3, 3)),
    ("4e_b3",      1, TRUNK_14, 512, 64, (1, 1, 1)),
    ("4f_fused",   1, TRUNK_14, 528, 448, (1, 1, 1)),
    ("4f_b1b",     1, TRUNK_14, 160, 320, (3, 3, 3)),
    ("4f_b2b",     1, TRUNK_14, 32, 128, (3, 3, 3)),
    ("4f_b3",      1, TRUNK_14, 528, 128, (1, 1, 1)),
    ("5b_fused",   3, HEAD, 832, 448, (1, 1, 1)),
    ("5b_b1b",     3, HEAD, 160, 320, (3, 3, 3)),
    ("5b_b2b",     3, HEAD, 32, 128, (3, 3, 3)),
    ("5b_b3",      3, HEAD, 832, 128, (1, 1, 1)),
    ("5c_fused",   3, HEAD, 832, 624, (1, 1, 1)),
    ("5c_b1b",     3, HEAD, 192, 384, (3, 3, 3)),
    ("5c_b2b",     3, HEAD, 48, 128, (3, 3, 3)),
    ("5c_b3",      3, HEAD, 832, 128, (1, 1, 1)),
    ("downsample", 3, HEAD, 1024, 256, (1, 1, 1)),
    ("loc_res",    3, LOCAL, 1088, 1024, (1, 1, 1)),
    ("loc_conv2",  3, LOCAL, 1088, 256, (1, 1, 1)),
    ("loc_3x3",    9, LOCAL, 256, 256, (1, 3, 3)),
    # bottleneck_exit: 256 -> 1024 (+x, relu) -> 256.  Per refinement step two exits store Y and feed the next block's
    # conv1 (ReLU); the last one feeds downsample2 (bias, no ReLU) and does not store Y.
    ("loc_exit",   6, LOCAL, 256, 1024, "exit"),
    ("loc_exit_ds", 3, LOCAL, 256, 1024, "exit_ds"),
]


def conv_tiles():
    """(BK, BN) pairs of STEP_CONV_TILES in conv_umma.cu, or None for a tree without the list."""
    src = open(os.path.join(ROOT, "step_b200", "csrc", "conv_umma.cu")).read()
    m = re.search(r"#define STEP_CONV_TILES\(X\)(.*?)\n\n", src, re.S)
    return [(int(a), int(b)) for a, b in re.findall(r"X\((\d+),\s*(\d+)\)", m.group(1))] if m else None


def plan(Cin, Cout, tiles):
    """(BK, BN, n_tiles) as build_plan picks them."""
    bk = 16 if Cin <= 16 else (32 if -(-Cin // 32) * 32 < -(-Cin // 64) * 64 else 64)
    best = min((-(-Cout // bn) * bn - Cout, -(-Cout // bn), bn) for b, bn in tiles if b == bk)
    return bk, best[2], best[1]


def kernel_of(N, T, H, W, Cin, Cout, k):
    if Cin == 24 and k == (4, 4, 4):
        return "stem"
    taps = k[0] * k[1] * k[2]
    halo = taps > 1 and Cin in (16, 32, 64) and Cout <= 256 and Cin <= 32 and min(H, W) >= 14
    return "halo" if halo else "umma"


def time_us(f, reps=20):
    for _ in range(3):
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3


def ksweep():
    N, T, H, W = HEAD
    M, Cout = N * T * H * W, 256
    tiles = -(-M // 128)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    waves = -(-tiles // sms)
    print("ksweep: 1x1x1 conv, M = %d, Cout = %d, %d tiles of 128 x 256 on %d SMs (%d waves)" % (M, Cout, tiles, sms, waves))
    ks, per_wave = [], []
    for Cin in (256, 512, 1024, 2048):
        x = Act(torch.randn(N, T, H, W, Cin, device="cuda").half())
        w = (torch.randn(Cout, 1, Cin, device="cuda") / Cin ** 0.5).half()
        out = Act(torch.empty(N, T, H, W, Cout, device="cuda", dtype=torch.float16))
        sc, sh = torch.ones(Cout, device="cuda"), torch.zeros(Cout, device="cuda")
        us = time_us(lambda: E.conv(x, w, sc, sh, out, (1, 1, 1), (1, 1, 1), None, True, None), reps=50)
        ks.append(Cin)
        per_wave.append(us / waves)
        print("K %5d  %8.1f us  %6.2f us per wave  %6.1f TFLOP/s" % (Cin, us, us / waves, 2.0 * M * Cin * Cout / us / 1e6))
    n = len(ks)
    mk, mt = sum(ks) / n, sum(per_wave) / n
    slope = sum((k - mk) * (t - mt) for k, t in zip(ks, per_wave)) / sum((k - mk) ** 2 for k in ks)
    icept = mt - slope * mk
    t1024 = icept + slope * 1024
    print("fit per wave: %.2f us + %.4f us per K (%.2f us per 64-channel block); intercept = %.0f %% of a K = 1024 tile"
          % (icept, slope, slope * 64, 100.0 * icept / t1024))


def main():
    print(json.dumps(card(0)), flush=True)
    if "--ksweep" in sys.argv:
        ksweep()
        return
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    check = "--check" in sys.argv
    tiles = conv_tiles()
    torch.manual_seed(0)
    total_ms = 0.0
    print("%-11s %3s %4s %9s %9s %3s %4s %3s %9s %8s" % ("layer", "n", "kern", "GMAC", "exec_GMAC", "BK", "BN", "nt",
                                                         "us", "TFLOP/s"))
    for name, count, (N, T, H, W), Cin, Cout, k in LAYERS:
        if args and name not in args:
            continue
        M = N * T * H * W
        if k in ("exit", "exit_ds"):
            h = Act(torch.randn(N, T, H, W, Cin, device="cuda").half())
            w3 = (torch.randn(Cout, 1, Cin, device="cuda") / Cin ** 0.5).half()
            x = Act(torch.randn(N, T, H, W, Cout, device="cuda").half())
            w1 = (torch.randn(Cin, 1, Cout, device="cuda") / Cout ** 0.5).half()
            z = Act(torch.empty(N, T, H, W, Cin, device="cuda", dtype=torch.float16))
            if k == "exit":
                y = Act(torch.empty(N, T, H, W, Cout, device="cuda", dtype=torch.float16))
                f = lambda: E.bottleneck_exit(h, w3, x, w1, None, True, z, y)
            else:
                b = torch.randn(Cin, device="cuda")
                f = lambda: E.bottleneck_exit(h, w3, x, w1, b, False, z)
            gmac = 2.0 * M * Cin * Cout / 1e9
            kern, exec_gmac, tile = "exit", gmac, ("-", "-", "-")
        elif name == "stem_s2d":
            # Unit3Dpy.forward_s2d's problem: 24 live channels in rows of 32 and pack_stem_s2d weights, whose zero last t
            # tap plane channels 16..23 the stem kernel does not multiply (88 k16 steps per pixel)
            buf = torch.randn(N, T, H, W, 32, device="cuda").half()
            buf[..., 24:] = 0
            x = Act(buf, Cin)
            w = E.pack_stem_s2d(torch.randn(Cout, 3, 7, 7, 7, device="cuda") / 1029 ** 0.5)
            out = Act(torch.empty(N, T, H, W, Cout, device="cuda", dtype=torch.float16))
            sc, sh = torch.ones(Cout, device="cuda"), torch.zeros(Cout, device="cuda")
            pad = (1, 1, 1)
            f = lambda: E.conv(x, w, sc, sh, out, k, (1, 1, 1), pad, True, None, a_mode=L.A_HALO, zero_cin_last_kt=12)
            gmac = M * Cout * 3 * 7 ** 3 / 1e9
            kern, exec_gmac, tile = kernel_of(N, T, H, W, Cin, Cout, k), M * Cout * 88 * 16 / 1e9, ("-", "-", "-")
        else:
            taps = k[0] * k[1] * k[2]
            x = Act(torch.randn(N, T, H, W, Cin, device="cuda").half())
            w = (torch.randn(Cout, taps, Cin, device="cuda") / (Cin * taps) ** 0.5).half()
            out = Act(torch.empty(N, T, H, W, Cout, device="cuda", dtype=torch.float16))
            sc, sh = torch.ones(Cout, device="cuda"), torch.zeros(Cout, device="cuda")
            pad = (1, 1, 1) if name == "stem_s2d" else None
            f = lambda: E.conv(x, w, sc, sh, out, k, (1, 1, 1), pad, True, None)
            gmac = M * Cin * Cout * taps / 1e9
            kern = kernel_of(N, T, H, W, Cin, Cout, k)
            if kern == "umma" and tiles:
                bk, bn, nt = plan(Cin, Cout, tiles)
                exec_gmac = M * (-(-Cin // bk) * bk) * (bn * nt) * taps / 1e9
                tile = (bk, bn, nt)
            else:
                exec_gmac, tile = float("nan"), ("-", "-", "-")
        us = time_us(f)
        total_ms += us * count / 1e3
        line = "%-11s %3d %4s %9.2f %9.2f %3s %4s %3s %9.1f %8.1f" % (name, count, kern, gmac, exec_gmac, tile[0], tile[1],
                                                                     tile[2], us, 2 * gmac / us * 1e3)
        if check and not isinstance(k, str):   # spot check against torch on two images (tool only: the parity tests live in tests/)
            import torch.nn.functional as F
            xs = x.buf[:2].float().permute(0, 4, 1, 2, 3)
            ws = w.float().view(Cout, k[0], k[1], k[2], w.shape[2]).permute(0, 4, 1, 2, 3)
            pd = pad if pad is not None else tuple(E.same_pad(kk, 1)[0] for kk in k)
            hi = tuple(kk - 1 - q for kk, q in zip(k, pd))
            ref = torch.relu(F.conv3d(F.pad(xs, (pd[2], hi[2], pd[1], hi[1], pd[0], hi[0])), ws).permute(0, 2, 3, 4, 1))
            line += "  rel_err %.1e" % float((out.buf[:2].float() - ref).abs().max() / ref.abs().max())
        print(line, flush=True)
    print("sum over the step (time x count): %.3f ms" % total_ms)


if __name__ == "__main__":
    main()
