"""GPU: every (BK, BN) tile of the wgmma convolution (STEP_CONV_TILES in step_b200/csrc/conv_umma.cu) against the SIMT
kernel on identical fp16 inputs and against the float64 convolution (bound derived in test_gpu_forward_layers.py): a Cout
that leaves the last N tile ragged, a residual, a destination split inside an N tile, and M not a multiple of the 128-row
tile (98 M tiles)."""
import os
import re
import sys

import pytest
import torch

from step_b200 import _lib as L
from step_b200 import engine as E
from step_b200.engine import Act

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _tape_reference as R  # noqa: E402

pytestmark = pytest.mark.gpu

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "step_b200", "csrc", "conv_umma.cu")


def conv_tiles():
    src = open(SRC).read()
    body = re.search(r"#define STEP_CONV_TILES\(X\)(.*?)\n\n", src, re.S).group(1)
    return [(int(a), int(b)) for a, b in re.findall(r"X\((\d+),\s*(\d+)\)", body)]


TILES = conv_tiles()


def plan(Cin, Cout):
    """(BK, BN) as pick_bk / pick_tile choose them."""
    bk = 16 if Cin <= 16 else (32 if -(-Cin // 32) * 32 < -(-Cin // 64) * 64 else 64)
    best = min((-(-Cout // bn) * bn - Cout, -(-Cout // bn), bn) for b, bn in TILES if b == bk)
    return bk, best[2]


def shape_for(bk, bn):
    """(Cin, Cout) that selects tile (bk, bn), with a ragged last N tile where the dispatcher allows one."""
    Cin = {64: 64, 32: 96, 16: 16}[bk]
    assert plan(Cin, 8)[0] == bk
    hits = [c for c in range(8, 2 * bn + 1, 8) if plan(Cin, c) == (bk, bn)]
    ragged = [c for c in hits if c % bn]
    assert hits, (bk, bn)
    return Cin, max(ragged or hits)


def run(x, w, k, scale, shift, residual, a_mode, outs):
    """conv into the channel slices `outs` = [(buffer, coff, C), ...] (more than one: split epilogue)."""
    xa = Act(x)
    acts = [Act(b, c, off) for b, off, c in outs]
    E.conv(xa, E.pack_conv_weight(w, L.F16), scale, shift, acts[0], k, (1, 1, 1), None, True,
           Act(residual) if residual is not None else None, a_mode=a_mode, extra_outs=acts[1:] or None)
    torch.cuda.synchronize()


@pytest.mark.parametrize("bk,bn", TILES, ids=["bk%d_bn%d" % t for t in TILES])
def test_every_tile_matches_simt(bk, bn):
    Cin, Cout = shape_for(bk, bn)
    N, T, H, W = 4, 4, 27, 29                      # M = 12528 = 97 x 128 + 112
    g = torch.Generator().manual_seed(bn * 100 + bk)
    x = torch.randn(N, T, H, W, Cin, generator=g).half().cuda()
    scale = (torch.rand(Cout, generator=g) + 0.5).cuda()
    shift = torch.randn(Cout, generator=g).cuda()
    res = torch.randn(N, T, H, W, Cout, generator=g).half().cuda()
    for k in ((1, 3, 3), (1, 1, 1)):
        w = (torch.randn(Cout, Cin, *k, generator=g) / (Cin * k[0] * k[1] * k[2]) ** 0.5).half().cuda()
        # residual, output in a channel slice of a wider buffer
        ref = torch.zeros(N, T, H, W, Cout + 16, dtype=torch.float16, device="cuda")
        got = torch.zeros_like(ref)
        run(x, w, k, scale, shift, res, L.A_SIMT, [(ref, 8, Cout)])
        run(x, w, k, scale, shift, res, L.A_IM2COL if k != (1, 1, 1) else L.A_AUTO, [(got, 8, Cout)])
        tol = 2e-3 * float(ref.float().abs().max()) + 2e-3
        err = float((got.float() - ref.float()).abs().max())
        assert err <= tol, (k, Cin, Cout, err, tol)
        assert float(got[..., :8].abs().max()) == 0 and float(got[..., 8 + Cout:].abs().max()) == 0
        pad = tuple(E.same_pad(kk, 1)[0] for kk in k)
        (y,), (xw,), (epi,) = R.conv_fwd(x, E.pack_conv_weight(w, L.F16), scale, shift, res, k, (1, 1, 1), pad, (T, H, W),
                                         True)
        R.check_fwd(got[..., 8:8 + Cout], y, xw, epi, R.conv_steps(k, Cin), (bk, bn, k))
    # destination split inside the first N tile (and a second one further on when Cout allows), 1x1x1, no residual
    s0 = 16
    s1 = s0 + 16 * max(1, (Cout - s0) // 32) if Cout - s0 > 16 else None
    cuts = [0, s0] + ([s1] if s1 is not None and s1 < Cout else []) + [Cout]
    w = (torch.randn(Cout, Cin, 1, 1, 1, generator=g) / Cin ** 0.5).half().cuda()
    bufs = [torch.zeros(N, T, H, W, b - a + 8, dtype=torch.float16, device="cuda") for a, b in zip(cuts, cuts[1:])]
    run(x, w, (1, 1, 1), scale, shift, None, L.A_AUTO, [(b, 8, c1 - c0) for b, c0, c1 in zip(bufs, cuts, cuts[1:])])
    ref = torch.zeros(N, T, H, W, Cout, dtype=torch.float16, device="cuda")
    run(x, w, (1, 1, 1), scale, shift, None, L.A_SIMT, [(ref, 0, Cout)])
    tol = 2e-3 * float(ref.float().abs().max()) + 2e-3
    for b, c0, c1 in zip(bufs, cuts, cuts[1:]):
        assert float((b[..., 8:].float() - ref[..., c0:c1].float()).abs().max()) <= tol, (c0, c1)
        assert float(b[..., :8].abs().max()) == 0
    widths = [c1 - c0 for c0, c1 in zip(cuts, cuts[1:])]
    ys, xws, epis = R.conv_fwd(x, E.pack_conv_weight(w, L.F16), scale, shift, None, (1, 1, 1), (1, 1, 1), (0, 0, 0), (T, H, W),
                               True, widths)
    for b, y, xw, epi in zip(bufs, ys, xws, epis):
        R.check_fwd(b[..., 8:], y, xw, epi, R.conv_steps((1, 1, 1), Cin), (bk, bn, "split", b.shape[-1]))
