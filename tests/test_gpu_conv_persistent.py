"""GPU: the persistent tile loop of the wgmma convolution (conv_umma.cu), where every CTA runs several tiles in turn.  Every
(BK, BN) tile of STEP_CONV_TILES at the refinement heads' shape (88 tubes x 8 frames x 7 x 7: 270 M tiles, the last one 64
rows) with an N tile count that does not divide the SM count, so one CTA meets different N tiles and with them different
scale / shift.  Against the SIMT kernel on identical fp16 inputs and against the float64 convolution: 1x3x3 IM2COL and
1x1x1 LINEAR with a residual into a channel slice between untouched neighbours, a 1x1x1 split into three destinations, and
a 3x3x3 BOX-mode case."""
import os
import sys

import pytest
import torch

from step_b200 import _lib as L
from step_b200 import engine as E

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _tape_reference as R  # noqa: E402
from test_gpu_conv_tiles import TILES, plan, run  # noqa: E402

pytestmark = pytest.mark.gpu

N, T, H, W = 88, 8, 7, 7                           # M = 34496 = 269 x 128 + 64
CIN = {64: 64, 32: 96, 16: 16}


def cout_for(bk, bn, sms):
    """Cout that selects tile (bk, bn) with at least two N tiles, preferring a count that does not divide the grid (one or
    two CTAs per SM), so that the grid stride moves a CTA to another N tile, then a ragged last N tile, then the fewest
    tiles."""
    hits = [c for c in range(bn + 8, 8 * bn + 1, 8) if plan(CIN[bk], c) == (bk, bn)]
    assert hits, (bk, bn)
    return min(hits, key=lambda c: ((2 * sms) % -(-c // bn) == 0, c % bn == 0, -(-c // bn), c))


def check(x, w, k, scale, shift, res, a_mode, Cout, what):
    """conv into a channel slice [8, 8 + Cout) of a wider buffer: SIMT comparison, untouched neighbours, float64 bound."""
    ref = torch.zeros(N, T, H, W, Cout + 16, dtype=torch.float16, device="cuda")
    got = torch.zeros_like(ref)
    run(x, w, k, scale, shift, res, L.A_SIMT, [(ref, 8, Cout)])
    run(x, w, k, scale, shift, res, a_mode, [(got, 8, Cout)])
    tol = 2e-3 * float(ref.float().abs().max()) + 2e-3
    err = float((got.float() - ref.float()).abs().max())
    assert err <= tol, (what, err, tol)
    assert float(got[..., :8].abs().max()) == 0 and float(got[..., 8 + Cout:].abs().max()) == 0, what
    pad = tuple(E.same_pad(kk, 1)[0] for kk in k)
    (y,), (xw,), (epi,) = R.conv_fwd(x, E.pack_conv_weight(w, L.F16), scale, shift, res, k, (1, 1, 1), pad, (T, H, W), True)
    R.check_fwd(got[..., 8:8 + Cout], y, xw, epi, R.conv_steps(k, x.shape[-1]), what)


def inputs(bk, bn, Cout, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, T, H, W, CIN[bk], generator=g).half().cuda()
    scale = (torch.rand(Cout, generator=g) + 0.5).cuda()
    shift = torch.randn(Cout, generator=g).cuda()
    res = torch.randn(N, T, H, W, Cout, generator=g).half().cuda()
    return g, x, scale, shift, res


@pytest.mark.parametrize("bk,bn", TILES, ids=["bk%d_bn%d" % t for t in TILES])
def test_every_tile_over_many_tiles_per_cta(bk, bn):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    Cout = cout_for(bk, bn, sms)
    n_tiles = -(-Cout // bn)
    assert -(-N * T * H * W // 128) * n_tiles > 2 * sms     # every CTA of the grid (at most 2 per SM) runs several tiles
    g, x, scale, shift, res = inputs(bk, bn, Cout, bn * 100 + bk)
    Cin = CIN[bk]
    for k, a_mode in (((1, 3, 3), L.A_IM2COL), ((1, 1, 1), L.A_AUTO)):
        w = (torch.randn(Cout, Cin, *k, generator=g) / (Cin * k[0] * k[1] * k[2]) ** 0.5).half().cuda()
        check(x, w, k, scale, shift, res, a_mode, Cout, (bk, bn, Cout, k))
    # two cuts, at multiples of 16 inside different N tiles: three destinations, 1x1x1, no residual
    cuts = [0, 16 * (Cout // 48), 16 * (Cout // 24), Cout]
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


def test_box_mode_over_many_tiles_per_cta():
    """3x3x3 in BOX mode (boxes of output pixels with overhang rows past the 7 x 7 x 8 map), BK 64 / BN 256."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    bk, bn = 64, 256
    Cout = cout_for(bk, bn, sms)
    g, x, scale, shift, res = inputs(bk, bn, Cout, 7)
    k = (3, 3, 3)
    w = (torch.randn(Cout, CIN[bk], *k, generator=g) / (CIN[bk] * 27) ** 0.5).half().cuda()
    check(x, w, k, scale, shift, res, L.A_BOX, Cout, ("box", Cout))
