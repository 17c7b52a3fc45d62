"""GPU: the ROIAlign and ROIPool backwards are deterministic in both layouts.

1. The channels-last entries reproduce tests/golden/roi_bwd_bits.npz, the SHA-256 of their outputs as the build before
   the shared kernels made them (tests/golden/make_roi_bwd_golden.py): train_step's ROI backward kept its summation
   order bit for bit.
2. The reference-layout entries (NCHW, the ones roi_layers.py's autograd Functions call) equal the channels-last ones,
   transposed, bit for bit.
3. At the edges both agree with float64 within the bound of tests/_tape_reference.py: sampling ratio 0 and 2, ROIs
   across, outside and of zero area, unsorted rows on several frames, frames without a row, R = 0, C = 1, 3 and 832, and
   a plane larger than one CTA's shared-memory tile.  A row whose frame index is outside [0, K) contributes nothing and
   nothing outside grad_in is written.
4. Every entry gives the same bytes when called again, and on another stream.
5. The unedited drivers repeat: two train.py / train_cls.py iterations (tests/test_gpu_autograd.py) from the same nets,
   clips and generator state give bit-identical gradients and bit-identical parameters after step_b200.optim.Adam."""
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.join(HERE, "golden"), os.path.dirname(HERE)]
import _tape_reference as TR  # noqa: E402
import make_roi_bwd_golden as G  # noqa: E402
from step_b200 import _lib as L  # noqa: E402

pytestmark = pytest.mark.gpu
SCALE = 1.0 / 16.0


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def bits():
    return np.load(os.path.join(HERE, "golden", "roi_bwd_bits.npz"))


# ---- 1. the pinned bits --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [c["name"] for c in G.CASES])
def test_channels_last_entries_reproduce_the_pinned_bits(bits, name):
    assert json.loads(str(bits["cases"])) == G.CASES
    c = next(c for c in G.CASES if c["name"] == name)
    for tag, dt in (("f32", torch.float32), ("f16", torch.float16)):
        gin, am = G.run(c, dt)
        if am is not None:
            assert G.sha(am) == str(bits["%s_argmax_sha" % name])
        if name in G.EDGE:
            np.testing.assert_array_equal(gin.cpu().numpy(), bits["%s_%s_out" % (name, tag)])
        assert G.sha(gin) == str(bits["%s_%s_sha" % (name, tag)]), (name, tag)


# ---- helpers -------------------------------------------------------------------------------------------------------------
def align_nchw(g, rois, K, H, W, sr, out=None):
    """step_roi_align_bwd_nchw_f32: g [R, C, ph, pw] fp32 -> grad_in [K, C, H, W] (into `out` when given)."""
    R, C, ph, pw = g.shape
    gin = torch.full((K, C, H, W), 7.0, device="cuda") if out is None else out
    L.check(L.lib().step_roi_align_bwd_nchw_f32(L.ptr(g), L.ptr(rois), R, SCALE, ph, pw, K, C, H, W, sr, L.ptr(gin), L.stream()))
    return gin


def align_nhwc(g, rois, K, H, W, sr):
    """step_roi_align_bwd_nhwc: g [R, ph, pw, C] -> grad_in [K, H, W, C]."""
    R, ph, pw, C = g.shape
    gin = torch.full((K, H, W, C), 7.0, device="cuda")
    L.check(L.lib().step_roi_align_bwd_nhwc(L.ptr(g), L.dt(g), C, L.ptr(rois), R, SCALE, ph, pw, K, H, W, C, sr, L.ptr(gin), C,
                                            L.stream()))
    return gin


def pool_fwd_nchw(feat, rois, ph=7, pw=7):
    K, C, H, W = feat.shape
    R = rois.shape[0]
    out = torch.empty((R, C, ph, pw), device="cuda")
    am = torch.empty((R, C, ph, pw), dtype=torch.int32, device="cuda")
    L.check(L.lib().step_roi_pool_fwd_nchw_f32(L.ptr(feat), K, C, H, W, L.ptr(rois), R, SCALE, ph, pw, L.ptr(out), L.ptr(am),
                                               L.stream()))
    return out, am


def pool_nchw(g, am, rois, K, H, W, out=None):
    R, C, ph, pw = g.shape
    gin = torch.full((K, C, H, W), 7.0, device="cuda") if out is None else out
    L.check(L.lib().step_roi_pool_bwd_nchw_f32(L.ptr(g), L.ptr(am), L.ptr(rois), R, ph, pw, K, C, H, W, L.ptr(gin), L.stream()))
    return gin


def pool_nhwc(g, am, rois, K, H, W):
    """step_roi_pool_bwd_slice_nhwc over the whole map (roi_T = feat_T = K, t_start = 0) on a zeroed grad_in."""
    R, ph, pw, C = g.shape
    gin = torch.zeros((K, H, W, C), device="cuda")
    L.check(L.lib().step_roi_pool_bwd_slice_nhwc(L.ptr(g), L.dt(g), C, L.ptr(am), L.ptr(rois), R, ph, pw, K, H, W, C, K, K, 0,
                                                 L.ptr(gin), C, L.stream()))
    return gin


def edge_rois(K, H, W, R, seed, frames=None):
    """R rows on frames drawn from [0, frames) (default K) in no order, boxes across and beyond the map, one of zero area,
    one wholly outside, one larger than the map."""
    rng = np.random.default_rng(seed)
    iw, ih = W / SCALE, H / SCALE
    f = rng.integers(0, K if frames is None else frames, R)
    x1, y1 = rng.uniform(-0.2, 1.0, R) * iw, rng.uniform(-0.2, 1.0, R) * ih
    r = np.stack([f, x1, y1, x1 + rng.uniform(0, 0.8, R) * iw, y1 + rng.uniform(0, 0.8, R) * ih], 1).astype(np.float32)
    if R >= 3:
        r[0, 3:] = r[0, 1:3]
        r[1, 1:] = [iw * 1.3, ih * 1.2, iw * 1.6, ih * 1.5]
        r[2, 1:] = [-iw, -ih, 2 * iw, 2 * ih]
    return cu(r)


nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()


# ---- 2. layouts agree ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,H,W,C,R,sr", [(18, 25, 25, 832, 204, 0), (3, 9, 7, 12, 10, 2), (2, 100, 100, 8, 6, 0)])
def test_nchw_entries_equal_the_channels_last_ones(K, H, W, C, R, sr):
    rois = edge_rois(K, H, W, R, seed=K + C)
    g = torch.randn(R, C, 7, 7, generator=torch.Generator().manual_seed(1)).cuda()
    assert torch.equal(nhwc(align_nchw(g, rois, K, H, W, sr)), align_nhwc(nhwc(g), rois, K, H, W, sr))
    if H * W <= 6400:   # the channels-last ROIPool backward's documented limit
        feat = torch.randn(K, C, H, W, generator=torch.Generator().manual_seed(2)).cuda()
        _, am = pool_fwd_nchw(feat, rois)
        assert torch.equal(nhwc(pool_nchw(g, am, rois, K, H, W)), pool_nhwc(nhwc(g), nhwc(am), rois, K, H, W))


# ---- 3. edges against float64 --------------------------------------------------------------------------------------------
def check_align(got_nchw, g, rois, K, H, W, sr):
    ref, mag, n = TR.roi_align_bwd(nhwc(g), rois, SCALE, 7, 7, K, H, W, sampling_ratio=sr)
    got = nhwc(got_nchw)
    assert TR.roi_align_bwd_check(got, torch.zeros_like(got), ref, mag, n) <= 1.0


def pool_ref(g, am, rois, K, H, W):
    """float64 ROIPool backward and the sum of |terms| per element: grad_in[frame(r), c, argmax] += g (the scatter of
    ROIPool_cuda.cu:103-132)."""
    R, C, ph, pw = g.shape
    out = torch.zeros(K, C, H * W, dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(out)
    cidx = torch.arange(C, device="cuda").unsqueeze(1).expand(C, ph * pw)
    for r in range(R):
        f = int(rois[r, 0])
        if not 0 <= f < K:
            continue
        a, v = am[r].reshape(C, -1).long(), g[r].reshape(C, -1).double()
        ok = a >= 0
        out[f].index_put_((cidx[ok], a[ok]), v[ok], accumulate=True)
        mag[f].index_put_((cidx[ok], a[ok]), v[ok].abs(), accumulate=True)
    return out.view(K, C, H, W), mag.view(K, C, H, W)


def check_pool(got, ref, mag):
    """fp32 sums of at most 64 terms here: within 64 roundings of the float64 sum (u32 = 2^-24)."""
    assert bool(((got.double() - ref).abs() <= 64 * 2 ** -24 * mag).all())


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.flatten().contiguous().view(torch.uint8),
                                                                     b.flatten().contiguous().view(torch.uint8))


@pytest.mark.parametrize("C", [1, 3, 832])
@pytest.mark.parametrize("sr", [0, 2])
def test_nchw_edges_against_float64(C, sr):
    K, H, W, R = 5, 13, 11, 23
    rois = edge_rois(K, H, W, R, seed=C * 10 + sr, frames=K - 1)        # frame K - 1 has no row
    g = torch.randn(R, C, 7, 7, generator=torch.Generator().manual_seed(C)).cuda()
    got = align_nchw(g, rois, K, H, W, sr)
    check_align(got, g, rois, K, H, W, sr)
    assert bool((got[K - 1] == 0).all()) and not bool(torch.signbit(got[K - 1]).any())
    feat = torch.randn(K, C, H, W, generator=torch.Generator().manual_seed(3)).cuda()
    _, am = pool_fwd_nchw(feat, rois)
    check_pool(pool_nchw(g, am, rois, K, H, W), *pool_ref(g, am, rois, K, H, W))


def test_plane_larger_than_one_tile_against_float64():
    K, C, H, W, R = 2, 8, 100, 100, 9
    rois = edge_rois(K, H, W, R, seed=7)
    g = torch.randn(R, C, 7, 7, generator=torch.Generator().manual_seed(4)).cuda()
    check_align(align_nchw(g, rois, K, H, W, 0), g, rois, K, H, W, 0)
    feat = torch.randn(K, C, H, W, generator=torch.Generator().manual_seed(5)).cuda()
    _, am = pool_fwd_nchw(feat, rois)
    check_pool(pool_nchw(g, am, rois, K, H, W), *pool_ref(g, am, rois, K, H, W))


def test_no_rows_gives_zeros():
    rois = torch.zeros((0, 5), device="cuda")
    g = torch.zeros((0, 3, 7, 7), device="cuda")
    assert bool((align_nchw(g, rois, 2, 5, 6, 0) == 0).all())
    assert bool((pool_nchw(g, torch.zeros((0, 3, 7, 7), dtype=torch.int32, device="cuda"), rois, 2, 5, 6) == 0).all())


def test_rows_outside_the_frame_range():
    """The forward reads the frame the index addresses in the storage around the input (no bounds check, as in the
    reference's kernels); the backward drops such a row and writes nothing outside grad_in."""
    from step_b200.roi_layers import roi_align
    K, C, H, W = 3, 4, 9, 9
    big = torch.randn(K + 2, C, H, W, generator=torch.Generator().manual_seed(6)).cuda()
    inner = big[1:K + 1]
    box = [20.0, 16.0, 100.0, 120.0]
    rois = torch.tensor([[-1.0] + box, [float(K)] + box, [1.0] + box], device="cuda")
    out = roi_align(inner, rois, (7, 7), SCALE, 0)
    want = roi_align(big, rois + torch.tensor([1.0, 0, 0, 0, 0], device="cuda"), (7, 7), SCALE, 0)
    assert torch.equal(out, want)               # frames -1 and K of `inner` are big[0] and big[K + 1]
    g = torch.randn(3, C, 7, 7, generator=torch.Generator().manual_seed(8)).cuda()
    guard = torch.full((K + 2, C, H, W), 3.0, device="cuda")
    align_nchw(g, rois, K, H, W, 0, out=guard[1:K + 1])
    assert bool((guard[0] == 3).all()) and bool((guard[K + 1] == 3).all())
    alone = align_nchw(g[2:], rois[2:], K, H, W, 0)
    assert torch.equal(guard[1:K + 1], alone)
    _, am = pool_fwd_nchw(big[1:K + 1].contiguous(), rois[2:])
    am = torch.cat([am, am, am])
    guard.fill_(3.0)
    pool_nchw(g, am, rois, K, H, W, out=guard[1:K + 1])
    assert bool((guard[0] == 3).all()) and bool((guard[K + 1] == 3).all())
    assert torch.equal(guard[1:K + 1], pool_nchw(g[2:], am[2:], rois[2:], K, H, W))


# ---- 4. run to run -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["shipped_step9", "pool_shipped_step9", "shipped_whole", "edge_sr2"])
def test_channels_last_entries_repeat_on_any_stream(name):
    c = next(c for c in G.CASES if c["name"] == name)
    for dt in (torch.float32, torch.float16):
        a, _ = G.run(c, dt)
        b, _ = G.run(c, dt)
        s, _ = G.run(c, dt, stream=torch.cuda.Stream())
        assert same_bits(a, b) and same_bits(a, s)


def test_nchw_entries_repeat_on_any_stream():
    K, C, H, W, R = 18, 832, 25, 25, 612
    rois = edge_rois(K, H, W, R, seed=9)
    g = torch.randn(R, C, 7, 7, generator=torch.Generator().manual_seed(9)).cuda()
    feat = torch.randn(K, C, H, W, generator=torch.Generator().manual_seed(10)).cuda()
    _, am = pool_fwd_nchw(feat, rois)
    runs = []
    for s in (None, None, torch.cuda.Stream()):
        with torch.cuda.stream(s or torch.cuda.current_stream()):
            runs.append((align_nchw(g, rois, K, H, W, 0), pool_nchw(g, am, rois, K, H, W)))
        torch.cuda.synchronize()
    for a, p in runs[1:]:
        assert same_bits(a, runs[0][0]) and same_bits(p, runs[0][1])


# ---- 5. the drivers repeat -----------------------------------------------------------------------------------------------
def driver_twice(workload, pool_mode, fp16, scale):
    from step_b200 import optim, synth
    from test_gpu_autograd import named, train_cls_iteration, train_py_iteration
    gen = torch.cuda.default_generators[0]
    state = gen.get_state()
    out = []
    for _ in range(2):
        cfg, nets, clips, st, sg = synth.make_workload(workload, fp16=fp16, pool_mode=pool_mode, dropout=0.3)
        opt = optim.Adam(list(named(nets).values()), lr=1e-5)
        gen.set_state(state)
        if workload == "cls":
            train_cls_iteration(cfg, nets, clips, st, sg)
        else:
            train_py_iteration(cfg, nets, clips, st, sg, scale=scale)
        grads = {k: p.grad.detach().clone() for k, p in named(nets).items()}
        for p in named(nets).values():
            p.grad.div_(scale)
        opt.step()
        out.append((grads, {k: p.detach().clone() for k, p in named(nets).items()}))
        del nets, opt
    return out


@pytest.mark.parametrize("workload,pool_mode,fp16,scale", [
    ("shipped", "align", False, 1.0), ("shipped", "pool", False, 1.0), ("shipped", "align", True, 1024.0),
    ("cls", "align", False, 1.0)])
def test_driver_iterations_repeat_bit_for_bit(workload, pool_mode, fp16, scale):
    (ga, pa), (gb, pb) = driver_twice(workload, pool_mode, fp16, scale)
    assert set(ga) == set(gb) and ga
    differ = [k for k in ga if not same_bits(ga[k], gb[k])]
    assert not differ, differ[:10]
    differ = [k for k in pa if not same_bits(pa[k], pb[k])]
    assert not differ, differ[:10]
