"""GPU: the launches of train_step outside the tape, each against a float64 reference on the operands it read
(tests/_tape_reference.py derives every bound), and the ROIAlign backward on its own at the shapes and edges where it can
go wrong.

ROIAlign backward (step_roi_align_bwd_nhwc and step_roi_align_bwd_slice_nhwc, fp32 and fp16 gradients), against
roi_align_bwd within (n + 3) u32 (sum |term| + |init|), elements without a term bit-identical to their initial value:
  * the shipped geometry: 2 clips x 9 frames of 25x25x832, 34 tubes per clip (synth.make_train_case at 400x400), the three
    steps' slices (roi_T 3 / 3 / 9, t_start 3 / 3 / 0) into one pre-filled buffer, the fp16 gradient read at row pitch
    832 + 256 as from the head's concat buffer;
  * edge cases on 28x28 maps: a whole-image ROI (grid exactly 4x4: 784 samples, one full sample table), ROIs of grid 5x5
    and up (two or more passes over the table) for 7x7 and 5x3 bins, sampling_ratio 2, a degenerate ROI (x2 < x1),
    corners in [-16, 0) (samples in [-1, 0] clamped) and below -16 (samples dropped), ROIs touching and passing the
    bottom and right edges, a frame with 40 overlapping ROIs, a slice frame without ROI and frames outside the slice.

train_step launch by launch: one un-instrumented and one instrumented step in three geometries (the shipped
configuration with ROIAlign, the same with ROIPool, the class-only stage).  Test-local wrappers around
training.head_losses, cls_loss, linear_backward, context_grad_reduce, roi_align_backward_slice and
roi_pool_backward_slice clone what each launch reads before it and what it wrote right after, on the issuing stream;
tape_backward is spied as in test_gpu_backward_layers.py for the gradient seeds, from which the raw launches
(mean_mid_bwd of the classifier's temporal mean and of ContextNet's spatial mean, f32_accum_f16 of the regressors' input
gradient and of the trunk's output gradient) are checked exactly: each is one fp32 operation on an fp16 zero and one
rounding.  The ROIPool backward is checked against a float64 scatter through the recorded argmax with the same
(n + 3) u32 bound, after checking that every argmax points at a maximum of its ROIPool bin and that the pooled value the
head read is that pixel's value (wrappers around ROINet.pool_into).  The space-to-depth clip the stem reads (a wrapper
around Unit3Dpy.forward_s2d) must unpack to the fp16 clip exactly, with zero padding channels.  Finally every step::
kernel a profiled train_step launches must be on CHECKED, which names the test that compares it with float64.
"""
import json
import math
import os
import re
import subprocess
import sys
import time

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [HERE, ROOT]
import _tape_reference as R  # noqa: E402
from _train_case import SHIPPED  # noqa: E402
from step_b200.synth import device_nets  # noqa: E402
from step_b200 import synth  # noqa: E402

pytestmark = pytest.mark.gpu
SCALE = 1.0 / 16.0
FWD = "tests/test_gpu_forward_layers.py::test_every_launch_against_float64"
BWD_CHAIN = "tests/test_gpu_backward_layers.py::test_chain_of_real_gradients_through_heads_context_and_trunk"
BWD_ENTRY = "tests/test_gpu_backward_layers.py::test_every_tape_entry_in_isolation"
HERE_LAUNCH = "tests/test_gpu_train_launches.py::test_every_launch_against_float64"
# Every step:: kernel of train_step, by name pattern, and the test that checks it against float64 on its own operands.
CHECKED = [
    (r"step::conv_umma_kernel", FWD + " / " + BWD_CHAIN + " (dgrad)"),
    (r"step::conv_halo_kernel", FWD + " / " + BWD_CHAIN + " (dgrad)"),
    (r"step::conv_stem_kernel", FWD),
    (r"step::conv3d_simt_kernel", FWD),
    (r"step::bottleneck_exit_kernel", FWD),
    (r"step::clip_to_s2d_rgb_kernel", HERE_LAUNCH + " (exact: R.unpack_s2d of the stem's input is the fp16 clip)"),
    (r"step::maxpool3d\w*_kernel", FWD),
    (r"step::mean_mid\w*_kernel", FWD + " / " + HERE_LAUNCH + " (the context mean of each step)"),
    (r"step::linear_(mma|splitk|reduce)_kernel", FWD),
    (r"step::head_reg_reduce_kernel", FWD),
    (r"step::roi_align_fwd_nhwc\w*_kernel", FWD),
    (r"step::roi_pool_fwd_nhwc_kernel", HERE_LAUNCH + " (exact: every argmax at a maximum of its bin, out == feat[argmax])"),
    (r"step::act_bwd_kernel", BWD_ENTRY),
    (r"step::colsum_(partial|reduce)_kernel", BWD_ENTRY),
    (r"step::conv1x1_wgrad_(partial|reduce)_kernel", BWD_ENTRY),
    (r"step::maxpool_(argmax|bwd)_kernel", BWD_ENTRY),
    (r"step::head_losses_kernel", HERE_LAUNCH),
    (r"step::cls_loss_kernel", HERE_LAUNCH),
    (r"step::linear_bwd_(dw|dx)_kernel", HERE_LAUNCH),
    (r"step::mean_mid_bwd_kernel", HERE_LAUNCH),
    (r"step::f32_accum_f16_kernel", HERE_LAUNCH),
    (r"step::ctx_grad_reduce_kernel", HERE_LAUNCH),
    (r"step::roi_align_bwd_slice_nhwc_kernel", HERE_LAUNCH),
    (r"step::roi_pool_bwd_slice_nhwc_kernel", HERE_LAUNCH),
]
WORST = {}                       # launch kind -> largest |err| / bound seen (printed at the end of the module)


def _note(kind, ratio):
    WORST[kind] = max(WORST.get(kind, 0.0), ratio)


# ---- ROIAlign backward on its own ---------------------------------------------------------------------------------------
def _grad_act(g, ld, dtype):
    """g [R, ph, pw, C] -> Act [R, 1, ph, pw, ld] slice of its first C channels, in dtype, the rest of the row garbage."""
    from step_b200.engine import Act
    Rr, ph, pw, C = g.shape
    buf = torch.randn(Rr, 1, ph, pw, ld, device="cuda").to(dtype)
    buf[..., :C] = g.view(Rr, 1, ph, pw, C).to(dtype)
    return Act(buf, C, 0)


def _run_nhwc(g_act, rois, K, H, W, sr, what):
    from step_b200 import training
    got = training.roi_align_backward_nhwc_strided(g_act, rois, SCALE, K, H, W, sr)
    ph, pw = g_act.H, g_act.W
    ref, mag, n = R.roi_align_bwd(R.act_view(g_act).reshape(-1, ph, pw, g_act.C), rois, SCALE, ph, pw, K, H, W, sampling_ratio=sr)
    _note("roi_align_bwd_nhwc", R.roi_align_bwd_check(got, torch.zeros_like(got), ref, mag, n, what))


def _run_slice(g_act, rois, grad_in, roi_T, feat_T, t_start, sr, what):
    from step_b200 import training
    K, H, W, _ = grad_in.shape
    init = grad_in.clone()
    training.roi_align_backward_slice(g_act, rois, SCALE, grad_in, roi_T, feat_T, t_start, sr)
    ph, pw = g_act.H, g_act.W
    ref, mag, n = R.roi_align_bwd(R.act_view(g_act).reshape(-1, ph, pw, g_act.C), rois, SCALE, ph, pw, K, H, W, roi_T, feat_T,
                                  t_start, sr)
    _note("roi_align_bwd_slice", R.roi_align_bwd_check(grad_in, init, ref, mag, n, what))
    return n


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_roi_align_bwd_at_the_shipped_geometry(dtype):
    """2 clips x 9 frames of 25x25x832, 34 tubes per clip from synth.make_train_case at 400x400: the three steps' slices
    into one pre-filled buffer (fp16 gradient at row pitch 832 + 256), and the un-sliced entry on step 3's ROIs."""
    cfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(400, 400))
    st, _ = synth.make_train_case(cfg, 2, 34, 400, 400, seed=31)
    gen = torch.Generator(device="cuda").manual_seed(32)
    B, T_all, H, W, C = 2, 9, 25, 25, 832
    # pre-filled at the magnitude of one step's contributions (0.1 w / count), so that |init| does not dominate the bound
    grad_in = torch.randn(B * T_all, H, W, C, device="cuda", generator=gen) * 1e-3
    ld = C + 256 if dtype == torch.float16 else C
    from step_b200.training import step_frames
    for i, tubes in enumerate(st):
        t_start, t_len = step_frames(cfg, i + 1)
        rois = tubes.view(-1, 5).cuda()
        g = torch.randn(rois.shape[0], 7, 7, C, device="cuda", generator=gen) * 0.1
        _run_slice(_grad_act(g, ld, dtype), rois, grad_in, t_len, T_all, t_start, 0, ("shipped", i, dtype))
        torch.cuda.synchronize()
    _run_nhwc(_grad_act(g, ld, dtype), rois, B * T_all, H, W, 0, ("shipped nhwc", dtype))


EDGE_ROIS = [
    # frame, x1, y1, x2, y2 in image pixels (scale 1/16) on 28 x 28 maps
    [0, 0.0, 0.0, 448.0, 448.0],         # the whole image: 28 px, grid exactly 4 x 4 at 7 x 7 (784 samples)
    [0, 300.0, 200.0, 250.0, 150.0],     # degenerate: x2 < x1, y2 < y1
    [3, 16.0, 32.0, 576.0, 592.0],       # 35 px: grid 5 x 5 at 7 x 7 (1225 samples, two passes)
    [3, -200.0, -100.0, 900.0, 1000.0],  # grid 10 x 10 and more than 3 passes, corners below -16, past both far edges
    [3, -10.0, -5.0, 200.0, 150.0],      # corners in [-16, 0): samples in [-1, 0] clamped
    [3, -100.0, -60.0, 100.0, 120.0],    # corners below -16: samples dropped
    [3, 300.0, 300.0, 447.0, 447.0],     # touching the bottom and right edges
    [3, 350.0, 380.0, 600.0, 700.0],     # passing them
]


def _edge_rois():
    rois = torch.tensor(EDGE_ROIS, dtype=torch.float32)
    # frame 1: 40 overlapping ROIs; frame 2: none
    g = torch.Generator().manual_seed(33)
    xy = torch.rand(40, 2, generator=g) * 200.0
    wh = 16.0 + torch.rand(40, 2, generator=g) * 200.0
    many = torch.cat([torch.ones(40, 1), xy, xy + wh], 1)
    return torch.cat([rois, many]).cuda()


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("bins,sr", [((7, 7), 0), ((5, 3), 0), ((7, 7), 2)])
def test_roi_align_bwd_edges(dtype, bins, sr):
    """The edge ROIs through both entries.  Slice entry: 2 clips of 4 frames, ROI frames 0..3 relative to the 2-frame slice
    from t 1: ROI frames 0, 1, 2, 3 land on grad_in frames 1, 2, 5, 6.  ROI frame 2 has no ROI, so grad_in frame 5, the first
    slice frame of clip 1, takes no term; t 0 and 3 of each clip (grad_in frames 0, 3, 4, 7) are outside the slice.  The
    pre-fills are scaled to the contributions so that the bound is not dominated by |init|."""
    gen = torch.Generator(device="cuda").manual_seed(34)
    rois = _edge_rois()
    ph, pw = bins
    H = W = 28
    C = 64
    g = torch.randn(rois.shape[0], ph, pw, C, device="cuda", generator=gen)
    ld = C + 16 if dtype == torch.float16 else C
    act = _grad_act(g, ld, dtype)
    what = ("edges", bins, sr, dtype)
    _run_nhwc(act, rois, 6, H, W, sr, what + ("nhwc",))
    grad_in = torch.randn(8, H, W, C, device="cuda", generator=gen) * 1e-2
    n = _run_slice(act, rois, grad_in, 2, 4, 1, sr, what + ("slice",))
    per_frame = n.view(8, -1).sum(1).tolist()
    assert [f > 0 for f in per_frame] == [False, True, True, False, False, False, True, False], per_frame
    if sr == 0 and bins == (7, 7):
        # the whole-image ROI fills exactly one sample table; the 35 px one needs two passes
        groups = R.roi_align_terms(rois[:3], SCALE, ph, pw, H, W)
        assert sorted(gr["count"] for gr in groups) == [1, 16, 25]


# ---- train_step launch by launch --------------------------------------------------------------------------------------------
def _geoms():
    from test_oracle_cls import CLS_CFG
    return {
        "align": (dict(**SHIPPED), "align", False, 34),
        "pool": (dict(**SHIPPED), "pool", False, 34),
        "cls": (dict(CLS_CFG), "align", True, 34),
    }


def setup(name):
    kw, mode, cls_only, N = _geoms()[name]
    cfg = synth.make_cfg(fp16=True, **dict(kw, image_size=(400, 400)))
    x = synth.make_clips(2, 36, 400, 400, seed=41).cuda()
    if cls_only:
        tb, tg = synth.make_cls_case(cfg, 2, N, 400, 400, seed=42)
        st, tgs = [tb], [tg]
        heads = [synth.cls_head_state_dict(100, cfg)]
    else:
        st, tgs = synth.make_train_case(cfg, 2, N, 400, 400, seed=42)
        heads = [synth.head_state_dict(100 + i, cfg) for i in range(len(st))]
    nets = device_nets(cfg, heads, pool_mode=mode, context=not getattr(cfg, "no_context", True), cls_only=cls_only)
    return cfg, nets, x, [t.cuda() for t in st], [t.cuda() for t in tgs]


def step(cfg, nets, x, st, tgs):
    from step_b200 import training
    r = training.train_step(cfg, nets, x, st, tgs, lr=None, loss_scale=1024.0)
    torch.cuda.synchronize()
    return r


def profiled_kernel_names(name):
    """Kernel names of one un-instrumented train_step under torch.profiler, in a child process (see
    test_gpu_forward_layers.profiled_kernel_names)."""
    cfg, nets, x, st, tgs = setup(name)
    step(cfg, nets, x, st, tgs)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(cfg, nets, x, st, tgs)
    return sorted({e.key for e in prof.key_averages()})


def _c(t):
    return t.detach().clone() if t is not None else None


def install(mp, recs):
    from step_b200 import i3d, networks, training
    orig_s2d, orig_pool_into = i3d.Unit3Dpy.forward_s2d, networks.ROINet.pool_into

    def forward_s2d(self, x_s2d):
        recs.append(dict(kind="s2d", s2d=x_s2d.buf.clone(), cin=self.conv3d.in_channels))
        return orig_s2d(self, x_s2d)

    def pool_into(self, feat, flat_tubes, out, roi_T, feat_T, t_start, argmax=None):
        ret = orig_pool_into(self, feat, flat_tubes, out, roi_T, feat_T, t_start, argmax)
        recs.append(dict(kind="roi_fwd", mode=self.pool_mode, out=R.act_view(out).clone(), argmax=_c(argmax)))
        return ret

    mp.setattr(i3d.Unit3Dpy, "forward_s2d", forward_s2d)
    mp.setattr(networks.ROINet, "pool_into", pool_into)
    orig = {k: getattr(training, k) for k in ("head_losses", "cls_loss", "linear_backward", "context_grad_reduce",
                                              "roi_align_backward_slice", "roi_pool_backward_slice", "tape_backward",
                                              "context_forward", "head_forward_backward")}

    def head_losses(logits, local_loc, first_loc, last_loc, tubes, targets, T, lambda_reg=5.0, lambda_neighbor=1.0,
                    want_grads=False):
        r = dict(kind="head_losses", args=[_c(t).float() for t in (logits, local_loc, first_loc, last_loc, tubes, targets)], T=T,
                 lam=(lambda_reg, lambda_neighbor))
        out = orig["head_losses"](logits, local_loc, first_loc, last_loc, tubes, targets, T, lambda_reg, lambda_neighbor, want_grads)
        r["out"] = [_c(t) for t in out[:3]] + ([{k: _c(v) for k, v in out[3].items()}] if want_grads else [])
        recs.append(r)
        return out

    def cls_loss(logits, targets, want_grads=False):
        r = dict(kind="cls_loss", args=[_c(logits).float(), _c(targets).float()])
        out = orig["cls_loss"](logits, targets, want_grads)
        r["out"] = [_c(t) for t in out] if want_grads else [_c(out)]
        recs.append(r)
        return out

    def linear_backward(x, w, dy, need_dx=True, need_dw=True, dx_out=None, accumulate_dx=False):
        r = dict(kind="linear_bwd", x=_c(x), w=_c(w).float(), dy=_c(dy).float(), init=_c(dx_out) if accumulate_dx else None)
        out = orig["linear_backward"](x, w, dy, need_dx, need_dw, dx_out, accumulate_dx)
        r["out"] = [_c(t) for t in out]
        recs.append(r)
        return out

    def context_grad_reduce(dctx, tubes, acc, t_start):
        r = dict(kind="ctx_grad_reduce", dctx=_c(dctx).float(), tubes=_c(tubes).float(), acc=_c(acc), t_start=t_start)
        out = orig["context_grad_reduce"](dctx, tubes, acc, t_start)
        r["out"] = _c(acc)
        recs.append(r)
        return out

    def roi_align_backward_slice(grad_act, rois, spatial_scale, grad_in, roi_T, feat_T, t_start, sampling_ratio=0, ws=None):
        r = dict(kind="roi_align_bwd", g=R.act_view(grad_act).clone(), rois=_c(rois), scale=spatial_scale, init=_c(grad_in),
                 roi_T=roi_T, feat_T=feat_T, t_start=t_start, sr=sampling_ratio, ld=grad_act.ld)
        out = orig["roi_align_backward_slice"](grad_act, rois, spatial_scale, grad_in, roi_T, feat_T, t_start, sampling_ratio, ws)
        r["out"] = _c(grad_in)
        recs.append(r)
        return out

    def roi_pool_backward_slice(grad_act, rois, argmax, grad_in, roi_T, feat_T, t_start):
        r = dict(kind="roi_pool_bwd", g=R.act_view(grad_act).clone(), rois=_c(rois), argmax=_c(argmax), init=_c(grad_in),
                 roi_T=roi_T, feat_T=feat_T, t_start=t_start)
        out = orig["roi_pool_backward_slice"](grad_act, rois, argmax, grad_in, roi_T, feat_T, t_start)
        r["out"] = _c(grad_in)
        recs.append(r)
        return out

    def tape_backward(tape, grads, loss_scale=1.0, need_input_grad=None):
        r = dict(kind="tape", seeds={k: v.clone() for k, v in grads.bufs.items()}, shapes={k: tuple(v.shape) for k, v in grads.bufs.items()},
                 loss_scale=loss_scale)
        recs.append(r)
        out = orig["tape_backward"](tape, grads, loss_scale, need_input_grad)
        r["final"] = {k: v.clone() for k, v in grads.bufs.items()}
        return out

    def context_forward(context_net, feat):
        ctx, state = orig["context_forward"](context_net, feat)
        recs.append(dict(kind="ctx_fwd", ctx=_c(ctx), feat_ptr=feat.buf.data_ptr()))
        return ctx, state

    def head_forward_backward(net, global_feat, tubes, targets, context_feat=None, **kw):
        r = dict(kind="head", ctx_mean=_c(context_feat[0]) if isinstance(context_feat, tuple) else None, T=kw["cat"].T)
        recs.append(r)
        return orig["head_forward_backward"](net, global_feat, tubes, targets, context_feat, **kw)

    for k, fn in dict(head_losses=head_losses, cls_loss=cls_loss, linear_backward=linear_backward,
                      context_grad_reduce=context_grad_reduce, roi_align_backward_slice=roi_align_backward_slice,
                      roi_pool_backward_slice=roi_pool_backward_slice, tape_backward=tape_backward,
                      context_forward=context_forward, head_forward_backward=head_forward_backward).items():
        mp.setattr(training, k, fn)


@pytest.fixture(scope="module", params=["align", "pool", "cls"])
def geom(request):
    name = request.param
    t0 = time.time()
    child = subprocess.run([sys.executable, os.path.abspath(__file__), name], cwd=ROOT, capture_output=True, text=True,
                           timeout=900)
    assert child.returncode == 0, child.stderr[-4000:]
    names = set(json.loads(child.stdout.strip().splitlines()[-1]))
    cfg, nets, x, st, tgs = setup(name)
    plain = step(cfg, nets, x, st, tgs)
    plain_grads = {p: g.clone() for p, g in plain["grads"].items()}
    recs = []
    with pytest.MonkeyPatch.context() as mp:
        install(mp, recs)
        inst = step(cfg, nets, x, st, tgs)
    yield dict(name=name, cfg=cfg, nets=nets, x=x, st=st, recs=recs, plain=plain_grads, inst=inst, names=names, t0=t0)
    print("\n%s: %.1f s; largest |err| / bound per launch kind: %s" % (name, time.time() - t0, json.dumps(WORST, sort_keys=True)))


def _census(recs):
    got = {}
    for r in recs:
        got[r["kind"]] = got.get(r["kind"], 0) + 1
    return got


def test_launch_census_and_bit_identical_gradients(geom):
    """Per-kind launch counts from the step structure (per full head: the classifier, its context columns, local_reg and
    the two neighbour regressors), and the instrumented step's gradients equal the un-instrumented step's bit for bit."""
    name = geom["name"]
    n_steps = len(geom["st"])
    ctx = name != "cls" or not getattr(geom["cfg"], "no_context", True)
    want = {"head": n_steps, "tape": n_steps + 1 + (1 if ctx else 0), "s2d": 1, "roi_fwd": n_steps}
    if name == "cls":
        want.update(cls_loss=1, linear_bwd=1 + (1 if ctx else 0))
    else:
        want.update(head_losses=n_steps, linear_bwd=5 * n_steps)
    if ctx:
        want.update(ctx_grad_reduce=n_steps, ctx_fwd=1)
    want["roi_pool_bwd" if name == "pool" else "roi_align_bwd"] = n_steps
    assert _census(geom["recs"]) == want
    inst = geom["inst"]["grads"]
    assert set(inst) == set(geom["plain"])
    for p, g in geom["plain"].items():
        assert torch.equal(inst[p], g), tuple(p.shape)


def _bin_argmax_ok(feat, rois, argmax, out, roi_T, feat_T, t_start, ps):
    """Every recorded argmax of a ROIPool bin points at a pixel inside the bin that holds the bin's maximum, and the pooled
    value the head read (out [R, ps, ps, C] fp16) is that pixel's value bit for bit; an empty bin records -1 and pools 0.  Bins by the reference's ROIPool rules (ROIPool_cuda.cu): corners round(coord * scale) (half away
    from zero), size max(end - start + 1, 1), bin p spans [floor(p * bin), ceil((p + 1) * bin)) in fp32, shifted by the
    corner and clipped to the map.  On the CPU."""
    import numpy as np
    f32 = np.float32
    Fr, H, W, C = feat.shape
    feat = feat.cpu()
    rois = rois.cpu()
    fr = R.roi_frames(rois, roi_T, feat_T, t_start)
    am = argmax.cpu().view(-1, ps, ps, C).long()
    out = out.cpu().reshape(-1, ps, ps, C)
    cround = lambda v: int(math.copysign(math.floor(abs(v) + 0.5), v))

    def edges(start, size, p):
        b = f32(size) / f32(ps)
        lo = int(math.floor(f32(p) * b)) + start
        hi = int(math.ceil(f32(p + 1) * b)) + start
        return lo, hi

    for r in range(rois.shape[0]):
        x1, y1, x2, y2 = (cround(float(f32(float(v)) * f32(SCALE))) for v in rois[r, 1:5])
        rw, rh = max(x2 - x1 + 1, 1), max(y2 - y1 + 1, 1)
        f = feat[int(fr[r])]
        for p in range(ps):
            hs, he = (min(max(v, 0), H) for v in edges(y1, rh, p))
            for q in range(ps):
                ws, we = (min(max(v, 0), W) for v in edges(x1, rw, q))
                a = am[r, p, q]
                if he <= hs or we <= ws:
                    assert bool((a == -1).all()) and not bool(out[r, p, q].any()), (r, p, q)
                    continue
                assert bool(((a // W >= hs) & (a // W < he) & (a % W >= ws) & (a % W < we)).all()), (r, p, q)
                got = f.reshape(H * W, C).gather(0, a.view(1, C)).view(C)
                assert torch.equal(got, f[hs:he, ws:we].reshape(-1, C).max(0).values), (r, p, q)
                assert torch.equal(out[r, p, q], got.half()), (r, p, q)


def _roi_pool_ref(g, rois, argmax, K, H, W, roi_T, feat_T, t_start):
    """Float64 scatter of g [R, ps, ps, C] through argmax into [K, H, W, C], with sum |term| and the terms per element."""
    Rr, ph, pw, C = g.shape
    fr = R.roi_frames(rois, roi_T, feat_T, t_start)
    a = argmax.view(Rr, ph * pw, C).long()
    live = a >= 0
    idx = (fr.view(Rr, 1, 1) * (H * W) + a.clamp(min=0)) * C + torch.arange(C, device=g.device).view(1, 1, C)
    gd = torch.where(live, g.reshape(Rr, ph * pw, C).double(), torch.zeros_like(a, dtype=torch.float64))
    ref = torch.zeros(K * H * W * C, dtype=torch.float64, device=g.device)
    mag, n = torch.zeros_like(ref), torch.zeros_like(ref)
    ref.index_add_(0, idx.flatten(), gd.flatten())
    mag.index_add_(0, idx.flatten(), gd.abs().flatten())
    n.index_add_(0, idx.flatten(), live.double().flatten())
    v = lambda t: t.view(K, H, W, C)
    return v(ref), v(mag), v(n)


def test_every_launch_against_float64(geom):
    """Each recorded launch against its float64 reference and bound (tests/_tape_reference.py), the raw launches exactly
    from the tape seeds, and the frames outside each ROI slice unchanged."""
    recs = geom["recs"]
    for i, r in enumerate(recs):
        what = (geom["name"], i, r["kind"])
        k = r["kind"]
        if k == "head_losses":
            logits, loc, first, last, tubes, targets = r["args"]
            ref = R.head_losses(logits, loc, first, last, tubes, targets, r["T"], *r["lam"])
            lc, ll, ln, g = r["out"]
            for key, got in (("loss_cls", lc), ("loss_loc", ll), ("loss_nb", ln), ("dlogits", g["logits"]), ("dlocal", g["local_loc"]),
                             ("dfirst", g["first_loc"]), ("dlast", g["last_loc"])):
                _note("head_losses", R._check_within(got.cpu(), ref[key][0], ref[key][1], what + (key,)))
        elif k == "cls_loss":
            ref = R.cls_loss(*r["args"])
            lc, dl = r["out"]
            _note("cls_loss", R._check_within(lc.cpu(), ref["loss"], ref["loss_tol"], what + ("loss",)))
            _note("cls_loss", R._check_within(dl.cpu(), ref["dlogits"], ref["dlogits_tol"], what + ("dlogits",)))
        elif k == "linear_bwd":
            ref = R.linear_bwd(r["x"], r["w"], r["dy"], r["init"])
            dx, dw, db = r["out"]
            M, Nn = r["dy"].shape
            _note("linear_bwd", R.linear_bwd_check(dw, ref["dw"], ref["dw_abs"], M, what + ("dw",)))
            _note("linear_bwd", R.linear_bwd_check(db, ref["db"], ref["db_abs"], M, what + ("db",)))
            if dx is not None:
                _note("linear_bwd", R.linear_bwd_check(dx, ref["dx"], ref["dx_abs"], Nn, what + ("dx",)))
        elif k == "ctx_grad_reduce":
            # exact: per clip the rows in ascending order, one fp32 division by T_len, one addition per frame
            acc = r["acc"].clone()
            T_len = r["tubes"].shape[1]
            clip = torch.div(r["tubes"][:, 0, 0], torch.full_like(r["tubes"][:, 0, 0], float(T_len))).floor().long()
            for b in range(acc.shape[0]):
                s = torch.zeros(acc.shape[2], device="cuda")
                for row in (clip == b).nonzero().view(-1).tolist():
                    s = s + r["dctx"][row]
                acc[b, r["t_start"]:r["t_start"] + T_len] += s / torch.full_like(s, T_len)
            assert torch.equal(r["out"], acc), what
        elif k == "roi_align_bwd":
            K, H, W, C = r["init"].shape
            g = r["g"].reshape(-1, 7, 7, C)
            ref, mag, n = R.roi_align_bwd(g, r["rois"], r["scale"], 7, 7, K, H, W, r["roi_T"], r["feat_T"], r["t_start"], r["sr"])
            _note("roi_align_bwd_slice", R.roi_align_bwd_check(r["out"], r["init"], ref, mag, n, what))
            outside = [f for f in range(K) if not (r["t_start"] <= f % r["feat_T"] < r["t_start"] + r["roi_T"])]
            assert torch.equal(r["out"][outside], r["init"][outside]), what
        elif k == "roi_pool_bwd":
            K, H, W, C = r["init"].shape
            g = r["g"].reshape(-1, 7, 7, C)
            ref, mag, n = _roi_pool_ref(g, r["rois"], r["argmax"], K, H, W, r["roi_T"], r["feat_T"], r["t_start"])
            _note("roi_pool_bwd_slice", R.roi_align_bwd_check(r["out"], r["init"], ref, mag, n, what))
            outside = [f for f in range(K) if not (r["t_start"] <= f % r["feat_T"] < r["t_start"] + r["roi_T"])]
            assert torch.equal(r["out"][outside], r["init"][outside]), what
            # the forward that recorded this argmax: the pool_into of the same step (the same argmax buffer)
            fwd = [q for q in recs[:i] if q["kind"] == "roi_fwd"][-1]
            assert torch.equal(fwd["argmax"], r["argmax"]), what
            feat = _trunk_feat(geom)
            _bin_argmax_ok(feat.view(-1, *feat.shape[2:]), r["rois"], r["argmax"], fwd["out"], r["roi_T"], r["feat_T"], r["t_start"], 7)
        elif k == "s2d":
            # clip_to_s2d: exact.  R.unpack_s2d of the 8 * cin live channels is the fp16 clip, the padding channels are zero
            x = geom["x"]                                                  # [N, T, C, H, W] fp32, what train_step was given
            live = 8 * r["cin"]
            assert torch.equal(R.unpack_s2d(r["s2d"], r["cin"]), x.half().permute(0, 2, 1, 3, 4)), what
            assert not bool(r["s2d"][..., live:].any()), (what, "padding channels")
        torch.cuda.synchronize()
    _check_seeds(geom)


_FEAT = {}


def _trunk_feat(geom):
    """conv_feat of the geometry's clips (the trunk forward is deterministic: the same values train_step pooled)."""
    if geom["name"] not in _FEAT:
        with torch.no_grad():
            f = geom["nets"]["base_net"].forward_act(geom["x"])
        _FEAT[geom["name"]] = R.act_view(f).float().clone()
    return _FEAT[geom["name"]]


def _check_seeds(geom):
    """The raw launches, exactly, from the tape seeds: the classifier's mean_mid_bwd (fp16(0 + dxbar 1024 / T')) and the
    regressors' f32_accum_f16 (fp16(0 + dlf2 1024)) in every head; ContextNet's mean_mid_bwd (fp16(0 + d_ctx 1024 / (H W)));
    the trunk's f32_accum_f16 (fp16(0 + (total / 1024) 1024)); and each step's context mean (step_mean_mid_strided) within
    mean_mid's bound."""
    recs = geom["recs"]
    heads = [i for i, r in enumerate(recs) if r["kind"] == "head"]
    tapes = [r for r in recs if r["kind"] == "tape"]
    ls = 1024.0
    for h, i in enumerate(heads):
        end = heads[h + 1] if h + 1 < len(heads) else len(recs)
        seg = recs[i:end]
        lins = [r for r in seg if r["kind"] == "linear_bwd"]
        tape = [r for r in seg if r["kind"] == "tape"][0]
        T_ = recs[i]["T"]
        dxbar = lins[0]["out"][0]                                      # [N, 49 fc]
        cat_keys = [k for k, s in tape["shapes"].items() if s[-1] > 832]
        assert len(cat_keys) == 1
        seed = tape["seeds"][cat_keys[0]]
        Nr, _, P1, P2, ld = seed.shape
        fc = ld - 832
        want = ((dxbar * ls) / torch.full_like(dxbar, T_)).half().view(Nr, 1, P1, P2, fc).expand(Nr, T_, P1, P2, fc)
        assert torch.equal(seed[..., 832:], want), (h, "mean_mid_bwd")
        assert not bool(seed[..., :832].any()), (h, "the ROI channels are seeded by the tape")
        full = [r for r in seg if r["kind"] == "head_losses"]
        if full:
            ctx = recs[i]["ctx_mean"] is not None
            loc, n1, n2 = lins[2 if ctx else 1:5 if ctx else 4]
            dlf2 = loc["out"][0].clone().view(Nr, T_, -1)
            s0, s1, e0, e1 = R.head_chunks(3, T_)
            dlf2[:, s0:s1] += n1["out"][0].view(Nr, s1 - s0, -1)
            dlf2[:, e0:e1] += n2["out"][0].view(Nr, e1 - e0, -1)
            lf_keys = [k for k in tape["seeds"] if k != cat_keys[0]]
            assert len(lf_keys) == 1
            lseed = tape["seeds"][lf_keys[0]]
            assert lseed.shape[-1] * 49 * T_ * Nr == dlf2.numel(), (h, "local_feat2 is not a dense buffer", tuple(lseed.shape))
            assert torch.equal(lseed.reshape(Nr, T_, -1), (dlf2 * ls).half().view(Nr, T_, -1)), (h, "f32_accum_f16")
        if recs[i]["ctx_mean"] is not None:
            fwd = [r for r in recs if r["kind"] == "ctx_fwd"][0]["ctx"]       # [B, T', 1024]
            t_start = [r for r in seg if r["kind"] == "ctx_grad_reduce"][0]["t_start"]
            x = fwd[:, t_start:t_start + T_].unsqueeze(2)                    # [B, T_len, 1, 1024]
            ref, mabs = R.mean_mid(x)
            _note("mean_mid_strided", R._check_within(recs[i]["ctx_mean"], ref, R.mean_mid_tol(ref, mabs, T_), (h, "context mean")))
    # ContextNet: its tape's seed is the spatial mean's backward of the final d_ctx
    red = [r for r in recs if r["kind"] == "ctx_grad_reduce"]
    if red:
        ctape = tapes[len(heads)]
        d_ctx = red[-1]["out"]                                              # [B, T', 1024]
        (key, seed), = ctape["seeds"].items()
        Bc, Tc_, Hc, Wc, ldc = seed.shape
        want = ((d_ctx * ls) / torch.full_like(d_ctx, Hc * Wc)).half().view(Bc, Tc_, 1, 1, -1).expand(Bc, Tc_, Hc, Wc, d_ctx.shape[-1])
        assert torch.equal(seed[..., ldc - d_ctx.shape[-1]:], want), "context mean_mid_bwd"
    # the trunk: fp16(0 + (total / 1024) 1024) with total = the ROI backward of every step + ContextNet's input gradient
    ttape = tapes[-1]
    roi = [r for r in recs if r["kind"] in ("roi_align_bwd", "roi_pool_bwd")]
    total = roi[-1]["out"].clone()
    if red:
        ctape = tapes[len(heads)]
        rows = total.numel() // 832
        gfeat = [v for k, v in ctape["final"].items() if k not in ctape["seeds"] and v.shape[-1] >= 832
                 and v.numel() // v.shape[-1] == rows]
        assert len(gfeat) == 1
        g = gfeat[0]
        total.add_(g[..., g.shape[-1] - 832:].reshape(total.shape).float())
    d = total.mul_(1.0 / ls)
    (tkey, tseed), = ttape["seeds"].items()
    assert torch.equal(tseed[..., tseed.shape[-1] - 832:].reshape(d.shape), (d * ls).half()), "trunk f32_accum_f16"


def test_every_train_step_kernel_has_a_float64_check(geom):
    """Closure: every step:: kernel of a profiled train_step matches a pattern of CHECKED."""
    kernels = sorted(n for n in geom["names"] if "step::" in n)
    assert kernels, "the profile recorded no step:: kernel"
    missing = [n for n in kernels if not any(re.search(p, n) for p, _ in CHECKED)]
    assert not missing, missing
    base = sorted({re.search(r"step::(\w+)", n).group(1) for n in kernels})
    print("\n%s: %d step:: kernels: %s" % (geom["name"], len(base), " ".join(base)))


if __name__ == "__main__":                                     # the fixture's child process: python <this file> <geometry>
    print(json.dumps(profiled_kernel_names(sys.argv[1])))
