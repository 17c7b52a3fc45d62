"""GPU: the inference forward launch by launch, against the float64 references of tests/_tape_reference.py on the SAME
operands each launch read: the fp16 activations, the packed fp16 filters, the fp32 folded scale / shift, the fp16 residual.

The forward runs as the benchmark runs it (eager; Inception branches on side streams, the fused 1x1 triple, the fused
bottleneck exit, the A_BEST choice between the patch and the im2col kernels), with test-local wrappers around engine.conv,
engine.maxpool, engine.bottleneck_exit, engine.mean_mid, engine.linear_small_n, ROINet.pool_into and
TwoBranchNet.forward_act (whose results carry step_head_regress's outputs; its input is the last exit's z).  Each wrapper
clones what the launch reads before it and what it wrote right after it, on the issuing stream.  At the end every written
region must still equal its snapshot (a later launch writing outside its channel slice or past a tile edge fails), and the
instrumented run's outputs must equal an un-instrumented run bit for bit.

Two geometries: the benchmark's C4 batch (8 clips of 32 x 224 x 224, 11 proposals, 3 steps: every layer of
profiles/h100_conv_layers_c4.txt on its benchmarked kernel) and the shipped configuration (one 36 x 400 x 400 clip,
ContextNet, steps of 3, 3 and 9 frames: the patch kernel's TT = 4 with a partly filled last plane group at OT = 18 and 9,
the stem on a 200 x 200 map, ContextNet's 25 x 25 map and mean).  At C4 the trunk's convolutions are compared on clips 0
and 7 (the first M tile and the ragged last one); every other launch, and every head row, is compared whole.

Tolerances (u32 = 2^-24, the fp32 unit roundoff; ulp16(v) the fp16 spacing at |v|):
  * Convolutions and both GEMMs of the exit, elementwise:
        |got - ref| <= m + 1/2 ulp16(|ref| + m),
        m = 2^-12 |scale| (|x| * |w|) + 2^-21 (|acc scale| + |shift| + |res|).
    The wgmma accumulation adds 16 exact products per k16 step into an fp32 accumulator, truncating: each step errs by
    less than one fp32 ulp of the partial sum, 2 u32 |partial| <= 2 u32 (|x| * |w|).  The longest chain in the network is
    Mixed_5c's 3x3x3 convolution over 192 channels, 27 x 12 = 324 steps: 648 u32 < 2^-14.6 < 2^-12 (each launch asserts
    steps x 2 u32 <= 2^-12).  The epilogue is fmaf(acc, scale, shift), + residual in fp32: two roundings, each within u32
    of |acc scale| + |shift| + |res|, far below 2^-21 of it.  The fp16 store rounds to nearest: 1/2 ulp at the perturbed
    value.  ReLU is 1-Lipschitz.  The exit's z inherits y's tolerance: the kernel feeds GEMM2 its own fp16 y, which may sit
    up to m_y + 1/2 ulp from the float64 y and so up to m_y + 1 ulp from fp16(y); |w1| times that is added to z's m.
  * Bias, per launch.  The elementwise bound is loose by about sqrt(K), so a layer scaled by 1 + 2^-8 or rounded toward
    zero can hide inside it.  Over the elements with |ref| >= 64 m, d_i = (got - ref) sign(ref) / ulp16(ref) is a
    round-to-nearest error in [-1/2, 1/2] (mean 0 when the rounded values' low bits are spread out) plus the accumulation
    error.  Hoeffding bounds the mean of n values of width 1 by sqrt(ln(2 / delta) / (2 n)) except with probability delta
    = 2^-40; the truncating accumulation loses on average half an fp32 ulp of the partial per step, at most
    steps x u32 x |scale| (|x| * |w|) per element (plus the inherited carry for z).  |mean d| must stay under the sum.
    Round toward zero moves the mean by -1/2, a 2^-8 scale by 4 to 8.
  * Max pools: torch.equal (a maximum of fp16 values is exact).
  * mean_mid: B fp32 additions in index order and one division: B u32 mean|x| + u32 |ref|.
  * linear_small_n / step_head_regress: split-K over 512-column chunks; inside a chunk 32 mma k16 steps at 2 u32 (the fp32
    SIMT path: 16 FMAs and 5 shuffle additions per lane, fewer), then the chunks in fixed order, the bias and the
    accumulate, each within u32 of the abs sum: (64 + ceil(K / 512) + 2) u32 (|x| |w|^T + |b| + |y0|).  The sigmoid is
    1/4-Lipschitz, and 1 / (1 + expf(-v)) adds expf's 2 ulp and two roundings: < 2^-21 |y|.  first / last = local +
    neighbour: both tolerances plus one fp32 rounding of the sum.
  * ROIAlign, packed half2 (exact = 0): <= 16 merged pixels per bin, weights rounded to fp16 (2^-11 relative, 2^-25
    absolute), one half2 FMA rounding per pixel (2^-11 of the running sum, 2^-25 absolute): 17 x 2^-11 sum |w| |v| +
    2^-20 sum |w| |v| (the fp32 merge) + 16 x 2^-25 (1 + max |v|).
"""
import json
import os
import re
import subprocess
import sys

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [HERE, ROOT]
import _tape_reference as R  # noqa: E402
from step_b200 import synth  # noqa: E402
from test_gpu_pipeline import build  # noqa: E402

pytestmark = pytest.mark.gpu
GEOMS = {
    # cfg, clips, T_in, image side, proposals per clip, ContextNet
    "c4": (dict(T=8, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 1}, image_size=(224, 224)), 8, 32, 224, 11, False),
    "shipped": (dict(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False, image_size=(400, 400)), 1, 36, 400, 11,
                True),
}
# Launches per kind, from the module structure.  Trunk: stem, conv3d_2b / 2c, 7 Mixed x (fused 1x1 triple, two 3x3x3, the
# branch-3 1x1) = 31 convs; 3 strided pools + 7 branch-3 pools.  A head step: Mixed_5b / 5c (8 convs, 2 pools), downsample,
# the local branch with the fused exits (conv2 / conv3 / conv1 of block 0, conv2 of blocks 1 and 2: 5 convs; 3 exits), the
# temporal mean, the classifier (+ its context columns), step_head_regress, one ROIAlign.  ContextNet: its pool and two
# Mixed (8 convs, 3 pools) and the spatial mean; with it every step also takes the mean of the context rows.
CENSUS = {
    "c4": dict(conv=31 + 3 * 14, pool=10 + 3 * 2, exit=3 * 3, mean_mid=3, linear=3, roi=3, regress=3),
    "shipped": dict(conv=31 + 8 + 3 * 14, pool=10 + 3 + 3 * 2, exit=3 * 3, mean_mid=1 + 3 * 2, linear=3 * 2, roi=3, regress=3),
}


class _Cai(object):
    """__cuda_array_interface__ over a raw device pointer (engine.mean_mid takes one)."""

    def __init__(self, ptr, dtype, shape, strides):
        self.__cuda_array_interface__ = dict(shape=tuple(shape), typestr={torch.float16: "<f2", torch.float32: "<f4"}[dtype],
                                             data=(ptr, False), version=2,
                                             strides=tuple(s * (2 if dtype == torch.float16 else 4) for s in strides))


class Recorder(object):
    def __init__(self):
        self.recs = []
        self.rows = None            # clips whose trunk convolutions are compared (None: all)

    def sel(self):
        return slice(None) if self.rows is None else list(self.rows)


def _clone(t):
    return t.detach().clone() if t is not None else None


def install(mp, rec, fused_exit=True):
    """The wrappers.  Each clones what its launch reads before calling the original and what it wrote right after, on the
    current (issuing) stream.  fused_exit: the full head runs the fused bottleneck exit (the fp16 inference path; the
    fp32 path runs it as separate convolutions and its regressors read downsample2's conv output)."""
    from step_b200 import _lib as L
    from step_b200 import engine as E
    from step_b200 import networks, two_branch
    orig = dict(conv=E.conv, maxpool=E.maxpool, exit=E.bottleneck_exit, mean_mid=E.mean_mid, linear=E.linear_small_n,
                pool_into=networks.ROINet.pool_into, forward_act=two_branch.TwoBranchNet.forward_act)

    def conv(x, w_packed, scale, shift, out, k, stride=(1, 1, 1), pad_lo=None, relu=True, residual=None, a_mode=None,
             out_dims=None, extra_outs=None, zero_cin_last_kt=0, tag=None):
        sel = rec.sel() if x.T > 1 else slice(None)
        r = dict(kind="conv", x=R.act_view(x)[sel].clone(), w=_clone(w_packed), scale=_clone(scale), shift=_clone(shift),
                 res=R.act_view(residual)[sel].clone() if residual is not None else None, k=tuple(k), stride=tuple(stride),
                 pad_lo=tuple(pad_lo) if pad_lo is not None else tuple(E.same_pad(kk, s)[0] for kk, s in zip(k, stride)),
                 out_dims=tuple(out_dims) if out_dims is not None else E.same_out_dims((x.T, x.H, x.W), k, stride),
                 relu=relu, sel=sel, n=x.N)
        ret = orig["conv"](x, w_packed, scale, shift, out, k, stride, pad_lo, relu, residual, a_mode, out_dims, extra_outs,
                           zero_cin_last_kt, tag)
        r["outs"] = [(o, R.act_view(o).clone()) for o in [out] + list(extra_outs or [])]
        rec.recs.append(r)
        return ret

    def maxpool(x, k, s, out=None):
        xs = R.act_view(x).clone()
        o = orig["maxpool"](x, k, s, out)
        geo = [E.pool_out(d, kk, ss) for d, kk, ss in zip((x.T, x.H, x.W), k, s)]
        rec.recs.append(dict(kind="pool", x=xs, k=tuple(k), stride=tuple(s), pad_lo=tuple(g[1] for g in geo),
                             pad_hi=tuple(g[2] for g in geo), outs=[(o, R.act_view(o).clone())]))
        return o

    def bottleneck_exit(h, w3, x, w1, shift2, relu2, z, y=None):
        rows = lambda a: R.act_view(a).reshape(-1, a.C)
        r = dict(kind="exit", h=rows(h).clone(), w3=_clone(w3), x=rows(x).clone(), w1=_clone(w1), shift2=_clone(shift2),
                 relu2=relu2)
        ret = orig["exit"](h, w3, x, w1, shift2, relu2, z, y)
        r["outs"] = [(a, R.act_view(a).clone()) for a in [z] + ([y] if y is not None else [])]
        rec.recs.append(r)
        return ret

    def mean_mid(x_ptr, code, A, B, P, C, ld, device, out_code=L.F32):
        dt = E.torch_dtype(code)
        x = torch.as_tensor(_Cai(int(x_ptr), dt, (A, B, P, C), (B * P * ld, P * ld, ld, 1)), device=device).clone()
        y = orig["mean_mid"](x_ptr, code, A, B, P, C, ld, device, out_code)
        rec.recs.append(dict(kind="mean_mid", x=x, outs=[(y, y.clone())]))
        return y

    def linear_small_n(x, M, K, x_ld, w, bias, N, y=None, act=0, accumulate=False, row_map=None):
        r = dict(kind="linear", x=x.reshape(-1, x_ld)[:, :K].clone(), M=M, K=K, w=_clone(w), bias=_clone(bias), act=act,
                 y0=y[:M, :N].clone() if accumulate else None, y0_of=y if accumulate else None, row_map=_clone(row_map))
        out = orig["linear"](x, M, K, x_ld, w, bias, N, y, act, accumulate, row_map)
        r["outs"] = [(out, out.clone())]
        rec.recs.append(r)
        return out

    def pool_into(self, feat, flat_tubes, out, roi_T, feat_T, t_start, argmax=None):
        f = R.act_view(feat)
        r = dict(kind="roi", feat=f.reshape(-1, *f.shape[2:]).clone(), rois=flat_tubes.reshape(-1, 5).clone(), roi_T=roi_T,
                 feat_T=feat_T, t_start=t_start, mode=self.pool_mode, size=self.pool_size)
        ret = orig["pool_into"](self, feat, flat_tubes, out, roi_T, feat_T, t_start, argmax)
        r["outs"] = [(out, R.act_view(out).clone())]
        rec.recs.append(r)
        return ret

    def forward_act(self, cat, ctx_mean=None, ctx_row_map=None, want_logits=False, keep=None):
        start = len(rec.recs)
        res = orig["forward_act"](self, cat, ctx_mean, ctx_row_map, want_logits, keep)
        if not self.cls_only:
            exits = [r for r in rec.recs[start:] if r["kind"] == "exit"]
            if fused_exit:
                assert exits, "the inference head runs the fused exit"
                lf2 = exits[-1]["outs"][0][1]
            else:
                assert not exits, "this head was expected to run its exits unfused"
                lf2 = [r for r in rec.recs[start:] if r["kind"] == "conv"][-1]["outs"][0][1]    # downsample2
            rec.recs.append(dict(kind="regress", x=lf2.reshape(-1, *lf2.shape[2:]), mods=(self.local_reg, self.neighbor_reg1,
                                 self.neighbor_reg2), Tc=self.T, T=cat.T, outs=[(t, t.clone()) for t in res[1:4]]))
        return res

    mp.setattr(E, "conv", conv)
    mp.setattr(E, "maxpool", maxpool)
    mp.setattr(E, "bottleneck_exit", bottleneck_exit)
    mp.setattr(E, "mean_mid", mean_mid)
    mp.setattr(E, "linear_small_n", linear_small_n)
    mp.setattr(networks.ROINet, "pool_into", pool_into)
    mp.setattr(two_branch.TwoBranchNet, "forward_act", forward_act)


def run(cfg, nets, x, tubes, context):
    import step_b200
    with torch.no_grad():
        cf = nets["base_net"](x)
        ctx = nets["context_net"](cf) if context else None
        hist, _ = step_b200.inference(cfg, cf, ctx, nets, cfg.max_iter, tubes, want_trajectory=False)
    outs = [cf.clone()] + ([ctx.clone()] if ctx is not None else [])
    for h in hist:
        outs += [h[k].clone() for k in ("pred_prob", "pred_loc", "pred_first_loc", "pred_last_loc") if h[k] is not None]
    return outs


def setup(name):
    from step_b200 import engine as E
    kw, B, T_in, side, N, context = GEOMS[name]
    assert E.BRANCH_STREAMS and E.FUSE_1X1 and E.FUSE_EXIT and E.A_MODE == E.L.A_BEST, "engine switches off their defaults"
    cfg = synth.make_cfg(fp16=True, **kw)
    nets = build(cfg, context)
    x = synth.make_clips(B, T_in, side, side).cuda()
    tubes = synth.make_proposals(B, N, cfg.T * cfg.NUM_CHUNKS[1], side, side)
    return cfg, nets, x, tubes, context, B


def profiled_kernel_names(name):
    """Kernel names of one un-instrumented eager run under torch.profiler.  Runs in a child process: a profiling session of
    this size leaves CUPTI's kernel records off for later sessions in the same process (test_gpu_stem.py's)."""
    cfg, nets, x, tubes, context, _ = setup(name)
    run(cfg, nets, x, tubes, context)                           # weights packed outside the profiled window
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(cfg, nets, x, tubes, context)
        torch.cuda.synchronize()
    return sorted({e.key for e in prof.key_averages()})


@pytest.fixture(scope="module", params=sorted(GEOMS))
def geom(request):
    """One geometry: the kernel names of a profiled run (child process), an un-instrumented eager run (reference
    outputs), then the instrumented run."""
    name = request.param
    child = subprocess.run([sys.executable, os.path.abspath(__file__), name], cwd=ROOT, capture_output=True, text=True,
                           timeout=600)
    assert child.returncode == 0, child.stderr[-4000:]
    names = set(json.loads(child.stdout.strip().splitlines()[-1]))
    cfg, nets, x, tubes, context, B = setup(name)
    plain = run(cfg, nets, x, tubes, context)
    torch.cuda.synchronize()
    rec = Recorder()
    with pytest.MonkeyPatch.context() as mp:
        install(mp, rec)
        import step_b200
        with torch.no_grad():
            rec.rows = (0, B - 1) if B > 2 else None
            cf = nets["base_net"](x)
            ctx = nets["context_net"](cf) if context else None
            rec.rows = None
            hist, _ = step_b200.inference(cfg, cf, ctx, nets, cfg.max_iter, tubes, want_trajectory=False)
        inst = [cf.clone()] + ([ctx.clone()] if ctx is not None else [])
        for h in hist:
            inst += [h[k].clone() for k in ("pred_prob", "pred_loc", "pred_first_loc", "pred_last_loc") if h[k] is not None]
        torch.cuda.synchronize()
    yield dict(name=name, cfg=cfg, recs=rec.recs, plain=plain, inst=inst, names=names)


def test_launch_census(geom):
    got = {}
    for r in geom["recs"]:
        got[r["kind"]] = got.get(r["kind"], 0) + 1
    assert got == CENSUS[geom["name"]], got
    convs = [r for r in geom["recs"] if r["kind"] == "conv"]
    if geom["name"] == "shipped":
        # Mixed_3b / 4b's 16-channel 3x3x3 convolutions on 18 and 9 planes: the patch kernel with TT = 4 and a last plane
        # group of 2 and 1 planes (conv_halo.cu halo_launch_cols; A_BEST takes the patch kernel for Cin <= 32 on maps >= 14)
        ots = sorted({r["out_dims"][0] for r in convs if r["x"].shape[-1] == 16 and r["k"] == (3, 3, 3)})
        assert ots == [9, 18], ots


def _c4_tiles():
    """(BK, BN) of every wgmma layer of the C4 table (its `after` section: this tree's kernel per layer)."""
    text = open(os.path.join(ROOT, "profiles", "h100_conv_layers_c4.txt")).read()
    sec = re.search(r"== after:.*?\n(.*?)\n== ", text, re.S).group(1)
    rows = re.findall(r"^(\S+)\s+\d+\s+(umma|halo|exit)\s+\S+\s+\S+\s+(\S+)\s+(\S+)", sec, re.M)
    assert len(rows) >= 40, "profiles/h100_conv_layers_c4.txt changed its layout: update this parser"
    return {(int(bk), int(bn)) for _, kern, bk, bn in rows if kern == "umma"}


def test_kernels_reached(geom):
    """The profiled eager run reaches the kernels this file is meant to cover.  If the C4 table or the tile list of
    conv_umma.cu changes, this says so instead of silently covering less."""
    names = geom["names"]
    has = lambda pat: any(re.search(pat, n) for n in names)
    src = open(os.path.join(ROOT, "step_b200", "csrc", "conv_umma.cu")).read()
    body = re.search(r"#define STEP_CONV_TILES\(X\)(.*?)\n\n", src, re.S).group(1)
    tiles = {(int(a), int(b)) for a, b in re.findall(r"X\((\d+),\s*(\d+)\)", body)}
    table = _c4_tiles()
    assert table == tiles - {(16, 64)}, ("the C4 layer table and STEP_CONV_TILES disagree", sorted(table ^ (tiles - {(16, 64)})))
    need = ["conv_stem_kernel", r"conv_halo_kernel<\d+, \d+, 4>", "bottleneck_exit_kernel", "maxpool3d_333_march_kernel",
            r"maxpool3d_march_kernel<[^,]+, 1, 3, 3,", r"maxpool3d_march_kernel<[^,]+, 3, 3, 3,", "linear_mma_kernel",
            "roi_align_fwd_nhwc_f16_packed_kernel"]
    if geom["name"] == "c4":
        need += [r"conv_umma_kernel<%d, %d>" % t for t in sorted(table)]
    missing = [p for p in need if not has(p)]
    assert not missing, (missing, sorted(n for n in names if "kernel" in n))


def test_instrumented_run_is_bit_identical_and_writes_persist(geom):
    check_instrumented_run(geom)


def check_instrumented_run(geom):
    """The instrumented run's outputs equal the plain run's bit for bit, every region a launch wrote still holds what it
    wrote when the forward ends, and an accumulating linear launch read what the launch before it wrote."""
    assert len(geom["plain"]) == len(geom["inst"])
    for a, b in zip(geom["plain"], geom["inst"]):
        assert torch.equal(a, b)
    accumulated = {id(r["y0_of"]) for r in geom["recs"] if r["kind"] == "linear" and r["y0_of"] is not None}
    for i, r in enumerate(geom["recs"]):
        for o, snap in r["outs"]:
            if torch.is_tensor(o):
                if id(o) in accumulated and r.get("y0_of") is None:
                    continue                                     # accumulated into by the next launch: checked below
                live = o
            else:
                live = R.act_view(o)
            assert torch.equal(live, snap), (i, r["kind"], "written region changed after the launch")
    # an accumulating launch read exactly what the launch before it wrote
    lin = [r for r in geom["recs"] if r["kind"] == "linear"]
    for prev, r in zip(lin, lin[1:]):
        if r["y0"] is not None:
            assert r["y0_of"] is prev["outs"][0][0] and torch.equal(r["y0"], prev["outs"][0][1][:r["M"]])


def _conv(r, what):
    widths = [snap.shape[-1] for _, snap in r["outs"]]
    ys, xws, epis = R.conv_fwd(r["x"], r["w"], r["scale"], r["shift"], r["res"], r["k"], r["stride"], r["pad_lo"],
                               r["out_dims"], r["relu"], widths)
    steps = R.conv_steps(r["k"], r["x"].shape[-1])
    assert steps * 2 * R.U32 <= R.U12, (what, steps)
    for j, ((_, snap), y, xw, epi) in enumerate(zip(r["outs"], ys, xws, epis)):
        R.check_fwd(snap[r["sel"]], y, xw, epi, steps, (what, j))


def _exit(r, what):
    ref = R.exit_fwd(r["h"], r["w3"], r["x"], r["w1"], r["shift2"], r["relu2"])
    M = r["h"].shape[0]
    z = r["outs"][0][1].reshape(M, -1)
    R.check_fwd(z, ref["z"], ref["z_xw"], ref["z_epi"], R.conv_steps((1, 1, 1), r["x"].shape[1]), (what, "z"),
                extra=ref["z_carry"])
    if len(r["outs"]) > 1:
        R.check_fwd(r["outs"][1][1].reshape(M, -1), ref["y"], ref["y_xw"], ref["y_epi"], R.conv_steps((1, 1, 1), r["h"].shape[1]),
                    (what, "y"))
    # the fused launch == the two step_conv3d_fwd launches it replaces, bit for bit (same fp16 y, same K order)
    from step_b200 import engine as E
    from step_b200.engine import Act
    rows = lambda t: Act(t.contiguous().view(M, 1, 1, 1, t.shape[1]))
    y2 = rows(torch.empty(M, r["x"].shape[1], dtype=torch.float16, device="cuda"))
    z2 = rows(torch.empty(M, z.shape[1], dtype=torch.float16, device="cuda"))
    E.conv(rows(r["h"]), r["w3"], None, None, y2, (1, 1, 1), relu=True, residual=rows(r["x"]))
    E.conv(y2, r["w1"], None, r["shift2"], z2, (1, 1, 1), relu=r["relu2"])
    assert torch.equal(z2.buf.view(M, -1), z), (what, "fused exit != two launches")
    if len(r["outs"]) > 1:
        assert torch.equal(y2.buf.view(M, -1), r["outs"][1][1].reshape(M, -1)), (what, "y")


def _within(got, ref, tol, what):
    err = (got.double() - ref).abs()
    ok = err <= tol
    assert bool(ok.all()), (what, int((~ok).sum()), float((err - tol).max()))


def _mean_mid(r, what):
    ref, mabs = R.mean_mid(r["x"])
    _within(r["outs"][0][1], ref, R.mean_mid_tol(ref, mabs, r["x"].shape[1]), what)


def _linear(r, what):
    x = r["x"] if r["row_map"] is not None else r["x"][:r["M"]]
    y, _, a = R.linear(x, r["w"], r["bias"], r["y0"], r["row_map"], r["act"])
    got = r["outs"][0][1][:r["M"], :y.shape[1]]
    _within(got, y, R.linear_tol(y, a, r["K"], r["act"]), what)


def _regress(r, what):
    ref = R.head_regress(r["x"], *r["mods"], r["Tc"], r["T"])
    for (_, got), key in zip(r["outs"], ("local", "first", "last")):
        _within(got, ref[key], ref[key + "_tol"], (what, key))


def _roi(r, what):
    assert r["mode"] == "align"
    ps = r["size"]
    out, out_abs = R.roi_align(r["feat"], r["rois"], 1.0 / 16.0, ps, ps, r["roi_T"], r["feat_T"], r["t_start"])
    got = r["outs"][0][1].reshape(-1, ps, ps, r["feat"].shape[-1]).cpu()
    _within(got, out, R.roi_align_tol(out_abs, float(r["feat"].abs().max())), what)


def _pool(r, what):
    ref = R.pool_fwd(r["x"], r["k"], r["stride"], r["pad_lo"], r["pad_hi"])
    assert torch.equal(r["outs"][0][1].cpu().double(), ref), what


def test_every_launch_against_float64(geom):
    """Each recorded launch against its float64 reference with the derived bound (module docstring)."""
    check = dict(conv=_conv, pool=_pool, exit=_exit, mean_mid=_mean_mid, linear=_linear, roi=_roi, regress=_regress)
    for i, r in enumerate(geom["recs"]):
        what = (geom["name"], i, r["kind"])
        if r["kind"] == "conv":
            what += (r["k"], r["x"].shape[-1], tuple(r["out_dims"]))
        check[r["kind"]](r, what)
        torch.cuda.synchronize()


if __name__ == "__main__":                                     # the fixture's child process: python <this file> <geometry>
    print(json.dumps(profiled_kernel_names(sys.argv[1])))
