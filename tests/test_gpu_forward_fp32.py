"""GPU: the fp32 forward (cfg.fp16=False, the reference's default precision) against exact replays and float64 references
on the operands each launch read.

  * The SIMT convolution at its edges (conv3d_simt_kernel, fp32 storage and, through a_mode=A_SIMT, __half storage):
    engine.conv on Acts, every output equal to tests/_simt_replay.py's bit-exact replay, and the guard columns around
    every output slice untouched.  Cin 4 (the stem's padded clip, channel 3 zero), 12, 20, 48, 832, 1024; Cout 8, 63,
    64, 65, 112, 208, 384; M off the 64-row tile over several clips; the stride-2 7x7x7 stem, (1,3,3) and (3,3,3) at
    stride 1 and 2, 1x1; TF-SAME asymmetric padding on odd extents; channel slices of the input, residual and output;
    scale / shift / ReLU / residual present and absent.  Also every shape tests/test_gpu_conv_tiles.py runs through the
    __half instance, which those tests (and test_gpu_conv_persistent.py, the wgmma-vs-SIMT tests of test_gpu_conv.py)
    use as their reference.
  * The forward launch by launch (the wrappers of tests/test_gpu_forward_layers.py around engine.conv, engine.maxpool,
    engine.mean_mid, engine.linear_small_n, ROINet.pool_into and TwoBranchNet.forward_act; the fp32 head runs its
    bottleneck exits and Mixed 1x1 convolutions unfused) on three geometries: the shipped inference configuration (one
    36 x 400 x 400 clip, ContextNet, steps of 3, 3 and 9 frames), the classification stage's class-only head at 400 x 400
    (T = 9, ContextNet's per-clip mean), and a 14 x 66 x 82 clip (odd extents at every strided pool, ragged M tiles in
    every layer).  Per launch:
      conv:      torch.equal with the replay on every row of the first and the last 64-row M tile, every row of the first
                 and the last output plane whose window touches the padding, and 4096 seeded random rows; and all
                 outputs within R.check_fwd32's bound (one fmaf chain of taps x Cin terms, three epilogue roundings);
      pools:     torch.equal (a maximum is exact);
      mean_mid:  torch.equal with B fp32 additions in index order and one division;
      linear / step_head_regress: R.linear_tol, R.head_regress with the fp32 weights;
      ROIAlign:  R.roi_align within R.roi_align_tol;
      clip_to_ndhwc: the stem's input equals the clip channels-last, its padding channel zero.
    A census of launches per kind, derived from the module structure; every written region unchanged at the end; the
    instrumented run's outputs bit-identical to a plain run's; and a profiled child-process run that reaches every fp32
    forward kernel."""
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
import _simt_replay as S  # noqa: E402
import _tape_reference as R  # noqa: E402
import test_gpu_forward_layers as FL  # noqa: E402
from step_b200 import synth  # noqa: E402
from test_gpu_pipeline import build  # noqa: E402

pytestmark = pytest.mark.gpu
WORST = {}
SENTINEL = -1234.0               # guard-column fill (exact in fp16 and fp32)


def _note(kind, v):
    WORST[kind] = max(WORST.get(kind, 0.0), v)


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    print("\nfp32 forward, worst error / bound:", {k: "%.3g" % v for k, v in sorted(WORST.items())})


# ---- the SIMT convolution at its edges ------------------------------------------------------------------------------
# name: N, T, H, W, Cin, in (ld, coff), Cout, k, stride, epilogue "scale shift relu" (1 / 0), residual (ld, coff) | None,
#       out (ld, coff)
EDGE = {
    "stem_7x7x7_s2_cin4": (1, 9, 21, 19, 4, (4, 0), 64, (7, 7, 7), (2, 2, 2), "111", None, (72, 4)),
    "k133_cin12_cout63_in_slice": (2, 3, 13, 11, 12, (20, 4), 63, (1, 3, 3), (1, 1, 1), "100", (70, 3), (63, 0)),
    "k333_cin20_cout65": (3, 5, 7, 9, 20, (20, 0), 65, (3, 3, 3), (1, 1, 1), "011", (65, 0), (80, 12)),
    "k333_cin48_cout112_slices": (2, 4, 9, 7, 48, (56, 8), 112, (3, 3, 3), (1, 1, 1), "111", (120, 8), (120, 4)),
    "1x1_cin832_cout208": (2, 3, 7, 7, 832, (1088, 0), 208, (1, 1, 1), (1, 1, 1), "111", None, (480, 272)),
    "1x1_cin1024_cout384_res": (3, 1, 7, 7, 1024, (1024, 0), 384, (1, 1, 1), (1, 1, 1), "010", (400, 16), (392, 8)),
    "1x1_cin20_cout8": (3, 5, 5, 3, 20, (24, 4), 8, (1, 1, 1), (1, 1, 1), "001", None, (8, 0)),
    "k133_s122_odd_cin16_cout64": (2, 3, 15, 13, 16, (16, 0), 64, (1, 3, 3), (1, 2, 2), "111", (64, 0), (64, 0)),
    "k333_s2_odd_cin24_cout65": (1, 7, 9, 11, 24, (32, 8), 65, (3, 3, 3), (2, 2, 2), "110", (72, 7), (65, 0)),
}


def _edge_operands(name, dtype):
    from step_b200 import _lib as L, engine as E
    from step_b200.engine import Act
    N, T, H, W, Cin, (in_ld, coff), Cout, k, stride, epi, res, (out_ld, out_coff) = EDGE[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    code = L.F16 if dtype == torch.float16 else L.F32
    xb = torch.randn(N, T, H, W, in_ld, generator=g)
    cin_w = 3 if Cin == 4 and k == (7, 7, 7) else Cin      # the stem: 3 live channels, the 4th zero in input and filter
    if cin_w != Cin:
        xb[..., coff + cin_w:coff + Cin] = 0.0
    x = Act(xb.to(dtype).cuda(), Cin, coff)
    w = torch.randn(Cout, cin_w, *k, generator=g) / (cin_w * k[0] * k[1] * k[2]) ** 0.5
    wp = E.pack_conv_weight(w.cuda(), code, cin_pad=Cin if dtype == torch.float32 else None)
    scale = (torch.rand(Cout, generator=g) + 0.5).cuda() if epi[0] == "1" else None
    shift = torch.randn(Cout, generator=g).cuda() if epi[1] == "1" else None
    pad_lo = tuple(E.same_pad(kk, s)[0] for kk, s in zip(k, stride))
    od = E.same_out_dims((T, H, W), k, stride)
    residual = None
    if res is not None:
        residual = Act(torch.randn(N, *od, res[0], generator=g).to(dtype).cuda(), Cout, res[1])
    out = Act(torch.full((N,) + od + (out_ld,), SENTINEL, dtype=dtype, device="cuda"), Cout, out_coff)
    return x, wp, scale, shift, residual, out, k, stride, pad_lo, od, epi[2] == "1"


def _run_and_replay(x, wp, scale, shift, residual, out, k, stride, pad_lo, od, relu, a_mode, what):
    """engine.conv into `out`, then: every output equals the replay, the guard columns hold SENTINEL."""
    from step_b200 import engine as E
    dtype = x.buf.dtype
    E.conv(x, wp, scale, shift, out, k, stride, pad_lo, relu, residual, a_mode=a_mode, out_dims=od)
    torch.cuda.synchronize()
    M = x.N * od[0] * od[1] * od[2]
    got = R.act_view(out).reshape(M, out.C)
    want = S.simt_conv_replay(R.act_view(x), wp, scale, shift, R.act_view(residual) if residual is not None else None, k,
                              stride, pad_lo, od, relu, dtype=dtype)
    if not torch.equal(got, want):
        bad = (got != want).nonzero()
        m, c = (int(v) for v in bad[0])
        raise AssertionError("%s: %d of %d outputs differ from the replay; first at row %d column %d: got %r want %r" % (
            what, bad.shape[0], got.numel(), m, c, float(got[m, c]), float(want[m, c])))
    guard = torch.cat([out.buf[..., :out.coff].reshape(-1), out.buf[..., out.coff + out.C:].reshape(-1)])
    assert bool((guard == SENTINEL).all()), (what, "a guard column around the output slice was written")
    return got


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["fp32", "fp16_simt"])
@pytest.mark.parametrize("name", list(EDGE))
def test_simt_conv_edges_bit_exact(name, dtype):
    from step_b200 import _lib as L
    ops = _edge_operands(name, dtype)
    _run_and_replay(*ops, a_mode=L.A_SIMT if dtype == torch.float16 else None, what=(name, str(dtype)))


def test_simt_fp16_reference_shapes_of_conv_tiles():
    """The __half instance on every shape test_gpu_conv_tiles.py compares the wgmma tiles against: per tile its (Cin,
    Cout), (1,3,3) and (1,1,1) filters, scale, shift, residual, ReLU, the output in a channel slice, M = 12528."""
    from step_b200 import _lib as L, engine as E
    from step_b200.engine import Act
    import test_gpu_conv_tiles as CT
    N, T, H, W = 4, 4, 27, 29
    for bk, bn in CT.TILES:
        Cin, Cout = CT.shape_for(bk, bn)
        g = torch.Generator().manual_seed(bn * 100 + bk)
        x = Act(torch.randn(N, T, H, W, Cin, generator=g).half().cuda())
        scale = (torch.rand(Cout, generator=g) + 0.5).cuda()
        shift = torch.randn(Cout, generator=g).cuda()
        res = Act(torch.randn(N, T, H, W, Cout, generator=g).half().cuda())
        for k in ((1, 3, 3), (1, 1, 1)):
            w = (torch.randn(Cout, Cin, *k, generator=g) / (Cin * k[0] * k[1] * k[2]) ** 0.5).half().cuda()
            out = Act(torch.full((N, T, H, W, Cout + 16), SENTINEL, dtype=torch.float16, device="cuda"), Cout, 8)
            pad = tuple(E.same_pad(kk, 1)[0] for kk in k)
            _run_and_replay(x, E.pack_conv_weight(w, L.F16), scale, shift, res, out, k, (1, 1, 1), pad, (T, H, W), True,
                            a_mode=L.A_SIMT, what=(bk, bn, k))


# ---- the fp32 forward launch by launch ------------------------------------------------------------------------------
GEOMS = {
    # cfg, clips, T_in, H, W, proposals per clip, head kind
    "shipped": (dict(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False, image_size=(400, 400)), 1, 36, 400, 400,
                11, "full"),
    "cls_stage": (dict(T=9, max_iter=1, NUM_CHUNKS={1: 1}, no_context=False, image_size=(400, 400)), 1, 36, 400, 400, 11, "cls"),
    "odd_14x66x82": (dict(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 1}, no_context=False, image_size=(82, 66)), 1, 14, 66, 82,
                     7, "full"),
}
# Launches per kind, from the module structure.  Trunk: stem, conv3d_2b / 2c, 7 Mixed x 6 unfused convs = 45 convs; 3
# strided pools + 7 branch-3 pools.  ContextNet: its pool and two Mixed (12 convs, 3 pools) and the spatial mean.  A step
# of a full head: Mixed_5b / 5c (12 convs, 2 pools), downsample, the local branch (4 + 3 + 3 convs), downsample2 = 24
# convs, the temporal mean of the context rows and of the features, the classifier and its context columns,
# step_head_regress, one ROIAlign.  The class-only head: 13 convs, 2 pools, both means, both linear launches, one ROIAlign.
CENSUS = {
    "shipped": dict(conv=45 + 12 + 3 * 24, pool=10 + 3 + 3 * 2, mean_mid=1 + 3 * 2, linear=3 * 2, roi=3, regress=3),
    "cls_stage": dict(conv=45 + 12 + 13, pool=10 + 3 + 2, mean_mid=1 + 2, linear=2, roi=1),
    "odd_14x66x82": dict(conv=45 + 12 + 3 * 24, pool=10 + 3 + 3 * 2, mean_mid=1 + 3 * 2, linear=3 * 2, roi=3, regress=3),
}


def setup(name):
    kw, B, T_in, H, W, n, head = GEOMS[name]
    cfg = synth.make_cfg(fp16=False, **kw)
    if head == "cls":
        nets = build(synth.make_cfg(fp16=False, **dict(kw, max_iter=0)), True)
        nets["det_net0"] = synth.device_head(cfg, synth.cls_head_state_dict(100, cfg), cls_only=True)
    else:
        nets = build(cfg, True)
    x = synth.make_clips(B, T_in, H, W).cuda()
    tubes = synth.make_proposals(B, n, cfg.T * cfg.NUM_CHUNKS[1], W, H)
    return cfg, nets, x, tubes, head


def _cls_step(cfg, nets, cf, ctx, tubes):
    """The classification stage's head on one step, as inference_device runs a step: ROIAlign into the concat buffer,
    the context's temporal mean per clip, the class-only head with the tube -> clip row map."""
    from step_b200 import _lib as L, engine as E
    from step_b200.engine import Act
    from step_b200.inference import stage_tubes
    from step_b200.networks import act_of
    feat = act_of(cf)
    dev = cf.device
    flat, clip_of_tube, _ = stage_tubes(tubes, dev)
    head = nets["det_net0"]
    T_len = cfg.NUM_CHUNKS[1] * cfg.T
    cat = Act.empty(flat.shape[0], T_len, head.pool_size, head.pool_size, 832 + head.fc_dim, L.F32, dev)
    nets["roi_net"].pool_into(feat, flat, cat.frames().slice(0, 832), T_len, feat.T, 0)
    ctx_all = ctx.detach().float().reshape(feat.N, ctx.shape[1], feat.T).permute(0, 2, 1).contiguous()
    sl = ctx_all[:, :T_len].contiguous()
    ctx_mean = E.mean_mid(sl.data_ptr(), L.F32, feat.N, T_len, 1, sl.shape[2], sl.shape[2], dev)
    return [head.forward_act(cat, ctx_mean, clip_of_tube)[0]]


def run(cfg, nets, x, tubes, head):
    import step_b200
    with torch.no_grad():
        cf = nets["base_net"](x)
        ctx = nets["context_net"](cf)
        outs = [cf.clone(), ctx.clone()]
        if head == "cls":
            return outs + [t.clone() for t in _cls_step(cfg, nets, cf, ctx, tubes)]
        hist, _ = step_b200.inference(cfg, cf, ctx, nets, cfg.max_iter, tubes, want_trajectory=False)
    for h in hist:
        outs += [h[k].clone() for k in ("pred_prob", "pred_loc", "pred_first_loc", "pred_last_loc") if h[k] is not None]
    return outs


def profiled_kernel_names(name):
    """Kernel names of one un-instrumented run under torch.profiler, in a child process (test_gpu_forward_layers.py's
    profiled_kernel_names says why)."""
    cfg, nets, x, tubes, head = setup(name)
    run(cfg, nets, x, tubes, head)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(cfg, nets, x, tubes, head)
        torch.cuda.synchronize()
    return sorted({e.key for e in prof.key_averages()})


@pytest.fixture(scope="module", params=sorted(GEOMS))
def geom(request):
    name = request.param
    child = subprocess.run([sys.executable, os.path.abspath(__file__), name], cwd=ROOT, capture_output=True, text=True,
                           timeout=900)
    assert child.returncode == 0, child.stderr[-4000:]
    names = set(json.loads(child.stdout.strip().splitlines()[-1]))
    cfg, nets, x, tubes, head = setup(name)
    plain = run(cfg, nets, x, tubes, head)
    torch.cuda.synchronize()
    rec = FL.Recorder()
    with pytest.MonkeyPatch.context() as mp:
        FL.install(mp, rec, fused_exit=False)
        inst = run(cfg, nets, x, tubes, head)
        torch.cuda.synchronize()
    yield dict(name=name, cfg=cfg, recs=rec.recs, plain=plain, inst=inst, names=names, clip=x)


def test_launch_census(geom):
    got = {}
    for r in geom["recs"]:
        got[r["kind"]] = got.get(r["kind"], 0) + 1
    assert got == CENSUS[geom["name"]], got
    convs = [r for r in geom["recs"] if r["kind"] == "conv"]
    assert all(r["x"].dtype == torch.float32 and len(r["outs"]) == 1 for r in convs)
    assert convs[0]["k"] == (7, 7, 7) and convs[0]["stride"] == (2, 2, 2) and convs[0]["x"].shape[-1] == 4
    if geom["name"] == "odd_14x66x82":
        # every strided pool sees an odd extent, and no layer's M is a multiple of the 64-row tile
        strided = [r for r in geom["recs"] if r["kind"] == "pool" and r["stride"] != (1, 1, 1)]
        assert strided and all(any(d % 2 for d, s in zip(r["x"].shape[1:4], r["stride"]) if s == 2) for r in strided)
        ms = [r["x"].shape[0] * r["out_dims"][0] * r["out_dims"][1] * r["out_dims"][2] for r in convs]
        assert all(m % 64 for m in ms), sorted(set(m for m in ms if m % 64 == 0))


def test_kernels_reached(geom):
    names = geom["names"]
    has = lambda pat: any(re.search(pat, n) for n in names)
    need = [r"conv3d_simt_kernel<float>", r"maxpool3d_333_march_kernel<float>", r"maxpool3d_march_kernel<float,",
            r"maxpool3d_kernel<float,", r"mean_mid_kernel<float, float>", r"linear_splitk_kernel<float>", "linear_reduce_kernel",
            r"roi_align_fwd_nhwc_kernel<float, true>", r"clip_to_ndhwc_kernel<float>"]
    if geom["name"] != "cls_stage":
        need.append("head_reg_reduce_kernel")
    missing = [p for p in need if not has(p)]
    assert not missing, (missing, sorted(n for n in names if "kernel" in n))
    assert not has(r"conv_(umma|halo|stem)_kernel|bottleneck_exit_kernel|linear_mma_kernel"), "an fp16 kernel ran on the fp32 path"


def test_instrumented_run_is_bit_identical_and_writes_persist(geom):
    FL.check_instrumented_run(geom)


def sample_rows(r, gen):
    """Flat output pixels the replay checks: the first and the last 64-row M tile, every pixel of the first and the last
    output plane whose window touches the padding, and 4096 seeded random pixels."""
    x = r["x"]
    od, k, stride, pad = r["out_dims"], r["k"], r["stride"], r["pad_lo"]
    M = x.shape[0] * od[0] * od[1] * od[2]
    dev = x.device
    every = torch.arange(M, device=dev)
    _, ot, _, _ = S.conv_rows(every, od)
    edge = ((ot == 0) | (ot == od[0] - 1)) & S.touches_padding(every, tuple(x.shape[1:4]), k, stride, pad, od)
    parts = [every[:64], every[(M - 1) // 64 * 64:], every[edge], torch.randint(M, (4096,), generator=gen).to(dev)]
    return torch.unique(torch.cat(parts))


def _conv(r, gen, what):
    (o, snap), = r["outs"]
    od = r["out_dims"]
    M = r["x"].shape[0] * od[0] * od[1] * od[2]
    Cin = r["x"].shape[-1]
    rows = sample_rows(r, gen)
    want = S.simt_conv_replay(r["x"], r["w"], r["scale"], r["shift"], r["res"], r["k"], r["stride"], r["pad_lo"], od, r["relu"],
                              rows=rows)
    got = snap.reshape(M, -1)[rows]
    if not torch.equal(got, want):
        bad = (got != want).nonzero()
        i, c = (int(v) for v in bad[0])
        raise AssertionError("%s: %d of %d sampled outputs differ from the replay; first at row %d column %d: got %r want %r"
                             % (what, bad.shape[0], got.numel(), int(rows[i]), c, float(got[i, c]), float(want[i, c])))
    (y,), (xw,), (epi,) = R.conv_fwd(r["x"], r["w"], r["scale"], r["shift"], r["res"], r["k"], r["stride"], r["pad_lo"], od,
                                     r["relu"])
    n = r["k"][0] * r["k"][1] * r["k"][2] * Cin
    _note("conv", R.check_fwd32(snap, y, xw, epi, n, what))


def _pool(r, what):
    ref = R.pool_fwd(r["x"], r["k"], r["stride"], r["pad_lo"], r["pad_hi"])
    assert torch.equal(r["outs"][0][1].cpu().double(), ref), what


def _mean_mid(r, what):
    assert r["x"].dtype == torch.float32
    assert torch.equal(r["outs"][0][1], S.mean_mid_replay(r["x"])), what
    ref, mabs = R.mean_mid(r["x"])
    _note("mean_mid", R._check_within(r["outs"][0][1], ref, R.mean_mid_tol(ref, mabs, r["x"].shape[1]), what))


def _linear(r, what):
    x = r["x"] if r["row_map"] is not None else r["x"][:r["M"]]
    y, _, a = R.linear(x, r["w"], r["bias"], r["y0"], r["row_map"], r["act"])
    got = r["outs"][0][1][:r["M"], :y.shape[1]]
    _note("linear", R._check_within(got, y, R.linear_tol(y, a, r["K"], r["act"]), what))


def _regress(r, what):
    ref = R.head_regress(r["x"], *r["mods"], r["Tc"], r["T"], wdtype=torch.float32)
    for (_, got), key in zip(r["outs"], ("local", "first", "last")):
        _note("regress", R._check_within(got, ref[key], ref[key + "_tol"], (what, key)))


def _roi(r, what):
    assert r["mode"] == "align"
    ps = r["size"]
    out, out_abs = R.roi_align(r["feat"], r["rois"], 1.0 / 16.0, ps, ps, r["roi_T"], r["feat_T"], r["t_start"])
    got = r["outs"][0][1].reshape(-1, ps, ps, r["feat"].shape[-1]).cpu()
    _note("roi_align", R._check_within(got, out, R.roi_align_tol(out_abs, float(r["feat"].abs().max())), what))


def test_every_launch_against_replay_and_float64(geom):
    """The stem's input is the clip channels-last with a zero padding channel; every recorded launch against its exact
    replay and / or float64 reference (module docstring)."""
    stem = next(r for r in geom["recs"] if r["kind"] == "conv")
    clip = geom["clip"].permute(0, 1, 3, 4, 2)
    assert torch.equal(stem["x"][..., :3], clip) and bool((stem["x"][..., 3] == 0).all()), "clip_to_ndhwc"
    gen = torch.Generator().manual_seed(0)
    for i, r in enumerate(geom["recs"]):
        what = (geom["name"], i, r["kind"])
        if r["kind"] == "conv":
            _conv(r, gen, what + (r["k"], r["x"].shape[-1], tuple(r["out_dims"])))
        elif r["kind"] == "pool":
            _pool(r, what)
        else:
            dict(mean_mid=_mean_mid, linear=_linear, regress=_regress, roi=_roi)[r["kind"]](r, what)
        torch.cuda.synchronize()


if __name__ == "__main__":                                     # the fixture's child process: python <this file> <geometry>
    print(json.dumps(profiled_kernel_names(sys.argv[1])))
