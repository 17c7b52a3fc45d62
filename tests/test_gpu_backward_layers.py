"""GPU: the training backward (training.tape_backward and the kernels behind it) layer by layer, against the float64
reference of tests/_tape_reference.py on the SAME fp16 operands: the recorded fp16 activations, the packed fp16 filters,
the fp32 BatchNorm scale and the fp16 output gradient.  Only accumulation order and the final fp16 rounding differ, so
every tolerance below is derived, not fitted.

Tolerances (u32 = 2^-24, the fp32 unit roundoff):
  * dz, dres: torch.equal.  act_bwd_kernel does dz = fp16(fp32(dy) * [y > 0] * scale) and dres = fp16(dres + masked dy)
    in IEEE fp32 with round-to-nearest, exactly what the reference does.
  * dW: |got - ref| <= 2^-12 (|dz|^T |x|) elementwise, and relative L2 <= 1e-4.  The wgrad kernel sums each 2048-pixel
    chunk with wmma (16 products per step, fp32 accumulate: 128 steps) and then the chunks in order (<= 352 at the shipped
    stem), each fp32 addition erring by at most 2 u32 of the running |sum| <= the abs sum (2 for the tensor cores'
    truncating adds): (2 * 128 + 352) u32 < 2^-14.7 < 2^-12.  The 1/loss_scale factor is a power of two: exact.
  * db: the same bound with |dz| summed: colsum adds <= M / 64 + 64 fp32 terms in a chain (< 1200 here): < 2^-13.8.
  * dgrad dx (the forward wgmma kernels on flipped, transposed filters): 2^-12 (|dz| * |w|) for the fp32 accumulation of
    <= taps * Cout / 16 wgmma steps (<= 27 * 1088 / 16 = 1836 at 2 u32: 2^-12.0), plus one fp16 rounding of the result
    bounded by 1 ulp at |ref| + that margin.
  * pool dx: at most 1 fp16 ulp of the reference, ties included: maxpool_bwd_kernel sums <= 27 fp16 gradients in fp32
    (exact to far below an fp16 ulp) and rounds once.
  * chain: an activation's final gradient is its seed plus every consumer's contribution, each added with one fp16
    rounding: the sum of the contributions' margins plus one ulp per accumulation at the running magnitude.
"""
import os
import sys

import pytest
import torch

from step_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _tape_reference as R  # noqa: E402
from _train_case import SHIPPED  # noqa: E402
from step_b200.synth import device_head, device_nets  # noqa: E402

pytestmark = pytest.mark.gpu

U12 = 2.0 ** -12
# (conv entries, pool entries) of each tape, from the module structure: a Mixed block records its fused 1x1 triple, two
# 3x3x3 convs, the branch-3 pool and its 1x1; the trunk adds the stem, conv3d_2b / 2c and three strided pools; ContextNet a
# (1,3,3)/(1,2,2) pool; a full head downsample, 3 + 2 x 3 bottleneck convs plus conv1's projection, downsample2
COUNTS = {"trunk": (3 + 7 * 4, 3 + 7), "context": (2 * 4, 1 + 2), "head": (2 * 4 + 1 + 4 + 2 * 3 + 1, 2), "cls_head": (2 * 4 + 1, 2)}


def counts(tape):
    return sum(e["kind"] == "conv" for e in tape), sum(e["kind"] == "pool" for e in tape)


def record(fn):
    """Run fn with the tape on, as training.trunk_forward_backward does."""
    from step_b200 import engine as E
    tape = []
    with E.recording(tape), torch.no_grad():
        fn()
    return tape


def nets(cfg):
    n = device_nets(cfg, [synth.head_state_dict(100, cfg)], context=True)
    ccfg = synth.make_cfg(fp16=True, T=cfg.T, no_context=True)
    cls = device_head(ccfg, synth.cls_head_state_dict(101, ccfg), cls_only=True)
    return n["base_net"], n["context_net"], n["det_net0"], cls


def head_tape(net, R_, T_, seed, ctx=True):
    from step_b200 import _lib as L
    from step_b200.engine import Act
    gen = torch.Generator(device="cuda").manual_seed(seed)
    cat = Act.empty(R_, T_, 7, 7, 832 + net.fc_dim, L.F16, torch.device("cuda"))
    cat.buf.normal_(generator=gen).relu_()                     # ROI features come out of a ReLU: many exact zeros
    ctx_mean = torch.randn(R_, 1024, device="cuda", generator=gen) if ctx else None
    return record(lambda: net.forward_act(cat, ctx_mean, None, want_logits=True, keep={}))


@pytest.fixture(scope="module")
def tapes():
    """Every tape geometry: the trunk on one 36x400x400 clip (the shipped input) and ContextNet on its output, full heads of
    3 and 9 frames, a class-only head, and the trunk / ContextNet on a 14x66x82 clip, whose extents are odd at every
    strided pool (T 7 at the (3,3,3)/(2,2,2) pool; H 33, 17, 9 and W 41, 21, 11 at the three strided trunk pools; 5 x 6
    at ContextNet's)."""
    cfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(400, 400))
    base, ctx, head, cls = nets(cfg)
    out = {}
    for name, shape in (("shipped", (36, 400, 400)), ("odd", (14, 66, 82))):
        x = synth.make_clips(1, *shape, seed=7).cuda()
        box = {}
        out["trunk_" + name] = record(lambda: box.__setitem__("feat", base.forward_act(x)))
        out["context_" + name] = record(lambda: ctx.forward_act(box["feat"], keep={}))
    out["head_T3"] = head_tape(head, 4, 3, 1)
    out["head_T9"] = head_tape(head, 3, 9, 2)
    out["cls_head"] = head_tape(cls, 4, 3, 3, ctx=False)
    return out


def kernel_dz(e, dys):
    """dz as tape_backward forms it (step_act_bwd_f16 per output into one dense buffer), for the exact comparison."""
    from step_b200 import _lib as L
    outs = [e["out"]] + e["extra_outs"]
    o0 = outs[0]
    n_total = sum(o.C for o in outs)
    dz = torch.empty((o0.N, o0.T, o0.H, o0.W, n_total), dtype=torch.float16, device="cuda")
    col = 0
    for o, dy in zip(outs, dys):
        sc = e["scale"][col:col + o.C] if e["scale"] is not None else None
        L.check(L.lib().step_act_bwd_f16(L.ptr(dy), o.C, L.c_void_p(o.data_ptr()), o.ld, L.ptr(sc), 1 if e["relu"] else 0,
                                         o.N * o.T * o.H * o.W, o.C, L.c_void_p(dz.data_ptr() + 2 * col), n_total, None, 0, L.stream()))
        col += o.C
    return dz


def check_wgrad(got, ref, bound, what):
    got = got.double()
    err = (got - ref).abs()
    assert bool((err <= U12 * bound).all()), (what, float((err / bound.clamp(min=1e-300)).max()))
    rn = float(ref.norm())
    if rn == 0.0:
        assert float(got.abs().max()) == 0.0, what
    else:
        assert float(err.norm()) <= 1e-4 * rn, (what, float(err.norm()) / rn)


def dgrad_tol(ref, bound):
    margin = U12 * bound
    return margin + R.ulp16(ref.abs() + margin)


def check_params(grads, ref, what):
    n = 0
    for w, dW, bW, bias, db, bdb in ref["params"]:
        if w.requires_grad:
            check_wgrad(grads[w], dW, bW, (what, "weight", tuple(w.shape)))
            n += 1
        if bias is not None and bias.requires_grad:
            check_wgrad(grads[bias], db, bdb, (what, "bias", tuple(bias.shape)))
            n += 1
    assert len(grads) == n, what


def entry_shift(e):
    """The fp32 shift the forward launch of a conv entry read: the folded BatchNorm of its Unit3Dpy container(s), or the
    bias of an nn.Conv container (engine.conv keeps the scale on the tape, not the shift)."""
    from step_b200 import _lib as L
    parts = []
    for tg, o in zip(R.tags_of(e), [e["out"]] + e["extra_outs"]):
        if isinstance(tg, tuple):                              # ("s2d", stem unit)
            parts.append(tg[1].packed(L.F16, s2d=True)[2])
        elif hasattr(tg, "packed"):
            parts.append(tg.packed(L.F16)[2])
        else:
            parts.append(tg.bias.detach().float() if tg.bias is not None else torch.zeros(o.C, device="cuda"))
    return torch.cat(parts) if any(p is not None for p in parts) else None


def check_conv_forward(e, what):
    """The entry's forward outputs against conv_fwd (tests/test_gpu_forward_layers.py derives the bound)."""
    outs = [e["out"]] + e["extra_outs"]
    o0 = outs[0]
    res = R.act_view(e["residual"]) if e["residual"] is not None else None
    ys, xws, epis = R.conv_fwd(R.act_view(e["x"]), e["w"], e["scale"], entry_shift(e), res, e["k"], e["stride"], e["pad_lo"],
                               (o0.T, o0.H, o0.W), e["relu"], [o.C for o in outs])
    steps = R.conv_steps(e["k"], e["x"].C)
    for j, (o, y, xw, epi) in enumerate(zip(outs, ys, xws, epis)):
        R.check_fwd(R.act_view(o), y, xw, epi, steps, (what, "forward", j))


def isolate_conv(e, gen, loss_scale, what):
    from step_b200 import training
    outs = [e["out"]] + e["extra_outs"]
    check_conv_forward(e, what)
    gs = training.GradStore()
    dys = []
    for o in outs:
        dy = torch.randn((o.N, o.T, o.H, o.W, o.C), device="cuda", generator=gen).half()
        R.act_view(gs.of(o)).copy_(dy)
        dys.append(dy)
    grads = training.tape_backward([e], gs, loss_scale)
    ref = R.conv_entry(e, dys, loss_scale)
    assert torch.equal(kernel_dz(e, dys), ref["dz"]), what
    if e["residual"] is not None:                              # fresh store: dres = fp16(0 + masked dy), exact
        assert torch.equal(R.act_view(gs.of(e["residual"])).float(), ref["dres"]), what
    check_params(grads, ref, what)
    if ref["dx"] is not None:
        got = R.act_view(gs.of(e["x"])).double()
        err = (got - ref["dx"]).abs()
        tol = dgrad_tol(ref["dx"], ref["dx_abs"])
        assert bool((err <= tol).all()), (what, "dx", float((err / tol).max()))
        busy = {o.buf.data_ptr() for o in outs} | ({e["residual"].buf.data_ptr()} if e["residual"] is not None else set())
        if e["x"].buf.data_ptr() not in busy:                  # nothing outside x's channel slice is written
            g = gs.of(e["x"]).buf
            rest = torch.ones(g.shape[-1], dtype=torch.bool, device="cuda")
            rest[e["x"].coff:e["x"].coff + e["x"].C] = False
            assert float(g[..., rest].abs().max()) == 0.0 if bool(rest.any()) else True, what


def isolate_pool(e, gen, what):
    from step_b200 import training
    y = e["out"]
    gs = training.GradStore()
    dy = torch.randn((y.N, y.T, y.H, y.W, y.C), device="cuda", generator=gen).half()
    R.act_view(gs.of(y)).copy_(dy)
    assert training.tape_backward([e], gs, 1024.0) == {}
    y_ref, dx_ref = R.pool_entry(e, dy)
    assert torch.equal(R.act_view(y).cpu().double(), y_ref), (what, "forward")
    got = R.act_view(gs.of(e["x"])).cpu().double()
    err = (got - dx_ref).abs()
    assert bool((err <= R.ulp16(dx_ref)).all()), (what, "pool dx", float(err.max()))


@pytest.mark.parametrize("name", ["trunk_shipped", "context_shipped", "head_T3", "head_T9", "cls_head", "trunk_odd", "context_odd"])
def test_every_tape_entry_in_isolation(tapes, name):
    """Each conv / pool entry of the tape alone: its forward output against conv_fwd / the pool reference, then a fresh
    GradStore seeded with a random fp16 output gradient, tape_backward([entry]), and dz, dres, dW / db, dx against the
    float64 reference."""
    tape = tapes[name]
    kind = name.rsplit("_", 1)[0] if name.startswith(("trunk", "context")) else ("cls_head" if name == "cls_head" else "head")
    assert counts(tape) == COUNTS[kind], (name, counts(tape))
    gen = torch.Generator(device="cuda").manual_seed(len(name))
    for i, e in enumerate(tape):
        what = (name, i, e["k"], e["x"].C, tuple(e["x"].buf.shape[1:4]))
        if e["kind"] == "pool":
            isolate_pool(e, gen, what)
        else:
            isolate_conv(e, gen, 1024.0, what)
        torch.cuda.synchronize()


@pytest.fixture(scope="module")
def chain():
    """One train_step in the shipped configuration (2 clips of 36x66x82: odd H and W at every strided pool; context on;
    steps of 3, 3 and 9 frames) with tape_backward wrapped so that each call's tape, GradStore, the gradients seeded
    before it and its parameter gradients are kept: three heads, then ContextNet, then the trunk."""
    from step_b200 import training
    cfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(66, 82))
    nets_ = device_nets(cfg, [synth.head_state_dict(100 + i, cfg) for i in range(3)], context=True)
    x = synth.make_clips(2, 36, 66, 82, seed=13).cuda()
    st, tg = synth.make_train_case(cfg, 2, 3, 82, 66, seed=5)
    calls, orig = [], training.tape_backward

    def spy(tape, grads, loss_scale=1.0, need_input_grad=None):
        seeds = {k: v.clone() for k, v in grads.bufs.items()}
        out = orig(tape, grads, loss_scale, need_input_grad)
        calls.append(dict(tape=list(tape), grads=grads, seeds=seeds, loss_scale=loss_scale, out=out))
        return out
    training.tape_backward = spy
    try:
        training.train_step(cfg, nets_, x, [t.cuda() for t in st], [t.cuda() for t in tg], lr=None, loss_scale=1024.0)
    finally:
        training.tape_backward = orig
    torch.cuda.synchronize()
    return calls


def check_chain(call, what):
    """Every entry's dW / db from its output's final gradient, and every activation's final gradient as its seed plus the
    reference contributions of all its consumers (convolution input gradients, pool backward, residual gradients)."""
    grads, seeds = call["grads"], call["seeds"]
    acc = {}

    def slot(a):
        key = a.buf.data_ptr()
        g = grads.bufs[key]
        if key not in acc:
            acc[key] = {k: torch.zeros(g.shape, dtype=torch.float64, device="cuda") for k in ("ref", "bound", "mag", "n")}
        return {k: v.view(a.buf.shape)[..., a.coff:a.coff + a.C] for k, v in acc[key].items()}

    def add(a, val, margin=None):
        s = slot(a)
        s["ref"] += val
        s["mag"] += val.abs()
        s["n"] += 1
        if margin is not None:
            s["bound"] += margin

    n_conv = n_pool = 0
    for i, e in enumerate(call["tape"]):
        if e["kind"] == "pool":
            dy = R.act_view(grads.of(e["out"]))
            _, dx = R.pool_entry(e, dy)
            add(e["x"], dx.cuda())
            n_pool += 1
            continue
        dys = [R.act_view(grads.of(o)) for o in [e["out"]] + e["extra_outs"]]
        ref = R.conv_entry(e, dys, call["loss_scale"])
        for w, dW, bW, bias, db, bdb in ref["params"]:
            if w.requires_grad:
                check_wgrad(call["out"][w], dW, bW, (what, i, "weight"))
            if bias is not None and bias.requires_grad:
                check_wgrad(call["out"][bias], db, bdb, (what, i, "bias"))
        if ref["dres"] is not None:
            add(e["residual"], ref["dres"].double())
        if ref["dx"] is not None:
            add(e["x"], ref["dx"], U12 * ref["dx_abs"])
        n_conv += 1
    for key, s in acc.items():
        seed = seeds[key].double() if key in seeds else torch.zeros_like(s["ref"])
        ref = seed + s["ref"]
        tol = s["bound"] + s["n"] * R.ulp16(seed.abs() + s["mag"] + s["bound"])
        tol = torch.where(s["n"] > 0, tol, torch.zeros_like(tol))            # untouched elements keep their seed exactly
        err = (grads.bufs[key].double() - ref).abs()
        assert bool((err <= tol).all()), (what, tuple(grads.bufs[key].shape), float((err - tol).max()))
    return n_conv, n_pool


def test_chain_of_real_gradients_through_heads_context_and_trunk(chain):
    assert [counts(c["tape"]) for c in chain] == [COUNTS["head"]] * 3 + [COUNTS["context"], COUNTS["trunk"]]
    for i, call in enumerate(chain):
        assert check_chain(call, i) == counts(call["tape"])


# ---- the other backward kernels on their own -----------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(3, 4, 49, 256, 264, 8), (2, 9, 1, 1024, 1024, 0), (5, 2, 3, 24, 40, 16)])
def test_mean_mid_bwd_and_f32_accum_into_channel_slices(shape):
    """mean_mid_bwd: dx[a, b, p, coff + c] = fp16(dx + g[a, p * C + c] * gscale / B), f32_accum_f16:
    dst[m, coff + c] = fp16(dst + src[m, c] * gscale), both on a channel slice (ld > C, coff > 0) of a buffer that already
    holds gradients; every other channel stays as it was.  Exact: both are single fp32 operations then one rounding."""
    from step_b200 import _lib as L
    A, B, P, C, ld, coff = shape
    gen = torch.Generator(device="cuda").manual_seed(A * B + C)
    g = torch.randn(A, P * C, device="cuda", generator=gen)
    dx0 = torch.randn(A, B, P, ld, device="cuda", generator=gen).half()
    dx = dx0.clone()
    L.check(L.lib().step_mean_mid_bwd(L.ptr(g), A, B, P, C, 1024.0, L.c_void_p(dx.data_ptr() + 2 * coff), ld, L.stream()))
    ref = dx0.clone()
    ref[..., coff:coff + C] = (dx0[..., coff:coff + C].float() + (g.view(A, 1, P, C) * 1024.0) / torch.full_like(g, B).view(A, 1, P, C)).half()
    assert torch.equal(dx, ref)
    M = A * B * P
    src = torch.randn(M, C, device="cuda", generator=gen)
    dst0 = torch.randn(M, ld, device="cuda", generator=gen).half()
    dst = dst0.clone()
    L.check(L.lib().step_f32_accum_f16(L.ptr(src), M, C, 256.0, L.c_void_p(dst.data_ptr() + 2 * coff), ld, L.stream()))
    ref = dst0.clone()
    ref[:, coff:coff + C] = (dst0[:, coff:coff + C].float() + src * 256.0).half()
    assert torch.equal(dst, ref)


def test_ctx_grad_reduce_at_clip_boundaries_and_empty_clips():
    """Frame indices exactly at multiples of T_len (the first frame of a clip) and at the last frame of a clip, a clip with
    no tube, and a tube-less call: acc[b, t_start:t_start + T_len] += (sum of the clip's rows, ascending) / T_len, bit for
    bit the same fp32 operation order."""
    from step_b200 import training
    B, T_all, C, T_len, t_start = 4, 9, 1024, 3, 3
    gen = torch.Generator(device="cuda").manual_seed(3)
    frames = [0.0, 3.0, 5.0, 3.0, 9.0, 11.0, 9.0]                # clips 0, 1, 1, 1, 3, 3, 3; clip 2 has none
    R_ = len(frames)
    tubes = torch.rand(R_, T_len, 5, device="cuda", generator=gen)
    tubes[:, 0, 0] = torch.tensor(frames, device="cuda")
    dctx = torch.randn(R_, C, device="cuda", generator=gen)
    acc0 = torch.randn(B, T_all, C, device="cuda", generator=gen)
    acc = training.context_grad_reduce(dctx, tubes, acc0.clone(), t_start)
    ref = acc0.clone()
    for b in range(B):
        s = torch.zeros(C, device="cuda")
        for r in range(R_):
            if int(frames[r] // T_len) == b:
                s = s + dctx[r]
        ref[b, t_start:t_start + T_len] += s / torch.full_like(s, T_len)   # a true division, not torch's reciprocal product
    assert torch.equal(acc, ref)
    assert torch.equal(training.context_grad_reduce(dctx[:0], tubes[:0], acc0.clone(), t_start), acc0)


@pytest.mark.parametrize("shape", [(37, 8, 16), (1000, 264, 272), (64 * 50 + 3, 520, 520), (64, 24, 40)])
def test_colsum_partial_chunks_and_wide_rows(shape):
    """Bias gradients: colsum over M rows (M < 64, M % 64 != 0) of C columns (C > 256: a second CTA column) at a row pitch
    ld > C, against float64 within 2^-12 of the abs sum (chain of <= M / 64 + 64 fp32 additions)."""
    from step_b200 import _lib as L
    M, C, ld = shape
    gen = torch.Generator(device="cuda").manual_seed(M)
    x = torch.randn(M, ld, device="cuda", generator=gen).half()
    out = torch.empty(C, device="cuda")
    ws = torch.empty(64 * C, device="cuda")
    L.check(L.lib().step_colsum_f16(L.ptr(x), ld, M, C, 0.5, L.ptr(out), L.ptr(ws), L.stream()))
    ref = x[:, :C].double().sum(0) * 0.5
    bound = x[:, :C].double().abs().sum(0) * 0.5
    check_wgrad(out, ref, bound, shape)


@pytest.mark.parametrize("shape", [
    (1, 3, 7, 9, 16, 24, (3, 3, 3), (1, 1, 1), 24),
    (2, 1, 13, 11, 48, 112, (1, 3, 3), (0, 1, 1), 120),
    (1, 5, 31, 29, 208, 16, (1, 1, 1), (0, 0, 0), 16),
    (1, 4, 9, 10, 24, 208, (3, 3, 3), (1, 1, 1), 208),
    (2, 9, 13, 13, 112, 48, (3, 3, 3), (1, 1, 1), 48),
    (1, 3, 9, 7, 64, 24, (4, 4, 4), (1, 1, 1), 32),
])
def test_conv_wgrad_thin_channels_partial_chunks_and_taps(shape):
    """step_conv_wgrad_f16 with M not a multiple of 32 or 2048, Cout / Cin of 16, 24, 48, 112, 208, (1,3,3), (3,3,3) and
    the stem's (4,4,4) pad 1 (24 of the s2d buffer's 32 channels), x at a row pitch >= Cin, against float64."""
    from step_b200 import _lib as L
    N, T, H, W, Cout, Cin, k, pad, x_ld = shape
    gen = torch.Generator(device="cuda").manual_seed(Cout * Cin)
    x = torch.randn(N, T, H, W, x_ld, device="cuda", generator=gen).half()
    dz = torch.randn(N, T, H, W, Cout, device="cuda", generator=gen).half()
    taps = k[0] * k[1] * k[2]
    M = N * T * H * W
    dw = torch.empty((Cout, taps, Cin), dtype=torch.float32, device="cuda")
    nbytes = L.lib().step_conv_wgrad_workspace_bytes(M, Cout, Cin, taps)
    ws = torch.empty((nbytes // 4,), dtype=torch.float32, device="cuda")
    L.check(L.lib().step_conv_wgrad_f16(L.ptr(dz), Cout, L.ptr(x), x_ld, N, T, H, W, Cout, Cin, k[0], k[1], k[2], pad[0], pad[1],
                                        pad[2], 1.0 / 64.0, L.ptr(dw), Cin, 0, L.ptr(ws), nbytes, L.stream()))
    xr = R.ncdhw(x[..., :Cin].double())
    w0 = torch.zeros((Cout, Cin) + k, dtype=torch.float64, device="cuda")
    ref, _ = R.conv_grads(xr, w0, R.ncdhw(dz.double()), k, (1, 1, 1), pad, want_dx=False)
    bound, _ = R.conv_grads(xr.abs(), w0, R.ncdhw(dz.double()).abs(), k, (1, 1, 1), pad, want_dx=False)
    to_kernel = lambda t: t.permute(0, 2, 3, 4, 1).reshape(Cout, taps, Cin) / 64.0
    check_wgrad(dw, to_kernel(ref), to_kernel(bound), shape)
