"""GPU: the training step on the fp32 path (cfg.fp16=False: fp32 activations, activation gradients, ROI concat buffer and
packed weights), the reference's default precision.

  * per launch: step_conv_wgrad_f32 (the stride-2 7x7x7 stem with Cin = 4, asymmetric TF-SAME padding, a ragged last
    pixel chunk, Cout / Cin off the 64-wide tile, channel slices) and the fp32 siblings of the fp16 backward entries,
    against float64 on the same fp32 operands;
  * per tape entry: every conv and max-pool entry of the trunk, ContextNet, a full head and a class-only head alone,
    against float64 on the operands it read;
  * against the reference's own fp32 autograd (tests/golden/head_grads.npz, trunk_grads.npz, ctx_temporal_grads.npz,
    cls_grads.npz) and the oracle's torch-CPU autograd for whole tensors;
  * train_step end to end with step_b200.optim.Adam in the shipped and the classification-stage configurations, with
    ROIAlign and ROIPool, against torch.optim.Adam on the oracle's gradients, and bit-identical from run to run.

Bounds.  An fp32 sum of n terms carries at most n u |terms| of rounding (u = 2^-24).  step_conv_wgrad_f32 adds each
output's chunk of pixels with one fmaf chain and the chunk sums in chunk order, then scales once: n = chunk + chunks + 1
(`wgrad_terms`, the kernel's shape-only chunk plan).  The SIMT input gradient is one fmaf chain over taps x Cout.
ReLU masks, BatchNorm scales, the residual gradient and the elementwise accumulations are single fp32 operations and are
compared exactly."""
import math
import os
import sys

import pytest
import torch

from oracle import model as om
from step_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _tape_reference as R  # noqa: E402
import test_oracle_cls  # noqa: E402
import test_oracle_context  # noqa: E402
from _train_case import SHIPPED, device_head, device_nets, rel_l2, trainable  # noqa: E402

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -24
# The bar against the reference's and the oracle's fp32 autograd: relative error of every gradient norm (NORM_TOL) and
# relative L2 error of every gradient tensor (L2_TOL).  A ReLU net's gradient is discontinuous where a ReLU input sits at 0
# or two max-pool candidates tie: a change of a few ulps in the operands (the device sums in another order than the CPU
# oracle) moves such a decision, and every gradient upstream of it by up to ~1e-3.  The oracle shows it on its own: scaling
# its head inputs and weights by (1 + 5e-7 randn) moves its local-branch weight gradients by 8.5e-4 and its feature
# gradient by 2.4e-3, while fp32 against float64 agrees to 7e-7.  So a tensor may miss L2_TOL only when the forward the
# device recorded holds such a decision downstream of it (`near_decisions`: a ReLU input within NEAR of 0 relative to
# |x||w| + |epilogue terms|, or a max-pool window whose two largest values are within NEAR of each other), and then only
# up to CHAIN_L2_TOL / TRAIN_TRUNK_L2_TOL; every other tensor is held to L2_TOL.
# Measured on an H100 (worst case over the module): trunk alone 2.3e-6, head_grads c1 head 6.6e-4, class-only head 3.3e-4,
# context heads 1.4e-3 (the local-branch bottlenecks of head 0), ContextNet's
# conv_feat gradient 3.4e-3, train_step heads 5.9e-3 and trunk 6.8e-3; every tensor above L2_TOL was flagged.  The
# recorded forwards hold up to 171 near decisions per context head, 106 in ContextNet and 406 outside the trunk in one
# train_step; the other tensors meet L2_TOL.
NORM_TOL = 1e-3
L2_TOL = 1e-3
NEAR = 2.0 ** -20
CHAIN_L2_TOL = 1e-2
TRAIN_TRUNK_L2_TOL = 2e-2
WORST = {}


def _note(kind, v):
    WORST[kind] = max(WORST.get(kind, 0.0), v)


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    print("\nfp32 training, worst relative errors:", {k: "%.2e" % v for k, v in sorted(WORST.items())})


def wgrad_terms(M, Cout, cols):
    """Additions on the path of one term of step_conv_wgrad_f32 (its chunk plan: about 2048 CTAs of 64 x 64 tiles, chunks
    of >= 256 pixels in steps of 16): chunk + chunks + 1."""
    tiles = math.ceil(Cout / 64) * math.ceil(cols / 64)
    want = max(1, min(math.ceil(2048 / tiles), math.ceil(M / 256)))
    chunk = math.ceil(math.ceil(M / want) / 16) * 16
    return chunk + math.ceil(M / chunk) + 1


def fp32_cfg(**kw):
    return synth.make_cfg(fp16=False, **kw)


def act_of(t, C=None, coff=0):
    from step_b200.engine import Act
    return Act(t, C, coff)


# ---- step_conv_wgrad_f32 on its own ------------------------------------------------------------------------------------
WGRAD_CASES = {
    # name: N, T, H, W, Cin, x_ld, Cout, k, stride
    "stem_7x7x7_s2_cin4": (1, 10, 22, 18, 4, 4, 64, (7, 7, 7), (2, 2, 2)),
    "asymmetric_pad_k243": (2, 5, 9, 7, 12, 16, 68, (2, 4, 3), (1, 1, 1)),
    "spatial_s2_k133_slices": (2, 3, 13, 11, 36, 40, 20, (1, 3, 3), (1, 2, 2)),
    "1x1_ragged_m": (3, 7, 29, 31, 132, 136, 72, (1, 1, 1), (1, 1, 1)),
    "3x3x3_cin_cout_off_tile": (1, 4, 10, 9, 100, 100, 196, (3, 3, 3), (1, 1, 1)),
}


@pytest.mark.parametrize("name", list(WGRAD_CASES))
def test_conv_wgrad_f32_against_float64(name):
    """dW of one launch against float64 on the same fp32 operands, per element within wgrad_terms u |dz|^T|x|; repeatable
    bit for bit; scale and accumulate."""
    from step_b200 import engine as E, training
    N, T, H, W, Cin, x_ld, Cout, k, stride = WGRAD_CASES[name]
    gen = torch.Generator(device="cuda").manual_seed(len(name))
    pad_lo = tuple(E.same_pad(kk, s)[0] for kk, s in zip(k, stride))
    OT, OH, OW = E.same_out_dims((T, H, W), k, stride)
    xb = torch.randn(N, T, H, W, x_ld, device="cuda", generator=gen)
    x = act_of(xb, Cin, x_ld - Cin)                         # the last Cin channels of the row: a channel slice
    dzb = torch.randn(N, OT, OH, OW, Cout, device="cuda", generator=gen) * 0.1
    dz = act_of(dzb)
    dw = training.conv_wgrad_f32(dz, x, k, stride, pad_lo)
    x64 = R.ncdhw(R.act_view(x).double())
    dz64 = R.ncdhw(dzb.double())
    zero = torch.zeros((Cout, Cin) + k, dtype=torch.float64, device="cuda")
    ref, _ = R.conv_grads(x64, zero, dz64, k, stride, pad_lo, False)
    bound, _ = R.conv_grads(x64.abs(), zero, dz64.abs(), k, stride, pad_lo, False)
    taps = k[0] * k[1] * k[2]
    ref = ref.permute(0, 2, 3, 4, 1).reshape(Cout, taps, Cin)
    bound = bound.permute(0, 2, 3, 4, 1).reshape(Cout, taps, Cin)
    n = wgrad_terms(N * OT * OH * OW, Cout, taps * Cin)
    err = (dw.double() - ref).abs()
    ratio = float((err / (n * U32 * bound).clamp(min=1e-300)).max())
    _note("conv_wgrad_f32 err / bound", ratio)
    assert ratio <= 1.0, (name, ratio)
    assert torch.equal(dw, training.conv_wgrad_f32(dz, x, k, stride, pad_lo)), name
    dw2 = training.conv_wgrad_f32(dz, x, k, stride, pad_lo, scale=0.5, out=dw.clone(), accumulate=True)
    assert torch.equal(dw2, dw + 0.5 * dw), name


def test_fp32_backward_siblings_against_float64():
    """step_act_bwd_f32 (ReLU mask, BatchNorm scale, residual accumulation on channel slices), step_f32_accum_f32 and
    step_mean_mid_bwd_f32 are single fp32 operations per element: exact.  step_colsum_f32 within (M / 64 + 65) u sum|x|."""
    from step_b200 import _lib as L
    gen = torch.Generator(device="cuda").manual_seed(8)
    M, C, ld = 37 * 5, 24, 32
    dy = torch.randn(M, ld, device="cuda", generator=gen)
    y = torch.randn(M, ld, device="cuda", generator=gen).relu_()
    sc = torch.rand(C, device="cuda", generator=gen) + 0.5
    dres = torch.randn(M, ld, device="cuda", generator=gen)
    dres0 = dres.clone()
    dz = torch.full((M, C), float("nan"), device="cuda")
    o = 4                                                   # channel offset of every slice (16 bytes)
    L.check(L.lib().step_act_bwd_f32(L.c_void_p(dy.data_ptr() + 4 * o), ld, L.c_void_p(y.data_ptr() + 4 * o), ld, L.ptr(sc), 1, M, C,
                                     L.ptr(dz), C, L.c_void_p(dres.data_ptr() + 4 * o), ld, L.stream()))
    g = torch.where(y[:, o:o + C] > 0, dy[:, o:o + C], torch.zeros_like(dz))
    assert torch.equal(dz, g * sc)
    want = dres0.clone()
    want[:, o:o + C] += g
    assert torch.equal(dres, want)
    # colsum at a row pitch wider than C, M not a multiple of the 64 row chunks
    Mc, Cc, ldc = 1000, 264, 272
    x = torch.randn(Mc, ldc, device="cuda", generator=gen)
    out = torch.empty(Cc, device="cuda")
    ws = torch.empty(64 * Cc, device="cuda")
    L.check(L.lib().step_colsum_f32(L.ptr(x), ldc, Mc, Cc, 0.5, L.ptr(out), L.ptr(ws), L.stream()))
    ref = x[:, :Cc].double().sum(0) * 0.5
    tol = (math.ceil(Mc / 64) + 65) * U32 * x[:, :Cc].double().abs().sum(0) * 0.5
    assert bool(((out.double() - ref).abs() <= tol).all())
    # mean_mid_bwd / f32_accum into channel slices
    A, B, P, Cm, ldm, coff = 3, 4, 49, 256, 264, 8
    gm = torch.randn(A, P * Cm, device="cuda", generator=gen)
    dx = torch.randn(A, B, P, ldm, device="cuda", generator=gen)
    dx0 = dx.clone()
    L.check(L.lib().step_mean_mid_bwd_f32(L.ptr(gm), A, B, P, Cm, 1024.0, L.c_void_p(dx.data_ptr() + 4 * coff), ldm, L.stream()))
    want = dx0.clone()
    want[..., coff:coff + Cm] = dx0[..., coff:coff + Cm] + (gm.view(A, 1, P, Cm) * 1024.0) / float(B)
    assert torch.equal(dx, want)
    src = torch.randn(A * B * P, Cm, device="cuda", generator=gen)
    dst = torch.randn(A * B * P, ldm, device="cuda", generator=gen)
    dst0 = dst.clone()
    L.check(L.lib().step_f32_accum_f32(L.ptr(src), A * B * P, Cm, 256.0, L.c_void_p(dst.data_ptr() + 4 * coff), ldm, L.stream()))
    want = dst0.clone()
    want[:, coff:coff + Cm] = dst0[:, coff:coff + Cm] + src * 256.0
    assert torch.equal(dst, want)


# ---- every tape entry of the fp32 forward in isolation --------------------------------------------------------------------
def _nets32():
    import step_b200
    cfg = fp32_cfg(**SHIPPED, image_size=(400, 400))
    base = step_b200.BaseNet(cfg)
    base.load_state_dict(synth.base_net_state_dict())
    ctx = step_b200.ContextNet(cfg)
    ctx.load_state_dict(synth.context_net_state_dict())
    head = step_b200.TwoBranchNet(cfg)
    head.load_state_dict(synth.head_state_dict(100, cfg))
    ccfg = fp32_cfg(T=cfg.T, no_context=True)
    cls = step_b200.TwoBranchNet(ccfg, cls_only=True)
    cls.load_state_dict(synth.cls_head_state_dict(101, ccfg))
    out = [m.cuda().eval() for m in (base, ctx, head, cls)]
    for m in out[2:]:
        m.set_device("cuda:0")
    return out


def _record(fn):
    from step_b200 import engine as E
    tape = []
    with E.recording(tape), torch.no_grad():
        fn()
    return tape


def _head_tape(net, R_, T_, seed, ctx=True):
    from step_b200 import _lib as L
    from step_b200.engine import Act
    gen = torch.Generator(device="cuda").manual_seed(seed)
    cat = Act.empty(R_, T_, 7, 7, 832 + net.fc_dim, L.F32, torch.device("cuda"))
    cat.buf.normal_(generator=gen).relu_()
    ctx_mean = torch.randn(R_, 1024, device="cuda", generator=gen) if ctx else None
    return _record(lambda: net.forward_act(cat, ctx_mean, None, want_logits=True, keep={}))


@pytest.fixture(scope="module")
def tapes32():
    """The fp32 tapes: the trunk on a 14x66x82 clip (odd extents at every strided pool) and ContextNet on its output, a
    full head of 3 frames and a class-only head."""
    base, ctx, head, cls = _nets32()
    x = synth.make_clips(1, 14, 66, 82, seed=7).cuda()
    box = {}
    out = {"trunk": _record(lambda: box.__setitem__("feat", base.forward_act(x)))}
    out["context"] = _record(lambda: ctx.forward_act(box["feat"], keep={}))
    out["head"] = _head_tape(head, 4, 3, 1)
    out["cls_head"] = _head_tape(cls, 4, 3, 3, ctx=False)
    return out


def _isolate_conv(e, gen, loss_scale, what):
    from step_b200 import _lib as L, training
    outs = [e["out"]] + e["extra_outs"]
    x, k, stride, pad_lo = e["x"], e["k"], e["stride"], e["pad_lo"]
    gs = training.GradStore()
    dys, gmask, col = [], [], 0
    for o in outs:
        dy = torch.randn((o.N, o.T, o.H, o.W, o.C), device="cuda", generator=gen)
        R.act_view(gs.of(o)).copy_(dy)
        dys.append(dy)
        gmask.append(torch.where(R.act_view(o) > 0, dy, torch.zeros_like(dy)) if e["relu"] else dy)
    strided = stride != (1, 1, 1)
    grads = training.tape_backward([e], gs, loss_scale, need_input_grad=lambda _: not strided)
    # dz exactly as the act_bwd launch forms it: fp32(masked dy * scale)
    sc = e["scale"]
    parts, col = [], 0
    for o, g in zip(outs, gmask):
        parts.append(g * sc[col:col + o.C] if sc is not None else g)
        col += o.C
    dz = torch.cat(parts, -1)
    o0 = outs[0]
    n_total = dz.shape[-1]
    kd = torch.empty_like(dz)
    col = 0
    for o, dy in zip(outs, dys):
        s = sc[col:col + o.C] if sc is not None else None
        L.check(L.lib().step_act_bwd_f32(L.ptr(dy), o.C, L.c_void_p(o.data_ptr()), o.ld, L.ptr(s), 1 if e["relu"] else 0,
                                         o.N * o.T * o.H * o.W, o.C, L.c_void_p(kd.data_ptr() + 4 * col), n_total, None, 0, L.stream()))
        col += o.C
    assert torch.equal(kd, dz), what
    if e["residual"] is not None:                          # fresh store: 0 + masked dy, exact
        assert torch.equal(R.act_view(gs.of(e["residual"])), sum(gmask[1:], gmask[0])), what
    inv = 1.0 / loss_scale
    x64 = R.ncdhw(R.act_view(x).double())
    dz64 = R.ncdhw(dz.double())
    w = R.packed_weight(e["w"], k, x.C).double()
    dW, dx = R.conv_grads(x64, w, dz64, k, stride, pad_lo, not strided)
    bW, bx = R.conv_grads(x64.abs(), w.abs(), dz64.abs(), k, stride, pad_lo, not strided)
    M = o0.N * o0.T * o0.H * o0.W
    taps = k[0] * k[1] * k[2]
    n = wgrad_terms(M, n_total, taps * x.C) + 1             # + the loss-scale multiplication
    checked, row = 0, 0
    for tg, o in zip(R.tags_of(e), outs):
        sl = slice(row, row + o.C)
        row += o.C
        conv = getattr(tg, "conv3d", tg)
        cin = conv.weight.shape[1]
        if conv.weight.requires_grad:
            ref = dW[sl, :cin].reshape(conv.weight.shape) * inv
            tol = n * U32 * bW[sl, :cin].reshape(conv.weight.shape) * inv
            err = (grads[conv.weight].double() - ref).abs()
            r = float((err / tol.clamp(min=1e-300)).max())
            _note("tape wgrad err / bound", r)
            assert r <= 1.0, (what, "weight", r)
            checked += 1
        if conv.bias is not None and conv.bias.requires_grad:
            d = dz64[:, sl]
            ref = d.sum((0, 2, 3, 4)) * inv
            tol = (math.ceil(M / 64) + 66) * U32 * d.abs().sum((0, 2, 3, 4)) * inv
            assert bool(((grads[conv.bias].double() - ref).abs() <= tol).all()), (what, "bias")
            checked += 1
    assert len(grads) == checked, what
    if dx is not None:
        got = R.act_view(gs.of(x)).double()
        tol = (taps * n_total + 1) * U32 * R.ndhwc(bx)
        r = float(((got - R.ndhwc(dx)).abs() / tol.clamp(min=1e-300)).max())
        _note("tape dgrad err / bound", r)
        assert r <= 1.0, (what, "dx", r)


def _isolate_pool(e, gen, what):
    from step_b200 import training
    y = e["out"]
    gs = training.GradStore()
    dy = torch.randn((y.N, y.T, y.H, y.W, y.C), device="cuda", generator=gen)
    R.act_view(gs.of(y)).copy_(dy)
    assert training.tape_backward([e], gs, 1024.0) == {}
    y_ref, dx_ref = R.pool_entry(e, dy)
    _, dx_abs = R.pool_entry(e, dy.abs())
    assert torch.equal(R.act_view(y).cpu().double(), y_ref), (what, "forward")
    got = R.act_view(gs.of(e["x"])).cpu().double()
    taps = e["k"][0] * e["k"][1] * e["k"][2]
    assert bool(((got - dx_ref).abs() <= taps * U32 * dx_abs).all()), (what, "pool dx")


@pytest.mark.parametrize("name", ["trunk", "context", "head", "cls_head"])
def test_every_fp32_tape_entry_in_isolation(tapes32, name):
    """Each conv / pool entry of an fp32 tape alone: a fresh GradStore seeded with a random fp32 output gradient,
    tape_backward([entry]), and dz, dres, dW / db (the stem's from the stride-2 step_conv_wgrad_f32), dx and the pool's dx
    against float64 on the entry's own operands."""
    tape = tapes32[name]
    assert tape and all(e["x"].code == 0 for e in tape)
    if name == "trunk":
        assert tape[0]["stride"] == (2, 2, 2) and tape[0]["k"] == (7, 7, 7) and tape[0]["x"].C == 4
    gen = torch.Generator(device="cuda").manual_seed(len(name))
    for i, e in enumerate(tape):
        what = (name, i, e["k"], e["x"].C, tuple(e["x"].buf.shape[1:4]))
        if e["kind"] == "pool":
            _isolate_pool(e, gen, what)
        else:
            _isolate_conv(e, gen, 1024.0, what)
        torch.cuda.synchronize()


def test_strided_input_gradient_is_refused(tapes32):
    from step_b200 import training
    e = tapes32["trunk"][0]
    with pytest.raises(NotImplementedError, match="strided"):
        training.tape_backward([e], training.GradStore(), 1.0)


# ---- against the reference's fp32 autograd -------------------------------------------------------------------------------
def _entry_shift(e):
    """The fp32 shift a conv entry's forward read: the folded BatchNorm of its Unit3Dpy, or an nn.Conv container's bias."""
    from step_b200 import _lib as L
    parts = []
    for tg, o in zip(R.tags_of(e), [e["out"]] + e["extra_outs"]):
        if hasattr(tg, "packed"):
            parts.append(tg.packed(L.F32)[2])
        else:
            parts.append(tg.bias.detach().float() if tg.bias is not None else None)
    if all(p is None for p in parts):
        return None
    return torch.cat([p if p is not None else torch.zeros(o.C, device="cuda") for p, o in zip(parts, [e["out"]] + e["extra_outs"])])


def near_decisions(tape):
    """Per tape entry, the decisions of the recorded forward that a few ulps of its operands can move: ReLU inputs z with
    |z| <= NEAR (|x||w| + |epilogue terms|) (float64 on the entry's own operands), and max-pool windows whose largest value
    is positive and within NEAR of, but not equal to, the second largest (zero padding and the ceil-mode overhang
    included).  Exact zeros (every product and epilogue term 0) and exact ties are not counted: they are the same values on
    both sides (a ReLU's zeros, one pixel copied into several ROIPool bins, the test's inputs) and decide the same way."""
    import torch.nn.functional as F
    counts = []
    for e in tape:
        if e["kind"] == "pool":
            x = R.ncdhw(R.act_view(e["x"]).double())
            y = e["out"]
            xp = F.pad(x, R._fpad(list(zip(e["pad_lo"], e["pad_hi"]))))
            extra = [(o - 1) * s + kk - d for o, s, kk, d in zip((y.T, y.H, y.W), e["stride"], e["k"], xp.shape[2:])]
            xp = F.pad(xp, (0, max(extra[2], 0), 0, max(extra[1], 0), 0, max(extra[0], 0)), value=float("-inf"))
            for d, (kk, s) in enumerate(zip(e["k"], e["stride"])):
                xp = xp.unfold(2 + d, kk, s)
            top = xp.reshape(xp.shape[:5] + (-1,)).topk(2, dim=-1).values if xp.shape[-1] * xp.shape[-2] * xp.shape[-3] > 1 else None
            gap = None if top is None else top[..., 0] - top[..., 1]
            counts.append(0 if top is None else int(((top[..., 0] > 0) & (gap > 0) & (gap <= NEAR * top[..., 0])).sum()))
            continue
        if not e["relu"]:
            counts.append(0)
            continue
        outs = [e["out"]] + e["extra_outs"]
        o0 = outs[0]
        res = R.act_view(e["residual"]) if e["residual"] is not None else None
        zs, xws, epis = R.conv_fwd(R.act_view(e["x"]), e["w"], e["scale"], _entry_shift(e), res, e["k"], e["stride"], e["pad_lo"],
                                   (o0.T, o0.H, o0.W), False, [o.C for o in outs])
        counts.append(sum(int(((xw + ep > 0) & (z.abs() <= NEAR * (xw + ep))).sum()) for z, xw, ep in zip(zs, xws, epis)))
    return counts


def downstream_flags(tape, counts):
    """{parameter: True when an entry at or after the one that owns it (nearer the loss) holds a near decision}."""
    flags = {}
    for j, e in enumerate(tape):
        if e["kind"] != "conv":
            continue
        for tg in R.tags_of(e):
            conv = getattr(tg, "conv3d", tg)
            for t in (conv.weight, conv.bias):
                if t is not None:
                    flags[t] = sum(counts[j:]) > 0
    return flags


class Recorder:
    """Keeps every tape the training entry points record (engine.recording wrapped)."""

    def __init__(self, monkeypatch):
        from step_b200 import engine as E
        self.tapes, orig = [], E.recording

        def recording(tape):
            if tape is not None:
                self.tapes.append(tape)
            return orig(tape)
        monkeypatch.setattr(E, "recording", recording)


def _check_named(got, ref_norm, ref_grad, kind, flagged=False, cap=CHAIN_L2_TOL):
    """Norm against the reference's golden norm (None: not compared) and the tensor against the oracle's autograd: within
    NORM_TOL / L2_TOL, or, when a near decision lies downstream (flagged), within cap."""
    tol = cap if flagged else L2_TOL
    if ref_norm is not None:
        gn = float(got.double().norm())
        _note(kind + " norm", abs(gn - ref_norm) / ref_norm)
        assert abs(gn - ref_norm) <= max(NORM_TOL, tol if flagged else 0.0) * ref_norm, (kind, gn, ref_norm)
    r = rel_l2(got, ref_grad)
    _note(kind + " L2", r)
    if r > L2_TOL:
        _note(kind + " L2 above L2_TOL, flagged", r)
    assert r <= tol, (kind, r, "flagged" if flagged else "no near decision downstream")


def test_fp32_head_backward_matches_reference_autograd(golden):
    """The whole head (head_grads.npz, case c1) on the fp32 path: the 34 trainable tensors and the pooled features'
    gradient."""
    from step_b200 import training
    g = golden("head_grads")
    T_, chunks, n, _ = synth.LOSS_CASES["c1"]
    cfg = fp32_cfg(T=T_, max_iter=1, NUM_CHUNKS={1: chunks}, image_size=(112, 112))
    _, _, feat, tb, tg = synth.make_loss_case("c1", cfg.num_classes)
    net = device_head(cfg, synth.head_state_dict(100, cfg))
    r = training.head_forward_backward(net, feat.cuda(), tb.cuda(), tg.cuda(), lambda_reg=5.0, lambda_neighbor=1.0, loss_scale=1.0)
    torch.cuda.synchronize()
    assert abs(float(r["loss"]) - float(g["loss"][0])) <= 1e-5 * abs(float(g["loss"][0]))
    sd = trainable(synth.head_state_dict(100, cfg))
    fr = feat.clone().requires_grad_(True)
    prob, loc, first, last, logits = om.two_branch(fr, sd, cfg.T, None, cfg.fc_dim, cfg.pool_size, return_logits=True)
    lc, ll, ln = om.two_branch_losses(logits, loc, first, last, tb, tg, cfg.T)
    (lc.mean() + ll.mean() * 5.0 + ln.mean() * 1.0).backward()
    names = {p: k for k, p in net.named_parameters()}
    got = {names[p]: v for p, v in r["grads"].items()}
    assert len(got) == 34
    for k, v in got.items():
        assert tuple(v.shape) == tuple(sd[k].shape), k
        _check_named(v, float(g["gn:" + k][0]), sd[k].grad, "head")
    _check_named(r["feat_grad"], float(g["feat_grad_norm"][0]), fr.grad, "head feat_grad")


def test_fp32_trunk_backward_matches_reference_autograd(golden):
    """The I3D trunk on the fp32 path (trunk_grads.npz): 45 Unit3D weight gradients, the stem's from the stride-2 7x7x7
    step_conv_wgrad_f32 over the clip padded to 4 channels."""
    import step_b200
    from step_b200 import training
    g = golden("trunk_grads")
    cfg = fp32_cfg(T=2, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(64, 64))
    net = step_b200.BaseNet(cfg)
    net.load_state_dict(synth.base_net_state_dict(), strict=True)
    net = net.cuda().eval()
    x = synth.make_clips(1, 8, 64, 64, seed=4321)
    proj = torch.randn((1, 2, 832, 4, 4), generator=torch.Generator().manual_seed(99))
    numel = proj.numel()
    feat, grads = training.trunk_forward_backward(net, x.cuda(), lambda f: (proj / numel).permute(0, 1, 3, 4, 2).contiguous().cuda(),
                                                  loss_scale=1.0)
    torch.cuda.synchronize()
    sd = {k: v.clone().requires_grad_(k.endswith("conv3d.weight")) for k, v in synth.base_net_state_dict().items()}
    cf = om.base_net(x.clone(), sd)
    ((cf * proj).sum() / cf.numel()).backward()
    names = {p: k for k, p in net.named_parameters()}
    got = {names[p]: v for p, v in grads.items()}
    checked = 0
    for key in g.files:
        if not key.startswith("gn:"):
            continue
        k = key[3:]
        assert tuple(got[k].shape) == tuple(sd[k].grad.shape), k
        _check_named(got[k], float(g[key][0]), sd[k].grad, "trunk")
        checked += 1
    assert checked == 45 and len(got) == 45


def test_fp32_context_heads_and_context_net_match_reference_autograd(golden, monkeypatch):
    """ctx_temporal_grads.npz on the fp32 path: the three heads of the shipped configuration with the per-tube context
    feature (34 tensors each, the pooled features' and the context input's gradient), then ContextNet's backward from the
    oracle's d(loss)/d(context) (12 tensors and the context branch's gradient of conv_feat)."""
    import step_b200
    from step_b200 import _lib as L, training
    from step_b200.networks import to_act
    g = golden("ctx_temporal_grads")
    cfg, cf, step_tubes, step_targets = test_oracle_context.golden_case()
    cf = cf.requires_grad_(True)
    sd_ctx = trainable(synth.context_net_state_dict())
    sds = [trainable(synth.head_state_dict(100 + i, cfg)) for i in range(3)]
    loss, pooled, ctx = test_oracle_context.oracle_objective(cf, sd_ctx, sds, cfg, step_tubes, step_targets, pooled_leaves=True)
    ctx.retain_grad()
    loss.backward()
    dcfg = fp32_cfg(**SHIPPED, image_size=(400, 400))
    rec = Recorder(monkeypatch)
    for i in range(3):
        t0, tl = training.step_frames(cfg, i + 1)
        flat = step_tubes[i]
        clip = [int(flat[p, 0, 0].item() / tl) for p in range(flat.shape[0])]
        tctx = torch.stack([ctx.detach()[c, :, t0:t0 + tl] for c in clip]).requires_grad_(True)
        pl = pooled[i].detach().clone().requires_grad_(True)
        sd = trainable(synth.head_state_dict(100 + i, cfg))
        _, loc, first, last, logits = om.two_branch(pl, sd, cfg.T, tctx, cfg.fc_dim, cfg.pool_size, return_logits=True)
        lc, ll, ln = om.two_branch_losses(logits, loc, first, last, flat, step_targets[i], cfg.T)
        (lc.mean() + 5.0 * ll.mean() + 1.0 * ln.mean()).backward()
        net = device_head(dcfg, synth.head_state_dict(100 + i, dcfg))
        r = training.head_forward_backward(net, pooled[i].detach().cuda(), flat.cuda(), step_targets[i].cuda(),
                                           context_feat=tctx.detach().cuda(), loss_scale=1.0)
        torch.cuda.synchronize()
        tape = rec.tapes[-1]
        counts = near_decisions(tape)
        flags = downstream_flags(tape, counts)
        _note("context heads near decisions", sum(counts))
        names = {p: k for k, p in net.named_parameters()}
        got = {names[p]: v for p, v in r["grads"].items()}
        assert len(got) == 34
        for p, v in r["grads"].items():
            k = names[p]
            _check_named(v, float(g["gn:h%d:%s" % (i, k)][0]), sd[k].grad, "context heads", flags.get(p, False))
        _check_named(r["feat_grad"], float(g["pooled_grad_norm%d" % (i + 1)][0]), pl.grad, "context heads feat_grad", sum(counts) > 0)
        r_ctx = rel_l2(r["ctx_grad"], tctx.grad)
        _note("context heads ctx_grad L2", r_ctx)
        assert r_ctx <= L2_TOL, r_ctx
    net = step_b200.ContextNet(dcfg)
    net.load_state_dict(synth.context_net_state_dict(), strict=True)
    net = net.cuda().eval()
    feat = to_act(cf.detach().cuda(), L.F32)
    c, state = training.context_forward(net, feat)
    d_ctx = ctx.grad.view(2, 1024, 9).permute(0, 2, 1).contiguous().cuda()
    grads, gfeat = training.context_backward(state, d_ctx, 1.0)
    torch.cuda.synchronize()
    counts = near_decisions(state["tape"])
    flags = downstream_flags(state["tape"], counts)
    _note("context_net near decisions", sum(counts))
    names = {p: k for k, p in net.named_parameters()}
    assert len(grads) == 12
    for p, v in grads.items():
        _check_named(v, float(g["gn:ctx:" + names[p]][0]), sd_ctx[names[p]].grad, "context_net", flags[p])
    _check_named(gfeat.permute(0, 1, 4, 2, 3), float(g["ctx_feat_grad_norm"][0]), cf.grad, "context_net feat_grad", sum(counts) > 0)


def test_fp32_cls_head_backward_matches_reference_autograd(golden):
    """cls_grads.npz on the fp32 path: a class-only head with the context as train_step feeds it (per-clip mean and row
    map): 16 tensors and the pooled features' gradient."""
    from step_b200 import training
    g = golden("cls_grads")
    cfg, cf, flat_tubes, flat_targets = test_oracle_cls.golden_case()
    ctx = om.context_net(cf, synth.context_net_state_dict(), global_mean=True).detach()
    clip = [int(flat_tubes[p, 0, 0].item() / cfg.T) for p in range(flat_tubes.shape[0])]
    tctx = torch.stack([ctx[c, :, :cfg.T] for c in clip])
    _, _, pooled, _, _ = test_oracle_cls.cls_objective(cf, synth.context_net_state_dict(), synth.cls_head_state_dict(100, cfg), cfg,
                                                       flat_tubes, flat_targets, pooled_leaf=True)
    pooled = pooled.detach().requires_grad_(True)
    sd = trainable(synth.cls_head_state_dict(100, cfg))
    prob, loc, first, last, logits = om.two_branch(pooled, sd, cfg.T, tctx, cfg.fc_dim, cfg.pool_size, cls_only=True, return_logits=True)
    lc, _, _ = om.two_branch_losses(logits, loc, first, last, flat_tubes, flat_targets, cfg.T, cls_only=True)
    lc.mean().backward()
    dcfg = fp32_cfg(**test_oracle_cls.CLS_CFG, image_size=(400, 400))
    net = device_head(dcfg, synth.cls_head_state_dict(100, dcfg), cls_only=True)
    context = (ctx.view(2, 1024, 9).mean(2).cuda(), torch.tensor(clip, dtype=torch.int32, device="cuda"))
    r = training.head_forward_backward(net, pooled.detach().cuda(), flat_tubes.cuda(), flat_targets.cuda(), context_feat=context,
                                       loss_scale=1.0)
    torch.cuda.synchronize()
    assert abs(float(r["loss"]) - float(g["loss"][0])) <= 1e-5 * float(g["loss"][0])
    names = {p: k for k, p in net.named_parameters()}
    got = {names[p]: v for p, v in r["grads"].items()}
    assert len(got) == 16
    for k, v in got.items():
        _check_named(v, float(g["gn:h0:" + k][0]), sd[k].grad, "cls head")
    _check_named(r["feat_grad"], float(g["pooled_grad_norm"][0]), pooled.grad, "cls head feat_grad")


# ---- train_step end to end with Adam ------------------------------------------------------------------------------------
def _case(stage, pool_mode):
    """(cfg, clips, step_tubes, step_targets, nets, {module: oracle state dict}, oracle objective) at 2 clips of 36x64x64."""
    cls = stage == "cls"
    if cls:
        cfg = fp32_cfg(**test_oracle_cls.CLS_CFG, image_size=(64, 64))
        tubes, targets = synth.make_cls_case(cfg, 2, 6, 64, 64, seed=3)
        step_tubes, step_targets = [tubes], [targets]
        heads = [synth.cls_head_state_dict(100, cfg)]
    else:
        cfg = fp32_cfg(**SHIPPED, image_size=(64, 64))
        step_tubes, step_targets = synth.make_train_case(cfg, 2, 3, 64, 64, seed=3)
        heads = [synth.head_state_dict(100 + i, cfg) for i in range(3)]
    x = synth.make_clips(2, 36, 64, 64, seed=11)
    nets = device_nets(cfg, heads, pool_mode, context=True, cls_only=cls)
    return cfg, x, step_tubes, step_targets, nets, heads


def _oracle(stage, cfg, x, step_tubes, step_targets, heads, monkeypatch, pool_mode):
    if pool_mode == "pool":
        import test_gpu_train_pool
        monkeypatch.setattr(test_oracle_cls if stage == "cls" else test_oracle_context, "tv_roi_align", test_gpu_train_pool.pool_as_align)
    sd_b = {k: v.clone().requires_grad_(k.endswith("conv3d.weight")) for k, v in synth.base_net_state_dict().items()}
    sd_ctx = trainable(synth.context_net_state_dict())
    sds = [trainable(sd) for sd in heads]
    cf = om.base_net(x.clone(), sd_b)
    if stage == "cls":
        total = test_oracle_cls.cls_objective(cf, sd_ctx, sds[0], cfg, step_tubes[0], step_targets[0])[0]
    else:
        total = test_oracle_context.oracle_objective(cf, sd_ctx, sds, cfg, step_tubes, step_targets)[0]
    total.backward()
    mods = {"base_net": sd_b, "context_net": sd_ctx}
    mods.update({"det_net%d" % i: sd for i, sd in enumerate(sds)})
    return float(total.detach()), mods


LR, WD = 1e-4, 1e-4


@pytest.mark.parametrize("stage", ["shipped", "cls"])
@pytest.mark.parametrize("pool_mode", ["align", "pool"])
def test_fp32_train_step_with_adam_matches_oracle_and_repeats(stage, pool_mode, monkeypatch):
    """train_step(..., optimizer=step_b200.optim.Adam(...)) with loss_scale=1.0 -- the reference's fp32 arithmetic -- against
    the oracle's torch-CPU autograd: every gradient within L2_TOL unless a near decision of the recorded forwards lies
    downstream of it (a head's own tape for its tensors, ContextNet's for its own; any tape, and with ROIPool the argmax
    of every bin, for the trunk's, which receive the sum of the heads' and ContextNet's conv_feat gradients).  The update
    is bit-identical to torch.optim.Adam(foreach=False) run on the device's gradients, and a second run from the same
    parameters gives the same gradients and parameters bit for bit."""
    from step_b200 import optim, training
    cfg, x, step_tubes, step_targets, nets, heads = _case(stage, pool_mode)
    total, mods = _oracle(stage, cfg, x, step_tubes, step_targets, heads, monkeypatch, pool_mode)
    named = [(m, k, p) for m in nets if m != "roi_net" for k, p in nets[m].named_parameters() if p.requires_grad]
    init = {(m, k): p.detach().clone() for m, k, p in named}

    rec = Recorder(monkeypatch)

    def run():
        with torch.no_grad():
            for m, k, p in named:
                p.copy_(init[(m, k)])
        opt = optim.Adam([p for _, _, p in named], lr=LR, weight_decay=WD)
        r = training.train_step(cfg, nets, x.cuda(), [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets],
                                loss_scale=1.0, optimizer=opt)
        torch.cuda.synchronize()
        return r, {(m, k): p.detach().clone() for m, k, p in named}
    r, after = run()
    assert not r["skipped"]
    assert abs(float(r["loss"]) - total) <= 1e-4 * abs(total)
    # near decisions of every recorded forward (trunk, ContextNet, heads), and the tensors downstream of them
    flags, trunk_tape, others = {}, None, 0
    base_params = set(nets["base_net"].parameters())
    for tape in rec.tapes:
        counts = near_decisions(tape)
        f = downstream_flags(tape, counts)
        flags.update(f)
        if any(p in base_params for p in f):
            trunk_tape = (f, counts)
        else:
            others += sum(counts)
    _note("train_step near decisions outside the trunk", others)
    upstream = others > 0 or pool_mode == "pool"
    n = 0
    for m in mods:
        params = dict(nets[m].named_parameters())
        for k, sdv in mods[m].items():
            if sdv.grad is None:
                continue
            p = params[k]
            trunk = m == "base_net"
            _check_named(r["grads"][p], None, sdv.grad, "train_step %s %s" % (stage, m.rstrip("012")),
                         flags.get(p, False) or (trunk and upstream), TRAIN_TRUNK_L2_TOL if trunk else CHAIN_L2_TOL)
            n += 1
    assert trunk_tape is not None and n == len(named) == len(r["grads"])
    # the update: torch.optim.Adam on the device's own gradients, bit for bit
    ref_p = [init[(m, k)].clone().requires_grad_(True) for m, k, _ in named]
    for q, (_, _, p) in zip(ref_p, named):
        q.grad = r["grads"][p].detach().clone()
    torch.optim.Adam(ref_p, lr=LR, weight_decay=WD, foreach=False).step()
    for q, (m, k, _) in zip(ref_p, named):
        assert torch.equal(after[(m, k)], q.detach()), (m, k)
    # bit-identical from run to run
    rec.tapes.clear()
    r2, after2 = run()
    assert all(torch.equal(after[key], after2[key]) for key in after)
    assert all(torch.equal(r["grads"][p], r2["grads"][p]) for _, _, p in named)
