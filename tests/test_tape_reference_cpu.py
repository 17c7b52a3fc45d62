"""CPU: the float64 tape reference of tests/_tape_reference.py pinned to the modules' meaning on small shapes, and the
argument checks of the backward entry points (step_act_bwd_f16, step_conv_wgrad_f16, step_maxpool3d_bwd_f16).

The reference rounds dz = dy * [y > 0] * scale to fp16 as act_bwd_kernel does; autograd of the module keeps it exact.
That rounding moves each dz by at most half an fp16 ulp, 2^-11 |dz|, so a weight or input gradient moves by at most
2^-11 (|dz|^T |x|) or 2^-11 (|dz| * |w|): the bound every comparison below uses.  Everything else is float64."""
import ctypes
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _tape_reference as R  # noqa: E402

from step_b200 import _lib as L  # noqa: E402
from step_b200 import engine as E  # noqa: E402
from step_b200.engine import Act  # noqa: E402

HALF_ULP = 2.0 ** -11


def half_values(*shape, gen, scale=1.0):
    return (torch.randn(*shape, generator=gen) * scale).half()


def same_pads(dims, k, s):
    lo = tuple(E.same_pad(kk, ss)[0] for kk, ss in zip(k, s))
    hi = tuple(E.same_pad(kk, ss)[1] for kk, ss in zip(k, s))
    return lo, hi


def fpad(lo, hi):
    return (lo[2], hi[2], lo[1], hi[1], lo[0], hi[0])


def entry(x, w_packed, scale, out, k, pad_lo, relu, residual=None, tag=None):
    return dict(kind="conv", x=x, w=w_packed, scale=scale, out=out, extra_outs=[], k=tuple(k), stride=(1, 1, 1),
                pad_lo=tuple(pad_lo), relu=relu, residual=residual, tag=tag)


def within(got, ref, bound, factor=HALF_ULP, slack=1e-12):
    err = (got.double() - ref.double()).abs()
    lim = factor * bound.double() + slack
    assert bool((err <= lim).all()), float((err - lim).max())


def test_unit3d_with_folded_bn_relu_and_same_padding():
    """Unit3Dpy(8 -> 16, 3x3x3, SAME, BatchNorm eval, ReLU): dW and dx of the reference against autograd of
    relu(batch_norm(conv3d(pad(x), w))) in float64 on the same fp16 x / w."""
    from step_b200.i3d import Unit3Dpy
    gen = torch.Generator().manual_seed(1)
    u = Unit3Dpy(8, 16, kernel_size=(3, 3, 3)).eval()
    with torch.no_grad():
        u.conv3d.weight.copy_(torch.randn(u.conv3d.weight.shape, generator=gen) * 0.2)
        u.batch3d.weight.copy_(torch.rand(16, generator=gen) + 0.5)
        u.batch3d.bias.copy_(torch.randn(16, generator=gen) * 0.2)
        u.batch3d.running_mean.copy_(torch.randn(16, generator=gen) * 0.1)
        u.batch3d.running_var.copy_(torch.rand(16, generator=gen) + 0.5)
    N, T, H, W = 2, 3, 5, 6
    x16 = half_values(N, T, H, W, 8, gen=gen)
    w_packed, scale, shift = u.packed(L.F16)
    k = (3, 3, 3)
    lo, hi = same_pads((T, H, W), k, (1, 1, 1))
    # the module's meaning in float64
    xr = R.ncdhw(x16.double()).requires_grad_(True)
    wr = u.conv3d.weight.detach().half().double().requires_grad_(True)
    bn = u.batch3d
    z = F.conv3d(F.pad(xr, fpad(lo, hi)), wr)
    y = torch.relu(F.batch_norm(z, bn.running_mean.double(), bn.running_var.double(), bn.weight.double(), bn.bias.double(),
                                False, 0.0, bn.eps))
    dy16 = half_values(N, T, H, W, 16, gen=gen)
    y.backward(R.ncdhw(dy16.double()))
    y16 = R.ndhwc(y.detach()).half().contiguous()
    e = entry(Act(x16.contiguous()), w_packed, scale, Act(y16), k, lo, True, tag=u)
    r = R.conv_entry(e, [dy16], loss_scale=1.0)
    (p, dW, bW, _, db, _), = r["params"]
    assert p is u.conv3d.weight and db is None
    within(dW, wr.grad, bW)
    within(r["dx"], R.ndhwc(xr.grad), r["dx_abs"])
    # the same with a loss scale: every parameter gradient is divided by it
    r2 = R.conv_entry(e, [dy16], loss_scale=1024.0)
    assert torch.equal(r2["params"][0][1] * 1024.0, dW)
    # dz is the fp16 rounding of dy * [y > 0] * scale, and zero wherever the ReLU was off
    assert torch.equal(r["dz"], (dy16.float() * (y16.float() > 0) * scale).half())


def test_bottleneck_resample_residual_path_and_biased_downsample():
    """A head Bottleneck_resample (two_branch.py:86-111): conv1 has no ReLU and feeds conv4's residual input; conv4 adds it
    before its ReLU.  The reference's dres of the conv4 entry, fed to the conv1 entry as its output gradient, gives
    conv1's dW and its share of dx; against autograd of the block.  Then the biased 1x1x1 `downsample` (no activation)."""
    from step_b200.two_branch import Bottleneck_resample
    gen = torch.Generator().manual_seed(2)
    blk = Bottleneck_resample(16, 32, 8)
    for m in (blk.conv1, blk.conv2, blk.conv3, blk.conv4):
        with torch.no_grad():
            m.weight.copy_(torch.randn(m.weight.shape, generator=gen) * 0.3)
    Fr, P = 3, 5
    x16 = half_values(Fr, 1, P, P, 16, gen=gen)
    w = {n: getattr(blk, n).weight.detach().half().double().requires_grad_(True) for n in ("conv1", "conv2", "conv3", "conv4")}
    xr = R.ncdhw(x16.double())[:, :, 0].requires_grad_(True)               # frames as 2-D images [F, C, 5, 5]
    res = F.conv2d(xr, w["conv1"])
    res.retain_grad()
    o2 = torch.relu(F.conv2d(xr, w["conv2"]))
    o3 = torch.relu(F.conv2d(o2, w["conv3"], padding=1))
    out = torch.relu(F.conv2d(o3, w["conv4"]) + res)
    dy16 = half_values(Fr, 1, P, P, 32, gen=gen)
    out.backward(R.ncdhw(dy16.double())[:, :, 0], retain_graph=True)
    to_act = lambda t: Act(R.ndhwc(t.detach().unsqueeze(2)).half().contiguous())
    res_a, o3_a, out_a = to_act(res), to_act(o3), to_act(out)
    e4 = entry(o3_a, E.pack_conv_weight(blk.conv4.weight, L.F16), None, out_a, (1, 1, 1), (0, 0, 0), True, residual=res_a,
               tag=blk.conv4)
    r4 = R.conv_entry(e4, [dy16])
    (p4, dW4, bW4, _, _, _), = r4["params"]
    assert p4 is blk.conv4.weight
    within(dW4, w["conv4"].grad, bW4)
    # the residual gradient is dy masked by the block's ReLU, exactly
    assert torch.equal(r4["dres"].double(), R.ndhwc(res.grad.unsqueeze(2)))
    e1 = entry(Act(x16.contiguous()), E.pack_conv_weight(blk.conv1.weight, L.F16), None, res_a, (1, 1, 1), (0, 0, 0), False,
               tag=blk.conv1)
    r1 = R.conv_entry(e1, [r4["dres"].half()])
    (p1, dW1, bW1, _, _, _), = r1["params"]
    assert p1 is blk.conv1.weight
    within(dW1, w["conv1"].grad, bW1, slack=1e-10)
    # conv1's input-gradient contribution: autograd of res alone
    (gx1,) = torch.autograd.grad(res, xr, res.grad)
    within(r1["dx"][:, 0], R.ndhwc(gx1.unsqueeze(2))[:, 0], r1["dx_abs"][:, 0], slack=1e-10)
    # downsample: 1x1x1 Conv3d with bias, no activation
    ds = torch.nn.Conv3d(16, 24, 1, bias=True)
    wd = ds.weight.detach().half().double().requires_grad_(True)
    bd = ds.bias.detach().double().requires_grad_(True)
    g16 = half_values(2, 3, 4, 4, 16, gen=gen)
    yd = F.conv3d(R.ncdhw(g16.double()), wd, bd)
    dyd = half_values(2, 3, 4, 4, 24, gen=gen)
    yd.backward(R.ncdhw(dyd.double()))
    ed = entry(Act(g16.contiguous()), E.pack_conv_weight(ds.weight, L.F16), None, Act(R.ndhwc(yd.detach()).half().contiguous()),
               (1, 1, 1), (0, 0, 0), False, tag=ds)
    (_, dWd, bWd, bias, db, bdb), = R.conv_entry(ed, [dyd], loss_scale=4.0)["params"]
    assert bias is ds.bias
    within(dWd * 4.0, wd.grad, bWd * 4.0)
    within(db * 4.0, bd.grad, bdb * 4.0)


def s2d_pack(clip):
    """clip [N, C, T, H, W] -> [N, T/2, H/2, W/2, 32]: channel ((rt * 2 + rh) * 2 + rw) * C + c holds
    clip[2 t2 + rt, 2 h2 + rh, 2 w2 + rw] (written out here index by index, independently of R.unpack_s2d)."""
    N, C, T, H, W = clip.shape
    out = torch.zeros(N, T // 2, H // 2, W // 2, 32, dtype=clip.dtype)
    for rt in range(2):
        for rh in range(2):
            for rw in range(2):
                for c in range(C):
                    out[..., ((rt * 2 + rh) * 2 + rw) * C + c] = clip[:, c, rt::2, rh::2, rw::2]
    return out


def test_stem_s2d_packing_and_wgrad_unpack_match_the_strided_convolution():
    """The stem (Unit3Dpy 3 -> 64, 7x7x7, stride 2, SAME) runs as a 4x4x4 stride-1 convolution with pad 1 over the
    space-to-depth clip with engine.pack_stem_s2d's filter.  Checks, in float64 on the same fp16 values: that forward
    equals the strided convolution of the clip; training.stem_s2d_wgrad applied to the 4x4x4 weight gradient equals
    autograd's 7x7x7 one; and the reference's s2d entry gives that gradient too."""
    from step_b200 import training
    from step_b200.i3d import Unit3Dpy
    gen = torch.Generator().manual_seed(3)
    u = Unit3Dpy(3, 64, kernel_size=(7, 7, 7), stride=(2, 2, 2))
    with torch.no_grad():
        u.conv3d.weight.copy_(torch.randn(u.conv3d.weight.shape, generator=gen) * 0.05)
    N, T, H, W = 1, 6, 10, 8
    clip = torch.randn(N, 3, T, H, W, generator=gen).half().double()
    w7 = u.conv3d.weight.detach().half().double().requires_grad_(True)
    y = F.conv3d(F.pad(clip, (2, 3, 2, 3, 2, 3)), w7, stride=2)                   # same_pad(7, 2) = (2, 3)
    assert tuple(y.shape[2:]) == (T // 2, H // 2, W // 2)
    xs = s2d_pack(clip)
    assert torch.equal(R.unpack_s2d(xs, 3), clip)
    w4 = E.pack_stem_s2d(u.conv3d.weight).double()                              # [64, 64 taps, 32]
    w4_5d = w4.reshape(64, 4, 4, 4, 32).permute(0, 4, 1, 2, 3)
    y4 = F.conv3d(F.pad(R.ncdhw(xs), (1, 2, 1, 2, 1, 2)), w4_5d)
    assert float((y4 - y).abs().max()) <= 1e-12 * float(y.abs().max())
    dz16 = torch.randn(y.shape, generator=gen).half()
    y.backward(dz16.double())
    # the 4x4x4 weight gradient in the kernel's [Cout, taps, 32] layout, unpacked as tape_backward does
    dW4, _ = R.conv_grads(R.ncdhw(xs), w4_5d, dz16.double(), (4, 4, 4), (1, 1, 1), (1, 1, 1), want_dx=False)
    g7 = training.stem_s2d_wgrad(dW4.permute(0, 2, 3, 4, 1).reshape(64, 64, 32), 3)
    assert float((g7 - w7.grad).abs().max()) <= 1e-12 * float(w7.grad.abs().max())
    # the reference's stem entry: the same gradient from the s2d activations, divided by the loss scale
    y16 = R.ndhwc(y.detach()).half().contiguous()
    e = dict(kind="conv", x=Act(xs.half().contiguous(), 24, 0), w=E.pack_stem_s2d(u.conv3d.weight), scale=None,
             out=Act(y16), extra_outs=[], k=(4, 4, 4), stride=(1, 1, 1), pad_lo=(1, 1, 1), relu=False, residual=None,
             tag=("s2d", u))
    r = R.conv_entry(e, [R.ndhwc(dz16)], loss_scale=2.0)
    (p, dW, bW, _, _, _), = r["params"]
    assert p is u.conv3d.weight and r["dx"] is None
    assert float((dW * 2.0 - w7.grad).abs().max()) <= 1e-12 * float(w7.grad.abs().max())
    assert bool((dW.abs() <= bW + 1e-15).all())


def first_max_pool_bwd(x, k, s, lo, hi, out_dims, dy):
    """Max-pool backward by the rule the kernel implements, written as loops: the window's positions in (kt, kh, kw)
    order; positions in the zero padding hold 0 and take part, positions past it do not exist; the first strict maximum
    wins and a win by padding drops the gradient.  x [T, H, W] float64, dy [OT, OH, OW]."""
    T, H, W = x.shape
    dx = torch.zeros_like(x)
    for ot in range(out_dims[0]):
        for oh in range(out_dims[1]):
            for ow in range(out_dims[2]):
                best, arg = None, None
                for kt in range(k[0]):
                    for kh in range(k[1]):
                        for kw in range(k[2]):
                            p = (ot * s[0] + kt - lo[0], oh * s[1] + kh - lo[1], ow * s[2] + kw - lo[2])
                            dims = (T, H, W)
                            if any(q < -l or q >= d + h for q, l, d, h in zip(p, lo, dims, hi)):
                                continue
                            real = all(0 <= q < d for q, d in zip(p, dims))
                            v = float(x[p]) if real else 0.0
                            if best is None or v > best:
                                best, arg = v, (p if real else None)
                if arg is not None:
                    dx[arg] += float(dy[ot, oh, ow])
    return dx


@pytest.mark.parametrize("geom", [((1, 3, 3), (1, 2, 2), (2, 7, 9)), ((3, 3, 3), (2, 2, 2), (7, 5, 9)),
                                  ((1, 3, 3), (1, 2, 2), (1, 25, 25)), ((3, 3, 3), (1, 1, 1), (3, 4, 5))])
def test_pool_reference_ties_and_asymmetric_padding(geom):
    """R.pool_entry (ATen: zero F.pad + max_pool3d(ceil_mode=True)) against the loop rule above on values drawn from
    {-1, 0, 1} after a ReLU-like clamp: almost every window holds ties, among themselves and with the padding.
    Geometries: the trunk's (1,3,3)/(1,2,2) and (3,3,3)/(2,2,2) on odd extents, ContextNet's 25 -> 13 with its ceil-mode
    overhang, and the stride-1 branch-3 pool."""
    k, s, dims = geom
    gen = torch.Generator().manual_seed(sum(dims))
    C = 2
    x16 = torch.randint(-1, 2, (1,) + dims + (C,), generator=gen).clamp_(min=0).half()
    x16[..., 1] = torch.randint(-1, 2, (1,) + dims, generator=gen).half()          # channel 1 keeps negatives
    lo, hi, od = [], [], []
    for d, kk, ss in zip(dims, k, s):
        o, l_, h_ = E.pool_out(d, kk, ss)
        od.append(o); lo.append(l_); hi.append(h_)
    dy16 = torch.randn((1,) + tuple(od) + (C,), generator=gen).half()
    y_ref = F.max_pool3d(F.pad(R.ncdhw(x16.double()), fpad(lo, hi)), k, s, ceil_mode=True)
    e = dict(kind="pool", x=Act(x16.contiguous()), out=Act(R.ndhwc(y_ref).half().contiguous()), k=k, stride=s,
             pad_lo=tuple(lo), pad_hi=tuple(hi))
    y, dx = R.pool_entry(e, dy16)
    assert tuple(y.shape[1:4]) == tuple(od)
    for c in range(C):
        ref = first_max_pool_bwd(x16[0, ..., c].double(), k, s, lo, hi, od, dy16[0, ..., c].double())
        assert torch.equal(dx[0, ..., c], ref), (geom, c)


# ---- argument checks of the backward entry points (no device work happens before them) --------------------------------
@pytest.fixture(scope="module")
def lib():
    return L.lib()


@pytest.fixture(scope="module")
def buf():
    b = (ctypes.c_char * (4096 + 16))()
    addr = (ctypes.addressof(b) + 15) & ~15                 # 16-byte aligned fake device pointer (never dereferenced)
    return b, ctypes.c_void_p(addr)


def expect(lib, rc, *words, code=L.E_ARG):
    assert rc == code
    msg = lib.step_last_error().decode()
    for w in words:
        assert w in msg, (w, msg)


def act_bwd(lib, p, dy_ld=16, y_ld=16, relu=1, M=10, C=16, dz_ld=16, dres="p", dres_ld=16, dy="p", y="p", dz="p", scale=None):
    pick = lambda v: p if v == "p" else v
    return lib.step_act_bwd_f16(pick(dy), dy_ld, pick(y), y_ld, scale, relu, M, C, pick(dz), dz_ld, pick(dres), dres_ld, None)


def test_act_bwd_rejects_partial_vectors_and_misalignment(lib, buf):
    p = buf[1]
    assert act_bwd(lib, p, M=0) == L.E_ARG
    for kw in (dict(C=12), dict(dy_ld=20), dict(y_ld=12), dict(dz_ld=20), dict(dres_ld=12)):
        expect(lib, act_bwd(lib, p, **kw), "act_bwd: bad arguments")
    expect(lib, act_bwd(lib, p, y=None), "act_bwd: bad arguments")                 # the ReLU mask needs y
    for which in ("dy", "y", "dz", "dres"):
        expect(lib, act_bwd(lib, p, **{which: ctypes.c_void_p(p.value + 8)}), "16-byte aligned")


def wgrad(lib, p, dz_ld=16, x_ld=16, N=1, T=3, H=4, W=5, Cout=16, Cin=16, k=(3, 3, 3), pad=(1, 1, 1), dw_ld=16, ws_bytes=1 << 30,
          dz="p", x="p", dw="p", ws="p"):
    pick = lambda v: p if v == "p" else v
    return lib.step_conv_wgrad_f16(pick(dz), dz_ld, pick(x), x_ld, N, T, H, W, Cout, Cin, k[0], k[1], k[2], pad[0], pad[1], pad[2],
                                   1.0, pick(dw), dw_ld, 0, pick(ws), ws_bytes, None)


def test_conv_wgrad_rejects_bad_channels_alignment_padding_and_workspace(lib, buf):
    p = buf[1]
    for kw in (dict(Cout=12, dz_ld=16), dict(Cin=20, x_ld=24, dw_ld=24), dict(dz_ld=12), dict(x_ld=20), dict(dw_ld=8)):
        expect(lib, wgrad(lib, p, **kw), "conv_wgrad", "multiples of 8")
    for which in ("dz", "x"):
        expect(lib, wgrad(lib, p, **{which: ctypes.c_void_p(p.value + 8)}), "16-byte aligned")
    for pad in ((3, 1, 1), (1, 3, 1), (1, 1, -1), (0, 0, 3)):
        expect(lib, wgrad(lib, p, pad=pad), "conv_wgrad: bad padding")
    expect(lib, wgrad(lib, p, k=(1, 1, 1), pad=(0, 1, 0)), "conv_wgrad: bad padding")  # a 1-tap filter has no padding
    expect(lib, wgrad(lib, p, ws=None), "conv_wgrad: bad arguments")
    need = lib.step_conv_wgrad_workspace_bytes(60, 16, 16, 27)
    expect(lib, wgrad(lib, p, ws_bytes=need - 4), "workspace", code=L.E_WORKSPACE)


def pool_bwd(lib, p, C=16, k=(3, 3, 3), s=(2, 2, 2), lo=(1, 1, 1), hi=(1, 1, 1), dims=(7, 9, 9), out=(4, 5, 5), x="p", ws="p"):
    pick = lambda v: p if v == "p" else v
    return lib.step_maxpool3d_bwd_f16(pick(x), C, p, C, 1, dims[0], dims[1], dims[2], C, k[0], k[1], k[2], s[0], s[1], s[2],
                                      lo[0], lo[1], lo[2], hi[0], hi[1], hi[2], out[0], out[1], out[2], p, C, pick(ws), None)


def test_maxpool_bwd_rejects_oversized_windows_zero_strides_and_padding_outside_the_window(lib, buf):
    p = buf[1]
    # tap indices are bytes with 254 (padding won) and 255 (empty window) reserved: at most 253 taps
    expect(lib, pool_bwd(lib, p, k=(1, 1, 254), lo=(0, 0, 1)), "maxpool3d_bwd: bad arguments")
    expect(lib, pool_bwd(lib, p, k=(2, 11, 12), lo=(1, 1, 1)), "maxpool3d_bwd: bad arguments")
    expect(lib, pool_bwd(lib, p, x=None), "maxpool3d_bwd: bad arguments")
    expect(lib, pool_bwd(lib, p, ws=None), "maxpool3d_bwd: bad arguments")
    for s in ((0, 2, 2), (2, 0, 2), (2, 2, 0)):
        expect(lib, pool_bwd(lib, p, s=s), "maxpool3d_bwd", "must be positive")
    expect(lib, pool_bwd(lib, p, out=(4, 0, 5)), "must be positive")
    for lo, hi in (((3, 1, 1), (1, 1, 1)), ((1, -1, 1), (1, 1, 1)), ((1, 1, 1), (1, 1, -1))):
        expect(lib, pool_bwd(lib, p, lo=lo, hi=hi), "maxpool3d_bwd: bad padding")


# ---- the forward helpers ----------------------------------------------------------------------------------------------
def _bn_unit(cin, cout, k, stride=(1, 1, 1), seed=0):
    from step_b200.i3d import Unit3Dpy
    gen = torch.Generator().manual_seed(seed)
    u = Unit3Dpy(cin, cout, kernel_size=k, stride=stride).eval()
    with torch.no_grad():
        u.conv3d.weight.copy_(torch.randn(u.conv3d.weight.shape, generator=gen) * 0.2)
        u.batch3d.weight.copy_(torch.rand(cout, generator=gen) + 0.5)
        u.batch3d.bias.copy_(torch.randn(cout, generator=gen) * 0.2)
        u.batch3d.running_mean.copy_(torch.randn(cout, generator=gen) * 0.1)
        u.batch3d.running_var.copy_(torch.rand(cout, generator=gen) + 0.5)
    return u, gen


def _module_fwd(u, x16, stride, residual=None):
    """relu(batch_norm(conv3d(SAME pad(x), w)) + residual) in float64 on the module's fp16-rounded weight."""
    k = u.kernel_size
    lo, hi = zip(*(E.same_pad(kk, ss) for kk, ss in zip(k, stride)))
    bn = u.batch3d
    z = F.conv3d(F.pad(R.ncdhw(x16.double()), fpad(lo, hi)), u.conv3d.weight.detach().half().double(), stride=stride)
    z = F.batch_norm(z, bn.running_mean.double(), bn.running_var.double(), bn.weight.double(), bn.bias.double(), False, 0.0,
                     bn.eps)
    if residual is not None:
        z = z + R.ncdhw(residual.double())
    return R.ndhwc(torch.relu(z))


def _fold_within(got, ref, scale_err):
    """conv_fwd uses engine.fold_bn's fp32 scale / shift: within a few fp32 ulps of the float64 BatchNorm."""
    err = (got - ref).abs()
    assert bool((err <= scale_err).all()), float((err - scale_err).max())


@pytest.mark.parametrize("k,stride,residual", [((3, 3, 3), (1, 1, 1), False), ((1, 1, 1), (1, 1, 1), True),
                                               ((3, 3, 3), (2, 2, 2), False), ((1, 3, 3), (1, 1, 1), True)])
def test_conv_fwd_matches_the_module(k, stride, residual):
    """conv_fwd (packed fp16 filter, fp32 folded scale / shift, fp16 residual) against the Unit3Dpy's meaning in float64:
    SAME padding (asymmetric at stride 2 on odd extents), BatchNorm eval, residual, ReLU; and its magnitude terms."""
    u, gen = _bn_unit(8, 16, k, stride, seed=sum(k) + stride[0])
    N, T, H, W = 2, 5, 7, 6
    x16 = half_values(N, T, H, W, 8, gen=gen)
    w, scale, shift = u.packed(L.F16)
    od = E.same_out_dims((T, H, W), k, stride)
    lo = tuple(E.same_pad(kk, ss)[0] for kk, ss in zip(k, stride))
    res = half_values(N, *od, 16, gen=gen) if residual else None
    (y,), (xw,), (epi,) = R.conv_fwd(x16, w, scale, shift, res, k, stride, lo, od, True)
    ref = _module_fwd(u, x16, stride, res)
    assert y.shape == ref.shape
    _fold_within(y, ref, 2.0 ** -20 * (epi + 1.0))
    # the magnitude terms bound what they claim to: |acc * scale| <= xw, |y| <= epi
    assert bool((y.abs() <= epi + 1e-12).all())
    assert bool((xw >= 0).all()) and bool((epi >= 0).all())


def test_conv_fwd_splits_the_fused_1x1_and_runs_the_stem_and_frame_convs():
    """The three-way fused 1x1 (one packed filter, outputs split by width) equals three separate conv_fwd calls; the s2d
    stem (4x4x4 pad 1 over the 24 live channels, pack_stem_s2d filter) equals the stride-2 7x7x7 module; a biased (1,3,3)
    frame conv (nn.Conv2d on frames) equals F.conv2d."""
    units = [_bn_unit(24, c, (1, 1, 1), seed=c)[0] for c in (16, 8, 24)]
    gen = torch.Generator().manual_seed(9)
    x16 = half_values(1, 3, 4, 5, 24, gen=gen)
    parts = [u.packed(L.F16) for u in units]
    w = torch.cat([p[0] for p in parts], 0)
    sc = torch.cat([p[1] for p in parts])
    sh = torch.cat([p[2] for p in parts])
    ys, xws, epis = R.conv_fwd(x16, w, sc, sh, None, (1, 1, 1), (1, 1, 1), (0, 0, 0), (3, 4, 5), True, [16, 8, 24])
    assert [y.shape[-1] for y in ys] == [16, 8, 24]
    for (wp, s, b), y, xw in zip(parts, ys, xws):
        (y1,), (xw1,), _ = R.conv_fwd(x16, wp, s, b, None, (1, 1, 1), (1, 1, 1), (0, 0, 0), (3, 4, 5), True)
        assert torch.equal(y, y1) and torch.equal(xw, xw1)
    # the stem
    from step_b200.i3d import Unit3Dpy
    stem = Unit3Dpy(3, 64, kernel_size=(7, 7, 7), stride=(2, 2, 2)).eval()
    with torch.no_grad():
        stem.conv3d.weight.copy_(torch.randn(stem.conv3d.weight.shape, generator=gen) * 0.05)
    clip = torch.randn(1, 3, 6, 10, 8, generator=gen).half()
    xs = s2d_pack(clip.double()).half()
    ws, ss, bs = stem.packed(L.F16, s2d=True)
    (y,), _, _ = R.conv_fwd(xs[..., :24], ws, ss, bs, None, (4, 4, 4), (1, 1, 1), (1, 1, 1), (3, 5, 4), True)
    ref = _module_fwd(stem, R.ndhwc(clip), (2, 2, 2))
    _fold_within(y, ref, 2.0 ** -20 * (ref.abs() + 1.0))
    # a frame conv with bias, no BatchNorm, no activation
    conv = torch.nn.Conv2d(16, 8, 3, padding=1, bias=True)
    xf = half_values(4, 1, 6, 5, 16, gen=gen)
    wp = E.pack_conv_weight(conv.weight, L.F16)
    (y,), _, _ = R.conv_fwd(xf, wp, None, conv.bias.detach().float(), None, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 6, 5), False)
    ref = F.conv2d(R.ncdhw(xf.double())[:, :, 0], conv.weight.detach().half().double(), conv.bias.detach().float().double(),
                   padding=1)
    assert float((y[:, 0] - ref.permute(0, 2, 3, 1)).abs().max()) <= 1e-12


@pytest.mark.parametrize("relu2,bias", [(True, False), (False, True)])
def test_exit_fwd_equals_two_conv_fwd(relu2, bias):
    """y and z of exit_fwd are two conv_fwd calls: the 1x1 with residual and ReLU, then the 1x1 on fp16(y); z_carry is
    |w1| applied to y's full tolerance."""
    gen = torch.Generator().manual_seed(5)
    M = 37
    h = half_values(M, 64, gen=gen)
    w3 = half_values(128, 1, 64, gen=gen, scale=0.125)
    x = half_values(M, 128, gen=gen)
    w1 = half_values(32, 1, 128, gen=gen, scale=0.1)
    b = torch.randn(32, generator=gen) if bias else None
    r = R.exit_fwd(h, w3, x, w1, b, relu2)
    rows = lambda t: t.reshape(M, 1, 1, 1, t.shape[-1])
    (y,), (yxw,), (yepi,) = R.conv_fwd(rows(h), w3, None, None, rows(x), (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), True)
    assert torch.equal(y.reshape(M, -1), r["y"]) and torch.equal(yxw.reshape(M, -1), r["y_xw"])
    assert torch.equal(yepi.reshape(M, -1), r["y_epi"])
    y16 = r["y"].half()
    (z,), (zxw,), (zepi,) = R.conv_fwd(rows(y16), w1, None, b, None, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), relu2)
    for a, key in ((z, "z"), (zxw, "z_xw"), (zepi, "z_epi")):
        assert float((a.reshape(M, -1) - r[key]).abs().max()) <= 1e-12 * (1.0 + float(r[key].abs().max())), key
    my = R.fwd_margin(r["y_xw"], r["y_epi"])
    carry = (my + R.ulp16(r["y"].abs() + my)) @ w1[:, 0].double().abs().t()
    assert torch.allclose(carry, r["z_carry"], rtol=1e-12, atol=0)


def test_check_fwd_accepts_rounding_and_rejects_a_scaled_or_truncated_output():
    """check_fwd on a synthetic 1x1 layer: the float64 result rounded to nearest passes; the same scaled by 1 + 2^-8 fails;
    rounded toward zero it stays inside the elementwise bound and fails the bias test."""
    gen = torch.Generator().manual_seed(11)
    x16 = half_values(4, 4, 14, 14, 256, gen=gen)
    w = half_values(64, 1, 256, gen=gen, scale=1.0 / 16)
    (ref,), (xw,), (epi,) = R.conv_fwd(x16, w, None, None, None, (1, 1, 1), (1, 1, 1), (0, 0, 0), (4, 14, 14), False)
    steps = R.conv_steps((1, 1, 1), 256)
    n, d, thr = R.check_fwd(ref.half(), ref, xw, epi, steps, "nearest")
    assert n > 10000 and abs(d) < thr < 0.5
    with pytest.raises(AssertionError, match="scaled"):
        R.check_fwd((ref * (1.0 + 2.0 ** -8)).half(), ref, xw, epi, steps, "scaled")
    rtz = ref.half().double()
    rtz = torch.where(rtz.abs() > ref.abs(), rtz - rtz.sign() * R.ulp16(rtz - rtz.sign() * R.ulp16(rtz) / 2), rtz)
    assert bool(((rtz - ref).abs() < R.ulp16(ref) + 1e-30).all()) and bool((rtz.abs() <= ref.abs()).all())
    with pytest.raises(AssertionError, match="bias"):
        R.check_fwd(rtz, ref, xw, epi, steps, "toward zero")


def test_mean_mid_and_linear_references():
    """mean_mid is the mean over B; linear is x[row_map] w^T + bias (+ y0), sigmoid on request."""
    gen = torch.Generator().manual_seed(12)
    x = torch.randn(3, 5, 2, 8, generator=gen).half()
    m, mabs = R.mean_mid(x)
    assert torch.allclose(m, x.double().permute(0, 2, 3, 1).reshape(3, 16, 5).mean(-1), rtol=0, atol=1e-15)
    assert bool((m.abs() <= mabs).all())
    xs = torch.randn(7, 40, generator=gen)
    w = torch.randn(5, 40, generator=gen)
    b = torch.randn(5, generator=gen)
    y0 = torch.randn(4, 5, generator=gen)
    rows = torch.tensor([6, 0, 3, 3], dtype=torch.int32)
    y, v, a = R.linear(xs, w, b, y0, rows, act=1)
    ref = xs.double()[rows.long()] @ w.double().t() + b.double() + y0.double()
    assert torch.allclose(v, ref, rtol=1e-14, atol=0) and torch.allclose(y, torch.sigmoid(ref), rtol=1e-14, atol=0)
    assert bool((v.abs() <= a).all())


def test_head_regress_matches_nn_linear_on_the_nchw_flatten():
    """head_regress from the three nn.Linear modules equals nn.Linear on the reference's (c, h, w) flatten of the
    downsample2 output, chunk slices included; and the channels-last product with two_branch._perm_flat's weight is the
    same number (what the kernel computes)."""
    from step_b200.two_branch import _perm_flat
    gen = torch.Generator().manual_seed(13)
    C, ps, R_, T, Tc = 16, 7, 3, 9, 3
    mods = [torch.nn.Linear(C * ps * ps, 4) for _ in range(3)]
    feat = half_values(R_ * T, ps, ps, C, gen=gen)
    r = R.head_regress(feat, *mods, Tc, T)
    flat = feat.double().permute(0, 3, 1, 2).reshape(R_ * T, -1)                # NCHW flatten (two_branch.py:261)
    outs = [(flat @ m.weight.detach().half().double().t() + m.bias.detach().double()).view(R_, T, 4) for m in mods]
    s0, s1, e0, e1 = R.head_chunks(Tc, T)
    assert (s0, s1, e0, e1) == (0, 3, 6, 9)
    assert torch.allclose(r["local"], outs[0], rtol=1e-13, atol=1e-13)
    assert torch.allclose(r["first"], (outs[0] + outs[1])[:, s0:s1], rtol=1e-13, atol=1e-13)
    assert torch.allclose(r["last"], (outs[0] + outs[2])[:, e0:e1], rtol=1e-13, atol=1e-13)
    cl = feat.double().reshape(R_ * T, -1) @ _perm_flat(mods[0].weight, C, ps).half().double().t()
    assert torch.allclose(cl.view(R_, T, 4) + mods[0].bias.detach().double(), outs[0], rtol=1e-13, atol=1e-13)
    assert bool((r["local_tol"] > 0).all())


def _roi_align_loops(feat, roi, scale, ph, pw):
    """ROIAlign of one roi, written as the loops of the reference's CPU op (float32 coordinates, float64 sums)."""
    f32 = lambda v: float(torch.tensor(float(v), dtype=torch.float32))
    K, H, W, C = feat.shape
    b = int(roi[0])
    sw, sh, ew, eh = (f32(f32(roi[j]) * f32(scale)) for j in (1, 2, 3, 4))
    rw, rh = max(f32(ew - sw), 1.0), max(f32(eh - sh), 1.0)
    bh, bw = f32(rh / ph), f32(rw / pw)
    gh, gw = int(math.ceil(f32(rh / ph))), int(math.ceil(f32(rw / pw)))
    out = torch.zeros(ph, pw, C, dtype=torch.float64)
    fd = feat.double()
    for p in range(ph):
        for q in range(pw):
            for iy in range(gh):
                y = f32(f32(sh + f32(p * bh)) + f32(f32(f32(iy + 0.5) * bh) / gh))
                for ix in range(gw):
                    x = f32(f32(sw + f32(q * bw)) + f32(f32(f32(ix + 0.5) * bw) / gw))
                    if y < -1.0 or y > H or x < -1.0 or x > W:
                        continue
                    yy, xx = max(y, 0.0), max(x, 0.0)
                    yl, xl = int(yy), int(xx)
                    if yl >= H - 1:
                        yh = yl = H - 1
                        yy = float(yl)
                    else:
                        yh = yl + 1
                    if xl >= W - 1:
                        xh = xl = W - 1
                        xx = float(xl)
                    else:
                        xh = xl + 1
                    ly, lx = f32(yy - yl), f32(xx - xl)
                    hy, hx = f32(1.0 - ly), f32(1.0 - lx)
                    out[p, q] += (f32(hy * hx) * fd[b, yl, xl] + f32(hy * lx) * fd[b, yl, xh] + f32(ly * hx) * fd[b, yh, xl]
                                  + f32(ly * lx) * fd[b, yh, xh])
    return out / (gh * gw)


def test_roi_align_reference_matches_the_loop_rule():
    """R.roi_align (vectorised) against the per-sample loops on ROIs inside, across and past the map edge (samples beyond
    [-1, H] dropped, the last row / column clamped), a small ROI (grid 1x1) and a large one (grid 3x3), with the
    roi_T / feat_T / t_start frame map."""
    gen = torch.Generator().manual_seed(14)
    K, H, W, C = 6, 9, 11, 8
    feat = half_values(K, H, W, C, gen=gen)
    rois = torch.tensor([[0, 10.0, 20.0, 90.0, 100.0], [1, -30.0, -20.0, 60.0, 40.0], [2, 100.0, 90.0, 200.0, 170.0],
                         [3, 40.0, 40.0, 44.0, 47.0], [4, 0.0, 0.0, 175.0, 143.0]], dtype=torch.float32)
    out, out_abs = R.roi_align(feat, rois, 1.0 / 16.0, 7, 7)
    for r in range(rois.shape[0]):
        ref = _roi_align_loops(feat, rois[r], 1.0 / 16.0, 7, 7)
        assert torch.allclose(out[r], ref, rtol=1e-12, atol=1e-12), r
    assert bool((out.abs() <= out_abs + 1e-15).all())
    # frame map: roi frame f of a 2-frame slice starting at t 1 of 3-frame clips -> (f // 2) * 3 + 1 + f % 2
    fm, _ = R.roi_align(feat, rois[:4], 1.0 / 16.0, 7, 7, roi_T=2, feat_T=3, t_start=1)
    direct = rois[:4].clone()
    direct[:, 0] = torch.tensor([1.0, 2.0, 4.0, 5.0])
    ref, _ = R.roi_align(feat, direct, 1.0 / 16.0, 7, 7)
    assert torch.equal(fm, ref)


# ---- the references of train_step's launches outside the tape ---------------------------------------------------------
EDGE_ROIS = [[0, 10.0, 20.0, 90.0, 100.0],      # inside
             [1, -30.0, -20.0, 60.0, 40.0],     # corners in [-16, 0): samples in [-1, 0] clamped to 0
             [2, -100.0, -90.0, 40.0, 30.0],    # corners below -16: samples dropped
             [3, 100.0, 90.0, 200.0, 170.0],    # past the bottom and right edges: last row / column clamped
             [4, 40.0, 40.0, 44.0, 47.0],       # grid 1x1
             [5, 0.0, 0.0, 175.0, 143.0],       # the whole map
             [0, 60.0, 50.0, 20.0, 30.0],       # degenerate: x2 < x1, y2 < y1 (width and height clamped to 1)
             [1, -40.0, 5.0, 1000.0, 700.0]]    # grid 10 x 7: more than one sample table of the kernel


def _edge_case(gen, K=6, H=9, W=11, C=8):
    feat = half_values(K, H, W, C, gen=gen).double()
    rois = torch.tensor(EDGE_ROIS, dtype=torch.float32)
    return feat, rois


@pytest.mark.parametrize("sr", [0, 2])
def test_roi_align_bwd_is_the_adjoint_of_roi_align(sr):
    """<roi_align(feat), g> = <feat, roi_align_bwd(g)> in float64, to 1e-12, on ROIs inside, across and past every edge,
    degenerate and larger than one sample table; the same with the roi_T / feat_T / t_start frame map."""
    gen = torch.Generator().manual_seed(21 + sr)
    feat, rois = _edge_case(gen)
    K, H, W, C = feat.shape
    g = torch.randn(rois.shape[0], 7, 7, C, generator=gen, dtype=torch.float64)
    out, _ = R.roi_align(feat, rois, 1.0 / 16.0, 7, 7, sampling_ratio=sr)
    gin, mag, n = R.roi_align_bwd(g, rois, 1.0 / 16.0, 7, 7, K, H, W, sampling_ratio=sr)
    lhs, rhs = float((out * g).sum()), float((feat * gin).sum())
    assert abs(lhs - rhs) <= 1e-12 * float((out.abs() * g.abs()).sum()), (lhs, rhs)
    assert bool((gin.abs() <= mag + 1e-15).all()) and bool((n >= 0).all())
    # frame map: 2 clips of 3 frames, a 2-frame slice from t 1; ROI frames 0..3
    fm = rois[:4].clone()
    fm[:, 0] = torch.tensor([0.0, 1.0, 2.0, 3.0])
    out, _ = R.roi_align(feat, fm, 1.0 / 16.0, 5, 3, roi_T=2, feat_T=3, t_start=1, sampling_ratio=sr)
    g = g[:4, :5, :3]
    gin, _, n = R.roi_align_bwd(g.contiguous(), fm, 1.0 / 16.0, 5, 3, K, H, W, roi_T=2, feat_T=3, t_start=1, sampling_ratio=sr)
    assert abs(float((out * g).sum()) - float((feat * gin).sum())) <= 1e-12 * float((out.abs() * g.abs()).sum())
    assert float(n[[0, 3]].sum()) == 0.0 and float(n[[1, 2, 4, 5]].sum()) > 0          # frames 0 and 3 are outside the slice


def test_roi_align_bwd_matches_torchvision_autograd():
    """On ROIs whose fp32 sample coordinates and weights are exact (corners on multiples of 1/16 of a pixel, sizes giving
    power-of-two bins and grids), roi_align_bwd equals float64 autograd of torchvision.ops.roi_align(aligned=False),
    including samples clamped at the far edges and dropped ones."""
    tv = pytest.importorskip("torchvision")
    gen = torch.Generator().manual_seed(22)
    K, H, W, C = 3, 10, 12, 4
    feat = torch.randn(K, C, H, W, generator=gen, dtype=torch.float64, requires_grad=True)
    rois = torch.tensor([[0, 16.0, 32.0, 80.0, 96.0], [1, 0.0, 0.0, 256.0, 256.0], [2, 128.0, 96.0, 256.0, 224.0],
                         [0, -32.0, -24.0, 32.0, 40.0], [2, -64.0, 40.0, 0.0, 104.0], [1, 96.0, 48.0, 112.0, 64.0]],
                        dtype=torch.float64)
    for ph, pw in ((4, 4), (2, 8)):
        out = tv.ops.roi_align(feat, rois, (ph, pw), 1.0 / 16.0, 0, aligned=False)
        g = torch.randn(out.shape, generator=gen, dtype=torch.float64)
        (ref,) = torch.autograd.grad(out, feat, g)
        gin, _, _ = R.roi_align_bwd(g.permute(0, 2, 3, 1).contiguous(), rois.float(), 1.0 / 16.0, ph, pw, K, H, W)
        assert torch.allclose(gin.permute(0, 3, 1, 2), ref, rtol=0, atol=1e-13), (ph, pw)


def _shift_clamped_tap(groups, H, W):
    """A copy of roi_align_terms' groups with tap 0 of one sample clamped at the last row (its taps 0 and 2 on one pixel)
    moved up by one row.  Returns (groups, True) or (groups, False) when there is no such sample."""
    out = []
    moved = False
    for gr in groups:
        gr = dict(gr, pix=gr["pix"].clone())
        if not moved:
            p = gr["pix"].view(gr["pix"].shape[0], -1, 4)
            w = gr["w"].view_as(p)
            hit = ((p[..., 0] == p[..., 2]) & (p[..., 0] >= (H - 1) * W) & (w[..., 0] > 0)).nonzero()
            if hit.shape[0]:
                r, s = hit[0].tolist()
                p[r, s, 0] -= W
                moved = True
        out.append(gr)
    return out, moved


def test_roi_align_bwd_check_rejects_perturbed_references():
    """roi_align_bwd_check accepts the float64 result rounded to fp32 on top of an initial gradient, and rejects the
    reference with the 1/count dropped, with one tap of a clamped sample moved by a pixel, with the frame map off by one
    frame, and scaled by 1 + 2^-12."""
    gen = torch.Generator().manual_seed(23)
    K, H, W, C = 6, 9, 11, 8
    rois = torch.tensor(EDGE_ROIS, dtype=torch.float32)
    rois[:, 0] = torch.tensor([0.0, 1.0, 2.0, 3.0, 0.0, 1.0, 2.0, 3.0])
    args = (rois, 1.0 / 16.0, 7, 7, K, H, W)
    fmap = dict(roi_T=2, feat_T=3, t_start=1)
    g = half_values(rois.shape[0], 7, 7, C, gen=gen)
    init = torch.randn(K, H, W, C, generator=gen) * 0.01
    ref, mag, n = R.roi_align_bwd(g, *args, **fmap)
    got = (init.double() + ref).float()
    assert R.roi_align_bwd_check(got, init, ref, mag, n) < 1.0
    groups = R.roi_align_terms(rois, 1.0 / 16.0, 7, 7, H, W)
    no_count = [dict(gr, count=1) for gr in groups]
    assert any(gr["count"] > 1 for gr in groups)
    shifted, moved = _shift_clamped_tap(groups, H, W)
    assert moved
    bad = {"1/count dropped": R.roi_align_bwd(g, *args, groups=no_count, **fmap),
           "clamped tap moved": R.roi_align_bwd(g, *args, groups=shifted, **fmap),
           "frame map off by one": R.roi_align_bwd(g, *args, roi_T=2, feat_T=3, t_start=0),
           "scaled": (ref * (1.0 + 2.0 ** -12), mag, n)}
    for what, (r_, m_, n_) in bad.items():
        with pytest.raises(AssertionError):
            R.roi_align_bwd_check(got, init, r_, m_, n_, what)


def _roi_fma_chain(feat, rois, groups, nbins):
    """What the fp16 ROIAlign with fp32 FMAs computes (csrc/roi.cu: roi_align_fwd_nhwc_kernel<__half, false> and the
    direct form of the packed kernel), restated on the CPU: fp32 weights w * fp32(1 / count), one fp32 rounding per tap
    added in (bin, iy, ix, tap) order, an fp16 store.  fp16 [R, nbins, C]."""
    K, H, W, C = feat.shape
    f = feat.reshape(K, H * W, C).double()
    fr = R.roi_frames(rois)
    out = torch.zeros(rois.shape[0], nbins, C, dtype=torch.float16)
    for gr in groups:
        G = gr["idx"].numel()
        ic = torch.tensor(1.0, dtype=torch.float32) / gr["count"]
        live = gr["pix"] >= 0
        w = torch.where(live, gr["w"].float() * ic, torch.zeros(())).double().view(G, nbins, -1)
        v = f[fr[gr["idx"]].view(-1, 1), gr["pix"].clamp(min=0)].view(G, nbins, -1, C)
        acc = torch.zeros(G, nbins, C, dtype=torch.float32)
        for k in range(w.shape[-1]):
            acc = (acc.double() + w[..., k, None] * v[..., k, :]).float()
        out[gr["idx"]] = acc.half()
    return out


@pytest.mark.parametrize("sr", [0, 3])
def test_roi_align_fma_tol_accepts_the_fma_chain_and_rejects_perturbed_references(sr):
    """The fp32-FMA ROIAlign restated on the CPU is within roi_align_fma_tol of the float64 reference on the edge ROIs;
    the bound rejects the reference scaled by 1 + 2^-10, with the 1/count dropped, and with one tap of a clamped sample
    moved by a pixel."""
    gen = torch.Generator().manual_seed(25 + sr)
    feat, rois = _edge_case(gen)
    K, H, W, C = feat.shape
    groups = R.roi_align_terms(rois, 1.0 / 16.0, 7, 7, H, W, sr)
    ref, out_abs = R.roi_align(feat, rois, 1.0 / 16.0, 7, 7, sampling_ratio=sr)
    tol = R.roi_align_fma_tol(out_abs, R.roi_samples_per_bin(groups, rois.shape[0]))
    got = _roi_fma_chain(feat, rois, groups, 49).view_as(ref)
    assert R._check_within(got, ref, tol, ("fma chain", sr)) < 1.0
    no_count = [dict(gr, count=1) for gr in groups]
    assert any(gr["count"] > 1 for gr in groups)
    shifted, moved = _shift_clamped_tap(groups, H, W)
    assert moved
    bad = {"scaled": ref * (1.0 + 2.0 ** -10),
           "1/count dropped": R.roi_align(feat, rois, 1.0 / 16.0, 7, 7, groups=no_count)[0],
           "clamped tap moved": R.roi_align(feat, rois, 1.0 / 16.0, 7, 7, groups=shifted)[0]}
    for what, r_ in bad.items():
        with pytest.raises(AssertionError):
            R._check_within(got, r_, tol, what)


def _packed_table_terms(groups, nbins):
    """roi_align_terms' groups with every tap of a bin whose pixel is not among the bin's first ROI_MERGED distinct pixels,
    in (iy, ix, tap) order, zeroed: what a merged table that silently drops pixels past its capacity would sum."""
    out = []
    for gr in groups:
        G = gr["idx"].numel()
        pix = gr["pix"].view(G, nbins, -1)
        w = gr["w"].clone().view_as(pix)
        for g in range(G):
            for b in range(nbins):
                seen = set()
                for k, p in enumerate(pix[g, b].tolist()):
                    if p < 0 or p in seen:
                        continue
                    if len(seen) < R.ROI_MERGED:
                        seen.add(p)
                    else:
                        w[g, b, k] = 0.0
        out.append(dict(gr, w=w.view_as(gr["w"])))
    return out


def test_roi_align_tol_rejects_a_bin_with_pixels_past_the_table_dropped():
    """sampling_ratio 3 with 10-pixel bins (a 70 px ROI inside an 80 x 80 map, at 7 x 7): a bin's 9 samples touch 36
    distinct pixels.  roi_align_tol rejects the sum over the first 16 alone (the 17th..36th pixel dropped); at
    sampling_ratio 2 no bin exceeds 16 pixels and nothing is dropped."""
    gen = torch.Generator().manual_seed(27)
    H = W = 80
    feat = (0.5 + 0.5 * torch.rand(1, H, W, 8, generator=gen)).half()
    rois = torch.tensor([[0, 80.0, 80.0, 1200.0, 1200.0]], dtype=torch.float32)
    vmax = float(feat.abs().max())
    for sr, most in ((3, 36), (2, 16)):
        groups = R.roi_align_terms(rois, 1.0 / 16.0, 7, 7, H, W, sr)
        assert max(int(R.roi_distinct_pixels(gr, 49).max()) for gr in groups) == most
        ref, out_abs = R.roi_align(feat, rois, 1.0 / 16.0, 7, 7, sampling_ratio=sr)
        packed, _ = R.roi_align(feat, rois, 1.0 / 16.0, 7, 7, groups=_packed_table_terms(groups, 49))
        tol = R.roi_align_tol(out_abs, vmax)
        if most > R.ROI_MERGED:
            with pytest.raises(AssertionError):
                R._check_within(packed, ref, tol, "17th..36th pixel dropped")
        else:
            assert torch.equal(packed, ref)


@pytest.mark.parametrize("xdtype", [torch.float16, torch.float32])
def test_linear_bwd_matches_autograd_and_its_check_rejects_perturbations(xdtype):
    """linear_bwd's dx / dW / db equal float64 autograd of x w^T + b (dx accumulated onto init_dx); linear_bwd_check
    accepts them rounded to fp32 and rejects a 1 + 2^-12 scale and one transposed index (two columns of x swapped)."""
    gen = torch.Generator().manual_seed(24)
    M, K, Nn = 37, 96, 4
    x = torch.randn(M, K, generator=gen).to(xdtype)
    w = torch.randn(Nn, K, generator=gen)
    dy = torch.randn(M, Nn, generator=gen)
    init = torch.randn(M, K, generator=gen)
    xd, wd = x.double().requires_grad_(True), w.double().requires_grad_(True)
    bd = torch.zeros(Nn, dtype=torch.float64, requires_grad=True)
    (xd @ wd.t() + bd).backward(dy.double())
    r = R.linear_bwd(x, w, dy, init_dx=init)
    assert torch.allclose(r["dx"], xd.grad + init.double(), rtol=1e-14, atol=1e-14)
    assert torch.allclose(r["dw"], wd.grad, rtol=1e-14, atol=1e-14) and torch.allclose(r["db"], bd.grad, rtol=1e-14, atol=1e-14)
    for key, steps in (("dx", Nn), ("dw", M), ("db", M)):
        assert R.linear_bwd_check(r[key].float(), r[key], r[key + "_abs"], steps, key) < 1.0
        with pytest.raises(AssertionError):
            R.linear_bwd_check(r[key].float(), r[key] * (1.0 + 2.0 ** -12), r[key + "_abs"], steps, key)
    xs = x.clone()
    xs[:, [3, 4]] = xs[:, [4, 3]]
    with pytest.raises(AssertionError):
        rs = R.linear_bwd(xs, w, dy)
        R.linear_bwd_check(r["dw"].float(), rs["dw"], rs["dw_abs"], M, "dw transposed")


def _loss_case(gen, N=6, cls=5, T=3, chunks=3):
    Tl = T * chunks
    logits = torch.randn(N, cls, generator=gen) * 3
    box = torch.rand(N, 1, 2, generator=gen) * 200
    size = 20 + torch.rand(N, 1, 2, generator=gen) * 80
    tubes = torch.cat([torch.zeros(N, Tl, 1), (box + torch.rand(N, Tl, 2, generator=gen) * 4),
                       (box + size + torch.rand(N, Tl, 2, generator=gen) * 4)], 2)
    tg = torch.zeros(N, 3, 6 + cls)
    tg[:, :, :2] = box + torch.rand(N, 3, 2, generator=gen) * 10
    tg[:, :, 2:4] = box + size + torch.rand(N, 3, 2, generator=gen) * 10
    tg[:, :, 4:6] = (torch.rand(N, 3, 2, generator=gen) > 0.3).float()
    tg[0, :, 4:6] = 1.0
    tg[:, :, 6:] = (torch.rand(N, 3, cls, generator=gen) > 0.6).float()
    # predictions near the encoded targets, some coordinates past |d| = 1 (the linear branch of smooth-L1)
    local = torch.randn(N, Tl, 4, generator=gen) * 0.8
    first = torch.randn(N, T, 4, generator=gen) * 0.8
    last = torch.randn(N, T, 4, generator=gen) * 0.8
    return logits, local, first, last, tubes, tg, T


def test_loss_references_match_autograd_and_their_checks_reject_perturbations():
    """head_losses: the losses of oracle.model.two_branch_losses; dlocal is autograd's through first_loc = local[s0:] + a,
    last_loc = local[e0:] + b (the head's structure), dfirst / dlast d/da, d/db.  cls_loss: d mean(BCE) / d logits =
    (sigmoid - t) / (N cls).  Every bound accepts the float64 values rounded to fp32 and rejects a 1 + 2^-12 scale and
    one transposed index."""
    from oracle.model import two_branch_losses
    gen = torch.Generator().manual_seed(25)
    logits, local, first, last, tubes, tg, T = _loss_case(gen)
    ref = R.head_losses(logits, local, first, last, tubes, tg, T, 5.0, 1.0)
    loc = local.double().requires_grad_(True)
    s0, _, e0, _ = R.head_chunks(T, local.shape[1])
    a = (first.double() - local.double()[:, s0:s0 + T]).requires_grad_(True)
    b = (last.double() - local.double()[:, e0:e0 + T]).requires_grad_(True)
    x = logits.double().requires_grad_(True)
    lc, ll, ln = two_branch_losses(x, loc, loc[:, s0:s0 + T] + a, loc[:, e0:e0 + T] + b, tubes.double(), tg.double(), T)
    (lc.mean() + 5.0 * ll.mean() + 1.0 * ln.mean()).backward()
    for key, g in (("dlogits", x.grad), ("dlocal", loc.grad), ("dfirst", a.grad), ("dlast", b.grad)):
        assert torch.allclose(ref[key][0], g, rtol=1e-12, atol=1e-15), key
    for key, v in (("loss_cls", lc), ("loss_loc", ll), ("loss_nb", ln)):
        assert torch.allclose(ref[key][0], v.detach(), rtol=1e-12, atol=0), key
    t = tg[:, 1, 6:].double() * tg[:, 1, 4:5].double()
    assert torch.allclose(ref["dlogits"][0], (torch.sigmoid(logits.double()) - t) / logits.numel(), rtol=1e-12, atol=1e-18)
    cref = R.cls_loss(logits, tg)
    assert torch.equal(cref["loss"], ref["loss_cls"][0]) and torch.allclose(cref["dlogits"], ref["dlogits"][0], rtol=1e-14, atol=0)
    assert bool((ref["dlocal"][0] != 0).sum() > 0) and bool((ref["dlast"][0].abs() > 0).any())
    assert bool((ref["dlocal"][0].abs() >= 1.0 / 6).any()), "no coordinate on smooth-L1's linear branch"
    for key, (v, tol) in ref.items():
        assert R._check_within(v.float(), v, tol + 0.0, key) <= 1.0
        with pytest.raises(AssertionError):
            R._check_within(v.float(), v * (1.0 + 2.0 ** -12), tol, key)
    # one transposed index: two logits / two box coordinates swapped in the inputs
    lg = logits.clone()
    lg[:, [0, 1]] = lg[:, [1, 0]]
    lo = local.clone()
    lo[:, :, [0, 2]] = lo[:, :, [2, 0]]
    fi = first.clone()
    fi[:, :, [1, 3]] = fi[:, :, [3, 1]]
    for args, keys in (((lg, local, first, last), ("loss_cls", "dlogits")), ((logits, lo, first, last), ("loss_loc", "dlocal")),
                       ((logits, local, fi, last), ("loss_nb", "dfirst"))):
        bad = R.head_losses(*args, tubes, tg, T, 5.0, 1.0)
        for key in keys:
            with pytest.raises(AssertionError):
                R._check_within(ref[key][0].float(), bad[key][0], bad[key][1], (key, "transposed"))
