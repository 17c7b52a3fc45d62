"""CPU: the float64 tape reference of tests/_tape_reference.py pinned to the modules' meaning on small shapes, and the
argument checks of the backward entry points (step_act_bwd_f16, step_conv_wgrad_f16, step_maxpool3d_bwd_f16).

The reference rounds dz = dy * [y > 0] * scale to fp16 as act_bwd_kernel does; autograd of the module keeps it exact.
That rounding moves each dz by at most half an fp16 ulp, 2^-11 |dz|, so a weight or input gradient moves by at most
2^-11 (|dz|^T |x|) or 2^-11 (|dz| * |w|): the bound every comparison below uses.  Everything else is float64."""
import ctypes
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

STEP_E_ARG, STEP_E_WORKSPACE = 10001, 10003
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
    l = L.lib()
    l.step_last_error.restype = ctypes.c_char_p
    return l


@pytest.fixture(scope="module")
def buf():
    b = (ctypes.c_char * (4096 + 16))()
    addr = (ctypes.addressof(b) + 15) & ~15                 # 16-byte aligned fake device pointer (never dereferenced)
    return b, ctypes.c_void_p(addr)


def expect(lib, rc, *words, code=STEP_E_ARG):
    assert rc == code
    msg = lib.step_last_error().decode()
    for w in words:
        assert w in msg, (w, msg)


def act_bwd(lib, p, dy_ld=16, y_ld=16, relu=1, M=10, C=16, dz_ld=16, dres="p", dres_ld=16, dy="p", y="p", dz="p", scale=None):
    pick = lambda v: p if v == "p" else v
    return lib.step_act_bwd_f16(pick(dy), dy_ld, pick(y), y_ld, scale, relu, M, C, pick(dz), dz_ld, pick(dres), dres_ld, None)


def test_act_bwd_rejects_partial_vectors_and_misalignment(lib, buf):
    p = buf[1]
    assert act_bwd(lib, p, M=0) == STEP_E_ARG
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
    expect(lib, wgrad(lib, p, ws_bytes=need - 4), "workspace", code=STEP_E_WORKSPACE)


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
