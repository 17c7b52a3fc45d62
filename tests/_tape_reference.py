"""Float64 reference of the backward of one tape entry (step_b200/engine.py: the dicts `engine.conv` and `engine.maxpool`
append to engine.TAPE), fed the same fp16 operands the kernels read: the fp16 activations `x`, the packed fp16 weights
`e["w"]`, the fp32 BatchNorm scale and the fp16 output gradient.  Only the accumulation order and the final fp16 rounding
of the kernels differ from it, so the tests can derive their tolerances instead of fitting them.

Convolutions go through torch.nn.grad in float64 on the zero-padded input (the SAME padding of i3dpt.py:14-31 is
asymmetric, so it is applied with F.pad); pools through autograd of F.pad + F.max_pool3d(ceil_mode=True) in float64 on the
CPU.  Never fp32 on the GPU: cuDNN convolutions default to TF32 there.
"""
import torch
import torch.nn.functional as F


def act_view(a):
    """Act -> [N, T, H, W, C] view of its channel slice."""
    return a.buf[..., a.coff:a.coff + a.C]


def ncdhw(t):
    return t.permute(0, 4, 1, 2, 3)


def ndhwc(t):
    return t.permute(0, 2, 3, 4, 1)


def ulp16(v):
    """Spacing of the fp16 numbers at |v| (2^-24 in the subnormal range), float64."""
    v = v.abs().double()
    _, e = torch.frexp(v)                                   # v = m 2^e, m in [0.5, 1)
    return torch.ldexp(torch.ones_like(v), (e - 1).clamp(min=-14) - 10)


def act_bwd(dy, y, scale, relu):
    """What act_bwd_kernel forms from an output gradient: dz = fp16(fp32(dy) * [y > 0] * scale) and the fp32 masked
    gradient that flows into the residual input (exact: the mask only zeroes fp16 values)."""
    g = dy.float()
    if relu:
        g = torch.where(y.float() > 0, g, torch.zeros_like(g))
    dz = g * scale.float() if scale is not None else g
    return dz.half(), g


def unpack_s2d(xs, cin):
    """Inverse of the space-to-depth clip (csrc/pool_layout.cu clip_to_s2d): [N, T/2, H/2, W/2, >= 8 cin] with channel
    ((rt * 2 + rh) * 2 + rw) * cin + c at (t2, h2, w2)  ->  [N, cin, T, H, W] holding clip[2 t2 + rt, 2 h2 + rh, 2 w2 + rw]."""
    N, T2, H2, W2 = xs.shape[:4]
    v = xs[..., :8 * cin].reshape(N, T2, H2, W2, 2, 2, 2, cin)
    return v.permute(0, 7, 1, 4, 2, 5, 3, 6).reshape(N, cin, 2 * T2, 2 * H2, 2 * W2)


def _pads(dims, out_dims, k, stride, pad_lo):
    """(lo, hi) zero padding per dimension such that a VALID strided convolution of the padded input has out_dims."""
    return [(pl, (o - 1) * s + kk - d - pl) for d, o, kk, s, pl in zip(dims, out_dims, k, stride, pad_lo)]


def _fpad(pads):
    (tl, th), (hl, hh), (wl, wh) = pads
    return (wl, wh, hl, hh, tl, th)


def conv_grads(x, w, dz, k, stride, pad_lo, want_dx=True):
    """float64 x [N, Cin, T, H, W], w [Cout, Cin, *k], dz [N, Cout, OT, OH, OW] -> (dW, dx | None) of the zero-padded
    (pad_lo, and whatever the high side needs for dz's extent) strided convolution."""
    pads = _pads(x.shape[2:], dz.shape[2:], k, stride, pad_lo)
    xp = F.pad(x, _fpad(pads))
    dW = torch.nn.grad.conv3d_weight(xp, w.shape, dz, stride=stride)
    dx = None
    if want_dx:
        dxp = torch.nn.grad.conv3d_input(xp.shape, w, dz, stride=stride)
        (tl, _), (hl, _), (wl, _) = pads
        T, H, W = x.shape[2:]
        dx = dxp[:, :, tl:tl + T, hl:hl + H, wl:wl + W]
    return dW, dx


def entry_weight(e):
    """The fp16 filter of a stride-1 conv entry as [Cout, Cin, KT, KH, KW] (engine.pack_conv_weight: [Cout, taps, cin_pad],
    taps in (kt, kh, kw) order)."""
    KT, KH, KW = e["k"]
    w = e["w"][:, :, :e["x"].C]
    return w.reshape(w.shape[0], KT, KH, KW, w.shape[2]).permute(0, 4, 1, 2, 3)


def tags_of(e):
    return list(e["tag"]) if isinstance(e["tag"], list) else [e["tag"]]


def conv_entry(e, dys, loss_scale=1.0, want_dx=True):
    """Reference backward of one conv tape entry.  dys: the fp16 output gradients, one [N, T, H, W, C_i] tensor per output
    ([e["out"]] + e["extra_outs"]).  Returns a dict:
      dz    fp16 [N, T, H, W, sum C_i]  gradient w.r.t. the raw convolution output, rounded as the kernel rounds it;
      dres  fp32 [N, T, H, W, C] | None  what flows into the residual input (exact fp16 values);
      params list of (weight, dW, |dz|^T|x| bound, bias | None, db | None, sum|dz| bound | None) in the parameters' own
            layout, divided by loss_scale, for every output that has a parameter container (the s2d stem: the 7x7x7 weight);
      dx / dx_abs  float64 [N, T, H, W, Cin]: the input gradient and |dz| * |w| (None for the stem and without want_dx)."""
    outs = [e["out"]] + e["extra_outs"]
    scale = e["scale"]
    dzs, col = [], 0
    dres = None
    for o, dy in zip(outs, dys):
        sc = scale[col:col + o.C] if scale is not None else None
        dz, g = act_bwd(dy, act_view(o), sc, e["relu"])
        dzs.append(dz)
        if e["residual"] is not None:
            dres = g if dres is None else dres + g
        col += o.C
    dz = torch.cat(dzs, -1)
    dz64 = ncdhw(dz.double())
    inv = 1.0 / float(loss_scale)
    tag = e["tag"]
    if isinstance(tag, tuple) and tag[0] == "s2d":
        unit = tag[1]
        cin = unit.conv3d.in_channels
        x = unpack_s2d(act_view(e["x"]).double(), cin)
        k, stride = unit.kernel_size, unit.stride
        pad_lo = tuple((max(kk - s, 0)) // 2 for kk, s in zip(k, stride))
        shape = (dz.shape[-1], cin) + tuple(k)
        dW, _ = conv_grads(x, torch.zeros(shape, dtype=torch.float64, device=x.device), dz64, k, stride, pad_lo, False)
        bW, _ = conv_grads(x.abs(), torch.zeros(shape, dtype=torch.float64, device=x.device), dz64.abs(), k, stride, pad_lo, False)
        return dict(dz=dz, dres=dres, params=[(unit.conv3d.weight, dW * inv, bW * inv, None, None, None)], dx=None, dx_abs=None)
    x = ncdhw(act_view(e["x"]).double())
    w = entry_weight(e).double()
    dW, dx = conv_grads(x, w, dz64, e["k"], e["stride"], e["pad_lo"], want_dx)
    bW, bx = conv_grads(x.abs(), w.abs(), dz64.abs(), e["k"], e["stride"], e["pad_lo"], want_dx)
    params, row = [], 0
    for tg, o in zip(tags_of(e), outs):
        sl = slice(row, row + o.C)
        row += o.C
        if tg is None:
            continue
        conv = getattr(tg, "conv3d", tg)
        shp = conv.weight.shape
        db = bdb = None
        if conv.bias is not None:
            d = dz64[:, sl]
            db, bdb = d.sum((0, 2, 3, 4)) * inv, d.abs().sum((0, 2, 3, 4)) * inv
        params.append((conv.weight, dW[sl].reshape(shp) * inv, bW[sl].reshape(shp) * inv, conv.bias, db, bdb))
    return dict(dz=dz, dres=dres, params=params, dx=ndhwc(dx) if dx is not None else None,
                dx_abs=ndhwc(bx) if bx is not None else None)


def pool_entry(e, dy):
    """Reference backward of one max-pool tape entry: zero F.pad with the entry's pad_lo / pad_hi, then
    F.max_pool3d(ceil_mode=True), autograd in float64 on the CPU (ATen's rule: the first maximum in scan order wins, strict
    '>', a padded zero takes part and its gradient is dropped).  dy: fp16 [N, OT, OH, OW, C].  Returns (y, dx): the pooled
    values (to check the forward the backward is paired with) and dx, both channels-last float64 on the CPU."""
    x = ncdhw(act_view(e["x"]).detach().cpu().double()).contiguous().requires_grad_(True)
    pads = list(zip(e["pad_lo"], e["pad_hi"]))
    y = F.max_pool3d(F.pad(x, _fpad(pads)), e["k"], e["stride"], ceil_mode=True)
    y.backward(ncdhw(dy.detach().cpu().double()))
    return ndhwc(y.detach()), ndhwc(x.grad)
