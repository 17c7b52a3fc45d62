"""Float64 reference of the backward of one tape entry (step_b200/engine.py: the dicts `engine.conv` and `engine.maxpool`
append to engine.TAPE), fed the same fp16 operands the kernels read: the fp16 activations `x`, the packed fp16 weights
`e["w"]`, the fp32 BatchNorm scale and the fp16 output gradient.  Only the accumulation order and the final fp16 rounding
of the kernels differ from it, so the tests can derive their tolerances instead of fitting them.

Convolutions go through torch.nn.grad in float64 on the zero-padded input (the SAME padding of i3dpt.py:14-31 is
asymmetric, so it is applied with F.pad); pools through autograd of F.pad + F.max_pool3d(ceil_mode=True) in float64 on the
CPU.  Never fp32 on the GPU: cuDNN convolutions default to TF32 there.

The second half holds the float64 references of the inference forward's launches (conv_fwd, exit_fwd, mean_mid, linear,
head_regress, roi_align; pool_entry's `y` for the pools), fed what the kernel read, with the magnitude terms their error
bounds are built from (tests/test_gpu_forward_layers.py derives the bounds), and check_fwd, the elementwise + bias check
of one fp16 convolution output.
"""
import math

import torch
import torch.nn.functional as F

U32 = 2.0 ** -24                                            # fp32 unit roundoff
U12 = 2.0 ** -12


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


def packed_weight(w_packed, k, cin):
    """A packed filter [Cout, taps, w_ld] (engine.pack_conv_weight / pack_stem_s2d, taps in (kt, kh, kw) order) as
    [Cout, cin, KT, KH, KW]: the first cin channels of every tap, the ones the kernels read."""
    KT, KH, KW = k
    w = w_packed[:, :, :cin]
    return w.reshape(w.shape[0], KT, KH, KW, cin).permute(0, 4, 1, 2, 3)


def entry_weight(e):
    """The fp16 filter of a stride-1 conv entry as [Cout, Cin, KT, KH, KW]."""
    return packed_weight(e["w"], e["k"], e["x"].C)


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
    y = _pool(x, e["k"], e["stride"], e["pad_lo"], e["pad_hi"])
    y.backward(ncdhw(dy.detach().cpu().double()))
    return ndhwc(y.detach()), ndhwc(x.grad)


def _pool(x, k, stride, pad_lo, pad_hi):
    return F.max_pool3d(F.pad(x, _fpad(list(zip(pad_lo, pad_hi)))), k, stride, ceil_mode=True)


def pool_fwd(x, k, stride, pad_lo, pad_hi):
    """pool_entry's forward alone: x [N, T, H, W, C] -> the pooled values, channels-last float64 on the CPU."""
    return ndhwc(_pool(ncdhw(x.detach().cpu().double()), k, stride, pad_lo, pad_hi))


# ---- forward ------------------------------------------------------------------------------------------------------------
def conv_fwd(x, w_packed, scale, shift, residual, k, stride, pad_lo, out_dims, relu, widths=None):
    """Float64 reference of one step_conv3d_fwd launch on what it read: x fp16 [N, T, H, W, Cin] (the input channel slice),
    the packed fp16 filter, the fp32 folded scale / shift (or None), the fp16 residual [N, OT, OH, OW, Cout] (or None).
    Zero padding pad_lo below and whatever out_dims needs above, strided conv3d, * scale + shift + residual, ReLU.
    widths: channel counts of [out] + extra_outs (default: one output).  Returns three lists split like the outputs, each
    [N, OT, OH, OW, C_i] float64 channels-last:
      y    the result;
      xw   |scale| * (|x| * |w|), what the accumulation error scales with;
      epi  |acc * scale| + |shift| + |residual|, what the fp32 epilogue's roundings scale with."""
    cin = x.shape[-1]
    w = packed_weight(w_packed, k, cin).double()
    xd = ncdhw(x.double())
    pads = _fpad(_pads(xd.shape[2:], out_dims, k, stride, pad_lo))
    acc = F.conv3d(F.pad(xd, pads), w, stride=stride)
    mag = F.conv3d(F.pad(xd.abs(), pads), w.abs(), stride=stride)
    one = lambda v: v.double().view(1, -1, 1, 1, 1)
    s = one(scale) if scale is not None else torch.ones_like(acc[:1, :, :1, :1, :1])
    b = one(shift) if shift is not None else torch.zeros_like(s)
    z = acc * s + b
    epi = (acc * s).abs() + b.abs()
    if residual is not None:
        r = ncdhw(residual.double())
        z = z + r
        epi = epi + r.abs()
    y = torch.relu(z) if relu else z
    outs = [ndhwc(t) for t in (y, mag * s.abs(), epi)]
    widths = widths or [acc.shape[1]]
    cuts = [sum(widths[:i]) for i in range(len(widths) + 1)]
    return [[o[..., a:b_] for a, b_ in zip(cuts, cuts[1:])] for o in outs]


def conv_steps(k, cin):
    """wgmma k16 steps one output accumulates over: taps x ceil(cin / 16)."""
    return k[0] * k[1] * k[2] * -(-cin // 16)


def fwd_margin(xw, epi, extra=None):
    """m = 2^-12 |scale| (|x| |w|) + 2^-21 (|acc scale| + |shift| + |res|) (+ an inherited operand tolerance)."""
    m = U12 * xw + 2.0 ** -21 * epi
    return m if extra is None else m + extra


def fwd_tol(ref, m):
    """m plus half an fp16 ulp (round to nearest) at |ref| + m."""
    return m + 0.5 * ulp16(ref.abs() + m)


BIAS_DELTA = 2.0 ** -40          # failure probability of the bias check's rounding term (Hoeffding)


def check_fwd(got, ref, xw, epi, steps, what, extra=None):
    """One fp16 convolution output against its reference:
      elementwise |got - ref| <= m + 0.5 ulp16(|ref| + m);
      bias over the elements with |ref| >= 64 m: |mean((got - ref) sign(ref) / ulp16(ref))| <= the Hoeffding bound of n
      round-to-nearest errors in [-1/2, 1/2] plus the mean expected truncation loss steps * u32 * xw / ulp16(ref)
      (tests/test_gpu_forward_layers.py derives both).  Returns (n checked by the bias test, mean, threshold)."""
    got, ref = got.double(), ref.double()
    m = fwd_margin(xw, epi, extra)
    err = (got - ref).abs()
    tol = fwd_tol(ref, m)
    ok = err <= tol
    if not bool(ok.all()):
        i = int((err - tol).flatten().argmax())
        raise AssertionError("%s: %d of %d elements out of bound; worst at flat %d: got %r ref %r tol %r" % (
            what, int((~ok).sum()), ok.numel(), i, float(got.flatten()[i]), float(ref.flatten()[i]), float(tol.flatten()[i])))
    sel = ref.abs() >= 64.0 * m
    n = int(sel.sum())
    if n == 0:
        return 0, 0.0, 0.0
    u = ulp16(ref[sel])
    d = float(((got - ref)[sel] * ref[sel].sign() / u).mean())
    trunc = steps * U32 * xw[sel] + (extra[sel] if extra is not None else 0.0)
    thr = math.sqrt(math.log(2.0 / BIAS_DELTA) / (2.0 * n)) + float((trunc / u).mean())
    assert abs(d) <= thr, (what, "bias", n, d, thr)
    return n, d, thr


def exit_fwd(h, w3, x, w1, shift2, relu2):
    """Float64 reference of step_bottleneck_exit_f16 on rows: h fp16 [M, planes], w3 [inplanes, 1, planes], x fp16
    [M, inplanes], w1 [outplanes, 1, inplanes], shift2 fp32 [outplanes] | None.
      y = fp16(relu(h w3^T + x)),  z = act(y w1^T + shift2)   (act = ReLU if relu2, else identity).
    Returns dict(y, y_xw, y_epi, z, z_xw, z_epi, z_carry): y is the float64 value before its fp16 rounding; z is formed from
    fp16(y); z_carry = |w1| (m_y + ulp16(|y| + m_y)) bounds how far the kernel's y (within m_y + 1/2 ulp of the float64
    value) can sit from fp16(y) (another 1/2 ulp away), pushed through GEMM2."""
    hd, xd = h.double(), x.double()
    w3d, w1d = w3[:, 0].double(), w1[:, 0].double()
    a1 = hd @ w3d.t()
    y = torch.relu(a1 + xd)
    y_xw = hd.abs() @ w3d.abs().t()
    y_epi = a1.abs() + xd.abs()
    y16 = y.half().double()
    a2 = y16 @ w1d.t()
    b = shift2.double() if shift2 is not None else torch.zeros_like(a2[0])
    z = a2 + b
    z = torch.relu(z) if relu2 else z
    my = fwd_margin(y_xw, y_epi)
    carry = (my + ulp16(y.abs() + my)) @ w1d.abs().t()
    return dict(y=y, y_xw=y_xw, y_epi=y_epi, z=z, z_xw=y16.abs() @ w1d.abs().t(), z_epi=a2.abs() + b.abs(), z_carry=carry)


def mean_mid(x):
    """x [A, B, P, C] -> (mean over B, mean over B of |x|) as [A, P * C] float64."""
    xd = x.double()
    return xd.mean(1).flatten(1), xd.abs().mean(1).flatten(1)


def mean_mid_tol(ref, mabs, B):
    """step_mean_mid: fp32 sum over b in index order (B - 1 additions, each within u32 of a partial <= B mean|x|), one
    fp32 division by B (u32 of the quotient): (B - 1) u32 mean|x| + u32 (|ref| + that) <= B u32 mean|x| + u32 |ref|."""
    return B * U32 * mabs + U32 * ref.abs()


LIN_KC = 512                     # split-K chunk of step_linear_small_n / step_head_regress (csrc/pool_layout.cu kLinKC)


def linear(x, w, bias=None, y0=None, row_map=None, act=0):
    """Float64 step_linear_small_n: v = x[row_map] w^T + bias (+ y0 when accumulating), then sigmoid if act == 1.
    Returns (y, v, |x| |w|^T + |bias| + |y0|)."""
    xd = x.double()
    if row_map is not None:
        xd = xd[row_map.long()]
    wd = w.double()
    v = xd @ wd.t()
    a = xd.abs() @ wd.abs().t()
    for t in (bias, y0):
        if t is not None:
            v = v + t.double()
            a = a + t.double().abs()
    return (torch.sigmoid(v) if act == 1 else v), v, a


def linear_ops(K):
    """fp32 roundings an output of the split-K linear sees, each within u32 of the abs sum: inside a 512-column chunk
    2 u32 per k16 mma step (32 steps: 64 u32; the fp32 SIMT path has 16 FMAs + 5 shuffle adds per lane, fewer), then one
    addition per chunk in fixed order, the bias and the accumulate."""
    return 2 * (LIN_KC // 16) + -(-K // LIN_KC) + 2


def linear_tol(y, a, K, act):
    """linear_ops(K) u32 |x||w| before the activation; the sigmoid is 1/4-Lipschitz and 1 / (1 + expf(-v)) adds expf's
    2 ulp (2^-22 relative) and two fp32 roundings: < 2^-21 |y|."""
    pre = linear_ops(K) * U32 * a
    return pre / 4.0 + 2.0 ** -21 * y.abs() if act == 1 else pre


def head_chunks(Tc, T):
    """(s0, s1, e0, e1) of two_branch.py:263-270: the frames first_loc and last_loc cover."""
    half = int(Tc / 2)
    chunks = int(T / Tc)
    s0, s1 = max(int(Tc / 2) - half, 0), min(int(Tc / 2) + half + 1, T)
    e0 = max((chunks - 1) * Tc + int(Tc / 2) - half, 0)
    e1 = min((chunks - 1) * Tc + int(Tc / 2) + half + 1, T)
    return s0, s1, e0, e1


def head_regress(feat, local_reg, neighbor_reg1, neighbor_reg2, Tc, T, wdtype=torch.float16):
    """Float64 local_reg / neighbor_reg1 / neighbor_reg2 (two_branch.py:261-270) from the modules' own nn.Linear weights in
    the reference's (c, h, w) flattening: feat [R * T, ps, ps, C] channels-last (the downsample2 output), weights rounded to
    the kernel's dtype.  Returns dict(local [R, T, 4], first, last, and their tolerances): local within linear_ops u32
    |x||w|, first / last = local + neighbour within the sum of the two tolerances plus one fp32 rounding of the sum."""
    RT = feat.shape[0]
    R = RT // T
    x = ncdhw(feat.unsqueeze(1).double())[:, :, 0].reshape(RT, -1)       # [R T, C * ps * ps], column c * ps^2 + p
    outs, tols = [], []
    for m in (local_reg, neighbor_reg1, neighbor_reg2):
        w = m.weight.detach().to(wdtype).double()
        v = x @ w.t() + m.bias.detach().double()
        a = x.abs() @ w.abs().t() + m.bias.detach().double().abs()
        outs.append(v.view(R, T, 4))
        tols.append((linear_ops(x.shape[1]) * U32 * a).view(R, T, 4))
    s0, s1, e0, e1 = head_chunks(Tc, T)
    first, last = outs[0] + outs[1], outs[0] + outs[2]
    tf = tols[0] + tols[1] + U32 * first.abs()
    tl = tols[0] + tols[2] + U32 * last.abs()
    return dict(local=outs[0], local_tol=tols[0], first=first[:, s0:s1], first_tol=tf[:, s0:s1], last=last[:, e0:e1],
                last_tol=tl[:, e0:e1])


ROI_MERGED = 16                  # most distinct pixels one bin of the packed ROIAlign merges (csrc/roi.cu kMaxMerged)


def roi_align(feat, rois, scale, ph, pw, roi_T=0, feat_T=0, t_start=0):
    """Float64 ROIAlign (legacy sampling, sampling_ratio 0: adaptive grid ceil(roi / pooled), samples outside [-1, H]
    dropped, 4-tap bilinear, mean over the grid) of channels-last frames feat [K, H, W, C], on the CPU.  Sample coordinates
    and tap weights are formed in fp32 in the kernel's operation order (csrc/roi.cu roi_geometry / sample_coord /
    make_tap, oracle/step_oracle.c), the weighted sums in float64.  rois [R, 5] (frame, x1, y1, x2, y2); with roi_T > 0 the
    frame index f maps to (f // roi_T) * feat_T + t_start + f % roi_T.  Returns (out, out of |feat|) as [R, ph, pw, C]."""
    f32 = torch.float32
    K, H, W, C = feat.shape
    fd = feat.detach().cpu().double()
    rois = rois.detach().cpu().to(f32)
    R = rois.shape[0]
    out = torch.zeros(R, ph * pw, C, dtype=torch.float64)
    out_abs = torch.zeros_like(out)
    sc = torch.tensor(scale, dtype=f32)
    one = torch.tensor(1.0, dtype=f32)

    def taps(start, bin_, grid, n_bins, extent):
        """per (bin, sample): low / high index and weights (lo, hi) along one axis, and validity."""
        p = torch.arange(n_bins, dtype=f32).view(-1, 1)
        i = torch.arange(grid, dtype=f32).view(1, -1)
        c = (start + p * bin_) + ((i + 0.5) * bin_) / torch.tensor(float(grid), dtype=f32)
        valid = (c >= -1.0) & (c <= float(extent))
        c = torch.where(c <= 0.0, torch.zeros_like(c), c)
        low = c.to(torch.int64)
        top = low >= extent - 1
        low = torch.where(top, torch.full_like(low, extent - 1), low)
        high = torch.where(top, low, low + 1)
        c = torch.where(top, low.to(f32), c)
        l_ = c - low.to(f32)
        return low, high, one - l_, l_, valid

    for r in range(R):
        b = int(rois[r, 0])
        frame = (b // roi_T) * feat_T + t_start + b % roi_T if roi_T > 0 else b
        sw, sh, ew, eh = (rois[r, j] * sc for j in (1, 2, 3, 4))
        rw, rh = torch.maximum(ew - sw, one), torch.maximum(eh - sh, one)
        bin_h, bin_w = rh / torch.tensor(float(ph), dtype=f32), rw / torch.tensor(float(pw), dtype=f32)
        gh, gw = int(torch.ceil(rh / float(ph))), int(torch.ceil(rw / float(pw)))
        yl, yh, hy, ly, vy = taps(sh, bin_h, gh, ph, H)                 # [ph, gh]
        xl, xh, hx, lx, vx = taps(sw, bin_w, gw, pw, W)                 # [pw, gw]
        # every (p, q, iy, ix) sample: four pixels with fp32 weights hy hx, hy lx, ly hx, ly lx
        e = lambda t: t.view(ph, 1, gh, 1)
        f = lambda t: t.view(1, pw, 1, gw)
        ok = (e(vy) & f(vx)).double()
        pix = [e(yl) * W + f(xl), e(yl) * W + f(xh), e(yh) * W + f(xl), e(yh) * W + f(xh)]
        wts = [e(hy) * f(hx), e(hy) * f(lx), e(ly) * f(hx), e(ly) * f(lx)]
        M = torch.zeros(ph * pw, H * W, dtype=torch.float64)
        rows = torch.arange(ph * pw).view(ph, pw, 1, 1).expand(ph, pw, gh, gw)
        for p_, w_ in zip(pix, wts):
            M.index_put_((rows.reshape(-1), p_.expand(ph, pw, gh, gw).reshape(-1)),
                         (w_.double() * ok).expand(ph, pw, gh, gw).reshape(-1), accumulate=True)
        M /= gh * gw
        fr = fd[frame].reshape(H * W, C)
        out[r] = M @ fr
        out_abs[r] = M @ fr.abs()
    return out.view(R, ph, pw, C), out_abs.view(R, ph, pw, C)


def roi_align_tol(out_abs, vmax):
    """The packed-half2 path (exact=0): per bin <= 16 merged pixels whose fp32 weights (sum of tap weights / count) are
    rounded to fp16 (2^-11 relative, 2^-25 absolute below the normal range) and summed with one rounding per half2 FMA
    (2^-11 of the running sum <= the abs sum, 2^-25 absolute): 17 x 2^-11 x sum |w| |v| + 16 x 2^-25 (1 + max |v|) + the
    fp32 merge (< 2^-20 relative)."""
    return (ROI_MERGED + 1) * 2.0 ** -11 * out_abs + 2.0 ** -20 * out_abs + ROI_MERGED * 2.0 ** -25 * (1.0 + vmax)
