"""Float64 reference of the backward of one tape entry (step_b200/engine.py: the dicts `engine.conv` and `engine.maxpool`
append to engine.TAPE), fed the same fp16 operands the kernels read: the fp16 activations `x`, the packed fp16 weights
`e["w"]`, the fp32 BatchNorm scale and the fp16 output gradient.  Only the accumulation order and the final fp16 rounding
of the kernels differ from it, so the tests can derive their tolerances instead of fitting them.

Convolutions go through torch.nn.grad in float64 on the zero-padded input (the SAME padding of i3dpt.py:14-31 is
asymmetric, so it is applied with F.pad); pools through autograd of F.pad + F.max_pool3d(ceil_mode=True) in float64 on the
CPU.  Never fp32 on the GPU: cuDNN convolutions default to TF32 there.

The second part holds the float64 references of the inference forward's launches (conv_fwd, exit_fwd, mean_mid, linear,
head_regress, roi_align; pool_entry's `y` for the pools), fed what the kernel read, with the magnitude terms their error
bounds are built from (tests/test_gpu_forward_layers.py derives the bounds), and check_fwd, the elementwise + bias check
of one fp16 convolution output.  roi_align_tol and roi_align_fma_tol bound the fp16 ROIAlign forward's packed-table and
fp32-FMA paths (tests/test_gpu_roi_fwd_edges.py).

The third part holds the references of train_step's launches outside the tape (tests/test_gpu_train_launches.py):
roi_align_bwd (the transpose of the ROIAlign matrix roi_align uses, built once by roi_align_terms / roi_align_matrix),
linear_bwd, head_losses and cls_loss, each with its bound derived in its docstring and a checker that applies it.
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


def check_fwd32(got, ref, xw, epi, n, what):
    """One fp32 SIMT convolution output (csrc/conv_simt.cu, fp32 storage) against its reference, elementwise:
        |got - ref| <= gamma_n |scale| (|x| |w|) + 3 u32 (|acc scale| + |shift| + |res|),   gamma_n = n u32 / (1 - n u32),
    n = taps x Cin: the accumulation is one fmaf chain of n terms (each rounding within u32 of a partial sum <= the abs
    sum), the epilogue's multiply and two additions round once each, ReLU is 1-Lipschitz and the store is exact.  xw / epi
    are conv_fwd's.  Returns the largest |err| / bound."""
    assert n * U32 < 0.5, (what, n)
    tol = n * U32 / (1.0 - n * U32) * xw.double() + 3.0 * U32 * epi.double()
    return _check_within(got, ref, tol, what)


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
ROI_CHUNK = 64                   # ROIs per batched matrix product of the ROIAlign references


def roi_frames(rois, roi_T=0, feat_T=0, t_start=0):
    """Feature frame of every ROI row: int(frame) (truncation, as the kernels' (int) cast), mapped to
    (f // roi_T) * feat_T + t_start + f % roi_T when roi_T > 0 (ROINet.pool_into's frame map).  int64 [R]."""
    b = rois[:, 0].to(torch.float32).trunc().to(torch.int64)
    return (b // roi_T) * feat_T + t_start + b % roi_T if roi_T > 0 else b


def roi_align_terms(rois, scale, ph, pw, H, W, sampling_ratio=0):
    """Every term of the legacy ROIAlign (aligned=False; adaptive grid ceil(roi / pooled) for sampling_ratio 0; samples
    outside [-1, extent] dropped; 4-tap bilinear; mean over the grid) of rois [R, 5] (frame, x1, y1, x2, y2) on H x W maps,
    on the rois' device.  Sample coordinates and tap weights are formed in fp32 in the kernels' operation order
    (csrc/roi_math.cuh roi_geometry / sample_coord / make_tap, which csrc/roi.cu and csrc/train.cu roi_align_bwd_frame
    share, oracle/step_oracle.c).  A clamped sample (past H-1 / W-1) keeps its duplicate taps of one pixel as separate terms, as
    the kernels add them.  ROIs are grouped by sampling grid so that each group is one batched tensor expression.
    Returns a list of groups dict(idx [G] int64 ROI rows, bin [S] int64, pix [G, S] int64 (-1: dropped sample),
    w [G, S] float64 holding the fp32 tap weights, count = gh * gw, grid = (gh, gw), bin_hw = the fp32 bin sizes [G] x 2),
    S = ph pw gh gw 4 in the kernels' (bin, iy, ix, tap) order."""
    f32 = torch.float32
    dev = rois.device
    r = rois.detach().to(f32)
    sc = torch.tensor(scale, dtype=f32, device=dev)
    sw, sh, ew, eh = (r[:, j] * sc for j in (1, 2, 3, 4))
    one = torch.ones((), dtype=f32, device=dev)
    rw, rh = torch.maximum(ew - sw, one), torch.maximum(eh - sh, one)
    bin_h = rh / torch.tensor(float(ph), dtype=f32, device=dev)
    bin_w = rw / torch.tensor(float(pw), dtype=f32, device=dev)
    if sampling_ratio > 0:
        gh_all = torch.full_like(bin_h, sampling_ratio, dtype=torch.int64)
        gw_all = gh_all
    else:
        gh_all, gw_all = torch.ceil(bin_h).to(torch.int64), torch.ceil(bin_w).to(torch.int64)   # ceilf(roi / pooled)

    def taps(start, bin_, grid, n_bins, extent):
        """[G, n_bins, grid]: low / high index, weights (hi, lo) along one axis, and validity."""
        p = torch.arange(n_bins, dtype=f32, device=dev).view(1, -1, 1)
        i = torch.arange(grid, dtype=f32, device=dev).view(1, 1, -1)
        s, b = start.view(-1, 1, 1), bin_.view(-1, 1, 1)
        c = (s + p * b) + ((i + 0.5) * b) / torch.tensor(float(grid), dtype=f32, device=dev)
        valid = (c >= -1.0) & (c <= float(extent))
        c = torch.where(c <= 0.0, torch.zeros_like(c), c)
        low = c.to(torch.int64)
        top = low >= extent - 1
        low = torch.where(top, torch.full_like(low, extent - 1), low)
        high = torch.where(top, low, low + 1)
        c = torch.where(top, low.to(f32), c)
        l_ = c - low.to(f32)
        return low, high, 1.0 - l_, l_, valid

    groups = []
    keys = torch.stack([gh_all, gw_all], 1).cpu()
    for gh, gw in sorted({(int(a), int(b)) for a, b in keys.tolist()}):
        idx = ((gh_all == gh) & (gw_all == gw)).nonzero().view(-1)
        G = idx.numel()
        yl, yh, hy, ly, vy = taps(sh[idx], bin_h[idx], gh, ph, H)          # [G, ph, gh]
        xl, xh, hx, lx, vx = taps(sw[idx], bin_w[idx], gw, pw, W)          # [G, pw, gw]
        e = lambda t: t.view(G, ph, 1, gh, 1)
        f = lambda t: t.view(G, 1, pw, 1, gw)
        ok = e(vy) & f(vx)
        pix = torch.stack([e(yl) * W + f(xl), e(yl) * W + f(xh), e(yh) * W + f(xl), e(yh) * W + f(xh)], -1)
        wts = torch.stack([e(hy) * f(hx), e(hy) * f(lx), e(ly) * f(hx), e(ly) * f(lx)], -1)
        ok = ok.unsqueeze(-1).expand_as(pix)
        pix = torch.where(ok, pix, torch.full_like(pix, -1)).reshape(G, -1)
        wts = torch.where(ok, wts, torch.zeros_like(wts)).double().reshape(G, -1)
        b_ = torch.arange(ph * pw, device=dev).view(ph, pw, 1, 1, 1).expand(ph, pw, gh, gw, 4).reshape(-1)
        groups.append(dict(idx=idx, bin=b_, pix=pix, w=wts, count=gh * gw, grid=(gh, gw), bin_hw=(bin_h[idx], bin_w[idx])))
    return groups


def roi_align_matrix(group, sel, nbins, npix):
    """The per-ROI matrices of rows `sel` of one roi_align_terms group: M [g, nbins, npix] float64 with
    M[bin, pix] = sum of the bin's tap weights on pix / count (the ROIAlign forward is out = M @ frame), and the number of
    taps behind each entry, [g, nbins, npix] float64.  Shared by roi_align and roi_align_bwd."""
    pix, w = group["pix"][sel], group["w"][sel]
    g = pix.shape[0]
    live = pix >= 0
    lin = group["bin"].view(1, -1) * npix + pix.clamp(min=0)
    M = torch.zeros((g, nbins * npix), dtype=torch.float64, device=pix.device)
    M.scatter_add_(1, lin, torch.where(live, w, torch.zeros_like(w)) / group["count"])
    n = torch.zeros_like(M)
    n.scatter_add_(1, lin, live.double())
    return M.view(g, nbins, npix), n.view(g, nbins, npix)


def _roi_chunks(groups, frames, K):
    """(group, row selection, ROI rows, frames) per chunk of <= ROI_CHUNK ROIs whose frame lies in [0, K)."""
    for gr in groups:
        fr = frames[gr["idx"]]
        keep = ((fr >= 0) & (fr < K)).nonzero().view(-1)
        for a in range(0, keep.numel(), ROI_CHUNK):
            sel = keep[a:a + ROI_CHUNK]
            yield gr, sel, gr["idx"][sel], fr[sel]


def roi_distinct_pixels(group, nbins):
    """Distinct pixels with a live tap per bin of every ROI of one roi_align_terms group: int64 [G, nbins].  The packed
    ROIAlign merges a bin's taps per pixel into a table of ROI_MERGED entries."""
    G = group["pix"].shape[0]
    p = group["pix"].view(G, nbins, -1).sort(-1).values
    first = torch.ones_like(p[..., :1], dtype=torch.bool)
    new = torch.cat([first, p[..., 1:] != p[..., :-1]], -1) & (p >= 0)
    return new.sum(-1)


def roi_samples_per_bin(groups, R):
    """gh * gw of every ROI row: int64 [R]."""
    spb = torch.zeros(R, dtype=torch.int64)
    for gr in groups:
        spb[gr["idx"].cpu()] = gr["count"]
    return spb


def roi_align_fma_tol(out_abs, spb):
    """The fp16 ROIAlign with fp32 FMAs (step_roi_align_fwd_nhwc exact=2, the table-less fallback of exact=0, and the
    direct form of the packed kernel): per sample the four taps w_k v_k are added into an fp32 accumulator by one fmaf each,
    with the weights w_k (1 / count) formed in fp32 (1 / count and the product each rounded once), then the sum is stored as
    fp16.  u32 = 2^-24.  The weight of a term is w / count (1 + d1)(1 + d2); each of the n = 4 spb fmaf rounds its result
    once, (1 + d); so every term of the sum carries at most n + 2 factors (1 + d), |d| <= u32, and the fp32 result is within
    gamma_(n+2) sum |w| |v| / count of the float64 value, gamma_k = k u32 / (1 - k u32) (about (4 spb + 2) u32; no
    underflow: the weights are >= 2^-61, far above fp32's normal range, and the fp32 subnormal spacing 2^-149 is below the
    absolute term).  The fp16 store rounds once more: at most half an fp16 ulp, <= 2^-11 |x| + 2^-25.  out_abs [R, ph, pw, C]
    the sum |w| |v| / count (roi_align's second output), spb [R] the samples per bin (roi_samples_per_bin)."""
    k = (4.0 * spb.double() + 2.0).view(-1, *([1] * (out_abs.dim() - 1)))
    gamma = k * U32 / (1.0 - k * U32)
    fp32 = gamma * out_abs
    return fp32 + 2.0 ** -11 * (out_abs + fp32) + 2.0 ** -25


def roi_align(feat, rois, scale, ph, pw, roi_T=0, feat_T=0, t_start=0, sampling_ratio=0, groups=None):
    """Float64 ROIAlign of channels-last frames feat [K, H, W, C] (roi_align_terms' rules; the weighted sums in float64),
    computed on feat's device.  rois [R, 5]; with roi_T > 0 the frame index f maps to (f // roi_T) * feat_T + t_start +
    f % roi_T.  groups: roi_align_terms' output, to evaluate a modified set of terms.  Returns (out, out of |feat|) as
    [R, ph, pw, C] on the CPU."""
    K, H, W, C = feat.shape
    dev = feat.device
    fd = feat.detach().double().reshape(K, H * W, C)
    rois = rois.detach().to(dev)
    R = rois.shape[0]
    out = torch.zeros(R, ph * pw, C, dtype=torch.float64, device=dev)
    out_abs = torch.zeros_like(out)
    if groups is None:
        groups = roi_align_terms(rois, scale, ph, pw, H, W, sampling_ratio)
    for gr, sel, rows, fr in _roi_chunks(groups, roi_frames(rois, roi_T, feat_T, t_start), K):
        M, _ = roi_align_matrix(gr, sel, ph * pw, H * W)
        x = fd[fr]
        out[rows] = torch.bmm(M, x)
        out_abs[rows] = torch.bmm(M, x.abs())
    return out.view(R, ph, pw, C).cpu(), out_abs.view(R, ph, pw, C).cpu()


def roi_align_bwd(grad, rois, scale, ph, pw, K, H, W, roi_T=0, feat_T=0, t_start=0, sampling_ratio=0, groups=None):
    """Float64 ROIAlign backward, the transpose of roi_align's per-ROI matrix: grad [R, ph, pw, C] (the values the kernel
    read, any dtype) -> grad_in [K, H, W, C] float64 with grad_in[frame(r)] += M_r^T grad[r], on grad's device.  ROIs whose
    (mapped) frame is outside [0, K) contribute nothing, as in the kernels.  groups: roi_align_terms' output, to evaluate a
    modified set of terms.  Returns (grad_in, mag, n): mag = sum over the terms of |g w / count| (float64), n [K, H, W, 1]
    the number of terms per pixel (every channel of a pixel has the same terms).

    Bound (roi_align_bwd_check), u32 = 2^-24: the kernels form each term as fl(fl(g w) / count) from the fp32 value of g
    and the fp32 weight w, within (1 + u32)^2 - 1 < 2.01 u32 of g w / count (no underflow: |g| >= 2^-24 or 0, w >= 2^-48
    or 0).  They add the n terms of an element and its initial value into one fp32 result in some order (per ROI, then
    per frame, then into grad_in); whatever the order, that is a tree of n additions, each within u32 of its result, and
    every partial sum is at most the sum of the absolute values: n u32 (1 + n u32) (sum |term| + |init|).  In total
    |got - init - ref| <= (n + 3) u32 (mag + |init|) for n <= 2^11, and an element with no term keeps its initial value
    bit for bit."""
    dev = grad.device
    R = grad.shape[0]
    C = grad.shape[-1]
    g = grad.detach().double().reshape(R, ph * pw, C)
    gin = torch.zeros(K, H * W, C, dtype=torch.float64, device=dev)
    mag = torch.zeros_like(gin)
    n = torch.zeros(K, H * W, 1, dtype=torch.float64, device=dev)
    rois = rois.detach().to(dev)
    if groups is None:
        groups = roi_align_terms(rois, scale, ph, pw, H, W, sampling_ratio)
    for gr, sel, rows, fr in _roi_chunks(groups, roi_frames(rois, roi_T, feat_T, t_start), K):
        M, cnt = roi_align_matrix(gr, sel, ph * pw, H * W)
        Mt = M.transpose(1, 2)
        gin.index_add_(0, fr, torch.bmm(Mt, g[rows]))
        mag.index_add_(0, fr, torch.bmm(Mt, g[rows].abs()))
        n.index_add_(0, fr, cnt.sum(1).unsqueeze(-1))
    return gin.view(K, H, W, C), mag.view(K, H, W, C), n.view(K, H, W, 1)


def roi_align_bwd_check(got, init, ref, mag, n, what="roi_align_bwd"):
    """got (the kernel's grad_in after the launch) against init (before it) + ref within (n + 3) u32 (mag + |init|)
    (roi_align_bwd derives it); elements with n == 0 equal init exactly.  Returns the largest |err| / bound."""
    got, init = got.double(), init.double()
    assert bool((n <= 2 ** 11).all()), (what, "more terms per element than the bound is derived for")
    touched = (n > 0).expand_as(got)
    same = (got == init) | touched
    if not bool(same.all()):
        i = int((~same).flatten().nonzero()[0])
        raise AssertionError("%s: an element without a term changed at flat %d: %r -> %r" % (
            what, i, float(init.flatten()[i]), float(got.flatten()[i])))
    err = (got - init - ref).abs()
    tol = (n + 3.0) * U32 * (mag + init.abs())
    ok = (err <= tol) | ~touched
    if not bool(ok.all()):
        i = int((err - tol).masked_fill(~touched, -1.0).flatten().argmax())
        raise AssertionError("%s: %d of %d elements out of bound; worst at flat %d: got %r init %r ref %r tol %r" % (
            what, int((~ok).sum()), ok.numel(), i, float(got.flatten()[i]), float(init.flatten()[i]), float(ref.flatten()[i]),
            float(tol.flatten()[i])))
    return float((err / tol.clamp(min=1e-300)).masked_fill(~touched, 0.0).max()) if bool(touched.any()) else 0.0


def roi_align_tol(out_abs, vmax):
    """The packed-half2 path (exact=0): per bin <= 16 merged pixels whose fp32 weights (sum of tap weights / count) are
    rounded to fp16 (2^-11 relative, 2^-25 absolute below the normal range) and summed with one rounding per half2 FMA
    (2^-11 of the running sum <= the abs sum, 2^-25 absolute): 17 x 2^-11 x sum |w| |v| + 16 x 2^-25 (1 + max |v|) + the
    fp32 merge (< 2^-20 relative)."""
    return (ROI_MERGED + 1) * 2.0 ** -11 * out_abs + 2.0 ** -20 * out_abs + ROI_MERGED * 2.0 ** -25 * (1.0 + vmax)


# ---- the launches of train_step outside the tape -----------------------------------------------------------------------
def linear_bwd(x, w, dy, init_dx=None):
    """Float64 backward of y = x w^T + b on what step_linear_small_n_bwd read: x [M, K] (fp16 | fp32), w [Nn, K] fp32,
    dy [M, Nn] fp32, init_dx [M, K] what dx accumulates onto (or None).  Returns dict(dx, dx_abs, dw, dw_abs, db, db_abs):
    the values and |dy| |w| (+ |init_dx|), |dy|^T |x|, sum |dy|.

    Bounds (linear_bwd_check): linear_bwd_dw_kernel forms dW[n, k] as an fmaf chain over the M rows in order and db[n] as a
    chain of M fp32 additions; linear_bwd_dx_kernel forms dx[m, k] as an fmaf chain over the Nn columns, starting from 0 or
    from dx when accumulating.  Each fmaf / addition rounds once, within u32 of its result, and every partial sum is at
    most the abs sum: a chain of s roundings errs by at most s u32 (1 + s u32) abs <= (s + 1) u32 abs for s <= 2^12
    (s = M for dW and db, Nn for dx; one more for a later fp32 addition of dx into another buffer)."""
    xd, wd, g = x.double(), w.double(), dy.double()
    dx = g @ wd
    dx_abs = g.abs() @ wd.abs()
    if init_dx is not None:
        dx = dx + init_dx.double()
        dx_abs = dx_abs + init_dx.double().abs()
    return dict(dx=dx, dx_abs=dx_abs, dw=g.t() @ xd, dw_abs=g.abs().t() @ xd.abs(), db=g.sum(0), db_abs=g.abs().sum(0))


def linear_bwd_check(got, ref, abs_, steps, what):
    """|got - ref| <= (steps + 1) u32 abs elementwise (linear_bwd derives it).  Returns the largest |err| / bound."""
    assert steps <= 2 ** 12, (what, steps)
    return _check_within(got, ref, (steps + 1) * U32 * abs_, what)


def _check_within(got, ref, tol, what):
    got, ref, tol = got.double(), ref.double().to(got.device), tol.double().to(got.device)
    err = (got - ref).abs()
    ok = err <= tol
    if not bool(ok.all()):
        i = int((err - tol).flatten().argmax())
        raise AssertionError("%s: %d of %d elements out of bound; worst at flat %d: got %r ref %r tol %r" % (
            what, int((~ok).sum()), ok.numel(), i, float(got.flatten()[i]), float(ref.flatten()[i]), float(tol.flatten()[i])))
    return float((err / tol.clamp(min=1e-300)).max()) if err.numel() else 0.0


# The loss bounds keep the first-order terms (u32 times a magnitude); this factor covers the neglected products of two such
# terms, each below 2^-12 of its magnitude for box coordinates below 2^10.
SECOND_ORDER = 1.0 + 2.0 ** -10


def _cls_terms(x, t):
    """Classification part of the loss bounds (cls_loss_pass), float64: x the logits, t = label * mask.
    loss l = (1 - t) x - (min(x, 0) - log1p(exp(-|x|))): expf errs by <= 2 ulp (4 u32 relative), log1pf by 1 ulp (2 u32)
    and carries expf's error scaled by e / (1 + e) <= log1p(e) / e * e, so L = log1pf(expf(-|x|)) is within 6 u32 L; four
    more roundings ((1 - t), * x, the two subtractions), each within u32 of A = |(1 - t) x| + |min(x, 0)| + L: 10 u32 A.
    gradient (sigmoid(x) - t) / (N cls): sg = 1 / (1 + expf(-x)) is within 6 u32 sg (expf's 4 u32 scaled by
    e / (1 + e) <= 1, two roundings) plus 2^-126 where expf(-x) overflows; sg - t, the fp32 1 / (N cls) and the product
    round three times more: (6 u32 sg + 3 u32 |sg - t| + 2^-126) / (N cls)."""
    L = torch.log1p(torch.exp(-x.abs()))
    A = ((1.0 - t) * x).abs() + torch.clamp(x, max=0.0).abs() + L
    sg = torch.sigmoid(x)
    return 10.0 * U32 * A, 6.0 * U32 * sg + 3.0 * U32 * (sg - t).abs() + 2.0 ** -126


def cls_loss(logits, targets):
    """Float64 reference of cls_loss_kernel on its fp32 inputs (oracle.model.two_branch_losses, cls_only): returns
    dict(loss [N cls] or the [1] zero without a classification sample, loss_tol, dlogits = d mean(loss) / d logits by
    float64 autograd, dlogits_tol) with _cls_terms' bounds times SECOND_ORDER."""
    from oracle.model import two_branch_losses
    x = logits.detach().double().cpu().requires_grad_(True)
    tg = targets.detach().double().cpu()
    N, cls = x.shape
    z = torch.zeros(N, 1, 4, dtype=torch.float64)
    lc, _, _ = two_branch_losses(x, z, z, z, torch.zeros(N, 1, 5, dtype=torch.float64), tg, 1, cls_only=True)
    t = tg[:, 1, 6:] * tg[:, 1, 4:5]
    lt, gt = _cls_terms(x.detach(), t)
    has = bool(tg[:, 1, 4].sum() != 0)
    if has:
        lc.mean().backward()
        g = x.grad
    else:
        g = torch.zeros_like(x)
    return dict(loss=lc.detach(), loss_tol=(lt.flatten() if has else torch.zeros(1, dtype=torch.float64)) * SECOND_ORDER,
                dlogits=g.detach(), dlogits_tol=(gt / (N * cls) if has else torch.zeros_like(g)) * SECOND_ORDER)


def _encode_terms(gt, anchor):
    """encode_one of csrc/tube_math.cuh (tube_utils.py:143-163) in float64 and its fp32 error bound, per [N, 4] row.
    With B = |c0| + |c2| + 1 per axis of a box (c0, c2 its two coordinates on the axis): the width fl(fl(c2 - c0) + 1) is
    within 2 u32 B, the centre fl(c0 + 0.5 w) within 2.5 u32 B < 3 u32 B.  (gx - ax) / aw: the difference within
    3 u32 (Bg + Ba) + u32 |num|, the division adds |enc| 2 u32 Ba / |aw| (the width) and u32 |enc|.  log(gw / aw): the ratio
    is within delta = 2 u32 Bg / |gw| + 2 u32 Ba / |aw| + u32 relative, which moves the log by delta; logf adds 1 ulp,
    2 u32 |enc|."""
    enc, err = [], []
    for lo, hi in ((0, 2), (1, 3)):
        gw, aw = gt[:, hi] - gt[:, lo] + 1.0, anchor[:, hi] - anchor[:, lo] + 1.0
        Bg, Ba = gt[:, lo].abs() + gt[:, hi].abs() + 1.0, anchor[:, lo].abs() + anchor[:, hi].abs() + 1.0
        num = (gt[:, lo] + 0.5 * gw) - (anchor[:, lo] + 0.5 * aw)
        e = num / aw
        enc.append(e)
        err.append((3.0 * U32 * (Bg + Ba) + U32 * num.abs()) / aw.abs() + e.abs() * 2.0 * U32 * Ba / aw.abs() + U32 * e.abs())
    for lo, hi in ((0, 2), (1, 3)):
        gw, aw = gt[:, hi] - gt[:, lo] + 1.0, anchor[:, hi] - anchor[:, lo] + 1.0
        Bg, Ba = gt[:, lo].abs() + gt[:, hi].abs() + 1.0, anchor[:, lo].abs() + anchor[:, hi].abs() + 1.0
        e = torch.log(gw / aw)
        enc.append(e)
        err.append(2.0 * U32 * Bg / gw.abs() + 2.0 * U32 * Ba / aw.abs() + U32 + 2.0 * U32 * e.abs())
    return torch.stack(enc, 1), torch.stack(err, 1)


def head_losses(logits, local_loc, first_loc, last_loc, tubes, targets, T, lambda_reg=5.0, lambda_neighbor=1.0):
    """Float64 reference of head_losses_kernel on its fp32 inputs: oracle.model.two_branch_losses, and float64 autograd of
    mean(loss_cls) + lambda_reg loss_loc + lambda_neighbor loss_nb.  The kernel adds d/d first_loc and d/d last_loc into
    d/d local_loc at the frames first_loc / last_loc are slices of (two_branch.py:265-270; head_chunks), so dlocal here is
    autograd's plus those two.  Returns dict of (value, tol) pairs: loss_cls, loss_loc, loss_nb, dlogits, dlocal, dfirst,
    dlast, each tol times SECOND_ORDER.

    Regression bounds, per coordinate of a tube (masks are 0 / 1, S their fp32 sum, exact below 2^24): d = fl(pred - enc)
    errs by E_d = E_enc + u32 |d| (_encode_terms); smooth-L1 and its derivative clamp(d, -1, 1) are continuous at |d| = 1 with
    slopes min(|d|, 1) and 1, so a branch flip near the boundary stays inside E_l = min(|d| + E_d, 1) E_d + u32 |l| and
    E_g = E_d; the gradient fl(fl(g m w) / S) adds two roundings: (w / S) E_g + 2 u32 |grad|; each addition of a first / last
    gradient into local_loc one more (u32 of the sum).  The loss sums 4N (8N for the neighbours) terms in tube order:
    sum E_l + 4N u32 sum |l| (8N), then / S: one rounding."""
    from oracle.model import two_branch_losses
    d64 = lambda t: t.detach().double().cpu()
    x = d64(logits).requires_grad_(True)
    loc, fst, lst = (d64(t).requires_grad_(True) for t in (local_loc, first_loc, last_loc))
    tb, tg = d64(tubes), d64(targets)
    N, cls = x.shape
    Tl, Tc = loc.shape[1], fst.shape[1]
    for j in range(3):
        assert bool(((tg[:, j, 4:6] == 0) | (tg[:, j, 4:6] == 1)).all()), "masks of 0 / 1 (the bound assumes exact products)"
    lc, ll, ln = two_branch_losses(x, loc, fst, lst, tb, tg, T)
    obj = lc.mean() + lambda_reg * ll.mean() + lambda_neighbor * ln.mean()
    gx, gl, gf, gla = (torch.zeros_like(t) for t in (x, loc, fst, lst))
    if obj.requires_grad:
        gs = torch.autograd.grad(obj, (x, loc, fst, lst), allow_unused=True)
        gx, gl, gf, gla = (g if g is not None else z for g, z in zip(gs, (gx, gl, gf, gla)))
    chunks = int(Tl / T)
    half = int(T / 2)
    centre, first_i, last_i = (chunks // 2) * T + half, half, (chunks - 1) * T + half
    s0, e0 = first_i - half, last_i - half
    dlocal = gl.clone()
    dlocal[:, s0:s0 + Tc] += gf
    dlocal[:, e0:e0 + Tc] += gla
    sums = gl.abs()
    sums[:, s0:s0 + Tc] += gf.abs()
    sums[:, e0:e0 + Tc] += gla.abs()
    # classification
    t = tg[:, 1, 6:] * tg[:, 1, 4:5]
    lt, gt_ = _cls_terms(x.detach(), t)
    has_cls = bool(tg[:, 1, 4].sum() != 0)
    out = dict(loss_cls=(lc.detach(), (lt.flatten() if has_cls else torch.zeros(1, dtype=torch.float64)) * SECOND_ORDER),
               dlogits=(gx, (gt_ / (N * cls) if has_cls else torch.zeros_like(gx)) * SECOND_ORDER))
    # regression: (target row, tube frame, prediction) of the centre, first and last terms
    terms = []
    for j, frame, pred in ((1, centre, loc[:, centre]), (0, first_i, fst[:, half]), (2, last_i, lst[:, half])):
        enc, e_enc = _encode_terms(tg[:, j, :4], tb[:, frame, 1:5])
        d = pred.detach() - enc
        E_d = e_enc + U32 * d.abs()
        ad = d.abs()
        l = torch.where(ad < 1.0, 0.5 * d * d, ad - 0.5)
        E_l = torch.minimum(ad + E_d, torch.ones_like(ad)) * E_d + U32 * l
        terms.append((tg[:, j, 5:6], l, E_l, E_d))
    grads_tol = {}
    for name, parts, lam in (("loss_loc", terms[:1], lambda_reg), ("loss_nb", terms[1:], lambda_neighbor)):
        S = sum(float(m.sum()) * 4 for m, _, _, _ in parts)
        if S == 0:
            out[name] = ((ll if name == "loss_loc" else ln).detach(), torch.zeros(1, dtype=torch.float64))
            grads_tol[name] = [torch.zeros_like(p[1]) for p in parts]
            continue
        sum_E = sum(float((E_l * m).sum()) for m, _, E_l, _ in parts)
        sum_l = sum(float((l * m).sum()) for m, l, _, _ in parts)
        v = (ll if name == "loss_loc" else ln).detach()
        out[name] = (v, ((sum_E + 4 * N * len(parts) * U32 * sum_l) / S + U32 * v.abs()) * SECOND_ORDER)
        # |grad| = (lambda / S) |clamp(d, -1, 1)| m <= (lambda / S) m
        grads_tol[name] = [(lam / S) * m * (E_d + 2.0 * U32) for m, _, _, E_d in parts]
    tl = torch.zeros_like(gl)
    tl[:, centre] = grads_tol["loss_loc"][0]
    tf, tla = torch.zeros_like(gf), torch.zeros_like(gla)
    tf[:, half] = grads_tol["loss_nb"][0]
    tla[:, half] = grads_tol["loss_nb"][1]
    tlocal = tl.clone()
    tlocal[:, s0:s0 + Tc] += tf
    tlocal[:, e0:e0 + Tc] += tla
    tlocal = tlocal + 2.0 * U32 * sums                               # the (up to two) additions of first / last into local
    out.update(dlocal=(dlocal, tlocal * SECOND_ORDER), dfirst=(gf, tf * SECOND_ORDER), dlast=(gla, tla * SECOND_ORDER))
    return out
