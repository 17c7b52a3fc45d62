"""Exact replays, in float64 arithmetic, of the fp32 forward kernels whose operation order is fixed: the SIMT convolution
(csrc/conv_simt.cu conv3d_simt_kernel, both storage types) and the fp32 temporal / spatial mean (csrc/pool_layout.cu
mean_mid_kernel<float, float>).  Each returns the bits the launch must have written, so a test can require torch.equal on
every output instead of a tolerance loose by about sqrt(n).

conv3d_simt_kernel, as its SASS for sm_90a shows (conv_simt.cu is compiled with FMA contraction, it is not in
step_b200/build.py NO_FMAD):
  * main loop: every output is one sequential fmaf chain over the filter taps in (t, h, w) order, then the 16-channel
    blocks, then k = 0..15 inside a block; a padded tap or a channel at or past Cin contributes fmaf(0, w, acc) == acc
    (acc starts at +0 and never becomes -0, and the operands are finite), so the chain is the taps x Cin products in
    (tap, channel) order;
  * epilogue, not contracted: a predicated FMUL (scale), FADD (shift), FADD (residual) and FMNMX with 0 (ReLU), each
    rounded on its own; then the store: the fp32 value, or its __half round-to-nearest.
fma32 is a correctly rounded fp32 fused multiply-add: the product of two fp32 values is exact in float64, TwoSum gives the
sum as s + e exactly, s is rounded to odd with e (53 bits), and rounding that to fp32 (24 bits) is correctly rounded
(round-to-odd at p + 2 or more bits followed by round-to-nearest is a single correct rounding).  All of it runs on the
operands' device; CUDA's float64 add / multiply and the float64 -> fp32 conversion are IEEE round-to-nearest-even, as on
the CPU.
"""
import torch

ROW_CHUNK = 8192                 # output pixels per vectorised replay pass (bounds the gathered operand tensor)


def _d(t, like):
    if torch.is_tensor(t):
        return t.to(device=like.device, dtype=torch.float64)
    return torch.tensor(float(t), dtype=torch.float64, device=like.device)


def _fma32_d(a, b, c):
    """fma32 on float64 tensors holding fp32 values; returns float64 holding the fp32 result."""
    p = a * b                                               # exact: 24 + 24 significant bits, exponent in range
    s = p + c
    bb = s - p                                              # TwoSum: s + e == p + c exactly
    e = (p - (s - bb)) + (c - bb)
    e = torch.where(torch.isfinite(s), e, torch.zeros_like(e))
    even = (s.view(torch.int64) & 1) == 0
    toward = torch.where(e > 0, torch.full_like(s, float("inf")), torch.full_like(s, float("-inf")))
    s = torch.where((e != 0) & even, torch.nextafter(s, toward), s)   # round to odd
    return s.float().double()


def fma32(a, b, c):
    """Correctly rounded fp32 fmaf(a, b, c) of fp32 values (tensors or numbers, broadcast), computed in float64 on the
    operands' device.  Returns float32."""
    like = next((t for t in (a, b, c) if torch.is_tensor(t)), torch.zeros(()))
    return _fma32_d(_d(a, like), _d(b, like), _d(c, like)).float()


def _taps(k):
    KT, KH, KW = k
    return [(kt, kh, kw) for kt in range(KT) for kh in range(KH) for kw in range(KW)]


def conv_rows(rows, out_dims):
    """Flat output pixels m (int64 tensor) -> (n, ot, oh, ow), the kernel's decomposition."""
    OT, OH, OW = out_dims
    ow = rows % OW
    r = rows // OW
    oh = r % OH
    r = r // OH
    return r // OT, r % OT, oh, ow


def gather_patches(x, rows, k, stride, pad_lo, out_dims):
    """The operands the kernel's A loader reads for output pixels `rows`: x [N, T, H, W, Cin] -> float64 [R, taps, Cin]
    in (t, h, w) tap order, zero where the tap falls into the padding."""
    N, T, H, W, Cin = x.shape
    n, ot, oh, ow = conv_rows(rows, out_dims)
    out = torch.zeros((rows.numel(), len(_taps(k)), Cin), dtype=torch.float64, device=x.device)
    for j, (kt, kh, kw) in enumerate(_taps(k)):
        it = ot * stride[0] + kt - pad_lo[0]
        ih = oh * stride[1] + kh - pad_lo[1]
        iw = ow * stride[2] + kw - pad_lo[2]
        ok = (it >= 0) & (it < T) & (ih >= 0) & (ih < H) & (iw >= 0) & (iw < W)
        idx = ok.nonzero().view(-1)
        if idx.numel():
            out[idx, j] = x[n[idx], it[idx], ih[idx], iw[idx]].double()
    return out


def touches_padding(rows, dims, k, stride, pad_lo, out_dims):
    """bool per output pixel: its window reaches outside the input in some dimension."""
    _, ot, oh, ow = conv_rows(rows, out_dims)
    hit = torch.zeros_like(rows, dtype=torch.bool)
    for o, d, kk, s, pl in zip((ot, oh, ow), dims, k, stride, pad_lo):
        lo = o * s - pl
        hit |= (lo < 0) | (lo + kk > d)
    return hit


def simt_conv_replay(x, w_packed, scale, shift, residual, k, stride, pad_lo, out_dims, relu, rows=None,
                     dtype=torch.float32):
    """What conv3d_simt_kernel writes, bit for bit, with R.conv_fwd's arguments: x [N, T, H, W, Cin] (the input channel
    slice, fp32 or fp16), w_packed [Cout, taps, w_ld], scale / shift fp32 [Cout] or None, residual [N, OT, OH, OW, Cout]
    (the residual channel slice) or None.  rows: int64 flat output pixels (default all, N * OT * OH * OW).  dtype: the
    storage type (torch.float32 or torch.float16).  Returns [len(rows), Cout] in dtype on x's device."""
    N, Cin = x.shape[0], x.shape[-1]
    Cout = w_packed.shape[0]
    dev = x.device
    M = N * out_dims[0] * out_dims[1] * out_dims[2]
    if rows is None:
        rows = torch.arange(M, device=dev)
    rows = rows.to(dev)
    w = w_packed[:, :, :Cin].to(dev).double()                # [Cout, taps, Cin]
    taps = w.shape[1]
    assert taps == k[0] * k[1] * k[2], (taps, k)
    sc = scale.to(dev).double().view(1, -1) if scale is not None else None
    sh = shift.to(dev).double().view(1, -1) if shift is not None else None
    res = residual.reshape(M, Cout) if residual is not None else None
    out = torch.empty((rows.numel(), Cout), dtype=dtype, device=dev)
    for a in range(0, rows.numel(), ROW_CHUNK):
        rs = rows[a:a + ROW_CHUNK]
        xg = gather_patches(x, rs, k, stride, pad_lo, out_dims)
        acc = torch.zeros((rs.numel(), Cout), dtype=torch.float64, device=dev)
        for t in range(taps):
            for c in range(Cin):
                acc = _fma32_d(xg[:, t, c:c + 1], w[:, t, c].view(1, -1), acc)
        v = acc
        if sc is not None:
            v = (v * sc).float().double()
        if sh is not None:
            v = (v + sh).float().double()
        if res is not None:
            v = (v + res[rs.to(res.device)].to(dev).double()).float().double()
        if relu:
            v = torch.clamp_min(v, 0.0)
        out[a:a + ROW_CHUNK] = v.to(dtype)
    return out


def mean_mid_replay(x):
    """mean_mid_kernel<float, float>: x fp32 [A, B, P, C] -> [A, P * C] fp32: B fp32 additions in index order starting
    from 0, then one fp32 division by B.  The divisor is a tensor: torch divides a CUDA tensor by a Python scalar as a
    multiplication by its reciprocal, which rounds twice."""
    s = torch.zeros_like(x[:, 0])
    for b in range(x.shape[1]):
        s = s + x[:, b]                                     # fp32 tensors: one IEEE rounding per addition
    return (s / torch.full_like(s, float(x.shape[1]))).flatten(1)
