"""Host-side glue between the ported modules and the C ABI: the channels-last activation handle
(`Act`), weight packing / BatchNorm folding, and thin launch helpers.  No arithmetic happens here;
torch supplies device memory and the current stream only.
"""
import contextlib
import math
import os

import torch

from . import _lib as L

# Addressing mode of the fp16 implicit-GEMM for filters larger than 1x1x1 (include/step_b200.h a_mode):
# "box" = tiled TMA boxes with zero-filled halo, "im2col" = TMA im2col mode (dense M tiles; both are validated
# byte-for-byte by tests/test_gpu_conv.py::test_tma_tile_addressing), "halo" = input patch staged once in shared
# memory (csrc/conv_halo.cu), "best" (default) = halo where it measures faster (thin inputs on large maps), else im2col.
A_MODE = {"box": L.A_BOX, "im2col": L.A_IM2COL, "auto": L.A_AUTO, "simt": L.A_SIMT, "best": L.A_BEST}[
    os.environ.get("STEP_B200_AMODE", "best")]


# When set to a list, conv() appends (params, tensors-kept-alive) for every launch: bench.py replays
# exactly those launches to time the dominant kernel class in isolation (roofline.achieved).
RECORDER = None
# When set to a list, conv() and maxpool() append what the backward pass needs (step_b200/training.py): operands, outputs,
# geometry and the owning parameter container(s) (`tag`).  Activations stay alive through the tape.
TAPE = None
DEBUG_SYNC = os.environ.get("STEP_B200_DEBUG_SYNC", "0") == "1"
STEM_HALO = os.environ.get("STEP_B200_STEM_HALO", "1") != "0"


# Independent branches of an Inception block (models/i3dpt.py:157-163 runs them serially) are issued on
# side streams: at these shapes one branch often has < 148 tiles, so overlapping the four branches is what
# fills the SMs.  Under CUDA-graph capture the fork/join events become graph edges.
BRANCH_STREAMS = os.environ.get("STEP_B200_BRANCH_STREAMS", "1") != "0"
FUSE_1X1 = os.environ.get("STEP_B200_FUSE_1X1", "1") != "0"
_side_streams = {}


@contextlib.contextmanager
def recording(tape):
    """Set TAPE to `tape` for the block and restore TAPE and BRANCH_STREAMS on exit.  A list turns BRANCH_STREAMS off
    too, so that every launch runs on one stream and the tape order is the execution order; None only stops recording."""
    global TAPE, BRANCH_STREAMS
    saved = TAPE, BRANCH_STREAMS
    TAPE = tape
    if tape is not None:
        BRANCH_STREAMS = False
    try:
        yield tape
    finally:
        TAPE, BRANCH_STREAMS = saved


def side_streams(device, n=3):
    # keyed by the CALLER's stream too: a side stream then only ever runs work forked from (and joined back into) one
    # stream, so a block freed by the caller and re-used on the side stream is ordered behind the caller's consumer
    key = (device.type, device.index, torch.cuda.current_stream(device).cuda_stream)
    st = _side_streams.get(key)
    if st is None or len(st) < n:
        st = [torch.cuda.Stream(device=device) for _ in range(n)]
        _side_streams[key] = st
    return st[:n]


def run_parallel(device, main_fn, side_fns, first_side=0):
    """Run main_fn on the current stream and each side_fn on its own side stream; join before returning.
    first_side: index of the first side stream to use (nested calls must not share a stream)."""
    if not BRANCH_STREAMS or not side_fns:
        main_fn()
        for f in side_fns:
            f()
        return
    cur = torch.cuda.current_stream(device)
    fork = cur.record_event()
    streams = side_streams(device, first_side + len(side_fns))[first_side:]
    joins = []
    for st, f in zip(streams, side_fns):
        st.wait_event(fork)
        with torch.cuda.stream(st):
            f()
            joins.append(st.record_event())
    main_fn()
    for ev in joins:
        cur.wait_event(ev)


def torch_dtype(code):
    return torch.float16 if code == L.F16 else torch.float32


def dtype_code(fp16):
    env = os.environ.get("STEP_B200_PRECISION")
    if env:
        return {"fp16": L.F16, "fp32": L.F32}[env]
    return L.F16 if fp16 else L.F32


class Act:
    """A channel slice [coff, coff+C) of a channels-last buffer `buf` [N, T, H, W, ld]."""
    __slots__ = ("buf", "C", "coff")

    def __init__(self, buf, C=None, coff=0):
        assert buf.dim() == 5 and buf.is_contiguous()
        self.buf = buf
        self.C = buf.shape[4] - coff if C is None else C
        self.coff = coff

    @staticmethod
    def empty(N, T, H, W, C, code, device, ld=None):
        return Act(torch.empty((N, T, H, W, ld or C), dtype=torch_dtype(code), device=device), C, 0)

    N = property(lambda s: s.buf.shape[0])
    T = property(lambda s: s.buf.shape[1])
    H = property(lambda s: s.buf.shape[2])
    W = property(lambda s: s.buf.shape[3])
    ld = property(lambda s: s.buf.shape[4])
    code = property(lambda s: L.dt(s.buf))
    device = property(lambda s: s.buf.device)

    def slice(self, coff, C):
        return Act(self.buf, C, self.coff + coff)

    def data_ptr(self):
        return self.buf.data_ptr() + self.coff * self.buf.element_size()

    def logical(self):
        """[N, T, C, H, W] view (the reference's activation layout, networks.py:80-81)."""
        return self.buf[..., self.coff:self.coff + self.C].permute(0, 1, 4, 2, 3)

    def frames(self):
        """view as N*T images: Act [N*T, 1, H, W, ld] (Conv2d on frames, two_branch.py:258)."""
        return Act(self.buf.view(self.N * self.T, 1, self.H, self.W, self.ld), self.C, self.coff)


FUSE_EXIT = os.environ.get("STEP_B200_FUSE_EXIT", "1") != "0"


def bottleneck_exit(h, w3, x, w1, shift2, relu2, z, y=None):
    """step_bottleneck_exit_f16: y = relu(h * w3^T + x); z = act(y * w1^T + shift2) on frames Acts (rows = N*T*H*W).
    h [.., planes], x / y [.., inplanes], z [.., outplanes]; w3 / w1 packed 1x1 filters [Cout, 1, Cin] fp16."""
    L.same_device(h.buf, x.buf, z.buf, w3, w1)
    M = h.N * h.T * h.H * h.W
    args = (h.data_ptr(), h.ld, L.ptr(w3), x.data_ptr(), x.ld, L.ptr(w1), L.ptr(shift2) if shift2 is not None else None,
            1 if relu2 else 0, y.data_ptr() if y is not None else None, y.ld if y is not None else 0, z.data_ptr(), z.ld,
            M, h.C, x.C, z.C)
    L.check(L.lib().step_bottleneck_exit_f16(*args, L.stream()))
    if RECORDER is not None:   # (launch arguments, buffers kept alive, algorithmic bytes) for bench.py's replay of the conv class
        alg = 2 * (M * (h.C + x.C + z.C + (x.C if y is not None else 0)) + w3.numel() + w1.numel())
        RECORDER.append((("exit", args, alg), (h.buf, w3, x.buf, w1, shift2, y.buf if y is not None else None, z.buf)))
    return z


def can_fuse_exit(code, planes, inplanes, outplanes):
    """The fused kernel exists for the reference's head widths and the fp16 path; it does not record the per-layer tape
    entries the reverse pass walks, so the training forward keeps the two launches."""
    return FUSE_EXIT and TAPE is None and code == L.F16 and planes == 256 and inplanes == 1024 and outplanes == 256


def same_pad(k, s):
    """models/i3dpt.py:14-31 per dimension: (low, high)."""
    pad = max(k - s, 0)
    return pad // 2, pad - pad // 2


def same_out_dims(dims, k, stride):
    """Output extent of the reference's SAME emulation, i3dpt.py:14-31,95-98: pad max(k - s, 0) in total, then a
    VALID convolution -> (D + max(k - s, 0) - k) // s + 1 (= floor(D / s) for odd D when k > s, not ceil)."""
    return tuple((d + max(kk - s, 0) - kk) // s + 1 for d, kk, s in zip(dims, k, stride))


def pack_conv_weight(w, code, cin_pad=None):
    """[Cout, Cin, *k] (Conv3d / Conv2d layout) -> [Cout, taps, cin_pad] in the compute dtype."""
    Cout, Cin = w.shape[0], w.shape[1]
    taps = int(math.prod(w.shape[2:]))
    align = 8 if code == L.F16 else 4
    cin_pad = cin_pad or (Cin + align - 1) // align * align
    out = torch.zeros((Cout, taps, cin_pad), dtype=torch_dtype(code), device=w.device)
    out[:, :, :Cin] = w.detach().reshape(Cout, Cin, taps).permute(0, 2, 1).to(out.dtype)
    return out


def pack_stem_s2d(w):
    """7x7x7 stride-2 stem (i3dpt.py:184-189) as a 4x4x4 stride-1 filter over the space-to-depth
    clip: input index i = 2*o + k - 2 = 2*(o + q) + r  =>  k = 2*(q+1) + r, q in [-1,2], r in {0,1}.
    [64, 3, 7,7,7] -> [64, 64 taps (qt,qh,qw), 32 (rt,rh,rw,c + 8 zero)] fp16."""
    Cout, Cin = w.shape[0], w.shape[1]
    assert tuple(w.shape[2:]) == (7, 7, 7)
    w8 = torch.zeros((Cout, Cin, 8, 8, 8), dtype=torch.float32, device=w.device)
    w8[:, :, :7, :7, :7] = w.detach().float()
    w8 = w8.view(Cout, Cin, 4, 2, 4, 2, 4, 2).permute(0, 2, 4, 6, 3, 5, 7, 1)  # co, qt,qh,qw, rt,rh,rw, c
    out = torch.zeros((Cout, 64, 32), dtype=torch.float16, device=w.device)
    out[:, :, :8 * Cin] = w8.reshape(Cout, 64, 8 * Cin).to(torch.float16)
    return out


def fold_bn(bn, conv_bias, Cout, device):
    """BatchNorm3d(eval) (+ conv bias) -> per-channel (scale, shift) fp32: y = conv*scale + shift
    (i3dpt.py:105-108; eps = bn.eps)."""
    if bn is None:
        if conv_bias is None:
            return None, None
        return None, conv_bias.detach().float().contiguous()
    s = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
    b = bn.bias.detach().float() - bn.running_mean.detach().float() * s
    if conv_bias is not None:
        b = b + conv_bias.detach().float() * s
    return s.contiguous(), b.contiguous()


def params_key(*tensors):
    return tuple((t.data_ptr(), t._version, t.device, t.dtype) for t in tensors if t is not None)


# Whether a batch-statistics forward updates the BatchNorms' running statistics.  training.train_step turns it off to repeat
# a forward whose statistics the caller's own training-mode forward has already counted (train.py:266-269).
UPDATE_RUNNING_STATS = True


@contextlib.contextmanager
def running_stats_update(on):
    global UPDATE_RUNNING_STATS
    saved = UPDATE_RUNNING_STATS
    UPDATE_RUNNING_STATS = bool(on)
    try:
        yield
    finally:
        UPDATE_RUNNING_STATS = saved


def check_batch_stats_bn(bn):
    """The BatchNorm settings the batch-statistics kernels implement: an exponential running average (momentum) that is
    tracked, as the reference's BatchNorm3d defaults are."""
    if bn.momentum is None or not bn.track_running_stats:
        raise ValueError("BatchNorm with batch statistics needs track_running_stats=True and a momentum (got momentum=%r, "
                         "track_running_stats=%r): the cumulative average and untracked statistics are not implemented"
                         % (bn.momentum, bn.track_running_stats))


def _conv_batch_stats(x, w_packed, shift, outs, bns, k, stride, pad_lo, relu, a_mode, out_dims, zero_cin_last_kt, tag):
    """conv() for Unit3Dpy outputs whose BatchNorms normalise with batch statistics (bns: one BatchNorm3d per output of outs):
    the convolution writes z [M, sum C] with the identity epilogue (+ the conv bias `shift`), step_bn_stats forms each
    BatchNorm's statistics over z's column range (and, when UPDATE_RUNNING_STATS, updates its running statistics once), and
    one step_bn_apply writes y = relu(scale z + shift) to every output.  The tape entry also keeps z, mean, rstd and bns."""
    code, dev = x.code, x.device
    o0 = outs[0]
    n_total = sum(o.C for o in outs)
    z = Act.empty(o0.N, o0.T, o0.H, o0.W, n_total, code, dev)
    with recording(None):
        conv(x, w_packed, None, shift, z, k, stride, pad_lo, relu=False, a_mode=a_mode, out_dims=out_dims,
             zero_cin_last_kt=zero_cin_last_kt)
    M = o0.N * o0.T * o0.H * o0.W
    stats = torch.empty((4, n_total), dtype=torch.float32, device=dev)          # mean, rstd, scale, shift
    nbytes = L.lib().step_bn_stats_workspace_bytes(M, max(o.C for o in outs))
    ws = torch.empty((max(nbytes, 4) // 4,), dtype=torch.float32, device=dev)
    bn_stats = L.lib().step_bn_stats_f16 if code == L.F16 else L.lib().step_bn_stats_f32
    esz = z.buf.element_size()
    col = 0
    for o, bn in zip(outs, bns):
        check_batch_stats_bn(bn)
        upd = UPDATE_RUNNING_STATS
        at = lambda r, col=col: L.c_void_p(stats[r].data_ptr() + 4 * col)
        L.check(bn_stats(L.c_void_p(z.buf.data_ptr() + esz * col), n_total, M, o.C, L.ptr(bn.weight.detach()),
                         L.ptr(bn.bias.detach()), float(bn.eps), float(bn.momentum), L.ptr(bn.running_mean) if upd else None,
                         L.ptr(bn.running_var) if upd else None, at(0), at(1), at(2), at(3), L.ptr(ws), nbytes, L.stream()))
        if upd:
            # written in place by the kernel: the version bump re-keys the folded weights of a later eval-mode forward
            torch.autograd.graph.increment_version(bn.running_mean)
            torch.autograd.graph.increment_version(bn.running_var)
            bn.num_batches_tracked.add_(1)
        col += o.C
    ys = list(outs) + [None] * (3 - len(outs))
    splits = [o0.C, o0.C + (outs[1].C if len(outs) > 1 else 0)]
    bn_apply = L.lib().step_bn_apply_f16 if code == L.F16 else L.lib().step_bn_apply_f32
    L.check(bn_apply(L.c_void_p(z.buf.data_ptr()), n_total, M, n_total, L.ptr(stats[2]), L.ptr(stats[3]), 1 if relu else 0,
                     L.c_void_p(o0.data_ptr()), o0.ld, splits[0],
                     L.c_void_p(ys[1].data_ptr()) if ys[1] is not None else None, ys[1].ld if ys[1] is not None else 0, splits[1],
                     L.c_void_p(ys[2].data_ptr()) if ys[2] is not None else None, ys[2].ld if ys[2] is not None else 0, L.stream()))
    if TAPE is not None:
        TAPE.append(dict(kind="conv", x=x, w=w_packed, scale=None, out=o0, extra_outs=list(outs[1:]), k=tuple(k),
                         stride=tuple(stride), pad_lo=tuple(pad_lo), relu=bool(relu), residual=None, tag=tag, z=z,
                         mean=stats[0], rstd=stats[1], bn=list(bns)))
    return o0


def conv(x, w_packed, scale, shift, out, k, stride=(1, 1, 1), pad_lo=None, relu=True, residual=None,
         a_mode=None, out_dims=None, extra_outs=None, zero_cin_last_kt=0, tag=None, bn=None):
    """Launch step_conv3d_fwd: x (Act) * w_packed [Cout, taps, w_ld] -> out (Act slice).
    extra_outs: up to two more Act slices; output channels are then split [out.C | extra[0].C | extra[1].C]
    (horizontally fused 1x1x1 layers sharing the input).
    bn: None, or one BatchNorm3d per output that normalises with batch statistics (freeze_stats=False in training mode):
    scale must then be None, shift is the conv bias (or None), and there is no residual (_conv_batch_stats)."""
    code = x.code
    if bn is not None:
        if scale is not None or residual is not None or len(bn) != 1 + len(extra_outs or []):
            raise RuntimeError("conv: batch statistics take one BatchNorm per output, no folded scale and no residual")
        if pad_lo is None:
            pad_lo = tuple(same_pad(k[i], stride[i])[0] for i in range(3))
        return _conv_batch_stats(x, w_packed, shift, [out] + list(extra_outs or []), bn, k, stride, pad_lo, relu, a_mode,
                                 out_dims, zero_cin_last_kt, tag)
    if pad_lo is None:
        pad_lo = tuple(same_pad(k[i], stride[i])[0] for i in range(3))
    if out_dims is None:
        out_dims = same_out_dims((x.T, x.H, x.W), k, stride)
    p = L.step_conv_params()
    p.dtype = code
    p.N, p.T, p.H, p.W = x.N, x.T, x.H, x.W
    p.Cin, p.in_ld = x.C, x.ld
    p.Cout, p.out_ld, p.out_coff = out.C + sum(e.C for e in (extra_outs or [])), out.ld, out.coff
    if extra_outs:
        p.n_splits = len(extra_outs)
        edge = out.C
        for i, e in enumerate(extra_outs):
            p.split[i] = edge
            p.y_extra[i] = e.buf.data_ptr()
            p.ld_extra[i], p.coff_extra[i] = e.ld, e.coff
            edge += e.C
    p.KT, p.KH, p.KW = k
    p.ST, p.SH, p.SW = stride
    p.PT, p.PH, p.PW = pad_lo
    p.OT, p.OH, p.OW = out_dims
    p.relu = 1 if relu else 0
    p.w_ld = w_packed.shape[2]
    p.x = x.data_ptr()
    p.w = w_packed.data_ptr()
    p.scale = scale.data_ptr() if scale is not None else None
    p.shift = shift.data_ptr() if shift is not None else None
    if residual is not None:
        p.residual = residual.buf.data_ptr()
        p.res_ld, p.res_coff = residual.ld, residual.coff
    p.y = out.buf.data_ptr()
    p.zero_cin_last_kt = int(zero_cin_last_kt)
    p.a_mode = A_MODE if a_mode is None else a_mode
    if p.a_mode in (L.A_BOX, L.A_IM2COL, L.A_BEST) and k == (1, 1, 1):
        p.a_mode = L.A_AUTO
    assert (out.N, out.T, out.H, out.W) == (x.N,) + tuple(out_dims), "conv: output buffer shape mismatch"
    L.check(L.lib().step_conv3d_fwd(p, L.stream()))
    if DEBUG_SYNC:   # STEP_B200_DEBUG_SYNC=1: find the launch an asynchronous fault belongs to
        try:
            torch.cuda.synchronize()
        except Exception:
            print("conv fault:", {f: getattr(p, f) for f, _ in p._fields_ if isinstance(getattr(p, f), int)}, flush=True)
            raise
    if TAPE is not None:
        TAPE.append(dict(kind="conv", x=x, w=w_packed, scale=scale, out=out, extra_outs=list(extra_outs or []), k=tuple(k),
                         stride=tuple(stride), pad_lo=tuple(pad_lo), relu=bool(relu), residual=residual, tag=tag))
    if RECORDER is not None:
        RECORDER.append((p, (x.buf, w_packed, scale, shift, out.buf, residual.buf if residual is not None else None,
                             [e.buf for e in (extra_outs or [])])))
    return out


def pool_out(size, k, s):
    """Output extent of ConstantPad3d(TF-SAME) + MaxPool3d(ceil_mode=True) (i3dpt.py:114-126)."""
    lo, hi = same_pad(k, s)
    P = size + lo + hi
    o = -(-(P - k) // s) + 1
    if (o - 1) * s >= P:
        o -= 1
    return o, lo, hi


def maxpool(x, k, s, out=None):
    (ot, pt, ht), (oh, ph, hh), (ow, pw, hw) = (pool_out(d, kk, ss) for d, kk, ss in zip((x.T, x.H, x.W), k, s))
    if out is None:
        out = Act.empty(x.N, ot, oh, ow, x.C, x.code, x.device)
    L.check(L.lib().step_maxpool3d_fwd(L.c_void_p(x.data_ptr()), x.code, x.N, x.T, x.H, x.W, x.C, x.ld, k[0], k[1],
                                       k[2], s[0], s[1], s[2], pt, ph, pw, ht, hh, hw, ot, oh, ow,
                                       L.c_void_p(out.data_ptr()), out.ld, L.stream()))
    if TAPE is not None:
        TAPE.append(dict(kind="pool", x=x, out=out, k=tuple(k), stride=tuple(s), pad_lo=(pt, ph, pw), pad_hi=(ht, hh, hw)))
    return out


def mean_mid(x_ptr, code, A, B, P, C, ld, device, out_code=L.F32):
    """x [A, B, P, C] (pixel stride ld) -> [A, P*C] mean over B."""
    y = torch.empty((A, P * C), dtype=torch_dtype(out_code), device=device)
    L.check(L.lib().step_mean_mid(L.c_void_p(x_ptr), code, A, B, P, C, ld, L.ptr(y), out_code, L.stream()))
    return y


def linear_small_n(x, M, K, x_ld, w, bias, N, y=None, act=0, accumulate=False, row_map=None):
    if y is None:
        y = torch.empty((M, N), dtype=torch.float32, device=x.device)
    nbytes = L.lib().step_linear_small_n_workspace_bytes(M, K, N)
    ws = torch.empty((max(nbytes, 4) // 4,), dtype=torch.float32, device=x.device)
    L.check(L.lib().step_linear_small_n(L.ptr(x), L.dt(x), M, K, x_ld, L.ptr(w), L.ptr(bias), N, L.ptr(y),
                                        y.shape[1], act, 1 if accumulate else 0, L.ptr(row_map), L.ptr(ws), nbytes,
                                        L.stream()))
    return y
