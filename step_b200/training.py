"""The training step on the device (SURVEY.md section 8f rank 1; the reference: train.py:263-348).

What exists: the head's three losses and the gradient of the training objective with respect to the head outputs
(`head_losses`), the backward of the head's small-N linears (`linear_backward`), a deterministic channels-last ROIAlign
backward (`roi_align_backward_nhwc`, and `roi_align_backward_slice` for the temporal slices of train.py:294-309), its
ROIPool counterpart through the recorded maxima (`roi_pool_backward_slice`), the
tensor-core weight gradient of the convolutions, max-pool backward, the backward of the whole head including the context
columns of `global_cls` (`head_forward_backward`), of ContextNet (`context_forward` / `context_backward`) and of the I3D
trunk (`trunk_forward_backward`), the SGD update with the gradient all-reduce (`sgd_step`) and the whole step in spatial
and temporal mode with or without the context branch (`train_step`), which can also update through the optimizers of
`optim` with dynamic loss scaling.  The backward walks the tape the modules' forward records; the trunk's, ContextNet's
and the head's are split into forward and backward halves (trunk_forward / trunk_backward, context_forward /
context_backward, head_forward / head_backward, with head_outputs_backward for any upstream gradients of the head's
outputs), which train_step calls in order and the modules' torch.autograd Functions (step_b200/autograd.py) call from
autograd's backward.
Every piece runs on both precision paths of the modules (cfg.fp16): fp16 activations and activation gradients with the
tensor-core weight gradient, or fp32 storage throughout (the reference's default precision) with the fp32 SIMT kernels and
`conv_wgrad_f32`.  Weight gradients are fp32 on both.
"""
import contextlib
import ctypes

import torch

from . import _lib as L


def head_losses(logits, local_loc, first_loc, last_loc, tubes, targets, T, lambda_reg=5.0, lambda_neighbor=1.0,
                want_grads=False):
    """models/two_branch.py:276-333 on the device.  logits [N,cls] (pre-sigmoid), local_loc [N,T',4],
    first_loc / last_loc [N,Tc,4], tubes [N,T',5], targets [N,3,6+cls].
    Returns (loss_global_cls, loss_local_loc, loss_neighbor_loc) shaped like the reference's `.view(-1)` outputs
    (loss_global_cls is the element-wise BCE [N*cls], or the scalar 0 when no sample is positive) and, with
    want_grads, a dict with the gradients of  mean(loss_cls) + lambda_reg * loss_loc + lambda_neighbor * loss_nb
    (train.py:335-336; scripts/train_step.sh:43-44) w.r.t. logits / local_loc / first_loc / last_loc."""
    dev = L.same_device(logits, local_loc, first_loc, last_loc, tubes, targets)
    f32 = lambda t: t.detach().to(torch.float32).contiguous()
    logits, local_loc, first_loc, last_loc, tubes, targets = map(f32, (logits, local_loc, first_loc, last_loc, tubes, targets))
    N, cls = logits.shape
    T_len, Tc = local_loc.shape[1], first_loc.shape[1]
    if targets.shape != (N, 3, 6 + cls) or tubes.shape != (N, T_len, 5):
        raise RuntimeError("head_losses: targets %s / tubes %s do not match N=%d, T'=%d, classes=%d"
                           % (tuple(targets.shape), tuple(tubes.shape), N, T_len, cls))
    with torch.cuda.device(dev):
        loss_cls = torch.empty((N * cls,), dtype=torch.float32, device=dev)
        loss_loc = torch.empty((1,), dtype=torch.float32, device=dev)
        loss_nb = torch.empty((1,), dtype=torch.float32, device=dev)
        flags = torch.empty((3,), dtype=torch.int32, device=dev)
        scratch = torch.empty((N * 12,), dtype=torch.float32, device=dev)
        g = None
        if want_grads:
            g = {"logits": torch.empty_like(logits), "local_loc": torch.empty_like(local_loc),
                 "first_loc": torch.empty_like(first_loc), "last_loc": torch.empty_like(last_loc)}
        L.check(L.lib().step_head_losses_f32(L.ptr(logits), L.ptr(local_loc), L.ptr(first_loc), L.ptr(last_loc), L.ptr(tubes),
                                             L.ptr(targets), N, cls, T_len, int(T), Tc, float(lambda_reg), float(lambda_neighbor),
                                             L.ptr(loss_cls), L.ptr(loss_loc), L.ptr(loss_nb), L.ptr(flags),
                                             L.ptr(g["logits"]) if g else None, L.ptr(g["local_loc"]) if g else None,
                                             L.ptr(g["first_loc"]) if g else None, L.ptr(g["last_loc"]) if g else None,
                                             L.ptr(scratch), L.stream()))
        # `if mask.sum():` in the reference is the same host read-back (two_branch.py:293)
        if int(flags[0].item()) == 0:
            loss_cls = torch.zeros((1,), dtype=torch.float32, device=dev)
    return (loss_cls, loss_loc, loss_nb) if not want_grads else (loss_cls, loss_loc, loss_nb, g)


def cls_loss(logits, targets, want_grads=False):
    """The loss of a class-only head (TwoBranchNet(cls_only=True), models/two_branch.py:291-297) on the device: logits
    [N,cls] (pre-sigmoid), targets [N,3,6+cls] (train_cls.py:260-297 tiles one frame three times; the centre row is read).
    Returns loss_cls, the element-wise BCE [N*cls] or the [1] zero of the reference when no row has the classification flag,
    and with want_grads also d mean(loss_cls) / d logits [N,cls] (zeros in that case).  Bit for bit the classification part
    of `head_losses`."""
    dev = L.same_device(logits, targets)
    logits = logits.detach().to(torch.float32).contiguous()
    targets = targets.detach().to(torch.float32).contiguous()
    N, cls = logits.shape
    if targets.shape != (N, 3, 6 + cls):
        raise RuntimeError("cls_loss: targets %s do not match N=%d, classes=%d" % (tuple(targets.shape), N, cls))
    with torch.cuda.device(dev):
        loss_cls = torch.empty((N * cls,), dtype=torch.float32, device=dev)
        flags = torch.empty((1,), dtype=torch.int32, device=dev)
        dlogits = torch.empty_like(logits) if want_grads else None
        L.check(L.lib().step_cls_loss_f32(L.ptr(logits), L.ptr(targets), N, cls, L.ptr(loss_cls), L.ptr(flags), L.ptr(dlogits),
                                          L.stream()))
        # `if mask.sum():` in the reference is the same host read-back (two_branch.py:293)
        if int(flags[0].item()) == 0:
            loss_cls = torch.zeros((1,), dtype=torch.float32, device=dev)
    return (loss_cls, dlogits) if want_grads else loss_cls


def linear_backward(x, w, dy, need_dx=True, need_dw=True, dx_out=None, accumulate_dx=False):
    """Backward of y = x W^T + b (nn.Linear, or the 1x1x1 `global_cls` on flattened features) for the head's small-N
    layers: x [M,K] fp16|fp32, w [Nn,K] fp32, dy [M,Nn] fp32 -> (dx [M,K] fp32 | None, dw [Nn,K] | None, db [Nn] | None)."""
    dev = L.same_device(x, w, dy)
    M, K = x.shape
    Nn = dy.shape[1]
    dy = dy.detach().float().contiguous()
    w32 = w.detach().float().contiguous() if w is not None else None
    with torch.cuda.device(dev):
        dx = None
        if need_dx:
            dx = dx_out if dx_out is not None else torch.empty((M, K), dtype=torch.float32, device=dev)
        dw = torch.empty((Nn, K), dtype=torch.float32, device=dev) if need_dw else None
        db = torch.empty((Nn,), dtype=torch.float32, device=dev) if need_dw else None
        xs = x.detach()
        if xs.stride(1) != 1:
            xs = xs.contiguous()
        L.check(L.lib().step_linear_small_n_bwd(L.ptr(xs), L.dt(xs), M, K, xs.stride(0), L.ptr(w32), L.ptr(dy), Nn, L.ptr(dx),
                                                1 if accumulate_dx else 0, L.ptr(dw), L.ptr(db), L.stream()))
    return dx, dw, db


def roi_align_backward_nhwc(grad_out, rois, spatial_scale, K, H, W, sampling_ratio=0):
    """grad_out [R,ph,pw,C] (channels-last, fp16|fp32) -> grad_in [K,H,W,C] fp32.  Deterministic: no atomics."""
    from .engine import Act
    go = grad_out.detach().contiguous()
    R, ph, pw, C = go.shape
    return roi_align_backward_nhwc_strided(Act(go.view(R, 1, ph, pw, C)), rois, spatial_scale, K, H, W, sampling_ratio)


def roi_align_backward_nhwc_strided(grad_act, rois, spatial_scale, K, H, W, sampling_ratio=0):
    """ROIAlign backward from a channel slice of a wider buffer: grad_act (Act [R, T', ph, pw, ld] slice of C channels,
    fp16 | fp32; its R * T' rows are the rows of rois) -> grad_in [K,H,W,C] fp32.  Deterministic: no atomics."""
    ph, pw, C = grad_act.H, grad_act.W, grad_act.C
    R = grad_act.N * grad_act.T
    dev = L.same_device(grad_act.buf, rois)
    r = rois.detach().float().contiguous()
    with torch.cuda.device(dev):
        gin = torch.empty((K, H, W, C), dtype=torch.float32, device=dev)
        L.check(L.lib().step_roi_align_bwd_nhwc(L.c_void_p(grad_act.data_ptr()), grad_act.code, grad_act.ld, L.ptr(r), R,
                                                float(spatial_scale), ph, pw, K, H, W, C, int(sampling_ratio), L.ptr(gin), C,
                                                L.stream()))
    return gin


def roi_align_backward_slice(grad_act, rois, spatial_scale, grad_in, roi_T, feat_T, t_start, sampling_ratio=0, ws=None):
    """grad_in [B*feat_T, H, W, C] fp32 += ROIAlign backward of grad_act (Act [R, roi_T, ph, pw, ld] slice of C channels,
    fp16 | fp32) for ROIs whose frame index is relative to the frames [t_start, t_start + roi_T) of every clip (the frame map
    of ROINet.pool_into).  Frames outside the slice are untouched.  ws: optional fp32 workspace tensor, reused when large
    enough; the one used is returned."""
    ph, pw, C = grad_act.H, grad_act.W, grad_act.C
    R = grad_act.N * grad_act.T
    dev = L.same_device(grad_act.buf, rois, grad_in)
    K, H, W = grad_in.shape[0], grad_in.shape[1], grad_in.shape[2]
    r = rois.detach().float().contiguous()
    with torch.cuda.device(dev):
        nbytes = L.lib().step_roi_align_bwd_slice_workspace_bytes(K, H, W, C, roi_T, feat_T)
        if ws is None or ws.numel() * 4 < nbytes:
            ws = torch.empty((max(nbytes, 16) // 4,), dtype=torch.float32, device=dev)
        L.check(L.lib().step_roi_align_bwd_slice_nhwc(L.c_void_p(grad_act.data_ptr()), grad_act.code, grad_act.ld, L.ptr(r), R,
                                                      float(spatial_scale), ph, pw, K, H, W, C, int(sampling_ratio), int(roi_T),
                                                      int(feat_T), int(t_start), L.ptr(grad_in), grad_in.shape[3], L.ptr(ws),
                                                      ws.numel() * 4, L.stream()))
    return ws


def roi_pool_backward_slice(grad_act, rois, argmax, grad_in, roi_T, feat_T, t_start):
    """grad_in [B*feat_T, H, W, C] fp32 += ROIPool backward of grad_act (Act [R, roi_T, ph, pw, ld] slice of C channels,
    fp16 | fp32) through argmax (int32 [R*roi_T, ph, pw, C], as ROINet.pool_into records it) for ROIs whose frame index is
    relative to the frames [t_start, t_start + roi_T) of every clip.  Frames outside the slice are untouched.
    Deterministic, no atomics: every element sums its contributions in ascending (ROI row, ph, pw) order."""
    ph, pw, C = grad_act.H, grad_act.W, grad_act.C
    R = grad_act.N * grad_act.T
    if argmax.dtype != torch.int32 or not argmax.is_contiguous() or argmax.numel() < R * ph * pw * C:
        raise RuntimeError("roi_pool_backward_slice: argmax must be a contiguous int32 tensor of >= %d elements" % (R * ph * pw * C))
    dev = L.same_device(grad_act.buf, rois, argmax, grad_in)
    K, H, W = grad_in.shape[0], grad_in.shape[1], grad_in.shape[2]
    r = rois.detach().float().contiguous()
    with torch.cuda.device(dev):
        L.check(L.lib().step_roi_pool_bwd_slice_nhwc(L.c_void_p(grad_act.data_ptr()), grad_act.code, grad_act.ld, L.ptr(argmax), L.ptr(r),
                                                     R, ph, pw, K, H, W, C, int(roi_T), int(feat_T), int(t_start), L.ptr(grad_in),
                                                     grad_in.shape[3], L.stream()))
    return grad_in


def conv1x1_wgrad(dz, x, scale=1.0, out=None, accumulate=False):
    """dz [M,Cout] fp16, x [M,Cin] fp16 (row-major, channel strides allowed) -> dW [Cout,Cin] fp32 = scale * dz^T x."""
    dev = L.same_device(dz, x)
    if dz.dtype != torch.float16 or x.dtype != torch.float16:
        raise RuntimeError("conv1x1_wgrad: fp16 operands")
    M, Cout = dz.shape
    Cin = x.shape[1]
    with torch.cuda.device(dev):
        dw = out if out is not None else torch.empty((Cout, Cin), dtype=torch.float32, device=dev)
        nbytes = L.lib().step_conv1x1_wgrad_workspace_bytes(M, Cout, Cin)
        ws = torch.empty((nbytes // 4,), dtype=torch.float32, device=dev)
        L.check(L.lib().step_conv1x1_wgrad_f16(L.ptr(dz), dz.stride(0), L.ptr(x), x.stride(0), M, Cout, Cin, float(scale), L.ptr(dw),
                                               dw.stride(0), 1 if accumulate else 0, L.ptr(ws), nbytes, L.stream()))
    return dw


def conv_wgrad_f32(dz, x, k, stride=(1, 1, 1), pad_lo=(0, 0, 0), scale=1.0, out=None, accumulate=False):
    """Weight gradient of a convolution on the fp32 path: dz Act [N, OT, OH, OW, Cout] (the gradient of the raw convolution
    output), x Act [N, T, H, W, Cin] (its input; channel slices allowed) -> dW [Cout, taps, Cin] fp32 (+)= scale * dz^T x
    over every tap, for any filter k, stride and low padding pad_lo (step_conv_wgrad_f32: fp32 FFMA, deterministic)."""
    dev = L.same_device(dz.buf, x.buf)
    if dz.code != L.F32 or x.code != L.F32:
        raise RuntimeError("conv_wgrad_f32: fp32 operands")
    taps = k[0] * k[1] * k[2]
    M = dz.N * dz.T * dz.H * dz.W
    with torch.cuda.device(dev):
        dw = out if out is not None else torch.empty((dz.C, taps, x.C), dtype=torch.float32, device=dev)
        nbytes = L.lib().step_conv_wgrad_f32_workspace_bytes(M, dz.C, x.C, taps)
        ws = torch.empty((max(nbytes, 4) // 4,), dtype=torch.float32, device=dev)
        L.check(L.lib().step_conv_wgrad_f32(L.c_void_p(dz.data_ptr()), dz.ld, L.c_void_p(x.data_ptr()), x.ld, x.N, x.T, x.H, x.W,
                                            dz.T, dz.H, dz.W, dz.C, x.C, k[0], k[1], k[2], stride[0], stride[1], stride[2],
                                            pad_lo[0], pad_lo[1], pad_lo[2], float(scale), L.ptr(dw), dw.shape[2],
                                            1 if accumulate else 0, L.ptr(ws), nbytes, L.stream()))
    return dw


# ---- backward of the conv / pool tape ----------------------------------------------------------------------------------
class GradStore:
    """Gradient buffers, one per activation buffer of the forward (same shape and storage type -- fp16 or fp32 --,
    zero-initialised on first use).
    Every consumer ACCUMULATES into the slice it read, so fan-out (Inception branches, residuals, the shared concat
    buffer of two_branch.py:256) needs no special casing."""

    def __init__(self):
        self.bufs = {}

    def of(self, act):
        """Act view of the gradient of `act` (same channel slice of the gradient buffer)."""
        from .engine import Act
        key = act.buf.data_ptr()
        g = self.bufs.get(key)
        if g is None:
            g = torch.zeros_like(act.buf)
            self.bufs[key] = g
        # `act` may be another view of the same memory (Act.frames(): [N*T, 1, H, W, ld] over [N, T, H, W, ld])
        return Act(g.view(act.buf.shape), act.C, act.coff)


def _dgrad_weights(entry):
    """[Cout, taps, cin_pad] forward weights -> [Cin, taps, Cout] for the input gradient: dx = conv(dz, flip(w)^T)."""
    c = entry.get("_wT")
    if c is None:
        cin = entry["x"].C
        c = entry["w"][:, :, :cin].flip(1).permute(2, 1, 0).contiguous()
        entry["_wT"] = c
    return c


def stem_s2d_wgrad(dw, cin):
    """Weight gradient of the stride-2 7x7x7 stem from that of the 4x4x4 filter it runs as over the space-to-depth clip
    (engine.pack_stem_s2d): dw [Cout, 64 taps (qt, qh, qw), >= 8 cin channels (rt, rh, rw, c)] -> [Cout, cin, 7, 7, 7].
    Tap q and sub-position r hold filter position k = 2 q + r; k = 7 is padding and is dropped."""
    n = dw.shape[0]
    g8 = dw[:, :, :8 * cin].reshape(n, 4, 4, 4, 2, 2, 2, cin).permute(0, 7, 1, 4, 2, 5, 3, 6).reshape(n, cin, 8, 8, 8)
    return g8[:, :, :7, :7, :7].contiguous()


TIMING = None     # set to {} to collect per-phase device times of tape_backward (tools/train_bench.py)


@contextlib.contextmanager
def _phase(name):
    """Adds the block's device time to TIMING[name] when TIMING is a dict."""
    if TIMING is None:
        yield
        return
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    try:
        yield
    finally:
        e1.record()
        TIMING.setdefault(name, []).append((e0, e1))


def timing_summary():
    torch.cuda.synchronize()
    return {k: round(sum(a.elapsed_time(b) for a, b in v), 2) for k, v in (TIMING or {}).items()}


def trainable_bn(tag):
    """The BatchNorm3d of a tape tag (a Unit3Dpy) whose weight (gamma) or bias (beta) requires grad -- freeze_affine=False,
    networks.py:136-142 / two_branch.py:46-50 -- else None."""
    bn = getattr(tag, "batch3d", None) if getattr(tag, "use_bn", False) else None
    if bn is None or not (bn.weight.requires_grad or bn.bias.requires_grad):
        return None
    return bn


def check_bn_affine(nets):
    """Raise ValueError naming the first BatchNorm of nets ({key: module}) whose affine parameters train and that has a
    channel with gamma == 0 and beta > 0: that channel's output is relu(beta), constant, and its normalised input, which the
    gamma gradient needs, cannot be recovered from it.  One device-to-host read for all layers, none when no BatchNorm
    trains."""
    bns = [("%s.%s" % (key, name), m) for key, mod in nets.items() if mod is not None for name, m in mod.named_modules()
           if isinstance(m, torch.nn.BatchNorm3d) and (m.weight.requires_grad or m.bias.requires_grad)]
    if not bns:
        return
    with torch.no_grad():
        bad = torch.stack([((m.weight == 0) & (m.bias > 0)).any() for _, m in bns]).cpu()
    if bool(bad.any()):
        name = bns[int(bad.nonzero()[0, 0])][0]
        raise ValueError("BatchNorm %s has a channel with gamma == 0 and beta > 0: its output is constant and gamma's gradient "
                         "cannot be recovered from it; freeze that layer's affine parameters or give gamma a non-zero value"
                         % name)


def tape_backward(tape, grads, loss_scale=1.0, need_input_grad=None):
    """Reverse pass over the conv / max-pool tape recorded by engine.TAPE, in the storage type of each entry's activations
    (fp16: tensor-core weight gradient; fp32: step_conv_wgrad_f32).  `grads` (GradStore) must already hold
    d(loss * loss_scale)/d(output) of the last layers.  Returns {parameter tensor: fp32 gradient in the parameter's own
    layout}: conv weights and biases, and the weight (gamma) and bias (beta) of every Unit3Dpy BatchNorm whose affine
    parameters require grad (freeze_affine=False; step_act_bn_bwd_*, from the stored output: wherever its gradient is
    non-zero, y = gamma * xhat + beta).  Each BatchNorm tensor is returned only if it requires grad.  An entry recorded with
    batch statistics (freeze_stats=False, engine.conv's `bn`) goes through step_bn_bwd_* instead: dz through the batch mean
    and variance from the kept z, and gamma / beta gradients when they require grad.  With the running statistics a channel
    with gamma == 0 gives dgamma = 0, exact unless beta > 0, which `check_bn_affine` refuses.
    The input gradient of every layer is produced by the SAME convolution kernels as its forward (wgmma on fp16, SIMT on
    fp32), run on the transposed, flipped filter (stride-1 convolutions: dx = conv(dz, flip(w)^T)), accumulated through
    their residual input.  need_input_grad(entry) -> bool limits which entries form it (default: all).  A strided
    convolution (the fp32 trunk's 7x7x7 stem) gets its weight gradient only; asking for its input gradient raises."""
    from . import engine as E
    from .engine import Act
    out = {}
    lib = L.lib()
    inv = 1.0 / float(loss_scale)

    def add(param, g):
        out[param] = out[param] + g if param in out else g

    for e in reversed(tape):
        f16 = e["x"].code == L.F16
        if e["kind"] == "pool":
            x, y = e["x"], e["out"]
            gy, gx = grads.of(y), grads.of(x)
            k, s, pl, ph = e["k"], e["stride"], e["pad_lo"], e["pad_hi"]
            ws = torch.empty((y.N * y.T * y.H * y.W * y.C,), dtype=torch.uint8, device=x.device)
            pool_bwd = lib.step_maxpool3d_bwd_f16 if f16 else lib.step_maxpool3d_bwd_f32
            with _phase("pool_bwd"):
                L.check(pool_bwd(L.c_void_p(x.data_ptr()), x.ld, L.c_void_p(gy.data_ptr()), gy.ld, x.N, x.T, x.H,
                                                   x.W, x.C, k[0], k[1], k[2], s[0], s[1], s[2], pl[0], pl[1], pl[2], ph[0], ph[1],
                                                   ph[2], y.T, y.H, y.W, L.c_void_p(gx.data_ptr()), gx.ld, L.ptr(ws), L.stream()))
            continue
        x, w, k = e["x"], e["w"], e["k"]
        strided = e["stride"] != (1, 1, 1)
        if strided and (f16 or need_input_grad is None or need_input_grad(e)):
            raise NotImplementedError("tape_backward: a strided convolution has a weight gradient on the fp32 path only, and no "
                                      "input gradient (the trunk's stem needs none)")
        outs = [e["out"]] + e["extra_outs"]
        y0 = e["out"]
        M = y0.N * y0.T * y0.H * y0.W
        n_total = sum(o.C for o in outs)
        dz = torch.empty((y0.N, y0.T, y0.H, y0.W, n_total), dtype=x.buf.dtype, device=x.device)
        esz = dz.element_size()
        act_bwd = lib.step_act_bwd_f16 if f16 else lib.step_act_bwd_f32
        s2d = isinstance(e["tag"], tuple) and e["tag"][0] == "s2d"
        out_tags = [e["tag"][1]] if s2d else list(e["tag"]) if isinstance(e["tag"], (list, tuple)) else [e["tag"]]
        out_tags += [None] * (len(outs) - len(out_tags))        # every output gets its activation backward
        col = 0
        if e.get("bn") is not None and e.get("sync") is not None:
            # batch statistics of every rank's rows (engine.batch_stats_sync): this rank's sums of every output, one
            # exchange for the entry, then dz from the sums of all ranks (added in rank order: the same on every rank)
            with _phase("bn_bwd"):
                z = e["z"]
                sums_fn = lib.step_bn_bwd_sums_f16 if f16 else lib.step_bn_bwd_sums_f32
                merge_dz = lib.step_bn_bwd_merge_dz_f16 if f16 else lib.step_bn_bwd_merge_dz_f32
                nbytes = max(lib.step_bn_bwd_sums_workspace_bytes(M, max(o.C for o in outs)),
                             lib.step_bn_bwd_merge_dz_workspace_bytes(max(o.C for o in outs)))
                ws = torch.empty((max(nbytes, 4) // 4,), dtype=torch.float32, device=x.device)
                sums = torch.empty((2, n_total), dtype=torch.float32, device=x.device)
                at = lambda t, c, es=4: L.c_void_p(t.data_ptr() + es * c)
                for o, bn in zip(outs, e["bn"]):
                    gy = grads.of(o)
                    gam, bet = bn.weight, bn.bias
                    dgam = torch.empty((o.C,), dtype=torch.float32, device=x.device) if gam.requires_grad else None
                    dbet = torch.empty((o.C,), dtype=torch.float32, device=x.device) if bet.requires_grad else None
                    L.check(sums_fn(L.c_void_p(gy.data_ptr()), gy.ld, L.c_void_p(o.data_ptr()), o.ld, at(z.buf, col, esz), n_total, M,
                                    o.C, at(e["mean"], col), at(e["rstd"], col), 1 if e["relu"] else 0, inv, at(sums, col), n_total,
                                    L.ptr(dgam), L.ptr(dbet), L.ptr(ws), nbytes, L.stream()))
                    if dgam is not None:
                        add(gam, dgam)
                    if dbet is not None:
                        add(bet, dbet)
                    col += o.C
                gathered = E.all_gather_rows(sums, e["sync"]["group"])
                col = 0
                for o, bn in zip(outs, e["bn"]):
                    gy = grads.of(o)
                    L.check(merge_dz(at(gathered, col), gathered.shape[0], n_total, e["sync"]["M_total"], L.c_void_p(gy.data_ptr()),
                                     gy.ld, L.c_void_p(o.data_ptr()), o.ld, at(z.buf, col, esz), n_total, M, o.C, at(e["mean"], col),
                                     at(e["rstd"], col), L.ptr(bn.weight.detach()), 1 if e["relu"] else 0, at(dz, col, esz), n_total,
                                     L.ptr(ws), nbytes, L.stream()))
                    col += o.C
        elif e.get("bn") is not None:   # batch statistics (engine._conv_batch_stats): dz through mean and variance
            with _phase("bn_bwd"):
                bn_bwd = lib.step_bn_bwd_f16 if f16 else lib.step_bn_bwd_f32
                nbytes = lib.step_bn_bwd_workspace_bytes(M, max(o.C for o in outs))
                ws = torch.empty((max(nbytes, 4) // 4,), dtype=torch.float32, device=x.device)
                z = e["z"]
                for o, bn in zip(outs, e["bn"]):
                    gy = grads.of(o)
                    gam, bet = bn.weight, bn.bias
                    dgam = torch.empty((o.C,), dtype=torch.float32, device=x.device) if gam.requires_grad else None
                    dbet = torch.empty((o.C,), dtype=torch.float32, device=x.device) if bet.requires_grad else None
                    L.check(bn_bwd(L.c_void_p(gy.data_ptr()), gy.ld, L.c_void_p(o.data_ptr()), o.ld,
                                   L.c_void_p(z.buf.data_ptr() + esz * col), n_total, M, o.C,
                                   L.c_void_p(e["mean"].data_ptr() + 4 * col), L.c_void_p(e["rstd"].data_ptr() + 4 * col),
                                   L.ptr(gam.detach()), 1 if e["relu"] else 0, inv, L.c_void_p(dz.data_ptr() + esz * col), n_total,
                                   L.ptr(dgam), L.ptr(dbet), L.ptr(ws), nbytes, L.stream()))
                    if dgam is not None:
                        add(gam, dgam)
                    if dbet is not None:
                        add(bet, dbet)
                    col += o.C
        else:
            with _phase("act_bwd"):
                for o, tg in zip(outs, out_tags):
                    gy = grads.of(o)
                    sc = e["scale"][col:col + o.C] if e["scale"] is not None else None
                    res = e["residual"]
                    gres = grads.of(res) if res is not None else None
                    args = (L.c_void_p(gy.data_ptr()), gy.ld, L.c_void_p(o.data_ptr()), o.ld, L.ptr(sc), 1 if e["relu"] else 0, M,
                            o.C, L.c_void_p(dz.data_ptr() + esz * col), n_total,
                            L.c_void_p(gres.data_ptr()) if gres is not None else None, gres.ld if gres is not None else 0)
                    bn = trainable_bn(tg)
                    if bn is None:
                        L.check(act_bwd(*args, L.stream()))
                    else:   # the same dz / dres, and the BatchNorm's gamma / beta gradients from the same pass
                        gam, bet = bn.weight, bn.bias
                        dgam = torch.empty((o.C,), dtype=torch.float32, device=x.device) if gam.requires_grad else None
                        dbet = torch.empty((o.C,), dtype=torch.float32, device=x.device) if bet.requires_grad else None
                        nbytes = lib.step_act_bn_bwd_workspace_bytes(M, o.C)
                        ws = torch.empty((nbytes // 4,), dtype=torch.float32, device=x.device)
                        act_bn_bwd = lib.step_act_bn_bwd_f16 if f16 else lib.step_act_bn_bwd_f32
                        L.check(act_bn_bwd(*args, L.ptr(bet.detach()), L.ptr(gam.detach()), inv, L.ptr(dgam), L.ptr(dbet), L.ptr(ws),
                                           nbytes, L.stream()))
                        if dgam is not None:
                            add(gam, dgam)
                        if dbet is not None:
                            add(bet, dbet)
                    col += o.C
        # ---- weight (and bias) gradients
        taps = k[0] * k[1] * k[2]
        pl = e["pad_lo"]
        with _phase("wgrad_k%d" % taps):
            if f16:
                dw = torch.empty((n_total, taps, x.C), dtype=torch.float32, device=x.device)
                nbytes = lib.step_conv_wgrad_workspace_bytes(M, n_total, x.C, taps)
                ws = torch.empty((nbytes // 4,), dtype=torch.float32, device=x.device)
                L.check(lib.step_conv_wgrad_f16(L.ptr(dz), n_total, L.c_void_p(x.data_ptr()), x.ld, x.N, x.T, x.H, x.W, n_total, x.C,
                                                k[0], k[1], k[2], pl[0], pl[1], pl[2], inv, L.ptr(dw), x.C, 0, L.ptr(ws), nbytes,
                                                L.stream()))
            else:
                dw = conv_wgrad_f32(Act(dz), x, k, e["stride"], pl, inv)
        if s2d:
            unit = e["tag"][1]
            if unit.conv3d.weight.requires_grad:
                add(unit.conv3d.weight, stem_s2d_wgrad(dw, unit.conv3d.in_channels))
            continue                                   # the clip itself needs no gradient
        tags = e["tag"] if isinstance(e["tag"], (list, tuple)) else [e["tag"]]
        row = 0
        for tg, o in zip(tags, outs):
            if tg is None:
                row += o.C
                continue
            conv = getattr(tg, "conv3d", tg)          # Unit3Dpy holds its nn.Conv3d; nn.Conv2d / nn.Conv3d containers are themselves
            cin = conv.weight.shape[1]                # x.C, or fewer on the fp32 stem (the clip's padding channel)
            g = dw[row:row + o.C, :, :cin].reshape((o.C,) + tuple(conv.weight.shape[2:]) + (cin,))
            g = g.permute(0, g.dim() - 1, *range(1, g.dim() - 1)).contiguous()        # [Cout, Cin, *k]
            if conv.weight.requires_grad:
                add(conv.weight, g)
            if conv.bias is not None and conv.bias.requires_grad:
                db = torch.empty((o.C,), dtype=torch.float32, device=x.device)
                wsb = torch.empty((64 * o.C,), dtype=torch.float32, device=x.device)
                colsum = lib.step_colsum_f16 if f16 else lib.step_colsum_f32
                L.check(colsum(L.c_void_p(dz.data_ptr() + esz * row), n_total, M, o.C, inv, L.ptr(db), L.ptr(wsb), L.stream()))
                add(conv.bias, db)
            row += o.C
        # ---- input gradient: the forward kernel on the transposed, flipped filter, accumulated into grad(x)
        if need_input_grad is None or need_input_grad(e):
            gx = grads.of(x)
            wT = _dgrad_weights(e)
            pad = tuple(kk - 1 - p for kk, p in zip(k, pl))
            with E.recording(None), _phase("dgrad"):
                E.conv(Act(dz), wT, None, None, gx, k, (1, 1, 1), pad, relu=False, residual=gx, out_dims=(x.T, x.H, x.W))
    return out


# ---- the heads' dropout (two_branch.py:244, 261) -------------------------------------------------------------------------
_DEVICE_GEOMETRY = {}


def dropout_draw(device, p, n):
    """Take the draw that torch.nn.functional.dropout(x, p, training=True) makes for an n-element fp32 tensor x on `device`
    from torch.cuda.default_generators[device]: returns the step_dropout_draw of the generator's state before it (seed,
    offset, p, and the device's launch geometry), and advances the generator's offset as that call does.  The library
    reproduces the call's keep mask from the draw (step_b200.h, step_dropout_*).  0 < p < 1 and n % 4 == 0, or it raises
    before touching the generator; inside CUDA stream capture it raises (the offset moves on the host)."""
    torch.cuda.init()                     # default_generators is empty until CUDA is initialised
    device = torch.device(device)
    index = device.index if device.index is not None else torch.cuda.current_device()
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("dropout_draw: the draw advances the generator's offset on the host and cannot be captured in a CUDA graph")
    geom = _DEVICE_GEOMETRY.get(index)
    if geom is None:
        prop = torch.cuda.get_device_properties(index)
        geom = _DEVICE_GEOMETRY[index] = (prop.multi_processor_count, prop.max_threads_per_multi_processor)
    gen = torch.cuda.default_generators[index]
    # keep = (float)(1 - p) with 1 - p in double, as ATen's dropout_cuda forms it (ctypes rounds the double to float)
    draw = L.step_dropout_draw(seed=gen.initial_seed(), offset=gen.get_offset(), keep=1.0 - float(p), sm_count=geom[0],
                               threads_per_sm=geom[1])
    step = ctypes.c_uint64()
    L.check(L.lib().step_dropout_check(draw, int(n), ctypes.byref(step)))
    gen.set_offset(draw.offset + step.value)
    return draw


def dropout_mask(draw, n, device):
    """The keep mask of a draw of n elements (uint8 [n], 1 = kept), in the dropped tensor's element order."""
    with torch.cuda.device(device):
        mask = torch.empty((n,), dtype=torch.uint8, device=device)
        L.check(L.lib().step_dropout_mask_u8(draw, int(n), L.ptr(mask), L.stream()))
    return mask


def head_dropout_draws(net, R, T, context=True):
    """The draws head `net` makes in a training forward over R tubes of T frames (two_branch.py:244, then 261), taken from
    the default generator of the head's device: (global, local) -- local None for class-only heads -- or None when the head
    draws nothing (net.dropout in eval mode, or p == 0).  context: whether the classifier reads the context columns."""
    p = float(net.dropout.p)
    if not net.dropout.training or p == 0.0:
        return None
    if p >= 1.0:
        raise ValueError("head_dropout_draws: dropout p = %g zeroes the head's inputs; only p < 1 is supported" % p)
    dev = net.global_cls.weight.device
    D = net.fc_dim * net.pool_size ** 2
    ctx_cols = net.global_cls.weight.shape[1] - D if context else 0
    g = dropout_draw(dev, p, R * (D + ctx_cols) * T)
    return g, None if net.cls_only else dropout_draw(dev, p, R * T * D)


def head_forward_backward(net, global_feat, tubes, targets, context_feat=None, lambda_reg=5.0, lambda_neighbor=1.0,
                          loss_scale=1024.0, cat=None, objective_scale=1.0, dropout=False):
    """One training-time evaluation of a TwoBranchNet on the device (train.py:323-347 for one refinement step): forward
    with targets, the three losses, and the gradient of  mean(loss_cls) + lambda_reg * loss_loc + lambda_neighbor * loss_nb
    with respect to every trainable parameter of the head and to the pooled ROI features, on the head's precision path
    (net.fp16): fp16 or fp32 activations / activation gradients, fp32 weight gradients, with the static loss scale
    `loss_scale` applied to the activation gradients on both (apex-style; on fp32 a power of two is exact, and 1.0 is the
    reference's fp32 arithmetic).  Dropout is the identity (eval mode), like the reference's gradient goldens, unless
    dropout=True and the head's nn.Dropout is in training mode with 0 < p < 1: then the head makes the reference's two draws
    (`head_dropout_draws`) from the CUDA generator of its device, exactly the masks F.dropout would draw there, and the
    forward and backward go through them (two_branch.py:244, 261; see step_b200.h, step_dropout_*).
    Class-only heads (TwoBranchNet(cls_only=True), the first training stage of train_cls.py) have no local branch: the
    objective is mean(loss_cls) alone (`cls_loss`), the regression losses are the reference's [1] zeros and grads holds the
    16 tensors of Mixed_5b / Mixed_5c, `downsample` and `global_cls`.  With freeze_affine=False grads also holds the gamma
    and beta of the head's Unit3D BatchNorms that require grad (tape_backward).
    context_feat (heads built with the context columns, cfg.no_context=False), in one of two forms:
      * [N,1024,T',1,1], the per-tube context feature the reference passes (train.py:317-321, two_branch.py:242-249);
      * (ctx_mean, row_map): ctx_mean fp32 [rows, 1024] is the mean of the context feature over the step's frames and
        row_map int32 [N] (or None = identity) the row of each tube (ContextNet output per clip, as train_step feeds it);
        with dropout the frames themselves are needed: (ctx_mean, row_map, ctx, t_start), ctx the ContextNet output
        [clips, T'', 1024] fp32 and t_start the step's first frame in it (row_map then gives each tube's clip).
    Returns dict(prob, loc, first, last, losses=(cls, loc, nb), loss, grads={param: grad}, feat_grad=[N,T',832,7,7] fp32,
    ctx_grad): grads holds the whole global_cls.weight (context columns included); ctx_grad is the gradient with respect to
    the context input, [N,1024,T',1,1] for the first form and the per-tube [N,1024] gradient of the row each tube reads for
    the second (None without context).  With dropout the second form's ctx_grad is the gradient of each tube's dropped
    context mean, and ctx_dropout holds what `context_grad_reduce` needs to take it through the draw."""
    from . import engine as E
    with torch.cuda.device(cat.device if cat is not None else global_feat.device), torch.no_grad():
        fwd, state = head_forward(net, global_feat, tubes, targets, context_feat=context_feat, cat=cat, dropout=dropout)
        prob, loc, first, last, logits = fwd["prob"], fwd["loc"], fwd["first"], fwd["last"], fwd["logits"]
        dev = state["dev"]
        if net.cls_only:
            # class-only heads: the regression losses are the reference's zeros (two_branch.py:252,276-280)
            lc, dlogits = cls_loss(logits, targets, want_grads=True)
            ll, ln = torch.zeros((1,), dtype=torch.float32, device=dev), torch.zeros((1,), dtype=torch.float32, device=dev)
            g = {"logits": dlogits}
        else:
            lc, ll, ln, g = head_losses(logits, loc, first, last, tubes, targets, net.T, lambda_reg, lambda_neighbor, want_grads=True)
        if objective_scale != 1.0:
            for k_ in g:
                g[k_].mul_(objective_scale)
        r = head_backward(state, g, loss_scale)
    loss = lc.mean() + lambda_reg * ll.mean() + lambda_neighbor * ln.mean()
    return dict(prob=prob, loc=loc, first=first, last=last, losses=(lc, ll, ln), loss=loss, **r)


def head_forward(net, global_feat, tubes, targets, context_feat=None, cat=None, dropout=False):
    """The forward half of head_forward_backward (same arguments): the head's forward with the tape on, and with
    dropout=True the reference's draws when the head's nn.Dropout trains.  Returns (dict(prob, loc, first, last, logits),
    state for head_backward).  The state holds none of the returned tensors."""
    from . import engine as E
    from .engine import Act
    from .networks import to_act
    code = E.dtype_code(net.fp16)
    fc, ps = net.fc_dim, net.pool_size
    if cat is None:
        dev = L.same_device(global_feat, tubes, targets)
        N, Tl, C, Wd, Hd = global_feat.shape
    else:   # ROI features already pooled into the [ROI | downsample] concat buffer (ROINet.pool_into)
        dev = L.same_device(cat.buf, tubes, targets)
        N, Tl, Wd, Hd, C = cat.N, cat.T, cat.H, cat.W, cat.ld - fc
        if cat.code != code:
            raise RuntimeError("head_forward_backward: the concat buffer is %s but the head runs on the %s path"
                               % (cat.buf.dtype, E.torch_dtype(code)))
    hw = net._head_weights()
    if (context_feat is None) != (hw["ctx_w"] is None):
        raise RuntimeError("head_forward_backward: global_cls has %d context columns but context_feat is %s"
                           % (0 if hw["ctx_w"] is None else hw["ctx_w"].shape[1], "None" if context_feat is None else "given"))
    with torch.cuda.device(dev), torch.no_grad():
        if cat is None:
            cat = Act.empty(N, Tl, Wd, Hd, C + fc, code, dev)
            src = to_act(global_feat, code)
            cat.buf[..., :C].copy_(src.buf[..., src.coff:src.coff + C])
        drop = head_dropout_draws(net, N, Tl, context=context_feat is not None) if dropout else None
        ctx_mean, row_map, ctx_module_form = None, None, False
        if isinstance(context_feat, (tuple, list)):
            ctx_mean, row_map = context_feat[:2]
            L.same_device(ctx_mean, row_map, cat.buf)
            ctx_mean = ctx_mean.float().contiguous()
            if drop is not None:
                if len(context_feat) != 4:
                    raise RuntimeError("head_forward_backward: dropout needs the context frames: (ctx_mean, row_map, ctx, t_start)")
                ctx, t0 = context_feat[2].detach().float().contiguous(), int(context_feat[3])
                L.same_device(ctx, cat.buf)
                K = ctx.shape[2]
                rm = row_map.to(torch.int32).contiguous() if row_map is not None else None
                ctx_mean = torch.empty((N, K), dtype=torch.float32, device=dev)
                L.check(L.lib().step_dropout_ctx_mean_f32(drop[0], ps * ps, fc, L.c_void_p(ctx.data_ptr() + 4 * t0 * K), L.ptr(rm),
                                                          ctx.shape[1] * K, K, 1, N, Tl, K, L.ptr(ctx_mean), L.stream()))
                row_map = None
        elif context_feat is not None:
            ctx_module_form = True
            if tuple(context_feat.shape) != (N, 1024, Tl, 1, 1):
                raise RuntimeError("head_forward_backward: context_feat %s, expected [%d,1024,%d,1,1]" % (tuple(context_feat.shape), N, Tl))
            cf = context_feat.detach().to(dev).float().contiguous().view(N * 1024, Tl)
            if drop is None:
                ctx_mean = E.mean_mid(cf.data_ptr(), L.F32, N * 1024, Tl, 1, 1, 1, dev).view(N, 1024)   # as TwoBranchNet.forward
            else:
                ctx_mean = torch.empty((N, 1024), dtype=torch.float32, device=dev)
                L.check(L.lib().step_dropout_ctx_mean_f32(drop[0], ps * ps, fc, L.ptr(cf), None, 1024 * Tl, 1, Tl, N, Tl, 1024,
                                                          L.ptr(ctx_mean), L.stream()))
        tape, keep = [], {}
        with E.recording(tape):
            prob, loc, first, last, logits = net.forward_act(cat, ctx_mean, row_map, want_logits=True, keep=keep, dropout=drop)
    state = dict(net=net, hw=hw, dev=dev, code=code, N=N, Tl=Tl, C=C, cat=cat, tape=tape, keep=keep, drop=drop, ctx_mean=ctx_mean,
                 row_map=row_map, ctx_module_form=ctx_module_form, feat_grad=global_feat is not None)
    return dict(prob=prob, loc=loc, first=first, last=last, logits=logits), state


def head_backward(state, g, loss_scale=1024.0):
    """The backward half of head_forward_backward from the gradients g of the head's tail outputs: fp32 g["logits"]
    [N,cls] (pre-sigmoid), and for full heads g["local_loc"] [N,T',4] (local_reg's output, with what flows back through
    the first / last slices already added) and g["first_loc"] / g["last_loc"] [N,Tc,4] (neighbor_reg1 / 2's outputs), each
    d(loss)/d(output) unscaled: the activation gradients are scaled by loss_scale and the results unscaled again.
    Returns dict(grads, feat_grad, roi_grad, ctx_grad, ctx_dropout) as head_forward_backward describes them."""
    from .engine import Act
    net, hw, dev, code = state["net"], state["hw"], state["dev"], state["code"]
    N, Tl, C, cat, keep, drop = state["N"], state["Tl"], state["C"], state["cat"], state["keep"], state["drop"]
    ctx_mean, row_map, ctx_module_form = state["ctx_mean"], state["row_map"], state["ctx_module_form"]
    fc, ps = net.fc_dim, net.pool_size
    D = fc * ps * ps
    with torch.cuda.device(dev), torch.no_grad():
        grads = GradStore()
        out = {}
        unperm = lambda w: w.view(-1, ps * ps, fc).permute(0, 2, 1).reshape(w.shape[0], -1)   # (p*fc + c) -> (c*49 + p)
        # ---- classifier: logits = mean_t(gconv) . W^T + ctx . W_ctx^T + b   (two_branch.py:242-249)
        dxbar, dw, db = linear_backward(keep["xbar"], hw["cls_w"], g["logits"])
        ctx_grad = None
        if ctx_mean is not None:
            # the context columns are not permuted; the rows each tube read (row_map) are gathered for dW_ctx
            xc = ctx_mean if row_map is None else ctx_mean.index_select(0, row_map.long())
            ctx_grad, dw_ctx, _ = linear_backward(xc, hw["ctx_w"], g["logits"])
            dw = torch.cat([unperm(dw), dw_ctx], 1)
            if ctx_module_form and drop is not None:
                # every tube is its own clip of T' frames: the reduce through the draw gives [N, T', 1024]
                own = torch.zeros((N, Tl, 5), dtype=torch.float32, device=dev)
                own[:, 0, 0] = torch.arange(N, dtype=torch.float32, device=dev) * Tl
                acc = torch.zeros((N, Tl, 1024), dtype=torch.float32, device=dev)
                context_grad_reduce(ctx_grad, own, acc, 0, dropout=(drop[0], ps * ps, fc))
                ctx_grad = acc.permute(0, 2, 1).contiguous().view(N, 1024, Tl, 1, 1)
            elif ctx_module_form:   # the classifier averages its per-frame logits over T' (two_branch.py:249)
                ctx_grad = (ctx_grad * (1.0 / Tl)).view(N, 1024, 1, 1, 1).expand(N, 1024, Tl, 1, 1).contiguous()
        else:
            dw = unperm(dw)
        out[net.global_cls.weight] = dw.reshape(net.global_cls.weight.shape)
        out[net.global_cls.bias] = db
        gcat = grads.of(cat)
        gconv_grad = L.c_void_p(gcat.data_ptr() + gcat.buf.element_size() * C)
        if drop is not None:
            L.check(L.lib().step_mean_mid_bwd_dropout(drop[0], 0 if ctx_mean is None else ctx_mean.shape[1], L.ptr(dxbar), N, Tl,
                                                      ps * ps, fc, float(loss_scale), gconv_grad, code, gcat.ld, L.stream()))
        else:
            mean_mid_bwd = L.lib().step_mean_mid_bwd if code == L.F16 else L.lib().step_mean_mid_bwd_f32
            L.check(mean_mid_bwd(L.ptr(dxbar), N, Tl, ps * ps, fc, float(loss_scale), gconv_grad, gcat.ld, L.stream()))
        # ---- regressors (two_branch.py:261-270): local_reg on every frame, neighbor_reg1 / 2 on the first / last chunk.
        # Class-only heads have no local branch: their tape ends at `downsample`.
        if not net.cls_only:
            lf2 = keep["local_feat2"]
            lf2v = keep["local_feat2_dropped"].buf.view(N, Tl, D)      # the regressors' input (lf2 itself without dropout)
            s0, s1, e0, e1 = keep["slices"]
            dlf2 = torch.zeros((N, Tl, D), dtype=torch.float32, device=dev)
            dx, dw, db = linear_backward(lf2v.reshape(N * Tl, D), hw["local_reg_w32"], g["local_loc"].reshape(N * Tl, 4), dx_out=dlf2.view(N * Tl, D))
            out[net.local_reg.weight], out[net.local_reg.bias] = unperm(dw), db
            for mod, nm, (a, b), gk in ((net.neighbor_reg1, "neighbor_reg1", (s0, s1), "first_loc"), (net.neighbor_reg2, "neighbor_reg2", (e0, e1), "last_loc")):
                xs = lf2v[:, a:b].reshape(-1, D).contiguous()
                dx, dw, db = linear_backward(xs, hw[nm + "_w32"], g[gk].reshape(-1, 4))
                dlf2[:, a:b] += dx.view(N, b - a, D)                      # disjoint frame ranges of one buffer (host-side glue)
                out[mod.weight], out[mod.bias] = unperm(dw), db
            glf2 = grads.of(lf2)
            if drop is not None:
                L.check(L.lib().step_f32_accum_dropout(drop[1], L.ptr(dlf2), N * Tl, ps * ps, fc, float(loss_scale),
                                                       L.c_void_p(glf2.data_ptr()), code, glf2.ld, L.stream()))
            else:
                f32_accum = L.lib().step_f32_accum_f16 if code == L.F16 else L.lib().step_f32_accum_f32
                L.check(f32_accum(L.ptr(dlf2), N * Tl * ps * ps, fc, float(loss_scale), L.c_void_p(glf2.data_ptr()), glf2.ld, L.stream()))
        # ---- every convolution and pool of the head, in reverse
        out.update(tape_backward(state["tape"], grads, loss_scale))
        gcat = grads.of(cat)
        fg = gcat.buf[..., :C].float().mul_(1.0 / loss_scale).permute(0, 1, 4, 2, 3).contiguous() if state["feat_grad"] else None
    ctx_dropout = (drop[0], ps * ps, fc) if drop is not None and ctx_mean is not None and not ctx_module_form else None
    return dict(grads=out, feat_grad=fg, roi_grad=Act(gcat.buf, C, 0), ctx_grad=ctx_grad, ctx_dropout=ctx_dropout)


def head_outputs_backward(logits, loc, first, last, tubes, targets, T, cls_only, g_prob=None, g_loc=None, g_first=None,
                          g_last=None, g_loss_cls=None, g_loss_loc=None, g_loss_nb=None):
    """The gradients of the head's tail (two_branch.py:272-342) from upstream gradients of its seven outputs
    (step_head_outputs_bwd_f32; None = zero): returns head_backward's g, {"logits"} and for full heads also {"local_loc",
    "first_loc", "last_loc"}.  logits [N,cls] (pre-sigmoid) and loc / first / last are the forward's; a loss whose mask
    sums to zero was a constant there and its upstream gradient is not read (decided on the device)."""
    dev = L.same_device(logits, targets)
    f32 = lambda t: None if t is None else t.detach().to(device=dev, dtype=torch.float32).contiguous()
    logits, targets = f32(logits), f32(targets)
    N, cls = logits.shape
    if targets.shape != (N, 3, 6 + cls):
        raise RuntimeError("head_outputs_backward: targets %s do not match N=%d, classes=%d" % (tuple(targets.shape), N, cls))
    ups = [f32(t) for t in (g_prob, g_loc, g_first, g_last, g_loss_cls, g_loss_loc, g_loss_nb)]
    with torch.cuda.device(dev):
        g = {"logits": torch.empty_like(logits)}
        if cls_only:
            loc = first = last = tubes = None
            T_len = Tc = 0
        else:
            loc, first, last, tubes = f32(loc), f32(first), f32(last), f32(tubes)
            T_len, Tc = loc.shape[1], first.shape[1]
            if tubes.shape != (N, T_len, 5) or loc.shape != (N, T_len, 4) or first.shape != last.shape or first.shape != (N, Tc, 4):
                raise RuntimeError("head_outputs_backward: local_loc %s / first %s / last %s / tubes %s do not match N=%d"
                                   % (tuple(loc.shape), tuple(first.shape), tuple(last.shape), tuple(tubes.shape), N))
            g.update(local_loc=torch.empty_like(loc), first_loc=torch.empty_like(first), last_loc=torch.empty_like(last))
        expect = [(N, cls), (N, T_len, 4), (N, Tc, 4), (N, Tc, 4), (N * cls,), (1,), (1,)]
        for i, (u, shape) in enumerate(zip(ups, expect)):
            if u is None or (cls_only and i in (1, 2, 3, 5, 6)):
                ups[i] = None
            elif i == 4 and u.numel() != N * cls:
                ups[i] = None       # the forward's [1] zero: no classification mask, the kernel reads nothing
            elif tuple(u.shape) != shape and u.numel() != int(torch.Size(shape).numel()):
                raise RuntimeError("head_outputs_backward: upstream gradient %d has shape %s, expected %s" % (i, tuple(u.shape), shape))
        L.check(L.lib().step_head_outputs_bwd_f32(L.ptr(logits), L.ptr(loc), L.ptr(first), L.ptr(last), L.ptr(tubes), L.ptr(targets),
                                                  N, cls, T_len, int(T), Tc, 1 if cls_only else 0, *[L.ptr(u) for u in ups],
                                                  L.ptr(g["logits"]), L.ptr(g.get("local_loc")), L.ptr(g.get("first_loc")),
                                                  L.ptr(g.get("last_loc")), L.stream()))
    return g


def context_forward(context_net, feat):
    """ContextNet.forward_act (two_branch.py:132-138) with the tape on, in the storage type of feat, the trunk's output Act
    [B,T',H',W',832] (fp16 or fp32, which must be the ContextNet's cfg.fp16 path).  Returns (ctx [B,T',1024] fp32, state
    for context_backward)."""
    from . import engine as E
    code = E.dtype_code(context_net.fp16)
    if feat.code != code:
        raise RuntimeError("context_forward: conv_feat is %s but the ContextNet runs on the %s path"
                           % (feat.buf.dtype, E.torch_dtype(code)))
    with torch.cuda.device(feat.device), torch.no_grad():
        tape, keep = [], {}
        with E.recording(tape):
            ctx = context_net.forward_act(feat, keep=keep)
    return ctx, dict(tape=tape, x=keep["mixed_5c"], feat=feat)


def context_backward(state, d_ctx, loss_scale=1024.0):
    """Backward of context_forward from d_ctx = d(loss)/d(ctx), fp32 [B,T',1024]: the spatial mean's backward into the
    gradient of Mixed_5c's output, then the tape (Mixed_5c, Mixed_5b, the (1,3,3)/(1,2,2) max-pool).  Returns
    ({parameter: fp32 gradient} for the 12 Unit3D convolutions, and their BatchNorms' gamma / beta when those require grad
    (freeze_affine=False, tape_backward), [B,T',H',W',832] in the
    forward's storage type (a channel-slice view) holding loss_scale * d(loss)/d(conv_feat) through the context branch)."""
    x = state["x"]
    with torch.cuda.device(x.device), torch.no_grad():
        grads = GradStore()
        gx = grads.of(x)
        d = d_ctx.float().contiguous()
        mean_mid_bwd = L.lib().step_mean_mid_bwd if gx.code == L.F16 else L.lib().step_mean_mid_bwd_f32
        L.check(mean_mid_bwd(L.ptr(d), x.N * x.T, x.H * x.W, 1, x.C, float(loss_scale), L.c_void_p(gx.data_ptr()), gx.ld, L.stream()))
        out = tape_backward(state["tape"], grads, loss_scale)
        gfeat = grads.of(state["feat"])
    return out, gfeat.buf[..., gfeat.coff:gfeat.coff + gfeat.C]


def context_grad_reduce(dctx, tubes, acc, t_start, dropout=None):
    """acc [B, T', 1024] fp32 += the gradient of ContextNet's output from one refinement step: dctx [R, 1024] is each
    tube's gradient of the context row it read, tubes [R, T_len, 5] the step's flat tubes (train.py:317-321: clip =
    floor(frame / T_len), frames [t_start, t_start + T_len) of the clip, weight 1 / T_len).  Deterministic.
    dropout: head_forward_backward's ctx_dropout when the classifier read the dropped context (dctx is then the gradient of
    each tube's dropped context mean, and every frame's term goes through its element of the head's global draw)."""
    dev = L.same_device(dctx, tubes, acc)
    R, T_len = tubes.shape[0], tubes.shape[1]
    B, T_all, C = acc.shape
    d = dctx.float().contiguous()
    tb = tubes.float().contiguous()
    with torch.cuda.device(dev):
        if dropout is not None:
            draw, P, Cg = dropout
            L.check(L.lib().step_ctx_grad_reduce_dropout_f32(draw, P, Cg, L.ptr(d), C, L.ptr(tb), R, T_len, B, T_all, int(t_start), C,
                                                             L.ptr(acc), L.stream()))
        else:
            L.check(L.lib().step_ctx_grad_reduce_f32(L.ptr(d), C, L.ptr(tb), R, T_len, B, T_all, int(t_start), C, L.ptr(acc), L.stream()))
    return acc


def trunk_forward_backward(base_net, clips, d_feat_fn, loss_scale=1024.0):
    """I3D trunk forward on base_net's precision path (cfg.fp16) with the tape on, then backward from d(loss)/d(conv_feat).
    On fp32 the stem is the stride-2 7x7x7 convolution over the clip padded to 4 channels; its weight gradient comes from
    step_conv_wgrad_f32 (on fp16 the stem runs as the space-to-depth 4x4x4 filter, stem_s2d_wgrad).
    d_feat_fn(feat_act) -> fp32 tensor [N,T',H',W',832] (channels-last) with the gradient of the loss w.r.t. the trunk
    output (e.g. the sum of the ROIAlign backward results of the refinement steps).
    Returns (feat Act, {parameter: fp32 gradient}): the conv weights, and the BatchNorms' gamma / beta where they require
    grad (freeze_affine=False, networks.py:136-142).  A base_net built with freeze_stats=False and in training mode normalises
    with batch statistics, and its forward updates the running statistics unless engine.running_stats_update(False) is on."""
    with torch.cuda.device(clips.device), torch.no_grad():
        feat, state = trunk_forward(base_net, clips)
        out = trunk_backward(state, d_feat_fn(feat), loss_scale)
    return feat, out


def trunk_forward(base_net, clips):
    """The forward half of trunk_forward_backward: base_net.forward_act(clips) with the tape on.  Returns (feat Act
    [N,T',H',W',832], state for trunk_backward)."""
    from . import engine as E
    with torch.cuda.device(clips.device), torch.no_grad():
        tape = []
        with E.recording(tape):
            feat = base_net.forward_act(clips)
    return feat, dict(tape=tape, feat=feat)


def trunk_backward(state, d_feat, loss_scale=1024.0):
    """The backward half of trunk_forward_backward from d_feat = d(loss)/d(conv_feat), [N,T',H',W',832] channels-last (any
    strides, any float dtype; made fp32 contiguous here).  Returns {parameter: fp32 gradient}."""
    feat, tape = state["feat"], state["tape"]
    with torch.cuda.device(feat.device), torch.no_grad():
        grads = GradStore()
        gfeat = grads.of(feat)
        d = d_feat.to(torch.float32).contiguous()
        M = feat.N * feat.T * feat.H * feat.W
        f32_accum = L.lib().step_f32_accum_f16 if feat.code == L.F16 else L.lib().step_f32_accum_f32
        L.check(f32_accum(L.ptr(d), M, feat.C, float(loss_scale), L.c_void_p(gfeat.data_ptr()), gfeat.ld, L.stream()))
        stem = tape[0]                                # the clip needs no gradient
        return tape_backward(tape, grads, loss_scale, need_input_grad=lambda e: e is not stem)


def _average_gradients(params_and_grads, world_size):
    """[(param, grad)] of the trainable parameters, the gradients averaged in place over the clip-parallel ranks (NCCL
    all-reduce of one flat bucket; an inf or NaN on any rank reaches every rank through the sum)."""
    items = [(p, g) for p, g in params_and_grads.items() if p.requires_grad]
    if world_size > 1 and items:
        import torch.distributed as dist
        flat = torch.cat([g.reshape(-1) for _, g in items])
        dist.all_reduce(flat, op=dist.ReduceOp.SUM)
        flat.div_(world_size)
        off = 0
        for _, g in items:
            g.copy_(flat[off:off + g.numel()].view_as(g))
            off += g.numel()
    return items


def sgd_step(params_and_grads, lr, momentum=0.9, weight_decay=0.0, state=None, world_size=1):
    """optim.SGD(momentum, weight_decay) (train.py:124) on the fp32 master parameters, after an optional gradient
    all-reduce over the clip-parallel ranks (NCCL; one flat bucket).  state: dict param -> momentum buffer.
    Host-side glue over torch.distributed + elementwise updates; the parameters change in place (their packed fp16
    copies are rebuilt by the modules' version-keyed caches on the next forward)."""
    state = {} if state is None else state
    items = _average_gradients(params_and_grads, world_size)
    with torch.no_grad():
        for p, g in items:
            g = g.to(p.device, p.dtype)
            if weight_decay:
                g = g.add(p, alpha=weight_decay)
            if momentum:
                buf = state.get(p)
                if buf is None:
                    buf = state[p] = g.clone()          # torch.optim.SGD: first step initialises the buffer with the gradient
                else:
                    buf.mul_(momentum).add_(g)
                g = buf
            p.add_(g, alpha=-lr)
    return state


def _sync_plan(cfg, nets, step_tubes, loss_scale, dev):
    """The refusals of a train_step whose heads synchronise their batch statistics, decided from one all-gather of every
    rank's number of steps, loss scale and per-step row counts, so that every rank raises the same error before anything
    changes.  Returns the rows of each step over all ranks."""
    import torch.distributed as dist
    from . import engine as E
    cap = int(cfg.max_iter)
    n_steps = len(step_tubes)
    mine = torch.zeros((2 + cap,), dtype=torch.float64)
    mine[0], mine[1] = n_steps, float(loss_scale)
    for i, t in enumerate(step_tubes[:cap]):
        mine[2 + i] = t.shape[0]
    plan = E.all_gather_rows(mine.to(dev), dist.group.WORLD).cpu()
    steps, scales, rows = plan[:, 0], plan[:, 1], plan[:, 2:]
    if bool((steps != steps[0]).any()) or bool((scales != scales[0]).any()):
        raise ValueError("train_step: the ranks disagree on the number of steps %s or the loss scale %s"
                         % (steps.long().tolist(), scales.tolist()))
    if n_steps > cap:
        raise ValueError("train_step: %d steps but cfg.max_iter = %d" % (n_steps, cap))
    rows = rows[:, :n_steps].long()
    if bool((rows == 0).any()):
        raise ValueError("train_step: a rank has no rows in some step (rows per rank and step: %s); synchronised batch "
                         "statistics need every rank to hold rows of every step" % rows.tolist())
    rows_total = rows.sum(0).tolist()
    for i in range(n_steps):
        head = nets["det_net%d" % i]
        values = rows_total[i] * step_frames(cfg, i + 1)[1] * head.pool_size ** 2
        if values < 2:
            raise ValueError("train_step: step %d's head BatchNorms would see %d value(s) per channel over all ranks: "
                             "Expected more than 1 value per channel when training" % (i + 1, values))
    return rows_total


def _broadcast_running_stats(bns):
    """Rank 0's running_mean, running_var and num_batches_tracked of every BatchNorm in bns to every rank: one broadcast of
    one flat byte buffer."""
    import torch.distributed as dist
    ts = [t for bn in bns for t in (bn.running_mean, bn.running_var, bn.num_batches_tracked)]
    if not ts:
        return
    flat = torch.cat([t.detach().reshape(-1).view(torch.uint8) for t in ts])
    dist.broadcast(flat, src=0)
    off = 0
    with torch.no_grad():
        for t in ts:
            n = t.numel() * t.element_size()
            t.copy_(flat[off:off + n].view(t.dtype).view_as(t))
            off += n


def step_frames(cfg, i):
    """(T_start, T_length) of refinement step i (1-based) -- train.py:294-298."""
    chunks = cfg.NUM_CHUNKS[i]
    return int((cfg.NUM_CHUNKS[cfg.max_iter] - chunks) / 2) * cfg.T, chunks * cfg.T


def train_step(cfg, nets, clips, step_tubes, step_targets, lr=None, momentum=0.9, weight_decay=0.0, lambda_reg=5.0,
               lambda_neighbor=1.0, loss_scale=1024.0, sgd_state=None, world_size=1, optimizer=None, scaler=None, dropout=False,
               trunk_stats_updated=False):
    """One optimisation step of train.py:263-348 on the device, for already selected training samples
    (`train_select`, utils/utils.py:135-423, is step_b200.select_samples, which returns step_tubes and step_targets):
        conv_feat = base_net(clips); context_feat = context_net(conv_feat) unless cfg.no_context      train.py:266-269
        for each refinement step i: T_start, T_length from cfg.NUM_CHUNKS / cfg.T / cfg.max_iter; ROI-pool the step's
            flat tubes from conv_feat[:, T_start:T_start+T_length]; run det_net[i-1] with targets and each tube's clip
            context over those frames;
            loss_back += loss_cls.mean() + lambda_reg * loss_loc.mean() + lambda_neighbor * loss_nb.mean()   train.py:294-336
        loss_back.backward(); optimizer.step()                                                             train.py:345-348
    step_tubes[i]: [R_i, T_length_i, 5] fp32 (frame index first, relative to the step's frame slice, as
    flatten_tubes(batch_idx=True) builds them), step_targets[i]: [R_i, 3, 6 + classes].
    Heads built with cls_only=True run the first training stage (train_cls.py:253-322, one step of T_length = cfg.T): their
    objective is loss_cls.mean() alone, and their gradients are those of Mixed_5b / Mixed_5c, `downsample` and `global_cls`.
    The gradient of conv_feat is, in this order, the ROI pooling backward of every step (each on its own frame slice) plus
    the context branch's; the pooling is nets['roi_net'].pool_mode's: ROIAlign ('align') or ROIPool ('pool', the
    reference's default, config.py:67), whose backward routes each gradient to the pixel of the maximum recorded by the
    step's forward.  Returns dict(loss, losses=[(cls, loc, nb)], grads={param: fp32 grad} (trunk, heads and, with
    the context branch, ContextNet's convolutions; with freeze_affine=False also every BatchNorm gamma / beta that requires
    grad), skipped, loss_scale).  When some BatchNorm's affine parameters train, a layer with a channel of gamma == 0 and
    beta > 0 raises ValueError before anything runs (check_bn_affine: one device-to-host read).
    Parameter update: with lr, `sgd_step` (one global rate); with optimizer (a step_b200.optim.Adam / SGD over the nets'
    parameters, e.g. built from the reference's get_params, and lr None), the gradients, averaged over the ranks, become
    p.grad and optimizer.step() runs -- it skips the update when a gradient is inf or NaN (skipped=True).  scaler (a
    step_b200.optim.LossScaler; needs optimizer) replaces loss_scale by its dynamic scale and is updated from the step.
    Precision: that of the nets (cfg.fp16, one value for all of them).  fp16 stores activations and their gradients in
    fp16 (apex O1-like); fp32 stores everything in fp32, the reference's default (config.py:26-27), and with
    loss_scale=1.0 and no scaler it is the reference's fp32 arithmetic.  Weight gradients and updates are fp32 on both.
    dropout=True: every head whose nn.Dropout is in training mode with 0 < p < 1 (the reference trains with --dropout 0.3,
    scripts/train_step.sh and train_cls.sh) draws its masks as the reference's training forward does, step by step, global
    then local, from the default CUDA generator of clips' device, and leaves that generator where those F.dropout calls
    leave it (head_forward_backward); nothing else here draws from it.  With one GPU this is the reference's draw sequence
    exactly.  Not in a CUDA graph: the draws move the generator's offset on the host.
    BatchNorm statistics: nets built with cfg.freeze_stats=False and in training mode (their train()) normalise with batch
    statistics in the trunk, ContextNet and heads, and the backward goes through them (step_bn_*).  Each head's running
    statistics are updated once by its forward.  trunk_stats_updated=True: the caller's own training-mode forward of
    base_net and context_net has already updated theirs (train.py:266-269); the step then normalises with the same batch
    statistics (the kernels are deterministic) and leaves their running statistics alone.  Without it the step updates
    them once.  A BatchNorm with momentum=None or track_running_stats=False raises ValueError before anything runs.
    Batch statistics with world_size > 1 (one process per GPU in the default process group of world_size ranks, rank r
    holding DataParallel's chunk r of the batch, clips [r * ceil(B / W), ...), and the rows its clips select) follow the
    reference's nn.DataParallel (train.py:141-148): the trunk and ContextNet normalise with each rank's own statistics and
    every rank ends with rank 0's running statistics (one broadcast); each head normalises with the statistics of every
    rank's rows of its step (engine.batch_stats_sync: an all-gather per convolution, forward and backward, and the same
    merge on every rank, so the heads' running statistics are identical on every rank).  The averaged gradients are those
    of (1 / W) sum_r L_r, the reference's whole-batch objective when every rank has the same rows in each step.  Without
    an initialised default process group this raises NotImplementedError; with one of another size, ranks that disagree on
    the number of steps or the loss scale, a rank with no rows in a step, or a head BatchNorm with fewer than 2 values per
    channel over all ranks, ValueError on every rank before anything changes (one all-gather up front)."""
    from . import engine as E
    from .engine import Act
    from .i3d import Unit3Dpy
    if optimizer is not None and lr is not None:
        raise ValueError("train_step: give either lr (sgd_step) or optimizer, not both")
    if scaler is not None:
        if optimizer is None:
            raise ValueError("train_step: scaler needs an optimizer (it is updated from optimizer.found_inf)")
        loss_scale = scaler.scale
    base, roi_net = nets["base_net"], nets["roi_net"]
    check_bn_affine(nets)
    stats_units = [m for mod in nets.values() if mod is not None for m in mod.modules()
                   if isinstance(m, Unit3Dpy) and m.batch_stats()]
    sync = bool(stats_units) and world_size > 1
    if sync:
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()):
            raise NotImplementedError("train_step: BatchNorm batch statistics (freeze_stats=False) with world_size > 1 need the "
                                      "default process group of the world_size ranks (torch.distributed.init_process_group): "
                                      "the heads' statistics are exchanged between the ranks")
        if dist.get_world_size() != world_size:
            raise ValueError("train_step: world_size=%d but the default process group has %d ranks"
                             % (world_size, dist.get_world_size()))
    for m in stats_units:
        E.check_batch_stats_bn(m.batch3d)
    pool_mode = roi_net.pool_mode
    if pool_mode not in ("align", "pool"):
        raise RuntimeError("train_step: ROINet pool_mode %r is neither 'align' nor 'pool'" % pool_mode)
    use_ctx = not getattr(cfg, "no_context", True)
    if use_ctx and nets.get("context_net") is None:
        raise RuntimeError("train_step: cfg.no_context is False but nets has no 'context_net'")
    dev = clips.device
    n_steps = len(step_tubes)
    rows_total = _sync_plan(cfg, nets, step_tubes, loss_scale, dev) if sync else None
    results = []
    all_grads = {}

    def d_feat(feat):
        # ContextNet and the heads first (they need conv_feat), then the sum of their conv_feat gradients is the trunk's
        # output gradient
        B, T_all = feat.N, feat.T
        ctx = ctx_state = d_ctx = None
        if use_ctx:
            ctx, ctx_state = context_forward(nets["context_net"], feat)                     # [B, T', 1024] fp32
            d_ctx = torch.zeros_like(ctx)
        total = torch.zeros((B * T_all, feat.H, feat.W, feat.C), dtype=torch.float32, device=dev)
        ws = None
        for i in range(n_steps):
            head = nets["det_net%d" % i]
            t_start, t_len = step_frames(cfg, i + 1)
            flat = step_tubes[i].to(dev).float().contiguous()
            R = flat.shape[0]
            if flat.shape[1] != t_len or t_start + t_len > T_all:
                raise RuntimeError("train_step: step %d pools frames [%d, %d) of T'=%d (cfg.T=%d, NUM_CHUNKS=%s) but its tubes have %d frames"
                                   % (i + 1, t_start, t_start + t_len, T_all, cfg.T, cfg.NUM_CHUNKS, flat.shape[1]))
            cat = Act.empty(R, t_len, head.pool_size, head.pool_size, 832 + head.fc_dim, feat.code, dev)
            argmax = None
            if pool_mode == "pool":   # the pixel of every maximum, for this step's ROIPool backward
                argmax = torch.empty((R * t_len * head.pool_size * head.pool_size * feat.C,), dtype=torch.int32, device=dev)
            roi_net.pool_into(feat, flat, cat.frames().slice(0, 832), t_len, T_all, t_start, argmax=argmax)
            context = None
            if use_ctx:
                # per-clip mean of the context over the step's frames; row_map = clip of each tube (train.py:317-321)
                sl = ctx[:, t_start:]
                ctx_mean = torch.empty((B, ctx.shape[2]), dtype=torch.float32, device=dev)
                L.check(L.lib().step_mean_mid_strided(L.c_void_p(sl.data_ptr()), L.F32, B, t_len, 1, ctx.shape[2], ctx.shape[2],
                                                      T_all * ctx.shape[2], L.ptr(ctx_mean), L.F32, L.stream()))
                row_map = torch.div(flat[:, 0, 0], float(t_len), rounding_mode="floor").to(torch.int32)
                context = (ctx_mean, row_map, ctx, t_start)
            # the heads' statistics: one update per step; with several ranks, those of every rank's rows of the step
            sync_heads = E.batch_stats_sync(dist.group.WORLD, rows_total[i]) if sync else contextlib.nullcontext()
            with E.running_stats_update(True), sync_heads:
                r = head_forward_backward(head, None, flat, step_targets[i].to(dev), context_feat=context, lambda_reg=lambda_reg,
                                          lambda_neighbor=lambda_neighbor, loss_scale=loss_scale, cat=cat, dropout=dropout)
            results.append(r)
            all_grads.update(r["grads"])
            if use_ctx and r["ctx_dropout"] is not None:
                context_grad_reduce(r["ctx_grad"], flat, d_ctx, t_start, dropout=r["ctx_dropout"])
            elif use_ctx:
                context_grad_reduce(r["ctx_grad"], flat, d_ctx, t_start)
            with _phase("roi_bwd"):
                if pool_mode == "pool":
                    roi_pool_backward_slice(r["roi_grad"], flat.view(-1, 5), argmax, total, t_len, T_all, t_start)
                else:
                    ws = roi_align_backward_slice(r["roi_grad"], flat.view(-1, 5), 1.0 / 16.0, total, t_len, T_all, t_start, ws=ws)
            argmax = None
        if use_ctx:
            cg, gfeat = context_backward(ctx_state, d_ctx, loss_scale)
            all_grads.update(cg)
            total.add_(gfeat.reshape(B * T_all, feat.H, feat.W, feat.C).float())             # scaled by loss_scale too
        return total.mul_(1.0 / loss_scale).view(B, T_all, feat.H, feat.W, feat.C)

    # the trunk's and ContextNet's forwards (d_feat runs ContextNet) update their running statistics unless the caller's did
    with E.running_stats_update(not trunk_stats_updated):
        feat, tg = trunk_forward_backward(base, clips, d_feat, loss_scale)
    all_grads.update(tg)
    if sync:   # DataParallel keeps device 0's replica's update of the trunk's and ContextNet's running statistics
        _broadcast_running_stats([m.batch3d for k in ("base_net", "context_net") if nets.get(k) is not None
                                  for m in nets[k].modules() if isinstance(m, Unit3Dpy) and m.batch_stats()])
    loss = sum(r["loss"] for r in results)
    skipped = False
    if optimizer is not None:
        for p, g in _average_gradients(all_grads, world_size):
            p.grad = g
        optimizer.step()
        skipped = bool(optimizer.found_inf)
        if scaler is not None:
            scaler.update(skipped)
    elif lr is not None:
        sgd_state = sgd_step(all_grads, lr, momentum, weight_decay, sgd_state, world_size)
    return dict(loss=loss, losses=[r["losses"] for r in results], grads=all_grads, sgd_state=sgd_state, skipped=skipped,
                loss_scale=loss_scale)
