"""Drop-in for `external.maskrcnn_benchmark.roi_layers` of the reference
(roi_layers/__init__.py:29-35): `nms`, `roi_align`, `ROIAlign`, `roi_pool`, `ROIPool` with the same
names, argument order, return types and error behaviour, implemented by libstep_b200.so.

Reference call sites: models/networks.py:28-31,44 (ROIAlign/ROIPool), test.py:192 / demo.py:158 /
train.py:547 (nms).

The ROIAlign / ROIPool backwards have no atomics (the reference's scatter with atomicAdd): their gradients repeat bit for
bit from run to run and on any stream, and equal the channels-last backward of training.train_step transposed
(tests/test_gpu_roi_bwd_det.py).
"""
import torch
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable
from torch.nn.modules.utils import _pair

from . import _lib as L

import functools

# One cached workspace per (device, stream) for the single-problem NMS entry point.
_nms_ws = {}


def _on_device_of(argpos):
    """Run the wrapped op with the CUDA device of its `argpos`-th argument current, so that allocations and the launch
    stream (L.stream()) belong to the device that owns the tensors (multi-GPU drivers: test.py:79-95)."""
    def deco(fn):
        @functools.wraps(fn)
        def wrapped(*a, **k):
            t = a[argpos]
            if torch.is_tensor(t) and t.is_cuda:
                with torch.cuda.device(t.device):
                    return fn(*a, **k)
            return fn(*a, **k)
        return wrapped
    return deco


def _workspace(device, nbytes):
    key = (device, torch.cuda.current_stream(device).cuda_stream)   # two streams must not share scratch memory
    buf = _nms_ws.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
        _nms_ws[key] = buf
    return buf


def nms(dets, scores, threshold):
    """nms(dets float[n,4], scores float[n], threshold) -> int64[k] kept original indices, ascending
    (roi_layers/nms.py:38 -> csrc/nms.h:34-51).

    CUDA tensors: runs on the tensors' device, returns a CUDA int64 tensor (as nms_cuda does).
    CPU tensors: every reference driver calls nms with CPU tensors (test.py:192); there is no CPU
    kernel here, so the rows are moved to the current CUDA device, resolved there with the CPU
    op's exact semantics (suppress when IoU >= thr, cpu/nms_cpu.cpp:84) and the indices are returned
    on the CPU.  Ties between equal scores are visited in ascending index order; NaN scores rank above every number,
    where scores.sort(descending=True) (nms_cpu.cpp:48) puts them, and -0.0 ties with +0.0.
    """
    if dets.dtype not in (torch.float32, torch.float64):
        raise RuntimeError('"nms" not implemented for \'%s\'' % str(dets.dtype).replace("torch.", ""))
    was_cpu = not dets.is_cuda
    if dets.numel() == 0:  # nms.h:41-42 / nms_cpu.cpp:37-39
        return torch.empty((0,), dtype=torch.int64, device="cpu")
    if not torch.cuda.is_available():
        raise RuntimeError("step_b200.nms: no CUDA device (there is no CPU fallback)")
    dev = dets.device if dets.is_cuda else torch.device("cuda", torch.cuda.current_device())
    boxes = dets.detach().to(device=dev, dtype=torch.float32).contiguous()
    sc = scores.detach().to(device=dev, dtype=torch.float32).contiguous()
    n = boxes.shape[0]
    if boxes.dim() != 2 or boxes.shape[1] != 4 or sc.numel() != n:
        raise RuntimeError("nms: expected dets [n,4] and scores [n]")
    with torch.cuda.device(dev):
        ws_bytes = L.lib().step_nms_workspace_bytes(n)
        ws = _workspace(dev, ws_bytes)
        keep = torch.empty((n,), dtype=torch.int64, device=dev)
        cnt = torch.empty((1,), dtype=torch.int32, device=dev)
        L.check(L.lib().step_nms_f32(L.ptr(boxes), L.ptr(sc), n, float(threshold), 1 if was_cpu else _CUDA_GE,
                                     L.ptr(keep), L.ptr(cnt), L.ptr(ws), ws.numel(), L.stream()))
        k = int(cnt.item())  # output length is data dependent: the one unavoidable D2H
    out = keep[:k]
    return out.cpu() if was_cpu else out


# The reference's CUDA kernel suppresses on '>' (cuda/nms.cu:84) while its CPU kernel uses '>='
# (cpu/nms_cpu.cpp:84).  All reference drivers use the CPU op, so '>=' is the exercised semantics;
# CUDA-tensor calls default to it too.  Set to 0 to reproduce nms.cu exactly.
_CUDA_GE = 1


@_on_device_of(0)
def nms_segmented(boxes, scores, seg_offsets, threshold, min_score=float("-inf"), ge=True, max_seg_rows=None):
    """Batched form of the per-clip x per-class loop of test.py:178-201: rows
    [seg_offsets[s], seg_offsets[s+1]) are independent NMS problems (<= 1024 rows each: pass the longest segment as
    `max_seg_rows` when the host knows it, otherwise it is read back once).  Only rows with score >= min_score take
    part: a NaN score never does, as scores.gt(conf_thresh) drops it in test.py:180 (unlike `nms`, which ranks it first).
    Returns a uint8 keep mask over all rows; stays on device."""
    L.same_device(boxes, scores, seg_offsets)
    if max_seg_rows is None:   # the host knows the segment lengths in every caller of ours; a stray caller pays one sync
        max_seg_rows = int((seg_offsets[1:] - seg_offsets[:-1]).max().item()) if seg_offsets.numel() > 1 else 0
    if max_seg_rows > L.lib().step_nms_segmented_max_rows():
        raise RuntimeError("nms_segmented: a segment of %d rows exceeds the %d-row shared-memory problem size"
                           % (max_seg_rows, L.lib().step_nms_segmented_max_rows()))
    boxes = boxes.contiguous().float()
    scores = scores.contiguous().float()
    seg_offsets = seg_offsets.contiguous().to(torch.int32)
    mask = torch.empty((boxes.shape[0],), dtype=torch.uint8, device=boxes.device)
    L.check(L.lib().step_nms_segmented_f32(L.ptr(boxes), L.ptr(scores), L.ptr(seg_offsets),
                                           seg_offsets.numel() - 1, float(threshold), 1 if ge else 0,
                                           float(min_score), L.ptr(mask), L.stream()))
    return mask


def _is_channels_last(x):
    # [K,C,H,W] logical shape whose memory is [K,H,W,C] (possibly a channel slice of a wider buffer)
    return x.dim() == 4 and x.stride(1) == 1 and x.stride(3) >= x.shape[1] and \
        x.stride(2) == x.shape[3] * x.stride(3) and x.stride(0) == x.shape[2] * x.stride(2)


class _ROIAlign(Function):
    """roi_layers/roi_align.py:45-76"""

    @staticmethod
    @_on_device_of(1)
    def forward(ctx, input, roi, output_size, spatial_scale, sampling_ratio):
        ctx.save_for_backward(roi)
        ctx.output_size = _pair(output_size)
        ctx.spatial_scale = spatial_scale
        ctx.sampling_ratio = sampling_ratio
        ctx.input_shape = input.size()
        L.same_device(input, roi)  # "no CPU fallback": ROIAlign.h:46 path is not reproduced
        ph, pw = ctx.output_size
        K, C, H, W = input.shape
        rois = roi.detach().to(torch.float32).contiguous()
        R = rois.shape[0]
        if input.dtype == torch.float64:
            raise RuntimeError("roi_align: float64 is not supported by the sm_90a kernels")
        if _is_channels_last(input) and input.dtype in (torch.float16, torch.float32) and C % 8 == 0:
            # channels-last storage (our own modules produce it): fast path, output keeps the layout
            ld = input.stride(3)
            out = torch.empty((R, ph, pw, C), dtype=input.dtype, device=input.device)
            L.check(L.lib().step_roi_align_fwd_nhwc(L.ptr(input), L.dt(input), K, H, W, C, ld, L.ptr(rois), R,
                                                    float(spatial_scale), ph, pw, int(sampling_ratio),
                                                    L.ptr(out), C, 0, 0, 0, 1, L.stream()))
            return out.permute(0, 3, 1, 2)
        x = input.detach().to(torch.float32).contiguous()  # ROIAlign_cuda.cu:310 does .contiguous() too
        out = torch.empty((R, C, ph, pw), dtype=torch.float32, device=input.device)
        L.check(L.lib().step_roi_align_fwd_nchw_f32(L.ptr(x), K, C, H, W, L.ptr(rois), R, float(spatial_scale),
                                                    ph, pw, int(sampling_ratio), L.ptr(out), L.stream()))
        return out.to(input.dtype)

    @staticmethod
    @once_differentiable
    @_on_device_of(1)
    def backward(ctx, grad_output):
        rois, = ctx.saved_tensors
        ph, pw = ctx.output_size
        bs, ch, h, w = ctx.input_shape
        L.need_cuda(grad_output)
        g = grad_output.to(torch.float32).contiguous()
        r = rois.detach().to(torch.float32).contiguous()
        gin = torch.empty((bs, ch, h, w), dtype=torch.float32, device=g.device)
        L.check(L.lib().step_roi_align_bwd_nchw_f32(L.ptr(g), L.ptr(r), r.shape[0], float(ctx.spatial_scale), ph, pw,
                                                    bs, ch, h, w, int(ctx.sampling_ratio), L.ptr(gin), L.stream()))
        return gin.to(grad_output.dtype), None, None, None, None


roi_align = _ROIAlign.apply


class ROIAlign(nn.Module):
    """roi_layers/roi_align.py:82-101"""

    def __init__(self, output_size, spatial_scale, sampling_ratio):
        super(ROIAlign, self).__init__()
        self.output_size = output_size
        self.spatial_scale = spatial_scale
        self.sampling_ratio = sampling_ratio

    def forward(self, input, rois):
        return roi_align(input, rois, self.output_size, self.spatial_scale, self.sampling_ratio)

    def __repr__(self):
        return "%s(output_size=%s, spatial_scale=%s, sampling_ratio=%s)" % (
            self.__class__.__name__, self.output_size, self.spatial_scale, self.sampling_ratio)


class _ROIPool(Function):
    """roi_layers/roi_pool.py:45-79"""

    @staticmethod
    @_on_device_of(1)
    def forward(ctx, input, roi, output_size, spatial_scale):
        ctx.output_size = _pair(output_size)
        ctx.spatial_scale = spatial_scale
        ctx.input_shape = input.size()
        L.need_cuda(input, roi)
        ph, pw = ctx.output_size
        K, C, H, W = input.shape
        x = input.detach().to(torch.float32).contiguous()
        rois = roi.detach().to(torch.float32).contiguous()
        R = rois.shape[0]
        out = torch.empty((R, C, ph, pw), dtype=torch.float32, device=input.device)
        argmax = torch.empty((R, C, ph, pw), dtype=torch.int32, device=input.device)
        L.check(L.lib().step_roi_pool_fwd_nchw_f32(L.ptr(x), K, C, H, W, L.ptr(rois), R, float(spatial_scale), ph, pw,
                                                   L.ptr(out), L.ptr(argmax), L.stream()))
        ctx.save_for_backward(rois, argmax)
        return out.to(input.dtype)

    @staticmethod
    @once_differentiable
    @_on_device_of(1)
    def backward(ctx, grad_output):
        rois, argmax = ctx.saved_tensors
        ph, pw = ctx.output_size
        bs, ch, h, w = ctx.input_shape
        g = grad_output.to(torch.float32).contiguous()
        gin = torch.empty((bs, ch, h, w), dtype=torch.float32, device=g.device)
        L.check(L.lib().step_roi_pool_bwd_nchw_f32(L.ptr(g), L.ptr(argmax), L.ptr(rois), rois.shape[0], ph, pw, bs,
                                                   ch, h, w, L.ptr(gin), L.stream()))
        return gin.to(grad_output.dtype), None, None, None


roi_pool = _ROIPool.apply


class ROIPool(nn.Module):
    """roi_layers/roi_pool.py:82-98"""

    def __init__(self, output_size, spatial_scale):
        super(ROIPool, self).__init__()
        self.output_size = output_size
        self.spatial_scale = spatial_scale

    def forward(self, input, rois):
        return roi_pool(input, rois, self.output_size, self.spatial_scale)

    def __repr__(self):
        return "%s(output_size=%s, spatial_scale=%s)" % (self.__class__.__name__, self.output_size, self.spatial_scale)


__all__ = ["nms", "roi_align", "ROIAlign", "roi_pool", "ROIPool", "nms_segmented"]
