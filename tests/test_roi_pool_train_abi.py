"""CPU: the ROIPool training entries (step_roi_pool_fwd_argmax_nhwc, step_roi_pool_bwd_slice_nhwc) validate their arguments
before any device work: STEP_E_ARG and a step_last_error() text that names the problem, for a null pointer, channel counts
that are not whole 16-byte vectors, a frame map outside the feature map, and a map larger than the backward's shared-memory
accumulator holds."""
import ctypes

import pytest

from step_b200 import _lib


@pytest.fixture(scope="module")
def lib():
    return _lib.lib()


@pytest.fixture(scope="module")
def buf():
    b = (ctypes.c_char * (4096 + 16))()
    addr = (ctypes.addressof(b) + 15) & ~15                 # 16-byte aligned fake device pointer (never dereferenced)
    return b, ctypes.c_void_p(addr)


def fwd(lib, p, dtype=_lib.F32, K=9, H=8, W=8, C=16, feat_ld=16, R=4, out_ld=16, roi_T=3, feat_T=9, t_start=3, argmax="p",
        feat="p", rois="p", out="p"):
    pick = lambda v: p if v == "p" else v
    return lib.step_roi_pool_fwd_argmax_nhwc(pick(feat), dtype, K, H, W, C, feat_ld, pick(rois), R, 1.0 / 16.0, 7, 7, pick(out),
                                             out_ld, roi_T, feat_T, t_start, pick(argmax), None)


def bwd(lib, p, dtype=_lib.F16, out_ld=16, R=4, K=9, H=8, W=8, C=16, roi_T=3, feat_T=9, t_start=3, in_ld=16, grad_out="p",
        argmax="p", rois="p", grad_in="p"):
    pick = lambda v: p if v == "p" else v
    return lib.step_roi_pool_bwd_slice_nhwc(pick(grad_out), dtype, out_ld, pick(argmax), pick(rois), R, 7, 7, K, H, W, C, roi_T,
                                            feat_T, t_start, pick(grad_in), in_ld, None)


def expect(lib, rc, *words):
    assert rc == _lib.E_ARG
    msg = lib.step_last_error().decode()
    for w in words:
        assert w in msg, (w, msg)


@pytest.mark.parametrize("which", ["feat", "rois", "out", "argmax"])
def test_forward_null_pointer(lib, buf, which):
    expect(lib, fwd(lib, buf[1], **{which: None}), "roi_pool_fwd_argmax_nhwc", "null pointer")


def test_forward_misaligned_channels_and_argmax(lib, buf):
    p = buf[1]
    expect(lib, fwd(lib, p, C=6, feat_ld=8, out_ld=8), "C=6", "multiples of 4")
    expect(lib, fwd(lib, p, dtype=_lib.F16, C=12, feat_ld=16, out_ld=16), "C=12", "multiples of 8")
    expect(lib, fwd(lib, p, feat_ld=18), "feat_ld=18")
    expect(lib, fwd(lib, p, argmax=ctypes.c_void_p(p.value + 4)), "argmax must be 16-byte aligned")


@pytest.mark.parametrize("fm", [(3, 9, 7), (3, 9, -1), (-1, 9, 0)])
def test_forward_bad_frame_map(lib, buf, fm):
    roi_T, feat_T, t_start = fm
    expect(lib, fwd(lib, buf[1], roi_T=roi_T, feat_T=feat_T, t_start=t_start), "bad frame map")


def test_forward_map_above_backward_limit(lib, buf):
    expect(lib, fwd(lib, buf[1], H=81, W=81), "H*W=6561", "6400")
    assert fwd(lib, buf[1], R=0, H=81, W=81) == 0           # no ROI: nothing to pool, no launch


@pytest.mark.parametrize("which", ["grad_out", "argmax", "rois", "grad_in"])
def test_backward_null_pointer(lib, buf, which):
    expect(lib, bwd(lib, buf[1], **{which: None}), "roi_pool_bwd_slice_nhwc", "null pointer")


def test_backward_misaligned_channels_and_grad_in(lib, buf):
    p = buf[1]
    expect(lib, bwd(lib, p, C=6, in_ld=8, out_ld=8), "C=6", "multiples of 4")
    expect(lib, bwd(lib, p, in_ld=18), "in_ld=18")
    expect(lib, bwd(lib, p, out_ld=8), "out_ld=8")
    expect(lib, bwd(lib, p, grad_in=ctypes.c_void_p(p.value + 4)), "grad_in must be 16-byte aligned")
    expect(lib, bwd(lib, p, dtype=7), "bad dtype")


@pytest.mark.parametrize("fm", [(3, 9, 7, 9), (3, 9, -1, 9), (0, 9, 0, 9), (3, 9, 3, 10), (3, 0, 0, 9)])
def test_backward_bad_frame_map(lib, buf, fm):
    roi_T, feat_T, t_start, K = fm
    expect(lib, bwd(lib, buf[1], roi_T=roi_T, feat_T=feat_T, t_start=t_start, K=K), "bad frame map")


def test_backward_map_above_shared_memory_limit(lib, buf):
    expect(lib, bwd(lib, buf[1], H=81, W=81), "H*W=6561", "6400-pixel limit")
    expect(lib, bwd(lib, buf[1], R=0, H=101, W=64), "H*W=6464")   # checked even when there is no ROI


def test_python_wrappers_reject_bad_argmax():
    import torch
    import step_b200
    from step_b200 import training
    from step_b200.engine import Act
    net = step_b200.ROINet("align", 7)
    with pytest.raises(RuntimeError, match="'pool' mode only"):
        net.pool_into(None, torch.zeros(1, 1, 5), None, 1, 1, 0, argmax=torch.zeros(49 * 8, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="argmax"):
        training.roi_pool_backward_slice(Act(torch.zeros(1, 1, 7, 7, 8)), torch.zeros(1, 5), torch.zeros(10, dtype=torch.int32),
                                         torch.zeros(1, 4, 4, 8), 1, 1, 0)
