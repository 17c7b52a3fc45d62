"""GPU: the space-to-depth stem kernel (csrc/conv_stem.cu) -- the stride-2 7x7x7 stem as a 4x4x4 filter over the 24 live
channels of the s2d clip, with pack_stem_s2d weights and folded BatchNorm."""
import os
import sys

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from step_b200 import _lib as L
from step_b200 import engine as E
from step_b200.engine import Act
from step_b200.i3d import Unit3Dpy

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _tape_reference as R  # noqa: E402

pytestmark = pytest.mark.gpu

# N, T, H, W of the clip; the s2d map is half of T, H, W
SHAPES = [
    (2, 8, 224, 224),      # the C4 plane size (112 x 112), whole 4 x 16 x 8 tiles
    (1, 10, 38, 26),       # s2d 5 x 19 x 13: ragged t, h and w tiles
    (3, 6, 34, 50),        # s2d 3 x 17 x 25
]


def _stem(seed):
    g = torch.Generator().manual_seed(seed)
    unit = Unit3Dpy(3, 64, kernel_size=(7, 7, 7), stride=(2, 2, 2))
    with torch.no_grad():
        unit.conv3d.weight.copy_(torch.randn(64, 3, 7, 7, 7, generator=g) / 1029 ** 0.5)
        bn = unit.batch3d
        bn.weight.copy_(torch.rand(64, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(64, generator=g) * 0.3)
        bn.running_mean.copy_(torch.randn(64, generator=g) * 0.1)
        bn.running_var.copy_(torch.rand(64, generator=g) + 0.5)
    return unit.cuda().eval()


def _clip(shape, seed):
    N, T, H, W = shape
    g = torch.Generator().manual_seed(seed)
    return torch.randn(N, T, 3, H, W, generator=g).cuda()


def _s2d(clip, pad_fill=None):
    N, T, C, H, W = clip.shape
    s2d = Act.empty(N, T // 2, H // 2, W // 2, 32, L.F16, clip.device)
    L.check(L.lib().step_clip_to_s2d_f16(L.ptr(clip), N, T, C, H, W, L.ptr(s2d.buf), 32, L.stream()))
    if pad_fill is not None:
        s2d.buf[..., 24:] = pad_fill
    return s2d


@pytest.mark.parametrize("shape", SHAPES)
def test_stem_kernel_matches_fp32_simt_stem(shape):
    """against the stride-2 fp32 SIMT convolution of the same layer; channels 24..31 of the s2d input hold NaN, so a read
    of them would poison the output."""
    unit = _stem(1)
    clip = _clip(shape, 2)
    N, T, H, W = shape
    got = unit.forward_s2d(_s2d(clip, float("nan"))).buf.float()
    a = Act.empty(N, T, H, W, 4, L.F32, clip.device)
    L.check(L.lib().step_clip_to_ndhwc(L.ptr(clip), N, T, 3, H, W, L.ptr(a.buf), L.F32, 4, L.stream()))
    ref = unit(a).buf
    torch.cuda.synchronize()
    assert got.shape == ref.shape
    assert bool(torch.isfinite(got).all())
    err = float((got - ref).abs().max())
    assert err <= 2e-2 * float(ref.abs().max()), err


@pytest.mark.parametrize("shape", SHAPES)
def test_stem_kernel_matches_32_channel_patch_kernel(shape):
    """against the generic patch kernel (conv_halo.cu) on today's 32-channel problem with zero padding channels: the
    same products except the zero ones, summed in another order."""
    unit = _stem(3)
    s2d = _s2d(_clip(shape, 4), 0.0)
    got = unit.forward_s2d(s2d).buf.float()
    w, scale, shift = unit.packed(L.F16, s2d=True)
    ref = Act.empty(s2d.N, s2d.T, s2d.H, s2d.W, 64, L.F16, s2d.device)
    E.conv(s2d, w, scale, shift, ref, (4, 4, 4), (1, 1, 1), (1, 1, 1), True, a_mode=L.A_HALO,
           out_dims=(s2d.T, s2d.H, s2d.W))
    torch.cuda.synchronize()
    ref = ref.buf.float()
    err = float((got - ref).abs().max())
    assert err <= 2e-3 * float(ref.abs().max()), err
    # and against the float64 4x4x4 / pad-1 convolution of the 24 live channels (bound: test_gpu_forward_layers.py)
    (y,), (xw,), (epi,) = R.conv_fwd(s2d.buf[..., :24], w, scale, shift, None, (4, 4, 4), (1, 1, 1), (1, 1, 1),
                                     (s2d.T, s2d.H, s2d.W), True)
    R.check_fwd(got, y, xw, epi, R.conv_steps((4, 4, 4), 24), shape)


def test_stem_shape_reaches_the_stem_kernel():
    """forward_s2d's problem (24 channels in a 32-channel row, pack_stem_s2d weights) runs conv_stem_kernel, and the
    32-channel problem still runs the generic patch kernel."""
    unit = _stem(5)
    s2d = _s2d(_clip((1, 8, 64, 64), 6), 0.0)
    unit.forward_s2d(s2d)                                  # weights packed outside the profiled window
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        unit.forward_s2d(s2d)
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    assert any("conv_stem_kernel" in k for k in names), names
    assert not any("conv_halo_kernel" in k for k in names), names
    w, scale, shift = unit.packed(L.F16, s2d=True)
    out = Act.empty(s2d.N, s2d.T, s2d.H, s2d.W, 64, L.F16, s2d.device)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        E.conv(s2d, w, scale, shift, out, (4, 4, 4), (1, 1, 1), (1, 1, 1), True, a_mode=L.A_HALO,
               out_dims=(s2d.T, s2d.H, s2d.W), zero_cin_last_kt=12)
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    assert any("conv_halo_kernel" in k for k in names), names
