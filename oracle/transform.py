"""TEST INFRASTRUCTURE ONLY -- numpy model of step_frames_to_clip_u8's arithmetic (step_b200/csrc/clip_prep.cu), i.e. of the
reference's BaseTransform (data/augmentations.py:601-615) as cv2 4.x computes it without IPP, followed by the dataset's
swap to RGB and permute.  tests/test_transform_model.py pins it bit for bit to tests/golden/transform_cases.npz (the
reference itself, run by tests/golden/make_transform_golden.py); the GPU tests then hold the kernel to the same goldens."""
import numpy as np

F32 = np.float32


def convert(u, scale):
    """ConvertFromInts: every step rounded in fp32."""
    x = u.astype(F32)
    if scale == 2:
        return (x * F32(2) / F32(255) - F32(1)).astype(F32)
    if scale == 1:
        return (x / F32(255)).astype(F32)
    return x


def linear_taps(n_dst, n_src, clamp_weight):
    """cv2 resize.cpp INTER_LINEAR: f = (float)((d + 0.5) * (1 / ((double)n_dst / n_src)) - 0.5), s = floor(f), f -= s.
    Columns clamp the tap and zero the weight at both ends; rows clip the tap indices only and keep the unclamped
    weight, so a border row is a replicated row weighted by (1 - f) and f, which can differ from it by an ulp."""
    scale = 1.0 / (float(n_dst) / n_src)
    f = ((np.arange(n_dst) + 0.5) * scale - 0.5).astype(F32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(F32)).astype(F32)
    if clamp_weight:
        lo, hi = s < 0, s >= n_src - 1
        f[lo | hi] = 0
        s[lo] = 0
        s[hi] = n_src - 1
    return np.clip(s, 0, n_src - 1), np.clip(s + 1, 0, n_src - 1), f


def resize(S, H, W):
    """cv2.resize(S, (W, H)) of one float32 frame S [H0, W0, C] (INTER_LINEAR, generic code)."""
    H0, W0 = S.shape[:2]
    if H0 == 2 * H and W0 == 2 * W:  # cv2 switches to INTER_AREA's fast path here
        a, b, c, d = S[0::2, 0::2], S[0::2, 1::2], S[1::2, 0::2], S[1::2, 1::2]
        return ((((a + b) + c) + d) * F32(0.25)).astype(F32)
    x0, x1, fx = linear_taps(W, W0, True)
    y0, y1, fy = linear_taps(H, H0, False)
    h = (S[:, x0] * (F32(1) - fx)[None, :, None] + S[:, x1] * fx[None, :, None]).astype(F32)
    return (h[y0] * (F32(1) - fy)[:, None, None] + h[y1] * fy[:, None, None]).astype(F32)


def base_transform(frames_rgb, size, mean=(0, 0, 0), stds=(1, 1, 1), scale=1):
    """frames_rgb: uint8 [T, 3, H0, W0] (after the dataset's swap); size = (W, H); mean / stds in BGR order as the
    reference's constructor takes them.  Returns fp32 [T, 3, H, W]."""
    W, H = size
    mean = np.asarray(mean, F32)[::-1]
    stds = np.asarray(stds, F32)[::-1]
    out = []
    for fr in frames_rgb:
        r = resize(convert(np.ascontiguousarray(fr.transpose(1, 2, 0)), scale), H, W)
        out.append((((r - mean).astype(F32)) / stds).astype(F32).transpose(2, 0, 1))
    return np.stack(out).astype(F32)
