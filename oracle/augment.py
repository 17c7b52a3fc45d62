"""TEST INFRASTRUCTURE ONLY -- numpy model of step_frames_to_clip_aug_u8's arithmetic (step_b200/csrc/clip_prep.cu), i.e. of
the reference's TubeAugmentation (data/augmentations.py:540-589) as cv2 4.x computes it without IPP, applied to the recipe
the host stage (step_b200.transforms.TubeAugmentation) drew, followed by the dataset's swap to RGB and permute.
tests/test_augment_cpu.py pins it bit for bit to tests/golden/augment_cases.npz (the reference itself, run by
tests/golden/make_augment_golden.py); the GPU tests then hold the kernel to the same goldens.

cv2's float32 HSV conversions (color_hsv.simd.hpp), as probed on cv2 4.13 against random pixels in [-40, 300]:
  BGR2HSV  v = max(b, g, r), diff = v - min(b, g, r), s = diff / (|v| + FLT_EPSILON), d = 60 / (diff + FLT_EPSILON) and
           h = fma(num, d, offset) with num = g - b (offset 0, or 360 when num < 0), b - r (120) or r - g (240) by the
           channel holding v.  That is its 8-lane vector loop.  The last W0 % 8 pixels of each row take the scalar loop:
           h = fma(num, d, offset without the 360), then h += 360 where h < 0.  Both match bit for bit.
  HSV2BGR  h6 = h * (6 / 360), sector = trunc(h6) mod 6, f = h6 - trunc(h6) and the table v, v * (1 - s),
           v * fma(-s, f, 1), v * fma(-s, 1 - f, 1) (the compiler fuses those two in both loops).  Bit for bit as well.
With IPP on, cv2 takes another HSV2BGR, whose results differ from these in the last bits."""
import numpy as np

from . import transform as ot

F32 = np.float32
FLT_EPSILON = F32(np.finfo(np.float32).eps)
HSV_LANES = 8


def fma(a, b, c):
    """fp32 fused multiply-add, correctly rounded: a * b is exact in float64, the sum's rounding error is recovered and
    settles the one case where rounding the float64 sum to fp32 again goes wrong (a tie)."""
    a, b = np.asarray(a, F32).astype(np.float64), np.asarray(b, F32).astype(np.float64)
    c = np.asarray(c, F32).astype(np.float64)
    p = a * b
    s = p + c
    t = s - p
    err = (p - (s - t)) + (c - t)
    r = s.astype(F32)
    r64 = r.astype(np.float64)
    other = np.where(s > r64, np.nextafter(r, F32(np.inf)), np.nextafter(r, F32(-np.inf)))
    tie = (s == (r64 + other.astype(np.float64)) / 2) & (err != 0)
    toward = np.sign(err) == np.sign(other.astype(np.float64) - r64)
    return np.where(tie & toward, other, r).astype(F32)


def bgr2hsv(x):
    """cv2.cvtColor(x, COLOR_BGR2HSV) of fp32 frames [..., W0, 3] (H in degrees)."""
    b, g, r = x[..., 0], x[..., 1], x[..., 2]
    v = np.maximum(np.maximum(r, g), b)
    diff = (v - np.minimum(np.minimum(r, g), b)).astype(F32)
    s = (diff / (np.abs(v) + FLT_EPSILON)).astype(F32)
    d = (F32(60) / (diff + FLT_EPSILON)).astype(F32)
    red, green = r == v, g == v
    num = np.where(red, g - b, np.where(green, b - r, r - g)).astype(F32)
    offset = np.where(red, F32(0), np.where(green, F32(120), F32(240))).astype(F32)
    vector = fma(num, d, offset + np.where(red & (num < 0), F32(360), F32(0)))
    scalar = fma(num, d, offset)
    scalar = np.where(scalar < 0, (scalar + F32(360)).astype(F32), scalar)
    W0 = x.shape[-2]
    tail = np.arange(W0) >= W0 - W0 % HSV_LANES
    h = np.where(tail, scalar, vector).astype(F32)
    return np.stack([h, s, v], -1)


SECTORS = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])


def hsv2bgr(x):
    """cv2.cvtColor(x, COLOR_HSV2BGR) of fp32 frames [..., 3] (H in degrees)."""
    h, s, v = x[..., 0], x[..., 1], x[..., 2]
    one = F32(1)
    h = (h * (F32(6) / F32(360))).astype(F32)
    pre = np.trunc(h).astype(F32)
    f = (h - pre).astype(F32)
    sector = (pre - np.trunc((pre * (one / F32(6))).astype(F32)) * F32(6)).astype(F32)
    tab = np.stack([v, (v * (one - s)).astype(F32), (v * fma(-s, f, one)).astype(F32),
                    (v * fma(-s, (one - f).astype(F32), one)).astype(F32)], -1)
    return np.take_along_axis(tab, SECTORS[sector.astype(np.int64) % 6], -1)


def photometric(x, rec):
    """PhotometricDistort with the recipe's draws on fp32 BGR frames [T, H0, W0, 3]."""
    if rec.brightness is not None:
        x = (x + rec.brightness).astype(F32)
    if rec.contrast_first and rec.contrast is not None:
        x = (x * rec.contrast).astype(F32)
    hsv = np.stack([bgr2hsv(fr) for fr in x])
    if rec.saturation is not None:
        hsv[..., 1] = (hsv[..., 1] * rec.saturation).astype(F32)
    if rec.hue is not None:
        h = (hsv[..., 0] + rec.hue).astype(F32)
        h = np.where(h > 360, (h - F32(360)).astype(F32), h)
        hsv[..., 0] = np.where(h < 0, (h + F32(360)).astype(F32), h)
    x = hsv2bgr(hsv)
    if not rec.contrast_first and rec.contrast is not None:
        x = (x * rec.contrast).astype(F32)
    return x[..., list(rec.perm)]


def augment(frames_rgb, rec, size, mean=(0, 0, 0), stds=(1, 1, 1), scale=1):
    """frames_rgb: uint8 [T, 3, H0, W0] (after the dataset's swap); rec: the host stage's AugRecipe; size = (W, H); mean /
    stds in BGR order.  Returns fp32 [T, 3, H, W]."""
    W, H = size
    x = np.ascontiguousarray(frames_rgb[:, ::-1].transpose(0, 2, 3, 1))  # BGR [T, H0, W0, 3], as the reference sees it
    if rec.photometric:
        x = photometric(x.astype(F32), rec)
        if scale == 2:
            x = np.clip(x, F32(0), F32(255))
    x = ot.convert(x, scale)
    x0, y0, w, h = rec.crop
    x = x[:, y0:y0 + h, x0:x0 + w]
    if rec.flip:
        x = x[:, :, ::-1]
    x = np.array(x)
    off = 0
    for x1, y1, x2, y2 in rec.erase:
        n = (y2 - y1) * (x2 - x1) * 3
        x[:, y1:y2, x1:x2] = rec.noise[off:off + n].reshape(y2 - y1, x2 - x1, 3)
        off += n
    mean = np.asarray(mean, F32)
    stds = np.asarray(stds, F32)
    out = []
    for fr in x:
        r = ot.resize(fr, H, W)
        out.append(((((r - mean).astype(F32)) / stds).astype(F32))[..., ::-1].transpose(2, 0, 1))
    return np.stack(out).astype(F32)
