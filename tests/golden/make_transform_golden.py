"""Generates tests/golden/transform_cases.npz by running the UNMODIFIED reference BaseTransform (data/augmentations.py,
imported from the reference checkout) on seeded uint8 frames, then the dataset's BGR->RGB swap and permute
(data/ava.py:333-338).  Each case runs with cv2's IPP on (the stock wheel's default) and off.  Only runnable where the
reference checkout and cv2 exist; the fixture it writes is committed.

    python tests/golden/make_transform_golden.py

Per case <name>: <name>_src, the key of its source `src_<key>` (uint8 [T, H0, W0, 3] BGR, as cv2.imread gives it; cases
may share one), <name>_size (W, H),
<name>_mean / <name>_stds (BGR, the constructor's), <name>_scale, <name>_rows (the output rows stored: all of them for small
outputs), <name>_ipp_off (fp32 [T, 3, len(rows), W]) and <name>_ipp_on_ulps (int32, the IPP output's bit pattern minus
the IPP-off output's: ipp_on = (ipp_off.view(int32) + ulps).view(float32)).  `cv2_version` and `cases` (names) are recorded.
"""
import importlib.util
import os
import sys

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refload  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "transform_cases.npz")


def load_augmentations():
    if refload.REF not in sys.path:
        sys.path.insert(0, refload.REF)
    spec = importlib.util.spec_from_file_location("ref_augmentations",
                                                  os.path.join(refload.REF, "data", "augmentations.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def frames(rs, T, H0, W0, sparse=29):
    """Seeded BGR frames: noise along every border (where cv2's border rules act) and in a sparse pattern of interior
    blocks, flat 16x16 blocks elsewhere so the fixture stays small."""
    y, x = np.mgrid[0:H0, 0:W0]
    out = []
    for _ in range(T):
        base = np.stack([(37 * (y // 16) + 11 * (x // 16) + 80 * c) % 256 for c in range(3)], -1)
        noise = rs.randint(0, 256, (H0, W0, 3))
        mask = (y < 2) | (y >= H0 - 2) | (x < 2) | (x >= W0 - 2) | ((y // 24 + x // 24) % sparse == 0)
        out.append(np.where(mask[..., None], noise, base).astype(np.uint8))
    return np.stack(out)


def main():
    assert refload.available(), "reference checkout not present"
    aug = load_augmentations()
    rs = np.random.RandomState(2024)
    f640 = frames(rs, 1, 360, 640)
    cases = [  # name, source, size (W, H), mean (BGR), stds (BGR), scale; a case may name an earlier case's source
        ("c4_360x640_224", f640, (224, 224), (0, 0, 0), (1, 1, 1), 2),
        ("ship_360x640_400", "c4_360x640_224", (400, 400), (0, 0, 0), (1, 1, 1), 2),
        ("w480_360x480_400", frames(rs, 1, 360, 480), (400, 400), (0, 0, 0), (1, 1, 1), 2),
        ("odd_361x641_400", frames(rs, 1, 361, 641), (400, 400), (0, 0, 0), (1, 1, 1), 2),
        ("area_800x800_400", frames(rs, 1, 800, 800, sparse=83), (400, 400), (0, 0, 0), (1, 1, 1), 2),
        ("up_200x300_400", frames(rs, 1, 200, 300), (400, 400), (0, 0, 0), (1, 1, 1), 2),
        ("same_64x96", frames(rs, 2, 64, 96), (96, 64), (0, 0, 0), (1, 1, 1), 2),
        ("row1_1x160_56", frames(rs, 2, 1, 160), (56, 40), (0, 0, 0), (1, 1, 1), 2),
        ("col1_90x1_56", frames(rs, 2, 90, 1), (56, 40), (0, 0, 0), (1, 1, 1), 2),
        ("scale0_72x128_56", frames(rs, 2, 72, 128), (56, 40), (0, 0, 0), (1, 1, 1), 0),
        ("scale1_72x128_56", frames(rs, 2, 72, 128), (56, 40), (0, 0, 0), (1, 1, 1), 1),
        ("meanstd_s0_72x128_56", frames(rs, 2, 72, 128), (56, 40), (104, 117, 123), (57.375, 57.12, 58.395), 0),
        ("meanstd_s1_72x128_56", frames(rs, 2, 72, 128), (56, 40), (0.406, 0.456, 0.485), (0.225, 0.224, 0.229), 1),
    ]
    rec = {"cv2_version": np.array(cv2.__version__), "cases": np.array([c[0] for c in cases])}
    for name, src, size, mean, stds, scale in cases:
        key = src if isinstance(src, str) else name
        src = rec["src_" + key] if isinstance(src, str) else src
        W, H = size
        rows = np.arange(H) if 3 * W * H <= 40000 else np.unique(np.r_[0:2, H - 2:H, 0:H:57])
        tr = aug.BaseTransform(size, mean, stds, scale)
        out = {}
        for ipp in (False, True):
            cv2.ipp.setUseIPP(ipp)
            images, _, _ = tr(src.copy())
            images = torch.from_numpy(np.ascontiguousarray(images[:, :, :, (2, 1, 0)])).permute(0, 3, 1, 2).numpy()
            assert images.dtype == np.float32 and images.shape == (src.shape[0], 3, H, W)
            out[ipp] = np.ascontiguousarray(images[:, :, rows])
        # the IPP output as its distance in ulps (int32 bit patterns) from the IPP-off output: exact, and mostly zeros
        rec[name + "_ipp_off"] = out[False]
        rec[name + "_ipp_on_ulps"] = (out[True].view(np.int32).astype(np.int64) - out[False].view(np.int32)).astype(np.int32)
        back = (out[False].view(np.uint32) + rec[name + "_ipp_on_ulps"].view(np.uint32)).view(np.float32)
        assert np.array_equal(back.view(np.int32), out[True].view(np.int32)), name
        rec["src_" + key] = src
        rec[name + "_src"] = np.array(key)
        rec.update({name + "_size": np.array(size), name + "_mean": np.array(mean, np.float32),
                    name + "_stds": np.array(stds, np.float32), name + "_scale": np.array(scale), name + "_rows": rows})
        d = np.abs(out[True] - out[False]).max()
        print("%-24s src %s -> %s, rows %d, max |ipp_on - ipp_off| %.3g" % (name, src.shape, size, len(rows), d))
    cv2.ipp.setUseIPP(True)
    np.savez_compressed(OUT, **rec)
    print("wrote %s (%.2f MB)" % (OUT, os.path.getsize(OUT) / 1e6))


if __name__ == "__main__":
    main()
