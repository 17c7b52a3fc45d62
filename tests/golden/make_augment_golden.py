"""Generates tests/golden/augment_cases.npz by running the reference's TubeAugmentation (data/augmentations.py, imported
from the reference checkout) on seeded uint8 frames, tubes and proposals, then the dataset's BGR->RGB swap and permute
(data/ava.py:333-338).  Each case runs with cv2's IPP off and on.  Only runnable where the reference checkout and cv2
exist; the fixture it writes is committed.

    python tests/golden/make_augment_golden.py

The module runs unmodified except for one shim on its `random` global (numpy.random): RandomSampleCrop's
`random.choice(self.sample_options)` raises under numpy >= 1.24 (the tuple of modes is an inhomogeneous array), so
choice over a tuple returns `options[numpy.random.choice(len(options))]`, the value numpy 1.x drew from the same stream.

The seeds are searched with the host stage (step_b200.transforms.TubeAugmentation, which draws what the reference draws)
so that the cases together hit every branch tests/test_augment_cpu.py asks for.

Per case <name>: <name>_src, the key of its source `src_<key>` (uint8 [T, H0, W0, 3] BGR, as cv2.imread gives it; cases
share them), <name>_tubes (float32 [N, K, 4 + 2], percent coordinates), <name>_proposals (float64 [P, K, 4], absent for
proposals=None), <name>_flags (do_flip, do_crop, do_photometric, do_erase), <name>_size (W, H), <name>_mean / <name>_stds (BGR), <name>_scale, <name>_seed (numpy.random.seed
before the call), <name>_rows (the output rows stored), <name>_ipp_off (fp32 [T, 3, len(rows), W]), <name>_ipp_on_ulps
(int32, the IPP output's bit pattern minus the IPP-off output's), <name>_out_tubes / <name>_out_proposals (what the
reference returned), <name>_state_keys / <name>_state_pos (numpy.random's state after the call).
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
from step_b200.transforms import TubeAugmentation  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "augment_cases.npz")
ALL = (True, True, True, True)
SOURCES = {}  # key -> uint8 BGR frames, shared by the cases that name it


class _ChoiceShim:
    """numpy.random, except that choice over a tuple draws the index (see the module docstring)."""

    def __getattr__(self, name):
        return getattr(np.random, name)

    @staticmethod
    def choice(a, *args, **kw):
        if isinstance(a, tuple) and not args and not kw:
            return a[np.random.choice(len(a))]
        return np.random.choice(a, *args, **kw)


def load_augmentations():
    if refload.REF not in sys.path:
        sys.path.insert(0, refload.REF)
    spec = importlib.util.spec_from_file_location("ref_augmentations",
                                                  os.path.join(refload.REF, "data", "augmentations.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.random = _ChoiceShim()
    return mod


def noise_frames(rs, T, H0, W0):
    return rs.randint(0, 256, (T, H0, W0, 3)).astype(np.uint8)


def sparse_frames(rs, T, H0, W0):
    """Noise along the borders and in sparse blocks, flat 16x16 blocks elsewhere, so a large source stays small."""
    y, x = np.mgrid[0:H0, 0:W0]
    out = []
    for _ in range(T):
        base = np.stack([(37 * (y // 16) + 11 * (x // 16) + 80 * c) % 256 for c in range(3)], -1)
        mask = (y < 2) | (y >= H0 - 2) | (x < 2) | (x >= W0 - 2) | ((y // 24 + x // 24) % 29 == 0)
        out.append(np.where(mask[..., None], rs.randint(0, 256, (H0, W0, 3)), base).astype(np.uint8))
    return np.stack(out)


def make_tubes(rs, N, K, zero_box=False, overlap=False):
    """N tubes of K boxes in percent coordinates, 2 label columns after the box."""
    x1, y1 = rs.uniform(0.05, 0.5, (2, N, 1))
    w, h = rs.uniform(0.25, 0.45, (2, N, 1))
    jitter = rs.uniform(-0.02, 0.02, (4, N, K))
    if overlap and N > 1:
        x1[1], y1[1] = x1[0] + 0.03, y1[0] + 0.02
    boxes = np.stack([x1 + jitter[0], y1 + jitter[1], x1 + w + jitter[2], y1 + h + jitter[3]], -1).clip(0, 1)
    if zero_box:
        boxes[0, 0] = 0  # an all-zero box (a chunk without the person): RandomMirror leaves it
    labels = rs.randint(0, 2, (N, K, 2))
    return np.concatenate([boxes, labels], -1).astype(np.float32)


def make_proposals(rs, P, K):
    x1, y1 = rs.uniform(0, 0.7, (2, P, 1))
    w, h = rs.uniform(0.01, 0.3, (2, P, 1))
    return np.tile(np.stack([x1, y1, x1 + w, y1 + h], -1), (1, K, 1)).astype(np.float64)


def features(rec, tubes, flags):
    """The branches one host-stage draw hits."""
    f = set()
    if flags[2]:
        f.add("photometric")
        for gate in ("brightness", "contrast", "saturation", "hue"):
            f.add("%s_%s" % (gate, "on" if getattr(rec, gate) is not None else "off"))
        f.add("contrast_first" if rec.contrast_first else "contrast_last")
        f.add("perm_%d%d%d" % rec.perm)
    if flags[1]:
        r = rec.crop_rejects
        f.add("crop_whole" if rec.crop_mode is None else "crop_min_iou" if rec.crop_mode[0] is not None else
              "crop_unconstrained")
        f.update("reject_" + k for k, v in r.items() if v)
    if flags[0]:
        f.add("flip_on" if rec.flip else "flip_off")
        if rec.flip and (tubes[..., :4].sum(-1) == 0).any():
            f.add("flip_zero_box")
    if flags[3]:
        f.add("erase_on" if rec.erase else "erase_off")
        e = rec.erase
        for i in range(len(e)):
            for j in range(i + 1, len(e)):
                if max(e[i][0], e[j][0]) < min(e[i][2], e[j][2]) and max(e[i][1], e[j][1]) < min(e[i][3], e[j][3]):
                    f.add("erase_overlap")
            x1, y1, x2, y2 = e[i]
            if x2 > x1 and y2 > y1 and (x1 == 0 or y1 == 0 or x2 == rec.crop[2] or y2 == rec.crop[3]):
                f.add("erase_border")
    return f


def draw(tr, seed, src, tubes, proposals):
    np.random.seed(seed)
    tr(src, tubes.copy(), None if proposals is None else proposals.copy())
    return tr.last_recipe


def search(template, want, tries=4000):
    """Seeds for one case template until no new branch of `want` turns up."""
    name, src, tubes, proposals, flags, size, mean, stds, scale = template
    src = SOURCES[src]
    tr = TubeAugmentation(size, mean, stds, *flags, scale=scale)
    seeds, got = [], set()
    for seed in range(tries):
        f = features(draw(tr, seed, src, tubes, proposals), tubes, flags) & want
        if f - got:
            seeds.append(seed)
            got |= f
        if got == want:
            break
    return seeds, got


def main():
    assert refload.available(), "reference checkout not present"
    aug = load_augmentations()
    rs = np.random.RandomState(2025)
    K = 3
    sources = SOURCES
    sources.update({"small": noise_frames(rs, 2, 48, 64),
                    "tail": noise_frames(rs, 2, 45, 70),  # 70 % 8 == 6: cv2's scalar HSV loop takes a row's last 6 pixels
                    "ship": sparse_frames(rs, 1, 360, 640)})
    small, tail = "small", "tail"
    tubes3 = make_tubes(rs, 3, K, zero_box=True, overlap=True)
    props = make_proposals(rs, 4, K)
    want = {"photometric", "contrast_first", "contrast_last", "crop_whole", "crop_min_iou", "crop_unconstrained",
            "reject_aspect", "reject_overlap", "reject_centre", "reject_modes", "flip_on", "flip_off", "flip_zero_box",
            "erase_on", "erase_off", "erase_overlap", "erase_border"}
    want |= {"%s_%s" % (g, s) for g in ("brightness", "contrast", "saturation", "hue") for s in ("on", "off")}
    want |= {"perm_%d%d%d" % p for p in ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0))}
    templates = [  # name, frames, tubes, proposals, flags (flip, crop, photometric, erase), size, mean, stds, scale
        ("all_s2", small, tubes3, props, ALL, (40, 32), (0, 0, 0), (1, 1, 1), 2),
    ]
    cases = []
    covered = set()
    for t in templates:
        seeds, got = search(t, want - covered)
        covered |= got
        cases += [("%s_seed%d" % (t[0], s),) + t[1:] + (s,) for s in seeds]
    missing = want - covered
    assert not missing, missing
    # cv2's scalar HSV loop: photometric cases on the 70-wide source without a crop, so the tile taps the last 70 % 8
    # columns of each row, read left to right and mirrored
    for t in [("tail_nocrop_s0", tail, tubes3, props, (True, False, True, True), (40, 32), (0, 0, 0), (1, 1, 1), 0),
              ("tail_nocrop_s2", tail, tubes3, None, (True, False, True, True), (40, 32), (0, 0, 0), (1, 1, 1), 2)]:
        seeds, got = search(t, {"flip_on", "flip_off"})
        assert got == {"flip_on", "flip_off"}, got
        cases += [("%s_seed%d" % (t[0], s),) + t[1:] + (s,) for s in seeds]
    cases += [  # scales, means and flags the search does not vary
        ("all_s0_meanstd", tail, tubes3, props, ALL, (40, 32), (104, 117, 123), (57.375, 57.12, 58.395), 0, 7),
        ("all_s1_meanstd", small, tubes3, None, ALL, (40, 32), (0.406, 0.456, 0.485), (0.225, 0.224, 0.229), 1, 8),
        ("photo_only_s2", small, tubes3, props, (False, False, True, False), (40, 32), (0, 0, 0), (1, 1, 1), 2, 9),
        ("geom_only_s1", tail, tubes3, props, (True, True, False, True), (40, 32), (0, 0, 0), (1, 1, 1), 1, 10),
        ("none_s2", small, tubes3, props, (False, False, False, False), (40, 32), (0, 0, 0), (1, 1, 1), 2, 11),
        ("ship_360x640_400", "ship", make_tubes(rs, 2, K), make_proposals(rs, 3, K), ALL,
         (400, 400), (0, 0, 0), (1, 1, 1), 2, 12),
    ]
    rec = {"src_" + k: v for k, v in sources.items()}
    rec.update({"cv2_version": np.array(cv2.__version__), "numpy_version": np.array(np.__version__),
                "cases": np.array([c[0] for c in cases])})
    for name, key, tubes, proposals, flags, size, mean, stds, scale, seed in cases:
        src = sources[key]
        W, H = size
        rows = np.arange(H) if 3 * W * H <= 40000 else np.unique(np.r_[0:2, H - 2:H, 0:H:57])
        tr = aug.TubeAugmentation(size, mean, stds, do_flip=flags[0], do_crop=flags[1], do_photometric=flags[2],
                                  do_erase=flags[3], scale=scale)
        out = {}
        for ipp in (False, True):
            cv2.ipp.setUseIPP(ipp)
            np.random.seed(seed)
            images, t_out, p_out = tr(src.copy(), tubes.copy(), None if proposals is None else proposals.copy())
            state = np.random.get_state()
            images = torch.from_numpy(np.ascontiguousarray(images[:, :, :, (2, 1, 0)])).permute(0, 3, 1, 2).numpy()
            assert images.dtype == np.float32 and images.shape == (src.shape[0], 3, H, W)
            out[ipp] = (np.ascontiguousarray(images[:, :, rows]), t_out, p_out, state)
        (off, t_out, p_out, state), on = out[False], out[True][0]
        assert np.array_equal(t_out, out[True][1]) and np.array_equal(out[True][3][1], state[1])
        rec[name + "_ipp_off"] = off
        rec[name + "_ipp_on_ulps"] = (on.view(np.int32).astype(np.int64) - off.view(np.int32)).astype(np.int32)
        rec.update({name + "_src": np.array(key), name + "_tubes": tubes, name + "_flags": np.array(flags),
                    name + "_size": np.array(size), name + "_mean": np.array(mean, np.float32),
                    name + "_stds": np.array(stds, np.float32), name + "_scale": np.array(scale),
                    name + "_seed": np.array(seed), name + "_rows": rows, name + "_out_tubes": t_out,
                    name + "_state_keys": state[1], name + "_state_pos": np.array(state[2])})
        if proposals is not None:
            rec[name + "_proposals"] = proposals
            rec[name + "_out_proposals"] = p_out
        d = np.abs(on - off).max()
        print("%-28s src %s -> %s, rows %d, max |ipp_on - ipp_off| %.3g" % (name, src.shape, size, len(rows), d))
    cv2.ipp.setUseIPP(True)
    np.savez_compressed(OUT, **rec)
    print("wrote %s (%.2f MB)" % (OUT, os.path.getsize(OUT) / 1e6))


if __name__ == "__main__":
    main()
