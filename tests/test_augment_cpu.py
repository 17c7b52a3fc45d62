"""CPU: the training augmentation's host stage (step_b200.transforms.TubeAugmentation) and the numpy model of its kernel
arithmetic (oracle/augment.py) against the reference's own TubeAugmentation (tests/golden/augment_cases.npz): the same
draws from numpy's global RandomState, the same tubes and proposals, and the clip bit for bit (cv2 without IPP).  Also the
argument errors of step_frames_to_clip_aug_u8 and the recipe's trip through a multi-worker DataLoader."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import augment as oa
from oracle import transform as ot
from step_b200 import _lib as L


def cases(golden):
    z = golden("augment_cases")
    return z, [str(n) for n in z["cases"]]


def source(z, n):
    return z["src_" + str(z[n + "_src"])]


def rgb_frames(src_bgr_hwc):
    return np.ascontiguousarray(src_bgr_hwc[..., ::-1].transpose(0, 3, 1, 2))


def transform(z, n):
    from step_b200.transforms import TubeAugmentation
    flip, crop, photometric, erase = (bool(v) for v in z[n + "_flags"])
    return TubeAugmentation(tuple(z[n + "_size"]), z[n + "_mean"], z[n + "_stds"], do_flip=flip, do_crop=crop,
                            do_photometric=photometric, do_erase=erase, scale=int(z[n + "_scale"]))


def host_stage(z, n):
    """Runs the host stage as the golden's reference run did; returns (transform, tubes, proposals, state after)."""
    tr = transform(z, n)
    proposals = z[n + "_proposals"].copy() if n + "_proposals" in z else None
    np.random.seed(int(z[n + "_seed"]))
    images, tubes, proposals = tr(source(z, n), z[n + "_tubes"].copy(), proposals)
    assert images is source(z, n) or np.array_equal(images, source(z, n))
    return tr, tubes, proposals, np.random.get_state()


def test_host_stage_draws_and_returns_what_the_reference_does(golden):
    z, names = cases(golden)
    for n in names:
        tr, tubes, proposals, state = host_stage(z, n)
        want = z[n + "_out_tubes"]
        assert tubes.dtype == want.dtype and np.array_equal(tubes.view(np.uint8), want.view(np.uint8)), n
        if n + "_proposals" in z:
            want = z[n + "_out_proposals"]
            assert proposals.dtype == want.dtype and np.array_equal(proposals.view(np.uint8), want.view(np.uint8)), n
        else:
            assert proposals is None, n
        assert np.array_equal(state[1], z[n + "_state_keys"]) and state[2] == int(z[n + "_state_pos"]), n


def test_numpy_model_is_bit_identical_to_the_reference_without_ipp(golden):
    z, names = cases(golden)
    assert len(names) >= 12
    for n in names:
        tr, _, _, _ = host_stage(z, n)
        got = oa.augment(rgb_frames(source(z, n)), tr.last_recipe, tuple(z[n + "_size"]), z[n + "_mean"],
                         z[n + "_stds"], int(z[n + "_scale"]))[:, :, z[n + "_rows"]]
        want = z[n + "_ipp_off"]
        assert got.shape == want.shape, n
        bad = got.view(np.int32) != want.view(np.int32)
        assert not bad.any(), "%s: %d values differ, first at %s" % (n, bad.sum(), np.argwhere(bad)[0])


def taps_hsv_tail(rec, size):
    """Whether the resize taps a source pixel among the last W0 % 8 of its row, which cv2's BGR2HSV computes in its
    scalar loop rather than its 8-lane one."""
    W, H = size
    x0, _, w, h = rec.crop
    if (w, h) == (2 * W, 2 * H):
        cols = np.arange(w)
    else:
        c0, c1, _ = ot.linear_taps(W, w, True)
        cols = np.unique(np.r_[c0, c1])
    src_cols = x0 + (w - 1 - cols if rec.flip else cols)
    W0 = rec.src_hw[1]
    return bool((src_cols >= W0 - W0 % oa.HSV_LANES).any())


def test_model_without_the_scalar_hsv_tail_fails_the_tail_cases(golden, monkeypatch):
    """The cases that tap cv2's scalar HSV loop do pin its rule: the model with the 8-lane rule on every pixel differs
    from the reference in each of them."""
    z, names = cases(golden)
    tail_cases = []
    for n in names:
        tr, _, _, _ = host_stage(z, n)
        if tr.last_recipe.photometric and taps_hsv_tail(tr.last_recipe, tuple(z[n + "_size"])):
            tail_cases.append((n, tr.last_recipe))
    assert {rec.flip for _, rec in tail_cases} == {False, True}
    monkeypatch.setattr(oa, "HSV_LANES", 1)
    for n, rec in tail_cases:
        got = oa.augment(rgb_frames(source(z, n)), rec, tuple(z[n + "_size"]), z[n + "_mean"], z[n + "_stds"],
                         int(z[n + "_scale"]))[:, :, z[n + "_rows"]]
        bad = int((got.view(np.int32) != z[n + "_ipp_off"].view(np.int32)).sum())
        assert bad > 0, n
        print("%s: %d values differ without the scalar HSV rule" % (n, bad))


def test_goldens_cover_every_branch(golden):
    """Every gate on and off, both photometric orders, every channel permutation, each crop mode and rejection path, the
    mirror with an all-zero box, overlapping erase regions and one at the crop's border, scales 0-2, a non-trivial mean
    and std, proposals present and absent, distorted pixels from cv2's scalar HSV loop (tapped, mirrored and not) and the
    shipped shape."""
    z, names = cases(golden)
    hit = set()
    for n in names:
        tr, _, _, _ = host_stage(z, n)
        rec = tr.last_recipe
        flip, crop, photometric, erase = (bool(v) for v in z[n + "_flags"])
        hit.add("scale%d" % int(z[n + "_scale"]))
        hit.add("proposals" if n + "_proposals" in z else "no_proposals")
        if np.any(z[n + "_mean"] != 0) and np.any(z[n + "_stds"] != 1):
            hit.add("meanstd")
        if not (flip or crop or photometric or erase):
            hit.add("all_off")
        if photometric:
            for gate in ("brightness", "contrast", "saturation", "hue"):
                hit.add("%s_%s" % (gate, "off" if getattr(rec, gate) is None else "on"))
            hit.add("contrast_first" if rec.contrast_first else "contrast_last")
            hit.add("perm%d%d%d" % rec.perm)
            if taps_hsv_tail(rec, tuple(z[n + "_size"])):
                hit.add("hsv_tail_flip" if rec.flip else "hsv_tail")
        if crop:
            hit.add("crop_whole" if rec.crop_mode is None else "crop_min_iou" if rec.crop_mode[0] is not None
                    else "crop_unconstrained")
            hit.update("reject_" + k for k, v in rec.crop_rejects.items() if v)
        if flip:
            hit.add("flip_on" if rec.flip else "flip_off")
            if rec.flip and (z[n + "_tubes"][..., :4].sum(-1) == 0).any():
                hit.add("flip_zero_box")
        if erase:
            e = rec.erase
            hit.add("erase_on" if e else "erase_off")
            for i, (x1, y1, x2, y2) in enumerate(e):
                if x2 > x1 and y2 > y1 and (x1 == 0 or y1 == 0 or x2 == rec.crop[2] or y2 == rec.crop[3]):
                    hit.add("erase_border")
                for a1, b1, a2, b2 in e[i + 1:]:
                    if max(x1, a1) < min(x2, a2) and max(y1, b1) < min(y2, b2):
                        hit.add("erase_overlap")
        if all((flip, crop, photometric, erase)) and source(z, n).shape[1:3] == (360, 640) and \
                tuple(z[n + "_size"]) == (400, 400):
            hit.add("shipped")
    want = {"scale0", "scale1", "scale2", "proposals", "no_proposals", "meanstd", "all_off", "contrast_first",
            "contrast_last", "hsv_tail", "hsv_tail_flip", "crop_whole", "crop_min_iou", "crop_unconstrained", "reject_aspect",
            "reject_overlap", "reject_centre", "reject_modes", "flip_on", "flip_off", "flip_zero_box", "erase_on",
            "erase_off", "erase_border", "erase_overlap", "shipped"}
    want |= {"%s_%s" % (g, s) for g in ("brightness", "contrast", "saturation", "hue") for s in ("on", "off")}
    want |= {"perm%d%d%d" % p for p in ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0))}
    assert want <= hit, sorted(want - hit)


def test_all_flags_off_is_base_transform():
    """With every flag off the host stage draws nothing and returns the tubes and proposals unchanged (up to the
    coordinate round trip's rounding, as the reference), and the model equals BaseTransform's."""
    from step_b200.transforms import BaseTransform, TubeAugmentation
    rs = np.random.RandomState(4)
    frames = rs.randint(0, 256, (3, 50, 70, 3)).astype(np.uint8)
    tubes = rs.uniform(0, 1, (2, 3, 6)).astype(np.float32)
    mean, stds = (104, 117, 123), (57.375, 57.12, 58.395)
    for scale in (0, 1, 2):
        tr = TubeAugmentation((40, 32), mean, stds, scale=scale)
        np.random.seed(3)
        before = np.random.get_state()[1].copy()
        images, t, p = tr(frames, tubes, None)
        assert images is frames and p is None and np.array_equal(np.random.get_state()[1], before)
        assert np.array_equal(t, (tubes * np.float32([70, 50, 70, 50, 1, 1]) / np.float32([70, 50, 70, 50, 1, 1])))
        rec = tr.last_recipe
        assert rec.crop == (0, 0, 70, 50) and not rec.flip and not rec.photometric and not rec.erase
        got = oa.augment(rgb_frames(frames), rec, (40, 32), mean, stds, scale)
        want = ot.base_transform(rgb_frames(frames), (40, 32), mean, stds, scale)
        assert np.array_equal(got.view(np.int32), want.view(np.int32))
        assert str(tr.base) == str(BaseTransform((40, 32), mean, stds, scale))


def test_hsv_model_round_trip_is_close():
    """A sanity bound on the HSV rules themselves (the goldens pin them exactly): the round trip of in-range pixels
    returns them to within a few ulps of 255."""
    x = np.random.RandomState(0).uniform(0, 255, (64, 70, 3)).astype(np.float32)
    back = oa.hsv2bgr(oa.bgr2hsv(x))
    assert np.abs(back - x).max() < 1e-3


def _call(table=16, params=16, erase=16, noise=16, B=1, T=1, H=8, W=8, scale=2, mean=True, std=True, out=16):
    m = (ctypes.c_float * 3)(0, 0, 0) if mean else None
    s = (ctypes.c_float * 3)(1, 1, 1) if std else None
    rc = L.lib().step_frames_to_clip_aug_u8(ctypes.c_void_p(table), ctypes.c_void_p(params), ctypes.c_void_p(erase),
                                            ctypes.c_void_p(noise), B, T, H, W, scale, m, s, ctypes.c_void_p(out),
                                            ctypes.c_void_p(0))
    return rc, L.lib().step_last_error().decode()


@pytest.mark.parametrize("kw, words", [
    (dict(table=0), "null pointer"), (dict(params=0), "null pointer"), (dict(out=0), "null pointer"),
    (dict(mean=False), "null pointer"), (dict(std=False), "null pointer"), (dict(erase=0), "both"),
    (dict(noise=0), "both"), (dict(B=0), "positive"), (dict(T=-1), "positive"), (dict(H=0), "positive"),
    (dict(W=0), "positive"), (dict(scale=3), "scale_mode 3"), (dict(scale=-1), "scale_mode -1"),
    (dict(B=300, T=300), "exceeds 65535"),
])
def test_frames_to_clip_aug_argument_errors(kw, words):
    rc, msg = _call(**kw)
    assert rc == L.E_ARG, (rc, msg)
    assert "frames_to_clip_aug_u8" in msg and words in msg, msg


class _FakeDataset(torch.utils.data.Dataset):
    """A reference-style dataset: transform on BGR frames, BGR->RGB swap, permute; returns (images, targets, tubes, info)
    with the sample's index in the frames, so a recipe can be matched to its sample."""

    def __init__(self, transform, n=12):
        self.transform, self.n = transform, n

    def __len__(self):
        return self.n

    def __getitem__(self, index):
        rs = np.random.RandomState(100 + index)
        frames = rs.randint(0, 256, (2, 30 + index, 40 + 2 * index, 3)).astype(np.uint8)
        tubes = np.array([[[0.2, 0.2, 0.7, 0.8, 1, 0]] * 3], np.float32)
        images, tubes, _ = self.transform(frames, tubes, None)
        images = torch.from_numpy(images[:, :, :, (2, 1, 0)]).permute(0, 3, 1, 2)
        return images, tubes, None, {"index": index}


def _ref_style_collate(batch):
    imgs = [s[0] for s in batch]
    if imgs[0] is not None:
        imgs = torch.stack(imgs, 0)
    return imgs, [s[1] for s in batch], [s[2] for s in batch], [s[3] for s in batch]


def test_every_recipe_arrives_with_its_own_sample():
    from step_b200.transforms import AugRecipe, TubeAugmentation, keep_recipes, with_recipes
    tr = TubeAugmentation((32, 24), do_flip=True, do_crop=True, do_photometric=True, do_erase=True, scale=2)
    ds = with_recipes(_FakeDataset(tr), tr)
    assert len(ds) == 12 and ds.n == 12
    loader = torch.utils.data.DataLoader(ds, batch_size=3, num_workers=2, shuffle=True,
                                         collate_fn=keep_recipes(_ref_style_collate))
    seen = []
    for pairs, targets, tubes, infos in loader:
        assert len(pairs) == len(targets) == len(infos) == 3 and tubes == [None] * 3
        for (frames, rec), info in zip(pairs, infos):
            i = info["index"]
            assert isinstance(rec, AugRecipe) and rec.src_hw == (30 + i, 40 + 2 * i) == tuple(frames.shape[2:])
            seen.append(i)
    assert sorted(seen) == list(range(12))
    with pytest.raises(RuntimeError):
        with_recipes(_FakeDataset(lambda *a: a), tr)[0]
