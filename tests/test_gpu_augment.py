"""GPU: the training augmentation (step_b200.transforms.TubeAugmentation.apply, kernel step_frames_to_clip_aug_u8) against
the reference's own TubeAugmentation output (tests/golden/augment_cases.npz): bit-identical to cv2 without IPP; mixed
source sizes and strided sources in one launch; BaseTransform's clip with every flag off; and a shipped-shape augmented
batch through train_step."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import augment as oa

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _train_case import SHIPPED  # noqa: E402
from step_b200.synth import device_nets  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ALL = dict(do_flip=True, do_crop=True, do_photometric=True, do_erase=True)


def source(z, n):
    return z["src_" + str(z[n + "_src"])]


def rgb(src_bgr_hwc):
    """The dataset's swap and permute of cv2's BGR [T, H0, W0, 3] frames, still uint8: a [T, 3, H0, W0] tensor."""
    return torch.from_numpy(np.ascontiguousarray(src_bgr_hwc[..., ::-1].transpose(0, 3, 1, 2)))


def seeded_bgr(seed, T, H0, W0):
    return np.random.RandomState(seed).randint(0, 256, (T, H0, W0, 3)).astype(np.uint8)


def seeded_tubes(seed, N=3, K=3):
    rs = np.random.RandomState(seed)
    x1, y1 = rs.uniform(0.05, 0.5, (2, N, 1))
    w, h = rs.uniform(0.25, 0.45, (2, N, 1))
    boxes = np.stack([x1, y1, x1 + w, y1 + h], -1).repeat(K, 1)
    return np.concatenate([boxes, np.ones((N, K, 2))], -1).astype(np.float32)


def test_golden_cases_bit_identical_to_cv2_without_ipp(golden):
    from step_b200.transforms import TubeAugmentation
    z = golden("augment_cases")
    worst = {}
    for n in [str(c) for c in z["cases"]]:
        flip, crop, photometric, erase = (bool(v) for v in z[n + "_flags"])
        tr = TubeAugmentation(tuple(z[n + "_size"]), z[n + "_mean"], z[n + "_stds"], do_flip=flip, do_crop=crop,
                              do_photometric=photometric, do_erase=erase, scale=int(z[n + "_scale"]))
        np.random.seed(int(z[n + "_seed"]))
        proposals = z[n + "_proposals"].copy() if n + "_proposals" in z else None
        tr(source(z, n), z[n + "_tubes"].copy(), proposals)
        got = tr.apply([(rgb(source(z, n)).to(DEV), tr.last_recipe)])[0]
        got = got[:, :, torch.from_numpy(z[n + "_rows"]).to(DEV)].cpu().numpy()
        off = z[n + "_ipp_off"]
        bad = got.view(np.int32) != off.view(np.int32)
        assert not bad.any(), "%s: %d values differ from cv2 (IPP off), first at %s" % (n, bad.sum(), np.argwhere(bad)[0])
        on = (off.view(np.uint32) + z[n + "_ipp_on_ulps"].view(np.uint32)).view(np.float32)
        worst[n] = float(np.abs(got - on).max())
    print("max |ours - cv2 with IPP| per case: %s" % ", ".join("%s %.3g" % kv for kv in worst.items()))


def _recipes(tr, clips_bgr, seed):
    np.random.seed(seed)
    recs = []
    for i, c in enumerate(clips_bgr):
        tr(c, seeded_tubes(seed + i), None)
        recs.append(tr.last_recipe)
    return recs


def test_mixed_sizes_and_strided_sources_equal_per_clip_results():
    """One launch over clips of different sizes, one of them HWC frames read through strides (the pixel's 3 bytes
    adjacent, rows 3 W0 apart), equals each clip launched alone and the numpy model."""
    from step_b200.transforms import TubeAugmentation
    tr = TubeAugmentation((400, 400), scale=2, **ALL)
    sizes = [(360, 640), (360, 480), (361, 641), (200, 300)]
    bgr = [seeded_bgr(20 + i, 3, h, w) for i, (h, w) in enumerate(sizes)]
    recs = _recipes(tr, bgr, 5)
    clips = [rgb(c).to(DEV) for c in bgr]
    hwc = torch.from_numpy(np.ascontiguousarray(bgr[1][..., ::-1])).to(DEV)
    clips[1] = hwc.permute(0, 3, 1, 2)  # a strided view of RGB HWC frames, not a copy
    assert clips[1].stride()[1:] == (1, 3 * sizes[1][1], 3)
    batch = tr.apply(list(zip(clips, recs)))
    assert batch.shape == (len(sizes), 3, 3, 400, 400)
    for i, (c, r) in enumerate(zip(clips, recs)):
        assert torch.equal(batch[i], tr.apply([(c.contiguous(), r)])[0]), sizes[i]
    for i in (0, 2):
        ref = oa.augment(rgb(bgr[i]).numpy(), recs[i], (400, 400), scale=2)
        assert np.array_equal(batch[i].cpu().numpy().view(np.int32), ref.view(np.int32)), sizes[i]
    pinned = tr.apply([(rgb(bgr[3]).pin_memory(), recs[3])])
    torch.cuda.synchronize()
    assert torch.equal(pinned[0], batch[3])


@pytest.mark.parametrize("scale", [0, 1, 2])
def test_all_flags_off_equals_base_transform(scale):
    from step_b200.transforms import BaseTransform, TubeAugmentation
    mean, stds = (104, 117, 123), (57.375, 57.12, 58.395)
    tr = TubeAugmentation((224, 224), mean, stds, scale=scale)
    base = BaseTransform((224, 224), mean, stds, scale)
    bgr = [seeded_bgr(30 + i, 4, 360, 640 - 160 * i) for i in range(2)]
    recs = _recipes(tr, bgr, 9)
    clips = [rgb(c).to(DEV) for c in bgr]
    assert torch.equal(tr.apply(list(zip(clips, recs))), base.apply(clips))


def test_shipped_shape_augmented_batch_feeds_train_step():
    """2 clips of 36 360x640 frames, all flags on, scale 2 -> 400x400, through train_step with the shipped configuration
    (ROIPool, ContextNet, three refinement steps)."""
    from step_b200 import synth, training
    from step_b200.transforms import TubeAugmentation
    tr = TubeAugmentation((400, 400), scale=2, **ALL)
    bgr = [seeded_bgr(40 + i, 36, 360, 640) for i in range(2)]
    recs = _recipes(tr, bgr, 13)
    x = tr.apply([(rgb(c).pin_memory(), r) for c, r in zip(bgr, recs)])
    assert x.shape == (2, 36, 3, 400, 400) and bool(torch.isfinite(x).all())
    assert float(x.min()) >= -1.0 and float(x.max()) <= 1.0
    cfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(400, 400))
    step_tubes, step_targets = synth.make_train_case(cfg, 2, 3, 400, 400, seed=3)
    nets = device_nets(cfg, [synth.head_state_dict(100 + i, cfg) for i in range(3)], "pool", context=True)
    r = training.train_step(cfg, nets, x, [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets], lr=0.01,
                            momentum=0.9, weight_decay=1e-4)
    torch.cuda.synchronize()
    assert np.isfinite(float(r["loss"])) and len(r["losses"]) == 3
    assert all(bool(torch.isfinite(g).all()) for g in r["grads"].values())


def test_full_width_641_source_matches_the_model_mirrored_and_not():
    """Without a crop, a 641-wide source's last column comes from cv2's scalar HSV loop (641 % 8 == 1): the kernel
    equals the numpy model there, with the clip mirrored and not."""
    from step_b200.transforms import TubeAugmentation
    tr = TubeAugmentation((400, 400), scale=0, do_flip=True, do_photometric=True)
    bgr = seeded_bgr(50, 2, 361, 641)
    flips = {}
    seed = 0
    while len(flips) < 2:
        np.random.seed(seed)
        tr(bgr, seeded_tubes(seed), None)
        flips.setdefault(tr.last_recipe.flip, tr.last_recipe)
        seed += 1
    clip = rgb(bgr).to(DEV)
    for flip, rec in flips.items():
        assert rec.photometric and rec.crop == (0, 0, 641, 361)
        got = tr.apply([(clip, rec)])[0].cpu().numpy()
        want = oa.augment(rgb(bgr).numpy(), rec, (400, 400), scale=0)
        bad = got.view(np.int32) != want.view(np.int32)
        assert not bad.any(), "flip %s: %d values differ, first at %s" % (flip, bad.sum(), np.argwhere(bad)[0])
