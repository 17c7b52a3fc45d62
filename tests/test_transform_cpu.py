"""CPU: the input transform's host-side pieces (argument errors of step_frames_to_clip_u8, the host stage, keep_frames) and the
numpy model of its kernel arithmetic (oracle/transform.py) against the reference's own BaseTransform output
(tests/golden/transform_cases.npz, cv2 without IPP), bit for bit."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import transform as ot
from step_b200 import _lib as L


def golden_cases(golden):
    z = golden("transform_cases")
    return z, [str(n) for n in z["cases"]]


def source(z, n):
    """Case n's uint8 BGR frames [T, H0, W0, 3] (cases may share a source)."""
    return z["src_" + str(z[n + "_src"])]


def rgb_frames(src_bgr_hwc):
    """The dataset's swap and permute (data/ava.py:333-338) of cv2's BGR [T, H0, W0, 3] frames, still uint8."""
    return np.ascontiguousarray(src_bgr_hwc[..., ::-1].transpose(0, 3, 1, 2))


def test_numpy_model_is_bit_identical_to_the_reference_without_ipp(golden):
    z, names = golden_cases(golden)
    assert len(names) >= 13
    for n in names:
        want = z[n + "_ipp_off"]
        got = ot.base_transform(rgb_frames(source(z, n)), tuple(z[n + "_size"]), z[n + "_mean"], z[n + "_stds"],
                                int(z[n + "_scale"]))[:, :, z[n + "_rows"]]
        assert got.shape == want.shape, n
        bad = got.view(np.int32) != want.view(np.int32)
        assert not bad.any(), "%s: %d values differ, first at %s" % (n, bad.sum(), np.argwhere(bad)[0])


def test_golden_covers_the_border_rows_and_the_area_switch(golden):
    z, names = golden_cases(golden)
    for n in names:
        H = int(z[n + "_size"][1])
        rows = z[n + "_rows"]
        assert rows[0] == 0 and rows[-1] == H - 1, n
    assert tuple(source(z, "area_800x800_400").shape[1:3]) == (800, 800)


def _call(table=16, B=1, T=1, H=8, W=8, scale=2, mean=True, std=True, out=16):
    m = (ctypes.c_float * 3)(0, 0, 0) if mean else None
    s = (ctypes.c_float * 3)(1, 1, 1) if std else None
    rc = L.lib().step_frames_to_clip_u8(ctypes.c_void_p(table), B, T, H, W, scale, m, s, ctypes.c_void_p(out),
                                        ctypes.c_void_p(0))
    return rc, L.lib().step_last_error().decode()


@pytest.mark.parametrize("kw, words", [
    (dict(table=0), "null pointer"), (dict(out=0), "null pointer"), (dict(mean=False), "null pointer"),
    (dict(std=False), "null pointer"), (dict(B=0), "positive"), (dict(T=-1), "positive"), (dict(H=0), "positive"),
    (dict(W=0), "positive"), (dict(scale=3), "scale_mode 3"), (dict(scale=-1), "scale_mode -1"),
    (dict(B=300, T=300), "exceeds 65535"),
])
def test_frames_to_clip_argument_errors(kw, words):
    rc, msg = _call(**kw)
    assert rc == L.E_ARG, (rc, msg)
    assert "frames_to_clip_u8" in msg and words in msg, msg


def test_host_stage_is_the_identity():
    from step_b200.transforms import BaseTransform
    tr = BaseTransform((400, 400), scale=2)
    frames = np.random.RandomState(0).randint(0, 256, (4, 36, 64, 3)).astype(np.uint8)
    tubes, proposals = np.zeros((2, 5)), np.ones((3, 3, 4))
    out = tr(frames, tubes, proposals)
    assert out[0] is frames and out[1] is tubes and out[2] is proposals
    assert tr(frames)[1:] == (None, None)
    with pytest.raises(ValueError):
        BaseTransform((400, 400), scale=3)


def _stacking_collate(batch):
    """A collate with the reference drivers' contract: images stacked unless the first is None, the rest as lists."""
    imgs, tubes, infos = [s[0] for s in batch], [s[1] for s in batch], [s[2] for s in batch]
    if imgs[0] is not None:
        imgs = torch.stack(imgs, 0)
    return imgs, tubes, infos


def test_keep_frames_returns_the_frames_and_the_other_fields_unchanged():
    from step_b200.transforms import keep_frames
    rs = np.random.RandomState(1)
    sizes = [(360, 640), (360, 480), (361, 641)]
    batch = [(torch.from_numpy(rs.randint(0, 256, (4, 3, h, w)).astype(np.uint8)), rs.randn(5, 3, 4), {"fid": i})
             for i, (h, w) in enumerate(sizes)]
    with pytest.raises(RuntimeError):
        _stacking_collate(batch)  # the stock collate cannot stack mixed sizes
    frames, tubes, infos = keep_frames(_stacking_collate)(batch)
    assert isinstance(frames, list) and all(f is s[0] for f, s in zip(frames, batch))
    same = [(torch.zeros(4, 3, 2, 2, dtype=torch.uint8),) + s[1:] for s in batch]
    _, tubes_ref, infos_ref = _stacking_collate(same)
    assert len(tubes) == len(tubes_ref) and all(a is b for a, b in zip(tubes, tubes_ref))
    assert infos == infos_ref
