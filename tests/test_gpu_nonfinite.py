"""GPU: the tube arithmetic, NMS and detection kernels on non-finite and boundary inputs (NaN, +-inf, -0.0, subnormals,
exp overflow, boxes at the degenerate-box rule and the image edge) through the C ABI (step_tube_*_f32, step_nms_f32,
step_nms_segmented_f32) and Detector / Merger, against the reference's own outputs (tests/golden/nonfinite_cases.npz)
and the oracles pinned to them (tests/test_nonfinite_cpu.py).

Bit for bit, except decode's expf on finite deltas, which keeps test_gpu_ops.py's tolerance; even there whether a value
is NaN, +inf or -inf, and whether valid_tubes replaced the box by the whole image, must match exactly.  Every box
valid_tubes and tube_update emit is finite: that is what keeps non-finite extents out of the ROI kernels, which are
never fed one here (a non-finite extent sizes a sampling grid of up to 2^31 steps).

NMS sizes 1023 .. 65,537 rows, with tied and NaN scores across the rank kernel's 1024-score tiles, are checked against
oracle/ops.nms; 65,537 rows give 1,025 column blocks, more than resolve_kernel has threads.  Above 393,216 rows
step_nms_f32 resolves with more than 48 KB of shared memory and needs a 19 GB workspace: that path is not tested here."""
import numpy as np
import pytest
import torch

from oracle import merge as om
from oracle import ops as oops
from step_b200 import _lib as L
from step_b200 import tube_utils as tu
from step_b200.postprocess import Detector, Merger, merged_results, result_lines

from _merge_case import LABELS, fixture_results, fixture_rows, infos, same_results
from test_nonfinite_cpu import DET_CASES, MODES, nms_cases, same_bits, same_class, update_from_decoded

pytestmark = pytest.mark.gpu

F = np.float32
DEV = torch.device("cuda:0")
EXT = {"none": L.EXT_NONE, "predict": L.EXT_PREDICT, "extrapolate": L.EXT_EXTRAPOLATE, "mean": L.EXT_MEAN}


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def exp_exact(d):
    """Rows whose exp(dw), exp(dh) are the same in every libm: 0, +-inf, NaN inputs, overflow and underflow."""
    e = d[:, 2:]
    return ((e == 0) | ~np.isfinite(e) | (e >= 89) | (e <= -1000)).all(1)


def test_decode(golden):
    z = golden("nonfinite_cases")
    a, d, ref = z["dec_anchors"], z["dec_deltas"], z["dec_out"]
    got = tu.decode_coef(cu(a), cu(d)).cpu().numpy()
    same_class(got, ref)
    fin = np.isfinite(ref)
    assert np.allclose(got[fin], ref[fin], rtol=1e-5, atol=1e-4)
    ex = exp_exact(d)
    assert ex.sum() >= 8
    same_bits(got[ex], ref[ex])


@pytest.mark.parametrize("W", [224, 400])
def test_valid_tubes(golden, W):
    z = golden("nonfinite_cases")
    v = z["val_in_%d" % W]
    got = tu.valid_tubes(cu(v.copy()), W, W).cpu().numpy()          # step_tube_valid_f32
    same_bits(got, z["val_torch_%d" % W])
    arr = v.copy().reshape(-1, 1, 4)
    assert tu.valid_tubes(arr, W, W) is arr                          # numpy in, mutated in place
    same_bits(arr.reshape(-1, 4), z["val_np_%d" % W])
    assert np.isfinite(got).all()


@pytest.mark.parametrize("T", [2, 3])
def test_extrapolate(golden, T):
    z = golden("nonfinite_cases")
    got = tu.extrapolate_tubes(z["ext_in_T%d" % T], T)               # step_tube_extrapolate_f32
    same_bits(got, z["ext_out_T%d" % T])
    with pytest.raises(ZeroDivisionError):
        tu.extrapolate_tubes(z["ext_in_T%d" % T], 1)


def test_extend(golden):
    z = golden("nonfinite_cases")
    same_bits(tu.extend_tubes(cu(z["extend_in"]), 1.2, 224, 224).cpu().numpy(), z["extend_out"])


@pytest.mark.parametrize("mode", MODES)
def test_tube_update(golden, mode):
    """step_tube_update_f32 against the reference's utils.py:61-129: decode up to expf (exact in class, and bit for bit
    where exp is exact), the whole-image replacements exactly, the next step's boxes within decode's tolerance and bit for
    bit from the device's own decode; every box of the next step finite."""
    z = golden("nonfinite_cases")
    p = "upd_%s_" % mode
    flat, loc, first, last = z[p + "flat"], z[p + "loc"], z[p + "first"], z[p + "last"]
    nums = z[p + "nums"].tolist()
    clip = np.repeat(np.arange(len(nums)), nums).astype(np.int32)
    nb = mode == "predict"
    pl_, pf_, pla_, fo = tu.tube_update(cu(flat), cu(loc), cu(first) if nb else None, cu(last) if nb else None, cu(clip),
                                        3, nb, EXT[mode], 224, 224)
    pairs = [(pl_, z[p + "pred_loc"], loc)]
    if nb:
        pairs += [(pf_, z[p + "pred_first"], first), (pla_, z[p + "pred_last"], last)]
    for dev, ref, d in pairs:
        got = dev.cpu().numpy()
        same_class(got, ref)
        fin = np.isfinite(ref)
        assert np.allclose(got[fin], ref[fin], rtol=1e-5, atol=1e-4)
        ex = exp_exact(d.reshape(-1, 4))
        same_bits(got.reshape(-1, 4)[ex], ref.reshape(-1, 4)[ex])
    got = fo.cpu().numpy()
    ref = z[p + "flat_out"]
    assert np.isfinite(got).all()
    whole = lambda f: (f[:, :, 1:] == F([0, 0, 224, 224])).all(2)
    assert np.array_equal(whole(got), whole(ref)) and whole(ref).any()
    assert np.array_equal(got[:, :, 0], ref[:, :, 0])
    assert np.allclose(got, ref, rtol=1e-5, atol=1e-4)
    args = (pf_.cpu().numpy(), pla_.cpu().numpy()) if nb else ()
    same_bits(got, update_from_decoded(z, mode, pl_.cpu().numpy(), *args))


def test_nms_fixture(golden):
    """step_nms_f32 on NaN / +-inf / signed-zero scores and NaN, infinite, zero- and negative-area boxes: the CPU-tensor
    call of the drivers and the CUDA-tensor call both give the reference's keep; '>' (ge = 0) gives the oracle's."""
    import step_b200.roi_layers as RL
    z = golden("nonfinite_cases")
    for name in nms_cases(z):
        p = "nms_%s_" % name
        b, s, thr = z[p + "boxes"], z[p + "scores"], float(z[p + "thr"])
        assert np.array_equal(RL.nms(torch.from_numpy(b), torch.from_numpy(s), thr).numpy(), z[p + "keep"]), name
        assert np.array_equal(RL.nms(cu(b), cu(s), thr).cpu().numpy(), z[p + "keep"]), name
        RL._CUDA_GE = 0
        try:
            assert np.array_equal(RL.nms(cu(b), cu(s), thr).cpu().numpy(), oops.nms(b, s, thr, ge=False)), name
        finally:
            RL._CUDA_GE = 1
    b, s = z["nms_iou_eq_thr_nan_boxes"], z["nms_iou_eq_thr_nan_scores"]
    assert not np.array_equal(oops.nms(b, s, 0.5, ge=False), oops.nms(b, s, 0.5))   # the flavours differ on this case


def test_nms_segmented_drops_nan_scores(golden):
    """step_nms_segmented_f32 with every fixture case as one segment: a NaN score fails s >= min_score and is dropped
    (scores.gt(conf_thresh) drops it in test.py:180); the rest is the oracle's NMS of the passing rows."""
    from step_b200.roi_layers import nms_segmented
    z = golden("nonfinite_cases")
    names = nms_cases(z)
    bs = [z["nms_%s_boxes" % n] for n in names]
    ss = [z["nms_%s_scores" % n] for n in names]
    offs = np.concatenate([[0], np.cumsum([len(s) for s in ss])]).astype(np.int32)
    b, s = np.concatenate(bs), np.concatenate(ss)
    for ge in (True, False):
        for min_score in (float("-inf"), 0.3):
            mask = nms_segmented(cu(b), cu(s), cu(offs), 0.5, min_score=min_score, ge=ge).cpu().numpy()
            exp = np.zeros(len(s), np.uint8)
            for i in range(len(names)):
                lo, hi = offs[i], offs[i + 1]
                sel = np.nonzero(s[lo:hi] >= min_score)[0]
                exp[lo + sel[oops.nms(b[lo:hi][sel], s[lo:hi][sel], 0.5, ge=ge)]] = 1
            assert np.array_equal(mask, exp), (ge, min_score)
            assert not mask[np.isnan(s)].any()


def size_case(n, seed):
    """n boxes in 64 clusters of heavy overlap, scores on 8 levels (ties inside and across 1024-score tiles), every
    97th score NaN and a few +-inf and -0.0."""
    rs = np.random.RandomState(seed)
    cell = rs.randint(0, 64, n)
    x1 = (cell % 8) * 120.0 + rs.uniform(0, 12, n)
    y1 = (cell // 8) * 120.0 + rs.uniform(0, 12, n)
    b = np.stack([x1, y1, x1 + rs.uniform(60, 80, n), y1 + rs.uniform(60, 80, n)], 1).astype(F)
    s = (rs.randint(0, 8, n) / 8.0).astype(F)
    s[::97] = np.nan
    s[5::1013] = np.inf
    s[7::1031] = -np.inf
    s[11::509] = -0.0
    return b, s


@pytest.mark.parametrize("n", [1023, 1024, 1025, 2049, 65537])
def test_nms_sizes_with_ties_and_nan(n):
    import step_b200.roi_layers as RL
    b, s = size_case(n, n)
    want = oops.nms(b, s, 0.4)
    assert np.array_equal(RL.nms(torch.from_numpy(b), torch.from_numpy(s), 0.4).numpy(), want)
    if n in (1025, 65537):
        RL._CUDA_GE = 0
        try:
            assert np.array_equal(RL.nms(cu(b), cu(s), 0.4).cpu().numpy(), oops.nms(b, s, 0.4, ge=False))
        finally:
            RL._CUDA_GE = 1
    # every NaN row leads in index order: the first NaN row is kept
    assert want[0] == 0 and np.isnan(s[0])


@pytest.mark.parametrize("name", DET_CASES)
def test_detector_and_merger(golden, name):
    """NaN and +-inf in prob and loc through Detector.run and Merger.run: demo.py's rows bit for bit (NaN scores dropped,
    +inf kept, non-finite coordinates clamped or replaced by the whole image), its merged dicts and results.txt text."""
    z = golden("nonfinite_cases")
    conf, nms, topk, width, height, thr = z[name + "_cfg"][:6].tolist()
    nums = z[name + "_nums"].tolist()
    det = Detector(nums, z[name + "_prob"].shape[1], DEV, conf, nms, width, height, topk=max(int(topk), 0))
    d = det.run(cu(z[name + "_prob"]), cu(z[name + "_loc"][:, None]))
    rows, count = det.det.cpu().numpy(), det.count.cpu().numpy()
    for b, clip in enumerate(fixture_rows(z, name)):
        assert int(count[b]) == len(clip)
        for k, (box, c, s) in enumerate(clip):
            same_bits(rows[b, k, :4], box)
            assert int(rows[b, k, 5]) == c and rows[b, k, 4] == F(s)
    assert np.isfinite(rows[:, :, :4]).all()
    got = merged_results(Merger(det, thr).run(d), d, LABELS)
    same_results(got, fixture_results(z, name))
    assert "".join(result_lines(got, infos(len(got)))) == str(z[name + "_text"])
    for b in range(len(nums)):
        clip = [(rows[b, k, :4], int(rows[b, k, 5]), float(rows[b, k, 4])) for k in range(int(count[b]))]
        same_results([got[b]], [om.demo_merge(clip, LABELS, thr)])
