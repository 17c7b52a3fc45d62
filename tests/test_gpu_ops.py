"""GPU: parity of the native ops (through the C ABI via step_b200's thin ctypes shim) against the
oracle and the committed golden vectors.  Bit-exact for NMS / ROIAlign fp32 / tube arithmetic
(exp/log excepted, tolerance stated)."""
import numpy as np
import pytest
import torch

from oracle import ops as oops
from oracle import tubes as otubes

pytestmark = pytest.mark.gpu

NMS_CASES = ["iou_eq_thr", "four", "third", "empty", "single", "rand63", "rand64", "rand65", "rand129",
             "rand1000", "intgrid"]


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("name", NMS_CASES)
def test_nms_golden(golden, name):
    from step_b200.roi_layers import nms
    g = golden("nms_cases")
    b, s, thr = g[name + "_boxes"], g[name + "_scores"], float(g[name + "_thr"])
    keep_cpu = nms(torch.from_numpy(b), torch.from_numpy(s), thr)        # the drivers' call pattern (CPU tensors)
    assert keep_cpu.dtype == torch.int64 and keep_cpu.device.type == "cpu"
    assert np.array_equal(keep_cpu.numpy(), g[name + "_keep"])
    if b.shape[0]:
        keep_gpu = nms(cu(b), cu(s), thr)
        assert keep_gpu.is_cuda and np.array_equal(keep_gpu.cpu().numpy(), g[name + "_keep"])


def test_nms_c3_10k_bit_exact_and_ties():
    from step_b200 import synth
    from step_b200.roi_layers import nms
    import step_b200.roi_layers as RL
    _, boxes, scores = synth.make_c3_rois()
    keep = nms(cu(boxes), cu(scores), 0.4).cpu().numpy()
    assert np.array_equal(keep, oops.nms(boxes, scores, 0.4))
    # tied scores: (score desc, index asc) contract, both comparison flavours
    s2 = np.round(scores * 8) / 8
    assert np.array_equal(nms(cu(boxes), cu(s2), 0.4).cpu().numpy(), oops.nms(boxes, s2, 0.4))
    RL._CUDA_GE = 0
    try:
        assert np.array_equal(nms(cu(boxes), cu(scores), 0.4).cpu().numpy(), oops.nms(boxes, scores, 0.4, ge=False))
    finally:
        RL._CUDA_GE = 1
    # size-independent properties: idempotence and sortedness
    again = nms(cu(boxes[keep]), cu(scores[keep]), 0.4).cpu().numpy()
    assert np.array_equal(again, np.arange(len(keep))) and np.all(np.diff(keep) > 0)


def test_nms_segmented_matches_per_segment_oracle():
    from step_b200.roi_layers import nms_segmented
    rs = np.random.RandomState(5)
    sizes = [0, 1, 11, 34, 34, 7, 300, 1024]
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    n = offs[-1]
    x1 = rs.uniform(0, 150, n); y1 = rs.uniform(0, 150, n)
    b = np.stack([x1, y1, x1 + rs.uniform(10, 100, n), y1 + rs.uniform(10, 100, n)], 1).astype(np.float32)
    s = rs.rand(n).astype(np.float32)
    s[::5] = 0.5
    mask = nms_segmented(cu(b), cu(s), cu(offs), 0.4, min_score=0.2).cpu().numpy()
    exp = np.zeros(n, np.uint8)
    for i in range(len(sizes)):
        lo, hi = offs[i], offs[i + 1]
        sel = np.nonzero(s[lo:hi] >= 0.2)[0]
        keep = oops.nms(b[lo:hi][sel], s[lo:hi][sel], 0.4)
        exp[lo + sel[keep]] = 1
    assert np.array_equal(mask, exp)


def test_roi_align_nchw_bit_exact(golden):
    from step_b200.roi_layers import ROIAlign, roi_align
    g = golden("roi_align_cases")
    feat, rois = cu(g["feat"]), cu(g["rois"])
    for sr in (0, 2):
        out = roi_align(feat, rois, (7, 7), 1.0 / 16.0, sr)
        assert np.array_equal(out.cpu().numpy(), g["out_sr%d" % sr])
    out = ROIAlign((3, 5), 0.5, 0)(feat, cu(g["rois"] * np.array([1, .1, .1, .1, .1], np.float32)))
    assert np.array_equal(out.cpu().numpy(), g["out_3x5_s0p5"])
    assert roi_align(feat, rois[:0], (7, 7), 1 / 16., 0).shape == (0, 5, 7, 7)


def test_roi_align_nhwc_fp32_bit_exact_and_fp16_close():
    from step_b200.roi_layers import roi_align
    rs = np.random.RandomState(2)
    K, C, H, W = 6, 64, 14, 14
    feat = rs.randn(K, C, H, W).astype(np.float32)
    R = 300
    x1 = rs.uniform(-20, 200, R); y1 = rs.uniform(-20, 200, R)
    rois = np.stack([rs.randint(0, K, R), x1, y1, x1 + rs.uniform(0, 400, R), y1 + rs.uniform(0, 150, R)], 1).astype(np.float32)
    ref = oops.roi_align_fwd(feat, rois, 1 / 16., 7, 7, 0)
    f_cl = cu(feat).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)   # channels-last storage
    out = roi_align(f_cl, cu(rois), (7, 7), 1 / 16., 0)
    assert out.stride(1) == 1                                               # stayed channels-last
    assert np.array_equal(out.cpu().numpy(), ref)
    h = roi_align(f_cl.half(), cu(rois), (7, 7), 1 / 16., 0)
    ref16 = oops.roi_align_fwd(feat.astype(np.float16).astype(np.float32), rois, 1 / 16., 7, 7, 0)
    assert h.dtype == torch.float16
    assert np.array_equal(h.float().cpu().numpy(), ref16.astype(np.float16).astype(np.float32))  # = round(exact fp32)


def test_roi_align_backward_matches_oracle():
    from step_b200.roi_layers import roi_align
    rs = np.random.RandomState(3)
    feat = torch.from_numpy(rs.randn(2, 4, 10, 12).astype(np.float32)).cuda().requires_grad_(True)
    rois = np.array([[0, 5, 5, 100, 90], [1, -10, 20, 60, 200], [1, 40, 40, 44, 44]], np.float32)
    out = roi_align(feat, cu(rois), (7, 7), 1 / 16., 0)
    gout = rs.randn(*out.shape).astype(np.float32)
    out.backward(cu(gout))
    ref = oops.roi_align_bwd(gout, rois, 1 / 16., 7, 7, 2, 4, 10, 12, 0)
    assert np.allclose(feat.grad.cpu().numpy(), ref, rtol=1e-5, atol=1e-6)   # float atomics: order differs


def test_roi_pool_forward_backward():
    from step_b200.roi_layers import roi_pool
    rs = np.random.RandomState(4)
    feat_np = rs.randn(3, 8, 14, 14).astype(np.float32)
    rois = np.array([[0, 0, 0, 223, 223], [1, 16, 16, 47, 47], [2, 500, 500, 600, 600], [2, 33.3, 70.1, 150.7, 99.9]], np.float32)
    feat = cu(feat_np).requires_grad_(True)
    out = roi_pool(feat, cu(rois), (7, 7), 1 / 16.)
    ref, arg = oops.roi_pool_fwd(feat_np, rois, 1 / 16., 7, 7)
    assert np.array_equal(out.detach().cpu().numpy(), ref)
    gout = rs.randn(*ref.shape).astype(np.float32)
    out.backward(cu(gout))
    assert np.allclose(feat.grad.cpu().numpy(), oops.roi_pool_bwd(gout, arg, rois, 7, 7, 3, 8, 14, 14), rtol=1e-5, atol=1e-6)


def test_tube_ops_golden(golden):
    from step_b200 import tube_utils as tu
    g = golden("tubes_cases")
    dec = tu.decode_coef(cu(g["dec_anchors"]), cu(g["dec_deltas"])).cpu().numpy()
    # expf differs from torch-CPU exp by <= 2 ulp: relative tolerance 1e-5 on finite rows
    fin = np.isfinite(g["dec_out"]).all(1)
    assert np.allclose(dec[fin], g["dec_out"][fin], rtol=1e-5, atol=1e-4)
    small = np.abs(g["dec_deltas"][:, 2:]).max(1) < 1e-30
    enc = tu.encode_coef(cu(g["enc_gt"]), cu(g["dec_anchors"])).cpu().numpy()
    assert np.allclose(enc, g["enc_out"], rtol=1e-5, atol=1e-6)
    v = tu.valid_tubes(cu(g["val_in"].copy()), 224, 224).cpu().numpy()
    assert np.array_equal(v, g["val_out_224"])
    arr = g["val_in"].copy()
    r = tu.valid_tubes(arr)                                  # numpy in, mutated in place like the reference
    assert r is arr and np.array_equal(arr, g["val_out_400"])
    for T in (2, 3, 4):
        e = tu.extrapolate_tubes(g["ext_in_T%d" % T], T)
        assert isinstance(e, np.ndarray) and np.array_equal(e, g["ext_out_T%d" % T])
    ex = tu.extend_tubes(cu(g["flat_out"]), 1.2, 224, 224).cpu().numpy()
    assert np.array_equal(ex, g["extend_out"])


@pytest.mark.parametrize("mode", ["none", "predict", "extrapolate", "mean"])
def test_tube_update_fused_matches_oracle_composition(mode):
    from step_b200 import _lib as L
    from step_b200 import tube_utils as tu
    rs = np.random.RandomState(9)
    R, T, Lf = 7, 3, 3
    boxes = rs.uniform(0, 100, (R, Lf, 2)).astype(np.float32)
    boxes = np.concatenate([boxes, boxes + rs.uniform(-2, 110, (R, Lf, 2)).astype(np.float32)], 2)
    clip = np.array([0, 0, 1, 1, 1, 3, 3], np.int32)
    flat = np.concatenate([np.zeros((R, Lf, 1), np.float32), boxes], 2)
    loc = (rs.randn(R, Lf, 4) * 0.3).astype(np.float32)
    first = (rs.randn(R, T, 4) * 0.3).astype(np.float32)
    last = (rs.randn(R, T, 4) * 0.3).astype(np.float32)
    ext = {"none": L.EXT_NONE, "predict": L.EXT_PREDICT, "extrapolate": L.EXT_EXTRAPOLATE, "mean": L.EXT_MEAN}[mode]
    nb = mode in ("none", "predict")
    pl_, pf_, pla_, fo = tu.tube_update(cu(flat), cu(loc), cu(first) if nb else None, cu(last) if nb else None,
                                        cu(clip), T, nb, ext, 224, 224)
    dexp = lambda v: np.exp(v.astype(np.float64)).astype(np.float32)
    dec = otubes.decode_coef(boxes.reshape(-1, 4), loc.reshape(-1, 4), exp=dexp).reshape(R, Lf, 4)
    assert np.allclose(pl_.cpu().numpy(), dec, rtol=1e-5, atol=1e-4)
    cur = pl_.cpu().numpy()   # continue from the device's own decode so the rest must be bit-exact
    if mode == "predict":
        prop = np.concatenate([pf_.cpu().numpy(), cur, pla_.cpu().numpy()], 1)
    elif mode == "extrapolate":
        prop = otubes.extrapolate_tubes(cur, T)
    elif mode == "mean":
        m = np.tile(np.mean(cur, axis=1, keepdims=True), (1, T, 1))
        prop = np.concatenate((m, cur, m), 1)
    else:
        prop = cur
    prop = otubes.valid_tubes(prop, 224, 224)
    Lo = prop.shape[1]
    idx = (clip[:, None] * Lo + np.arange(Lo)[None, :]).astype(np.float32)
    exp_flat = np.concatenate([idx[:, :, None], prop], 2)
    assert np.array_equal(fo.cpu().numpy(), exp_flat)


def test_roi_align_fp16_fast_paths_within_tolerance():
    """exact=2 (fp32 FMA) and exact=0 (merged taps, packed half2) against the exact fp16 kernel."""
    from step_b200 import _lib as L
    rs = np.random.RandomState(8)
    K, H, W, C = 5, 14, 14, 64
    feat = torch.from_numpy(rs.randn(K, H, W, C).astype(np.float32)).cuda().half()
    R = 400
    x1 = rs.uniform(-20, 200, R); y1 = rs.uniform(-20, 200, R)
    rois_np = np.stack([rs.randint(0, K, R), x1, y1, x1 + rs.uniform(0, 230, R), y1 + rs.uniform(0, 230, R)], 1).astype(np.float32)
    rois_np[:8, 3:] = rois_np[:8, 1:3] + 900.0          # huge ROIs: sampling grid > 3x3 -> per-ROI fallback
    rois = torch.from_numpy(rois_np).cuda()
    outs = {}
    for mode in (1, 2, 0):
        o = torch.empty((R, 7, 7, C), dtype=torch.float16, device="cuda")
        L.check(L.lib().step_roi_align_fwd_nhwc(L.ptr(feat), L.F16, K, H, W, C, C, L.ptr(rois), R, 1 / 16., 7, 7, 0,
                                                L.ptr(o), C, 0, 0, 0, mode, L.stream()))
        outs[mode] = o.float().cpu().numpy()
    ref = oops.roi_align_fwd(feat.float().cpu().numpy().transpose(0, 3, 1, 2), rois_np, 1 / 16., 7, 7, 0).transpose(0, 2, 3, 1)
    assert np.array_equal(outs[1], ref.astype(np.float16).astype(np.float32))
    mx = np.abs(ref).max()
    assert np.abs(outs[2] - ref).max() <= 1.5e-3 * mx          # <= 1 fp16 ulp of the largest value
    assert np.abs(outs[0] - ref).max() <= 6e-3 * mx            # packed half2: a few fp16 ulps


def test_detect_postprocess_matches_reference_loop():
    """Segmented on-device post-processing == the per-clip x per-class loop of test.py:156-218."""
    from oracle import postprocess as opp
    from step_b200 import postprocess as pp
    rs = np.random.RandomState(12)
    nums = [11, 11, 11]
    R, ncls, T = sum(nums), 60, 4
    prob = rs.rand(R, ncls).astype(np.float32) ** 3
    ctr = rs.uniform(40, 180, (R, 2)).astype(np.float32)
    wh = rs.uniform(20, 120, (R, 2)).astype(np.float32)
    box = np.concatenate([ctr - wh / 2, ctr + wh / 2], 1).astype(np.float32)
    box[3] = [50, 50, 51, 120]                                   # degenerate -> whole 400x400 image in valid_tubes
    loc = np.tile(box[:, None, :], (1, T, 1)) + rs.randn(R, T, 4).astype(np.float32)
    loc[:, T // 2] = box
    det = pp.detect(cu(np.tile(prob[:, None, :], (1, T, 1))), cu(loc), nums, 0.2, 0.4, 224.0, 224.0, topk=0)
    got = pp.to_lists(det, len(nums))
    ref = opp.detections(prob, box, nums, 0.2, 0.4, 224.0, 224.0, topk=0)
    for g, r in zip(got, ref):
        assert len(g) == len(r) and len(r) > 20
        gs = sorted((c, round(s, 6), tuple(np.round(b, 5))) for b, c, s in g)
        rs_ = sorted((c, round(s, 6), tuple(np.round(b, 5))) for b, c, s in r)
        assert gs == rs_
    # top-k per clip keeps exactly the k best kept scores
    det = pp.detect(cu(prob), cu(loc), nums, 0.2, 0.4, 224.0, 224.0, topk=10)
    got = pp.to_lists(det, len(nums))
    ref = opp.detections(prob, box, nums, 0.2, 0.4, 224.0, 224.0, topk=10)
    for g, r in zip(got, ref):
        assert [round(s, 6) for _, _, s in g] == [round(s, 6) for _, _, s in r]


@pytest.mark.parametrize("name", ["synth", "synth_topk", "c4"])
def test_detect_matches_reference_loop_rows(golden, name):
    """step_detect_f32 against the rows the reference's OWN evaluation loop (test.py:156-218, executed from the file where
    it lies by tests/golden/make_golden.py) wrote: ragged and empty clips, a score equal to conf_thresh, a degenerate
    box, near-duplicates, top-k.  The rows carry 4 significant digits ('{:.4}'), order included."""
    from step_b200 import postprocess as pp
    g = golden("postprocess_cases")
    conf, thr, topk, width, height = g[name + "_cfg"].tolist()
    prob, loc, nums = g[name + "_prob"], g[name + "_loc"], g[name + "_nums"].tolist()
    T = loc.shape[1]
    det = pp.detect(cu(np.ascontiguousarray(np.tile(prob[:, None, :], (1, T, 1)))), cu(loc), nums, conf, thr, width, height,
                    topk=int(topk))
    got = pp.to_lists(det)
    fmt = lambda v: float("{:.4}".format(float(v)))
    rows = [(b, c, fmt(s)) + tuple(fmt(v) for v in bx) for b, d in enumerate(got) for (bx, c, s) in d]
    ref = [(int(r[0]), int(r[1]), fmt(r[2])) + tuple(fmt(v) for v in r[3:7]) for r in g[name + "_rows"]]
    assert rows == ref            # same detections in the same (file) order


@pytest.mark.parametrize("name", ["ties", "ties_topk", "ties_topk_all"])
def test_detect_row_order_with_ties_matches_reference_loop(golden, name):
    """step_detect_f32 against the rows the reference's own loop wrote (make_golden.py::gen_detect_edges): exact score ties
    across and within classes, at and away from the top-k cut, scores equal to conf_thresh, degenerate boxes, an empty
    clip.  Same rows in the same order."""
    from step_b200 import postprocess as pp
    g = golden("detect_edge_cases")
    conf, thr, topk, width, height = g[name + "_cfg"].tolist()
    prob, loc, nums = g[name + "_prob"], g[name + "_loc"], g[name + "_nums"].tolist()
    det = pp.detect(cu(prob), cu(loc), nums, conf, thr, width, height, topk=int(topk))
    fmt = lambda v: float("{:.4}".format(float(v)))
    rows = [(b, c) + tuple(fmt(v) for v in (s,) + tuple(bx)) for b, d in enumerate(pp.to_lists(det)) for (bx, c, s) in d]
    ref = [(int(r[0]), int(r[1])) + tuple(fmt(v) for v in r[2:7]) for r in g[name + "_rows"]]
    assert rows == ref


def _oracle_rows(prob, box, nums, conf, thr, topk):
    """The corrected oracle's detections per clip as float32 [k, 8] rows laid out as step_detect_f32's det."""
    from oracle import postprocess as opp
    ref = opp.detections(prob, box, nums, conf, thr, 224.0, 224.0, topk=topk, with_tube=True)
    return [np.asarray([list(b) + [s, c, t, 0.0] for b, c, s, t in d], np.float32).reshape(-1, 8) for d in ref]


def _device_rows(det, b):
    return det["det"][b, :int(det["count"][b])].cpu().numpy()


def _same_rows(got, ref, what):
    """The same (class, tube) rows in the same order, scores and normalised boxes bit-equal as float32."""
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    if not np.array_equal(got.view(np.int32), ref.view(np.int32)):
        i = int(np.nonzero((got.view(np.int32) != ref.view(np.int32)).any(1))[0][0])
        raise AssertionError((what, "first differing row", i, got[i].tolist(), ref[i].tolist()))


def _detect_case(nums, ncls, seed, overlap=None, levels=None):
    """prob [R, T, ncls], loc [R, T, 4] and the centre-frame boxes [R, 4].  Boxes of the clips named in `overlap` are small
    jitters of one box (NMS keeps few of them); the others lie in distinct cells of a 12 x 12 grid over 400 px (disjoint:
    NMS keeps all).  Scores uniform, or drawn from `levels` (exact ties)."""
    rs = np.random.RandomState(seed)
    T = 3
    boxes = []
    for b, n in enumerate(nums):
        if overlap and b in overlap:
            x = rs.uniform(100, 104, (n, 2))
            boxes.append(np.concatenate([x, x + rs.uniform(60, 64, (n, 2))], 1))
        else:
            cell = rs.permutation(144)[:n] if n <= 144 else np.arange(n) % 144
            x = np.stack([cell % 12, cell // 12], 1) * 33.0 + rs.uniform(0, 3, (n, 2))
            boxes.append(np.concatenate([x, x + rs.uniform(20, 28, (n, 2))], 1))
    box = np.concatenate(boxes).astype(np.float32).reshape(-1, 4)
    R_ = box.shape[0]
    prob = rs.uniform(0, 1, (R_, ncls)).astype(np.float32) if levels is None else \
        np.asarray(levels, np.float32)[rs.randint(0, len(levels), (R_, ncls))]
    loc = (box[:, None, :] + rs.uniform(-2, 2, (R_, T, 4))).astype(np.float32)
    loc[:, T // 2] = box
    return np.ascontiguousarray(np.repeat(prob[:, None, :], T, 1)), loc, box


@pytest.mark.parametrize("topk", [0, 50])
def test_detect_at_scale_matches_corrected_oracle(topk):
    """Clips of 0, 1, 129 and 1024 tubes with 60 classes and a low conf_thresh (the 129-tube clip wraps the 128 threads
    of the rank and NMS loops; the 1024-tube clip is the per-(clip, class) limit, its boxes heavily overlapping so that NMS
    keeps few): the kept (class, tube) rows, scores and boxes bit-equal to the corrected oracle, in its order."""
    from step_b200 import postprocess as pp
    nums = [0, 1, 129, 1024]
    prob, loc, box = _detect_case(nums, 60, 61, overlap={3})
    det = pp.detect(cu(prob), cu(loc), nums, 0.05, 0.4, 224.0, 224.0, topk=topk)
    ref = _oracle_rows(prob[:, 1], box, nums, 0.05, 0.4, topk)
    for b in range(len(nums)):
        _same_rows(_device_rows(det, b), ref[b], ("clip", b, nums[b], topk))
    kept = det["keep"].cpu().numpy()
    assert 0 < int(kept[(129 + 1) * 60:].sum()) < 60 * 20                  # the 1024-tube clip: NMS keeps few


@pytest.mark.parametrize("topk", [0, 3000])
def test_detect_select_in_global_memory_matches_corrected_oracle(topk):
    """A clip of 140 tubes with disjoint boxes and every score above conf_thresh: 8400 survivors, more than the 4096 the
    select kernel ranks in shared memory, so it ranks against global memory.  Scores on three levels: the top-k cut falls
    inside a run of ties, which come out in reverse file order.  A 5-tube clip before it takes the shared-memory path."""
    from step_b200 import postprocess as pp
    nums = [5, 140]
    prob, loc, box = _detect_case(nums, 60, 62, levels=[0.25, 0.5, 0.75])
    det = pp.detect(cu(prob), cu(loc), nums, 0.1, 0.4, 224.0, 224.0, topk=topk)
    survivors = int(det["keep"][5 * 60:].sum())
    print("\nglobal-memory select: %d survivors" % survivors)
    assert survivors == 140 * 60 > 4096
    ref = _oracle_rows(prob[:, 1], box, nums, 0.1, 0.4, topk)
    for b in range(len(nums)):
        _same_rows(_device_rows(det, b), ref[b], ("clip", b, topk))
    if topk:
        full = _oracle_rows(prob[:, 1], box, nums, 0.1, 0.4, 10 ** 6)[1]
        assert full[topk - 1, 4] == full[topk, 4]                          # the cut splits a run of ties


@pytest.mark.parametrize("topk", [0, 3000])
def test_detect_cap_truncates_both_select_paths(topk):
    """An output of `cap` rows per clip keeps the first cap rows of the full result and counts min(rows, cap), in the
    shared-memory (5 tubes) and the global-memory (140 tubes) select paths."""
    from step_b200 import postprocess as pp
    nums = [5, 140]
    prob, loc, box = _detect_case(nums, 60, 63, levels=[0.25, 0.5, 0.75])
    full = pp.detect(cu(prob), cu(loc), nums, 0.1, 0.4, 224.0, 224.0, topk=topk)
    for cap in (7, 1000):
        d = pp.Detector(nums, 60, torch.device("cuda"), 0.1, 0.4, 224.0, 224.0, topk)
        d.cap = cap
        d.det = torch.full((len(nums), cap, 8), -1.0, device="cuda")
        got = d.run(cu(prob), cu(loc))
        for b in range(len(nums)):
            want = _device_rows(full, b)[:cap]
            assert int(got["count"][b]) == want.shape[0], (cap, b)
            _same_rows(_device_rows(got, b), want, ("cap", cap, b, topk))
    assert int(full["count"][0]) < 1000 < int(full["count"][1])


def test_detect_rejects_a_clip_over_1024_tubes_before_any_launch():
    """1025 tubes in one clip exceed the per-(clip, class) NMS problem: Detector raises, and so does the C entry when
    asked directly, and nothing is launched."""
    from step_b200 import _lib as L
    from step_b200 import postprocess as pp
    assert L.lib().step_nms_segmented_max_rows() == 1024
    nums = [3, 1025]
    prob, loc, _ = _detect_case(nums, 4, 64, overlap={1})
    before = L.launch_count()
    with pytest.raises(RuntimeError, match="1025 tubes"):
        pp.detect(cu(prob), cu(loc), nums, 0.1, 0.4, 224.0, 224.0)
    d = pp.Detector([3, 1024], 4, torch.device("cuda"), 0.1, 0.4, 224.0, 224.0)
    d.max_n = 1025
    with pytest.raises(RuntimeError, match="1025 tubes in one clip"):
        d.run(cu(prob[:1027]), cu(loc[:1027]))
    torch.cuda.synchronize()
    assert L.launch_count() == before


def test_roi_pool_and_align_backward_match_torchvision(golden):
    """The device ROIPool fwd/bwd and ROIAlign bwd against torchvision's CPU ops (the reference has no CPU
    implementation of them; see tests/golden/make_golden.py::gen_roi_cross)."""
    from step_b200.roi_layers import roi_align, roi_pool
    g, a = golden("roi_cross_cases"), golden("roi_align_cases")
    rois = cu(a["rois"])
    for sr in (0, 2):
        x = cu(a["feat"]).requires_grad_(True)
        y = roi_align(x, rois, (7, 7), 1.0 / 16.0, sr)
        y.backward(cu(g["align_gy_sr%d" % sr]))
        ref = g["align_gx_sr%d" % sr]
        assert np.abs(x.grad.cpu().numpy() - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max())
    x = cu(a["feat"]).requires_grad_(True)
    y = roi_pool(x, rois, (7, 7), 1.0 / 16.0)
    assert np.array_equal(y.detach().cpu().numpy(), g["pool_out"])
    y.backward(cu(g["pool_gy"]))
    assert np.abs(x.grad.cpu().numpy() - g["pool_gx"]).max() <= 2e-5 * max(1.0, np.abs(g["pool_gx"]).max())


def test_roi_align_c3_80000_rows_bit_exact():
    """BASELINE.json configs[2] (C3) at full size: 10 000 tubes x T' = 8 = 80 000 ROI rows over a [64,14,14,832] map,
    the exact channels-last kernels.  512 sampled rows are compared bit for bit with the C restatement of
    cpu/ROIAlign_cpu.cpp:137-243 (oracle/step_oracle.c, itself pinned to the reference's compiled op): fp32 exactly, fp16
    == round_to_half(exact fp32 on the half inputs).  Plus a size-independent property on ALL rows: pooling a constant
    map returns the constant wherever no sample falls outside the map."""
    from step_b200 import synth, _lib as L
    rois_np, _, _ = synth.make_c3_rois()
    R = rois_np.shape[0]
    assert R == 80000
    rois = cu(rois_np)
    g = torch.Generator().manual_seed(1234)
    feat32 = torch.randn(64, 14, 14, 832, generator=g).cuda()
    idx = np.random.RandomState(0).choice(R, 512, replace=False)
    for code, feat in ((L.F32, feat32), (L.F16, feat32.half())):
        o = torch.empty((R, 7, 7, 832), dtype=feat.dtype, device="cuda")
        L.check(L.lib().step_roi_align_fwd_nhwc(L.ptr(feat), code, 64, 14, 14, 832, 832, L.ptr(rois), R, 1 / 16., 7, 7, 0,
                                                L.ptr(o), 832, 0, 0, 0, 1, L.stream()))
        ref = oops.roi_align_fwd(feat.float().cpu().numpy().transpose(0, 3, 1, 2), rois_np[idx], 1 / 16., 7, 7, 0)
        got = o[torch.from_numpy(idx).cuda()].float().cpu().numpy().transpose(0, 3, 1, 2)
        refq = ref if code == L.F32 else ref.astype(np.float16).astype(np.float32)
        assert np.array_equal(got, refq)
        del o
    ones = torch.ones(64, 14, 14, 8, device="cuda")
    o = torch.empty((R, 7, 7, 8), dtype=torch.float32, device="cuda")
    L.check(L.lib().step_roi_align_fwd_nhwc(L.ptr(ones), L.F32, 64, 14, 14, 8, 8, L.ptr(rois), R, 1 / 16., 7, 7, 0,
                                            L.ptr(o), 8, 0, 0, 0, 1, L.stream()))
    assert float(o.min()) > 0.0 and float(o.max()) <= 1.0 + 1e-6
    inside = (rois_np[:, 1] >= 0) & (rois_np[:, 2] >= 0) & (rois_np[:, 3] <= 223) & (rois_np[:, 4] <= 223)
    assert float((o[torch.from_numpy(inside).cuda()] - 1.0).abs().max()) <= 1e-6


def test_roi_align_exact_huge_roi_uncached_grid():
    """ROIs far larger than the map (adaptive sampling grid > 4 x 4: the per-ROI tap table does not fit shared memory and
    the taps are recomputed per use) stay bit-exact, for 7 x 7 and for other output sizes."""
    from step_b200.roi_layers import roi_align
    rs = np.random.RandomState(8)
    K, C, H, W = 2, 16, 14, 14
    feat = rs.randn(K, C, H, W).astype(np.float32)
    rois = np.array([[0, -500, -300, 3000, 2500], [1, 0, 0, 1600, 223], [1, 10, 10, 900, 1200], [0, 3, 3, 100, 100]], np.float32)
    f_cl = cu(feat).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    for out_size in ((7, 7), (3, 5)):
        ref = oops.roi_align_fwd(feat, rois, 1 / 16., out_size[0], out_size[1], 0)
        out = roi_align(f_cl, cu(rois), out_size, 1 / 16., 0)
        assert np.array_equal(out.cpu().numpy(), ref)
