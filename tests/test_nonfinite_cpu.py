"""CPU: the oracle's tube arithmetic, NMS and detection post-processing on non-finite and boundary inputs (NaN, +-inf,
-0.0, subnormals, exp overflow, boxes at the degenerate-box rule and the image edge), pinned to the reference's own
outputs (tests/golden/nonfinite_cases.npz, tests/golden/make_nonfinite_golden.py); the GPU tests trust these oracles.

Also the rank rule of the device NMS (nms.cu, nms_rank_kernel) restated in numpy: with float compares every NaN score
and the best finite score share rank 0, so ranks repeat and some slots of the sorted order are never written; with the
integer order key the kernel uses, the ranks are the order torch.sort(descending=True) gives the reference, NaN first."""
import numpy as np
import pytest

from oracle import merge as om
from oracle import ops as oops
from oracle import postprocess as opp
from oracle import tubes as otubes

from _merge_case import LABELS, fixture_results, fixture_rows, same_results

F = np.float32
MODES = ["none", "predict", "extrapolate", "mean"]
DET_CASES = ["det_nonfinite", "det_nonfinite_topk"]


def nms_cases(z):
    return sorted(k[4:-5] for k in z.files if k.startswith("nms_") and k.endswith("_keep"))


def same_bits(a, b):
    """Equal shapes, NaN in the same places, every other element bit-identical (so -0.0 differs from +0.0)."""
    a, b = np.asarray(a, F), np.asarray(b, F)
    assert a.shape == b.shape
    na, nb = np.isnan(a), np.isnan(b)
    assert np.array_equal(na, nb)
    assert np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def same_class(a, b):
    """Where each array is NaN, +inf, -inf or finite: the part of decode that must match exactly even where expf may
    differ from the reference's exp by an ulp."""
    for f in (np.isnan, np.isposinf, np.isneginf):
        assert np.array_equal(f(a), f(b))


def test_fixture_covers_the_edges(golden):
    z = golden("nonfinite_cases")
    d = z["dec_deltas"]
    assert np.isnan(d).any() and np.isposinf(d).any() and np.isneginf(d).any()
    assert (d[:, 2:] >= 89).any() and (d[:, 2:] == F(88.7)).any() and (np.abs(d) == F(1e4)).any()
    assert np.isposinf(z["dec_out"]).any() and np.isnan(z["dec_out"]).any()
    assert (np.signbit(d) & (d == 0)).any() and ((d != 0) & (np.abs(d) < np.finfo(F).tiny)).any()
    for W in (224, 400):
        v = z["val_in_%d" % W]
        assert (v[:, 0] == v[:, 2] - 2).any() and (v == F(W)).any() and (v == np.nextafter(F(W), F(np.inf))).any()
    assert np.isnan(z["nms_nan_all_scores"]).all() and np.isnan(z["nms_nan_several_scores"]).sum() > 1


@pytest.mark.parametrize("W", [224, 400])
def test_valid_tubes_equals_both_reference_branches(golden, W):
    """numpy's np.maximum / np.minimum and torch.clamp keep NaN (the box then becomes the whole image) and -0.0; both
    branches of the reference agree bit for bit, and every box they emit is finite."""
    z = golden("nonfinite_cases")
    got = otubes.valid_tubes(z["val_in_%d" % W].reshape(-1, 1, 4), W, W).reshape(-1, 4)
    same_bits(got, z["val_np_%d" % W])
    same_bits(z["val_torch_%d" % W], z["val_np_%d" % W])
    assert np.isfinite(got).all()
    whole = (got == F([0, 0, W, W])).all(1)
    assert whole[np.isnan(z["val_in_%d" % W]).any(1)].all()
    assert (np.signbit(got) & (got == 0)).any()          # a kept -0.0


def test_decode_matches_reference(golden):
    z = golden("nonfinite_cases")
    with np.errstate(all="ignore"):
        got = otubes.decode_coef(z["dec_anchors"], z["dec_deltas"])
    ref = z["dec_out"]
    same_class(got, ref)
    fin = np.isfinite(ref)
    assert np.allclose(got[fin], ref[fin], rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize("T", [2, 3])
def test_extrapolate_matches_reference(golden, T):
    z = golden("nonfinite_cases")
    with np.errstate(all="ignore"):
        same_bits(otubes.extrapolate_tubes(z["ext_in_T%d" % T], T), z["ext_out_T%d" % T])


def test_extrapolate_at_T1_raises_like_the_reference(golden):
    z = golden("nonfinite_cases")
    with pytest.raises(ZeroDivisionError):
        otubes.extrapolate_tubes(z["ext_in_T2"], 1)
    from step_b200 import tube_utils as tu    # raises before it touches a device
    with pytest.raises(ZeroDivisionError):
        tu.extrapolate_tubes(z["ext_in_T2"], 1)


def test_extend_matches_reference(golden):
    z = golden("nonfinite_cases")
    with np.errstate(all="ignore"):
        same_bits(otubes.extend_tubes(z["extend_in"], 1.2, 224, 224), z["extend_out"])


def update_from_decoded(z, mode, pred_loc, pred_first=None, pred_last=None):
    """utils.py:100-129 in numpy from the decoded tubes: extension by temporal_mode, valid_tubes(224), flatten."""
    T = 3
    if mode == "predict":
        prop = np.concatenate([pred_first, pred_loc, pred_last], 1)
    elif mode == "extrapolate":
        prop = otubes.extrapolate_tubes(pred_loc, T)
    elif mode == "mean":
        m = np.tile(np.mean(pred_loc, axis=1, keepdims=True), (1, T, 1))
        prop = np.concatenate((m, pred_loc, m), 1)
    else:
        prop = pred_loc
    nums = z["upd_%s_nums" % mode].tolist()
    prop = otubes.valid_tubes(prop, 224, 224)
    lists, s = [], 0
    for n in nums:
        lists.append(prop[s:s + n]); s += n
    return otubes.flatten_tubes(lists, batch_idx=True)[0]


@pytest.mark.parametrize("mode", MODES)
def test_update_between_steps_matches_reference(golden, mode):
    """utils.py:61-129 with NaN, +-inf, exp overflow, -0.0 and subnormals in the regression outputs: the oracle's decode
    to the reference's up to exp's rounding (exactly in class), the rest bit for bit from the reference's decode; every
    box of the next step is finite."""
    z = golden("nonfinite_cases")
    p = "upd_%s_" % mode
    flat, loc = z[p + "flat"], z[p + "loc"]
    R_, L_ = loc.shape[:2]
    with np.errstate(all="ignore"):
        dec = otubes.decode_coef(flat[:, :, 1:].reshape(-1, 4), loc.reshape(-1, 4)).reshape(R_, L_, 4)
        same_class(dec, z[p + "pred_loc"])
        fin = np.isfinite(dec)
        assert np.allclose(dec[fin], z[p + "pred_loc"][fin], rtol=1e-5, atol=1e-4)
        args = (z[p + "pred_first"], z[p + "pred_last"]) if mode == "predict" else ()
        got = update_from_decoded(z, mode, z[p + "pred_loc"], *args)
    same_bits(got, z[p + "flat_out"])
    assert np.isfinite(got).all()
    assert (~np.isfinite(z[p + "pred_loc"])).any()


def test_oracle_nms_matches_reference(golden):
    z = golden("nonfinite_cases")
    names = nms_cases(z)
    assert len(names) >= 14
    for name in names:
        p = "nms_%s_" % name
        keep = oops.nms(z[p + "boxes"], z[p + "scores"], float(z[p + "thr"]))
        assert np.array_equal(keep, z[p + "keep"]), name


def float_rank(s):
    """nms_rank_kernel before it ranked on order keys: row i's slot is the number of rows that beat it, with float
    compares (an earlier row wins a tie)."""
    n = len(s)
    return np.array([sum(bool(s[t] >= s[i]) for t in range(i)) + sum(bool(s[t] > s[i]) for t in range(i + 1, n))
                     for i in range(n)])


def order_key(s):
    """nms.cu's order_key: an int32 with the order of the scores, NaN above +inf, -0.0 equal to +0.0."""
    s = np.asarray(s, F)
    b = np.where(s == 0, F(0), s).view(np.int32).astype(np.int64)
    k = np.where(b >= 0, b, b ^ 0x7FFFFFFF)
    return np.where(np.isnan(s), 0x7FFFFFFF, k)


def key_rank(s):
    k = order_key(s)
    n = len(s)
    return np.array([int((k[:i] >= k[i]).sum() + (k[i + 1:] > k[i]).sum()) for i in range(n)])


def test_float_rank_collides_on_nan_and_order_keys_do_not():
    s = F([.5, np.nan, .9, np.nan, .1])
    r = float_rank(s)
    assert r.tolist() == [1, 0, 0, 0, 2]                    # three rows in slot 0
    assert set(range(len(s))) - set(r.tolist()) == {3, 4}   # slots n - k .. n - 1 (k NaN rows) never written
    k = key_rank(s)
    order = np.empty(len(s), np.int64); order[k] = np.arange(len(s))
    assert order.tolist() == [1, 3, 2, 0, 4]                # torch.sort(descending=True), as nms_cpu.cpp:48 sorts


def test_order_key_ranks_like_the_oracle_sort():
    rs = np.random.RandomState(3)
    s = rs.choice(F([np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45, 1.2e-38, 0.5, -0.5, 3e38, -3e38]), 400)
    s = s.astype(F)
    r = key_rank(s)
    assert sorted(r.tolist()) == list(range(len(s)))
    order = np.empty(len(s), np.int64); order[r] = np.arange(len(s))
    # the same order as the oracle's comparator: NaN first, score descending, index ascending on ties (-0.0 == +0.0)
    key = [(0 if np.isnan(v) else 1, 0.0 if np.isnan(v) else -float(v), i) for i, v in enumerate(s)]
    assert order.tolist() == [i for *_, i in sorted(key)]
    assert bool((float_rank(s) != r).any())


@pytest.mark.parametrize("name", DET_CASES)
def test_postprocess_and_merge_oracles_match_reference(golden, name):
    """NaN and +-inf in prob and loc: NaN scores fail scores.gt(conf) and are dropped, +inf ones pass; a non-finite
    coordinate makes valid_tubes return a clamped or a whole-image box.  The oracle writes the rows demo.py's loop
    writes, bit for bit, and test.py's loop's rows at its 4 digits; the merge of those rows is the reference's."""
    z = golden("nonfinite_cases")
    conf, nms, topk, width, height, thr = z[name + "_cfg"][:6].tolist()
    dets = opp.detections(z[name + "_prob"], z[name + "_loc"], z[name + "_nums"].tolist(), conf, nms, width, height,
                          topk=int(topk))
    want = fixture_rows(z, name)
    for d, w in zip(dets, want):
        assert [(c, F(s)) for _, c, s in d] == [(c, F(s)) for _, c, s in w]
        assert all(np.array_equal(a[0], b[0]) for a, b in zip(d, w))
    fmt = lambda v: float("{:.4}".format(float(v)))
    rows = [(b, c, s) + tuple(bx) for b, d in enumerate(dets) for (bx, c, s) in d]
    assert [tuple(fmt(v) for v in r) for r in rows] == [tuple(fmt(v) for v in r) for r in z[name + "_tp_rows"]]
    assert any(np.isposinf(s) for d in dets for _, _, s in d)
    same_results([om.demo_merge(d, LABELS, thr) for d in want], fixture_results(z, name))
