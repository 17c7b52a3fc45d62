"""Generates tests/golden/nonfinite_cases.npz: the reference's tube arithmetic, NMS and detection loops on non-finite and
boundary inputs (NaN, +-inf, -0.0, subnormals, exp overflow, boxes exactly at the degenerate-box rule and at the image
edge), run by the UNMODIFIED reference (imported from its tree, native ops compiled from its own sources by
oracle/build_ref.py).  Only runnable where the reference tree exists; the fixture it writes is committed.

    python tests/golden/make_nonfinite_golden.py

Keys:
  dec_anchors, dec_deltas, dec_out           decode_coef (utils/tube_utils.py:165-189, torch)
  val_in, val_np_<W>, val_torch_<W>          valid_tubes [n, 1, 4] (tube_utils.py:59-92) on its numpy and its torch
                                             branch, W = 224 (width = height = 224) and 400 (the defaults)
  ext_in_T<T>, ext_out_T<T>                  extrapolate_tubes (tube_utils.py:10-27), T = 2, 3
  extend_in, extend_out                      extend_tubes(ratio 1.2, 224 x 224) (tube_utils.py:248-266)
  upd_<mode>_{flat,loc,first,last,nums,pred_loc,pred_first,pred_last,flat_out}
                                             the between-steps update of utils/utils.py:61-129, executed from the
                                             reference's file, for temporal_mode none (no extension), predict,
                                             extrapolate and mean; T = 3, image 224 x 224
  nms_<case>_{boxes,scores,thr,keep}         the compiled CPU nms (cpu/nms_cpu.cpp)
  det_<case>_*                               demo.py:130-217's per-class NMS, scores_list and cross-class merge (the
                                             layout of merge_cases.npz, see make_merge_golden.py), and _tp_rows: the
                                             rows test.py:156-218 writes for the same history (4 significant digits)
"""
import io
import os
import sys
import textwrap
import zipfile
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, OUT)
from oracle import refload  # noqa: E402
import make_golden  # noqa: E402  (run_reference_eval_loop: test.py:156-218 executed from the reference's file)
import make_merge_golden  # noqa: E402  (run_reference_demo_loop / case: demo.py:130-217)

R = refload.load()
TU = R.tube_utils
F = np.float32
T_ = torch.from_numpy
NAN, INF = F(np.nan), F(np.inf)
out = {}


def up(x):
    return np.nextafter(F(x), INF)


def dn(x):
    return np.nextafter(F(x), -INF)


def gen_decode():
    base_a = F([20, 30, 120, 150])
    base_d = F([0.1, -0.2, 0.3, -0.1])
    rows = [(base_a, base_d)]
    for c in range(4):
        for v in (NAN, INF, -INF):
            d = base_d.copy(); d[c] = v; rows.append((base_a, d))
            a = base_a.copy(); a[c] = v; rows.append((a, base_d))
    for v in (88.7, 89.0, 1e4, -1e4, -104.0):        # exp overflow (> 88.72) and underflow to 0
        for c in (2, 3):
            d = base_d.copy(); d[c] = v; rows.append((base_a, d))
        rows.append((base_a, F([0.1, -0.2, v, v])))
    for v in (1e38, -1e38, 3e38):                     # w * dx overflows: px = +-inf, px -+ 0.5 pw
        for c in (0, 1):
            d = base_d.copy(); d[c] = v; rows.append((base_a, d))
    rows.append((base_a, F([1e38, 0, 89.0, 0])))      # px = inf and pw = inf: inf - inf
    rows.append((base_a, F([-1e38, 0, 89.0, 0])))
    rows.append((base_a, F([-0.0, -0.0, -0.0, -0.0])))
    rows.append((F([-0.0, -0.0, 0, 0]), F([0, 0, 0, 0])))
    rows.append((F([0, 0, -1, -1]), F([0, 0, 0, 0])))   # w = h = 0: px = x1, pw = 0
    for v in (F(1e-45), F(-1e-45), F(1.2e-38)):         # subnormals
        rows.append((base_a, F([v, v, v, v])))
        rows.append((F([v, v, 100, 100]), base_d))
    a = np.stack([r[0] for r in rows]).astype(F)
    d = np.stack([r[1] for r in rows]).astype(F)
    out["dec_anchors"], out["dec_deltas"] = a, d
    with np.errstate(all="ignore"):
        out["dec_out"] = TU.decode_coef(T_(a.copy()), T_(d.copy())).numpy()


def valid_rows(W):
    base = F([20, 30, 120, 150])
    rows = [base]
    for c in range(4):
        for v in (NAN, INF, -INF):
            b = base.copy(); b[c] = v; rows.append(b)
    rows += [F([-0.0, -0.0, 120, 150]), F([20, 30, -0.0, 150]), F([-0.0, 30, 120, -0.0])]
    rows += [F([1e-45, -1e-45, 120, 150]), F([20, 30, 22 + 1e-5, 150]), F([-1.2e-38, 1.2e-38, 1e-45, 150])]
    # x1 == x2 - 2 (degenerate: not strictly less) and one ulp either side, in x and in y
    for lo in (F(98), dn(98), up(98)):
        rows.append(F([lo, 30, 100, 150]))
        rows.append(F([20, lo, 120, 100]))
    rows.append(F([0, 0, 2, 2])); rows.append(F([0, 0, up(2), up(2)]))
    # the far edge: at W, one ulp inside and one past (clamped to W), and x1 at W - 2 against a clamped x2
    for x2 in (F(W), dn(W), up(W), F(W + 50)):
        rows.append(F([20, 30, x2, 150]))
        rows.append(F([20, 30, 120, x2]))
    rows.append(F([W - 2, 30, up(W), 150])); rows.append(F([dn(W - 2), 30, up(W), 150]))
    rows.append(F([20, W - 2, 120, W + 1])); rows.append(F([20, dn(W - 2), 120, up(W)]))
    rows.append(F([NAN, NAN, NAN, NAN])); rows.append(F([-INF, -INF, INF, INF])); rows.append(F([INF, INF, -INF, -INF]))
    return np.stack(rows).astype(F)


def gen_valid():
    for W in (224, 400):
        v = valid_rows(W)
        out["val_in_%d" % W] = v
        kw = {} if W == 400 else dict(width=224, height=224)
        out["val_np_%d" % W] = TU.valid_tubes(v.copy().reshape(-1, 1, 4), **kw).reshape(-1, 4)
        out["val_torch_%d" % W] = TU.valid_tubes(T_(v.copy()).view(-1, 1, 4), **kw).view(-1, 4).numpy()


def gen_extrapolate():
    rs = np.random.RandomState(23)
    for Tt in (2, 3):
        n, L = 14, 2 * Tt
        t = np.concatenate([rs.uniform(5, 150, (n, L, 2)), rs.uniform(200, 380, (n, L, 2))], 2).astype(F)
        for k, (c, v) in enumerate([(c, v) for c in range(4) for v in (NAN, INF, -INF)]):
            t[k + 1, (k * 3) % L, c] = v
        t[13, :, :2] = -0.0                         # -0.0 through the recurrence and the clamp
        t[13, 0, 2:] = [399, 399]; t[13, 1, 2:] = [up(399), dn(399)]   # at the clamp (width - 1) and one ulp either side
        out["ext_in_T%d" % Tt] = t
        with np.errstate(all="ignore"):
            out["ext_out_T%d" % Tt] = TU.extrapolate_tubes(t.copy(), Tt)
    try:
        TU.extrapolate_tubes(out["ext_in_T2"].copy(), 1)
    except ZeroDivisionError:
        pass
    else:
        raise RuntimeError("the reference's extrapolate_tubes no longer raises at T = 1")


def gen_extend():
    rows = [F([20, 30, 120, 150])]
    for c in range(4):
        for v in (NAN, INF, -INF):
            b = rows[0].copy(); b[c] = v; rows.append(b)
    rows += [F([-0.0, -0.0, 0, 0]), F([0, 0, 223, 223]), F([1e-45, 1e-45, 222, 222])]
    b = np.stack(rows).astype(F)
    flat = np.concatenate([np.arange(len(b), dtype=F)[:, None], b], 1).reshape(-1, 1, 5)
    out["extend_in"] = flat
    out["extend_out"] = TU.extend_tubes(T_(flat.copy()), 1.2, 224, 224).numpy()


def _reference_update_source():
    """utils/utils.py:62-129, the update between two refinement steps (decode, extension by temporal_mode, valid_tubes,
    flatten_tubes), read from the file where it lies and dedented -- executed, never stored."""
    lines = open(os.path.join(refload.REF, "utils", "utils.py")).read().split("\n")
    start = next(i for i, l in enumerate(lines) if l.strip().startswith("pred_prob = global_prob.view("))
    end = next(i for i in range(start, len(lines)) if "flat_tubes = torch.FloatTensor(flat_tubes)" in lines[i])
    return textwrap.dedent("\n".join(lines[start:end + 1]))


def delta_variants():
    v = [F([0.1, -0.2, 0.3, -0.1]), F([0, 0, 0, 0]), F([-0.0, -0.0, -0.0, -0.0])]
    for c in range(4):
        for x in (NAN, INF, -INF):
            d = F([0.05, 0.1, -0.2, 0.1]); d[c] = x; v.append(d)
    v += [F([0, 0, 88.7, 0]), F([0, 0, 0, 89.0]), F([0, 0, 1e4, 1e4]), F([0, 0, -1e4, 0]), F([1e38, 0, 0, 0]),
          F([0, -1e38, 0, 0]), F([1e38, 0, 89.0, 0]), F([1e-45, -1e-45, 1e-45, -1e-45])]
    return v


def gen_update():
    rs = np.random.RandomState(29)
    T, L, C = 3, 3, 5
    nums = [7, 9]
    Rn = sum(nums)
    xy = rs.uniform(5, 120, (Rn, 1, 2)); wh = rs.uniform(20, 90, (Rn, 1, 2))
    boxes = (np.concatenate([xy, xy + wh], 2) + rs.uniform(-2, 2, (Rn, L, 4))).astype(F)
    clip = np.repeat(np.arange(len(nums)), nums)
    flat = np.concatenate([(clip[:, None] * L + np.arange(L)[None])[:, :, None].astype(F), boxes], 2).astype(F)
    var = delta_variants()
    base = lambda: (rs.randn(Rn, L, 4) * 0.2).astype(F)
    loc, first, last = base(), base(), base()
    slots = [(a, r, t) for a in (loc, first, last) for r in range(Rn) for t in range(L)]
    pick = rs.permutation(len(slots))
    for k, d in enumerate(var * 2):
        a, r, t = slots[pick[k]]
        a[r, t] = d
    prob = rs.uniform(0, 1, (Rn, C)).astype(F)
    for mode, i in (("none", 1), ("predict", 2), ("extrapolate", 2), ("mean", 2)):
        args = SimpleNamespace(num_classes=C, temporal_mode=mode if mode != "none" else "predict", max_iter=3,
                               NUM_CHUNKS={1: 1, 2: 1, 3: 3}, T=T, image_size=(224, 224))
        env = {"args": args, "i": i, "global_prob": T_(prob.copy()), "local_loc": T_(loc.copy()),
               "first_loc": T_(first.copy()), "last_loc": T_(last.copy()), "flat_tubes": T_(flat.copy()),
               "chunk_idx": [T // 2], "half_T": T // 2, "T_length": L, "tubes_nums": list(nums), "history": [], "trajectory": [],
               "conv_feat": torch.zeros(1), "np": np, "torch": torch, "decode_coef": TU.decode_coef,
               "extrapolate_tubes": TU.extrapolate_tubes, "valid_tubes": TU.valid_tubes,
               "flatten_tubes": TU.flatten_tubes}
        # pred_loc before valid_tubes: with no extension the reference's valid_tubes writes through the numpy view of it
        pred_loc = TU.decode_coef(T_(flat.copy()).view(-1, 5)[:, 1:], T_(loc.copy()).view(-1, 4)).view(Rn, L, 4).numpy()
        with np.errstate(all="ignore"):
            exec(compile(_reference_update_source(), "reference utils.py:62-129", "exec"), env)
        p = "upd_%s_" % mode
        out[p + "flat"], out[p + "loc"], out[p + "first"], out[p + "last"] = flat, loc, first, last
        out[p + "nums"] = np.asarray(nums, np.int64)
        out[p + "pred_loc"] = pred_loc
        if mode == "predict":
            out[p + "pred_first"] = env["pred_first_loc"].numpy().copy()
            out[p + "pred_last"] = env["pred_last_loc"].numpy().copy()
        out[p + "flat_out"] = env["flat_tubes"].numpy().copy()
        assert np.isfinite(out[p + "flat_out"]).all()


def nms_case(name, boxes, scores, thr):
    b = np.asarray(boxes, F).reshape(-1, 4)
    s = np.asarray(scores, F).reshape(-1)
    keep = R._C.nms(T_(b.copy()), T_(s.copy()), float(thr)).numpy().astype(np.int64)
    out["nms_%s_boxes" % name], out["nms_%s_scores" % name] = b, s
    out["nms_%s_thr" % name], out["nms_%s_keep" % name] = F(thr), keep


def gen_nms():
    cl = [[10, 10, 60, 60], [12, 12, 62, 62], [8, 11, 58, 61], [11, 9, 61, 59]]      # one overlapping cluster
    far = [[200, 200, 250, 250], [202, 201, 252, 251]]
    nms_case("nan_one", cl + far, [.5, NAN, .9, .3, .8, .1], 0.5)
    nms_case("nan_several", cl + far, [.5, NAN, .9, NAN, .1, NAN], 0.5)
    nms_case("nan_all", cl + far, [NAN] * 6, 0.5)
    nms_case("nan_first_last", cl + far, [NAN, .2, .9, .7, .8, NAN], 0.5)
    nms_case("inf_scores", cl + far, [INF, -INF, .5, INF, -INF, 0.0], 0.5)
    nms_case("nan_inf_scores", cl + far, [-INF, NAN, INF, .5, NAN, INF], 0.5)
    nms_case("signed_zero", cl + far, [-0.0, 0.0, -0.0, 0.0, 0.0, -0.0], 0.5)
    nms_case("signed_zero_rev", cl + far, [0.0, -0.0, 0.0, -0.0, -0.0, 0.0], 0.5)
    # non-finite coordinates in the earlier (higher score) and in the later row of an overlapping pair, pair k at 60*k
    for tag, vals in (("nan", (NAN,)), ("inf", (INF, -INF))):
        boxes, scores = [], []
        k = 0
        for v in vals:
            for c in range(4):
                for earlier in (True, False):
                    o = 60.0 * k
                    a, b = [o, o, o + 40, o + 40], [o + 2, o + 1, o + 41, o + 42]
                    (a if earlier else b)[c] = v
                    boxes += [a, b]
                    scores += [.9 - 0.01 * k, .8 - 0.01 * k]
                    k += 1
        nms_case("%s_coords" % tag, boxes, scores, 0.5)
        nms_case("%s_coords_rev" % tag, boxes, scores[::-1], 0.5)   # the later row of each pair goes first
    # zero-area (x2 = x1 - 1: width 0 with the "+1") and negative-area boxes against normal ones and each other
    boxes = [[10, 10, 9, 50], [10, 10, 50, 50], [100, 100, 90, 140], [100, 100, 140, 140], [200, 200, 199, 199],
             [200, 200, 199, 199], [300, 300, 280, 280], [290, 290, 300, 300], [400, 400, 380, 420], [400, 400, 380, 420]]
    nms_case("degenerate_areas", boxes, [.9, .8, .7, .6, .5, .4, .3, .2, .15, .1], 0.5)
    nms_case("degenerate_areas_rev", boxes, [.1, .2, .3, .4, .5, .6, .7, .8, .85, .9], 0.5)
    # IoU == thr exactly (ge suppresses, '>' keeps), next to NaN scores
    nms_case("iou_eq_thr_nan", [[0, 0, 9, 9], [0, 0, 9, 4], [100, 100, 109, 109], [100, 100, 109, 104]],
             [.9, .8, NAN, NAN], 0.5)


def gen_detect():
    """NaN and +-inf in prob and loc through demo.py's loop (rows and merged dicts) and test.py's loop (rows)."""
    rs = np.random.RandomState(31)
    nums, C = [6, 0, 9, 5], 7
    n = sum(nums)
    xy = rs.uniform(20, 250, (n, 2)); wh = rs.uniform(40, 120, (n, 2))
    loc = np.concatenate([xy, xy + wh], 1).astype(F)
    prob = rs.uniform(0, 1, (n, C)).astype(F)
    loc[0, 0] = NAN; loc[1, 2] = INF; loc[2, 3] = -INF; loc[3, 1] = -INF; loc[4, :] = NAN   # clip 0
    loc[7] = loc[6] + 1; loc[8, 2] = NAN; loc[9, 0] = INF; loc[10] = [-0.0, -0.0, 80, 90]   # clip 2
    loc[15, 3] = NAN; loc[16] = loc[15]                                                       # clip 3
    prob[0, 0] = NAN; prob[1, :3] = INF; prob[2, 1] = -INF; prob[3, :] = NAN; prob[5, 2] = NAN
    prob[6, 4] = INF; prob[7, 4] = INF; prob[8, :] = NAN; prob[9, 0] = INF; prob[11, 6] = -INF
    prob[15, 2] = INF; prob[16, 2] = NAN; prob[17, 5] = INF; prob[18, 5] = INF
    for name, topk in (("det_nonfinite", 0), ("det_nonfinite_topk", 9)):
        with np.errstate(all="ignore"):
            make_merge_golden.case(name, prob, loc, nums, 0.3, 0.4, topk if topk else -1)
            hist = [{"pred_prob": T_(prob[:, None, :].copy()), "pred_loc": T_(loc[:, None, :].copy()),
                     "tubes_nums": list(nums)}]
            dets = make_golden.run_reference_eval_loop(hist, len(nums), C, 0.3, 0.4, topk, 400, 400)[0]
        rows = [(b, c, s) + tuple(bx) for b, d in enumerate(dets) for (bx, c, s) in d]
        out[name + "_tp_rows"] = np.asarray(rows, np.float64).reshape(-1, 7)
    for k, v in make_merge_golden.out.items():
        if k.startswith("det_"):
            out[k] = v


def save_npz(path, arrays):
    """np.savez_compressed's layout with a fixed member date, so that a re-run writes the same bytes."""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k, v in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(v), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    gen_decode()
    gen_valid()
    gen_extrapolate()
    gen_extend()
    gen_update()
    gen_nms()
    gen_detect()
    save_npz(os.path.join(OUT, "nonfinite_cases.npz"), out)
    print("nonfinite cases:", len(out), "arrays")


if __name__ == "__main__":
    main()
