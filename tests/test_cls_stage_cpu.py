"""CPU: the classification pre-training stage's two device entries without a GPU.

- oracle/select_cls.py's train_cls_select, the numpy restatement of train_cls.py:260-297, against the reference's own
  select_proposals and flatten_tubes on every selection case of tests/golden/cls_stage_cases.npz: the flat rows bit for bit
  and numpy's and Python's generator states after the call;
- the fixture's validation cases: the reference's metrics lie inside oracle/evaluation.py's tie bracket of the CSV text
  train_cls.py:537-543 writes;
- step_select_params.target_mode: zero by default, the last field, and checked (train_cls rows need step 1, no extension);
- step_detect_scores_f32 / step_detect_scores_check refuse bad arguments with STEP_E_ARG before any launch;
- select_cls_samples refuses the inputs the reference fails on before anything touches CUDA, and leaves the generators."""
import ctypes
import os
import random
import sys

import numpy as np
import pytest

from oracle import evaluation as oev
from oracle import select_cls as osel
from step_b200 import _lib

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_cls_stage_golden import C, cls_detection_lines  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cls_stage_cases.npz")
z = np.load(GOLDEN)
SEL_CASES = [str(c) for c in z["sel_cases"]]
VAL_CASES = [str(c) for c in z["val_cases"]]


def selection_inputs(name):
    """(targets, proposals, (numpy state, Python state) before, after, (flat tubes, flat targets)) of one case."""
    nums, ngt = [int(v) for v in z[name + "_nums"]], [int(v) for v in z[name + "_ngt"]]
    targets = np.split(z[name + "_targets"], np.cumsum(ngt)[:-1])
    props = np.split(z[name + "_props"], np.cumsum(nums)[:-1])
    states = []
    for tag in ("", "_after"):
        np_state = ("MT19937", z[name + "_np_key" + tag], int(z[name + "_np_pos" + tag]), 0, 0.0)
        py_state = (3, tuple(int(v) for v in z[name + "_py_state" + tag]), None)
        states.append((np_state, py_state))
    return targets, props, states[0], states[1], (z[name + "_tubes"], z[name + "_targets_out"])


def set_states(st):
    np.random.set_state(st[0])
    random.setstate(st[1])


def states_equal(st):
    np_now, py_now = np.random.get_state(), random.getstate()
    return np.array_equal(np_now[1], st[0][1]) and np_now[2] == st[0][2] and py_now[1] == st[1][1]


def validation_inputs(name):
    keys = list(zip([str(v) for v in z[name + "_video"]], [int(f) for f in z[name + "_fid"]]))
    gkeys = list(zip([str(v) for v in z[name + "_gt_video"]], [int(f) for f in z[name + "_gt_fid"]]))
    excl = list(zip([str(v) for v in z[name + "_excl_video"]], [int(f) for f in z[name + "_excl_fid"]]))
    cats = [{"id": int(i), "name": str(n)} for i, n in zip(z["cat_ids"], z["cat_names"])]
    return keys, gkeys, excl, cats


@pytest.mark.parametrize("name", SEL_CASES)
def test_oracle_rows_match_reference(name):
    targets, props, before, after, (want_t, want_g) = selection_inputs(name)
    set_states(before)
    got_t, got_g = osel.train_cls_select(targets, props, C)
    assert states_equal(after)
    assert got_t.dtype == np.float32 and np.array_equal(got_t, want_t)
    assert np.array_equal(got_g, want_g)


def test_golden_covers_the_cases():
    _, _, before, after, _ = selection_inputs("shuffle_cut")
    assert before[1][1] != after[1][1]                       # random.shuffle drew from Python's generator
    targets, props, _, _, (t, g) = selection_inputs("extra_positives")
    clip = (t[:, 0, 0] // t.shape[1]).astype(int)
    assert any((g[clip == b, 1, :4].any(1)).sum() > tg.shape[0] for b, tg in enumerate(targets))
    targets, props, _, _, (t, g) = selection_inputs("no_free_negatives")
    clip = (t[:, 0, 0] // t.shape[1]).astype(int)
    assert (clip == 0).sum() == len(props[0]) and g[clip == 0, 1, :4].any(1).all()   # every proposal is a positive
    assert [len(selection_inputs(n)[0]) for n in ("b1_one_gt", "b4")] == [1, 4]
    assert selection_inputs("chunks3_b4")[0][0].shape[1] == 3
    assert all(p.dtype == np.float64 for n in SEL_CASES for p in selection_inputs(n)[1])
    for n in SEL_CASES:                                      # every row carries the classification flag, never regression
        g = z[n + "_targets_out"]
        assert (g[:, :, 4] == 1).all() and (g[:, :, 5] == 0).all() and (g[:, 0] == g[:, 1]).all() and (g[:, 2] == g[:, 1]).all()


@pytest.mark.parametrize("name", VAL_CASES)
def test_validation_reference_inside_the_oracle_bracket(name):
    keys, gkeys, excl, cats = validation_inputs(name)
    label_dict = [int(v) for v in z["label_dict"]]
    dlines = cls_detection_lines(z[name + "_prob"], z[name + "_tubes"], [int(n) for n in z[name + "_nums"]], keys,
                                 label_dict, float(z[name + "_conf"]), int(z[name + "_width"]), int(z[name + "_height"]))
    assert len(dlines) == int(z[name + "_rows"])
    glines = oev.gt_lines(gkeys, z[name + "_gt_boxes"], z[name + "_gt_labels"])
    lo, hi = oev.run(cats, glines, dlines, excl).ap_bounds()
    assert np.array_equal(lo, z[name + "_ap_lo"], equal_nan=True) and np.array_equal(hi, z[name + "_ap_hi"], equal_nan=True)
    ref = z[name + "_ref_ap"]
    ok = np.isnan(ref) | ((lo <= ref) & (ref <= hi))
    assert ok.all()
    exact = (lo == hi) & ~np.isnan(ref)
    assert np.array_equal(lo[exact], ref[exact])


# ---- ABI ----
@pytest.fixture(scope="module")
def lib():
    return _lib.lib()


@pytest.fixture(scope="module")
def fake():
    b = (ctypes.c_char * (4096 + 16))()
    return (ctypes.addressof(b) + 15) & ~15, b               # fake device pointer (never dereferenced)


def test_target_mode_is_the_last_field_and_defaults_to_select_rows():
    fields = [f[0] for f in _lib.step_select_params._fields_]
    assert fields[-1] == "target_mode"
    assert _lib.step_select_params().target_mode == _lib.TARGETS_SELECT == 0
    assert _lib.TARGETS_CLS == 1


def cls_params(p, **kw):
    d = dict(step=1, B=2, C=60, L=9, T=9, Lout=9, ext_mode=0, max_chunks=1, gt_mid=0, topk=0, max_pos=5, neg_ratio=3,
             sampling=0, max_rows=20, n_max=16, g_max=4, prop_f64=1, cls_thresh=0.75, target_mode=1)
    d.update({k: p for k in ("tube_off", "gt_off", "props", "targets", "mt", "out_tubes", "out_targets", "counts")})
    d.update(kw)
    return _lib.step_select_params(**d)


def test_select_target_mode_checks(lib, fake):
    before = _lib.launch_count()
    assert lib.step_select_check_f32(ctypes.byref(cls_params(None))) == 0
    for kw, words in ((dict(target_mode=2), "bad target_mode 2"), (dict(target_mode=-1), "bad target_mode -1"),
                      (dict(step=2, prob=fake[0], loc=fake[0]), "needs step 1"),
                      (dict(predict_nb=1, max_chunks=3, nb_last=2), "no neighbour rows")):
        prm = cls_params(fake[0], **kw)
        assert lib.step_select_check_f32(ctypes.byref(prm)) == _lib.E_ARG
        assert lib.step_select_step_f32(ctypes.byref(prm), None) == _lib.E_ARG
        msg = lib.step_last_error().decode()
        assert words in msg, (words, msg)
    assert _lib.launch_count() == before


def detect_args(p, **kw):
    d = dict(prob=p, prob_ld=60, box=p, box_ld=45, clip_offsets=p, n_clips=4, n_rows=80, max_per_clip=24, ncls=60,
             conf=0.01, norm_w=400.0, norm_h=400.0, cap=24 * 60, det=p, det_count=p)
    d.update(kw)
    return d


def call_check(lib, d):
    return lib.step_detect_scores_check(d["prob"], d["prob_ld"], d["box"], d["box_ld"], d["clip_offsets"], d["n_clips"],
                                        d["n_rows"], d["max_per_clip"], d["ncls"], d["cap"], d["det"], d["det_count"])


def call_run(lib, d):
    return lib.step_detect_scores_f32(d["prob"], d["prob_ld"], d["box"], d["box_ld"], d["clip_offsets"], d["n_clips"],
                                      d["n_rows"], d["max_per_clip"], d["ncls"], d["conf"], d["norm_w"], d["norm_h"],
                                      d["cap"], d["det"], d["det_count"], None)


@pytest.mark.parametrize("kw,words", [
    (dict(prob=None), "null pointer"), (dict(box=None), "null pointer"), (dict(clip_offsets=None), "null pointer"),
    (dict(det=None), "null pointer"), (dict(det_count=None), "null pointer"),
    (dict(ncls=0), "bad sizes"), (dict(n_clips=-1), "bad sizes"), (dict(max_per_clip=81), "max_per_clip 81"),
    (dict(prob_ld=59), "prob_ld 59"), (dict(box_ld=3), "box_ld 3"), (dict(cap=24 * 60 - 1), "cap 1439"),
    (dict(cap=0, max_per_clip=0), "cap 0"),
])
def test_detect_scores_refuses_bad_arguments(lib, fake, kw, words):
    d = detect_args(fake[0], **kw)
    before = _lib.launch_count()
    for fn in (call_check, call_run):
        assert fn(lib, d) == _lib.E_ARG
        msg = lib.step_last_error().decode()
        assert "step_detect_scores_f32" in msg and words in msg, (words, msg)
    assert _lib.launch_count() == before


def test_detect_scores_check_accepts_good_arguments(lib, fake):
    before = _lib.launch_count()
    assert call_check(lib, detect_args(fake[0])) == 0
    assert call_check(lib, detect_args(None, n_clips=0)) == 0     # nothing to do: no pointer is read
    assert call_run(lib, detect_args(None, n_clips=0)) == 0
    assert _lib.launch_count() == before


@pytest.mark.parametrize("which", ["no ground truth", "no proposals", "lists", "targets", "tubes", "sampling"])
def test_select_cls_samples_refuses_before_any_work(which):
    import step_b200
    targets, props, _, _, _ = selection_inputs("b4")
    if which == "no ground truth":
        targets = [targets[0][:0]] + targets[1:]
    elif which == "no proposals":
        props = props[:3] + [props[3][:0]]
    elif which == "lists":
        props = props[:3]
    elif which == "targets":
        targets = [t[:, :, :10] for t in targets]
    elif which == "tubes":
        props = [p[:, :, :3] for p in props]
    state, pystate = np.random.get_state(), random.getstate()
    with pytest.raises(ValueError, match="target lists" if which == "lists" else which):
        step_b200.select_cls_samples(targets, props, C, sampling="bad" if which == "sampling" else "uniform")
    assert np.array_equal(np.random.get_state()[1], state[1]) and random.getstate() == pystate
    if which in ("no ground truth", "no proposals"):
        with pytest.raises(ValueError, match=which):
            osel.train_cls_select(targets, props, C)
