"""CPU: oracle/select.py, the numpy restatement of train.py:291-310's sample selection, against the reference's own
train_select on every case of tests/golden/select_cases.npz: the flat tubes and targets of every step bit for bit, and
numpy's and Python's generator states after the call.  Also: the inputs the reference fails on raise ValueError, in the
oracle and in step_b200.select_samples, before anything touches CUDA."""
import json
import os
import random
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import select as osel

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "select_cases.npz")


def load_cases():
    z = np.load(GOLDEN)
    return z, [str(c) for c in z["cases"]]


def case_inputs(z, name):
    """(cfg, history with numpy arrays, targets, proposals, (numpy state, Python state) before, after) of one case."""
    d = json.loads(str(z[name + "_cfg"]))
    d["NUM_CHUNKS"] = {int(k): v for k, v in d["NUM_CHUNKS"].items()}
    cfg = SimpleNamespace(**d)
    nums, ngt = [int(v) for v in z[name + "_nums"]], [int(v) for v in z[name + "_ngt"]]
    targets = np.split(z[name + "_targets"], np.cumsum(ngt)[:-1])
    props = np.split(z[name + "_props"], np.cumsum(nums)[:-1])
    history = []
    for i in range(cfg.max_iter - 1):
        h = {"pred_prob": z["%s_prob%d" % (name, i)], "pred_loc": z["%s_loc%d" % (name, i)], "tubes_nums": nums}
        if "%s_first%d" % (name, i) in z:
            h["pred_first_loc"], h["pred_last_loc"] = z["%s_first%d" % (name, i)], z["%s_last%d" % (name, i)]
        history.append(h)
    states = []
    for tag in ("", "_after"):
        np_state = ("MT19937", z[name + "_np_key" + tag], int(z[name + "_np_pos" + tag]), 0, 0.0)
        py_state = (3, tuple(int(v) for v in z[name + "_py_state" + tag]), None)
        states.append((np_state, py_state))
    return cfg, history, targets, props, states[0], states[1]


def expected(z, name, cfg):
    return [(z["%s_tubes%d" % (name, i)], z["%s_targets_out%d" % (name, i)]) for i in range(cfg.max_iter)]


def set_states(st):
    np.random.set_state(st[0])
    random.setstate(st[1])


def states_equal(st):
    np_now, py_now = np.random.get_state(), random.getstate()
    return np.array_equal(np_now[1], st[0][1]) and np_now[2] == st[0][2] and py_now[1] == st[1][1]


z, CASES = load_cases()


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(name):
    cfg, history, targets, props, before, after = case_inputs(z, name)
    hist = [dict(h, pred_prob=np.broadcast_to(h["pred_prob"][:, None], (h["pred_prob"].shape[0], h["pred_loc"].shape[1],
                                                                         cfg.num_classes))) for h in history]
    set_states(before)
    st, sg = osel.select_samples(cfg, hist, targets, props)
    assert states_equal(after)
    for i, (t, g) in enumerate(expected(z, name, cfg)):
        assert st[i].dtype == np.float32 and np.array_equal(st[i], t), (name, i)
        assert np.array_equal(sg[i], g), (name, i)


def test_golden_covers_the_cases():
    rows = {n: [z["%s_tubes%d" % (n, i)].shape[0] for i in range(3)] for n in CASES}
    assert rows["empty_rows"] == [0, 0, 0]
    assert all(min(r) > 0 for n, r in rows.items() if n != "empty_rows")
    _, _, _, _, before, after = case_inputs(z, "many_gt_shuffle")
    assert before[1][1] != after[1][1]                       # random.shuffle drew from Python's generator
    cfg, _, targets, _, _, _ = case_inputs(z, "zero_gt_box")
    assert any((t[:, int(cfg.NUM_CHUNKS[cfg.max_iter] / 2), :4] == 0).all(-1).any() for t in targets)
    cfg, _, _, props, _, _ = case_inputs(z, "few_negatives")
    assert min(len(p) for p in props) < cfg.max_pos_num * (1 + cfg.neg_ratio)


def bad_inputs():
    cfg, history, targets, props, _, _ = case_inputs(z, "shipped_b2")
    yield "no ground truth", cfg, [targets[0][:0], targets[1]], props
    yield "no proposals", cfg, targets, [props[0], props[1][:0]]
    yield "candidates per class", SimpleNamespace(**dict(vars(cfg), topk=30)), targets, props


@pytest.mark.parametrize("k", range(3))
def test_reference_failures_raise_before_any_work(k):
    import step_b200
    msg, cfg, targets, props = list(bad_inputs())[k]
    with pytest.raises(ValueError, match=msg):
        osel.select_samples(cfg, [], targets, props)
    state = np.random.get_state()
    with pytest.raises(ValueError, match=msg):
        step_b200.select_samples(cfg, [], targets, props)     # no history and no CUDA needed to refuse
    assert np.array_equal(np.random.get_state()[1], state[1])
