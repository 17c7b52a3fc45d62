"""CPU: the selection entry (step_select_step_f32) validates its arguments before any device work: STEP_E_ARG and a
step_last_error() text that names the problem, for null pointers, rows per clip below max_pos * (1 + neg_ratio), a
T_length that does not match the candidates' frames and the extension, and the other out-of-range fields."""
import ctypes

import pytest

from step_b200 import _lib


@pytest.fixture(scope="module")
def lib():
    return _lib.lib()


@pytest.fixture(scope="module")
def buf():
    b = (ctypes.c_char * (4096 + 16))()
    return b, (ctypes.addressof(b) + 15) & ~15              # fake device pointer (never dereferenced)


def params(p, **kw):
    d = dict(step=2, B=2, C=60, L=3, T=3, Lout=9, ext_mode=1, max_chunks=3, gt_mid=1, predict_nb=0, nb_first=0, nb_last=2,
             topk=300, max_pos=5, neg_ratio=2, sampling=2, max_rows=15, n_max=34, g_max=3, prop_f64=1, cls_thresh=0.2,
             reg_thresh=0.2, width=400.0, height=400.0, prob_sr=60, prob_sl=0, prob_sc=1)
    d.update({k: p for k in ("tube_off", "gt_off", "prob", "loc", "first", "last", "props", "targets", "mt", "out_tubes",
                             "out_targets", "counts")})
    d.update(kw)
    return _lib.step_select_params(**d)


def expect(lib, prm, *words):
    assert lib.step_select_step_f32(ctypes.byref(prm), None) == _lib.E_ARG
    msg = lib.step_last_error().decode()
    for w in words:
        assert w in msg, (w, msg)


@pytest.mark.parametrize("which", ["tube_off", "gt_off", "targets", "mt", "out_tubes", "out_targets", "counts"])
def test_null_pointer(lib, buf, which):
    expect(lib, params(buf[1], **{which: None}), "select_step", "null pointer")


def test_null_step_inputs(lib, buf):
    expect(lib, params(buf[1], step=2, prob=None), "prob / loc")
    expect(lib, params(buf[1], step=2, first=None), "first / last")
    expect(lib, params(buf[1], step=1, ext_mode=0, Lout=3, props=None), "props")
    assert lib.step_select_step_f32(None, None) == _lib.E_ARG


def test_rows_above_the_bound(lib, buf):
    expect(lib, params(buf[1], max_rows=14), "max_rows 14")
    expect(lib, params(buf[1], max_pos=6), "max_pos 6")
    expect(lib, params(buf[1], neg_ratio=-1), "neg_ratio")


@pytest.mark.parametrize("shape", [(3, 3, 3, 1), (3, 9, 3, 0), (9, 9, 3, 1), (3, 9, 3, 7)])
def test_t_length_mismatch(lib, buf, shape):
    L, Lout, T, ext = shape
    msg = "bad ext_mode" if ext == 7 else "T_length %d" % Lout
    expect(lib, params(buf[1], L=L, Lout=Lout, T=T, ext_mode=ext), msg)


def test_other_fields(lib, buf):
    expect(lib, params(buf[1], step=1, L=3, Lout=9), "step 1")
    expect(lib, params(buf[1], topk=30), "topk=30")
    expect(lib, params(buf[1], sampling=3), "sampling 3")
    expect(lib, params(buf[1], gt_mid=3), "gt_mid 3")
    expect(lib, params(buf[1], predict_nb=1, nb_first=-1), "neighbour chunks")
    expect(lib, params(buf[1], n_max=0), "n_max 0")
    expect(lib, params(buf[1], ext_mode=2, T=1, Lout=5, L=3), "EXTRAPOLATE")
    expect(lib, params(buf[1], n_max=5000, topk=-1), "shared memory")


def test_check_entry_needs_no_pointer(lib, buf):
    """step_select_check_f32 runs the field and shared-memory checks alone: pointers may be null."""
    assert lib.step_select_check_f32(ctypes.byref(params(None))) == 0
    prm = params(None, n_max=5000, topk=-1)
    assert lib.step_select_check_f32(ctypes.byref(prm)) == _lib.E_ARG
    assert "shared memory" in lib.step_last_error().decode()


def shipped_host_inputs(n=34, G=3):
    from types import SimpleNamespace
    import numpy as np
    cfg = SimpleNamespace(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, cls_thresh=[0.2, 0.35, 0.5],
                          reg_thresh=[0.2, 0.35, 0.5], num_classes=60, topk=300, temporal_mode="predict",
                          image_size=[400, 400], max_pos_num=5, selection_sampling="softmax", neg_ratio=2)
    rs = np.random.RandomState(0)
    targets = [rs.uniform(0, 200, (G, 3, 64)).astype(np.float32) for _ in range(2)]
    tubes = [rs.uniform(0, 200, (n, 3, 4)) for _ in range(2)]
    return cfg, targets, tubes


def test_select_samples_checks_every_step_before_any_device_work():
    """A later step's problem (its history's frames, the shared memory a step needs) is reported before step 1 is uploaded
    or launched: no CUDA is needed to refuse, and the generators are left alone."""
    import numpy as np
    import torch
    import step_b200
    cfg, targets, tubes = shipped_host_inputs()
    R = 68
    bad_frames = [{"pred_prob": torch.zeros(R, 60), "pred_loc": torch.zeros(R, 3, 4), "tubes_nums": [34, 34]},
                  {"pred_prob": torch.zeros(R, 60), "pred_loc": torch.zeros(R, 5, 4), "tubes_nums": [34, 34],
                   "pred_first_loc": torch.zeros(R, 3, 4), "pred_last_loc": torch.zeros(R, 3, 4)}]
    state = np.random.get_state()
    with pytest.raises(RuntimeError, match="T_length 9 does not match L=5"):
        step_b200.select_samples(cfg, bad_frames, targets, tubes)
    big = [np.zeros((5000, 3, 4)), np.zeros((5000, 3, 4))]
    cfg.topk, cfg.max_iter, cfg.NUM_CHUNKS = -1, 1, {1: 1}
    targets = [t[:, :1] for t in targets]
    with pytest.raises(RuntimeError, match="shared memory"):
        step_b200.select_samples(cfg, [], targets, big)
    assert np.array_equal(np.random.get_state()[1], state[1])
