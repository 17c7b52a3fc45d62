"""CPU: the frame-mAP entries (step_eval_append, step_eval_run) validate their arguments before any device work:
STEP_E_ARG and a step_last_error() text that names the field, for null pointers, limits exceeded and bad tables; the
launch-free checks accept good arguments with no launch."""
import ctypes

import pytest

from step_b200 import _lib


@pytest.fixture(scope="module")
def lib():
    return _lib.lib()


@pytest.fixture(scope="module")
def fake():
    b = (ctypes.c_char * (4096 + 16))()
    return (ctypes.addressof(b) + 15) & ~15, b               # fake device pointer (never dereferenced)


def rows(p, **kw):
    d = dict(capacity=1000, counters=p, img_first=p, box=p, score=p, scode=p, img=p, cls=p)
    d.update(kw)
    return _lib.step_eval_rows(**d)


def append_params(p, img=(0, 1), rows_kw=None, **kw):
    d = dict(det=p, count=p, B=len(img), cap=300, ncls=60, class_of=p, rows=rows(p, **(rows_kw or {})))
    d.update(kw)
    prm = _lib.step_eval_append_params(**d)
    prm.img[:len(img)] = list(img)
    return prm


def run_params(lib, p, rows_kw=None, **kw):
    d = dict(rows=rows(p, **(rows_kw or {})), n_rows=500, n_classes=80, n_images=40, n_gt=100, max_gt_per_image=6,
             gt_box=p, gt_cls=p, gt_img_off=p, num_gt=p, workspace=p, ap=p)
    d.update(kw)
    d.setdefault("workspace_bytes", lib.step_eval_workspace_bytes(d["n_rows"], d["n_classes"], d["n_gt"]))
    return _lib.step_eval_params(**d)


def expect(lib, fn, prm, *words):
    before = _lib.launch_count()
    assert fn(ctypes.byref(prm), None) == _lib.E_ARG
    assert _lib.launch_count() == before
    msg = lib.step_last_error().decode()
    for w in words:
        assert w in msg, (w, msg)


def test_checks_accept_good_arguments(lib, fake):
    before = _lib.launch_count()
    assert lib.step_eval_append_check(ctypes.byref(append_params(fake[0]))) == 0
    assert lib.step_eval_check(ctypes.byref(run_params(lib, fake[0]))) == 0
    assert _lib.launch_count() == before


@pytest.mark.parametrize("field", ["det", "count", "class_of"])
def test_append_null_pointer(lib, fake, field):
    expect(lib, lib.step_eval_append, append_params(fake[0], **{field: None}), "eval_append", "null pointer")


@pytest.mark.parametrize("field", ["counters", "img_first", "box", "scode", "img", "cls"])
def test_rows_null_pointer(lib, fake, field):
    expect(lib, lib.step_eval_append, append_params(fake[0], rows_kw={field: None}), "null pointer", field)
    expect(lib, lib.step_eval_run, run_params(lib, fake[0], rows_kw={field: None}), "null pointer", field)


def test_append_limits(lib, fake):
    p = fake[0]
    expect(lib, lib.step_eval_append, append_params(p, B=65), "B 65")
    expect(lib, lib.step_eval_append, append_params(p, cap=0), "cap 0")
    expect(lib, lib.step_eval_append, append_params(p, img=(0, 1 << 20)), "img[1] 1048576")
    expect(lib, lib.step_eval_append, append_params(p, img=(-2,)), "img[0] -2")
    expect(lib, lib.step_eval_append, append_params(p, rows_kw={"capacity": (1 << 30) + 1}), "rows.capacity")
    expect(lib, lib.step_eval_append, append_params(p, B=64, cap=(1 << 24) + 1), "B * cap")
    assert lib.step_eval_append(None, None) == _lib.E_ARG


def test_run_limits_and_tables(lib, fake):
    p = fake[0]
    expect(lib, lib.step_eval_run, run_params(lib, p, n_classes=0), "n_classes 0")
    expect(lib, lib.step_eval_run, run_params(lib, p, n_classes=129), "n_classes 129")
    expect(lib, lib.step_eval_run, run_params(lib, p, n_images=(1 << 20) + 1), "n_images")
    expect(lib, lib.step_eval_run, run_params(lib, p, max_gt_per_image=1025), "max_gt_per_image 1025")
    expect(lib, lib.step_eval_run, run_params(lib, p, n_rows=1001), "n_rows 1001")
    expect(lib, lib.step_eval_run, run_params(lib, p, workspace_bytes=64), "workspace_bytes 64")
    for field in ("gt_img_off", "num_gt", "ap", "workspace"):
        expect(lib, lib.step_eval_run, run_params(lib, p, **{field: None}), "null pointer", field)
    expect(lib, lib.step_eval_run, run_params(lib, p, gt_box=None), "null pointer", "gt_box")
    assert lib.step_eval_check(ctypes.byref(run_params(lib, p, n_gt=0, gt_box=None, gt_cls=None))) == 0
    assert lib.step_eval_run(None, None) == _lib.E_ARG


def test_frame_ap_rejects_bad_tables_without_cuda():
    import step_b200
    cats = [{"id": 1, "name": "a"}, {"id": 3, "name": "b"}]
    with pytest.raises(ValueError, match="1-based"):
        step_b200.FrameAP([{"id": 0, "name": "z"}], [1], device="cuda:0")
    with pytest.raises(ValueError, match="exceeds 128"):
        step_b200.FrameAP([{"id": 129, "name": "z"}], [1], device="cuda:0")
    with pytest.raises(ValueError, match="no categories"):
        step_b200.FrameAP([], [1], device="cuda:0")
    with pytest.raises(RuntimeError, match="CUDA device"):
        step_b200.FrameAP(cats, [1, 3], device="cpu")
