"""CPU: demo.py's cross-class merge (demo.py:176-198).  The numpy restatement (oracle/merge.py) and the host line writer
(step_b200.postprocess.result_lines) against the reference's own loop (tests/golden/merge_cases.npz); the argument errors
of step_detect_merge_f32, returned before any launch."""
import ctypes

import numpy as np
import pytest

from oracle import merge as om
from oracle import postprocess as opp
from step_b200 import _lib
from step_b200.postprocess import result_lines

from _merge_case import CASES, LABELS, fixture_results, fixture_rows, infos, same_results


@pytest.mark.parametrize("name", CASES)
def test_oracle_merge_equals_reference(golden, name):
    z = golden("merge_cases")
    thr = float(z[name + "_cfg"][5])
    got = [om.demo_merge(d, LABELS, thr) for d in fixture_rows(z, name)]
    same_results(got, fixture_results(z, name))


@pytest.mark.parametrize("name", [c for c in CASES if c != "zero_area"])
def test_oracle_detections_give_the_reference_rows(golden, name):
    """The rows the merge reads are demo.py's scores_list: oracle.postprocess.detections on the same inputs."""
    z = golden("merge_cases")
    conf, nms, topk, width, height = z[name + "_cfg"][:5].tolist()
    dets = opp.detections(z[name + "_prob"], z[name + "_loc"], z[name + "_nums"].tolist(), conf, nms, width, height,
                          topk=int(topk))
    want = fixture_rows(z, name)
    for d, w in zip(dets, want):
        assert [(c, np.float32(s)) for _, c, s in d] == [(c, np.float32(s)) for _, c, s in w]
        assert all(np.array_equal(a[0], b[0]) for a, b in zip(d, w))


@pytest.mark.parametrize("name", CASES)
def test_result_lines_equal_reference_text(golden, name):
    z = golden("merge_cases")
    lines = result_lines(fixture_results(z, name), infos(len(z[name + "_nums"])))
    assert "".join(lines) == str(z[name + "_text"])


def test_fixture_edges_are_what_they_claim(golden):
    """The edge cases the fixture was built for: IoU exactly float32(0.8) stays apart, a repeated key, an empty clip and
    a one-row clip, and a group whose np.mean differs from a pairwise float32 sum."""
    z = golden("merge_cases")
    e = fixture_results(z, "edges")
    assert [len(r) for r in e] == [0, 4, 1, 0]
    rows = fixture_rows(z, "edges")[1]
    assert om.box_iou(rows[0][0], rows[1][0]) == np.float32(0.8)
    assert om.box_iou(rows[3][0], rows[4][0]) == np.nextafter(np.float32(0.8), np.float32(1))
    zr = fixture_rows(z, "zero_area")[0]
    assert len(zr) == 5 and len(fixture_results(z, "zero_area")[0]) == 3
    big = np.asarray([r[0] for r in fixture_rows(z, "big_group")[0]], np.float32)
    assert len(big) >= 100 and len(fixture_results(z, "big_group")[0]) == 1
    pairwise = np.asarray([np.sum(np.ascontiguousarray(big[:, c])) for c in range(4)], np.float32) / np.float32(len(big))
    assert not np.array_equal(big.mean(0), pairwise)


@pytest.fixture(scope="module")
def lib():
    return _lib.lib()


@pytest.fixture(scope="module")
def fake():
    b = (ctypes.c_char * (4096 + 256))()
    return (ctypes.addressof(b) + 255) & ~255, b           # fake device pointer (never dereferenced)


def expect(lib, p, *words, n_clips=4, cap=300, thresh=0.8, det=0, count=0, mbox=0, pairs=0, mcount=0, ws=0, ws_bytes=None):
    args = [p + det if det is not None else None, p if count is not None else None, n_clips, cap, thresh,
            p + mbox if mbox is not None else None, p if pairs is not None else None, p if mcount is not None else None,
            p + ws if ws is not None else None]
    if ws_bytes is None:
        ws_bytes = lib.step_detect_merge_workspace_bytes(n_clips, cap)
    before = _lib.launch_count()
    assert lib.step_detect_merge_f32(*args, ws_bytes, None) == _lib.E_ARG
    assert _lib.launch_count() == before
    msg = lib.step_last_error().decode()
    for w in words:
        assert w in msg, (w, msg)


def test_merge_argument_errors(lib, fake):
    p = fake[0]
    expect(lib, p, "n_clips -1", n_clips=-1)
    expect(lib, p, "n_clips 65536", n_clips=65536)
    expect(lib, p, "cap 0", cap=0)
    big = lib.step_detect_merge_max_rows() + 1
    expect(lib, p, "cap %d" % big, cap=big)
    for field in ("det", "count", "mbox", "pairs", "mcount", "ws"):
        expect(lib, p, "null pointer", **{field: None})
    expect(lib, p, "aligned", det=4)
    expect(lib, p, "aligned", mbox=8)
    expect(lib, p, "aligned", ws=16)
    need = lib.step_detect_merge_workspace_bytes(4, 300)
    expect(lib, p, "workspace %d < %d" % (need - 1, need), ws_bytes=need - 1)


def test_merge_sizes(lib):
    assert lib.step_detect_merge_max_rows() >= 34 * 60 * 16
    a, b = lib.step_detect_merge_workspace_bytes(8, 2040), lib.step_detect_merge_workspace_bytes(8, 300)
    assert a > b > 8 * 300 * 5 * 8
    assert a >= 8 * 2040 * 32 * 8                      # the bitmask: 2040 rows of 32 words per clip
    # no clips: nothing to do, not an error
    before = _lib.launch_count()
    assert lib.step_detect_merge_f32(None, None, 0, 300, 0.8, None, None, None, None, 0, None) == 0
    assert _lib.launch_count() == before
