"""GPU: step_b200.FrameAP (eval.cu) against oracle/evaluation.py and the reference's recorded metrics: the device CSV
rounding against Python's, every golden case bit for bit, Detector.run -> FrameAP end to end against the CSV text
test.py writes, add_detections without synchronisation, and over-limit input refused before any launch."""
import numpy as np
import pytest
import torch

from oracle import evaluation as oev

from test_oracle_eval import bits, case_text, load

pytestmark = pytest.mark.gpu


def categories():
    _, cats, _ = load()
    return cats


def run_device(z, cats, name):
    keys = list(zip([str(v) for v in z[name + "_video"]], [int(f) for f in z[name + "_fid"]]))
    gkeys = list(zip([str(v) for v in z[name + "_gt_video"]], [int(f) for f in z[name + "_gt_fid"]]))
    excl = list(zip([str(v) for v in z[name + "_excl_video"]], [int(f) for f in z[name + "_excl_fid"]]))
    import step_b200
    ev = step_b200.FrameAP(cats, [int(v) for v in z[name + "_label_dict"]], excl, device="cuda:0")
    ev.add_ground_truth(gkeys, z[name + "_gt_boxes"], z[name + "_gt_labels"])
    det, count = torch.from_numpy(z[name + "_det"]).cuda(), torch.from_numpy(z[name + "_count"]).cuda()
    b0 = 0
    for nb in z[name + "_batches"]:
        ev.add_detections({"det": det[b0:b0 + nb].contiguous(), "count": count[b0:b0 + nb].contiguous()}, keys[b0:b0 + nb])
        b0 += int(nb)
    return ev.evaluate(), ev.per_class_ap


@pytest.mark.parametrize("name", ["distinct", "ties", "ties_fine", "edge", "many"])
def test_golden_case(name):
    z, cats, _ = load()
    m, ap = run_device(z, cats, name)
    gt, det, excl = case_text(z, name)
    want = oev.run(cats, gt, det, excl).per_class_ap()
    assert np.array_equal(bits(ap), bits(want)), (ap, want)
    om = oev.metrics(cats, want)
    assert list(m) == list(om) and all(bits(m[k]) == bits(om[k]) for k in m)
    if bool(z[name + "_tie_free"]):
        assert np.array_equal(bits(ap), bits(z[name + "_ref_ap"]))
        assert bits(m["PascalBoxes_Precision/mAP@0.5IOU"]) == bits(z[name + "_ref_map"])


def rounding_inputs():
    vals = []
    for e in range(-45, 8):
        for base in (1.0, 1.0005, 1.00005, 9.9995, 5.0005, 1.2345, 0.99995, 2.5):
            x = np.float32(base * 10.0 ** e)
            if not np.isfinite(x) or x == 0:
                continue
            b = int(x.view(np.int32))
            vals.extend(np.arange(b - 64, b + 65, dtype=np.int64).astype(np.int32).view(np.float32).tolist())
    rs = np.random.RandomState(3)
    r = rs.randint(0, 2 ** 31 - 1, 1100000).astype(np.int32).view(np.float32)
    r = r[np.isfinite(r)][:1000000]
    v = np.concatenate([np.array(vals, np.float32), r, -r[:2000] * np.float32(1e-3), np.float32([0.0, -0.0])])
    return v[v > -10]


def test_device_rounding_equals_python():
    """Every value goes through add_detections as a score (box (0, 0, 1, 1)); the store's scores are the parsed CSV."""
    import step_b200
    v = rounding_inputs()
    n = v.size
    det = np.zeros((1, n, 8), np.float32)
    det[0, :, 2:4] = 1.0
    det[0, :, 4] = v
    ev = step_b200.FrameAP([{"id": 1, "name": "a"}], [1], device="cuda:0")
    ev.add_detections({"det": torch.from_numpy(det).cuda(), "count": torch.tensor([n], dtype=torch.int32).cuda()}, [("v", 1)])
    torch.cuda.synchronize()
    got = ev._score[:n].cpu().numpy()
    want = np.array([float(format(float(x), ".4")) for x in v])
    bad = np.where(got.view(np.int64) != want.view(np.int64))[0]
    assert bad.size == 0, [(repr(v[i]), got[i], want[i]) for i in bad[:5]]
    # box coordinates take the same path: a few, including subnormals and decade crossings
    box = np.float32([1e-45, 9.9995e-3, 0.99995, 1.00005e-3])
    det2 = np.zeros((1, 1, 8), np.float32)
    det2[0, 0, :4] = [box[0], box[1], box[2], 2.0]
    det2[0, 0, 4] = 0.5
    ev.reset()
    ev.add_detections({"det": torch.from_numpy(det2).cuda(), "count": torch.tensor([1], dtype=torch.int32).cuda()}, [("v", 1)])
    torch.cuda.synchronize()
    y1, x1, y2, x2 = ev._box[0].cpu().numpy()
    assert [x1, y1, x2, y2] == [oev.csv_round(b) for b in (box[0], box[1], box[2], 2.0)]


def test_end_to_end_detector_to_frame_ap():
    """2,000 frames in 8-clip batches: Detector.run on seeded scores and boxes, then FrameAP; against the oracle on the
    CSV text test.py:210-218 writes from postprocess.to_lists."""
    from step_b200.postprocess import Detector, to_lists
    import step_b200
    cats = categories()
    ld = sorted(c["id"] for c in cats)
    C, n_tubes, B, T = len(ld), 12, 8, 3
    rs = np.random.RandomState(11)
    ev = step_b200.FrameAP(cats, ld, [("v0", 905)], device="cuda:0")
    det_lines, gkeys, gboxes, glabels = [], [], [], []
    detector = Detector([n_tubes] * B, C, torch.device("cuda:0"), 0.05, 0.3, 400, 400)
    for fb in range(0, 2000, B):
        keys = [("v%d" % ((fb + b) // 100), 900 + (fb + b) % 100) for b in range(B)]
        locs = []
        for key in keys:
            g = rs.randint(1, 7)
            xy = rs.uniform(0, 0.6, (g, 2))
            wh = rs.uniform(0.1, 0.4, (g, 2))
            boxes = np.concatenate([xy, xy + wh], 1)
            for k in range(g):
                gkeys.append(key)
                gboxes.append(boxes[k])
                glabels.append(ld[rs.randint(0, C)])
            src = boxes[rs.randint(0, g, n_tubes)] * 400 + rs.normal(0, 12, (n_tubes, 4))
            locs.append(np.repeat(src[:, None], T, 1))
        prob = rs.dirichlet(np.full(C, 0.3), B * n_tubes).astype(np.float32)
        loc = np.concatenate(locs).astype(np.float32)
        out = detector.run(torch.from_numpy(prob).cuda(), torch.from_numpy(loc).cuda())
        ev.add_detections(out, keys)
        det_lines += oev.detection_lines(to_lists(out), keys, ld)
    ev.add_ground_truth(gkeys, gboxes, glabels)
    m = ev.evaluate()
    ref = oev.run(cats, oev.gt_lines(gkeys, gboxes, glabels), det_lines, [("v0", 905)])
    want = ref.per_class_ap()
    assert np.array_equal(bits(ev.per_class_ap), bits(want))
    om = oev.metrics(cats, want)
    assert all(bits(m[k]) == bits(om[k]) for k in om)
    assert np.isfinite(m["PascalBoxes_Precision/mAP@0.5IOU"])


def test_add_detections_does_not_synchronise():
    import step_b200
    z, cats, _ = load()
    name = "distinct"
    ev = step_b200.FrameAP(cats, [int(v) for v in z[name + "_label_dict"]], device="cuda:0")
    det, count = torch.from_numpy(z[name + "_det"][:8]).cuda(), torch.from_numpy(z[name + "_count"][:8]).cuda()
    keys = [("s", i) for i in range(8)]
    ev.reserve(100000)
    ev.add_detections({"det": det, "count": count}, keys)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(20):
            ev.add_detections({"det": det, "count": count}, [("s", 8 * (i + 1) + j) for j in range(8)])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    ev.evaluate()


def test_over_limit_input_is_refused_before_any_launch():
    import step_b200
    from step_b200 import _lib
    cats = categories()
    ev = step_b200.FrameAP(cats, sorted(c["id"] for c in cats), device="cuda:0")
    ev.add_ground_truth([("g", 1)] * 1025, np.tile([0.1, 0.1, 0.5, 0.5], (1025, 1)), [cats[0]["id"]] * 1025)
    before = _lib.launch_count()
    with pytest.raises(RuntimeError, match="max_gt_per_image 1025"):
        ev.evaluate()
    assert _lib.launch_count() == before
    ev.reset()
    ev._ids = {("k%d" % i): i for i in range(1 << 20)}          # every image id taken: the next one is out of range
    det = torch.zeros((1, 4, 8), dtype=torch.float32, device="cuda:0")
    with pytest.raises(RuntimeError, match="img\\[0\\] 1048576"):
        ev.add_detections({"det": det, "count": torch.ones(1, dtype=torch.int32, device="cuda:0")}, [("new", 1)])
    assert _lib.launch_count() == before
