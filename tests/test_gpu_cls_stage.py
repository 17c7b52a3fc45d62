"""GPU: the classification pre-training stage's sample selection and validation on the device.

- step_b200.select_cls_samples on every selection case of tests/golden/cls_stage_cases.npz (the reference's own
  select_proposals and flatten_tubes under train_cls.py's row building): the flat tubes and targets bit for bit, and
  numpy's and Python's generator states after the call;
- the reference's failures raise ValueError before any device work;
- train_step over the class-only heads gives the same loss and gradients on the device rows as on the same rows built on
  the host by oracle/select_cls.py;
- step_b200.postprocess.ClsDetector against a numpy restatement of train_cls.py:507-534, with scores exactly at
  conf_thresh and clips without a score above it;
- ClsDetector.run -> FrameAP.add_detections -> evaluate() against the reference's ava_evaluation metrics recorded in the
  fixture, under the tie contract of FrameAP (bit for bit in every class whose tie groups do not mix TPs and FPs, and
  bit for bit against oracle/evaluation.py everywhere);
- ClsDetector.run captured in a CUDA graph and replayed."""
import os
import random
import sys

import numpy as np
import pytest
import torch

from oracle import evaluation as oev
from oracle import select_cls as osel

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_cls_stage_cpu import (C, SEL_CASES, VAL_CASES, cls_detection_lines, selection_inputs, set_states,  # noqa: E402
                                states_equal, validation_inputs, z)

pytestmark = pytest.mark.gpu
F = np.float32


def bits(a):
    return np.asarray(a, np.float64).view(np.int64)


@pytest.mark.parametrize("name", SEL_CASES)
def test_selection_bit_identical_to_reference(name):
    import step_b200
    targets, props, before, after, (want_t, want_g) = selection_inputs(name)
    set_states(before)
    t, g = step_b200.select_cls_samples(targets, props, C)
    assert states_equal(after)
    assert t.is_cuda and g.is_cuda and t.dtype == torch.float32 and g.dtype == torch.float32
    assert tuple(t.shape) == want_t.shape and np.array_equal(t.cpu().numpy(), want_t)
    assert tuple(g.shape) == want_g.shape and np.array_equal(g.cpu().numpy(), want_g)


def test_selection_chains_the_generators_and_refuses_bad_clips():
    import step_b200
    targets, props, before, _, _ = selection_inputs("shuffle_cut")
    set_states(before)
    ref = [osel.train_cls_select(targets, props, C) for _ in range(2)]
    after = (np.random.get_state(), random.getstate())
    set_states(before)
    dev = [step_b200.select_cls_samples(targets, props, C) for _ in range(2)]
    assert states_equal(after)
    for (dt, dg), (rt, rg) in zip(dev, ref):
        assert np.array_equal(dt.cpu().numpy(), rt) and np.array_equal(dg.cpu().numpy(), rg)
    f32 = [p.astype(np.float32) for p in props]     # float32 proposals take the float32 IoU, as in numpy
    set_states(before)
    rt, rg = osel.train_cls_select(targets, f32, C)
    after = (np.random.get_state(), random.getstate())
    set_states(before)
    dt, dg = step_b200.select_cls_samples(targets, f32, C)
    assert states_equal(after)
    assert np.array_equal(dt.cpu().numpy(), rt) and np.array_equal(dg.cpu().numpy(), rg)
    state = np.random.get_state()
    with pytest.raises(ValueError, match="no ground truth"):
        step_b200.select_cls_samples([targets[0][:0], targets[1]], props, C)
    with pytest.raises(ValueError, match="no proposals"):
        step_b200.select_cls_samples(targets, [props[0], props[1][:0]], C)
    assert np.array_equal(np.random.get_state()[1], state[1])


def test_train_step_on_device_rows_equals_host_rows():
    """The selection of two clips at 64 x 64 (the fixture's boxes scaled by 64/400), then train_step over a class-only
    head with ContextNet on the device rows and on oracle/select_cls.py's host rows under the same generator states."""
    import step_b200
    from step_b200 import synth, training
    from test_oracle_cls import CLS_CFG
    targets, props, before, _, _ = selection_inputs("shuffle_cut")
    s = 64.0 / 400.0
    targets = [np.concatenate([t[:, :, :4] * F(s), t[:, :, 4:]], 2) for t in targets]
    props = [p * s for p in props]
    cfg = synth.make_cfg(fp16=True, **CLS_CFG, image_size=(64, 64))
    nets = synth.device_nets(cfg, [synth.cls_head_state_dict(100, cfg)], context=True, cls_only=True)
    x = synth.make_clips(2, 36, 64, 64, seed=11).cuda()
    set_states(before)
    dt, dg = step_b200.select_cls_samples(targets, props, cfg.num_classes)
    after = (np.random.get_state(), random.getstate())
    set_states(before)
    rt, rg = osel.train_cls_select(targets, props, cfg.num_classes)
    assert states_equal(after)
    assert np.array_equal(dt.cpu().numpy(), rt) and np.array_equal(dg.cpu().numpy(), rg)
    r_dev = training.train_step(cfg, nets, x, [dt], [dg])
    r_host = training.train_step(cfg, nets, x, [torch.from_numpy(rt).cuda()], [torch.from_numpy(rg).cuda()])
    torch.cuda.synchronize()
    assert float(r_dev["loss"]) == float(r_host["loss"])
    assert r_dev["grads"].keys() == r_host["grads"].keys() and len(r_dev["grads"]) > 0
    for p, g in r_dev["grads"].items():
        assert torch.equal(g, r_host["grads"][p])


def host_rows(prob, flat_tubes, nums, conf, width, height):
    """train_cls.py:507-534 in numpy: per clip the (box, score, class, proposal) rows in file order."""
    out, start = [], 0
    for n in nums:
        p, tb = prob[start:start + n], flat_tubes[start:start + n, flat_tubes.shape[1] // 2, 1:]
        start += n
        rows = []
        for cl in range(prob.shape[1]):
            keep = np.where(p[:, cl] > F(conf))[0]
            boxes = tb[keep].copy()
            boxes[:, ::2] /= width
            boxes[:, 1::2] /= height
            rows += [np.concatenate([boxes[k], [p[j, cl], cl, j, 0]]).astype(F) for k, j in enumerate(keep)]
        out.append(np.array(rows, F).reshape(-1, 8))
    return out


def batches(name):
    nums = [int(n) for n in z[name + "_nums"]]
    c0, r0 = 0, 0
    for nb in (int(v) for v in z[name + "_batches"]):
        n = nums[c0:c0 + nb]
        yield c0, nb, n, slice(r0, r0 + sum(n))
        c0, r0 = c0 + nb, r0 + sum(n)


@pytest.mark.parametrize("name", VAL_CASES)
def test_cls_detector_rows_equal_the_host_loop(name):
    from step_b200.postprocess import ClsDetector
    conf, W, H = float(z[name + "_conf"]), int(z[name + "_width"]), int(z[name + "_height"])
    prob, tubes = z[name + "_prob"], z[name + "_tubes"]
    at_conf = empty = 0
    for c0, nb, nums, rows in batches(name):
        d = ClsDetector(nums, C, "cuda:0", conf, W, H)
        res = d.run(torch.from_numpy(prob[rows]).cuda(), torch.from_numpy(tubes[rows]).cuda())
        assert res["det"].shape[1] == max(nums) * C and res["tubes_nums"] == nums
        det, cnt = res["det"].cpu().numpy(), res["count"].cpu().numpy()
        for b, want in enumerate(host_rows(prob[rows], tubes[rows], nums, conf, W, H)):
            assert cnt[b] == want.shape[0]
            assert np.array_equal(det[b, :cnt[b]], want), (name, c0 + b)
            empty += want.shape[0] == 0
        at_conf += int((prob[rows] == F(conf)).sum())
    if name == "val_ties":
        assert at_conf > 0 and empty > 0        # the strict threshold and clips without a row are exercised


@pytest.mark.parametrize("name", VAL_CASES)
def test_frame_ap_equals_reference_metrics(name):
    import step_b200
    from step_b200.postprocess import ClsDetector
    keys, gkeys, excl, cats = validation_inputs(name)
    label_dict = [int(v) for v in z["label_dict"]]
    conf, W, H = float(z[name + "_conf"]), int(z[name + "_width"]), int(z[name + "_height"])
    prob, tubes = z[name + "_prob"], z[name + "_tubes"]
    ev = step_b200.FrameAP(cats, label_dict, excl, device="cuda:0")
    ev.add_ground_truth(gkeys, z[name + "_gt_boxes"], z[name + "_gt_labels"])
    for c0, nb, nums, rows in batches(name):
        d = ClsDetector(nums, C, "cuda:0", conf, W, H)
        ev.add_detections(d.run(torch.from_numpy(prob[rows]).cuda(), torch.from_numpy(tubes[rows]).cuda()), keys[c0:c0 + nb])
    m = ev.evaluate()
    ap = ev.per_class_ap
    dlines = cls_detection_lines(prob, tubes, [int(n) for n in z[name + "_nums"]], keys, label_dict, conf, W, H)
    glines = oev.gt_lines(gkeys, z[name + "_gt_boxes"], z[name + "_gt_labels"])
    want = oev.run(cats, glines, dlines, excl).per_class_ap()
    assert np.array_equal(bits(ap), bits(want))
    ref, lo, hi = z[name + "_ref_ap"], z[name + "_ap_lo"], z[name + "_ap_hi"]
    exact = lo == hi
    assert np.array_equal(bits(ap[exact]), bits(ref[exact]))
    assert np.all(np.isnan(ref) | ((lo <= ap) & (ap <= hi)))
    if exact.all():
        assert bits(m["PascalBoxes_Precision/mAP@0.5IOU"]) == bits(z[name + "_ref_map"])


def test_cls_detector_run_in_a_cuda_graph():
    from step_b200.postprocess import ClsDetector
    name = "val_ties"
    conf, W, H = float(z[name + "_conf"]), int(z[name + "_width"]), int(z[name + "_height"])
    _, _, nums, rows = next(batches(name))
    prob = torch.from_numpy(z[name + "_prob"][rows]).cuda()
    tubes = torch.from_numpy(z[name + "_tubes"][rows]).cuda()
    d = ClsDetector(nums, C, "cuda:0", conf, W, H)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        d.run(prob, tubes)                      # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        d.run(prob, tubes)
    for seed in (1, 2):
        gen = torch.Generator(device="cuda").manual_seed(seed)
        prob.copy_(torch.rand(prob.shape, generator=gen, device="cuda") ** 4)
        g.replay()
        torch.cuda.synchronize()
        want = host_rows(prob.cpu().numpy(), tubes.cpu().numpy(), nums, conf, W, H)
        det, cnt = d.det.cpu().numpy(), d.count.cpu().numpy()
        for b, w in enumerate(want):
            assert cnt[b] == w.shape[0] and np.array_equal(det[b, :cnt[b]], w)
