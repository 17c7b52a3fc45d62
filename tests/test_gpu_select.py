"""GPU: step_b200.select_samples, the training-sample selection of train.py:291-310 on the device.

- every case of tests/golden/select_cases.npz (the reference's own train_select): with the history on the device as
  step_b200.inference returns it (pred_prob an expand view), the flat tubes and targets of every step are bit-identical,
  and numpy's and Python's generator states after the call are the reference's;
- histories with tied scores, a materialised [R, L, C] pred_prob and float32 proposals against oracle/select.py, whose tie
  rule the device shares;
- two consecutive calls chain the generators as two reference iterations do;
- end to end at the shipped configuration (scripts/train_step.sh) with the synthetic nets and ContextNet, in the ROIPool
  and ROIAlign modes: step_b200.inference as the pre-pass, then select_samples, against oracle/select.py on the history
  copied to the host under the same seeds; train_step on the two selections gives bit-identical losses and gradients."""
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import select as osel

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_oracle_select as tos  # noqa: E402
from _train_case import SHIPPED  # noqa: E402
from step_b200.synth import device_nets  # noqa: E402

pytestmark = pytest.mark.gpu


def device_history(cfg, history, materialise=False):
    out = []
    for h in history:
        L = h["pred_loc"].shape[1]
        prob = torch.from_numpy(h["pred_prob"]).cuda().view(-1, 1, cfg.num_classes).expand(-1, L, -1)
        d = {"pred_prob": prob.contiguous() if materialise else prob, "pred_loc": torch.from_numpy(h["pred_loc"]).cuda(),
             "pred_first_loc": None, "pred_last_loc": None, "tubes_nums": h["tubes_nums"]}
        if "pred_first_loc" in h:
            d["pred_first_loc"] = torch.from_numpy(h["pred_first_loc"]).cuda()
            d["pred_last_loc"] = torch.from_numpy(h["pred_last_loc"]).cuda()
        out.append(d)
    return out


def host_history(cfg, history):
    return [dict(h, pred_prob=np.broadcast_to(h["pred_prob"][:, None], (h["pred_prob"].shape[0], h["pred_loc"].shape[1],
                                                                         cfg.num_classes))) for h in history]


def assert_same(dev, ref, what):
    for i, (d, r) in enumerate(zip(dev, ref)):
        d = d.cpu().numpy()
        assert d.shape == r.shape, (what, i, d.shape, r.shape)
        assert np.array_equal(d, r), (what, i, np.argwhere(d != r)[:5])


@pytest.mark.parametrize("name", tos.CASES)
def test_golden_case_bit_identical(name):
    import step_b200
    cfg, history, targets, props, before, after = tos.case_inputs(tos.z, name)
    tos.set_states(before)
    st, sg = step_b200.select_samples(cfg, device_history(cfg, history), targets, props)
    assert tos.states_equal(after)
    exp = tos.expected(tos.z, name, cfg)
    assert_same(st, [e[0] for e in exp], "tubes")
    assert_same(sg, [e[1] for e in exp], "targets")
    for t in st + sg:
        assert t.is_cuda and t.dtype == torch.float32


def tie_case():
    """The shipped case with scores on a coarse grid (ties inside each class and across classes), float32 proposals."""
    cfg, history, targets, props, before, _ = tos.case_inputs(tos.z, "shipped_b2")
    for h in history:
        h["pred_prob"] = (np.round(h["pred_prob"] * 8) / 8).astype(np.float32)
    props = [p.astype(np.float32) for p in props]
    return cfg, history, targets, props, before


@pytest.mark.parametrize("materialise", [False, True])
def test_ties_follow_the_oracle(materialise):
    import step_b200
    cfg, history, targets, props, before = tie_case()
    tos.set_states(before)
    ref = osel.select_samples(cfg, host_history(cfg, history), targets, props)
    after = (np.random.get_state(), random.getstate())
    tos.set_states(before)
    st, sg = step_b200.select_samples(cfg, device_history(cfg, history, materialise), targets, props)
    assert tos.states_equal(after)
    assert_same(st, ref[0], "tubes")
    assert_same(sg, ref[1], "targets")


def test_two_calls_chain_the_generators():
    import step_b200
    cfg, history, targets, props, before, _ = tos.case_inputs(tos.z, "many_gt_shuffle")
    hh, dh = host_history(cfg, history), device_history(cfg, history)
    tos.set_states(before)
    ref = [osel.select_samples(cfg, hh, targets, props) for _ in range(2)]
    after = (np.random.get_state(), random.getstate())
    tos.set_states(before)
    dev = [step_b200.select_samples(cfg, dh, targets, props) for _ in range(2)]
    assert tos.states_equal(after)
    for d, r in zip(dev, ref):
        assert_same(d[0], r[0], "tubes")
        assert_same(d[1], r[1], "targets")
    assert not all(np.array_equal(a.cpu().numpy(), b.cpu().numpy()) for a, b in zip(dev[0][0], dev[1][0]))


def shipped_inputs(B=2, n=34, G=3, W=64, seed=4):
    from step_b200 import synth
    cfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(W, W))
    cfg.__dict__.update(cls_thresh=[0.2, 0.35, 0.5], reg_thresh=[0.2, 0.35, 0.5], topk=300, max_pos_num=5,
                        selection_sampling="softmax", neg_ratio=2)
    rs = np.random.RandomState(seed)
    targets, tubes = [], []
    for _ in range(B):
        x1, y1 = rs.uniform(0, 0.5 * W, (2, G, 1))
        w, h = rs.uniform(0.2 * W, 0.45 * W, (2, G, 1))
        box = np.concatenate([x1, y1, x1 + w, y1 + h], 1)
        tg = np.zeros((G, 3, 4 + cfg.num_classes), np.float32)
        tg[:, :, :4] = box[:, None] + rs.uniform(-1, 1, (G, 3, 4))
        tg[:, :, 4:] = rs.uniform(0, 1, (G, 3, cfg.num_classes)) > 0.9
        targets.append(tg)
        src = box[rs.randint(0, G, n)] + rs.normal(0, 0.1 * W, (n, 4))
        src[:, 2:] = np.maximum(src[:, 2:], src[:, :2] + 4)
        tubes.append(np.tile(src[:, None], (1, cfg.T, 1)))
    return cfg, targets, tubes


@pytest.mark.parametrize("pool_mode", ["pool", "align"])
def test_end_to_end_shipped_config(pool_mode):
    import step_b200
    from step_b200 import synth, training
    cfg, targets, tubes = shipped_inputs()
    nets = device_nets(cfg, [synth.head_state_dict(100 + i, cfg) for i in range(3)], pool_mode, context=True)
    x = synth.make_clips(2, 36, 64, 64, seed=11).cuda()
    with torch.no_grad():
        cf = nets["base_net"](x)
        ctx = nets["context_net"](cf)
        hist, _ = step_b200.inference(cfg, cf, ctx, nets, cfg.max_iter - 1, tubes, want_trajectory=False)
    np.random.seed(5)
    random.seed(6)
    st, sg = step_b200.select_samples(cfg, hist, targets, tubes)
    after = (np.random.get_state(), random.getstate())
    hh = [{k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in h.items()} for h in hist]
    np.random.seed(5)
    random.seed(6)
    rt, rg = osel.select_samples(cfg, hh, targets, tubes)
    assert tos.states_equal(after)
    assert_same(st, rt, "tubes")
    assert_same(sg, rg, "targets")
    assert [t.shape[1] for t in st] == [3, 3, 9] and all(t.shape[0] > 0 for t in st)
    r_dev = training.train_step(cfg, nets, x, st, sg)
    r_host = training.train_step(cfg, nets, x, [torch.from_numpy(t).cuda() for t in rt],
                                 [torch.from_numpy(g).cuda() for g in rg])
    torch.cuda.synchronize()
    assert float(r_dev["loss"]) == float(r_host["loss"])
    assert r_dev["grads"].keys() == r_host["grads"].keys()
    for p, g in r_dev["grads"].items():
        assert torch.equal(g, r_host["grads"][p])
