"""CPU: step_b200.optim's interface -- the reference's `get_params` routes the step_b200 modules' parameters into the
groups it builds for its own modules (tests/golden/shipped_param_groups.npz), the reference's WarmupCosineLR drives the
groups of `Adam` as it drives torch.optim.Adam's, unsupported options are refused and there is no CPU fallback."""
import os
import warnings
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from step_b200 import optim, synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "shipped_param_groups.npz")
# scripts/train_step.sh (rgb input, context on, 3 refinement steps) and config.py's default weight_decay
SHIPPED_ARGS = dict(base_lr=7.5e-5, det_lr0=1.5e-4, det_lr=7.5e-4, weight_decay=1e-7, input_type="rgb", no_context=False,
                    max_iter=3)
SHIPPED_CFG = dict(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False)


def shipped_modules(cfg=None):
    """The step_b200 modules of the shipped configuration (uninitialised weights; CPU)."""
    import step_b200
    cfg = cfg or synth.make_cfg(fp16=True, **SHIPPED_CFG, image_size=(64, 64))
    nets = {"base_net": step_b200.BaseNet(cfg), "context_net": step_b200.ContextNet(cfg)}
    for i in range(3):
        nets["det_net%d" % i] = step_b200.TwoBranchNet(cfg)
    return nets


def fixture_groups(nets, lr_scale=1.0):
    """The 159 parameter groups of the reference's get_params for the shipped configuration, built from the fixture:
    [{'params': [p], 'lr': lr * lr_scale, 'weight_decay': wd}] in the reference's order."""
    g = np.load(GOLDEN)
    named = {k: dict(n.named_parameters()) for k, n in nets.items()}
    return [{"params": [named[str(m)][str(n)]], "lr": float(lr) * lr_scale, "weight_decay": float(wd)}
            for m, n, lr, wd in zip(g["module"], g["name"], g["lr"], g["weight_decay"])]


def reference_solver():
    from oracle import refload
    if not refload.available():
        pytest.skip("reference tree not present")
    refload.load()
    from utils import solver
    return solver


def test_fixture_covers_every_trainable_tensor_of_the_shipped_nets():
    nets = shipped_modules()
    groups = fixture_groups(nets)
    trainable = [p for n in nets.values() for p in n.parameters() if p.requires_grad]
    assert len(groups) == len(trainable) == 159
    assert {id(g["params"][0]) for g in groups} == {id(p) for p in trainable}
    assert sum(g["params"][0].numel() for g in groups) == 44422936
    assert int(np.load(GOLDEN)["numel"].sum()) == 44422936


def test_reference_get_params_groups_step_b200_modules_as_its_own():
    solver = reference_solver()
    nets = shipped_modules()
    owner = {id(p): (k, n) for k, net in nets.items() for n, p in net.named_parameters()}
    got = solver.get_params(nets, SimpleNamespace(**SHIPPED_ARGS))
    g = np.load(GOLDEN)
    assert len(got) == len(g["name"]) == 159
    for grp, m, n, lr, wd in zip(got, g["module"], g["name"], g["lr"], g["weight_decay"]):
        assert len(grp["params"]) == 1
        assert owner[id(grp["params"][0])] == (str(m), str(n))
        assert grp["lr"] == lr and grp["weight_decay"] == wd, (str(m), str(n))


def test_reference_warmup_cosine_drives_adam_groups_like_torch():
    solver = reference_solver()
    ours = optim.Adam(fixture_groups(shipped_modules()), lr=SHIPPED_ARGS["det_lr"])
    ref = torch.optim.Adam(fixture_groups(shipped_modules()), lr=SHIPPED_ARGS["det_lr"])
    # train.py:88-89,131: milestones = [iterations of the run], min_ratio 0, cycle_decay 1, warmup_iters 1000
    s_ours = solver.WarmupCosineLR(ours, [1400], 0.0, 1.0, 1000)
    s_ref = solver.WarmupCosineLR(ref, [1400], 0.0, 1.0, 1000)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")             # scheduler.step() without optimizer.step(): no GPU here
        for it in range(1500):
            assert [g["lr"] for g in ours.param_groups] == [g["lr"] for g in ref.param_groups], it
            s_ours.step()
            s_ref.step()
    assert [g["lr"] for g in ours.param_groups] == [g["lr"] for g in ref.param_groups]
    assert ours.param_groups[-1]["lr"] == 0.0 and ref.param_groups[0]["initial_lr"] == SHIPPED_ARGS["base_lr"] / 8


@pytest.mark.parametrize("cls,kw", [
    (optim.Adam, dict(amsgrad=True)), (optim.Adam, dict(maximize=True)), (optim.Adam, dict(decoupled_weight_decay=True)),
    (optim.Adam, dict(differentiable=True)), (optim.Adam, dict(capturable=True)), (optim.Adam, dict(fused=True)),
    (optim.Adam, dict(foreach=True)), (optim.SGD, dict(nesterov=True, momentum=0.9)), (optim.SGD, dict(maximize=True)),
    (optim.SGD, dict(dampening=0.1)), (optim.SGD, dict(differentiable=True)), (optim.SGD, dict(fused=True)),
    (optim.SGD, dict(foreach=False))])
def test_unsupported_options_raise(cls, kw):
    with pytest.raises(ValueError):
        cls([torch.nn.Parameter(torch.zeros(3))], **kw)


def test_loaded_groups_with_unsupported_semantics_raise_at_step():
    p = torch.nn.Parameter(torch.zeros(3))
    ours = optim.Adam([p])
    ours.load_state_dict(torch.optim.Adam([p], amsgrad=True).state_dict())
    p.grad = torch.ones(3)
    with pytest.raises(ValueError, match="amsgrad"):
        ours.step()


def test_step_on_cpu_parameters_raises():
    for opt in (optim.Adam, optim.SGD):
        p = torch.nn.Parameter(torch.ones(4))
        o = opt([p], lr=0.1)
        p.grad = torch.ones(4)
        with pytest.raises(RuntimeError, match="CUDA"):
            o.step()
        assert torch.equal(p.detach(), torch.ones(4)) and len(o.state) == 0


def test_state_dict_has_torch_layout():
    p = torch.nn.Parameter(torch.zeros(3))
    ours, ref = optim.Adam([p], lr=0.01), torch.optim.Adam([p], lr=0.01)
    assert ours.state_dict()["param_groups"] == ref.state_dict()["param_groups"]
    ours, ref = optim.SGD([p], lr=0.01, momentum=0.9), torch.optim.SGD([p], lr=0.01, momentum=0.9)
    assert ours.state_dict()["param_groups"] == ref.state_dict()["param_groups"]


def test_loss_scaler_policy():
    s = optim.LossScaler()
    assert s.scale == 2.0 ** 16
    s.update(True)
    assert s.scale == 2.0 ** 15
    s = optim.LossScaler(init_scale=8.0, growth_interval=3)
    for _ in range(2):
        s.update(False)
    assert s.scale == 8.0
    s.update(False)
    assert s.scale == 16.0
    s.update(False); s.update(True); s.update(False); s.update(False)
    assert s.scale == 8.0                          # the overflow restarted the count of clean steps
    s.update(False)
    assert s.scale == 16.0


def test_train_step_rejects_lr_with_optimizer_and_scaler_without_optimizer():
    from step_b200 import training
    opt = optim.Adam([torch.nn.Parameter(torch.zeros(3))])
    with pytest.raises(ValueError, match="not both"):
        training.train_step(None, {}, None, [], [], lr=0.1, optimizer=opt)
    with pytest.raises(ValueError, match="needs an optimizer"):
        training.train_step(None, {}, None, [], [], scaler=optim.LossScaler())
