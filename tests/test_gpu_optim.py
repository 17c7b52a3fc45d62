"""GPU: step_b200.optim -- the multi-tensor Adam and SGD of csrc/optim.cu against torch.optim's single-tensor
implementations, the skip of a step with non-finite gradients, checkpoints exchanged with torch.optim.Adam, the weight caches
of the modules after an update, and train_step with an optimizer and dynamic loss scaling in the shipped configuration."""
import copy
import math
import os
import sys

import pytest
import torch

from step_b200 import optim, synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _train_case import SHIPPED  # noqa: E402
from step_b200.synth import device_head, device_nets  # noqa: E402
from test_optim_cpu import fixture_groups  # noqa: E402

pytestmark = pytest.mark.gpu

# 2^20 + 5 ends in a ragged tail of its last chunk; the 1000-element view at a 4-byte offset takes the scalar path
SIZES = (1, 3, 60, 4097, 2 ** 20 + 5)
GROUPS = (dict(lr=1e-3, weight_decay=0.0), dict(lr=3e-4, weight_decay=1e-2), dict(lr=2e-3, weight_decay=1e-7))


def make_case(seed=0):
    """Initial values [sizes..., view] on the CPU; the view's storage starts one element earlier."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for n in SIZES] + [torch.randn(1001, generator=g)]


def to_device(init):
    ps = [t.clone().cuda() for t in init[:-1]]
    view = init[-1].clone().cuda()[1:]
    assert view.data_ptr() % 16 == 4
    # the view is placed before the largest tensor, so the last element of the last tensor is in a vector-path tail
    return ps[:4] + [view, ps[4]]


def grouped(ps, **extra):
    return [dict(params=ps[0:2], **GROUPS[0], **extra), dict(params=ps[2:4], **GROUPS[1], **extra),
            dict(params=ps[4:], **GROUPS[2], **extra)]


def grads_of(ps, step, seed=7):
    g = torch.Generator().manual_seed(seed * 1000 + step)
    return [torch.randn(p.shape, generator=g).cuda() * (1.0 + 10.0 * (i % 2)) for i, p in enumerate(ps)]


def lr_factor(step):
    return 1.0 + 0.5 * math.sin(0.7 * step)


def run(opt_fn, init, steps=30, bad=None):
    """`steps` updates with seeded gradients and a different lr factor on every step; bad = (step, value) puts value into the
    last element of the last tensor's gradient on that step."""
    ps = to_device(init)
    opt = opt_fn(ps)
    base = [g["lr"] for g in opt.param_groups]
    for s in range(steps):
        for g, b in zip(opt.param_groups, base):
            g["lr"] = b * lr_factor(s)
        gs = grads_of(ps, s)
        if bad is not None and bad[0] == s:
            gs[-1][-1] = bad[1]
        for p, gr in zip(ps, gs):
            p.grad = gr
        opt.step()
    torch.cuda.synchronize()
    return ps, opt


def ours_adam(ps):
    return optim.Adam(grouped(ps), betas=(0.9, 0.999), eps=1e-8)


def torch_adam(ps):
    return torch.optim.Adam(grouped(ps), betas=(0.9, 0.999), eps=1e-8, foreach=False)


def ours_sgd(ps):
    return optim.SGD(grouped(ps, momentum=0.9))


def torch_sgd(ps):
    return torch.optim.SGD(grouped(ps, momentum=0.9), foreach=False)


def assert_close_params(got, ref, init, tol=1e-5):
    for g, r, p0 in zip(got, ref, to_device(init)):
        moved = float((r - p0).abs().max())
        assert moved > 0
        assert float((g - r).abs().max()) <= tol * moved, (g.numel(), float((g - r).abs().max()), moved)


def assert_close_state(o_got, p_got, o_ref, p_ref, keys, tol=1e-5):
    for pg, pr in zip(p_got, p_ref):
        for k in keys:
            a, b = o_got.state[pg][k], o_ref.state[pr][k]
            assert float((a - b).abs().max()) <= tol * float(b.abs().max()), (pg.numel(), k)


def max_differences(ours_fn, torch_fn, keys):
    """(max |p - p_torch|, max state difference) over every tensor: 0.0 / 0.0 when bit-identical."""
    init = make_case()
    pa, oa = run(ours_fn, init)
    pb, ob = run(torch_fn, init)
    dp = max(float((a - b).abs().max()) for a, b in zip(pa, pb))
    ds = max(float((oa.state[a][k] - ob.state[b][k]).abs().max()) for a, b in zip(pa, pb) for k in keys)
    return dp, ds


@pytest.mark.parametrize("ours_fn,torch_fn,keys", [(ours_adam, torch_adam, ("exp_avg", "exp_avg_sq")),
                                                   (ours_sgd, torch_sgd, ("momentum_buffer",))], ids=["adam", "sgd"])
def test_matches_torch_single_tensor_and_repeats(ours_fn, torch_fn, keys):
    init = make_case()
    pa, oa = run(ours_fn, init)
    pb, ob = run(torch_fn, init)
    assert_close_params(pa, pb, init)
    assert_close_state(oa, pa, ob, pb, keys)
    assert not oa.found_inf
    if "exp_avg" in keys:
        assert all(float(oa.state[p]["step"]) == 30.0 and oa.state[p]["step"].device.type == "cpu" for p in pa)
    pc, oc = run(ours_fn, init)
    for a, c in zip(pa, pc):
        assert torch.equal(a, c)
        for k in keys:
            assert torch.equal(oa.state[a][k], oc.state[c][k])


@pytest.mark.parametrize("value", [float("inf"), float("-inf"), float("nan")])
@pytest.mark.parametrize("ours_fn,torch_fn,keys", [(ours_adam, torch_adam, ("exp_avg", "exp_avg_sq")),
                                                   (ours_sgd, torch_sgd, ("momentum_buffer",))], ids=["adam", "sgd"])
def test_nonfinite_gradient_skips_the_step(ours_fn, torch_fn, keys, value):
    init = make_case(1)
    ps, opt = run(ours_fn, init, steps=4)
    before = [p.clone() for p in ps]
    state = {i: {k: v.clone() for k, v in opt.state[p].items()} for i, p in enumerate(ps)}
    gs = grads_of(ps, 4)
    gs[-1][-1] = value
    for p, g in zip(ps, gs):
        p.grad = g
    versions = [p._version for p in ps]
    opt.step()
    torch.cuda.synchronize()
    assert opt.found_inf
    for i, p in enumerate(ps):
        assert torch.equal(p, before[i]) and p._version == versions[i]
        for k, v in state[i].items():
            assert torch.equal(opt.state[p][k], v), k
    # the next clean step (step 5 of the seeded sequence) equals torch's run that never saw the bad gradients
    for g, b in zip(opt.param_groups, GROUPS):
        g["lr"] = b["lr"] * lr_factor(4)
    for p, g in zip(ps, grads_of(ps, 5)):
        p.grad = g
    opt.step()
    torch.cuda.synchronize()
    assert not opt.found_inf
    ref_ps = to_device(init)
    ref = torch_fn(ref_ps)
    for lr_step, grad_step in ((0, 0), (1, 1), (2, 2), (3, 3), (4, 5)):
        for g, b in zip(ref.param_groups, GROUPS):
            g["lr"] = b["lr"] * lr_factor(lr_step)
        for p, g in zip(ref_ps, grads_of(ref_ps, grad_step)):
            p.grad = g
        ref.step()
    assert_close_params(ps, ref_ps, init)
    assert_close_state(opt, ps, ref, ref_ps, keys)


def test_empty_step_and_first_step_overflow_keep_state_empty():
    ps = to_device(make_case())
    opt = optim.Adam(grouped(ps))
    opt.step()                                      # no gradients: nothing to do
    assert not opt.found_inf and len(opt.state) == 0
    for p in ps:
        p.grad = torch.full_like(p, float("nan"))
    opt.step()
    assert opt.found_inf and len(opt.state) == 0


def test_state_dict_round_trips_with_torch_adam():
    init = make_case(2)

    def continue_run(opt, ps, first):
        for s in range(first, first + 5):
            for p, g in zip(ps, grads_of(ps, s)):
                p.grad = g
            opt.step()
        torch.cuda.synchronize()

    def single_tensor(opt):
        # torch's single-tensor path, also after loading groups saved with foreach=None
        if isinstance(opt, torch.optim.Adam):
            for g in opt.param_groups:
                g["foreach"] = False
        return opt

    for first_cls, second_cls in ((optim.Adam, torch.optim.Adam), (torch.optim.Adam, optim.Adam)):
        ps = to_device(init)
        a = single_tensor(first_cls(grouped(ps)))
        continue_run(a, ps, 0)
        sd = copy.deepcopy(a.state_dict())           # load_state_dict keeps same-device state tensors: do not share them
        qs = [p.clone() for p in ps]
        b = second_cls(grouped(qs))
        b.load_state_dict(sd)
        single_tensor(b)
        assert all(b.state[q]["step"].device.type == "cpu" and float(b.state[q]["step"]) == 5.0 for q in qs)
        continue_run(a, ps, 5)
        continue_run(b, qs, 5)
        assert_close_params(qs, ps, init)
        assert_close_state(b, qs, a, ps, ("exp_avg", "exp_avg_sq"))


def test_update_invalidates_the_modules_weight_caches():
    """After opt.step() the next forward of the updated modules equals, bit for bit, that of fresh modules loaded with the
    updated weights (the packed fp16 / permuted caches are keyed on the parameters' _version)."""
    import step_b200
    cfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(64, 64))
    nets = device_nets(cfg, [synth.head_state_dict(100 + i, cfg) for i in range(3)], context=True)
    x = synth.make_clips(1, 36, 64, 64, seed=3).cuda()
    g = torch.Generator().manual_seed(4)
    feat = (torch.randn(4, 3, 832, 7, 7, generator=g) * 0.5).cuda()
    ctx = torch.randn(4, 1024, 3, 1, 1, generator=g).cuda()
    head, base = nets["det_net0"], nets["base_net"]
    head(feat, ctx)                                  # fill the caches with the old weights
    base(x)
    opt = optim.Adam(fixture_groups(nets))
    for grp in opt.param_groups:
        p = grp["params"][0]
        p.grad = torch.randn(p.shape, generator=g).cuda()
    opt.step()
    fresh_head = device_head(cfg, head.state_dict())
    fresh_base = step_b200.BaseNet(cfg)
    fresh_base.load_state_dict(base.state_dict())
    fresh_base = fresh_base.cuda().eval()
    for a, b in zip(head(feat, ctx)[:4], fresh_head(feat, ctx)[:4]):
        assert torch.equal(a, b)
    assert torch.equal(base(x), fresh_base(x))


def shipped_case(seed=3):
    cfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(64, 64))
    step_tubes, step_targets = synth.make_train_case(cfg, 2, 3, 64, 64, seed=seed)
    x = synth.make_clips(2, 36, 64, 64, seed=11).cuda()
    return cfg, (x, [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets])


def trainable(nets):
    return {(k, n): p for k, net in nets.items() for n, p in net.named_parameters() if p.requires_grad}


def test_train_step_with_adam_matches_torch_adam_on_the_returned_gradients():
    from step_b200 import training
    cfg, batch = shipped_case()
    heads_sd = [synth.head_state_dict(100 + i, cfg) for i in range(3)]
    nets_a, nets_b = device_nets(cfg, heads_sd, context=True), device_nets(cfg, heads_sd, context=True)
    p0 = {k: p.detach().clone() for k, p in trainable(nets_a).items()}
    opt = optim.Adam(fixture_groups(nets_a))
    ra = training.train_step(cfg, nets_a, *batch, optimizer=opt)
    rb = training.train_step(cfg, nets_b, *batch, lr=None)
    assert ra["skipped"] is False and ra["loss_scale"] == 1024.0 and rb["skipped"] is False
    assert float(ra["loss"]) == float(rb["loss"])
    ref = torch.optim.Adam(fixture_groups(nets_b), foreach=False)
    for p, gr in rb["grads"].items():
        p.grad = gr
    ref.step()
    torch.cuda.synchronize()
    pa, pb = trainable(nets_a), trainable(nets_b)
    assert len(pa) == 159
    for k in pa:
        moved = float((pb[k] - p0[k]).detach().abs().max())
        assert moved > 0, k
        assert float((pa[k] - pb[k]).detach().abs().max()) <= 1e-5 * moved, k


def test_overflowing_loss_scale_skips_then_backs_off_to_an_applied_step():
    from step_b200 import training
    cfg, batch = shipped_case()
    nets = device_nets(cfg, [synth.head_state_dict(100 + i, cfg) for i in range(3)], context=True)
    opt = optim.Adam(fixture_groups(nets))
    scaler = optim.LossScaler(init_scale=2.0 ** 40)
    before = {k: p.detach().clone() for k, p in trainable(nets).items()}
    r = training.train_step(cfg, nets, *batch, optimizer=opt, scaler=scaler)
    torch.cuda.synchronize()
    assert r["skipped"] is True and r["loss_scale"] == 2.0 ** 40 and scaler.scale == 2.0 ** 39
    assert any(not bool(torch.isfinite(g).all()) for g in r["grads"].values())
    after = trainable(nets)
    assert len(after) == 159 and all(torch.equal(after[k], v) for k, v in before.items())
    assert len(opt.state) == 0
    for call in range(1, 40):
        r = training.train_step(cfg, nets, *batch, optimizer=opt, scaler=scaler)
        if not r["skipped"]:
            break
    assert not r["skipped"], "no applied step down to loss scale %g" % scaler.scale
    assert all(bool(torch.isfinite(g).all()) for g in r["grads"].values())
    assert r["loss_scale"] == 2.0 ** (40 - call) and scaler.scale == r["loss_scale"]
    assert all(float(opt.state[p]["step"]) == 1.0 for p in after.values())


# One common factor on the shipped rates.  Adam's first steps move every element by about its rate, whatever its gradient's
# size; on these synthetic nets and this one batch the shipped rates (and 3e-3 of them) overshoot and the objective rises.
DESCENT_LR_SCALE = 1e-3


def test_adam_steps_descend_shipped_config():
    """Five Adam steps with the shipped per-group rates (times DESCENT_LR_SCALE) on one fixed batch: the objective never
    rises and ends lower.  No layer-wise normalisation: Adam's per-element scaling handles the regressor weights of std
    5e-5 next to O(0.05) conv weights."""
    from step_b200 import training
    cfg, batch = shipped_case(seed=7)
    nets = device_nets(cfg, [synth.head_state_dict(100 + i, cfg) for i in range(3)], context=True)
    opt = optim.Adam(fixture_groups(nets, DESCENT_LR_SCALE))
    losses = []
    for _ in range(5):
        r = training.train_step(cfg, nets, *batch, optimizer=opt)
        assert not r["skipped"]
        losses.append(float(r["loss"]))
    losses.append(float(training.train_step(cfg, nets, *batch, lr=None)["loss"]))
    assert all(b <= a for a, b in zip(losses, losses[1:])) and losses[-1] < losses[0], losses
