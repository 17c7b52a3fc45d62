"""GPU: the classification pre-training stage (scripts/train_cls.sh -> train_cls.py: T=9, max_iter=1, spatial mode, context
on, class-only heads): the class-only loss kernel against the classification part of the full loss kernel and the oracle,
the class-only head backward with context, train_step over class-only heads against the oracle's autograd, Adam with
dynamic loss scaling on it, and the transfer of its checkpoint into the full heads of the second stage (train.py:153-166).
References: tests/golden/cls_grads.npz (the reference's autograd) and the oracle's torch-CPU autograd, pinned to it by
tests/test_oracle_cls.py.  Tolerances are those of tests/test_gpu_train.py and tests/test_gpu_train_context.py for the same
fp32 losses and fp16 activation paths."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import model as om
from step_b200 import optim, synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _train_case import SHIPPED, compare_grads, rel_l2, trainable  # noqa: E402
from step_b200.synth import device_head, device_nets  # noqa: E402
from test_oracle_cls import CLS_CFG, cls_objective, golden_case, transfer_pretrained  # noqa: E402

pytestmark = pytest.mark.gpu

GROUPS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cls_param_groups.npz")


def loss_inputs(name):
    """(logits [N,60], tubes [N,T',5], targets [N,3,66], T): the train_cls.py-shaped case, where every row carries the
    classification flag and the last clip has negatives only, and two cases with mixed flags."""
    gen = torch.Generator().manual_seed(13)
    if name == "cls_case":
        cfg = synth.make_cfg(**CLS_CFG)
        tubes, targets = synth.make_cls_case(cfg, 3, 20, 400, 400)
        T_ = cfg.T
    else:
        T_, _, _, tubes, targets = synth.make_loss_case(name, 60)
    return torch.randn(targets.shape[0], 60, generator=gen) * 3.0, tubes, targets, T_


@pytest.mark.parametrize("name", ["cls_case", "c1", "c3"])
def test_cls_loss_equals_head_losses_and_matches_oracle(name):
    """step_cls_loss_f32 and step_head_losses_f32 on the same logits and targets: loss_cls and dlogits equal bit for bit, and
    both match the oracle's BCE and its autograd (expf / log1pf are not bit-exact: 1e-4 relative)."""
    from step_b200 import training
    logits, tubes, targets, T_ = loss_inputs(name)
    n, Tl = tubes.shape[0], tubes.shape[1]
    gen = torch.Generator().manual_seed(3)
    loc = torch.randn(n, Tl, 4, generator=gen) * 0.3
    lc, g = training.cls_loss(logits.cuda(), targets.cuda(), want_grads=True)
    lc_full, _, _, g_full = training.head_losses(logits.cuda(), loc.cuda(), loc[:, :T_].cuda(), loc[:, Tl - T_:].cuda(), tubes.cuda(),
                                                 targets.cuda(), T_, want_grads=True)
    torch.cuda.synchronize()
    assert lc.shape == (n * 60,) and g.shape == (n, 60)
    assert torch.equal(lc, lc_full) and torch.equal(g, g_full["logits"])
    x = logits.clone().requires_grad_(True)
    ref, _, _ = om.two_branch_losses(x, torch.zeros(1), torch.zeros(1), torch.zeros(1), tubes, targets, T_, cls_only=True)
    ref.mean().backward()
    assert np.allclose(lc.cpu().numpy(), ref.detach().numpy(), rtol=1e-4, atol=1e-6)
    assert np.allclose(g.cpu().numpy(), x.grad.numpy(), rtol=1e-4, atol=1e-8)
    again = training.cls_loss(logits.cuda(), targets.cuda(), want_grads=True)
    assert torch.equal(again[0], lc) and torch.equal(again[1], g)


def test_cls_loss_without_classification_flag_and_bad_arguments():
    from step_b200 import _lib as L
    from step_b200 import training
    logits, _, targets, _ = loss_inputs("cls_case")
    targets = targets.clone()
    targets[:, :, 4] = 0.0
    lc, g = training.cls_loss(logits.cuda(), targets.cuda(), want_grads=True)
    torch.cuda.synchronize()
    assert lc.shape == (1,) and float(lc) == 0.0                        # the reference's [1] zero (two_branch.py:290-297)
    assert g.shape == logits.shape and float(g.abs().max()) == 0.0
    assert float(training.cls_loss(logits.cuda(), targets.cuda()).abs().max()) == 0.0
    x, t = logits.cuda(), targets.cuda()
    out = torch.empty(x.numel(), device="cuda")
    flags = torch.empty(1, dtype=torch.int32, device="cuda")
    for args in ((x, t, 0, 60, out, flags), (x, t, x.shape[0], 0, out, flags), (None, t, x.shape[0], 60, out, flags),
                 (x, None, x.shape[0], 60, out, flags), (x, t, x.shape[0], 60, None, flags), (x, t, x.shape[0], 60, out, None)):
        with pytest.raises(RuntimeError, match="cls_loss"):
            L.check(L.lib().step_cls_loss_f32(L.ptr(args[0]), L.ptr(args[1]), args[2], args[3], L.ptr(args[4]), L.ptr(args[5]), None,
                                              L.stream()))
    with pytest.raises(RuntimeError, match="cls_loss"):
        training.cls_loss(x, t[:, :, :-1])


@pytest.fixture(scope="module")
def cls_oracle():
    """The golden case through the oracle on the CPU, with the per-tube context copy as a leaf: the gradients of the pooled
    features, of the context input and of the head's parameters."""
    cfg, cf, flat_tubes, flat_targets = golden_case()
    ctx = om.context_net(cf, synth.context_net_state_dict(), global_mean=True).detach()
    clip = [int(flat_tubes[p, 0, 0].item() / cfg.T) for p in range(flat_tubes.shape[0])]
    tctx = torch.stack([ctx[c, :, :cfg.T] for c in clip]).requires_grad_(True)
    _, _, pooled, _, _ = cls_objective(cf, synth.context_net_state_dict(), synth.cls_head_state_dict(100, cfg), cfg, flat_tubes,
                                       flat_targets, pooled_leaf=True)
    pooled = pooled.detach().requires_grad_(True)
    sd = trainable(synth.cls_head_state_dict(100, cfg))
    prob, loc, first, last, logits = om.two_branch(pooled, sd, cfg.T, tctx, cfg.fc_dim, cfg.pool_size, cls_only=True, return_logits=True)
    lc, _, _ = om.two_branch_losses(logits, loc, first, last, flat_tubes, flat_targets, cfg.T, cls_only=True)
    lc.mean().backward()
    return dict(cfg=cfg, ctx=ctx, clip=clip, tctx=tctx, pooled=pooled, sd=sd, prob=prob.detach(), lc=lc.detach(),
                tubes=flat_tubes, targets=flat_targets)


def test_cls_forward_with_targets_returns_the_reference_outputs(golden, cls_oracle):
    """TwoBranchNet(cls_only=True).forward(pooled, context, tubes, targets) -- train_cls.py:310 -- on the fp32 path: the seven
    outputs of the reference (probabilities, three [1] zeros, loss_cls, two [1] zero regression losses)."""
    g, o = golden("cls_grads"), cls_oracle
    cfg = synth.make_cfg(fp16=False, **CLS_CFG, image_size=(400, 400))
    net = device_head(cfg, synth.cls_head_state_dict(100, cfg), cls_only=True)
    with torch.no_grad():
        outs = net(o["pooled"].detach().cuda(), o["tctx"].detach().cuda(), tubes=o["tubes"].cuda(), targets=o["targets"].cuda())
    torch.cuda.synchronize()
    assert len(outs) == 7
    prob, loc, first, last, lc, ll, ln = [t.cpu() for t in outs]
    assert np.allclose(prob.numpy(), o["prob"].numpy(), rtol=1e-4, atol=2e-5)
    assert abs(float(prob.double().norm()) - float(g["prob_norm"][0])) <= 1e-4 * float(g["prob_norm"][0])
    assert np.array_equal(np.concatenate([t.reshape(-1).numpy() for t in (loc, first, last, ll, ln)]), g["other_outputs"])
    assert lc.shape == o["lc"].shape and np.allclose(lc.numpy(), o["lc"].numpy(), rtol=1e-4, atol=2e-6)
    assert abs(float(lc.mean()) - float(g["loss"][0])) <= 1e-4 * float(g["loss"][0])
    zero = o["targets"].clone()
    zero[:, :, 4] = 0.0
    with torch.no_grad():
        lz = net(o["pooled"].detach().cuda(), o["tctx"].detach().cuda(), tubes=o["tubes"].cuda(), targets=zero.cuda())[4]
    assert np.array_equal(lz.cpu().numpy(), g["zero_loss_cls"])


@pytest.mark.parametrize("form", ["per_tube", "row_map"])
def test_cls_head_backward_matches_reference_and_oracle(golden, cls_oracle, form):
    """head_forward_backward on a class-only head with the context in both forms: the reference's per-tube [R,1024,T,1,1]
    copy, and (per-clip mean, row map) as train_step feeds it.  16 tensors (Mixed_5b / 5c, downsample, global_cls), the
    gradient of the pooled features and of the context input; zero regression losses."""
    from step_b200 import training
    g, o = golden("cls_grads"), cls_oracle
    dcfg = synth.make_cfg(fp16=True, **CLS_CFG, image_size=(400, 400))
    net = device_head(dcfg, synth.cls_head_state_dict(100, dcfg), cls_only=True)
    if form == "per_tube":
        context = o["tctx"].detach().cuda()
    else:
        context = (o["ctx"].view(2, 1024, 9).mean(2).cuda(), torch.tensor(o["clip"], dtype=torch.int32, device="cuda"))
    r = training.head_forward_backward(net, o["pooled"].detach().cuda(), o["tubes"].cuda(), o["targets"].cuda(), context_feat=context)
    torch.cuda.synchronize()
    assert abs(float(r["loss"]) - float(g["loss"][0])) <= 5e-3 * float(g["loss"][0])
    lc, ll, ln = r["losses"]
    assert lc.shape == o["lc"].shape and ll.shape == (1,) and ln.shape == (1,) and float(ll) == 0.0 and float(ln) == 0.0
    names = {p: k for k, p in net.named_parameters()}
    got = {names[p]: v for p, v in r["grads"].items()}
    assert len(got) == 16
    for k, v in got.items():
        ref_n = float(g["gn:h0:" + k][0])
        assert tuple(v.shape) == tuple(o["sd"][k].shape), k
        assert abs(float(v.double().norm()) - ref_n) <= 3e-2 * ref_n, (k, float(v.double().norm()), ref_n)
        assert rel_l2(v, o["sd"][k].grad) <= 8e-2, (k, rel_l2(v, o["sd"][k].grad))
    assert abs(float(r["feat_grad"].double().norm()) - float(g["pooled_grad_norm"][0])) <= 3e-2 * float(g["pooled_grad_norm"][0])
    assert rel_l2(r["feat_grad"], o["pooled"].grad) <= 8e-2
    if form == "per_tube":
        assert tuple(r["ctx_grad"].shape) == tuple(o["tctx"].shape)
        assert rel_l2(r["ctx_grad"], o["tctx"].grad) <= 8e-2
    else:   # the gradient of the mean row each tube reads: the sum over the frames of its per-frame copy
        assert rel_l2(r["ctx_grad"], o["tctx"].grad.sum(2).view(-1, 1024)) <= 8e-2


def cls_case(seed=3, B=2, N=6):
    cfg = synth.make_cfg(fp16=True, **CLS_CFG, image_size=(64, 64))
    tubes, targets = synth.make_cls_case(cfg, B, N, 64, 64, seed=seed)
    return cfg, synth.make_clips(B, 36, 64, 64, seed=11), tubes, targets


def test_train_step_cls_config_matches_oracle_autograd():
    """train_step over a class-only head at reduced resolution (2 clips of 36x64x64, T'=9, one step pooling frames [0, 9),
    one clip with negatives only) against the oracle's autograd with torchvision's roi_align: 45 trunk, 12 ContextNet and 16
    head tensors."""
    from step_b200 import training
    cfg, x, tubes, targets = cls_case()
    nets = device_nets(cfg, [synth.cls_head_state_dict(100, cfg)], context=True, cls_only=True)
    sd_b = {k: v.clone().requires_grad_(k.endswith("conv3d.weight")) for k, v in synth.base_net_state_dict().items()}
    sd_ctx = trainable(synth.context_net_state_dict())
    sd_h = trainable(synth.cls_head_state_dict(100, cfg))
    cf = om.base_net(x.clone(), sd_b)
    total, _, _, _, _ = cls_objective(cf, sd_ctx, sd_h, cfg, tubes, targets)
    total.backward()
    total = float(total.detach())
    r = training.train_step(cfg, nets, x.cuda(), [tubes.cuda()], [targets.cuda()])
    torch.cuda.synchronize()
    assert abs(float(r["loss"]) - total) <= 5e-3 * abs(total)
    assert len(r["losses"]) == 1 and len(r["grads"]) == 45 + 12 + 16
    assert compare_grads(r, nets["det_net0"], sd_h, 3e-2, 1e-1) == 16
    assert compare_grads(r, nets["context_net"], sd_ctx, 3e-2, 1e-1) == 12
    assert compare_grads(r, nets["base_net"], sd_b, 1.5e-1, 2.5e-1) == 45


def test_train_step_cls_config_keeps_the_frame_and_context_checks():
    from step_b200 import training
    cfg, x, tubes, targets = cls_case()
    nets = device_nets(cfg, [synth.cls_head_state_dict(100, cfg)], context=True, cls_only=True)
    with pytest.raises(RuntimeError, match="step 1 pools frames"):
        training.train_step(cfg, nets, x.cuda(), [tubes[:, :3].contiguous().cuda()], [targets.cuda()])
    del nets["context_net"]
    with pytest.raises(RuntimeError, match="context_net"):
        training.train_step(cfg, nets, x.cuda(), [tubes.cuda()], [targets.cuda()])


def cls_groups(nets, lr_scale=1.0):
    """The 73 parameter groups of the reference's get_params for train_cls.py, from the fixture."""
    g = np.load(GROUPS)
    named = {k: dict(n.named_parameters()) for k, n in nets.items()}
    return [{"params": [named[str(m)][str(n)]], "lr": float(lr) * lr_scale, "weight_decay": float(wd)}
            for m, n, lr, wd in zip(g["module"], g["name"], g["lr"], g["weight_decay"])]


# One common factor on the rates of scripts/train_cls.sh, as in tests/test_gpu_optim.py::test_adam_steps_descend_shipped_config:
# Adam's first steps move every element by about its rate, and on these synthetic nets and one batch the shipped rates overshoot.
DESCENT_LR_SCALE = 1e-3


def test_adam_steps_descend_then_checkpoint_trains_the_shipped_heads():
    """Five Adam steps with a LossScaler over the class-only nets on one fixed mini-batch: the objective never rises and ends
    lower.  Their checkpoint then goes into three full heads as train.py:153-166 loads it (everything but `global_cls`),
    and a shipped-configuration train_step runs on them."""
    from step_b200 import training
    cfg, x, tubes, targets = cls_case(seed=7)
    nets = device_nets(cfg, [synth.cls_head_state_dict(100, cfg)], context=True, cls_only=True)
    opt = optim.Adam(cls_groups(nets, DESCENT_LR_SCALE))
    scaler = optim.LossScaler()
    batch = (x.cuda(), [tubes.cuda()], [targets.cuda()])
    losses = []
    for _ in range(5):
        r = training.train_step(cfg, nets, *batch, optimizer=opt, scaler=scaler)
        assert not r["skipped"] and r["loss_scale"] == 2.0 ** 16
        losses.append(float(r["loss"]))
    losses.append(float(training.train_step(cfg, nets, *batch, lr=None)["loss"]))
    assert all(b <= a for a, b in zip(losses, losses[1:])) and losses[-1] < losses[0], losses
    ckpt = {k: {n: v.detach().clone() for n, v in nets[k].state_dict().items()} for k in ("base_net", "context_net", "det_net0")}
    scfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(64, 64))
    full = device_nets(scfg, [synth.head_state_dict(100 + i, scfg) for i in range(3)], context=True)
    transfer_pretrained(ckpt, full, 3)
    moved = [k for k in ckpt["det_net0"] if "global_cls" not in k]
    for i in range(3):
        sd = full["det_net%d" % i].state_dict()
        assert all(torch.equal(sd[k], ckpt["det_net0"][k]) for k in moved)
    assert all(torch.equal(v, ckpt["base_net"][k]) for k, v in full["base_net"].state_dict().items())
    step_tubes, step_targets = synth.make_train_case(scfg, 2, 3, 64, 64, seed=3)
    r = training.train_step(scfg, full, x.cuda(), [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets], lr=None)
    torch.cuda.synchronize()
    assert len(r["grads"]) == 45 + 12 + 3 * 34 and np.isfinite(float(r["loss"]))
    assert all(bool(torch.isfinite(gr).all()) for gr in r["grads"].values())
