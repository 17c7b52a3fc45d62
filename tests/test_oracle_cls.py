"""CPU: the classification pre-training stage (scripts/train_cls.sh -> train_cls.py: T=9, max_iter=1, spatial mode, context
on, class-only heads).  The oracle's functional model (context_net(global_mean=True) + two_branch(cls_only=True) +
two_branch_losses(cls_only=True)) reproduces the reference's autograd (tests/golden/cls_grads.npz) -- once pinned here, it is
the element-level checker of the device's class-only training step.  The step_b200 class-only head has the reference's
state_dict, the reference's get_params groups its nets as its own (tests/golden/cls_param_groups.npz), and its checkpoint
transfers into full heads as train.py:153-166 loads it."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from torchvision.ops import roi_align as tv_roi_align

from oracle import model as om
from step_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _train_case import trainable  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cls_param_groups.npz")
# scripts/train_cls.sh (rgb input, context on, one refinement step) and config.py's default weight_decay
CLS_ARGS = dict(base_lr=5e-5, det_lr0=1e-4, det_lr=5e-4, weight_decay=1e-7, input_type="rgb", no_context=False, max_iter=1)
CLS_CFG = dict(T=9, max_iter=1, NUM_CHUNKS={1: 1}, no_context=False)


def cls_objective(cf, sd_ctx, sd, cfg, flat_tubes, flat_targets, pooled_leaf=False):
    """train_cls.py:266-311 through the oracle: conv_feat cf [B,T',832,H',W'] -> ContextNet, the ROIAlign of frames [0, T)
    (torchvision's roi_align, bit-identical to the reference's forward), the per-tube context copy of train_cls.py:304-308
    and loss_global_cls.mean() of the class-only head.  pooled_leaf: pool under no_grad and make the pooled features a leaf
    (the reference has no CPU ROIAlign backward).  Returns (loss, loss_cls, pooled, context_feat, prob)."""
    B, tl = cf.shape[0], cfg.T
    ctx = om.context_net(cf, sd_ctx, global_mean=True)                     # [B, 1024, T', 1, 1]
    fm = cf[:, :tl].reshape(B * tl, 832, cf.shape[3], cf.shape[4])
    with torch.set_grad_enabled(not pooled_leaf and torch.is_grad_enabled()):
        pooled = tv_roi_align(fm, flat_tubes.reshape(-1, 5), (7, 7), 1.0 / 16.0, 0, aligned=False).view(-1, tl, 832, 7, 7)
    if pooled_leaf:
        pooled = pooled.detach().requires_grad_(True)
    clip = [int(flat_tubes[p, 0, 0].item() / tl) for p in range(flat_tubes.shape[0])]
    tctx = torch.stack([ctx[c, :, :tl] for c in clip])                    # [R, 1024, T, 1, 1]
    prob, loc, first, last, logits = om.two_branch(pooled, sd, cfg.T, tctx, cfg.fc_dim, cfg.pool_size, cls_only=True,
                                                   return_logits=True)
    lc, _, _ = om.two_branch_losses(logits, loc, first, last, flat_tubes, flat_targets, cfg.T, cls_only=True)
    return lc.mean(), lc, pooled, ctx, prob


def golden_case(B=2, N=6):
    """The inputs of tests/golden/make_cls_golden.py."""
    cfg = synth.make_cfg(**CLS_CFG, image_size=(400, 400))
    flat_tubes, flat_targets = synth.make_cls_case(cfg, B, N, 400, 400)
    return cfg, synth.make_conv_feat(B, 9, 25, 25), flat_tubes, flat_targets


def test_make_cls_case_is_shaped_like_train_cls():
    cfg = synth.make_cfg(**CLS_CFG)
    tubes, targets = synth.make_cls_case(cfg, 3, 20, 400, 400)
    assert tuple(tubes.shape) == (60, 9, 5) and tuple(targets.shape) == (60, 3, 66)
    assert torch.equal(tubes[:, :, 0], (torch.arange(60).view(60, 1) // 20 * 9 + torch.arange(9).view(1, 9)).float())
    assert torch.equal(targets[:, 0], targets[:, 1]) and torch.equal(targets[:, 2], targets[:, 1])
    assert bool((targets[:, :, 4] == 1).all()) and bool((targets[:, :, 5] == 0).all())
    pos = targets[:, 1, 6:].sum(1) > 0
    assert pos.view(3, 20).sum(1).tolist() == [5, 5, 0]                 # at most 5 positives; the last clip negatives only
    assert bool((targets[~pos, 1, :4] == 0).all()) and bool((targets[pos, 1, 2:4] > targets[pos, 1, 0:2]).all())
    assert float(tubes[:, :, 1:].min()) >= 0 and float(tubes[:, :, 1:].max()) < 400


@pytest.mark.parametrize("zero_mask", [False, True])
def test_cls_gradients_oracle_matches_reference(golden, zero_mask):
    g = golden("cls_grads")
    cfg, cf, flat_tubes, flat_targets = golden_case()
    if zero_mask:
        flat_targets = flat_targets.clone()
        flat_targets[:, :, 4] = 0.0
    cf = cf.requires_grad_(True)
    sd_ctx = trainable(synth.context_net_state_dict())
    sd = trainable(synth.cls_head_state_dict(100, cfg))
    loss, lc, pooled, ctx, prob = cls_objective(cf, sd_ctx, sd, cfg, flat_tubes, flat_targets, pooled_leaf=True)
    if zero_mask:
        # no classification flag: the reference's [1] zero without a graph, and therefore no gradient
        assert lc.numel() == 1 and np.array_equal(lc.detach().numpy(), g["zero_loss_cls"])
        assert not loss.requires_grad and int(g["zero_loss_requires_grad"][0]) == 0
        assert np.allclose(prob.detach().double().norm().numpy(), g["zero_prob_norm"], rtol=1e-5)
        return
    loss.backward()
    assert lc.numel() == int(g["loss_cls_numel"][0])
    assert np.allclose(ctx.detach().double().norm().numpy(), g["context_feat_norm"], rtol=1e-5)
    assert np.allclose(prob.detach().double().norm().numpy(), g["prob_norm"], rtol=1e-5)
    assert np.allclose(loss.detach().numpy(), g["loss"], rtol=1e-5)
    assert np.allclose(pooled.detach().double().norm().numpy(), g["pooled_norm"], rtol=1e-6)
    assert np.allclose(pooled.grad.double().norm().numpy(), g["pooled_grad_norm"], rtol=1e-4)
    assert np.allclose(pooled.grad.reshape(-1)[:16].numpy(), g["pooled_grad_head"], rtol=1e-3, atol=1e-9)
    assert np.allclose(cf.grad.double().norm().numpy(), g["ctx_feat_grad_norm"], rtol=1e-4)
    assert np.allclose(cf.grad.reshape(-1)[:16].numpy(), g["ctx_feat_grad_head"], rtol=1e-3, atol=1e-10)
    checked = 0
    for key in g.files:
        if not key.startswith("gn:"):
            continue
        tag, k = key[3:].split(":", 1)
        p = (sd_ctx if tag == "ctx" else sd)[k]
        assert p.grad is not None, key
        assert np.allclose(p.grad.double().norm().numpy(), g[key], rtol=1e-4, atol=1e-12), key
        assert np.allclose(p.grad.reshape(-1)[:8].numpy(), g["gh:" + key[3:]], rtol=1e-3, atol=1e-9), key
        checked += 1
    assert checked == 12 + 16      # ContextNet's 12 Unit3D convolutions; Mixed_5b/5c, downsample and global_cls of the head


def cls_modules():
    """The step_b200 modules of train_cls.py (uninitialised weights; CPU)."""
    import step_b200
    cfg = synth.make_cfg(fp16=True, **CLS_CFG, image_size=(400, 400))
    return {"base_net": step_b200.BaseNet(cfg), "context_net": step_b200.ContextNet(cfg),
            "det_net0": step_b200.TwoBranchNet(cfg, cls_only=True)}


def test_cls_head_state_dict_matches_reference_keys_and_shapes():
    g = np.load(GOLDEN)
    sd = cls_modules()["det_net0"].state_dict()
    assert list(sd.keys()) == [str(k) for k in g["sd_key"]]
    for (k, v), row in zip(sd.items(), g["sd_shape"]):
        assert tuple(v.shape) == tuple(int(d) for d in row[1:1 + row[0]]), k
    assert set(synth.cls_head_state_dict(100, synth.make_cfg(**CLS_CFG))) == set(sd)


def test_fixture_covers_every_trainable_tensor_of_the_cls_nets():
    g = np.load(GOLDEN)
    nets = cls_modules()
    named = {k: dict(n.named_parameters()) for k, n in nets.items()}
    got = [named[str(m)][str(n)] for m, n in zip(g["module"], g["name"])]
    trainable_ = [p for n in nets.values() for p in n.parameters() if p.requires_grad]
    assert len(got) == len(trainable_) == 45 + 12 + 16
    assert {id(p) for p in got} == {id(p) for p in trainable_}
    assert [p.numel() for p in got] == [int(v) for v in g["numel"]]


def test_reference_get_params_groups_cls_modules_as_its_own():
    from oracle import refload
    if not refload.available():
        pytest.skip("reference tree not present")
    refload.load()
    from utils import solver
    nets = cls_modules()
    owner = {id(p): (k, n) for k, net in nets.items() for n, p in net.named_parameters()}
    got = solver.get_params(nets, SimpleNamespace(**CLS_ARGS))
    g = np.load(GOLDEN)
    assert len(got) == len(g["name"]) == 73
    for grp, m, n, lr, wd in zip(got, g["module"], g["name"], g["lr"], g["weight_decay"]):
        assert len(grp["params"]) == 1
        assert owner[id(grp["params"][0])] == (str(m), str(n))
        assert grp["lr"] == lr and grp["weight_decay"] == wd, (str(m), str(n))


def transfer_pretrained(checkpoint, nets, max_iter):
    """train.py:153-166: the trunk, ContextNet and, for every head, det_net0 of the classification checkpoint without the
    classifier `global_cls`."""
    nets["base_net"].load_state_dict(checkpoint["base_net"])
    if "context_net" in nets and "context_net" in checkpoint:
        nets["context_net"].load_state_dict(checkpoint["context_net"])
    for i in range(max_iter):
        model_dict = nets["det_net%d" % i].state_dict()
        pretrained = checkpoint.get("det_net%d" % i, checkpoint["det_net0"])
        pretrained = {k: v for k, v in pretrained.items() if k in model_dict and k.find("global_cls") <= -1}
        model_dict.update(pretrained)
        nets["det_net%d" % i].load_state_dict(model_dict)


def test_cls_checkpoint_transfers_into_full_heads():
    import step_b200
    cls_cfg = synth.make_cfg(fp16=True, **CLS_CFG, image_size=(400, 400))
    cls_head = step_b200.TwoBranchNet(cls_cfg, cls_only=True)
    cls_head.load_state_dict(synth.cls_head_state_dict(7, cls_cfg), strict=True)
    ckpt = {"base_net": step_b200.BaseNet(cls_cfg).state_dict(), "context_net": step_b200.ContextNet(cls_cfg).state_dict(),
            "det_net0": cls_head.state_dict()}
    cfg = synth.make_cfg(fp16=True, T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False, image_size=(400, 400))
    nets = {"base_net": step_b200.BaseNet(cfg), "context_net": step_b200.ContextNet(cfg)}
    for i in range(3):
        nets["det_net%d" % i] = step_b200.TwoBranchNet(cfg)
    own = {i: {k: v.clone() for k, v in nets["det_net%d" % i].state_dict().items()} for i in range(3)}
    transfer_pretrained(ckpt, nets, 3)
    for i in range(3):
        sd = nets["det_net%d" % i].state_dict()
        moved = [k for k in ckpt["det_net0"] if "global_cls" not in k]
        assert len(moved) == 74 and all(torch.equal(sd[k], ckpt["det_net0"][k]) for k in moved)
        # the classifier and the local branch keep the full head's own initialisation
        assert all(torch.equal(sd[k], own[i][k]) for k in sd if k not in moved)
        assert any(k.startswith("local_conv.") for k in sd if k not in moved)
