"""Shared by the batch-statistics tests (test_bn_stats_cpu.py, test_gpu_bn_stats.py): the oracle's functions with every
Unit3D's BatchNorm in training mode (`base_net`, `context_net`, `two_branch`), the objectives of the three cases of
tests/golden/make_bn_stats_golden.py through them, and the state dicts they train."""
import contextlib

import torch
import torch.nn.functional as F
from torchvision.ops import roi_align as tv_roi_align

from oracle import model as om
from step_b200 import synth

BN_MOMENTUM = 0.1  # torch.nn.BatchNorm3d's default, the reference's (i3dpt.py:101)


def unit3d_train(x, sd, p, stride=(1, 1, 1), relu=True):
    """oracle.model.unit3d with BatchNorm3d in training mode (freeze_stats=False): batch statistics, and sd's running
    statistics and num_batches_tracked updated in place, as BatchNorm3d.forward does."""
    w = sd[p + "conv3d.weight"]
    k = w.shape[2:]
    pads = [om.same_pad(k[i], stride[i]) for i in range(3)]
    x = F.pad(x, (pads[2][0], pads[2][1], pads[1][0], pads[1][1], pads[0][0], pads[0][1]))
    y = F.conv3d(x, w, sd.get(p + "conv3d.bias"), stride=stride)
    if p + "batch3d.weight" in sd:
        y = F.batch_norm(y, sd[p + "batch3d.running_mean"], sd[p + "batch3d.running_var"], sd[p + "batch3d.weight"],
                         sd[p + "batch3d.bias"], True, BN_MOMENTUM, om.BN_EPS)
        if p + "batch3d.num_batches_tracked" in sd:
            sd[p + "batch3d.num_batches_tracked"].add_(1)
    return F.relu(y) if relu else y


@contextlib.contextmanager
def _training_bn():
    """oracle.model's compositions (mixed, base_net, context_net, two_branch) reach every Unit3D through the module's
    `unit3d`; for the block it is the training-mode one, so the oracle's own composition code is what runs."""
    saved = om.unit3d
    om.unit3d = unit3d_train
    try:
        yield
    finally:
        om.unit3d = saved


def base_net_train(x, sd):
    with _training_bn():
        return om.base_net(x, sd)


def context_net_train(conv_feat, sd):
    with _training_bn():
        return om.context_net(conv_feat, sd, global_mean=True)


def two_branch_train(global_feat, sd, T, context_feat, fc_dim, pool_size, cls_only=False):
    """om.two_branch(..., return_logits=True) with its BatchNorms in training mode."""
    with _training_bn():
        return om.two_branch(global_feat, sd, T, context_feat, fc_dim, pool_size, cls_only=cls_only, return_logits=True)


def trainable_sd(sd, freeze_affine, convs_too=True):
    """A copy of sd whose float tensors require grad except the running statistics (updated in place by the oracle's
    training-mode BatchNorm) and, with freeze_affine, BatchNorm's gamma and beta; convs_too=False: only the conv weights and
    the BatchNorm affine may (the trunk's trainable set)."""
    def train(k, v):
        if not v.is_floating_point() or "running_" in k:
            return False
        if "batch3d" in k:
            return not freeze_affine
        return convs_too or k.endswith("conv3d.weight")
    return {k: v.clone().requires_grad_(train(k, v)) for k, v in sd.items()}


def trunk_cfg(fp16=False, freeze_affine=True):
    return synth.make_cfg(T=2, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(64, 64), freeze_stats=False,
                          freeze_affine=freeze_affine, dropout=0.0, fp16=fp16)


def trunk_objective(sd, x=None):
    """BaseNet in .train() on 1 clip of 8x64x64 and the seeded linear functional of make_bn_stats_golden.trunk_case.
    Returns (loss, conv_feat, proj)."""
    x = synth.make_clips(1, 8, 64, 64, seed=4321) if x is None else x
    cf = base_net_train(x, sd)
    proj = torch.randn(cf.shape, generator=torch.Generator().manual_seed(99))
    return (cf * proj).sum() / cf.numel(), cf, proj


def ctx_case(fp16=False, freeze_affine=True):
    """(cfg, conv_feat, step_tubes, step_targets) of make_bn_stats_golden.ctx_case."""
    cfg = synth.make_cfg(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False, image_size=(400, 400),
                         freeze_stats=False, freeze_affine=freeze_affine, dropout=0.0, fp16=fp16)
    step_tubes, step_targets = synth.make_train_case(cfg, 2, 3, 400, 400)
    return cfg, synth.make_conv_feat(2, 9, 25, 25), step_tubes, step_targets


def ctx_objective(cf, sd_ctx, sds, cfg, step_tubes, step_targets, leaves=True):
    """train.py:266-336 from conv_feat with every BatchNorm in training mode; with leaves the pooled features of each step
    enter as leaves (pooled under no_grad, as the reference's CPU case does), else the gradient flows through the pooling
    into conv_feat.  Returns (loss, context_feat, [per-step outputs], [pooled features])."""
    B = cf.shape[0]
    ctx = context_net_train(cf, sd_ctx)
    total, outs, pooled_all = 0.0, [], []
    for i in range(1, len(step_tubes) + 1):
        chunks = cfg.NUM_CHUNKS[i]
        t0 = int((cfg.NUM_CHUNKS[cfg.max_iter] - chunks) / 2) * cfg.T
        tl = chunks * cfg.T
        flat = step_tubes[i - 1]
        fm = cf[:, t0:t0 + tl].reshape(B * tl, 832, cf.shape[3], cf.shape[4])
        with torch.set_grad_enabled(not leaves and torch.is_grad_enabled()):
            pooled = tv_roi_align(fm, flat.reshape(-1, 5), (7, 7), 1.0 / 16.0, 0, aligned=False).view(-1, tl, 832, 7, 7)
        if leaves:
            pooled = pooled.detach().requires_grad_(True)
        pooled_all.append(pooled)
        clip = [int(flat[p, 0, 0].item() / tl) for p in range(flat.shape[0])]
        tctx = torch.stack([ctx[c, :, t0:t0 + tl] for c in clip])
        prob, loc, first, last, logits = two_branch_train(pooled, sds[i - 1], cfg.T, tctx, cfg.fc_dim, cfg.pool_size)
        outs.append((prob, loc, first, last))
        lc, ll, ln = om.two_branch_losses(logits, loc, first, last, flat, step_targets[i - 1], cfg.T)
        total = total + lc.mean() + 5.0 * ll.mean() + 1.0 * ln.mean()
    return total, ctx, outs, pooled_all


def ctx_objective_full(cf, sd_ctx, sds, cfg, step_tubes, step_targets):
    """The loss of ctx_objective with the gradient through the pooling (train_step's objective from conv_feat)."""
    return ctx_objective(cf, sd_ctx, sds, cfg, step_tubes, step_targets, leaves=False)[0]


def cls_case(fp16=False, freeze_affine=True):
    """(cfg, conv_feat, flat_tubes, flat_targets) of make_bn_stats_golden.cls_case (train_cls.py's shipped stage)."""
    cfg = synth.make_cfg(T=9, max_iter=1, NUM_CHUNKS={1: 1}, no_context=False, image_size=(400, 400), freeze_stats=False,
                         freeze_affine=freeze_affine, dropout=0.0, fp16=fp16)
    flat_tubes, flat_targets = synth.make_cls_case(cfg, 2, 6, 400, 400)
    return cfg, synth.make_conv_feat(2, 9, 25, 25), flat_tubes, flat_targets


def cls_objective(cf, sd_ctx, sd, cfg, flat_tubes, flat_targets):
    """train_cls.py:266-311 with BatchNorm in training mode.  Returns (loss, context_feat, prob, pooled leaf)."""
    B, tl = cf.shape[0], cfg.T
    ctx = context_net_train(cf, sd_ctx)
    fm = cf[:, :tl].reshape(B * tl, 832, cf.shape[3], cf.shape[4])
    with torch.no_grad():
        pooled = tv_roi_align(fm, flat_tubes.reshape(-1, 5), (7, 7), 1.0 / 16.0, 0, aligned=False).view(-1, tl, 832, 7, 7)
    pooled = pooled.detach().requires_grad_(True)
    clip = [int(flat_tubes[p, 0, 0].item() / tl) for p in range(flat_tubes.shape[0])]
    tctx = torch.stack([ctx[c, :, :tl] for c in clip])
    prob, loc, first, last, logits = two_branch_train(pooled, sd, cfg.T, tctx, cfg.fc_dim, cfg.pool_size, cls_only=True)
    lc, _, _ = om.two_branch_losses(logits, loc, first, last, flat_tubes, flat_targets, cfg.T, cls_only=True)
    return lc.mean(), ctx, prob, pooled
