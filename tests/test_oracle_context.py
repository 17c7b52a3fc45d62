"""CPU: the oracle's functional model (oracle/model.py: context_net(global_mean=True) + two_branch(context_feat) +
two_branch_losses) reproduces the reference's autograd for the shipped training configuration (scripts/train_step.sh:
T=3, temporal mode NUM_CHUNKS {1:1, 2:1, 3:3}, context on) -- tests/golden/ctx_temporal_grads.npz.  Once pinned here,
the oracle is the element-level checker of the device's context / temporal training step at any resolution."""
import os
import sys

import numpy as np
import torch
from torchvision.ops import roi_align as tv_roi_align

from oracle import model as om
from step_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _train_case import trainable  # noqa: E402


def oracle_objective(cf, sd_ctx, sds, cfg, step_tubes, step_targets, pooled_leaves=False):
    """train.py:266-336 through the oracle: conv_feat cf [B,T',832,H',W'] -> ContextNet, per refinement step the ROIAlign of
    the step's frame slice (torchvision's roi_align, bit-identical to the reference's forward), the per-tube context copy
    of train.py:317-321 and the head's objective.  pooled_leaves: pool under no_grad and make the pooled features leaves
    (the reference has no CPU ROIAlign backward).  Returns (loss, [pooled per step], context_feat)."""
    B = cf.shape[0]
    ctx = om.context_net(cf, sd_ctx, global_mean=True)                     # [B, 1024, T', 1, 1]
    total, pooled_all = 0.0, []
    for i in range(1, len(step_tubes) + 1):
        chunks = cfg.NUM_CHUNKS[i]
        t0 = int((cfg.NUM_CHUNKS[cfg.max_iter] - chunks) / 2) * cfg.T
        tl = chunks * cfg.T
        flat = step_tubes[i - 1]
        fm = cf[:, t0:t0 + tl].reshape(B * tl, 832, cf.shape[3], cf.shape[4])
        with torch.set_grad_enabled(not pooled_leaves and torch.is_grad_enabled()):
            pooled = tv_roi_align(fm, flat.reshape(-1, 5), (7, 7), 1.0 / 16.0, 0, aligned=False).view(-1, tl, 832, 7, 7)
        if pooled_leaves:
            pooled = pooled.detach().requires_grad_(True)
        pooled_all.append(pooled)
        clip = [int(flat[p, 0, 0].item() / tl) for p in range(flat.shape[0])]
        tctx = torch.stack([ctx[c, :, t0:t0 + tl] for c in clip])           # [R, 1024, T_len, 1, 1]
        sd = sds[i - 1]
        _, loc, first, last, logits = om.two_branch(pooled, sd, cfg.T, tctx, cfg.fc_dim, cfg.pool_size, return_logits=True)
        lc, ll, ln = om.two_branch_losses(logits, loc, first, last, flat, step_targets[i - 1], cfg.T)
        total = total + lc.mean() + 5.0 * ll.mean() + 1.0 * ln.mean()
    return total, pooled_all, ctx


def golden_case():
    cfg = synth.make_cfg(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False, image_size=(400, 400))
    step_tubes, step_targets = synth.make_train_case(cfg, 2, 3, 400, 400)
    return cfg, synth.make_conv_feat(2, 9, 25, 25), step_tubes, step_targets


def test_context_temporal_gradients_oracle_matches_reference(golden):
    g = golden("ctx_temporal_grads")
    cfg, cf, step_tubes, step_targets = golden_case()
    cf = cf.requires_grad_(True)
    sd_ctx = trainable(synth.context_net_state_dict())
    sds = [trainable(synth.head_state_dict(100 + i, cfg)) for i in range(3)]
    loss, pooled, ctx = oracle_objective(cf, sd_ctx, sds, cfg, step_tubes, step_targets, pooled_leaves=True)
    loss.backward()
    assert np.allclose(ctx.detach().double().norm().numpy(), g["context_feat_norm"], rtol=1e-5)
    assert np.allclose(loss.detach().numpy(), g["loss"], rtol=1e-5)
    for i, p in enumerate(pooled, 1):
        assert np.allclose(p.detach().double().norm().numpy(), g["pooled_norm%d" % i], rtol=1e-6)
        assert np.allclose(p.grad.double().norm().numpy(), g["pooled_grad_norm%d" % i], rtol=1e-4)
        assert np.allclose(p.grad.reshape(-1)[:16].numpy(), g["pooled_grad_head%d" % i], rtol=1e-3, atol=1e-9)
    assert np.allclose(cf.grad.double().norm().numpy(), g["ctx_feat_grad_norm"], rtol=1e-4)
    assert np.allclose(cf.grad.reshape(-1)[:16].numpy(), g["ctx_feat_grad_head"], rtol=1e-3, atol=1e-10)
    checked = 0
    for key in g.files:
        if not key.startswith("gn:"):
            continue
        tag, k = key[3:].split(":", 1)
        sd = sd_ctx if tag == "ctx" else sds[int(tag[1:])]
        p = sd[k]
        assert p.grad is not None, key
        assert np.allclose(p.grad.double().norm().numpy(), g[key], rtol=1e-4, atol=1e-12), key
        assert np.allclose(p.grad.reshape(-1)[:8].numpy(), g["gh:" + key[3:]], rtol=1e-3, atol=1e-9), key
        checked += 1
    assert checked == 12 + 3 * 34      # ContextNet's 12 Unit3D convolutions and every trainable tensor of the three heads
