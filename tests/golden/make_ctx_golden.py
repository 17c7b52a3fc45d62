"""Generates tests/golden/ctx_temporal_grads.npz by running the UNMODIFIED reference (through the loader and the module
builders of tests/golden/make_golden.py) on seeded synthetic inputs.  Only runnable in the build container; the fixture it
writes is committed.

    python tests/golden/make_ctx_golden.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, build_nets  # noqa: E402  (loads the reference once, as make_golden.py does)
from step_b200 import synth  # noqa: E402


def gen_ctx_temporal_grads():
    """The shipped training configuration (scripts/train_step.sh: T=3, iterative_mode=temporal -> NUM_CHUNKS {1:1, 2:1,
    3:3}, context on) from conv_feat on: ContextNet and three TwoBranchNet heads of the reference, eval-mode dropout, the
    per-tube context copy of train.py:317-321 and the objective of train.py:323-336.  conv_feat [2, 9, 832, 25, 25] is the
    trunk output at 36x400x400, the only size ContextNet's AvgPool3d((1,13,13)) accepts.  The reference has no CPU ROIAlign
    backward, so each step's pooled features come from its ROINet under no_grad and enter as leaves; ROIAlign backward is
    pinned separately (roi_cross_cases).  Stores the loss, per-parameter gradient norms and leading values of ContextNet
    and every head, the gradient of each step's pooled features and the context-only gradient of conv_feat."""
    cfg = synth.make_cfg(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False, image_size=(400, 400))
    B, N = 2, 3
    nets = build_nets(cfg, 3, context=True)
    for net in nets.values():
        for k, p_ in net.named_parameters():
            p_.requires_grad_("batch3d" not in k)          # BatchNorm affine is frozen (cfg.freeze_affine)
    cf = synth.make_conv_feat(B, 9, 25, 25).requires_grad_(True)
    step_tubes, step_targets = synth.make_train_case(cfg, B, N, 400, 400)
    context_feat = nets["context_net"](cf)
    out = {"context_feat_norm": context_feat.detach().double().norm().numpy().reshape(1)}
    loss_back = 0.0
    pooled_leaves = []
    for i in range(1, cfg.max_iter + 1):
        chunks = cfg.NUM_CHUNKS[i]
        T_start = int((cfg.NUM_CHUNKS[cfg.max_iter] - chunks) / 2) * cfg.T
        T_length = chunks * cfg.T
        flat_tubes = step_tubes[i - 1]
        with torch.no_grad():
            pooled = nets["roi_net"](cf[:, T_start:T_start + T_length].contiguous(), flat_tubes)
        _, C, W, H = pooled.size()
        pooled = pooled.view(-1, T_length, C, W, H).clone().requires_grad_(True)
        pooled_leaves.append(pooled)
        out["pooled_norm%d" % i] = pooled.detach().double().norm().numpy().reshape(1)
        temp_context_feat = torch.zeros((pooled.size(0), context_feat.size(1), T_length, 1, 1)).to(context_feat)
        for p in range(pooled.size(0)):      # train.py:317-321
            temp_context_feat[p] = context_feat[int(flat_tubes[p, 0, 0].item() / T_length), :, T_start:T_start + T_length].contiguous().clone()
        _, _, _, _, lc, ll, ln = nets["det_net%d" % (i - 1)](pooled, context_feat=temp_context_feat, tubes=flat_tubes,
                                                              targets=step_targets[i - 1])
        loss_back = loss_back + lc.mean() + ll.mean() * 5.0 + ln.mean() * 1.0
    loss_back.backward()
    out["loss"] = loss_back.detach().numpy().reshape(1)
    for i, pl in enumerate(pooled_leaves, 1):
        out["pooled_grad_norm%d" % i] = pl.grad.double().norm().numpy().reshape(1)
        out["pooled_grad_head%d" % i] = pl.grad.reshape(-1)[:16].numpy().copy()
    out["ctx_feat_grad_norm"] = cf.grad.double().norm().numpy().reshape(1)
    out["ctx_feat_grad_head"] = cf.grad.reshape(-1)[:16].numpy().copy()
    n = 0
    for tag, net in [("ctx", nets["context_net"])] + [("h%d" % i, nets["det_net%d" % i]) for i in range(3)]:
        for k, p_ in net.named_parameters():
            if p_.grad is None:
                continue
            out["gn:%s:%s" % (tag, k)] = p_.grad.double().norm().numpy().reshape(1)
            out["gh:%s:%s" % (tag, k)] = p_.grad.reshape(-1)[:8].numpy().copy()
            n += 1
    np.savez_compressed(os.path.join(OUT, "ctx_temporal_grads.npz"), **out)
    print("ctx temporal grads:", float(loss_back.detach()), n, "parameters with gradients")


if __name__ == "__main__":
    gen_ctx_temporal_grads()
