"""Generates tests/golden/cls_grads.npz and tests/golden/cls_param_groups.npz by running the UNMODIFIED reference (through the
loader and the module builders of tests/golden/make_golden.py) on seeded synthetic inputs.  Only runnable in the build
container; the fixtures it writes are committed.

    python tests/golden/make_cls_golden.py
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, R, build_nets, quiet  # noqa: E402  (loads the reference once, as make_golden.py does)
from step_b200 import synth  # noqa: E402

from utils import solver  # noqa: E402  (the reference tree is on sys.path once make_golden has loaded it)

# scripts/train_cls.sh (rgb input, context on, one refinement step) and config.py's default weight_decay
CLS_ARGS = dict(base_lr=5e-5, det_lr0=1e-4, det_lr=5e-4, weight_decay=1e-7, input_type="rgb", no_context=False, max_iter=1)
B, N = 2, 6


def cls_cfg():
    """scripts/train_cls.sh: T=9, max_iter=1, spatial mode (NUM_CHUNKS[1] = 1), align pooling of size 7, fc_dim 256, context
    on, 36x400x400 clips (conv_feat [B, 9, 832, 25, 25], the only size ContextNet's AvgPool3d((1,13,13)) accepts)."""
    return synth.make_cfg(T=9, max_iter=1, NUM_CHUNKS={1: 1}, no_context=False, image_size=(400, 400))


def cls_nets(cfg):
    """The reference's ROINet, ContextNet and one class-only head (train_cls.py:100-115) with the synthetic weights."""
    nets = build_nets(cfg, 0, context=True)
    h = quiet(R.models.TwoBranchNet, cfg, cls_only=True)
    h.load_state_dict(synth.cls_head_state_dict(100, cfg), strict=True)
    h.eval(); h.set_device("cpu")
    nets["det_net0"] = h
    for net in nets.values():
        for k, p_ in net.named_parameters():
            p_.requires_grad_("batch3d" not in k)          # BatchNorm affine is frozen (cfg.freeze_affine)
    return nets


def objective(nets, cfg, cf, flat_tubes, flat_targets):
    """train_cls.py:266-311 from conv_feat on, eval-mode dropout: ContextNet, the ROI pooling of frames [0, T) under no_grad
    (the reference has no CPU ROIAlign backward; the pooled features enter as a leaf), the per-tube context copy of
    train_cls.py:304-308 and loss_global_cls.mean()."""
    T_length = cfg.T
    context_feat = nets["context_net"](cf)
    with torch.no_grad():
        pooled = nets["roi_net"](cf[:, :T_length].contiguous(), flat_tubes)
    _, C, W, H = pooled.size()
    pooled = pooled.view(-1, T_length, C, W, H).clone().requires_grad_(True)
    temp_context_feat = torch.zeros((pooled.size(0), context_feat.size(1), T_length, 1, 1)).to(context_feat)
    for p in range(pooled.size(0)):
        temp_context_feat[p] = context_feat[int(flat_tubes[p, 0, 0].item() / T_length), :, :T_length].contiguous().clone()
    prob, loc, first, last, lc, ll, ln = nets["det_net0"](pooled, context_feat=temp_context_feat, tubes=flat_tubes,
                                                          targets=flat_targets)
    return dict(context_feat=context_feat, pooled=pooled, prob=prob, outs=(loc, first, last, lc, ll, ln), loss=lc.mean())


def gen_cls_grads():
    """Loss, gradient norms and leading values of every trainable head and ContextNet tensor, the gradients of the pooled
    features and the context-only gradient of conv_feat; then the same inputs with no classification flag set, where the
    reference's loss is a [1] zero without a graph (so every gradient is zero)."""
    cfg = cls_cfg()
    nets = cls_nets(cfg)
    cf = synth.make_conv_feat(B, 9, 25, 25).requires_grad_(True)
    flat_tubes, flat_targets = synth.make_cls_case(cfg, B, N, 400, 400)
    r = objective(nets, cfg, cf, flat_tubes, flat_targets)
    loc, first, last, lc, ll, ln = r["outs"]
    r["loss"].backward()
    out = {"loss": r["loss"].detach().numpy().reshape(1), "loss_cls_numel": np.asarray([lc.numel()]),
           "context_feat_norm": r["context_feat"].detach().double().norm().numpy().reshape(1),
           "prob_norm": r["prob"].detach().double().norm().numpy().reshape(1),
           "pooled_norm": r["pooled"].detach().double().norm().numpy().reshape(1),
           "pooled_grad_norm": r["pooled"].grad.double().norm().numpy().reshape(1),
           "pooled_grad_head": r["pooled"].grad.reshape(-1)[:16].numpy().copy(),
           "ctx_feat_grad_norm": cf.grad.double().norm().numpy().reshape(1),
           "ctx_feat_grad_head": cf.grad.reshape(-1)[:16].numpy().copy(),
           "other_outputs": np.concatenate([t.detach().reshape(-1).numpy() for t in (loc, first, last, ll, ln)])}
    n = 0
    for tag, net in (("ctx", nets["context_net"]), ("h0", nets["det_net0"])):
        for k, p_ in net.named_parameters():
            if p_.grad is None:
                continue
            out["gn:%s:%s" % (tag, k)] = p_.grad.double().norm().numpy().reshape(1)
            out["gh:%s:%s" % (tag, k)] = p_.grad.reshape(-1)[:8].numpy().copy()
            n += 1
    zero_targets = flat_targets.clone()
    zero_targets[:, :, 4] = 0.0
    z = objective(cls_nets(cfg), cfg, cf.detach(), flat_tubes, zero_targets)
    zl = z["outs"][3]
    out["zero_loss_cls"] = zl.detach().numpy().copy()
    out["zero_loss_requires_grad"] = np.asarray([int(z["loss"].requires_grad)])
    out["zero_prob_norm"] = z["prob"].detach().double().norm().numpy().reshape(1)
    np.savez_compressed(os.path.join(OUT, "cls_grads.npz"), **out)
    print("cls grads:", r["loss"].item(), n, "parameters with gradients; zero-mask loss", zl.tolist(), bool(z["loss"].requires_grad))


def gen_cls_param_groups():
    """The state_dict key names and shapes of a reference TwoBranchNet(cfg, cls_only=True), and the reference's get_params
    over the class-only nets of train_cls.py (base_net, context_net, det_net0), in group order: (module key, parameter name,
    lr, weight_decay, numel)."""
    cfg = cls_cfg()
    args = SimpleNamespace(**CLS_ARGS)
    nets = build_nets(cfg, 0, context=True)
    nets["det_net0"] = quiet(R.models.TwoBranchNet, cfg, cls_only=True)
    sd = nets["det_net0"].state_dict()
    shapes = np.zeros((len(sd), 6), np.int64)
    for i, v in enumerate(sd.values()):
        shapes[i, 0] = v.dim()
        shapes[i, 1:1 + v.dim()] = v.shape
    owner = {id(p): (key, name) for key, net in nets.items() for name, p in net.named_parameters()}
    groups = solver.get_params(nets, args)
    keys, names, lrs, wds = [], [], [], []
    for g in groups:
        assert len(g["params"]) == 1
        key, name = owner[id(g["params"][0])]
        keys.append(key)
        names.append(name)
        lrs.append(g["lr"])
        wds.append(g["weight_decay"])
    np.savez_compressed(os.path.join(OUT, "cls_param_groups.npz"), sd_key=np.array(list(sd.keys())), sd_shape=shapes,
                        module=np.array(keys), name=np.array(names), lr=np.array(lrs, np.float64),
                        weight_decay=np.array(wds, np.float64), numel=np.array([g["params"][0].numel() for g in groups], np.int64))
    print("cls param groups:", len(groups), "tensors,", sum(g["params"][0].numel() for g in groups), "parameters;",
          len(sd), "state_dict entries")


if __name__ == "__main__":
    gen_cls_grads()
    gen_cls_param_groups()
