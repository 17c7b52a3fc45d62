"""Generates tests/golden/bn_affine_grads.npz and tests/golden/bn_affine_param_groups.npz by running the UNMODIFIED reference
(through the loader and the module builders of tests/golden/make_golden.py) with freeze_affine=False: every BatchNorm's
weight (gamma) and bias (beta) trains, while the statistics stay frozen (freeze_stats=True, BatchNorm in eval mode).
Only runnable in the build container; the fixtures it writes are committed.

    python tests/golden/make_bn_affine_golden.py

bn_affine_grads.npz holds, for every batch3d.weight / batch3d.bias, the gradient norm ("gn:<case>:<name>") and its eight
leading values ("gh:<case>:<name>") in three cases, each the seeded case of an existing gradient golden:
  * trunk -- gen_trunk_grads of make_golden.py (BaseNet, 1 clip of 8x64x64, a seeded linear functional of conv_feat);
  * ctx   -- make_ctx_golden.py (shipped temporal configuration from conv_feat: ContextNet "ctx" and three heads "h0".."h2");
  * cls   -- make_cls_golden.py (the class-only head "h0" and ContextNet "ctx" of train_cls.py).
The head case c1 of head_grads.npz already holds its BatchNorm entries (all of the head's parameters trained there).
bn_affine_param_groups.npz: the reference's get_params over the shipped nets (make_optim_golden.py's arguments) built with
freeze_affine=False, in group order (module key, parameter name, lr, weight_decay, numel)."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, R, build_nets, quiet  # noqa: E402  (loads the reference once, as make_golden.py does)
import make_cls_golden  # noqa: E402
from make_optim_golden import shipped_args  # noqa: E402
from step_b200 import synth  # noqa: E402

from utils import solver  # noqa: E402  (the reference tree is on sys.path once make_golden has loaded it)


def _store(out, case, tag, net):
    n = 0
    for k, p_ in net.named_parameters():
        if "batch3d" not in k:
            continue
        assert p_.requires_grad and p_.grad is not None, (case, tag, k)
        out["gn:%s:%s:%s" % (case, tag, k)] = p_.grad.double().norm().numpy().reshape(1)
        out["gh:%s:%s:%s" % (case, tag, k)] = p_.grad.reshape(-1)[:8].numpy().copy()
        n += 1
    return n


def trunk_case(out):
    cfg = synth.make_cfg(T=2, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(64, 64), freeze_affine=False)
    net = quiet(R.models.BaseNet, cfg)
    net.load_state_dict(synth.base_net_state_dict()); net.eval()
    x = synth.make_clips(1, 8, 64, 64, seed=4321)
    cf = net(x)
    proj = torch.randn(cf.shape, generator=torch.Generator().manual_seed(99))
    loss = (cf * proj).sum() / cf.numel()
    loss.backward()
    out["loss:trunk"] = loss.detach().numpy().reshape(1)
    return _store(out, "trunk", "base", net)


def ctx_case(out):
    cfg = synth.make_cfg(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False, image_size=(400, 400),
                         freeze_affine=False)
    B, N = 2, 3
    nets = build_nets(cfg, 3, context=True)
    cf = synth.make_conv_feat(B, 9, 25, 25).requires_grad_(True)
    step_tubes, step_targets = synth.make_train_case(cfg, B, N, 400, 400)
    context_feat = nets["context_net"](cf)
    loss_back = 0.0
    for i in range(1, cfg.max_iter + 1):
        chunks = cfg.NUM_CHUNKS[i]
        T_start = int((cfg.NUM_CHUNKS[cfg.max_iter] - chunks) / 2) * cfg.T
        T_length = chunks * cfg.T
        flat_tubes = step_tubes[i - 1]
        with torch.no_grad():
            pooled = nets["roi_net"](cf[:, T_start:T_start + T_length].contiguous(), flat_tubes)
        _, C, W, H = pooled.size()
        pooled = pooled.view(-1, T_length, C, W, H).clone().requires_grad_(True)
        temp_context_feat = torch.zeros((pooled.size(0), context_feat.size(1), T_length, 1, 1)).to(context_feat)
        for p in range(pooled.size(0)):      # train.py:317-321
            temp_context_feat[p] = context_feat[int(flat_tubes[p, 0, 0].item() / T_length), :, T_start:T_start + T_length].contiguous().clone()
        _, _, _, _, lc, ll, ln = nets["det_net%d" % (i - 1)](pooled, context_feat=temp_context_feat, tubes=flat_tubes,
                                                              targets=step_targets[i - 1])
        loss_back = loss_back + lc.mean() + ll.mean() * 5.0 + ln.mean() * 1.0
    loss_back.backward()
    out["loss:ctx"] = loss_back.detach().numpy().reshape(1)
    n = _store(out, "ctx", "ctx", nets["context_net"])
    for i in range(3):
        n += _store(out, "ctx", "h%d" % i, nets["det_net%d" % i])
    return n


def cls_case(out):
    cfg = make_cls_golden.cls_cfg()
    cfg.freeze_affine = False
    nets = make_cls_golden.cls_nets(cfg)
    for net in nets.values():
        for p_ in net.parameters():
            p_.requires_grad_(True)
    cf = synth.make_conv_feat(make_cls_golden.B, 9, 25, 25).requires_grad_(True)
    flat_tubes, flat_targets = synth.make_cls_case(cfg, make_cls_golden.B, make_cls_golden.N, 400, 400)
    r = make_cls_golden.objective(nets, cfg, cf, flat_tubes, flat_targets)
    r["loss"].backward()
    out["loss:cls"] = r["loss"].detach().numpy().reshape(1)
    return _store(out, "cls", "ctx", nets["context_net"]) + _store(out, "cls", "h0", nets["det_net0"])


def gen_bn_affine_grads():
    out = {}
    counts = [trunk_case(out), ctx_case(out), cls_case(out)]
    np.savez_compressed(os.path.join(OUT, "bn_affine_grads.npz"), **out)
    print("bn affine grads: trunk / ctx / cls", counts, "BatchNorm tensors")


def gen_bn_affine_param_groups():
    args = shipped_args()
    cfg = synth.make_cfg(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False, image_size=(400, 400),
                         freeze_affine=False)
    nets = build_nets(cfg, args.max_iter, context=True)
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
    np.savez_compressed(os.path.join(OUT, "bn_affine_param_groups.npz"), module=np.array(keys), name=np.array(names),
                        lr=np.array(lrs, np.float64), weight_decay=np.array(wds, np.float64),
                        numel=np.array([g["params"][0].numel() for g in groups], np.int64))
    print("bn affine param groups:", len(groups), "tensors,", sum("batch3d" in n for n in names), "of them BatchNorm")


if __name__ == "__main__":
    gen_bn_affine_param_groups()
    gen_bn_affine_grads()
