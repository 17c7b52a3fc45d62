"""Generates tests/golden/bn_stats_cases.npz by running the UNMODIFIED reference (through the loader and the module builders of
tests/golden/make_golden.py) with freeze_stats=False: the nets' train() leaves every BatchNorm in training mode, so each
forward normalises with the batch statistics and updates the running statistics once (models/networks.py:85-99,
two_branch.py:146-161, 358-373).  cfg.dropout = 0, so no dropout mask enters.  Only runnable in the build container; the
fixture it writes is committed.

    python tests/golden/make_bn_stats_golden.py

Three cases, each the seeded case of make_bn_affine_golden.py, each with freeze_affine True ("fa1") and False ("fa0"):
  * trunk -- BaseNet in .train() on 1 clip of 8x64x64, a seeded linear functional of conv_feat;
  * ctx   -- the shipped temporal configuration from conv_feat: ContextNet "ctx" and three heads "h0".."h2" in .train();
  * cls   -- the class-only head "h0" and ContextNet "ctx" of train_cls.py in .train().
Keys, with <c> = <case>:<fa>:
  out:<c>:<name>     conv_feat (trunk) or the heads' and ContextNet's outputs: their norm ("n") and leading 64 values ("h")
  loss:<c>           the objective
  gn:<c>:<tag>:<p> / gh:<c>:<tag>:<p>   gradient norm and its eight leading values of every parameter with a gradient
  rm:<c>:<tag>:<bn> / rv:<c>:<tag>:<bn>   running_mean / running_var after the step: norm, then the 16 leading values
  nb:<c>:<tag>:<bn>   num_batches_tracked after the step"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, R, build_nets, quiet  # noqa: E402  (loads the reference once, as make_golden.py does)
import make_cls_golden  # noqa: E402
from step_b200 import synth  # noqa: E402


def _out(out, c, name, t):
    t = t.detach().double().reshape(-1)
    out["out:%s:%s:n" % (c, name)] = t.norm().numpy().reshape(1)
    out["out:%s:%s:h" % (c, name)] = t[:64].float().numpy().copy()


def _store(out, c, tag, net):
    n = 0
    for k, p_ in net.named_parameters():
        if p_.grad is None:
            continue
        out["gn:%s:%s:%s" % (c, tag, k)] = p_.grad.double().norm().numpy().reshape(1)
        out["gh:%s:%s:%s" % (c, tag, k)] = p_.grad.reshape(-1)[:8].numpy().copy()
        n += 1
    for k, m in net.named_modules():
        if isinstance(m, torch.nn.BatchNorm3d):
            assert m.training and int(m.num_batches_tracked) == 1, (c, tag, k)
            for kind, t in (("rm", m.running_mean), ("rv", m.running_var)):
                out["%s:%s:%s:%s" % (kind, c, tag, k)] = np.concatenate([t.double().norm().numpy().reshape(1),
                                                                         t[:16].double().numpy()])
            out["nb:%s:%s:%s" % (c, tag, k)] = m.num_batches_tracked.numpy().reshape(1).copy()
    return n


def _train(net, freeze_affine):
    net.train()
    for k, p_ in net.named_parameters():
        p_.requires_grad_(not (freeze_affine and "batch3d" in k))


def trunk_case(out, fa):
    c = "trunk:fa%d" % fa
    cfg = synth.make_cfg(T=2, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(64, 64), freeze_stats=False, freeze_affine=bool(fa),
                         dropout=0.0)
    net = quiet(R.models.BaseNet, cfg)
    net.load_state_dict(synth.base_net_state_dict())
    net.train()
    x = synth.make_clips(1, 8, 64, 64, seed=4321)
    cf = net(x)
    proj = torch.randn(cf.shape, generator=torch.Generator().manual_seed(99))
    loss = (cf * proj).sum() / cf.numel()
    loss.backward()
    _out(out, c, "conv_feat", cf)
    out["loss:" + c] = loss.detach().numpy().reshape(1)
    return _store(out, c, "base", net)


def ctx_case(out, fa):
    c = "ctx:fa%d" % fa
    cfg = synth.make_cfg(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False, image_size=(400, 400),
                         freeze_stats=False, freeze_affine=bool(fa), dropout=0.0)
    B, N = 2, 3
    nets = build_nets(cfg, 3, context=True)
    for k in ["context_net"] + ["det_net%d" % i for i in range(3)]:
        _train(nets[k], fa)
    cf = synth.make_conv_feat(B, 9, 25, 25).requires_grad_(True)
    step_tubes, step_targets = synth.make_train_case(cfg, B, N, 400, 400)
    context_feat = nets["context_net"](cf)
    _out(out, c, "ctx", context_feat)
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
        prob, loc, first, last, lc, ll, ln = nets["det_net%d" % (i - 1)](pooled, context_feat=temp_context_feat, tubes=flat_tubes,
                                                                         targets=step_targets[i - 1])
        for name, t in (("prob", prob), ("loc", loc), ("first", first), ("last", last)):
            _out(out, c, "h%d:%s" % (i - 1, name), t)
        loss_back = loss_back + lc.mean() + ll.mean() * 5.0 + ln.mean() * 1.0
    loss_back.backward()
    out["loss:" + c] = loss_back.detach().numpy().reshape(1)
    n = _store(out, c, "ctx", nets["context_net"])
    for i in range(3):
        n += _store(out, c, "h%d" % i, nets["det_net%d" % i])
    return n


def cls_case(out, fa):
    c = "cls:fa%d" % fa
    cfg = make_cls_golden.cls_cfg()
    cfg.freeze_stats, cfg.freeze_affine, cfg.dropout = False, bool(fa), 0.0
    nets = make_cls_golden.cls_nets(cfg)
    for k in ("context_net", "det_net0"):
        _train(nets[k], fa)
    cf = synth.make_conv_feat(make_cls_golden.B, 9, 25, 25).requires_grad_(True)
    flat_tubes, flat_targets = synth.make_cls_case(cfg, make_cls_golden.B, make_cls_golden.N, 400, 400)
    r = make_cls_golden.objective(nets, cfg, cf, flat_tubes, flat_targets)
    r["loss"].backward()
    _out(out, c, "ctx", r["context_feat"])
    _out(out, c, "h0:prob", r["prob"])
    out["loss:" + c] = r["loss"].detach().numpy().reshape(1)
    return _store(out, c, "ctx", nets["context_net"]) + _store(out, c, "h0", nets["det_net0"])


def gen_bn_stats_cases():
    out = {}
    counts = [f(out, fa) for f in (trunk_case, ctx_case, cls_case) for fa in (1, 0)]
    np.savez_compressed(os.path.join(OUT, "bn_stats_cases.npz"), **out)
    print("bn stats cases: trunk / ctx / cls x freeze_affine 1 / 0:", counts, "gradients,", len(out), "arrays")


if __name__ == "__main__":
    gen_bn_stats_cases()
