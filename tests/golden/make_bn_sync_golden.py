"""Generates tests/golden/bn_sync_cases.npz by running the UNMODIFIED reference (through the loader and the module builders of
tests/golden/make_golden.py) with freeze_stats=False as its nn.DataParallel runs it over two devices (train.py:141-148,
313-323): base_net and context_net replicated, each replica normalising its own chunk of the clips with that chunk's
statistics and only replica 0's running-statistic update kept; each head over every row of the batch.  On the CPU the
replicas run one after the other on the same module; chunk 1 updates copies of the running statistics, which are dropped.  Equal rows
per chunk, and every row a classification and regression sample, so the reference's whole-batch objective is the mean of
the chunks' objectives.  cfg.dropout = 0.  Only runnable in the build container; the fixture it writes is committed.

    python tests/golden/make_bn_sync_golden.py

Cases, each with freeze_affine True ("fa1") and False ("fa0"):
  * trunk -- BaseNet in .train() on two chunks of 1 clip of 8x64x64, the mean of a seeded linear functional of each
             chunk's conv_feat;
  * ctx   -- the shipped temporal configuration from the conv_feat of make_bn_stats_golden.ctx_case (two clips, one per
             chunk, 3 rows each): ContextNet per chunk and three heads over all rows;
  * cls   -- the class-only stage the same way (make_cls_case's rows, 3 per clip).
The pooled features enter the heads as leaves pooled under no_grad (the reference has no CPU ROI backward).
Keys as in make_bn_stats_golden.py (<c> = <case>:<fa>): loss:<c>, gn / gh:<c>:<tag>:<p>, rm / rv / nb:<c>:<tag>:<bn>,
out:<c>:<name>:n / :h."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden import OUT, R, build_nets, quiet  # noqa: E402  (loads the reference once, as make_golden.py does)
from make_bn_stats_golden import _out, _train  # noqa: E402
import _bn_sync_case as sc  # noqa: E402
from step_b200 import synth  # noqa: E402


def replicas(net, chunks):
    """net over each chunk in turn, with replica 0's running statistics kept (DataParallel's replicate / gather): the other
    chunks update copies of the buffers, which are dropped afterwards (the kept tensors are never written again, so the
    autograd graph's saved buffers stay valid)."""
    bns = [m for m in net.modules() if isinstance(m, torch.nn.BatchNorm3d)]
    names = ("running_mean", "running_var", "num_batches_tracked")
    outs = [net(chunks[0])]
    kept = [{k: getattr(m, k) for k in names} for m in bns]
    for x in chunks[1:]:
        for m in bns:
            for k in names:
                setattr(m, k, getattr(m, k).clone())
        outs.append(net(x))
    for m, b in zip(bns, kept):
        for k in names:
            setattr(m, k, b[k])
    return torch.cat(outs)


def _store(out, c, tag, net, nb=1):
    n = 0
    for k, p_ in net.named_parameters():
        if p_.grad is None:
            continue
        out["gn:%s:%s:%s" % (c, tag, k)] = p_.grad.double().norm().numpy().reshape(1)
        out["gh:%s:%s:%s" % (c, tag, k)] = p_.grad.reshape(-1)[:8].numpy().copy()
        n += 1
    for k, m in net.named_modules():
        if isinstance(m, torch.nn.BatchNorm3d):
            assert m.training and int(m.num_batches_tracked) == nb, (c, tag, k)
            for kind, t in (("rm", m.running_mean), ("rv", m.running_var)):
                out["%s:%s:%s:%s" % (kind, c, tag, k)] = np.concatenate([t.double().norm().numpy().reshape(1),
                                                                         t[:16].double().numpy()])
            out["nb:%s:%s:%s" % (c, tag, k)] = m.num_batches_tracked.numpy().reshape(1).copy()
    return n


def trunk_case(out, fa):
    c = "trunk:fa%d" % fa
    cfg = synth.make_cfg(T=2, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(64, 64), freeze_stats=False, freeze_affine=bool(fa),
                         dropout=0.0)
    net = quiet(R.models.BaseNet, cfg)
    net.load_state_dict(synth.base_net_state_dict())
    net.train()
    xs = sc.trunk_inputs()
    cf = replicas(net, xs)
    loss = 0.0
    for r in range(len(xs)):
        proj = torch.randn(cf[r:r + 1].shape, generator=torch.Generator().manual_seed(99 + r))
        loss = loss + (cf[r:r + 1] * proj).sum() / cf[r:r + 1].numel()
    loss = loss / len(xs)
    loss.backward()
    _out(out, c, "conv_feat", cf)
    out["loss:" + c] = loss.detach().numpy().reshape(1)
    return _store(out, c, "base", net)


def heads_case(out, name, fa):
    """ctx / cls: ContextNet replicated over the two clips, then train.py:294-336 (or train_cls.py:266-311) over all rows."""
    c = "%s:fa%d" % (name, fa)
    cfg, cf, step_tubes, step_targets = sc.feat_case(name, bool(fa))
    nets = build_nets(cfg, 3 if name == "ctx" else 0, context=True)
    if name == "cls":
        h = quiet(R.models.TwoBranchNet, cfg, cls_only=True)
        h.load_state_dict(synth.cls_head_state_dict(100, cfg), strict=True)
        h.set_device("cpu")
        nets["det_net0"] = h
    heads = ["det_net%d" % i for i in range(len(step_tubes))]
    for k in ["context_net"] + heads:
        _train(nets[k], fa)
    cf = cf.requires_grad_(True)
    context_feat = replicas(nets["context_net"], [cf[0:1], cf[1:2]])
    _out(out, c, "ctx", context_feat)
    loss_back = 0.0
    for i in range(len(step_tubes)):
        T_start, T_length = sc.step_frames(cfg, i + 1)
        flat_tubes = step_tubes[i]
        with torch.no_grad():
            pooled = nets["roi_net"](cf[:, T_start:T_start + T_length].contiguous(), flat_tubes)
        _, C, W, H = pooled.size()
        pooled = pooled.view(-1, T_length, C, W, H).clone().requires_grad_(True)
        temp_context_feat = torch.zeros((pooled.size(0), context_feat.size(1), T_length, 1, 1)).to(context_feat)
        for p in range(pooled.size(0)):      # train.py:317-321
            temp_context_feat[p] = context_feat[int(flat_tubes[p, 0, 0].item() / T_length), :, T_start:T_start + T_length].contiguous().clone()
        prob, loc, first, last, lc, ll, ln = nets[heads[i]](pooled, context_feat=temp_context_feat, tubes=flat_tubes,
                                                            targets=step_targets[i])
        _out(out, c, "h%d:prob" % i, prob)
        loss_back = loss_back + lc.mean() + (0.0 if name == "cls" else ll.mean() * 5.0 + ln.mean() * 1.0)
    loss_back.backward()
    out["loss:" + c] = loss_back.detach().numpy().reshape(1)
    n = _store(out, c, "ctx", nets["context_net"])
    for i, k in enumerate(heads):
        n += _store(out, c, "h%d" % i, nets[k])
    return n


def gen_bn_sync_cases():
    out = {}
    counts = [trunk_case(out, fa) for fa in (1, 0)]
    counts += [heads_case(out, name, fa) for name in ("ctx", "cls") for fa in (1, 0)]
    np.savez_compressed(os.path.join(OUT, "bn_sync_cases.npz"), **out)
    print("bn sync cases: trunk x fa 1 / 0, ctx x fa 1 / 0, cls x fa 1 / 0:", counts, "gradients,", len(out), "arrays")


if __name__ == "__main__":
    gen_bn_sync_cases()
