"""Shared by the synchronised batch-statistics tests (test_bn_sync_cpu.py, test_gpu_bn_sync.py, _bn_sync_worker.py): the
training-mode oracle of _bn_stats_case.py run as the reference's nn.DataParallel runs it over W devices, and the cases of
tests/golden/make_bn_sync_golden.py.

DataParallel (train.py:141-148) scatters the clips in chunks, clips [r * ceil(B / W), ...) to replica r; the trunk and
ContextNet normalise each chunk with its own statistics, and only replica 0's running-statistic update survives.  The heads
are not replicated: each runs over every row of the batch (train.py:313-323).  `sync_objective` computes
J = (1 / W) sum_r L_r, L_r the objective of rank r's rows, with the heads normalising over the concatenation of every
rank's rows; it is the reference's whole-batch objective when every rank has the same rows in each step and every row is
a classification and regression sample (each mean of the losses is then the mean of the ranks' means)."""
import math

import torch
from torchvision.ops import roi_pool as tv_roi_pool

from oracle import model as om
from step_b200 import synth

import _bn_stats_case as bc

W = 2
SHIPPED_KW = dict(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False)
CLS_KW = dict(T=9, max_iter=1, NUM_CHUNKS={1: 1}, no_context=False)


def case_cfg(name, fp16=False, freeze_affine=True):
    kw = SHIPPED_KW if name == "ctx" else CLS_KW
    return synth.make_cfg(fp16=fp16, image_size=(64, 64), freeze_stats=False, freeze_affine=freeze_affine, dropout=0.0, **kw)


def whole_case(name, cfg):
    """(clips [2, 36, 64, 64] input, step_tubes, step_targets) of the whole batch: the shipped case of
    test_gpu_bn_stats._shipped ("ctx") or the class-only stage ("cls"), 3 rows per clip, every row a classification and
    regression sample."""
    x = synth.make_clips(2, 36, 64, 64, seed=11)
    if name == "ctx":
        step_tubes, step_targets = synth.make_train_case(cfg, 2, 3, 64, 64, seed=3)
        for tg in step_targets:
            tg[:, :, 4:6] = 1.0
    else:
        flat_tubes, flat_targets = synth.make_cls_case(cfg, 2, 3, 64, 64)
        step_tubes, step_targets = [flat_tubes], [flat_targets]
    return x, step_tubes, step_targets


def step_frames(cfg, i):
    chunks = cfg.NUM_CHUNKS[i]
    return int((cfg.NUM_CHUNKS[cfg.max_iter] - chunks) / 2) * cfg.T, chunks * cfg.T


def split_rows(cfg, x, step_tubes, step_targets, world=W):
    """DataParallel's chunk r of the clips and the rows its clips select, with frame indices relative to the chunk:
    [(x_r, [tubes_r per step], [targets_r per step])]."""
    B = x.shape[0]
    per = math.ceil(B / world)
    out = []
    for r in range(world):
        c0, c1 = r * per, min((r + 1) * per, B)
        tubes_r, targets_r = [], []
        for i, (t, tg) in enumerate(zip(step_tubes, step_targets)):
            tl = step_frames(cfg, i + 1)[1]
            clip = torch.div(t[:, 0, 0], tl, rounding_mode="floor").long()
            sel = (clip >= c0) & (clip < c1)
            tr = t[sel].clone()
            tr[:, :, 0] -= c0 * tl
            tubes_r.append(tr)
            targets_r.append(tg[sel].clone())
        out.append((x[c0:c1].contiguous(), tubes_r, targets_r))
    return out


def _own_stats(sd):
    """sd with its own copies of the running statistics and num_batches_tracked (the parameters shared): a replica's."""
    return {k: (v.detach().clone() if "running_" in k or "num_batches" in k else v) for k, v in sd.items()}


def sync_objective(cfg, sds, ranks, cls_only=False, pool=None, from_feat=False):
    """J = (1 / W) sum_r L_r of the ranks [(x_r, tubes_r, targets_r)] with the trunk and ContextNet per rank (sds' running
    statistics take rank 0's update only) and each head over every rank's rows (its running statistics updated once).
    sds: "base_net", "context_net", "det_net<i>" state dicts.  pool(fm, rois, size, scale): torchvision's roi_pool (the
    shipped ROIPool) by default.  from_feat: x_r is rank r's conv_feat (no trunk), and the pooled features enter the heads
    as leaves pooled under no_grad by ROIAlign, as make_bn_sync_golden.py feeds the reference (it has no CPU ROI backward).
    Returns (J, [L_r], {"ctx<r>": ContextNet output of rank r, "h<i>:prob": the head's probabilities over all rows}."""
    if pool is None:
        pool = bc.tv_roi_align if from_feat else (lambda fm, rois, size, scale, *a, **k: tv_roi_pool(fm, rois, size, scale))
    feats, named = [], {}
    for r, (x, _, _) in enumerate(ranks):
        sb = sds.get("base_net") if r == 0 else _own_stats(sds.get("base_net", {}))
        sc = sds["context_net"] if r == 0 else _own_stats(sds["context_net"])
        cf = x if from_feat else bc.base_net_train(x, sb)
        ctx = bc.context_net_train(cf, sc)
        named["ctx%d" % r] = ctx
        feats.append((cf, ctx))
    losses = [0.0] * len(ranks)
    for i in range(len(ranks[0][1])):
        t0, tl = step_frames(cfg, i + 1)
        pooled, tctx, rows = [], [], []
        for (cf, ctx), (_, tubes_r, _) in zip(feats, ranks):
            B = cf.shape[0]
            flat = tubes_r[i]
            fm = cf[:, t0:t0 + tl].reshape(B * tl, 832, cf.shape[3], cf.shape[4])
            with torch.set_grad_enabled(not from_feat and torch.is_grad_enabled()):
                p = pool(fm, flat.reshape(-1, 5), (7, 7), 1.0 / 16.0, 0, aligned=False).view(-1, tl, 832, 7, 7)
            pooled.append(p.detach() if from_feat else p)
            clip = [int(flat[q, 0, 0].item() / tl) for q in range(flat.shape[0])]
            tctx.append(torch.stack([ctx[c, :, t0:t0 + tl] for c in clip]))
            rows.append(flat.shape[0])
        prob, loc, first, last, logits = bc.two_branch_train(torch.cat(pooled), sds["det_net%d" % i], cfg.T, torch.cat(tctx),
                                                             cfg.fc_dim, cfg.pool_size, cls_only=cls_only)
        named["h%d:prob" % i] = prob
        off = 0
        for r, (_, tubes_r, targets_r) in enumerate(ranks):
            s = slice(off, off + rows[r])
            off += rows[r]
            lc, ll, ln = om.two_branch_losses(logits[s], loc[s], first[s], last[s], tubes_r[i], targets_r[i], cfg.T,
                                              cls_only=cls_only)
            losses[r] = losses[r] + (lc.mean() if cls_only else lc.mean() + 5.0 * ll.mean() + 1.0 * ln.mean())
    return sum(losses) / len(ranks), losses, named


def trunk_sync_objective(sd, xs):
    """The trunk case of make_bn_sync_golden.py: BaseNet per rank chunk (rank 0's running-statistic update kept) and the
    mean over the ranks of the seeded linear functional of each chunk's conv_feat.  Returns (J, [conv_feat_r])."""
    losses, cfs = [], []
    for r, x in enumerate(xs):
        cf = bc.base_net_train(x, sd if r == 0 else _own_stats(sd))
        proj = torch.randn(cf.shape, generator=torch.Generator().manual_seed(99 + r))
        losses.append((cf * proj).sum() / cf.numel())
        cfs.append(cf)
    return sum(losses) / len(xs), cfs


def trunk_inputs():
    return [synth.make_clips(1, 8, 64, 64, seed=4321 + r) for r in range(W)]


def feat_case(name, freeze_affine):
    """(cfg, conv_feat [2, 9, 832, 25, 25], step_tubes, step_targets) of the fixture's ctx / cls cases: the conv_feat of
    _bn_stats_case's cases (25 x 25, the only map ContextNet's AvgPool3d((1, 13, 13)) takes in the reference), 3 rows per
    clip, every row a classification and regression sample."""
    if name == "ctx":
        cfg, cf, step_tubes, step_targets = bc.ctx_case(freeze_affine=freeze_affine)
        for tg in step_targets:
            tg[:, :, 4:6] = 1.0
        return cfg, cf, step_tubes, step_targets
    cfg = synth.make_cfg(T=9, max_iter=1, NUM_CHUNKS={1: 1}, no_context=False, image_size=(400, 400), freeze_stats=False,
                         freeze_affine=freeze_affine, dropout=0.0)
    flat_tubes, flat_targets = synth.make_cls_case(cfg, 2, 3, 400, 400)
    return cfg, synth.make_conv_feat(2, 9, 25, 25), [flat_tubes], [flat_targets]


def oracle_sds(name, cfg, fa):
    """Trainable oracle state dicts of the case's synthetic nets (the trunk's trainable set: conv weights and, with
    freeze_affine False, BatchNorm's affine)."""
    heads = [synth.cls_head_state_dict(100, cfg)] if name == "cls" else [synth.head_state_dict(100 + i, cfg) for i in range(3)]
    sds = {"base_net": bc.trainable_sd(synth.base_net_state_dict(), fa, convs_too=False),
           "context_net": bc.trainable_sd(synth.context_net_state_dict(), fa)}
    for i, h in enumerate(heads):
        sds["det_net%d" % i] = bc.trainable_sd(h, fa)
    return sds
