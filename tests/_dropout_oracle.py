"""The head's training forward with the reference's two dropout calls (models/two_branch.py:244, 261) given as fixed masks,
on top of the eval-mode oracle (oracle/model.py::two_branch), and the replay of the masks torch's F.dropout draws.

two_branch(..., dropout_masks=(global, local), p=...) multiplies, as nn.Dropout does in training mode,
  * the flattened global feature [N, C' = fc*ps^2 (+ 1024 with context), T', 1, 1] (two_branch.py:239-244), which only the
    classifier reads: the local branch concatenates the undropped downsample output (:256);
  * downsample2's output [N*T', fc, ps, ps] (:259-261), which feeds local_reg and both neighbour regressors;
by mask * scale, scale = (float)(1.0 / (double)(float)(1 - p)) (ATen's fused dropout).  Masks are in those shapes (bool or
0/1); local is ignored for class-only heads.  tests/test_dropout_cpu.py pins it against the reference's TwoBranchNet."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import model as om


def scale_of(p):
    return float(np.float32(1.0 / float(np.float32(1.0 - p))))


def _drop(x, mask, p):
    return x * mask.to(x.dtype) * scale_of(p)


def two_branch(global_feat, sd, T, context_feat=None, fc_dim=256, pool_size=7, cls_only=False, return_logits=False,
               dropout_masks=None, p=None):
    """oracle.model.two_branch with the reference's training-mode dropout at its two sites (dropout_masks None: the
    oracle itself)."""
    if dropout_masks is None:
        return om.two_branch(global_feat, sd, T, context_feat, fc_dim, pool_size, cls_only, return_logits)
    gmask, lmask = dropout_masks
    N, Tl, C, W, H = global_feat.shape
    chunks = int(Tl / T)
    chunk_idx = [j * T + int(T / 2) for j in range(chunks)]
    half_T = int(T / 2)
    g = global_feat.permute(0, 2, 1, 3, 4)
    g = om.mixed(g, sd, "i3d_conv.0.")
    g = om.mixed(g, sd, "i3d_conv.1.")
    gconv = F.conv3d(g, sd["downsample.weight"], sd["downsample.bias"])
    flat = gconv.permute(0, 2, 1, 3, 4).contiguous().view(N, Tl, -1, 1, 1).permute(0, 2, 1, 3, 4).contiguous()
    if context_feat is not None:
        flat = torch.cat([flat, context_feat], dim=1)
    flat = _drop(flat, gmask.view(flat.shape), p)
    cls = F.conv3d(flat, sd["global_cls.weight"], sd["global_cls.bias"]).squeeze(3).squeeze(3).mean(2)
    prob = torch.sigmoid(cls)
    if cls_only:
        z = torch.tensor([0.0])
        return (prob, z, z, z, cls) if return_logits else (prob, z, z, z)
    lf = torch.cat([global_feat.permute(0, 2, 1, 3, 4), gconv], dim=1)
    lf = lf.permute(0, 2, 1, 3, 4).contiguous().view(N * Tl, -1, W, H)
    lf = om._bottleneck(lf, sd, "local_conv.0.", True)
    lf = om._bottleneck(lf, sd, "local_conv.1.", False)
    lf = om._bottleneck(lf, sd, "local_conv.2.", False)
    lf = F.conv2d(lf, sd["downsample2.weight"], sd["downsample2.bias"])
    lf = _drop(lf, lmask.view(lf.shape), p)
    lf = lf.reshape(lf.size(0), -1)
    local_loc = F.linear(lf, sd["local_reg.weight"], sd["local_reg.bias"]).view(N, Tl, -1)
    D = fc_dim * pool_size ** 2
    s0, s1 = chunk_idx[0] - half_T, chunk_idx[0] + half_T + 1
    e0, e1 = chunk_idx[-1] - half_T, chunk_idx[-1] + half_T + 1
    first = local_loc[:, s0:s1].contiguous().clone()
    last = local_loc[:, e0:e1].contiguous().clone()
    first = first + F.linear(lf.view(N, Tl, -1)[:, s0:s1].contiguous().view(-1, D),
                             sd["neighbor_reg1.weight"], sd["neighbor_reg1.bias"]).view(N, T, -1)
    last = last + F.linear(lf.view(N, Tl, -1)[:, e0:e1].contiguous().view(-1, D),
                           sd["neighbor_reg2.weight"], sd["neighbor_reg2.bias"]).view(N, T, -1)
    if return_logits:
        return prob, local_loc, first, last, cls
    return prob, local_loc, first, last


def head_draw_sizes(R, T, fc_dim=256, pool_size=7, context=True, cls_only=False):
    """Element counts of a head's draws in the reference's order: [global] or [global, local]."""
    D = fc_dim * pool_size ** 2
    return [R * (D + (1024 if context else 0)) * T] + ([] if cls_only else [R * T * D])


def replay(sizes, p, device="cuda"):
    """The masks F.dropout draws, in order, for fp32 tensors of these element counts from the current state of the
    device's default generator (advancing it as the reference's forward does): a list of bool CPU tensors."""
    return [(F.dropout(torch.ones(n, device=device), p, True) != 0).cpu() for n in sizes]


def patch_heads(monkeypatch, masks, p):
    """Make oracle.model.two_branch apply the next (global[, local]) masks of `masks` at every call, in call order (the
    oracle objectives of the training tests call it once per refinement step)."""
    queue = list(masks)

    def patched(global_feat, sd, T, context_feat=None, fc_dim=256, pool_size=7, cls_only=False, return_logits=False):
        g = queue.pop(0)
        l_ = None if cls_only else queue.pop(0)
        return two_branch(global_feat, sd, T, context_feat, fc_dim, pool_size, cls_only, return_logits, (g, l_), p)
    monkeypatch.setattr(om, "two_branch", patched)
    return queue
