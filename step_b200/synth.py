"""Synthetic, seed-deterministic inputs for the STEP hot path (SURVEY.md section 8d).

There is no dataset or checkpoint offline, so parity tests and the benchmark use:
  * state dicts with the reference's key names (networks.py:107-132, two_branch.py:164-203) --
    He-normal conv weights, randomised BatchNorm statistics (the default init collapses
    activations to ~2e-5 and makes tolerances meaningless, SURVEY.md section 4);
  * clips ~ clamp(randn, -1, 1)  (the reference's scale_norm=2 input range, augmentations.py:80-82);
  * N grid proposals per clip built like data/data_utils.py:19-45 plus a centre and a full box.

The data is host-side numpy/torch-CPU generation; device_nets and make_workload load it into the nets and move them and
the step's inputs to a device, so that the benchmark tools and the training tests run the same workloads.
"""
import math
from collections import namedtuple
from types import SimpleNamespace

import numpy as np
import torch

from .networks import BaseNet, ROINet
from .tube_utils import flatten_tubes
from .two_branch import ContextNet, TwoBranchNet

# (in_channels, [b0, b1a, b1b, b2a, b2b, b3]) -- i3dpt.py:213-231
MIXED_PLAN = {
    "3b": (192, [64, 96, 128, 16, 32, 32]), "3c": (256, [128, 128, 192, 32, 96, 64]),
    "4b": (480, [192, 96, 208, 16, 48, 64]), "4c": (512, [160, 112, 224, 24, 64, 64]),
    "4d": (512, [128, 128, 256, 24, 64, 64]), "4e": (512, [112, 144, 288, 32, 64, 64]),
    "4f": (528, [256, 160, 320, 32, 128, 128]),
    "5b": (832, [256, 160, 320, 32, 128, 128]), "5c": (832, [384, 192, 384, 48, 128, 128]),
}
# position in BaseNet.base_model (nn.Sequential, networks.py:120-132)
TRUNK_MIXED = {5: "3b", 6: "3c", 8: "4b", 9: "4c", 10: "4d", 11: "4e", 12: "4f"}


def make_cfg(**kw):
    """The cfg attributes the ported modules read (SURVEY.md section 8b), C4 defaults."""
    d = dict(base_net="i3d", kinetics_pretrain=None, freeze_stats=True, freeze_affine=True, fp16=False,
             num_classes=60, T=8, fc_dim=256, dropout=0.3, pool_size=7, pool_mode="align",
             no_context=True, max_iter=3, temporal_mode="predict", NUM_CHUNKS={1: 1, 2: 1, 3: 1},
             image_size=(224, 224))
    d.update(kw)
    return SimpleNamespace(**d)


def _conv(g, sd, key, cout, cin, k, bias=False, std=None):
    fan_in = cin * int(np.prod(k))
    std = math.sqrt(2.0 / fan_in) if std is None else std
    sd[key + ".weight"] = torch.randn((cout, cin) + tuple(k), generator=g) * std
    if bias:
        sd[key + ".bias"] = torch.randn(cout, generator=g) * 0.1


def _bn(g, sd, key, c):
    sd[key + ".weight"] = torch.rand(c, generator=g) * 0.4 + 0.8
    sd[key + ".bias"] = torch.randn(c, generator=g) * 0.1
    sd[key + ".running_mean"] = torch.randn(c, generator=g) * 0.1
    sd[key + ".running_var"] = torch.rand(c, generator=g) + 0.5
    sd[key + ".num_batches_tracked"] = torch.tensor(0, dtype=torch.long)


def _unit(g, sd, p, cin, cout, k):
    _conv(g, sd, p + "conv3d", cout, cin, k)
    _bn(g, sd, p + "batch3d", cout)


def _mixed(g, sd, p, name):
    cin, o = MIXED_PLAN[name]
    _unit(g, sd, p + "branch_0.", cin, o[0], (1, 1, 1))
    _unit(g, sd, p + "branch_1.0.", cin, o[1], (1, 1, 1))
    _unit(g, sd, p + "branch_1.1.", o[1], o[2], (3, 3, 3))
    _unit(g, sd, p + "branch_2.0.", cin, o[3], (1, 1, 1))
    _unit(g, sd, p + "branch_2.1.", o[3], o[4], (3, 3, 3))
    _unit(g, sd, p + "branch_3.1.", cin, o[5], (1, 1, 1))


def base_net_state_dict(seed=1234):
    """Keys of BaseNet.state_dict() (networks.py:50-67, 120-132): base_model.{0..12}.*"""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    _unit(g, sd, "base_model.0.", 3, 64, (7, 7, 7))
    _unit(g, sd, "base_model.2.", 64, 64, (1, 1, 1))
    _unit(g, sd, "base_model.3.", 64, 192, (3, 3, 3))
    for idx, name in TRUNK_MIXED.items():
        _mixed(g, sd, "base_model.%d." % idx, name)
    return sd


def context_net_state_dict(seed=4321):
    """Keys of ContextNet.state_dict() (two_branch.py:113-130): i3d_conv_context.{1,2}.*"""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    _mixed(g, sd, "i3d_conv_context.1.", "5b")
    _mixed(g, sd, "i3d_conv_context.2.", "5c")
    return sd


def head_state_dict(seed, cfg, reg_std=5e-5, cls_std=2e-3):
    """Keys of TwoBranchNet.state_dict() (two_branch.py:164-203).

    The regressor / classifier weights get a small fixed std instead of the reference's
    xavier-normal init (two_branch.py:344-353): with He-scaled features xavier makes every
    delta O(10) -> exp() saturates -> all tubes collapse to the whole-image box in
    valid_tubes, which would make the progressive loop a degenerate test."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    _mixed(g, sd, "i3d_conv.0.", "5b")
    _mixed(g, sd, "i3d_conv.1.", "5c")
    fc, ps = cfg.fc_dim, cfg.pool_size
    D = fc * ps * ps
    _conv(g, sd, "downsample", fc, 1024, (1, 1, 1), bias=True)
    _conv(g, sd, "global_cls", cfg.num_classes, D + (0 if cfg.no_context else 1024), (1, 1, 1),
          bias=True, std=cls_std)
    _conv(g, sd, "local_conv.0.conv1", 1024, 832 + fc, (1, 1))
    _conv(g, sd, "local_conv.0.conv2", 256, 832 + fc, (1, 1))
    _conv(g, sd, "local_conv.0.conv3", 256, 256, (3, 3))
    _conv(g, sd, "local_conv.0.conv4", 1024, 256, (1, 1))
    for i in (1, 2):
        _conv(g, sd, "local_conv.%d.conv1" % i, 256, 1024, (1, 1))
        _conv(g, sd, "local_conv.%d.conv2" % i, 256, 256, (3, 3))
        _conv(g, sd, "local_conv.%d.conv3" % i, 1024, 256, (1, 1))
    _conv(g, sd, "downsample2", fc, 1024, (1, 1), bias=True)
    for name in ("local_reg", "neighbor_reg1", "neighbor_reg2"):
        sd[name + ".weight"] = torch.randn(4, D, generator=g) * reg_std
        sd[name + ".bias"] = torch.randn(4, generator=g) * 0.02
    return sd


CLS_HEAD_PREFIXES = ("i3d_conv.", "downsample.", "global_cls.")


def cls_head_state_dict(seed, cfg, **kw):
    """Keys of TwoBranchNet(cfg, cls_only=True).state_dict() (two_branch.py:181-189): head_state_dict without the local
    branch, so the shared tensors equal those of the full head of the same seed."""
    return {k: v for k, v in head_state_dict(seed, cfg, **kw).items() if k.startswith(CLS_HEAD_PREFIXES)}


def make_clips(B, T_in, H, W, seed=1234):
    """[B, T_in, 3, H, W] fp32 in [-1, 1] (the layout BaseNet.forward takes, networks.py:69-76)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, T_in, 3, H, W, generator=g).clamp_(-1.0, 1.0)


def grid_anchors(scales=(4.0 / 3.0,), steps=(5.0 / 6.0,)):
    """Normalised grid anchors in the spirit of data/data_utils.py:19-45: for each (scale, step),
    boxes of side 1/scale... laid on a regular grid; here one scale -> 3x3 = 9 boxes."""
    out = []
    for s, st in zip(scales, steps):
        side = 1.0 / s
        n = 3
        for iy in range(n):
            for ix in range(n):
                cx = 0.5 + (ix - 1) * (1.0 - side) / 2.0 * st * 1.2
                cy = 0.5 + (iy - 1) * (1.0 - side) / 2.0 * st * 1.2
                out.append([max(cx - side / 2, 0.0), max(cy - side / 2, 0.0),
                            min(cx + side / 2, 1.0), min(cy + side / 2, 1.0)])
    return np.asarray(out, dtype=np.float32)


def make_proposals(B, N, T, W, H):
    """list (len B) of [N, T, 4] fp32 tubes in input pixels: 9 grid anchors + centre + full frame,
    cycled / truncated to N, replicated over T frames (the reference tiles anchors over T,
    data/ava.py:343-345)."""
    base = np.concatenate([grid_anchors(),
                           np.array([[0.25, 0.25, 0.75, 0.75], [0.0, 0.0, 1.0, 1.0]], np.float32)], 0)
    idx = np.arange(N) % base.shape[0]
    boxes = base[idx] * np.array([W, H, W, H], np.float32)
    jit = (np.arange(N) // base.shape[0]).astype(np.float32)[:, None] * 3.0  # distinct if N > 11
    boxes = boxes + jit * np.array([1, 1, -1, -1], np.float32)
    tubes = np.tile(boxes[:, None, :], (1, T, 1)).astype(np.float32)
    return [tubes.copy() for _ in range(B)]


def make_c3_rois(n_tubes=10000, n_clips=8, Tp=8, W=224, seed=0):
    """BASELINE config 3: random tubes -> flat ROI rows [n_tubes*Tp, 5] (frame index b*Tp+t first)
    and the per-tube boxes [n_tubes, 4] used for the NMS microbench (SURVEY.md section 8d)."""
    rs = np.random.RandomState(seed)
    x1 = rs.uniform(0, 0.67 * W, n_tubes)
    y1 = rs.uniform(0, 0.67 * W, n_tubes)
    w = rs.uniform(0.09 * W, 0.54 * W, n_tubes)
    h = rs.uniform(0.09 * W, 0.54 * W, n_tubes)
    boxes = np.stack([x1, y1, np.minimum(x1 + w, W - 1), np.minimum(y1 + h, W - 1)], 1).astype(np.float32)
    clip = rs.randint(0, n_clips, n_tubes)
    frame = (clip[:, None] * Tp + np.arange(Tp)[None, :]).astype(np.float32)
    rois = np.concatenate([frame[:, :, None], np.tile(boxes[:, None, :], (1, Tp, 1))], 2).reshape(-1, 5)
    scores = rs.rand(n_tubes).astype(np.float32)
    return rois.astype(np.float32), boxes, scores


LOSS_CASES = {"c1": (3, 1, 5, "mixed"), "c3": (3, 3, 4, "mixed"), "nomask": (3, 1, 3, "zero")}


def make_loss_case(name, num_classes):
    """Seeded inputs of the training-time head call `TwoBranchNet.forward(feat, None, tubes=..., targets=...)`
    (two_branch.py:205-341): (T, feat [n,T',832,7,7], tubes [n,T',5], targets [n,3,6+cls]).  Shared by
    tests/golden/make_golden.py (reference run) and the oracle test."""
    T_, chunks, n, masks = LOSS_CASES[name]
    g = torch.Generator().manual_seed(77 + n)
    Tl = T_ * chunks
    feat = torch.randn(n, Tl, 832, 7, 7, generator=g) * 0.5
    x1 = torch.rand(n, Tl, generator=g) * 50
    y1 = torch.rand(n, Tl, generator=g) * 50
    w = 20 + torch.rand(n, Tl, generator=g) * 40
    h = 20 + torch.rand(n, Tl, generator=g) * 40
    tubes = torch.stack([torch.zeros(n, Tl), x1, y1, x1 + w, y1 + h], dim=2)
    tg = torch.zeros(n, 3, 6 + num_classes)
    gx1 = torch.rand(n, 3, generator=g) * 50
    gy1 = torch.rand(n, 3, generator=g) * 50
    tg[:, :, 0] = gx1
    tg[:, :, 1] = gy1
    tg[:, :, 2] = gx1 + 15 + torch.rand(n, 3, generator=g) * 45
    tg[:, :, 3] = gy1 + 15 + torch.rand(n, 3, generator=g) * 45
    if masks == "mixed":
        tg[:, :, 4] = (torch.rand(n, 3, generator=g) > 0.3).float()
        tg[:, :, 5] = (torch.rand(n, 3, generator=g) > 0.4).float()
        tg[0, :, 4] = 1.0
        tg[0, :, 5] = 1.0
    tg[:, :, 6:] = (torch.rand(n, 3, num_classes, generator=g) > 0.9).float()
    return T_, chunks, feat, tubes, tg


def make_train_case(cfg, B, N, W, H, seed=3):
    """Seeded selected samples of one training step (what train_select, utils/utils.py:135-423, hands to train.py:300-333)
    for refinement steps 1..cfg.max_iter: (step_tubes, step_targets), step_tubes[i] [B*N, T_length_i, 5] fp32 with the
    frame index relative to the step's frame slice first (flatten_tubes(batch_idx=True)), step_targets[i]
    [B*N, 3, 6 + classes].  Boxes lie inside a W x H image; every step has positive class and regression samples."""
    g = torch.Generator().manual_seed(seed)
    step_tubes, step_targets = [], []
    for i in range(1, cfg.max_iter + 1):
        t_len = cfg.NUM_CHUNKS[i] * cfg.T
        R = B * N
        x1 = torch.rand(R, 1, generator=g) * 0.3 * W
        y1 = torch.rand(R, 1, generator=g) * 0.3 * H
        w = (0.3 + torch.rand(R, 1, generator=g) * 0.3) * W
        hh = (0.3 + torch.rand(R, 1, generator=g) * 0.3) * H
        box = torch.cat([x1, y1, x1 + w, y1 + hh], 1)
        frame = (torch.arange(R) // N).view(R, 1, 1) * t_len + torch.arange(t_len).view(1, t_len, 1)
        jit = torch.rand(R, t_len, 4, generator=g) * 0.02 * W
        tubes = torch.cat([frame.float(), box.view(R, 1, 4).expand(R, t_len, 4) + jit], 2)
        tg = torch.zeros(R, 3, 6 + cfg.num_classes)
        tg[:, :, :4] = box.view(R, 1, 4) + torch.rand(R, 3, 4, generator=g) * 0.06 * W
        tg[:, :, 4] = (torch.rand(R, 3, generator=g) > 0.3).float()
        tg[:, :, 5] = (torch.rand(R, 3, generator=g) > 0.3).float()
        tg[0, :, 4:6] = 1.0
        tg[:, :, 6:] = (torch.rand(R, 3, cfg.num_classes, generator=g) > 0.9).float()
        step_tubes.append(tubes.contiguous())
        step_targets.append(tg)
    return step_tubes, step_targets


def make_cls_case(cfg, B, N, W, H, seed=3):
    """Seeded samples of one step of the classification pre-training stage, shaped as train_cls.py:260-297 builds them:
    (flat_tubes [B*N, cfg.T, 5] fp32 with the frame index b * T + t first (flatten_tubes(batch_idx=True)), flat_targets
    [B*N, 3, 6 + classes]).  Each clip has min(5, (N + 3) // 4) positives (select_proposals(..., 0.75, 5, 'uniform', 3)
    keeps at most 5) followed by negatives; with B > 1 the last clip has negatives only.  A positive row holds its ground
    truth box in columns :4 and its labels in 6:; every row has the classification flag (column 4) set and none the
    regression flag (column 5); the one target frame is tiled three times.  Boxes lie inside a W x H image."""
    g = torch.Generator().manual_seed(seed)
    T_, C = cfg.T, cfg.num_classes
    n_pos = min(5, (N + 3) // 4)
    tubes, targets = [], []
    for b in range(B):
        pos = 0 if (B > 1 and b == B - 1) else n_pos
        x1 = torch.rand(N, 1, generator=g) * 0.4 * W
        y1 = torch.rand(N, 1, generator=g) * 0.4 * H
        w = (0.2 + torch.rand(N, 1, generator=g) * 0.35) * W
        hh = (0.2 + torch.rand(N, 1, generator=g) * 0.35) * H
        box = torch.cat([x1, y1, x1 + w, y1 + hh], 1)
        jit = torch.rand(N, T_, 4, generator=g) * 0.02 * W
        frame = (b * T_ + torch.arange(T_, dtype=torch.float32)).view(1, T_, 1).expand(N, T_, 1)
        tubes.append(torch.cat([frame, box.view(N, 1, 4) + jit], 2))
        tg = torch.zeros(N, 1, 6 + C)
        if pos:
            tg[:pos, 0, :4] = box[:pos] + (torch.rand(pos, 4, generator=g) - 0.5) * 0.04 * W
            lab = (torch.rand(pos, C, generator=g) > 0.9).float()
            lab[torch.arange(pos), torch.randint(0, C, (pos,), generator=g)] = 1.0
            tg[:pos, 0, 6:] = lab
        tg[:, 0, 4] = 1.0
        targets.append(tg.repeat(1, 3, 1))
    return torch.cat(tubes).contiguous(), torch.cat(targets).contiguous()


def _on(net, device):
    net = net.to(device).eval()
    if hasattr(net, "set_device"):
        net.set_device(device)
    return net


def device_head(cfg, sd, cls_only=False, device="cuda:0"):
    """TwoBranchNet(cfg, cls_only) loaded with sd, on device in eval mode."""
    h = TwoBranchNet(cfg, cls_only=cls_only)
    h.load_state_dict(sd, strict=True)
    return _on(h, device)


def device_nets(cfg, heads_sd, pool_mode="align", context=False, cls_only=False, device="cuda:0"):
    """The nets dict of train_step and inference on device in eval mode: the synthetic trunk, ROINet(pool_mode, 7), with
    context the synthetic ContextNet, and one head det_net<i> per state dict of heads_sd."""
    nets = {"base_net": BaseNet(cfg), "roi_net": ROINet(pool_mode, 7)}
    nets["base_net"].load_state_dict(base_net_state_dict(), strict=True)
    if context:
        nets["context_net"] = ContextNet(cfg)
        nets["context_net"].load_state_dict(context_net_state_dict(), strict=True)
    nets = {k: _on(net, device) for k, net in nets.items()}
    for i, sd in enumerate(heads_sd):
        nets["det_net%d" % i] = device_head(cfg, sd, cls_only, device)
    return nets


# The named training workloads: make_cfg keywords, B clips of T_in x HW x HW and N tubes per clip.  The tools time them
# by name, so that numbers taken by different tools are numbers of the same step.
#   c4       BASELINE.json config 4 (bench.py's batch) trained: 3 spatial steps of T'=8, no context
#   shipped  scripts/train_step.sh: T=3, temporal mode (NUM_CHUNKS {1:1, 2:1, 3:3}: steps of 3, 3 and 9 frames),
#            context on
#   cls      scripts/train_cls.sh, the classification pre-training stage: one class-only head over T=9 frames,
#            context on
Workload = namedtuple("Workload", "cfg B N T_in HW")
WORKLOADS = {
    "c4": Workload(dict(T=8, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 1}), B=8, N=11, T_in=32, HW=224),
    "shipped": Workload(dict(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False),
                        B=2, N=34, T_in=36, HW=400),
    "cls": Workload(dict(T=9, max_iter=1, NUM_CHUNKS={1: 1}, no_context=False), B=4, N=20, T_in=36, HW=400),
}


def make_workload(name, fp16=True, pool_mode="align", B=None, device="cuda:0", **cfg_kw):
    """One training step of WORKLOADS[name] on device: (cfg, nets, clips, step_tubes, step_targets).  cfg takes the
    workload's keywords, fp16, pool_mode and cfg_kw (e.g. dropout=0.3, freeze_affine=False); nets are device_nets with
    ContextNet where the workload has context and heads seeded 100 + i (cls: one class-only head); B defaults to the
    workload's.  The samples are make_cls_case's (cls), make_train_case's (shipped), or for c4 the grid proposals of
    every clip with seeded targets, the same rows at every step."""
    w = WORKLOADS[name]
    B = w.B if B is None else B
    cfg = make_cfg(fp16=fp16, pool_mode=pool_mode, image_size=(w.HW, w.HW), **w.cfg, **cfg_kw)
    cls = name == "cls"
    heads = [cls_head_state_dict(100, cfg)] if cls else [head_state_dict(100 + i, cfg) for i in range(cfg.max_iter)]
    nets = device_nets(cfg, heads, pool_mode, context=not cfg.no_context, cls_only=cls, device=device)
    clips = make_clips(B, w.T_in, w.HW, w.HW).to(device)
    if cls:
        tubes, targets = make_cls_case(cfg, B, w.N, w.HW, w.HW)
        step_tubes, step_targets = [tubes], [targets]
    elif name == "shipped":
        step_tubes, step_targets = make_train_case(cfg, B, w.N, w.HW, w.HW)
    else:
        R = B * w.N
        tubes = torch.from_numpy(flatten_tubes(make_proposals(B, w.N, cfg.T, w.HW, w.HW), batch_idx=True)[0])
        g = torch.Generator().manual_seed(0)
        tg = torch.zeros(R, 3, 6 + cfg.num_classes)
        tg[:, :, :4] = tubes[:, 4:5, 1:] + torch.rand(R, 3, 4, generator=g) * 6
        tg[:, :, 4:6] = (torch.rand(R, 3, 2, generator=g) > 0.3).float()
        tg[0, :, 4:6] = 1
        tg[:, :, 6:] = (torch.rand(R, 3, cfg.num_classes, generator=g) > 0.9).float()
        step_tubes, step_targets = [tubes] * cfg.max_iter, [tg] * cfg.max_iter
    return cfg, nets, clips, [t.to(device) for t in step_tubes], [t.to(device) for t in step_targets]


def make_conv_feat(B, T, H, W, seed=2468):
    """A seeded stand-in for the trunk's output [B, T', 832, H', W'] (post-ReLU: non-negative)."""
    g = torch.Generator().manual_seed(seed)
    return torch.relu(torch.randn(B, T, 832, H, W, generator=g))

