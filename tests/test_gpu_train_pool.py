"""GPU: training with ROIPool (ROINet('pool', 7), the reference's default pool_mode, config.py:67): the argmax forward
(step_roi_pool_fwd_argmax_nhwc) and the deterministic ROIPool backward on a frame slice (step_roi_pool_bwd_slice_nhwc)
against torchvision's CPU roi_pool (tests/golden/roi_cross_cases.npz holds its outputs on the golden ROI case), the routing
inside train_step, and train_step end to end against the oracle's torch-CPU autograd with torchvision's roi_pool in place of
roi_align, in the three configurations the ROIAlign tests cover.

The backward sums every element's contributions in ascending (ROI row, ph, pw) order, the loop order of torchvision's CPU
backward, so fp32 results are compared bit for bit.  End to end, the tolerances are those of the ROIAlign tests
(tests/test_gpu_train.py, tests/test_gpu_train_context.py, tests/test_gpu_train_cls.py); max pooling adds one effect the
bilinear pooling does not have -- the fp16 trunk can reorder two near-equal values and route a gradient to another pixel --
and each case counts those argmax flips against the fp32 oracle and bounds them."""
import os
import sys

import numpy as np
import pytest
import torch
from torchvision.ops import roi_pool as tv_roi_pool

from oracle import model as om
from step_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_oracle_cls  # noqa: E402
import test_oracle_context  # noqa: E402
from _train_case import SHIPPED, compare_grads, spatial_case, trainable  # noqa: E402
from step_b200.synth import device_nets  # noqa: E402

pytestmark = pytest.mark.gpu


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def pool(feat, rois, ph=7, pw=7, roi_T=0, feat_T=0, t_start=0):
    """feat [K,H,W,C] (fp32 | fp16, CUDA) -> (pooled [R,ph,pw,C], argmax [R,ph,pw,C] int32, pooled by step_roi_pool_fwd_nhwc)."""
    from step_b200 import _lib as L
    K, H, W, C = feat.shape
    R = rois.shape[0]
    out = torch.full((R, ph, pw, C), 7.0, dtype=feat.dtype, device="cuda")
    plain = torch.full_like(out, 7.0)
    am = torch.full((R, ph, pw, C), -7, dtype=torch.int32, device="cuda")
    args = (L.ptr(feat), L.dt(feat), K, H, W, C, C, L.ptr(rois), R, 1.0 / 16.0, ph, pw)
    L.check(L.lib().step_roi_pool_fwd_argmax_nhwc(*args, L.ptr(out), C, roi_T, feat_T, t_start, L.ptr(am), L.stream()))
    L.check(L.lib().step_roi_pool_fwd_nhwc(*args, L.ptr(plain), C, roi_T, feat_T, t_start, L.stream()))
    return out, am, plain


def backward(gy, rois, am, gin, roi_T, feat_T, t_start):
    """gin [K,H,W,C] fp32 += ROIPool backward of gy [R,ph,pw,C] through am (training.roi_pool_backward_slice)."""
    from step_b200 import training
    from step_b200.engine import Act
    R, ph, pw, C = gy.shape
    training.roi_pool_backward_slice(Act(gy.contiguous().view(R, 1, ph, pw, C)), rois, am, gin, roi_T, feat_T, t_start)
    return gin


def tv_backward(x_nchw, rois, gy_nchw, ph=7, pw=7):
    """torchvision's CPU roi_pool forward and backward: (pooled, argmax, d input) in NCHW."""
    x = x_nchw.detach().cpu().float().clone().requires_grad_(True)
    y = tv_roi_pool(x, rois.cpu(), (ph, pw), 1.0 / 16.0)
    y.backward(gy_nchw.cpu().float())
    _, am = torch.ops.torchvision.roi_pool(x.detach(), rois.cpu(), 1.0 / 16.0, ph, pw)
    return y.detach(), am, x.grad


nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()
nchw = lambda t: t.permute(0, 3, 1, 2).contiguous()


def golden_map(a, C=8):
    """The golden case's [3,5,14,14] map, channels-last and padded to whole 16-byte vectors with zero channels."""
    K, C0, H, W = a["feat"].shape
    f = np.zeros((K, H, W, C), np.float32)
    f[..., :C0] = a["feat"].transpose(0, 2, 3, 1)
    return cu(f), C0


# ---- 1. forward -------------------------------------------------------------------------------------------------------
def test_forward_matches_plain_entry_golden_and_torchvision_argmax(golden):
    g, a = golden("roi_cross_cases"), golden("roi_align_cases")
    feat, C0 = golden_map(a)
    rois = cu(a["rois"])
    out, am, plain = pool(feat, rois)
    assert torch.equal(out, plain)
    assert np.array_equal(out.cpu().numpy().transpose(0, 3, 1, 2)[:, :C0], g["pool_out"])
    ty, tam, _ = tv_backward(nchw(feat), rois, torch.zeros(48, 8, 7, 7))
    assert torch.equal(out.cpu(), nhwc(ty)) and torch.equal(am.cpu(), nhwc(tam))
    assert int((am == -1).sum()) > 0                                   # the case has empty bins
    # fp16 storage: torchvision on the fp16-rounded map (ties then resolve identically)
    fh = feat.half()
    outh, amh, plainh = pool(fh, rois)
    assert torch.equal(outh, plainh)
    ty, tam, _ = tv_backward(nchw(fh.float()), rois, torch.zeros(48, 8, 7, 7))
    assert torch.equal(outh.float().cpu(), nhwc(ty)) and torch.equal(amh.cpu(), nhwc(tam))


def test_forward_ties_go_to_the_first_pixel_in_scan_order():
    gen = torch.Generator().manual_seed(21)
    feat = torch.randint(-1, 2, (2, 9, 11, 16), generator=gen).float()       # values in {-1, 0, 1}: ties everywhere
    rois = torch.tensor([[0, 0, 0, 170, 140], [1, 20, 30, 100, 60], [1, -30, -30, 400, 400], [0, 50, 50, 50, 50.]])
    for dt in (torch.float32, torch.float16):
        out, am, plain = pool(feat.to(dt).cuda(), rois.cuda())
        ty, tam, _ = tv_backward(nchw(feat), rois, torch.zeros(4, 16, 7, 7))
        assert torch.equal(out, plain) and torch.equal(out.float().cpu(), nhwc(ty)) and torch.equal(am.cpu(), nhwc(tam))


# ---- 2. backward, exact -----------------------------------------------------------------------------------------------
def test_backward_is_bit_identical_to_torchvision_and_repeatable(golden):
    g, a = golden("roi_cross_cases"), golden("roi_align_cases")
    feat, C0 = golden_map(a)
    K, H, W, C = feat.shape
    rois = cu(a["rois"])
    _, am, _ = pool(feat, rois)
    gy = np.zeros((48, 7, 7, C), np.float32)
    gy[..., :C0] = g["pool_gy"].transpose(0, 2, 3, 1)
    gy = cu(gy)
    gin = backward(gy, rois, am, torch.zeros(K, H, W, C, device="cuda"), K, K, 0)
    assert np.array_equal(gin.cpu().numpy().transpose(0, 3, 1, 2)[:, :C0], g["pool_gx"])
    assert float(gin[..., C0:].abs().max()) == 0.0
    again = backward(gy, rois, am, torch.zeros(K, H, W, C, device="cuda"), K, K, 0)
    assert torch.equal(again, gin)


# ---- 3. slice semantics -----------------------------------------------------------------------------------------------
def slice_case(C=16, H=10, W=12, N=4, B=2, seed=5):
    cfg = synth.make_cfg(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False)
    tubes = synth.make_train_case(cfg, B, N, 16 * W, 16 * H, seed=seed)[0][0]      # [B*N, 3, 5], frames of the 3-frame slice
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B * 9, H, W, C, generator=gen)
    return B, x, tubes, gen


def test_backward_slice_adds_the_torchvision_backward_and_leaves_other_frames():
    import step_b200
    from step_b200 import _lib as L
    from step_b200.engine import Act
    B, x, tubes, gen = slice_case()
    _, H, W, C = x.shape
    R = tubes.shape[0] * 3
    y = Act.empty(R, 1, 7, 7, C, L.F32, torch.device("cuda", 0))
    am = torch.empty(R * 49 * C, dtype=torch.int32, device="cuda")
    step_b200.ROINet("pool", 7).pool_into(Act(x.view(B, 9, H, W, C).cuda()), tubes.cuda(), y, 3, 9, 3, argmax=am)
    g = torch.randn(R, 7, 7, C, generator=gen)
    init = torch.randn(B * 9, H, W, C, generator=gen)
    acc = backward(g.cuda(), tubes.view(-1, 5).cuda(), am, init.clone().cuda(), 3, 9, 3).cpu()
    a, b = acc.view(B, 9, H, W, C), init.view(B, 9, H, W, C)
    assert torch.equal(a[:, :3], b[:, :3]) and torch.equal(a[:, 6:], b[:, 6:])
    xs = x.view(B, 9, H, W, C)[:, 3:6].reshape(B * 3, H, W, C)
    ty, tam, tgx = tv_backward(nchw(xs), tubes.view(-1, 5), nchw(g))
    assert torch.equal(y.buf.view(R, 7, 7, C).cpu(), nhwc(ty)) and torch.equal(am.view(R, 7, 7, C).cpu(), nhwc(tam))
    assert torch.equal(a[:, 3:6], b[:, 3:6] + nhwc(tgx).view(B, 3, H, W, C))
    # adjoint: <pool(x), g> == <x, bwd(g)>
    gin = backward(g.cuda(), tubes.view(-1, 5).cuda(), am, torch.zeros(B * 9, H, W, C, device="cuda"), 3, 9, 3).cpu()
    lhs = float((y.buf.cpu().double().view(-1) * g.double().view(-1)).sum())
    rhs = float((x.double() * gin.double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * max(1.0, abs(lhs))


def test_backward_at_the_shipped_shape_from_fp16_gradients():
    """25x25x832 maps (36x400x400 input), 34 tubes per clip over all 9 frames, fp16 gradients with a channel stride (the
    [ROI | downsample] concat buffer of train_step): 64-channel chunks, bit-identical to torchvision on the same values."""
    from step_b200.engine import Act
    from step_b200 import training
    cfg = synth.make_cfg(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False)
    B, H, W, C = 2, 25, 25, 832
    tubes = synth.make_train_case(cfg, B, 34, 400, 400, seed=8)[0][2]             # [68, 9, 5]
    x = synth.make_conv_feat(B, 9, H, W).reshape(B * 9, C, H, W)
    R = tubes.shape[0] * 9
    gen = torch.Generator().manual_seed(1)
    _, am, _ = pool(nhwc(x).half().cuda(), tubes.view(-1, 5).cuda(), roi_T=9, feat_T=9, t_start=0)
    gcat = (torch.randn(R, 7, 7, C + 256, generator=gen) * 100).half()
    gin = torch.zeros(B * 9, H, W, C, device="cuda")
    training.roi_pool_backward_slice(Act(gcat.cuda().view(R, 1, 7, 7, C + 256), C, 0), tubes.view(-1, 5).cuda(), am, gin, 9, 9, 0)
    _, tam, tgx = tv_backward(x.half().float(), tubes.view(-1, 5), nchw(gcat[..., :C].float()))
    assert torch.equal(am.cpu(), nhwc(tam))
    assert torch.equal(gin.cpu(), nhwc(tgx))


# ---- 4. edge cases ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", [(7, 7), (3, 5), (1, 1)])
def test_edge_cases_match_torchvision(size):
    """Empty bins (argmax -1, no contribution), ROIs partly and wholly outside the map, 1-pixel ROIs, 40 ROIs on one frame
    (several row batches of the block compaction at 8-channel chunks), a frame without ROIs, R = 0, pooled sizes != 7."""
    ph, pw = size
    gen = torch.Generator().manual_seed(ph * 10 + pw)
    K, H, W, C = 4, 6, 5, 8
    feat = torch.randint(-2, 3, (K, H, W, C), generator=gen).float() + torch.rand(K, H, W, C, generator=gen) * 0.5
    rows = [[0, -50, -50, 40, 40], [1, 500, 500, 600, 600], [2, 16, 16, 16, 16], [1, -100, 10, -60, 40], [2, 0, 0, 79, 95]]
    for i in range(40):
        x0, y0 = float(torch.randint(-20, 70, (1,), generator=gen)), float(torch.randint(-20, 90, (1,), generator=gen))
        rows.append([0, x0, y0, x0 + float(torch.randint(0, 60, (1,), generator=gen)), y0 + float(torch.randint(0, 60, (1,), generator=gen))])
    rois = torch.tensor(rows, dtype=torch.float32)
    R = rois.shape[0]
    out, am, plain = pool(feat.cuda(), rois.cuda(), ph, pw)
    gy = torch.randn(R, ph, pw, C, generator=gen)
    ty, tam, tgx = tv_backward(nchw(feat), rois, nchw(gy), ph, pw)
    assert torch.equal(out, plain) and torch.equal(out.cpu(), nhwc(ty)) and torch.equal(am.cpu(), nhwc(tam))
    assert bool((am[1] == -1).all()) and bool((out[1] == 0).all())           # wholly outside: every bin empty
    init = torch.randn(K, H, W, C, generator=gen)
    gin = backward(gy.cuda(), rois.cuda(), am, init.clone().cuda(), K, K, 0).cpu()
    assert torch.equal(gin[3], init[3])                                       # no ROI on frame 3: untouched
    gin0 = backward(gy.cuda(), rois.cuda(), am, torch.zeros(K, H, W, C, device="cuda"), K, K, 0).cpu()
    assert torch.equal(gin0, nhwc(tgx))
    # R = 0: nothing pooled, nothing added
    empty = torch.zeros(0, 5, device="cuda")
    out0, _, _ = pool(feat.cuda(), empty, ph, pw)
    assert out0.numel() == 0
    again = init.clone().cuda()
    backward(torch.zeros(0, ph, pw, C, device="cuda"), empty, torch.zeros(0, dtype=torch.int32, device="cuda"), again, K, K, 0)
    assert torch.equal(again.cpu(), init)


# ---- 5. routing inside train_step -------------------------------------------------------------------------------------
def test_train_step_feeds_the_trunk_the_roi_pool_backward(monkeypatch):
    """The conv_feat gradient train_step hands to the trunk is torchvision's CPU ROIPool backward of the step's own fp16
    conv_feat, its pooled-feature gradients and its tubes (summed over the steps, divided by the loss scale)."""
    from step_b200 import training
    cfg, x, step_tubes, step_targets = spatial_case()
    nets = device_nets(cfg, [synth.head_state_dict(100 + i, cfg) for i in range(2)], "pool")
    cap = {"roi_grad": []}
    head_fb, trunk_fb = training.head_forward_backward, training.trunk_forward_backward

    def head_spy(*a, **k):
        r = head_fb(*a, **k)
        g = r["roi_grad"]
        cap["roi_grad"].append(g.buf[..., g.coff:g.coff + g.C].float().cpu())
        return r

    def trunk_spy(base_net, clips, d_feat_fn, loss_scale=1024.0):
        def d(feat):
            out = d_feat_fn(feat)
            cap["feat"] = feat.buf[..., feat.coff:feat.coff + feat.C].float().cpu()
            cap["d"] = out.float().cpu()
            cap["scale"] = loss_scale
            return out
        return trunk_fb(base_net, clips, d, loss_scale)
    monkeypatch.setattr(training, "head_forward_backward", head_spy)
    monkeypatch.setattr(training, "trunk_forward_backward", trunk_spy)
    training.train_step(cfg, nets, x.cuda(), [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets])
    torch.cuda.synchronize()
    feat = cap["feat"]                                                    # [B, T', H', W', 832]
    B, Tp, H, W, C = feat.shape
    total = torch.zeros(B, Tp, H, W, C)
    for i, (tubes, rg) in enumerate(zip(step_tubes, cap["roi_grad"])):
        t0, tl = training.step_frames(cfg, i + 1)
        xs = nchw(feat[:, t0:t0 + tl].reshape(B * tl, H, W, C))
        _, _, gx = tv_backward(xs, tubes.reshape(-1, 5), nchw(rg.reshape(-1, 7, 7, C)))
        total[:, t0:t0 + tl] += nhwc(gx).view(B, tl, H, W, C)
    ref = total * (1.0 / cap["scale"])
    assert float(ref.abs().max()) > 0
    assert torch.allclose(cap["d"], ref, rtol=1e-6, atol=1e-12), float((cap["d"] - ref).abs().max())


# ---- 6. end to end against the oracle ---------------------------------------------------------------------------------
def pool_as_align(fm, rois, size, scale, sampling_ratio=0, aligned=False):
    """torchvision's roi_pool behind the oracle objectives' ROIAlign call."""
    return tv_roi_pool(fm, rois, size, scale)


def argmax_flips(nets, x, cf, cfg, step_tubes):
    """(elements whose device argmax differs from the fp32 oracle's, positive-valued ones of those, total) over every step."""
    from step_b200 import _lib as L
    from step_b200.engine import Act
    from step_b200 import training
    with torch.no_grad():
        feat = nets["base_net"].forward_act(x.cuda())
    B, Tp = cf.shape[0], cf.shape[1]
    flips = pos = total = 0
    for i, tubes in enumerate(step_tubes):
        t0, tl = training.step_frames(cfg, i + 1)
        R = tubes.shape[0] * tl
        out = Act.empty(R, 1, 7, 7, 832, L.F16, torch.device("cuda", 0))
        am = torch.empty(R * 49 * 832, dtype=torch.int32, device="cuda")
        nets["roi_net"].pool_into(feat, tubes.cuda(), out, tl, Tp, t0, argmax=am)
        fm = cf.detach()[:, t0:t0 + tl].reshape(B * tl, 832, cf.shape[3], cf.shape[4])
        oy, oam = torch.ops.torchvision.roi_pool(fm, tubes.reshape(-1, 5), 1.0 / 16.0, 7, 7)
        diff = am.view(R, 7, 7, 832).cpu() != nhwc(oam)
        flips += int(diff.sum())
        pos += int((diff & (nhwc(oy) > 0)).sum())           # flips among exact zeros (post-ReLU) reach no trunk weight
        total += diff.numel()
    return flips, pos, total


# At most 1 % of the pooled elements may take another pixel than the fp32 oracle's: the ROIAlign tests' tolerances below
# are kept unchanged on that condition (a failing comparison reports the counts).
MAX_FLIP_FRACTION = 1e-2


def test_train_step_pool_end_to_end_matches_oracle_autograd():
    from step_b200 import training
    cfg, x, step_tubes, step_targets = spatial_case()
    heads_sd = [synth.head_state_dict(100 + i, cfg) for i in range(2)]
    nets = device_nets(cfg, heads_sd, "pool")
    sd_b = {k: v.clone().requires_grad_(k.endswith("conv3d.weight")) for k, v in synth.base_net_state_dict().items()}
    sds = [trainable(sd) for sd in heads_sd]
    cf = om.base_net(x.clone(), sd_b)
    total = 0.0
    for i in range(2):
        fm = cf.reshape(-1, 832, cf.shape[3], cf.shape[4])
        pooled = tv_roi_pool(fm, step_tubes[i].view(-1, 5), (7, 7), 1.0 / 16.0).view(-1, 2, 832, 7, 7)
        _, loc, first, last, logits = om.two_branch(pooled, sds[i], cfg.T, None, cfg.fc_dim, cfg.pool_size, return_logits=True)
        lc, ll, ln = om.two_branch_losses(logits, loc, first, last, step_tubes[i], step_targets[i], cfg.T)
        total = total + lc.mean() + 5.0 * ll.mean() + 1.0 * ln.mean()
    total.backward()
    total = float(total.detach())
    flips, pos, n = argmax_flips(nets, x, cf, cfg, step_tubes)
    assert flips <= MAX_FLIP_FRACTION * n, (flips, pos, n)
    before = {k: p.detach().clone() for k, p in nets["base_net"].named_parameters()}
    r = training.train_step(cfg, nets, x.cuda(), [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets], lr=0.01,
                            momentum=0.9, weight_decay=1e-4)
    torch.cuda.synchronize()
    assert abs(float(r["loss"]) - total) <= 5e-3 * abs(total)
    assert compare_grads(r, nets["det_net0"], sds[0], 3e-2, 1e-1) == 34 and compare_grads(r, nets["det_net1"], sds[1], 3e-2, 1e-1) == 34
    assert compare_grads(r, nets["base_net"], sd_b, 1.5e-1, 2.5e-1) == 45, (flips, pos, n)
    names = {p: k for k, p in nets["base_net"].named_parameters()}
    for p, gdev in r["grads"].items():
        if p in names and names[p].endswith("12.branch_0.conv3d.weight"):
            exp = before[names[p]] - 0.01 * (gdev + 1e-4 * before[names[p]])
            assert torch.allclose(p.detach(), exp, rtol=1e-5, atol=1e-7)


def test_train_step_pool_shipped_config_matches_oracle_autograd(monkeypatch):
    from step_b200 import training
    monkeypatch.setattr(test_oracle_context, "tv_roi_align", pool_as_align)
    cfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(64, 64))
    B, N = 2, 3
    x = synth.make_clips(B, 36, 64, 64, seed=11)
    step_tubes, step_targets = synth.make_train_case(cfg, B, N, 64, 64, seed=3)
    nets = device_nets(cfg, [synth.head_state_dict(100 + i, cfg) for i in range(3)], "pool", context=True)
    sd_b = {k: v.clone().requires_grad_(k.endswith("conv3d.weight")) for k, v in synth.base_net_state_dict().items()}
    sd_ctx = trainable(synth.context_net_state_dict())
    sds = [trainable(synth.head_state_dict(100 + i, cfg)) for i in range(3)]
    cf = om.base_net(x.clone(), sd_b)
    total, _, _ = test_oracle_context.oracle_objective(cf, sd_ctx, sds, cfg, step_tubes, step_targets)
    total.backward()
    flips, pos, n = argmax_flips(nets, x, cf, cfg, step_tubes)
    assert flips <= MAX_FLIP_FRACTION * n, (flips, pos, n)
    before = {k: p.detach().clone() for k, p in nets["context_net"].named_parameters()}
    r = training.train_step(cfg, nets, x.cuda(), [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets], lr=0.01,
                            momentum=0.9, weight_decay=1e-4)
    torch.cuda.synchronize()
    assert abs(float(r["loss"]) - float(total)) <= 5e-3 * abs(float(total))
    assert len(r["losses"]) == 3
    for i in range(3):
        assert compare_grads(r, nets["det_net%d" % i], sds[i], 3e-2, 1e-1) == 34
    assert compare_grads(r, nets["context_net"], sd_ctx, 3e-2, 1e-1) == 12
    assert compare_grads(r, nets["base_net"], sd_b, 1.5e-1, 2.5e-1) == 45, (flips, pos, n)
    names = {p: k for k, p in nets["context_net"].named_parameters()}
    for p, gdev in r["grads"].items():
        if p in names and names[p].endswith("2.branch_0.conv3d.weight"):
            exp = before[names[p]] - 0.01 * (gdev + 1e-4 * before[names[p]])
            assert torch.allclose(p.detach(), exp, rtol=1e-5, atol=1e-7)


def test_train_step_pool_cls_config_matches_oracle_autograd(monkeypatch):
    from step_b200 import training
    monkeypatch.setattr(test_oracle_cls, "tv_roi_align", pool_as_align)
    cfg = synth.make_cfg(fp16=True, **test_oracle_cls.CLS_CFG, image_size=(64, 64))
    tubes, targets = synth.make_cls_case(cfg, 2, 6, 64, 64, seed=3)
    x = synth.make_clips(2, 36, 64, 64, seed=11)
    nets = device_nets(cfg, [synth.cls_head_state_dict(100, cfg)], "pool", context=True, cls_only=True)
    sd_b = {k: v.clone().requires_grad_(k.endswith("conv3d.weight")) for k, v in synth.base_net_state_dict().items()}
    sd_ctx = trainable(synth.context_net_state_dict())
    sd_h = trainable(synth.cls_head_state_dict(100, cfg))
    cf = om.base_net(x.clone(), sd_b)
    total, _, _, _, _ = test_oracle_cls.cls_objective(cf, sd_ctx, sd_h, cfg, tubes, targets)
    total.backward()
    total = float(total.detach())
    flips, pos, n = argmax_flips(nets, x, cf, cfg, [tubes])
    assert flips <= MAX_FLIP_FRACTION * n, (flips, pos, n)
    r = training.train_step(cfg, nets, x.cuda(), [tubes.cuda()], [targets.cuda()])
    torch.cuda.synchronize()
    assert abs(float(r["loss"]) - total) <= 5e-3 * abs(total)
    assert len(r["losses"]) == 1 and len(r["grads"]) == 45 + 12 + 16
    assert compare_grads(r, nets["det_net0"], sd_h, 3e-2, 1e-1) == 16
    assert compare_grads(r, nets["context_net"], sd_ctx, 3e-2, 1e-1) == 12
    assert compare_grads(r, nets["base_net"], sd_b, 1.5e-1, 2.5e-1) == 45, (flips, pos, n)
