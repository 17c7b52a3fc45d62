"""GPU: the training step in the reference's shipped configuration (scripts/train_step.sh: T=3, iterative_mode=temporal ->
NUM_CHUNKS {1:1, 2:1, 3:3}, context on): the temporal-slice ROIAlign backward, the context-gradient reduction, the head's
backward with the context columns, ContextNet's backward and train_step end to end, against the reference's autograd
(tests/golden/ctx_temporal_grads.npz) and the oracle's torch-CPU autograd (pinned to that golden by
tests/test_oracle_context.py).  Tolerances are those of tests/test_gpu_train.py for the same fp16 activation paths."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import model as om
from step_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _train_case import SHIPPED, compare_grads, rel_l2, trainable  # noqa: E402
from step_b200.synth import device_head, device_nets  # noqa: E402
from test_oracle_context import golden_case, oracle_objective  # noqa: E402

pytestmark = pytest.mark.gpu


def slice_case(dtype=torch.float16, seed=5):
    """B=2 clips of feat_T=9 frames, steps pooling roi_T=3 frames from t_start=3 (steps 1-2 of the shipped config)."""
    from step_b200.engine import Act
    from step_b200 import _lib as L
    gen = torch.Generator().manual_seed(seed)
    B, feat_T, H, W, C, N = 2, 9, 10, 12, 64, 4
    cfg = synth.make_cfg(**SHIPPED)
    tubes = synth.make_train_case(cfg, B, N, 16 * W, 16 * H, seed=seed)[0][0].cuda()      # [B*N, 3, 5]
    R = tubes.shape[0]
    go = Act((torch.randn(R, 3, 7, 7, C + 16, generator=gen) * 0.1).to(dtype).cuda(), C, 0)
    return B, feat_T, H, W, C, tubes, go, L


def test_roi_align_backward_slice_matches_existing_kernel_and_leaves_other_frames():
    from step_b200 import training
    B, feat_T, H, W, C, tubes, go, _ = slice_case()
    gen = torch.Generator().manual_seed(8)
    init = torch.randn(B * feat_T, H, W, C, generator=gen).cuda()
    acc = init.clone()
    training.roi_align_backward_slice(go, tubes.view(-1, 5), 1.0 / 16.0, acc, 3, feat_T, 3)
    # the existing kernel on the 3-frame slice maps (frame f of the slice = clip f // 3, frame 3 + f % 3)
    gin = training.roi_align_backward_nhwc_strided(go, tubes.view(-1, 5), 1.0 / 16.0, B * 3, H, W)
    a, b = acc.view(B, feat_T, H, W, C), init.view(B, feat_T, H, W, C)
    assert torch.equal(a[:, :3], b[:, :3]) and torch.equal(a[:, 6:], b[:, 6:])
    assert torch.equal(a[:, 3:6], b[:, 3:6] + gin.view(B, 3, H, W, C))
    again = init.clone()
    training.roi_align_backward_slice(go, tubes.view(-1, 5), 1.0 / 16.0, again, 3, feat_T, 3)
    assert torch.equal(again, acc)


def test_roi_align_backward_slice_spatial_equals_sum_of_existing_kernel():
    """t_start = 0, roi_T = feat_T: three accumulating calls on a zeroed buffer == gin0 + gin1 + gin2 bit for bit (what the
    spatial train_step did before)."""
    from step_b200 import training
    from step_b200.engine import Act
    gen = torch.Generator().manual_seed(2)
    B, T_, H, W, C, N = 2, 4, 8, 8, 32, 5
    cfg = synth.make_cfg(T=4, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 1})
    st = synth.make_train_case(cfg, B, N, 128, 128, seed=4)[0]
    acc = torch.zeros(B * T_, H, W, C, device="cuda")
    ref = None
    for t in st:
        go = Act((torch.randn(B * N, T_, 7, 7, C, generator=gen) * 0.1).half().cuda())
        training.roi_align_backward_slice(go, t.cuda().view(-1, 5), 1.0 / 16.0, acc, T_, T_, 0)
        gin = training.roi_align_backward_nhwc_strided(go, t.cuda().view(-1, 5), 1.0 / 16.0, B * T_, H, W)
        ref = gin if ref is None else ref.add_(gin)
    assert torch.equal(acc, ref)


def test_roi_align_backward_slice_is_adjoint_of_pool_into():
    """<pool_into(x), g> == <x, ROIAlign_slice^T(g)> at (roi_T=3, feat_T=9, t_start=3), fp32."""
    import step_b200
    from step_b200 import training
    from step_b200.engine import Act
    from step_b200 import _lib as L
    B, feat_T, H, W, C, tubes, _, _ = slice_case(torch.float32)
    gen = torch.Generator().manual_seed(6)
    x = Act(torch.randn(B, feat_T, H, W, C, generator=gen).cuda())
    R = tubes.shape[0]
    y = Act.empty(R * 3, 1, 7, 7, C, L.F32, x.device)
    step_b200.ROINet("align", 7).pool_into(x, tubes, y, 3, feat_T, 3)
    g = torch.randn(R * 3, 1, 7, 7, C, generator=gen).cuda()
    gin = torch.zeros(B * feat_T, H, W, C, device="cuda")
    training.roi_align_backward_slice(Act(g.view(R, 3, 7, 7, C)), tubes.view(-1, 5), 1.0 / 16.0, gin, 3, feat_T, 3)
    lhs = float((y.buf.double() * g.double()).sum())
    rhs = float((x.buf.reshape(-1).double() * gin.reshape(-1).double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * max(1.0, abs(lhs))
    assert float(gin.view(B, feat_T, -1)[:, :3].abs().max()) == 0.0 and float(gin.view(B, feat_T, -1)[:, 6:].abs().max()) == 0.0


def test_context_grad_reduce_matches_torch_and_is_deterministic():
    from step_b200 import training
    cfg = synth.make_cfg(**SHIPPED)
    B, N = 2, 5
    st = synth.make_train_case(cfg, B, N, 400, 400, seed=9)[0]
    gen = torch.Generator().manual_seed(1)
    acc0 = torch.randn(B, 9, 1024, generator=gen)
    dctx = [torch.randn(t.shape[0], 1024, generator=gen) for t in st]
    ref = acc0.clone()
    for i, (t, d) in enumerate(zip(st, dctx), 1):
        t0, tl = training.step_frames(cfg, i)
        clip = (t[:, 0, 0] / tl).floor().long()
        ref[:, t0:t0 + tl] += (torch.zeros(B, 1024).index_add_(0, clip, d) / tl).view(B, 1, 1024)

    def run():
        acc = acc0.clone().cuda()
        for i, (t, d) in enumerate(zip(st, dctx), 1):
            training.context_grad_reduce(d.cuda(), t.cuda(), acc, training.step_frames(cfg, i)[0])
        return acc
    got = run()
    assert torch.allclose(got.cpu(), ref, rtol=1e-5, atol=1e-5)
    assert torch.equal(run(), got)


@pytest.fixture(scope="module")
def golden_oracle():
    """The golden case through the oracle on the CPU, with the gradients of the context feature, of every step's pooled
    features and of every parameter."""
    cfg, cf, step_tubes, step_targets = golden_case()
    cf = cf.requires_grad_(True)
    sd_ctx = trainable(synth.context_net_state_dict())
    sds = [trainable(synth.head_state_dict(100 + i, cfg)) for i in range(3)]
    loss, pooled, ctx = oracle_objective(cf, sd_ctx, sds, cfg, step_tubes, step_targets, pooled_leaves=True)
    ctx.retain_grad()
    loss.backward()
    return dict(cfg=cfg, cf=cf, step_tubes=step_tubes, step_targets=step_targets, sd_ctx=sd_ctx, sds=sds, loss=loss,
                pooled=pooled, ctx=ctx)


def test_head_with_context_matches_reference_and_oracle(golden, golden_oracle):
    """head_forward_backward with the reference's per-tube context feature [R,1024,T',1,1] for the three heads of the
    shipped configuration (steps of 3, 3 and 9 frames): the 34 trainable tensors of each head, the gradient of the pooled
    features and of the context input."""
    from step_b200 import training
    g, o = golden("ctx_temporal_grads"), golden_oracle
    cfg = o["cfg"]
    dcfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(400, 400))
    ctx = o["ctx"].detach()
    total = 0.0
    for i in range(3):
        t0, tl = training.step_frames(cfg, i + 1)
        flat = o["step_tubes"][i]
        clip = [int(flat[p, 0, 0].item() / tl) for p in range(flat.shape[0])]
        tctx = torch.stack([ctx[c, :, t0:t0 + tl] for c in clip]).requires_grad_(True)
        pooled = o["pooled"][i].detach()
        # the oracle's gradient of this step's context input (the golden case's pooled features are leaves)
        pl = pooled.clone().requires_grad_(True)
        sd = trainable(synth.head_state_dict(100 + i, cfg))
        _, loc, first, last, logits = om.two_branch(pl, sd, cfg.T, tctx, cfg.fc_dim, cfg.pool_size, return_logits=True)
        lc, ll, ln = om.two_branch_losses(logits, loc, first, last, flat, o["step_targets"][i], cfg.T)
        (lc.mean() + 5.0 * ll.mean() + 1.0 * ln.mean()).backward()
        net = device_head(dcfg, synth.head_state_dict(100 + i, dcfg))
        r = training.head_forward_backward(net, pooled.cuda(), flat.cuda(), o["step_targets"][i].cuda(), context_feat=tctx.detach().cuda())
        torch.cuda.synchronize()
        total += float(r["loss"])
        names = {p: k for k, p in net.named_parameters()}
        got = {names[p]: v for p, v in r["grads"].items()}
        assert len(got) == 34
        for k, v in got.items():
            ref_n = float(g["gn:h%d:%s" % (i, k)][0])
            assert tuple(v.shape) == tuple(sd[k].shape), k
            assert abs(float(v.double().norm()) - ref_n) <= 3e-2 * ref_n, (i, k, float(v.double().norm()), ref_n)
            assert rel_l2(v, sd[k].grad) <= 8e-2, (i, k, rel_l2(v, sd[k].grad))
        assert abs(float(r["feat_grad"].double().norm()) - float(g["pooled_grad_norm%d" % (i + 1)][0])) <= 3e-2 * float(g["pooled_grad_norm%d" % (i + 1)][0])
        assert rel_l2(r["feat_grad"], pl.grad) <= 8e-2
        assert tuple(r["ctx_grad"].shape) == tuple(tctx.shape)
        assert rel_l2(r["ctx_grad"], tctx.grad) <= 8e-2, rel_l2(r["ctx_grad"], tctx.grad)
    assert abs(total - float(g["loss"][0])) <= 5e-3 * float(g["loss"][0])


def test_context_net_backward_matches_reference_and_oracle(golden, golden_oracle):
    """context_forward / context_backward at 25x25 (the trunk output at 36x400x400) from the oracle's d(loss)/d(context):
    ContextNet's 12 Unit3D weight gradients and the context-only gradient of conv_feat."""
    import step_b200
    from step_b200 import training
    from step_b200.networks import to_act
    from step_b200 import _lib as L
    g, o = golden("ctx_temporal_grads"), golden_oracle
    cfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(400, 400))
    net = step_b200.ContextNet(cfg)
    net.load_state_dict(synth.context_net_state_dict(), strict=True)
    net = net.cuda().eval()
    feat = to_act(o["cf"].detach().cuda(), L.F16)
    ctx, state = training.context_forward(net, feat)
    assert rel_l2(ctx, o["ctx"].detach().view(2, 1024, 9).permute(0, 2, 1)) <= 1e-2
    d_ctx = o["ctx"].grad.view(2, 1024, 9).permute(0, 2, 1).contiguous().cuda()
    grads, gfeat = training.context_backward(state, d_ctx, 1024.0)
    torch.cuda.synchronize()
    names = {p: k for k, p in net.named_parameters()}
    got = {names[p]: v for p, v in grads.items()}
    assert len(got) == 12
    for k, v in got.items():
        ref_n = float(g["gn:ctx:" + k][0])
        assert abs(float(v.double().norm()) - ref_n) <= 3e-2 * ref_n, (k, float(v.double().norm()), ref_n)
        assert rel_l2(v, o["sd_ctx"][k].grad) <= 8e-2, (k, rel_l2(v, o["sd_ctx"][k].grad))
    gf = gfeat.float().mul_(1.0 / 1024.0).permute(0, 1, 4, 2, 3)          # [B, T', 832, H', W']
    ref_n = float(g["ctx_feat_grad_norm"][0])
    assert abs(float(gf.double().norm()) - ref_n) <= 3e-2 * ref_n
    assert rel_l2(gf, o["cf"].grad) <= 8e-2, rel_l2(gf, o["cf"].grad)


def test_train_step_shipped_config_matches_oracle_autograd():
    """train_step in the shipped configuration at reduced resolution (2 clips of 36x64x64, T'=9: steps pool frames [3, 6),
    [3, 6) and [0, 9)) against the oracle's autograd with torchvision's roi_align: 45 trunk, 12 ContextNet and 3 x 34 head
    tensors, and the SGD update."""
    from step_b200 import training
    cfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(64, 64))
    B, N = 2, 3
    x = synth.make_clips(B, 36, 64, 64, seed=11)
    step_tubes, step_targets = synth.make_train_case(cfg, B, N, 64, 64, seed=3)
    nets = device_nets(cfg, [synth.head_state_dict(100 + i, cfg) for i in range(3)], context=True)
    sd_b = {k: v.clone().requires_grad_(k.endswith("conv3d.weight")) for k, v in synth.base_net_state_dict().items()}
    sd_ctx = trainable(synth.context_net_state_dict())
    sds = [trainable(synth.head_state_dict(100 + i, cfg)) for i in range(3)]
    cf = om.base_net(x.clone(), sd_b)
    total, _, _ = oracle_objective(cf, sd_ctx, sds, cfg, step_tubes, step_targets)
    total.backward()
    before = {k: p.detach().clone() for k, p in nets["context_net"].named_parameters()}
    r = training.train_step(cfg, nets, x.cuda(), [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets], lr=0.01,
                            momentum=0.9, weight_decay=1e-4)
    torch.cuda.synchronize()
    assert abs(float(r["loss"]) - float(total)) <= 5e-3 * abs(float(total))
    assert len(r["losses"]) == 3
    for i in range(3):
        assert compare_grads(r, nets["det_net%d" % i], sds[i], 3e-2, 1e-1) == 34
    assert compare_grads(r, nets["context_net"], sd_ctx, 3e-2, 1e-1) == 12
    assert compare_grads(r, nets["base_net"], sd_b, 1.5e-1, 2.5e-1) == 45
    names = {p: k for k, p in nets["context_net"].named_parameters()}
    for p, gdev in r["grads"].items():
        if p in names and names[p].endswith("2.branch_0.conv3d.weight"):
            exp = before[names[p]] - 0.01 * (gdev + 1e-4 * before[names[p]])
            assert torch.allclose(p.detach(), exp, rtol=1e-5, atol=1e-7)


def test_train_step_shipped_config_rejects_mismatched_tubes_and_missing_context_net():
    from step_b200 import training
    cfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(64, 64))
    step_tubes, step_targets = synth.make_train_case(cfg, 1, 2, 64, 64)
    nets = device_nets(cfg, [synth.head_state_dict(100 + i, cfg) for i in range(3)], context=True)
    x = synth.make_clips(1, 36, 64, 64).cuda()
    bad = [step_tubes[0], step_tubes[2], step_tubes[2]]                   # step 2 pools 3 frames, not 9
    with pytest.raises(RuntimeError, match="step 2 pools frames"):
        training.train_step(cfg, nets, x, [t.cuda() for t in bad], [t.cuda() for t in step_targets])
    del nets["context_net"]
    with pytest.raises(RuntimeError, match="context_net"):
        training.train_step(cfg, nets, x, [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets])


def test_sgd_steps_descend_shipped_config():
    """Four steps on one fixed mini-batch in the shipped configuration: the objective decreases monotonically, so the
    gradients of the temporal steps and of the context branch point downhill.  Layer-wise normalised step as in
    tests/test_gpu_train.py::test_sgd_steps_descend."""
    from step_b200 import training
    cfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(64, 64))
    nets = device_nets(cfg, [synth.head_state_dict(100 + i, cfg) for i in range(3)], context=True)
    step_tubes, step_targets = synth.make_train_case(cfg, 2, 3, 64, 64, seed=7)
    args = (cfg, nets, synth.make_clips(2, 36, 64, 64, seed=5).cuda(), [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets])
    losses = []
    for _ in range(4):
        r = training.train_step(*args, lr=None)
        losses.append(float(r["loss"]))
        assert len(r["grads"]) == 45 + 12 + 3 * 34
        for p, gr in r["grads"].items():
            pn, gn = float(p.detach().norm()), float(gr.norm())
            if pn > 0 and gn > 0:
                training.sgd_step({p: gr}, lr=3e-4 * pn / gn, momentum=0.0)
    losses.append(float(training.train_step(*args, lr=None)["loss"]))
    assert all(b < a for a, b in zip(losses, losses[1:])), losses
