"""GPU: back-propagation through BaseNet / ContextNet / TwoBranchNet with torch.autograd (step_b200.autograd).

1. step_head_outputs_bwd_f32 against torch's float64 autograd of the oracle's restatement of the head's tail
   (oracle/model.py::two_branch_losses + sigmoid + the first / last slices) on the same fp32 operands, for every upstream
   gradient, some of them, zero masks, class-only heads and T' != T; run-to-run bit identity; and, with the mean
   objective's upstream gradients, the gradients step_head_losses_f32 forms.
2. The modules' backward against the explicit halves of step_b200/training.py: the trunk's and ContextNet's parameter
   gradients bit for bit, the heads' within 1e-5 relative L2 (only the loss-gradient rounding differs); without autograd
   the forwards launch what they launched before and return the same bits.
3. A restatement of train.py:263-348 (and train_cls.py:246-322) on the synthetic workloads, fp32: after
   loss_back.backward() every trainable parameter's .grad is within 1e-4 relative L2 of train_step(loss_scale=1.0,
   dropout=True) from the same state and generator state; running statistics and the generator's offset agree, and
   step_b200.optim.Adam's update matches train_step(optimizer=...)'s.  The driver's ROIAlign / ROIPool backward is the
   NCHW one with float atomics, so the two paths differ by summation order only.
4. fp16: (loss * 1024).backward() against train_step(loss_scale=1024).
5. Refusals: a clip requiring grad, a second backward through one forward, a trainable parameter without a gradient."""
import os
import sys

import pytest
import torch

import step_b200
from oracle import model as om
from step_b200 import _lib as L
from step_b200 import synth, training

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _train_case import rel_l2  # noqa: E402

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -24


# ---- 1. the new entry ----------------------------------------------------------------------------------------------------
def tail_case(name, cls_only=False, seed=0):
    """(T, logits, loc, first, last, tubes, targets) fp32 on the CPU: make_loss_case's tubes and targets, seeded outputs."""
    T_, chunks, _, tubes, targets = synth.make_loss_case(name, 60)
    gen = torch.Generator().manual_seed(seed)
    N, Tl = tubes.shape[0], tubes.shape[1]
    logits = torch.randn(N, 60, generator=gen) * 3.0
    loc = torch.randn(N, Tl, 4, generator=gen)
    first = torch.randn(N, T_, 4, generator=gen)
    last = torch.randn(N, T_, 4, generator=gen)
    return T_, logits, loc, first, last, tubes, targets


def f64_tail_grads(T_, logits, loc, first, last, tubes, targets, ups, cls_only):
    """torch float64 autograd of prob = sigmoid(logits) and oracle two_branch_losses, with first / last = clones of loc's
    slices plus the neighbour regressors' outputs (two_branch.py:265-270), from the upstream gradients ups (None = zero).
    Returns (dlogits, dloc, dfirst, dlast) with dfirst / dlast the gradients of the neighbour regressors' outputs."""
    d = lambda t: t.double()
    lg = d(logits).requires_grad_(True)
    N, Tl = loc.shape[0], loc.shape[1]
    chunks = Tl // T_
    s0 = T_ // 2 - T_ // 2
    e0 = (chunks - 1) * T_ + T_ // 2 - T_ // 2
    lc_ = d(loc).requires_grad_(True)
    nb1 = (d(first) - d(loc)[:, s0:s0 + T_]).requires_grad_(True)
    nb2 = (d(last) - d(loc)[:, e0:e0 + T_]).requires_grad_(True)
    fl = lc_[:, s0:s0 + T_].contiguous().clone() + nb1
    ll = lc_[:, e0:e0 + T_].contiguous().clone() + nb2
    prob = torch.sigmoid(lg)
    losses = om.two_branch_losses(lg, lc_, fl, ll, d(tubes), d(targets), T_, cls_only=cls_only)
    outs = [prob] + ([] if cls_only else [lc_, fl, ll]) + list(losses)
    gs = [ups[0]] + ([] if cls_only else list(ups[1:4])) + list(ups[4:])
    pairs = [(o, d(g).view_as(o)) for o, g in zip(outs, gs) if g is not None and o.requires_grad and g.numel() == o.numel()]
    leaves = [lg] + ([] if cls_only else [lc_, nb1, nb2])
    grads = torch.autograd.grad([o for o, _ in pairs], leaves, [g for _, g in pairs], allow_unused=True)
    return [torch.zeros_like(l) if g is None else g for l, g in zip(leaves, grads)]


def random_ups(N, Tl, T_, cls, which, seed=1):
    gen = torch.Generator().manual_seed(seed)
    shapes = [(N, cls), (N, Tl, 4), (N, T_, 4), (N, T_, 4), (N * cls,), (1,), (1,)]
    return [torch.randn(*s, generator=gen) if i in which else None for i, s in enumerate(shapes)]


def device_tail(T_, logits, loc, first, last, tubes, targets, ups, cls_only):
    c = lambda t: None if t is None else t.cuda()
    g = training.head_outputs_backward(c(logits), c(loc), c(first), c(last), c(tubes), c(targets), T_, cls_only, *[c(u) for u in ups])
    keys = ["logits"] + ([] if cls_only else ["local_loc", "first_loc", "last_loc"])
    return [g[k].cpu() for k in keys]


def assert_few_roundings(got, ref, what):
    """max |got - ref| within 16 fp32 roundings of the tensor's largest element (exact zeros where ref is all zero)."""
    m = float(ref.abs().max())
    err = float((got.double() - ref).abs().max())
    assert err <= 16 * EPS32 * m, (what, err, m)


ALL = range(7)


@pytest.mark.parametrize("case,which,cls_only", [
    ("c1", ALL, False), ("c3", ALL, False), ("nomask", ALL, False),
    ("c3", (0, 4), False), ("c3", (1, 5), False), ("c3", (2, 3, 6), False), ("c1", (), False),
    ("c3", ALL, True), ("nomask", ALL, True), ("c1", (4,), True)])
def test_head_outputs_bwd_matches_float64_autograd(case, which, cls_only):
    T_, logits, loc, first, last, tubes, targets = tail_case(case)
    N, Tl = loc.shape[0], loc.shape[1]
    ups = random_ups(N, Tl, T_, 60, which)
    if case == "nomask":
        ups[4] = None if 4 not in which else torch.randn(1)     # the forward's [1] zero of loss_cls
    got = device_tail(T_, logits, loc, first, last, tubes, targets, ups, cls_only)
    ref = f64_tail_grads(T_, logits, loc, first, last, tubes, targets, ups, cls_only)
    for name, a, b in zip(("dlogits", "dloc", "dfirst", "dlast"), got, ref):
        assert_few_roundings(a, b, name)
    again = device_tail(T_, logits, loc, first, last, tubes, targets, ups, cls_only)
    assert all(torch.equal(a, b) for a, b in zip(got, again))


@pytest.mark.parametrize("case", ["c1", "c3", "nomask"])
def test_head_outputs_bwd_of_the_mean_objective_is_head_losses_gradient(case):
    T_, logits, loc, first, last, tubes, targets = tail_case(case)
    N = logits.shape[0]
    c = lambda t: t.cuda()
    _, _, _, g = training.head_losses(c(logits), c(loc), c(first), c(last), c(tubes), c(targets), T_, 5.0, 1.0, want_grads=True)
    ups = [None, None, None, None, torch.full((N * 60,), 1.0 / (N * 60)), torch.tensor([5.0]), torch.tensor([1.0])]
    got = device_tail(T_, logits, loc, first, last, tubes, targets, ups, False)
    for a, k in zip(got, ("logits", "local_loc", "first_loc", "last_loc")):
        b = g[k].cpu().double()
        assert float((a.double() - b).abs().max()) <= 16 * EPS32 * max(float(b.abs().max()), 1e-30), k


# ---- 2. modules against the explicit halves ------------------------------------------------------------------------------
def small_cfg(**kw):
    return synth.make_cfg(**dict(dict(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False, image_size=(64, 64)), **kw))


@pytest.mark.parametrize("fp16,train", [(False, False), (True, False), (False, True)])
def test_basenet_backward_is_trunk_backward_bit_for_bit(fp16, train):
    cfg = small_cfg(fp16=fp16, freeze_stats=not train, freeze_affine=not train)
    net = synth.device_nets(cfg, [])["base_net"]
    net.train(train)
    clips = synth.make_clips(1, 16, 64, 64, seed=5).cuda()
    with step_b200.engine.running_stats_update(False):
        conv = net(clips)
        assert conv.grad_fn is not None
        G = torch.randn(conv.shape, generator=torch.Generator().manual_seed(2)).to(conv.dtype).cuda()
        torch.autograd.backward(conv, G)
        feat, ref = training.trunk_forward_backward(net, clips, lambda f: G.permute(0, 1, 3, 4, 2), loss_scale=1.0)
    assert torch.equal(feat.logical(), conv.detach())
    params = [p for p in net.parameters() if p.requires_grad]
    assert len(params) == len(ref) and (not train or any("batch3d" in n for n, p in net.named_parameters() if p.requires_grad))
    for p in params:
        assert torch.equal(p.grad, ref[p])


@pytest.mark.parametrize("fp16", [False, True])
def test_contextnet_backward_is_context_backward_bit_for_bit(fp16):
    from step_b200.networks import to_act
    cfg = small_cfg(fp16=fp16)
    net = synth.device_nets(cfg, [], context=True)["context_net"]
    dt = torch.float16 if fp16 else torch.float32
    cf = synth.make_conv_feat(2, 9, 8, 8).to(dt).cuda().requires_grad_(True)
    out = net(cf)
    G = torch.randn(out.shape, generator=torch.Generator().manual_seed(4)).cuda()
    torch.autograd.backward(out, G)
    c, state = training.context_forward(net, to_act(cf.detach(), step_b200.engine.dtype_code(fp16)))
    assert torch.equal(c.permute(0, 2, 1).unsqueeze(-1).unsqueeze(-1), out.detach())
    ref, gfeat = training.context_backward(state, G.view(2, 1024, 9).permute(0, 2, 1), loss_scale=1.0)
    params = [p for p in net.parameters() if p.requires_grad]
    assert len(params) == len(ref)
    for p in params:
        assert torch.equal(p.grad, ref[p])
    assert torch.equal(cf.grad, gfeat.permute(0, 1, 4, 2, 3))


def head_case(cls_only, seed=3):
    cfg = synth.make_cfg(**synth.WORKLOADS["cls" if cls_only else "shipped"].cfg, image_size=(400, 400))
    sd = synth.cls_head_state_dict(100, cfg) if cls_only else synth.head_state_dict(100, cfg)
    head = synth.device_head(cfg, sd, cls_only)
    T_len = cfg.T if cls_only else cfg.T * 3
    _, _, feat, tubes, targets = synth.make_loss_case("c3", 60)
    if cls_only:
        feat, tubes = feat[:, :T_len], tubes[:, :T_len]
    gen = torch.Generator().manual_seed(seed)
    ctx = torch.rand(feat.shape[0], 1024, T_len, 1, 1, generator=gen)
    return cfg, head, feat.cuda(), ctx.cuda(), tubes.cuda(), targets.cuda()


@pytest.mark.parametrize("cls_only", [False, True])
def test_head_backward_matches_head_forward_backward(cls_only):
    cfg, head, feat, ctx, tubes, targets = head_case(cls_only)
    f, c = feat.clone().requires_grad_(True), ctx.clone().requires_grad_(True)
    outs = head(f, context_feat=c, tubes=tubes, targets=targets)
    loss = outs[4].mean() + 5.0 * outs[5].mean() + 1.0 * outs[6].mean()
    loss.backward()
    r = training.head_forward_backward(head, feat, tubes, targets, context_feat=ctx, loss_scale=1.0)
    assert torch.allclose(loss.detach(), r["loss"], rtol=1e-6)
    params = [p for p in head.parameters() if p.requires_grad]
    assert len(params) == len(r["grads"])
    for p in params:
        assert rel_l2(p.grad, r["grads"][p].cpu()) <= 1e-5
    assert rel_l2(f.grad, r["feat_grad"].cpu()) <= 1e-5
    assert rel_l2(c.grad, r["ctx_grad"].cpu()) <= 1e-5


def test_forwards_without_autograd_launch_and_return_what_they_did():
    cfg = small_cfg()
    heads = [synth.head_state_dict(100, cfg)]
    nets = synth.device_nets(cfg, heads, context=True)
    clips = synth.make_clips(1, 16, 64, 64, seed=5).cuda()
    _, _, feat, tubes, targets = synth.make_loss_case("c3", 60)
    feat, tubes, targets = feat.cuda(), tubes.cuda(), targets.cuda()

    def run(frozen):
        n0 = L.launch_count()
        conv = nets["base_net"](clips)
        cx = nets["context_net"](conv)
        outs = nets["det_net0"](feat, torch.rand(feat.shape[0], 1024, 9, 1, 1, generator=torch.Generator().manual_seed(1)).cuda(),
                                tubes, targets)
        torch.cuda.synchronize()
        assert all(t.grad_fn is None for t in (conv, cx) + tuple(outs))
        return L.launch_count() - n0, [conv, cx] + list(outs)

    with torch.no_grad():
        n_ng, a = run(False)
    saved = {p: p.requires_grad for net in nets.values() for p in net.parameters()}
    try:
        for p in saved:
            p.requires_grad_(False)
        n_fr, b = run(True)
    finally:
        for p, rg in saved.items():
            p.requires_grad_(rg)
    with torch.no_grad():     # what the forwards launched before: the same calls without the autograd dispatch
        n0 = L.launch_count()
        conv = nets["base_net"].forward_act(clips).logical()
        torch.cuda.synchronize()
        n_trunk = L.launch_count() - n0
    assert n_ng == n_fr and n_trunk < n_ng
    assert torch.equal(conv, a[0])
    for x, y in zip(a, b):
        assert torch.equal(x, y)


# ---- 3. the driver loops -------------------------------------------------------------------------------------------------
def train_py_iteration(cfg, nets, clips, step_tubes, step_targets, lambda_reg=5.0, lambda_neighbor=1.0, scale=1.0):
    """train.py:263-348 with the samples already selected (train_select is step_b200.select_samples) and no optimizer step:
    the modules' forwards, the driver's torch ops, loss_back.backward().  Returns loss_back."""
    for net in nets.values():
        net.train()
    conv_feat = nets["base_net"](clips)
    context_feat = None
    if not cfg.no_context:
        context_feat = nets["context_net"](conv_feat)
    loss_back = 0.
    for i in range(1, cfg.max_iter + 1):
        chunks = cfg.NUM_CHUNKS[i]
        T_start = int((cfg.NUM_CHUNKS[cfg.max_iter] - chunks) / 2) * cfg.T
        T_length = chunks * cfg.T
        flat_tubes, flat_targets = step_tubes[i - 1], step_targets[i - 1]
        pooled_feat = nets["roi_net"](conv_feat[:, T_start:T_start + T_length].contiguous(), flat_tubes)
        _, C, W, H = pooled_feat.size()
        pooled_feat = pooled_feat.view(-1, T_length, C, W, H)
        temp_context_feat = None
        if not cfg.no_context:
            temp_context_feat = torch.zeros((pooled_feat.size(0), context_feat.size(1), T_length, 1, 1)).to(context_feat)
            for p in range(pooled_feat.size(0)):
                temp_context_feat[p] = context_feat[int(flat_tubes[p, 0, 0].item() / T_length), :,
                                                    T_start:T_start + T_length].contiguous().clone()
        _, _, _, _, lc, ll, ln = nets["det_net%d" % (i - 1)](pooled_feat, context_feat=temp_context_feat, tubes=flat_tubes,
                                                             targets=flat_targets)
        cur = lc.mean() + ll.mean() * lambda_reg + ln.mean() * lambda_neighbor
        loss_back += cur.to(conv_feat.device)
    (loss_back * scale).backward()
    return loss_back


def train_cls_iteration(cfg, nets, clips, step_tubes, step_targets):
    """train_cls.py:246-322 with the rows already selected (step_b200.select_cls_samples), no optimizer step."""
    for net in nets.values():
        net.train()
    conv_feat = nets["base_net"](clips)
    context_feat = nets["context_net"](conv_feat)
    T_start, T_length = 0, cfg.T
    flat_tubes, flat_targets = step_tubes[0], step_targets[0]
    pooled_feat = nets["roi_net"](conv_feat[:, T_start:T_start + T_length].contiguous(), flat_tubes)
    _, C, W, H = pooled_feat.size()
    pooled_feat = pooled_feat.view(-1, T_length, pooled_feat.size(1), W, H)
    temp_context_feat = torch.zeros((pooled_feat.size(0), context_feat.size(1), T_length, 1, 1)).to(context_feat)
    for p in range(pooled_feat.size(0)):
        temp_context_feat[p] = context_feat[int(flat_tubes[p, 0, 0].item() / T_length), :, T_start:T_start + T_length].contiguous().clone()
    _, _, _, _, lc, _, _ = nets["det_net0"](pooled_feat, context_feat=temp_context_feat, tubes=flat_tubes, targets=flat_targets)
    loss = lc.mean()
    loss.backward()
    return loss


def named(nets):
    return {(k, n): p for k, net in nets.items() for n, p in net.named_parameters() if p.requires_grad}


def bn_buffers(nets):
    return {(k, n): b for k, net in nets.items() for n, b in net.named_buffers() if "running_" in n}


def driver_against_train_step(workload, pool_mode, freeze_stats, fp16=False, scale=1.0, lr=1e-5):
    """The driver iteration and step_b200.optim.Adam on one copy of the workload's nets, train_step(optimizer=...) on
    another, from the same generator state.  Returns (grads_a, grads_b, params_a, params_b, bufs_a, bufs_b, offsets)."""
    from step_b200 import optim
    mk = lambda: synth.make_workload(workload, fp16=fp16, pool_mode=pool_mode, dropout=0.3, freeze_stats=freeze_stats)
    cfg, nets_a, clips, step_tubes, step_targets = mk()
    _, nets_b, _, _, _ = mk()
    gen = torch.cuda.default_generators[0]
    state = gen.get_state()
    opt_a = optim.Adam(list(named(nets_a).values()), lr=lr)
    if workload == "cls":
        train_cls_iteration(cfg, nets_a, clips, step_tubes, step_targets)
    else:
        train_py_iteration(cfg, nets_a, clips, step_tubes, step_targets, scale=scale)
    grads_a = {k: p.grad.detach().clone() / scale for k, p in named(nets_a).items()}
    missing = [k for k, p in named(nets_a).items() if p.grad is None]
    assert not missing, missing
    for p in named(nets_a).values():
        p.grad.div_(scale)
    opt_a.step()
    off_a = gen.get_offset()
    gen.set_state(state)
    for net in nets_b.values():
        net.train()
    opt_b = optim.Adam(list(named(nets_b).values()), lr=lr)
    r = training.train_step(cfg, nets_b, clips, step_tubes, step_targets, loss_scale=scale, dropout=True, optimizer=opt_b)
    nb = named(nets_b)
    grads_b = {k: r["grads"][p] for k, p in nb.items()}
    assert set(grads_b) == set(grads_a)
    return (grads_a, grads_b, {k: p.detach() for k, p in named(nets_a).items()}, {k: p.detach() for k, p in nb.items()},
            bn_buffers(nets_a), bn_buffers(nets_b), (off_a, gen.get_offset()), nets_a)


def check_driver(res, bound, trunk_bound=None):
    """Gradients and Adam-updated parameters within `bound` relative L2 (the trunk's within trunk_bound when given), equal
    running statistics (to fp32 rounding) and the same generator offset."""
    grads_a, grads_b, pa, pb, ba, bb, (oa, ob), _ = res
    assert oa == ob
    lim = lambda k: trunk_bound if trunk_bound is not None and k[0] == "base_net" else bound
    over = [(k, what, e) for k in grads_a for what, e in (("grad", rel_l2(grads_a[k], grads_b[k].cpu())),
                                                          ("param", rel_l2(pa[k], pb[k].cpu()))) if e > lim(k)]
    assert not over, sorted(over, key=lambda t: -t[2])[:10]
    for k in ba:
        assert torch.allclose(ba[k], bb[k], rtol=1e-5, atol=1e-7), k


@pytest.mark.parametrize("pool_mode", ["align", "pool"])
@pytest.mark.parametrize("freeze_stats", [True, False])
def test_train_py_loop_matches_train_step(pool_mode, freeze_stats):
    res = driver_against_train_step("shipped", pool_mode, freeze_stats)
    check_driver(res, 1e-4)
    # torch's own Adam runs on the same gradients too
    nets_a = res[-1]
    params = list(named(nets_a).values())
    before = [p.detach().clone() for p in params]
    opt = torch.optim.Adam(params, lr=1e-5)
    opt.step()
    assert all(torch.isfinite(p).all() for p in params) and any(not torch.equal(p, q) for p, q in zip(params, before))


@pytest.mark.parametrize("freeze_stats", [True, False])
def test_train_cls_loop_matches_train_step(freeze_stats):
    check_driver(driver_against_train_step("cls", "align", freeze_stats), 1e-4)


def test_fp16_scaled_loss_matches_train_step():
    """fp16 storage: the driver's NCHW ROIAlign rounds its fp32 result to fp16 where train_step's channels-last pooling takes
    its fp16 fast path (within 1 fp16 ulp), and the autograd path stores conv_feat's summed gradient in fp16 where train_step
    keeps it in fp32.  Those fp16 differences grow through each backward: 3e-2 for ContextNet and the heads (1.02e-2
    measured on det_net0's local_conv.0.conv2 on an H100), 5e-2 for the trunk (2.4e-2 measured on the stem's weight),
    against the 1e-1 / 2.5e-1 tests/test_gpu_train_context.py allows train_step against the reference's autograd on the
    same fp16 path."""
    check_driver(driver_against_train_step("shipped", "align", True, fp16=True, scale=1024.0), 3e-2, trunk_bound=5e-2)


# ---- 5. refusals ---------------------------------------------------------------------------------------------------------
def test_clip_requiring_grad_is_refused():
    cfg = small_cfg()
    net = synth.device_nets(cfg, [])["base_net"]
    clips = synth.make_clips(1, 16, 64, 64).cuda().requires_grad_(True)
    with pytest.raises(RuntimeError, match="clip requires grad"):
        net(clips)


def test_second_backward_through_one_forward_raises():
    cfg, head, feat, ctx, tubes, targets = head_case(False)
    outs = head(feat.requires_grad_(True), context_feat=ctx, tubes=tubes, targets=targets)
    loss = outs[4].mean() + outs[5].mean()
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="second backward"):
        loss.backward()


def test_trainable_parameter_without_gradient_is_an_error():
    cfg, head, feat, ctx, tubes, targets = head_case(True)
    head.register_parameter("stray", torch.nn.Parameter(torch.zeros(3, device="cuda")))
    outs = head(feat, context_feat=ctx, tubes=tubes, targets=targets)
    with pytest.raises(RuntimeError, match="no gradient for the trainable parameter.*stray"):
        outs[4].mean().backward()
