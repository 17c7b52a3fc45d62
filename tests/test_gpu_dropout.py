"""GPU: the heads' training-mode dropout (models/two_branch.py:244, 261) through head_forward_backward and train_step.

  * mask parity with torch: step_dropout_mask_u8 against F.dropout(torch.ones(n), p, True) != 0 from the same state of the
    device's default generator, bit for bit, at the shipped draw sizes, a class-stage draw and the edges of torch's launch
    geometry (4 * n_threads elements is the last size whose threads make one curand_uniform4 call each), for three p,
    two seeds and two consecutive draws, with the generator's offset after them; the forward kernels' values against the
    permuted F.dropout output of the same fp32 tensors, bit for bit;
  * the head: head_forward_backward(dropout=True) on the fp32 path with loss_scale=1 against the oracle's autograd given
    the masks F.dropout draws when replayed from the same starting state (tests/_dropout_oracle.py), for full and
    class-only heads and both context forms, at the tolerances of test_gpu_train_fp32.py; the fp16 path at those of
    test_gpu_train.py;
  * train_step in the shipped configuration (ROIAlign and ROIPool) and the classification stage, heads in .train(): every
    gradient against the oracle with the replayed masks, and the generator's final offset against the replay's;
  * invariants: no draw and bit-identical results with p = 0 or heads in eval mode; bit-identical gradients from the same
    starting state; a draw inside CUDA stream capture raises."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import model as om
from step_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _dropout_oracle as DO  # noqa: E402
import test_gpu_train_fp32 as F32  # noqa: E402
import test_oracle_cls  # noqa: E402
import test_oracle_context  # noqa: E402
from _train_case import SHIPPED, rel_l2, trainable  # noqa: E402
from step_b200.synth import device_head, device_nets  # noqa: E402

pytestmark = pytest.mark.gpu
P = 0.3
FP16_L2_TOL = 1e-1


def _gen():
    torch.cuda.init()
    return torch.cuda.default_generators[0]


def _n_threads():
    prop = torch.cuda.get_device_properties(0)
    return 256 * prop.multi_processor_count * (prop.max_threads_per_multi_processor // 256)


def _sizes():
    nt = _n_threads()
    return [68 * 13568 * 3, 68 * 13568 * 9, 68 * 3 * 12544, 68 * 9 * 12544, 48 * 13568 * 9, 4, 1020, 4 * nt, 4 * nt + 4]


# ---- mask parity -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [0.1, 0.3, 0.5])
def test_masks_and_offsets_equal_torch_dropout(p):
    from step_b200 import training
    gen = _gen()
    for seed in (1234, (1 << 40) + 77):
        for n in _sizes():
            gen.manual_seed(seed)
            gen.set_offset(gen.get_offset() + 8)          # a draw that does not start at offset 0
            state = gen.get_state()
            ours = []
            for _ in range(2):
                d = training.dropout_draw("cuda:0", p, n)
                ours.append(training.dropout_mask(d, n, "cuda:0").bool())
            off_ours = gen.get_offset()
            gen.set_state(state)
            theirs = [F.dropout(torch.ones(n, device="cuda"), p, True) != 0 for _ in range(2)]
            assert gen.get_offset() == off_ours, (n, p, seed)
            for a, b in zip(ours, theirs):
                assert torch.equal(a, b), (n, p, seed, int((a != b).sum()))


def test_forward_kernels_equal_permuted_torch_dropout():
    """step_dropout_global_fwd / _ctx_mean_f32 / _local_fwd against F.dropout of the reference's tensors: the global
    [R, C' = fc*49 + 1024, T] (downsample output channel c at pixel p is c' = c*49 + p) and the local [R*T, fc, 49]."""
    from step_b200 import _lib as L, training
    R, T, Pp, fc, K = 68, 9, 49, 256, 1024
    gen = _gen()
    gen.manual_seed(99)
    flat = torch.randn((R, fc * Pp + K, T), device="cuda")
    state = gen.get_state()
    ref = F.dropout(flat, P, True)
    gen.set_state(state)
    d = training.dropout_draw("cuda:0", P, flat.numel())
    # the downsample part, read from a wider channels-last buffer (ld 300)
    cat = torch.zeros((R, T, Pp, 300), device="cuda")
    cat[..., 20:20 + fc] = flat[:, :fc * Pp].view(R, fc, Pp, T).permute(0, 3, 2, 1)
    y = torch.empty((R, T, Pp, fc), device="cuda")
    L.check(L.lib().step_dropout_global_fwd(d, L.c_void_p(cat.data_ptr() + 4 * 20), L.F32, 300, R, T, Pp, fc, K, L.ptr(y), fc,
                                            L.stream()))
    assert torch.equal(y, ref[:, :fc * Pp].reshape(R, fc, Pp, T).permute(0, 3, 2, 1))
    # the context part from ContextNet's [B, T', 1024] layout, two clips, frames from t_start = 2
    B, Tall, t0 = 2, T + 3, 2
    row_map = (torch.arange(R, device="cuda") % B).to(torch.int32)
    ctx = torch.randn((B, Tall, K), device="cuda")
    # each tube's slice must equal flat's context part for the comparison: rebuild flat's context from ctx
    flat2 = flat.clone()
    flat2[:, fc * Pp:] = ctx[row_map.long(), t0:t0 + T].permute(0, 2, 1)
    gen.set_state(state)
    ref2 = F.dropout(flat2, P, True)
    out = torch.empty((R, K), device="cuda")
    L.check(L.lib().step_dropout_ctx_mean_f32(d, Pp, fc, L.c_void_p(ctx.data_ptr() + 4 * t0 * K), L.ptr(row_map), Tall * K, K, 1, R, T,
                                              K, L.ptr(out), L.stream()))
    dropped = ref2[:, fc * Pp:]                                   # [R, K, T]
    s = torch.zeros((R, K), device="cuda")
    for t in range(T):
        s = s + dropped[:, :, t]
    assert torch.equal(out, torch.div(s, torch.full_like(s, float(T))))      # a true division (a scalar divisor multiplies)
    # local: [F, fc, 49] in the reference, [F, 49, fc] here
    Fr = R * T
    x = torch.randn((Fr, fc, Pp), device="cuda")
    state = gen.get_state()
    ref3 = F.dropout(x, P, True)
    gen.set_state(state)
    d3 = training.dropout_draw("cuda:0", P, x.numel())
    xl = x.permute(0, 2, 1).contiguous()
    yl = torch.empty_like(xl)
    L.check(L.lib().step_dropout_local_fwd(d3, L.ptr(xl), L.F32, fc, Fr, Pp, fc, L.ptr(yl), fc, L.stream()))
    assert torch.equal(yl, ref3.permute(0, 2, 1))


# ---- the head ------------------------------------------------------------------------------------------------------------
def _train_head(cfg, sd, cls_only=False):
    net = device_head(cfg, sd, cls_only)
    net.train()
    return net


def _head_case(form, fp16=False):
    """(cfg, net, feat, tubes, targets, context for head_forward_backward, oracle context [N,1024,T',1,1] or None, cls_only)."""
    cls_only = form == "cls_tuple"
    T_, chunks = 3, 3
    cfg = synth.make_cfg(fp16=fp16, T=T_, max_iter=1, NUM_CHUNKS={1: chunks}, no_context=form == "none", image_size=(112, 112), dropout=P)
    Tl = T_ * chunks
    N = 4
    g = torch.Generator().manual_seed(17)
    feat = torch.randn((N, Tl, 832, 7, 7), generator=g).relu()
    tubes, targets = synth.make_loss_case("c3", cfg.num_classes)[3:5]
    tubes, targets = tubes[:N], targets[:N]
    sd = synth.cls_head_state_dict(100, cfg) if cls_only else synth.head_state_dict(100, cfg)
    net = _train_head(cfg, sd, cls_only)
    ctx_dev, ctx_ref = None, None
    if form == "module":
        ctx_ref = torch.randn((N, 1024, Tl, 1, 1), generator=g).relu()
        ctx_dev = ctx_ref.cuda()
    elif form == "cls_tuple":
        B, t0 = 2, 1
        frames = torch.randn((B, Tl + 2, 1024), generator=g).relu()
        clip = torch.tensor([0, 1, 1, 0], dtype=torch.int32)
        ctx_ref = frames[clip.long(), t0:t0 + Tl].permute(0, 2, 1).reshape(N, 1024, Tl, 1, 1).contiguous()
        mean = frames[:, t0:t0 + Tl].mean(1)
        ctx_dev = (mean.cuda(), clip.cuda(), frames.cuda(), t0)
    return cfg, net, sd, feat, tubes, targets, ctx_dev, ctx_ref, cls_only


@pytest.mark.parametrize("form", ["none", "module", "cls_tuple"])
def test_head_forward_backward_with_dropout_matches_oracle(form, monkeypatch):
    from step_b200 import training
    cfg, net, sd, feat, tubes, targets, ctx_dev, ctx_ref, cls_only = _head_case(form)
    gen = _gen()
    gen.manual_seed(2024)
    state = gen.get_state()
    rec = F32.Recorder(monkeypatch)
    r = training.head_forward_backward(net, feat.cuda(), tubes.cuda(), targets.cuda(), context_feat=ctx_dev, loss_scale=1.0,
                                       dropout=True)
    torch.cuda.synchronize()
    off = gen.get_offset()
    gen.set_state(state)
    N, Tl = feat.shape[0], feat.shape[1]
    masks = DO.replay(DO.head_draw_sizes(N, Tl, cfg.fc_dim, cfg.pool_size, ctx_ref is not None, cls_only), P)
    assert gen.get_offset() == off
    sdo = trainable(sd)
    fr = feat.clone().requires_grad_(True)
    cr = ctx_ref.clone().requires_grad_(True) if ctx_ref is not None else None
    prob, loc, first, last, logits = DO.two_branch(fr, sdo, cfg.T, cr, cfg.fc_dim, cfg.pool_size, cls_only, True,
                                                   (masks[0], None if cls_only else masks[1]), P)
    lc, ll, ln = om.two_branch_losses(logits, loc, first, last, tubes, targets, cfg.T, cls_only=cls_only)
    loss = lc.mean() + (0.0 if cls_only else 5.0 * ll.mean() + ln.mean())
    loss.backward()
    assert abs(float(r["loss"]) - float(loss)) <= 1e-5 * abs(float(loss))
    counts = F32.near_decisions(rec.tapes[-1])
    flags = F32.downstream_flags(rec.tapes[-1], counts)
    names = {p: k for k, p in net.named_parameters()}
    assert len(r["grads"]) == (16 if cls_only else 34)
    for p, v in r["grads"].items():
        F32._check_named(v, None, sdo[names[p]].grad, "dropout head", flags.get(p, False))
    F32._check_named(r["feat_grad"], None, fr.grad, "dropout head feat_grad", sum(counts) > 0)
    if form == "module":
        assert rel_l2(r["ctx_grad"], cr.grad) <= F32.L2_TOL
    if form == "cls_tuple":
        # the tuple form's gradient of ContextNet's output, through the draw (context_grad_reduce)
        acc = torch.zeros((2, Tl + 2, 1024), device="cuda")
        own = torch.zeros((N, Tl, 5), device="cuda")
        own[:, 0, 0] = ctx_dev[1].float() * Tl
        training.context_grad_reduce(r["ctx_grad"], own, acc, ctx_dev[3], dropout=r["ctx_dropout"])
        want = torch.zeros((2, Tl + 2, 1024), dtype=torch.float64)
        for i, c in enumerate(ctx_dev[1].tolist()):
            want[c, 1:1 + Tl] += cr.grad[i, :, :, 0, 0].t().double()
        assert rel_l2(acc, want) <= F32.L2_TOL


def test_fp16_head_with_dropout_uses_the_same_masks():
    """The fp16 path draws the same masks (the products in fp32, rounded once to fp16): against the fp32 oracle with the
    replayed masks, every gradient norm within test_gpu_train.py's 2e-2 and every tensor within FP16_L2_TOL relative L2
    (measured on an H100: norms within 8.5e-3, tensors within 6.2e-2 -- fp16 activations and activation gradients against
    fp32 throughout; a wrong mask moves a tensor by O(1))."""
    from step_b200 import training
    cfg, net, sd, feat, tubes, targets, ctx_dev, ctx_ref, cls_only = _head_case("module", fp16=True)
    gen = _gen()
    gen.manual_seed(7)
    state = gen.get_state()
    r = training.head_forward_backward(net, feat.cuda(), tubes.cuda(), targets.cuda(), context_feat=ctx_dev, loss_scale=1024.0,
                                       dropout=True)
    torch.cuda.synchronize()
    gen.set_state(state)
    N, Tl = feat.shape[0], feat.shape[1]
    masks = DO.replay(DO.head_draw_sizes(N, Tl, cfg.fc_dim, cfg.pool_size, True, False), P)
    sdo = trainable(sd)
    prob, loc, first, last, logits = DO.two_branch(feat, sdo, cfg.T, ctx_ref, cfg.fc_dim, cfg.pool_size, False, True, masks, P)
    lc, ll, ln = om.two_branch_losses(logits, loc, first, last, tubes, targets, cfg.T)
    (lc.mean() + 5.0 * ll.mean() + ln.mean()).backward()
    names = {p: k for k, p in net.named_parameters()}
    worst = 0.0
    for p, v in r["grads"].items():
        ref = sdo[names[p]].grad.double()
        got = v.detach().cpu().double()
        rn, gn = float(ref.norm()), float(got.norm())
        worst = max(worst, rel_l2(got, ref))
        assert abs(gn - rn) <= 2e-2 * rn, (names[p], gn, rn)
    assert worst <= FP16_L2_TOL, worst


# ---- train_step ----------------------------------------------------------------------------------------------------------
def _step_case(stage, pool_mode):
    cls = stage == "cls"
    if cls:
        cfg = F32.fp32_cfg(**test_oracle_cls.CLS_CFG, image_size=(64, 64), dropout=P)
        tubes, targets = synth.make_cls_case(cfg, 2, 6, 64, 64, seed=3)
        step_tubes, step_targets = [tubes], [targets]
        heads = [synth.cls_head_state_dict(100, cfg)]
    else:
        cfg = F32.fp32_cfg(**SHIPPED, image_size=(64, 64), dropout=P)
        step_tubes, step_targets = synth.make_train_case(cfg, 2, 9, 64, 64, seed=3)     # 18 tubes: step 3 draws 2.2M elements
        heads = [synth.head_state_dict(100 + i, cfg) for i in range(3)]
    x = synth.make_clips(2, 36, 64, 64, seed=11)
    nets = device_nets(cfg, heads, pool_mode, context=True, cls_only=cls)
    for i in range(len(heads)):
        nets["det_net%d" % i].train()
    return cfg, x, step_tubes, step_targets, nets, heads


def _draw_sizes(cfg, step_tubes, cls):
    return [n for t in step_tubes for n in DO.head_draw_sizes(t.shape[0], t.shape[1], cfg.fc_dim, cfg.pool_size, True, cls)]


@pytest.mark.parametrize("stage,pool_mode", [("shipped", "align"), ("shipped", "pool"), ("cls", "align")])
def test_train_step_with_dropout_matches_oracle_with_replayed_masks(stage, pool_mode, monkeypatch):
    from step_b200 import training
    cfg, x, step_tubes, step_targets, nets, heads = _step_case(stage, pool_mode)
    sizes = _draw_sizes(cfg, step_tubes, stage == "cls")
    assert len(sizes) == (1 if stage == "cls" else 6)
    if stage == "shipped":
        assert max(sizes) > 4 * _n_threads()
    gen = _gen()
    gen.manual_seed(31)
    state = gen.get_state()
    rec = F32.Recorder(monkeypatch)
    r = training.train_step(cfg, nets, x.cuda(), [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets], loss_scale=1.0,
                            dropout=True)
    torch.cuda.synchronize()
    off = gen.get_offset()
    gen.set_state(state)
    masks = DO.replay(sizes, P)
    assert gen.get_offset() == off
    left = DO.patch_heads(monkeypatch, masks, P)
    total, mods = F32._oracle(stage, cfg, x, step_tubes, step_targets, heads, monkeypatch, pool_mode)
    assert not left
    assert abs(float(r["loss"]) - total) <= 1e-4 * abs(total)
    flags, others = {}, 0
    base_params = set(nets["base_net"].parameters())
    for tape in rec.tapes:
        counts = F32.near_decisions(tape)
        f = F32.downstream_flags(tape, counts)
        flags.update(f)
        if not any(p in base_params for p in f):
            others += sum(counts)
    upstream = others > 0 or pool_mode == "pool"
    n = 0
    for m in mods:
        params = dict(nets[m].named_parameters())
        for k, sdv in mods[m].items():
            if sdv.grad is None:
                continue
            p = params[k]
            trunk = m == "base_net"
            F32._check_named(r["grads"][p], None, sdv.grad, "dropout train_step %s %s" % (stage, m.rstrip("012")),
                             flags.get(p, False) or (trunk and upstream), F32.TRAIN_TRUNK_L2_TOL if trunk else F32.CHAIN_L2_TOL)
            n += 1
    assert n == len(r["grads"])


# ---- invariants ----------------------------------------------------------------------------------------------------------
def _run(nets, cfg, x, step_tubes, step_targets, dropout):
    from step_b200 import training
    r = training.train_step(cfg, nets, x.cuda(), [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets], loss_scale=1.0,
                            dropout=dropout)
    torch.cuda.synchronize()
    return r


def test_no_draw_without_training_mode_or_with_p_zero_and_repeatable_draws():
    cfg, x, step_tubes, step_targets, nets, heads = _step_case("shipped", "align")
    gen = _gen()
    gen.manual_seed(5)
    state = gen.get_state()
    r1 = _run(nets, cfg, x, step_tubes, step_targets, True)
    gen.set_state(state)
    r2 = _run(nets, cfg, x, step_tubes, step_targets, True)
    assert all(torch.equal(r1["grads"][p], r2["grads"][p]) for p in r1["grads"])
    heads_ = [nets["det_net%d" % i] for i in range(3)]
    base = _run(nets, cfg, x, step_tubes, step_targets, False)
    assert not all(torch.equal(base["grads"][p], r1["grads"][p]) for p in base["grads"])
    for setup in ("eval", "p0"):
        for h in heads_:
            if setup == "eval":
                h.eval()
            else:
                h.train()
                h.dropout.p = 0.0
        off = gen.get_offset()
        r = _run(nets, cfg, x, step_tubes, step_targets, True)
        assert gen.get_offset() == off, setup
        assert all(torch.equal(base["grads"][p], r["grads"][p]) for p in base["grads"]), setup
        assert torch.equal(base["loss"], r["loss"])


def test_draw_inside_stream_capture_raises():
    from step_b200 import training
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="CUDA graph"):
        with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
            training.dropout_draw("cuda:0", P, 1024)
