"""GPU: BatchNorm affine training with frozen statistics (freeze_affine=False, freeze_stats=True).

  * per launch, fp16 and fp32: step_act_bn_bwd_* writes dz and dres bit for bit as step_act_bwd_* does, and dgamma / dbeta
    within their fp32 accumulation bound of float64 on the same operands, bit-identical from run to run, at every
    BatchNorm layer shape of the shipped step (2 clips of 36x400x400, the channel slices the forward writes) and at the
    edges: M = 1, the narrowest C, a slice with ld > C and an offset, a residual, negative and small gamma, and gamma = 0
    with beta <= 0 (exactly 0);
  * per module, fp16: the heads, the trunk, ContextNet and the class-only head built with freeze_affine=False against the
    reference's gradients (bn_affine_grads.npz, head_grads.npz) and the oracle's autograd, at the tolerances the other
    parameters of those modules are held to;
  * train_step, fp32 (shipped configuration, ROIPool, context on, Adam over the reference's get_params groups,
    loss_scale=1.0) against the oracle, with the near-decision rule of the fp32 training tests; the forward after the
    update against the oracle's forward with the updated parameters; one fp16 step with a LossScaler;
  * selection (gamma only, beta only) and the refusal of gamma == 0 with beta > 0.

Bound of dgamma / dbeta: each term is one fp32 product (and one subtraction); a thread adds its ceil(chunk / rows) terms in
order, the block adds its `rows` partial sums, the reduce adds the chunks, and the result is scaled and divided once:
n = ceil(chunk / rows) + rows + chunks + 4 roundings of at most u |terms| (u = 2^-24)."""
import math
import os
import sys

import pytest
import torch

from oracle import model as om
from step_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_oracle_cls  # noqa: E402
import test_oracle_context  # noqa: E402
from _train_case import SHIPPED, device_head, device_nets, rel_l2  # noqa: E402
from test_bn_affine_cpu import affine_groups, bn_trainable  # noqa: E402
from test_gpu_train_fp32 import (CHAIN_L2_TOL, L2_TOL, TRAIN_TRUNK_L2_TOL, Recorder, downstream_flags,  # noqa: E402
                                 near_decisions)

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -24
WORST = {}


def _note(kind, v):
    WORST[kind] = max(WORST.get(kind, 0.0), v)


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    print("\nBatchNorm affine, worst ratios / errors:", {k: "%.2e" % v for k, v in sorted(WORST.items())})


# ---- the launch --------------------------------------------------------------------------------------------------------
def bn_terms(M, C, V):
    """Roundings on the path of one term (the kernel's plan: chunks of >= 256 pixels, at most 512 chunks, 256 threads over
    C / V vectors times 256 // (C / V) pixels)."""
    chunks = min(math.ceil(M / 256), 512)
    chunk = math.ceil(M / chunks)
    cols = min(C // V, 256)
    rows = 256 // cols
    return math.ceil(chunk / rows) + rows + chunks + 4


def run_launch(f16, M, C, ld, coff, gamma, beta, relu=True, residual=False, loss_scale=1.0, seed=0):
    """One step_act_bn_bwd_* call on seeded operands (y formed as relu(gamma * xhat + beta) and stored), beside
    step_act_bwd_* on the same operands: returns (dz, dres, dgamma, dbeta, dz_ref, dres_ref, y, dy)."""
    from step_b200 import _lib as L
    lib = L.lib()
    dt = torch.float16 if f16 else torch.float32
    gen = torch.Generator(device="cuda").manual_seed(seed)
    gamma = gamma.float().cuda().contiguous()
    beta = beta.float().cuda().contiguous()
    var = torch.rand(C, device="cuda", generator=gen) + 0.5
    scale = (gamma / torch.sqrt(var + 1e-3)).contiguous()
    y = torch.randn((M, ld), device="cuda", generator=gen).to(dt)
    xhat = torch.randn((M, C), device="cuda", generator=gen)
    pre = gamma * xhat + beta
    y[:, coff:coff + C] = (torch.relu(pre) if relu else pre).to(dt)
    dy = (torch.randn((M, ld), device="cuda", generator=gen) * loss_scale * 1e-2).to(dt)
    res0 = torch.randn((M, ld + 8), device="cuda", generator=gen).to(dt) if residual else None
    esz = y.element_size()

    def slc(t, off):
        return L.c_void_p(t.data_ptr() + esz * off)
    dz_ref = torch.full((M, C), float("nan"), device="cuda", dtype=dt)
    dres_ref = res0.clone() if residual else None
    act = lib.step_act_bwd_f16 if f16 else lib.step_act_bwd_f32
    L.check(act(slc(dy, coff), ld, slc(y, coff), ld, L.ptr(scale), int(relu), M, C, L.ptr(dz_ref), C,
                slc(dres_ref, 8) if residual else None, ld + 8 if residual else 0, L.stream()))
    outs = []
    for _ in range(2):
        dz = torch.full((M, C), float("nan"), device="cuda", dtype=dt)
        dres = res0.clone() if residual else None
        dg = torch.full((C,), float("nan"), device="cuda")
        db = torch.full((C,), float("nan"), device="cuda")
        nbytes = lib.step_act_bn_bwd_workspace_bytes(M, C)
        ws = torch.full((nbytes // 4,), float("nan"), device="cuda")
        fn = lib.step_act_bn_bwd_f16 if f16 else lib.step_act_bn_bwd_f32
        L.check(fn(slc(dy, coff), ld, slc(y, coff), ld, L.ptr(scale), int(relu), M, C, L.ptr(dz), C,
                   slc(dres, 8) if residual else None, ld + 8 if residual else 0, L.ptr(beta), L.ptr(gamma), 1.0 / loss_scale,
                   L.ptr(dg), L.ptr(db), L.ptr(ws), nbytes, L.stream()))
        outs.append((dz, dres, dg, db))
    torch.cuda.synchronize()
    (dz, dres, dg, db), (dz2, dres2, dg2, db2) = outs
    assert torch.equal(dg.view(torch.int32), dg2.view(torch.int32)) and torch.equal(db.view(torch.int32), db2.view(torch.int32))
    return dict(dz=dz, dres=dres, dg=dg, db=db, dz_ref=dz_ref, dres_ref=dres_ref, y=y[:, coff:coff + C], dy=dy[:, coff:coff + C],
                gamma=gamma, beta=beta)


def check_launch(f16, M, C, ld, coff, gamma, beta, relu=True, residual=False, loss_scale=1.0, seed=0, kind="launch"):
    r = run_launch(f16, M, C, ld, coff, gamma, beta, relu, residual, loss_scale, seed)
    bits = torch.int16 if f16 else torch.int32
    assert torch.equal(r["dz"].view(bits), r["dz_ref"].view(bits)), "dz differs from step_act_bwd"
    if residual:
        assert torch.equal(r["dres"].view(bits), r["dres_ref"].view(bits)), "dres differs from step_act_bwd"
    y, dy = r["y"].double(), r["dy"].double()
    g = dy * (y > 0) if relu else dy
    b64, g64 = r["beta"].double(), r["gamma"].double()
    t_beta = g
    t_gamma = g * (y - b64)
    n = bn_terms(M, C, 8 if f16 else 4)
    ref_b = t_beta.sum(0) / loss_scale
    ref_g = torch.where(g64 == 0, torch.zeros_like(g64), t_gamma.sum(0) / loss_scale / torch.where(g64 == 0, 1.0, g64))
    bound_b = n * U32 * t_beta.abs().sum(0) / loss_scale + 1e-30
    bound_g = n * U32 * t_gamma.abs().sum(0) / loss_scale / torch.where(g64 == 0, 1.0, g64.abs()) + 1e-30
    eb = (r["db"].double() - ref_b).abs()
    eg = (r["dg"].double() - ref_g).abs()
    _note(kind + " dbeta / bound", float((eb / bound_b).max()))
    _note(kind + " dgamma / bound", float((eg / bound_g).max()))
    assert bool((eb <= bound_b).all()), float((eb / bound_b).max())
    assert bool((eg <= bound_g).all()), float((eg / bound_g).max())
    zero = (g64 == 0) & (b64 <= 0)
    if bool(zero.any()):
        assert bool((r["dg"][zero] == 0).all()) and bool((r["db"][zero] == 0).all())
    return r


@pytest.fixture(scope="module")
def shipped_bn_shapes():
    """(M, C, ld, coff) of every BatchNorm output slice the forward of the shipped step writes: the trunk over 2 clips of
    36x400x400, ContextNet on its output, and a head over 6 tubes of the 9-frame step."""
    from step_b200 import _lib as L, engine as E, training
    from step_b200.engine import Act
    cfg = synth.make_cfg(fp16=True, **SHIPPED, image_size=(400, 400))
    nets = device_nets(cfg, [synth.head_state_dict(100, cfg)], context=True)
    x = synth.make_clips(2, 36, 400, 400, seed=5).cuda()
    tape = []
    with torch.no_grad(), E.recording(tape):
        feat = nets["base_net"].forward_act(x)
        nets["context_net"].forward_act(feat)
        head = nets["det_net0"]
        cat = Act.empty(6, 9, 7, 7, 832 + head.fc_dim, L.F16, "cuda")
        cat.buf.normal_()
        head.forward_act(cat, torch.randn((6, 1024), device="cuda"), None)
    shapes = set()
    for e in tape:
        if e["kind"] != "conv":
            continue
        s2d = isinstance(e["tag"], tuple) and e["tag"][0] == "s2d"
        tags = [e["tag"][1]] if s2d else e["tag"] if isinstance(e["tag"], (list, tuple)) else [e["tag"]]
        for tg, o in zip(tags, [e["out"]] + e["extra_outs"]):
            if getattr(tg, "use_bn", False):
                shapes.add((o.N * o.T * o.H * o.W, o.C, o.ld, o.coff))
    del nets, tape, feat
    torch.cuda.empty_cache()
    return sorted(shapes)


@pytest.mark.parametrize("f16", [True, False], ids=["f16", "f32"])
def test_launch_at_every_bn_shape_of_the_shipped_step(shipped_bn_shapes, f16):
    assert len(shipped_bn_shapes) >= 20 and max(s[0] for s in shipped_bn_shapes) == 2 * 18 * 200 * 200
    for i, (M, C, ld, coff) in enumerate(shipped_bn_shapes):
        gen = torch.Generator().manual_seed(100 + i)
        gamma = torch.rand(C, generator=gen) * 1.5 + 0.1
        beta = torch.randn(C, generator=gen) * 0.5
        check_launch(f16, M, C, ld, coff, gamma, beta, loss_scale=1024.0 if f16 else 1.0, seed=i, kind="shipped")
        torch.cuda.empty_cache()


EDGE_CASES = {
    # name: M, C (in vectors), ld extra vectors, coff vectors, gamma kind, residual, relu
    "m1": (1, 2, 0, 0, "rand", False, True),
    "narrowest_c": (777, 1, 0, 0, "rand", False, True),
    "slice_ld_offset": (3001, 3, 4, 2, "rand", False, True),
    "residual": (1000, 4, 2, 1, "rand", True, True),
    "no_relu": (513, 2, 0, 0, "rand", False, False),
    "negative_and_small_gamma": (4099, 4, 0, 0, "neg_small", False, True),
    "gamma_zero_beta_nonpositive": (2500, 2, 1, 1, "zero", False, True),
    "many_chunks_wide": (300000, 48, 0, 0, "rand", False, True),
}


@pytest.mark.parametrize("f16", [True, False], ids=["f16", "f32"])
@pytest.mark.parametrize("name", list(EDGE_CASES))
def test_launch_edges(name, f16):
    M, cvec, extra, offv, gk, residual, relu = EDGE_CASES[name]
    V = 8 if f16 else 4
    C, ld, coff = cvec * V, (cvec + extra + offv) * V, offv * V
    gen = torch.Generator().manual_seed(7)
    gamma = torch.rand(C, generator=gen) + 0.2
    beta = torch.randn(C, generator=gen) * 0.5
    if gk == "neg_small":
        gamma[0::3] = -gamma[0::3]
        gamma[1::3] = 1e-6 * torch.sign(torch.randn(len(gamma[1::3]), generator=gen))
    if gk == "zero":
        gamma[0::2] = 0.0
        beta[0::2] = -beta[0::2].abs()
        beta[0] = 0.0
    r = check_launch(f16, M, C, ld, coff, gamma, beta, relu=relu, residual=residual, seed=3, kind="edge")
    if gk == "zero":
        assert bool((r["dg"][0::2] == 0).all()) and bool((r["db"][0::2] == 0).all())
        assert bool((r["dg"][1::2] != 0).any())


# ---- modules, fp16 -----------------------------------------------------------------------------------------------------
def affine_cfg(fp16=True, **kw):
    return synth.make_cfg(fp16=fp16, freeze_affine=False, **kw)


def check_against(got, sd, g_norm, ntol, ttol, kind):
    """Every returned tensor against the oracle's autograd (relative L2 within ttol) and, where the golden holds it, its norm
    within ntol.  Returns the number of BatchNorm tensors checked."""
    n_bn = 0
    for k, v in got.items():
        assert tuple(v.shape) == tuple(sd[k].shape), k
        ref = sd[k].grad
        rel = rel_l2(v, ref)
        _note(kind + " L2", rel)
        assert rel <= ttol, (kind, k, rel)
        ref_n = g_norm(k)
        if ref_n is not None:
            gn = float(v.double().norm())
            _note(kind + " norm", abs(gn - ref_n) / ref_n)
            assert abs(gn - ref_n) <= ntol * ref_n, (kind, k, gn, ref_n)
        n_bn += "batch3d" in k
    return n_bn


def test_fp16_head_bn_gradients(golden):
    from step_b200 import training
    g = golden("head_grads")
    T_, chunks, _, _ = synth.LOSS_CASES["c1"]
    cfg = affine_cfg(T=T_, max_iter=1, NUM_CHUNKS={1: chunks}, image_size=(112, 112))
    _, _, feat, tb, tg = synth.make_loss_case("c1", cfg.num_classes)
    net = device_head(cfg, synth.head_state_dict(100, cfg))
    r = training.head_forward_backward(net, feat.cuda(), tb.cuda(), tg.cuda())
    torch.cuda.synchronize()
    sd = bn_trainable(synth.head_state_dict(100, cfg))
    prob, loc, first, last, logits = om.two_branch(feat.clone(), sd, cfg.T, None, cfg.fc_dim, cfg.pool_size, return_logits=True)
    lc, ll, ln = om.two_branch_losses(logits, loc, first, last, tb, tg, cfg.T)
    (lc.mean() + ll.mean() * 5.0 + ln.mean() * 1.0).backward()
    names = {p: k for k, p in net.named_parameters()}
    got = {names[p]: v for p, v in r["grads"].items()}
    assert len(got) == 34 + 24
    assert check_against(got, sd, lambda k: float(g["gn:" + k][0]), 3e-2, 8e-2, "fp16 head") == 24


def test_fp16_trunk_bn_gradients(golden):
    """The trunk's fp16 bounds are those of test_gpu_train.py's trunk test (fp16 storage of activations and their gradients
    compounds through 45 layers): norms within 1e-1, tensors within 1.5e-1."""
    import step_b200
    from step_b200 import training
    g = golden("bn_affine_grads")
    cfg = affine_cfg(T=2, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(64, 64))
    net = step_b200.BaseNet(cfg)
    net.load_state_dict(synth.base_net_state_dict(), strict=True)
    net = net.cuda().eval()
    x = synth.make_clips(1, 8, 64, 64, seed=4321)
    proj = torch.randn((1, 2, 832, 4, 4), generator=torch.Generator().manual_seed(99))
    numel = proj.numel()
    feat, grads = training.trunk_forward_backward(net, x.cuda(), lambda f: (proj / numel).permute(0, 1, 3, 4, 2).contiguous().cuda())
    torch.cuda.synchronize()
    sd = bn_trainable(synth.base_net_state_dict(), convs_too=False)
    cf = om.base_net(x.clone(), sd)
    ((cf * proj).sum() / cf.numel()).backward()
    names = {p: k for k, p in net.named_parameters()}
    got = {names[p]: v for p, v in grads.items()}
    assert len(got) == 45 + 90
    gn = lambda k: float(g["gn:trunk:base:" + k][0]) if "batch3d" in k else None
    assert check_against(got, sd, gn, 1e-1, 1.5e-1, "fp16 trunk") == 90


def test_fp16_context_heads_and_context_net_bn_gradients(golden):
    import step_b200
    from step_b200 import _lib as L, training
    from step_b200.networks import to_act
    g = golden("bn_affine_grads")
    cfg, cf, step_tubes, step_targets = test_oracle_context.golden_case()
    cf = cf.requires_grad_(True)
    sd_ctx = bn_trainable(synth.context_net_state_dict())
    sds = [bn_trainable(synth.head_state_dict(100 + i, cfg)) for i in range(3)]
    loss, pooled, ctx = test_oracle_context.oracle_objective(cf, sd_ctx, sds, cfg, step_tubes, step_targets, pooled_leaves=True)
    ctx.retain_grad()
    loss.backward()
    dcfg = affine_cfg(**SHIPPED, image_size=(400, 400))
    for i in range(3):
        t0, tl = training.step_frames(cfg, i + 1)
        flat = step_tubes[i]
        clip = [int(flat[p, 0, 0].item() / tl) for p in range(flat.shape[0])]
        tctx = torch.stack([ctx.detach()[c, :, t0:t0 + tl] for c in clip])
        sd = bn_trainable(synth.head_state_dict(100 + i, cfg))
        pl = pooled[i].detach().clone()
        _, loc, first, last, logits = om.two_branch(pl, sd, cfg.T, tctx, cfg.fc_dim, cfg.pool_size, return_logits=True)
        lc, ll, ln = om.two_branch_losses(logits, loc, first, last, flat, step_targets[i], cfg.T)
        (lc.mean() + 5.0 * ll.mean() + 1.0 * ln.mean()).backward()
        net = device_head(dcfg, synth.head_state_dict(100 + i, dcfg))
        r = training.head_forward_backward(net, pl.cuda(), flat.cuda(), step_targets[i].cuda(), context_feat=tctx.cuda())
        torch.cuda.synchronize()
        names = {p: k for k, p in net.named_parameters()}
        got = {names[p]: v for p, v in r["grads"].items()}
        assert len(got) == 34 + 24
        gn = lambda k: float(g["gn:ctx:h%d:%s" % (i, k)][0]) if "batch3d" in k else None
        assert check_against(got, sd, gn, 3e-2, 8e-2, "fp16 context heads") == 24
    net = step_b200.ContextNet(dcfg)
    net.load_state_dict(synth.context_net_state_dict(), strict=True)
    net = net.cuda().eval()
    c, state = training.context_forward(net, to_act(cf.detach().cuda(), L.F16))
    grads, _g = training.context_backward(state, ctx.grad.view(2, 1024, 9).permute(0, 2, 1).contiguous().cuda(), 1024.0)
    torch.cuda.synchronize()
    names = {p: k for k, p in net.named_parameters()}
    got = {names[p]: v for p, v in grads.items()}
    assert len(got) == 12 + 24
    gn = lambda k: float(g["gn:ctx:ctx:" + k][0]) if "batch3d" in k else None
    assert check_against(got, sd_ctx, gn, 3e-2, 8e-2, "fp16 context_net") == 24


def test_fp16_cls_head_bn_gradients(golden):
    from step_b200 import training
    g = golden("bn_affine_grads")
    cfg, cf, flat_tubes, flat_targets = test_oracle_cls.golden_case()
    ctx = om.context_net(cf, synth.context_net_state_dict(), global_mean=True).detach()
    clip = [int(flat_tubes[p, 0, 0].item() / cfg.T) for p in range(flat_tubes.shape[0])]
    tctx = torch.stack([ctx[c, :, :cfg.T] for c in clip])
    pooled = test_oracle_cls.cls_objective(cf, synth.context_net_state_dict(), synth.cls_head_state_dict(100, cfg), cfg,
                                           flat_tubes, flat_targets, pooled_leaf=True)[2].detach()
    sd = bn_trainable(synth.cls_head_state_dict(100, cfg))
    prob, loc, first, last, logits = om.two_branch(pooled, sd, cfg.T, tctx, cfg.fc_dim, cfg.pool_size, cls_only=True, return_logits=True)
    lc, _, _ = om.two_branch_losses(logits, loc, first, last, flat_tubes, flat_targets, cfg.T, cls_only=True)
    lc.mean().backward()
    dcfg = affine_cfg(**test_oracle_cls.CLS_CFG, image_size=(400, 400))
    net = device_head(dcfg, synth.cls_head_state_dict(100, dcfg), cls_only=True)
    context = (ctx.view(2, 1024, 9).mean(2).cuda(), torch.tensor(clip, dtype=torch.int32, device="cuda"))
    r = training.head_forward_backward(net, pooled.cuda(), flat_tubes.cuda(), flat_targets.cuda(), context_feat=context)
    torch.cuda.synchronize()
    names = {p: k for k, p in net.named_parameters()}
    got = {names[p]: v for p, v in r["grads"].items()}
    assert len(got) == 16 + 24
    gn = lambda k: float(g["gn:cls:h0:" + k][0]) if "batch3d" in k else None
    assert check_against(got, sd, gn, 3e-2, 8e-2, "fp16 cls head") == 24


# ---- selection and refusal ----------------------------------------------------------------------------------------------
def _head_case():
    T_, chunks, _, _ = synth.LOSS_CASES["c1"]
    cfg = affine_cfg(T=T_, max_iter=1, NUM_CHUNKS={1: chunks}, image_size=(112, 112))
    _, _, feat, tb, tg = synth.make_loss_case("c1", cfg.num_classes)
    return cfg, feat.cuda(), tb.cuda(), tg.cuda()


@pytest.mark.parametrize("fp16", [True, False], ids=["f16", "f32"])
def test_only_the_bn_tensors_that_require_grad_get_gradients(fp16):
    from step_b200 import training
    cfg, feat, tb, tg = _head_case()
    cfg.fp16 = fp16
    full = device_head(cfg, synth.head_state_dict(100, cfg))
    r_full = training.head_forward_backward(full, feat, tb, tg)["grads"]
    names = {p: k for k, p in full.named_parameters()}
    ref = {names[p]: v for p, v in r_full.items()}
    for keep in ("weight", "bias"):
        net = device_head(cfg, synth.head_state_dict(100, cfg))
        for k, p in net.named_parameters():
            if "batch3d" in k and not k.endswith(keep):
                p.requires_grad_(False)
        r = training.head_forward_backward(net, feat, tb, tg)["grads"]
        torch.cuda.synchronize()
        nm = {p: k for k, p in net.named_parameters()}
        got = {nm[p]: v for p, v in r.items()}
        bn = [k for k in got if "batch3d" in k]
        assert len(bn) == 12 and all(k.endswith("batch3d." + keep) for k in bn)
        assert len(got) == 34 + 12
        for k, v in got.items():       # the same launches, the same bits
            assert torch.equal(v, ref[k]), k


def test_gamma_zero_with_positive_beta_is_refused_before_any_update():
    from step_b200 import optim, training
    cfg = synth.make_cfg(fp16=False, freeze_affine=False, T=2, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(64, 64))
    x = synth.make_clips(1, 8, 64, 64, seed=11)
    tubes, targets = synth.make_train_case(cfg, 1, 2, 64, 64, seed=3)
    nets = device_nets(cfg, [synth.head_state_dict(100, cfg)])
    bn = nets["base_net"].base_model[5].branch_1[1].batch3d
    with torch.no_grad():
        bn.weight[3] = 0.0
        bn.bias[3] = 0.25
    params = [p for n in nets.values() for p in n.parameters() if p.requires_grad]
    before = [p.detach().clone() for p in params]
    opt = optim.Adam(params, lr=1e-3)
    with pytest.raises(ValueError, match=r"base_net\.base_model\.5\.branch_1\.1\.batch3d"):
        training.train_step(cfg, nets, x.cuda(), [t.cuda() for t in tubes], [t.cuda() for t in targets], loss_scale=1.0,
                            optimizer=opt)
    assert all(torch.equal(p.detach(), b) for p, b in zip(params, before))
    # with beta <= 0 the channel is dead: its gradients are exactly zero and the step runs
    with torch.no_grad():
        bn.bias[3] = -0.25
    r = training.train_step(cfg, nets, x.cuda(), [t.cuda() for t in tubes], [t.cuda() for t in targets], loss_scale=1.0,
                            optimizer=opt)
    torch.cuda.synchronize()
    assert float(r["grads"][bn.weight][3]) == 0.0 and float(r["grads"][bn.bias][3]) == 0.0


# ---- train_step ---------------------------------------------------------------------------------------------------------
def _shipped_case(fp16):
    cfg = affine_cfg(fp16=fp16, **SHIPPED, image_size=(64, 64))
    step_tubes, step_targets = synth.make_train_case(cfg, 2, 3, 64, 64, seed=3)
    heads = [synth.head_state_dict(100 + i, cfg) for i in range(3)]
    x = synth.make_clips(2, 36, 64, 64, seed=11)
    nets = device_nets(cfg, heads, "pool", context=True)
    return cfg, x, step_tubes, step_targets, nets, heads


def _bn_flags(tape, counts):
    """{BatchNorm gamma / beta: True when the entry that owns it or one nearer the loss holds a near decision}."""
    flags = {}
    for j, e in enumerate(tape):
        if e["kind"] != "conv":
            continue
        s2d = isinstance(e["tag"], tuple) and e["tag"][0] == "s2d"
        for tg in [e["tag"][1]] if s2d else e["tag"] if isinstance(e["tag"], (list, tuple)) else [e["tag"]]:
            if getattr(tg, "use_bn", False):
                flags[tg.batch3d.weight] = flags[tg.batch3d.bias] = sum(counts[j:]) > 0
    return flags


def test_fp32_train_step_trains_bn_affine_like_the_oracle(monkeypatch):
    """The shipped configuration on the fp32 path with ROIPool and context, Adam over the reference's get_params groups
    with freeze_affine=False (bn_affine_param_groups.npz), loss_scale=1.0: every BatchNorm gamma and beta gets a gradient
    and changes; every gradient matches the oracle's autograd (L2_TOL, or the chain bounds where a near decision lies
    downstream); the forward after the update equals the oracle's forward with the updated parameters."""
    import test_gpu_train_pool
    from step_b200 import optim, training
    cfg, x, step_tubes, step_targets, nets, heads = _shipped_case(False)
    monkeypatch.setattr(test_oracle_context, "tv_roi_align", test_gpu_train_pool.pool_as_align)
    sd_b = bn_trainable(synth.base_net_state_dict(), convs_too=False)
    sd_ctx = bn_trainable(synth.context_net_state_dict())
    sds = [bn_trainable(sd) for sd in heads]
    cf = om.base_net(x.clone(), sd_b)
    total = test_oracle_context.oracle_objective(cf, sd_ctx, sds, cfg, step_tubes, step_targets)[0]
    total.backward()
    mods = {"base_net": sd_b, "context_net": sd_ctx}
    mods.update({"det_net%d" % i: sd for i, sd in enumerate(sds)})
    groups = affine_groups(nets, 10.0)
    assert len(groups) == 345
    opt = optim.Adam(groups, lr=1e-4)
    bn_params = [(m, k, p) for m in mods for k, p in nets[m].named_parameters() if "batch3d" in k]
    assert len(bn_params) == 186 and all(p.requires_grad for _, _, p in bn_params)
    before = {p: p.detach().clone() for _, _, p in bn_params}
    rec = Recorder(monkeypatch)
    r = training.train_step(cfg, nets, x.cuda(), [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets], loss_scale=1.0,
                            optimizer=opt)
    torch.cuda.synchronize()
    assert not r["skipped"]
    assert abs(float(r["loss"]) - float(total)) <= 1e-4 * abs(float(total))
    assert len(r["grads"]) == 345
    for m, k, p in bn_params:
        assert p in r["grads"] and p.grad is not None, (m, k)
        assert not torch.equal(p.detach(), before[p]), (m, k)
    flags, others = {}, 0
    base_params = set(nets["base_net"].parameters())
    for tape in rec.tapes:
        counts = near_decisions(tape)
        f = downstream_flags(tape, counts)
        f.update(_bn_flags(tape, counts))
        flags.update(f)
        if not any(p in base_params for p in f):
            others += sum(counts)
    upstream = others > 0       # ROIPool's argmax decides every trunk gradient as well
    n = 0
    for m, sdv in mods.items():
        params = dict(nets[m].named_parameters())
        for k, ref in sdv.items():
            if ref.grad is None:
                continue
            p = params[k]
            trunk = m == "base_net"
            rel = rel_l2(r["grads"][p], ref.grad)
            flagged = flags.get(p, False) or trunk
            _note("train_step fp32 %s%s L2" % (m.rstrip("012"), " BatchNorm" if "batch3d" in k else ""), rel)
            assert rel <= (TRAIN_TRUNK_L2_TOL if trunk else CHAIN_L2_TOL) if flagged else L2_TOL, (m, k, rel, flagged, upstream)
            n += 1
    assert n == 345
    # the next forward reads the updated gamma / beta (Unit3Dpy.packed keys its folded scale and shift on their versions)
    sd_new = {k: (dict(nets["base_net"].named_parameters())[k].detach().cpu() if k in dict(nets["base_net"].named_parameters())
                  else v) for k, v in synth.base_net_state_dict().items()}
    with torch.no_grad():
        feat = nets["base_net"](x.cuda())
        ref = om.base_net(x.clone(), sd_new)
        old = om.base_net(x.clone(), synth.base_net_state_dict())
    torch.cuda.synchronize()
    err, moved = rel_l2(feat, ref), rel_l2(old.cuda(), ref)
    _note("forward after the update L2", err)
    assert err <= 1e-4 and moved > 10 * err, (err, moved)


def test_fp16_train_step_with_loss_scaler_updates_bn_affine():
    from step_b200 import optim, training
    cfg, x, step_tubes, step_targets, nets, heads = _shipped_case(True)
    opt = optim.Adam(affine_groups(nets, 10.0), lr=1e-4)
    scaler = optim.LossScaler(init_scale=1024.0)
    bn = [p for m in ("base_net", "context_net", "det_net0") for k, p in nets[m].named_parameters() if "batch3d" in k]
    before = [p.detach().clone() for p in bn]
    r = training.train_step(cfg, nets, x.cuda(), [t.cuda() for t in step_tubes], [t.cuda() for t in step_targets],
                            optimizer=opt, scaler=scaler)
    torch.cuda.synchronize()
    assert not r["skipped"] and r["loss_scale"] == 1024.0
    assert all(bool(torch.isfinite(r["grads"][p]).all()) for p in bn)
    assert all(not torch.equal(p.detach(), b) for p, b in zip(bn, before))
    # the fused 1x1 GEMM of a Mixed block (fp16) re-folds the updated BatchNorms on the next forward
    from step_b200 import _lib as L, engine as E
    mixed = nets["base_net"].base_model[5]
    w, scale, shift = mixed._fused_weights()
    units = (mixed.branch_0, mixed.branch_1[0], mixed.branch_2[0])
    want = torch.cat([E.fold_bn(u.batch3d, None, u.conv3d.out_channels, "cuda")[0] for u in units])
    assert torch.equal(scale, want)
