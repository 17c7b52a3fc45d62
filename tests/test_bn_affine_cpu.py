"""CPU: BatchNorm affine training (freeze_affine=False, BatchNorm statistics frozen).

* The oracle's functional autograd (oracle/model.py), with the batch3d weight / bias entries made trainable, reproduces the
  reference's gradients of every BatchNorm gamma and beta (tests/golden/bn_affine_grads.npz: trunk, ContextNet with the
  shipped temporal heads, the class-only head and ContextNet; head_grads.npz: the head case c1).  Once pinned here the
  oracle is the element-level checker of the device's BatchNorm gradients.
* step_b200's nets built with freeze_affine=False train, name for name and in order, the tensors of the reference's
  get_params groups (tests/golden/bn_affine_param_groups.npz), and step_b200.optim.Adam takes those groups.
* step_act_bn_bwd_f16 / _f32 refuse bad arguments before any launch (host addresses that are never dereferenced)."""
import ctypes
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import model as om
from step_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_oracle_cls  # noqa: E402
import test_oracle_context  # noqa: E402
from test_optim_cpu import SHIPPED_ARGS, SHIPPED_CFG, reference_solver  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bn_affine_param_groups.npz")


def bn_trainable(sd, convs_too=True):
    """A copy of the state dict sd in which every float tensor but the running statistics requires grad (BatchNorm's gamma
    and beta included); convs_too=False: only the conv weights and the BatchNorm affine (the trunk's trainable set)."""
    def train(k, v):
        if not v.is_floating_point() or "running_" in k:
            return False
        return convs_too or k.endswith("conv3d.weight") or "batch3d" in k
    return {k: v.clone().requires_grad_(train(k, v)) for k, v in sd.items()}


def check_bn(g, prefix, sds):
    """Every BatchNorm entry 'gn:<prefix><tag>:<name>' of the golden g against the .grad of sds[tag][name]."""
    checked = 0
    for key in g.files:
        if not key.startswith("gn:" + prefix):
            continue
        tag, k = key[3 + len(prefix):].split(":", 1)
        assert "batch3d" in k, key
        p = sds[tag][k]
        assert p.grad is not None, key
        ref = float(g[key][0])
        assert np.allclose(p.grad.double().norm().numpy(), g[key], rtol=1e-4, atol=1e-12), key
        assert np.allclose(p.grad.reshape(-1)[:8].numpy(), g["gh:" + key[3:]], rtol=1e-3, atol=1e-6 * ref), key
        checked += 1
    return checked


def test_trunk_bn_gradients_oracle_matches_reference(golden):
    g = golden("bn_affine_grads")
    sd = bn_trainable(synth.base_net_state_dict(), convs_too=False)
    x = synth.make_clips(1, 8, 64, 64, seed=4321)
    cf = om.base_net(x, sd)
    proj = torch.randn(cf.shape, generator=torch.Generator().manual_seed(99))
    loss = (cf * proj).sum() / cf.numel()
    loss.backward()
    assert np.allclose(loss.detach().numpy(), g["loss:trunk"], rtol=1e-4, atol=1e-8)
    assert check_bn(g, "trunk:", {"base": sd}) == 90        # gamma and beta of the 45 Unit3D of the trunk


def test_context_heads_bn_gradients_oracle_matches_reference(golden):
    g = golden("bn_affine_grads")
    cfg, cf, step_tubes, step_targets = test_oracle_context.golden_case()
    sd_ctx = bn_trainable(synth.context_net_state_dict())
    sds = [bn_trainable(synth.head_state_dict(100 + i, cfg)) for i in range(3)]
    loss, _, _ = test_oracle_context.oracle_objective(cf.requires_grad_(True), sd_ctx, sds, cfg, step_tubes, step_targets,
                                                      pooled_leaves=True)
    loss.backward()
    assert np.allclose(loss.detach().numpy(), g["loss:ctx"], rtol=1e-5)
    assert check_bn(g, "ctx:", {"ctx": sd_ctx, "h0": sds[0], "h1": sds[1], "h2": sds[2]}) == 24 + 3 * 24


def test_cls_head_bn_gradients_oracle_matches_reference(golden):
    g = golden("bn_affine_grads")
    cfg, cf, flat_tubes, flat_targets = test_oracle_cls.golden_case()
    sd_ctx = bn_trainable(synth.context_net_state_dict())
    sd = bn_trainable(synth.cls_head_state_dict(100, cfg))
    loss = test_oracle_cls.cls_objective(cf.requires_grad_(True), sd_ctx, sd, cfg, flat_tubes, flat_targets, pooled_leaf=True)[0]
    loss.backward()
    assert np.allclose(loss.detach().numpy(), g["loss:cls"], rtol=1e-5)
    assert check_bn(g, "cls:", {"ctx": sd_ctx, "h0": sd}) == 24 + 24


def test_head_bn_gradients_oracle_matches_reference(golden):
    """head_grads.npz trained every parameter of the head, BatchNorm's included: its 24 BatchNorm entries."""
    g = golden("head_grads")
    T_, chunks, _, _ = synth.LOSS_CASES["c1"]
    cfg = synth.make_cfg(T=T_, max_iter=1, NUM_CHUNKS={1: chunks}, image_size=(112, 112))
    _, _, feat, tb, tg = synth.make_loss_case("c1", cfg.num_classes)
    sd = bn_trainable(synth.head_state_dict(100, cfg))
    prob, loc, first, last, logits = om.two_branch(feat.clone(), sd, cfg.T, None, cfg.fc_dim, cfg.pool_size, return_logits=True)
    lc, ll, ln = om.two_branch_losses(logits, loc, first, last, tb, tg, cfg.T)
    (lc.mean() + ll.mean() * 5.0 + ln.mean() * 1.0).backward()
    checked = 0
    for key in g.files:
        if key.startswith("gn:") and "batch3d" in key:
            k = key[3:]
            ref = float(g[key][0])
            assert np.allclose(sd[k].grad.double().norm().numpy(), g[key], rtol=1e-4, atol=1e-12), k
            assert np.allclose(sd[k].grad.reshape(-1)[:8].numpy(), g["gh:" + k], rtol=1e-3, atol=1e-6 * ref), k
            checked += 1
    assert checked == 24


# ---- the parameter groups -----------------------------------------------------------------------------------------------
def affine_modules():
    """The step_b200 modules of the shipped configuration built with freeze_affine=False (uninitialised weights; CPU)."""
    import step_b200
    cfg = synth.make_cfg(fp16=True, **SHIPPED_CFG, image_size=(64, 64), freeze_affine=False)
    nets = {"base_net": step_b200.BaseNet(cfg), "context_net": step_b200.ContextNet(cfg)}
    for i in range(3):
        nets["det_net%d" % i] = step_b200.TwoBranchNet(cfg)
    return nets


def affine_groups(nets, lr_scale=1.0):
    """The reference's get_params groups for the shipped configuration with freeze_affine=False, from the fixture."""
    g = np.load(GOLDEN)
    named = {k: dict(n.named_parameters()) for k, n in nets.items()}
    return [{"params": [named[str(m)][str(n)]], "lr": float(lr) * lr_scale, "weight_decay": float(wd)}
            for m, n, lr, wd in zip(g["module"], g["name"], g["lr"], g["weight_decay"])]


def test_freeze_affine_false_trains_the_reference_groups():
    from step_b200 import optim
    nets = affine_modules()
    g = np.load(GOLDEN)
    groups = affine_groups(nets)
    trainable = [p for n in nets.values() for p in n.parameters() if p.requires_grad]
    assert len(groups) == len(trainable) == 159 + 186          # the 159 of freeze_affine=True and 93 BatchNorms' gamma / beta
    assert {id(gr["params"][0]) for gr in groups} == {id(p) for p in trainable}
    assert sum("batch3d" in str(n) for n in g["name"]) == 186
    assert [gr["params"][0].numel() for gr in groups] == g["numel"].tolist()
    # the reference's rates: a BatchNorm's gamma takes its layer's rate and weight decay, beta twice the rate and none
    for m, n, lr, wd in zip(g["module"], g["name"], g["lr"], g["weight_decay"]):
        if str(n).endswith("batch3d.bias"):
            assert wd == 0.0
        elif str(n).endswith("batch3d.weight"):
            assert wd == SHIPPED_ARGS["weight_decay"]
    opt = optim.Adam(groups, lr=1e-4)
    assert len(opt.param_groups) == 345
    # freeze_affine=True still trains none of them
    import step_b200
    frozen = step_b200.BaseNet(synth.make_cfg(fp16=True, **SHIPPED_CFG, image_size=(64, 64)))
    assert not any(p.requires_grad for k, p in frozen.named_parameters() if "batch3d" in k)


def test_reference_get_params_orders_the_step_b200_modules_as_the_fixture():
    solver = reference_solver()
    nets = affine_modules()
    owner = {id(p): (k, n) for k, net in nets.items() for n, p in net.named_parameters()}
    got = solver.get_params(nets, SimpleNamespace(**SHIPPED_ARGS))
    g = np.load(GOLDEN)
    assert len(got) == len(g["name"]) == 345
    for grp, m, n, lr, wd in zip(got, g["module"], g["name"], g["lr"], g["weight_decay"]):
        assert owner[id(grp["params"][0])] == (str(m), str(n))
        assert grp["lr"] == lr and grp["weight_decay"] == wd, (str(m), str(n))


# ---- argument checks of step_act_bn_bwd_* -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from step_b200 import _lib as L
    return L.lib()


@pytest.fixture(scope="module")
def buf():
    b = (ctypes.c_char * (1 << 16))()
    addr = (ctypes.addressof(b) + 15) & ~15
    return b, ctypes.c_void_p(addr)


def expect(lib, rc, *words, code=None):
    from step_b200 import _lib as L
    assert rc == (L.E_ARG if code is None else code)
    msg = lib.step_last_error().decode()
    for w in words:
        assert w in msg, (w, msg)


@pytest.mark.parametrize("dtype", ["f16", "f32"])
def test_act_bn_bwd_refuses_bad_arguments(lib, buf, dtype):
    _, p = buf
    V = 8 if dtype == "f16" else 4
    fn = getattr(lib, "step_act_bn_bwd_" + dtype)

    def call(dy="p", y="p", dz="p", dres=None, beta="p", gamma="p", dgamma="p", dbeta="p", ws="p", M=16, C=2 * V, ld=2 * V,
             dres_ld=0, ws_bytes=None):
        pick = lambda v: p if v == "p" else v
        if ws_bytes is None:
            ws_bytes = lib.step_act_bn_bwd_workspace_bytes(M, C)
        return fn(pick(dy), ld, pick(y), ld, None, 1, M, C, pick(dz), ld, pick(dres), dres_ld, pick(beta), pick(gamma), 1.0,
                  pick(dgamma), pick(dbeta), pick(ws), ws_bytes, None)
    for kw in (dict(dy=None), dict(y=None), dict(dz=None), dict(beta=None), dict(gamma=None), dict(ws=None),
               dict(dgamma=None, dbeta=None), dict(M=0), dict(C=0, ws_bytes=64)):
        expect(lib, call(**kw), "act_bn_bwd: bad arguments")
    for kw in (dict(C=V + V // 2, ld=2 * V), dict(ld=2 * V + 2), dict(C=2 * V, ld=V), dict(dres="p", dres_ld=V + 1)):
        expect(lib, call(**kw), "act_bn_bwd", "multiples of %d" % V)
    expect(lib, call(y=ctypes.c_void_p(p.value + 4)), "16-byte aligned")
    expect(lib, call(dres=ctypes.c_void_p(p.value + 8), dres_ld=2 * V), "16-byte aligned")
    need = lib.step_act_bn_bwd_workspace_bytes(16, 2 * V)
    assert need == 2 * 2 * V * 4                              # one chunk of (sum g, sum g (y - beta)) per channel
    from step_b200 import _lib as L
    expect(lib, call(ws_bytes=need - 4), "workspace", code=L.E_WORKSPACE)


def test_act_bn_bwd_workspace_follows_the_pixel_count_only(lib):
    assert lib.step_act_bn_bwd_workspace_bytes(0, 64) == 0 and lib.step_act_bn_bwd_workspace_bytes(100, 0) == 0
    assert lib.step_act_bn_bwd_workspace_bytes(1, 64) == 2 * 64 * 4
    assert lib.step_act_bn_bwd_workspace_bytes(257, 64) == 2 * 2 * 64 * 4
    big = 2 * 36 * 200 * 200 // 2
    assert lib.step_act_bn_bwd_workspace_bytes(big, 64) == lib.step_act_bn_bwd_workspace_bytes(10 * big, 64) == 512 * 2 * 64 * 4
