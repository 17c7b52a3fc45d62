"""CPU: BatchNorm with batch statistics (freeze_stats=False).

* The oracle with its BatchNorms in training mode (_bn_stats_case.py) reproduces the reference's outputs, losses,
  gradients and running statistics after the step (tests/golden/bn_stats_cases.npz: the trunk, ContextNet with the shipped
  temporal heads, and the class-only stage, each with freeze_affine True and False).  Once pinned here the oracle is the
  checker of the device's batch-statistics training.
* Nets built with freeze_stats=True never normalise with batch statistics, whatever their training mode; nets built with
  freeze_stats=False do exactly in training mode.
* step_bn_stats_* / step_bn_apply_* / step_bn_bwd_* refuse bad arguments before any launch."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from step_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _bn_stats_case as bc  # noqa: E402


def check_case(g, c, sds, outs):
    """Every gradient, running-statistic and output entry of case c of the golden g against the oracle's."""
    n = {"gn": 0, "rm": 0, "out": 0}
    for key in g.files:
        kind, rest = key.split(":", 1)
        if not rest.startswith(c + ":"):
            continue
        rest = rest[len(c) + 1:]
        if kind == "gn":
            tag, k = rest.split(":", 1)
            p = sds[tag][k]
            assert p.grad is not None, key
            ref = float(g[key][0])
            assert np.allclose(p.grad.double().norm().numpy(), g[key], rtol=1e-4, atol=1e-12), key
            assert np.allclose(p.grad.reshape(-1)[:8].numpy(), g["gh:" + c + ":" + rest], rtol=1e-3, atol=1e-6 * ref), key
            n["gn"] += 1
        elif kind in ("rm", "rv", "nb"):
            tag, bn = rest.split(":", 1)
            name = {"rm": "running_mean", "rv": "running_var", "nb": "num_batches_tracked"}[kind]
            got = sds[tag][bn + "." + name].detach()
            if kind != "nb":
                got = np.concatenate([got.double().norm().numpy().reshape(1), got[:16].double().numpy()])
            assert np.allclose(got, g[key], rtol=1e-5, atol=1e-7), key
            n["rm"] += kind == "rm"
        elif kind == "out" and rest.endswith(":n"):
            name = rest[:-2]
            t = outs[name].detach().double().reshape(-1)
            assert np.allclose(t.norm().numpy(), g[key], rtol=1e-5), key
            assert np.allclose(t[:64].float().numpy(), g["out:%s:%s:h" % (c, name)], rtol=1e-3, atol=1e-5), key
            n["out"] += 1
    return n


@pytest.mark.parametrize("fa", [1, 0], ids=["freeze_affine", "train_affine"])
def test_trunk_oracle_matches_reference(golden, fa):
    g = golden("bn_stats_cases")
    c = "trunk:fa%d" % fa
    sd = bc.trainable_sd(synth.base_net_state_dict(), fa, convs_too=False)
    loss, cf, _ = bc.trunk_objective(sd)
    loss.backward()
    assert np.allclose(loss.detach().numpy(), g["loss:" + c], rtol=1e-4, atol=1e-8)
    n = check_case(g, c, {"base": sd}, {"conv_feat": cf})
    assert n == {"gn": 45 + (0 if fa else 90), "rm": 45, "out": 1}


@pytest.mark.parametrize("fa", [1, 0], ids=["freeze_affine", "train_affine"])
def test_context_heads_oracle_matches_reference(golden, fa):
    g = golden("bn_stats_cases")
    c = "ctx:fa%d" % fa
    cfg, cf, step_tubes, step_targets = bc.ctx_case(freeze_affine=bool(fa))
    sd_ctx = bc.trainable_sd(synth.context_net_state_dict(), fa)
    sds = [bc.trainable_sd(synth.head_state_dict(100 + i, cfg), fa) for i in range(3)]
    loss, ctx, outs, _ = bc.ctx_objective(cf, sd_ctx, sds, cfg, step_tubes, step_targets)
    loss.backward()
    assert np.allclose(loss.detach().numpy(), g["loss:" + c], rtol=1e-5)
    named = {"ctx": ctx}
    for i, o in enumerate(outs):
        named.update({"h%d:%s" % (i, k): t for k, t in zip(("prob", "loc", "first", "last"), o)})
    n = check_case(g, c, {"ctx": sd_ctx, "h0": sds[0], "h1": sds[1], "h2": sds[2]}, named)
    assert n["rm"] == 4 * 12 and n["out"] == 1 + 3 * 4


@pytest.mark.parametrize("fa", [1, 0], ids=["freeze_affine", "train_affine"])
def test_cls_stage_oracle_matches_reference(golden, fa):
    g = golden("bn_stats_cases")
    c = "cls:fa%d" % fa
    cfg, cf, flat_tubes, flat_targets = bc.cls_case(freeze_affine=bool(fa))
    sd_ctx = bc.trainable_sd(synth.context_net_state_dict(), fa)
    sd = bc.trainable_sd(synth.cls_head_state_dict(100, cfg), fa)
    loss, ctx, prob, _ = bc.cls_objective(cf, sd_ctx, sd, cfg, flat_tubes, flat_targets)
    loss.backward()
    assert np.allclose(loss.detach().numpy(), g["loss:" + c], rtol=1e-5)
    n = check_case(g, c, {"ctx": sd_ctx, "h0": sd}, {"ctx": ctx, "h0:prob": prob})
    assert n["rm"] == 2 * 12 and n["out"] == 2


# ---- which units normalise with batch statistics --------------------------------------------------------------------------
def _nets(freeze_stats):
    import step_b200
    cfg = synth.make_cfg(fp16=True, T=3, no_context=False, image_size=(64, 64), freeze_stats=freeze_stats)
    return [step_b200.BaseNet(cfg), step_b200.ContextNet(cfg), step_b200.TwoBranchNet(cfg),
            step_b200.TwoBranchNet(cfg, cls_only=True)]


def _units(net):
    from step_b200.i3d import Unit3Dpy
    return [m for m in net.modules() if isinstance(m, Unit3Dpy)]


def test_freeze_stats_never_marks_a_unit_for_batch_statistics():
    for net in _nets(True):
        units = _units(net)
        assert units
        # freshly built (training mode), after train(), after eval(), and with the BatchNorms forced back into training mode
        for setup in (lambda: None, lambda: net.train(), lambda: net.eval(), lambda: [u.batch3d.train() for u in units]):
            setup()
            assert not any(u.batch_stats() for u in units)
        net.train()
        assert not any(u.batch3d.training for u in units)      # the reference's train(): BatchNorm back in eval mode


def test_freeze_stats_false_marks_every_unit_in_training_mode_only():
    for net in _nets(False):
        units = _units(net)
        net.train()
        assert all(u.batch_stats() for u in units)
        net.eval()
        assert not any(u.batch_stats() for u in units)


# ---- argument checks ------------------------------------------------------------------------------------------------------
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
def test_bn_stats_refuses_bad_arguments(lib, buf, dtype):
    _, p = buf
    V = 8 if dtype == "f16" else 4
    fn = getattr(lib, "step_bn_stats_" + dtype)

    def call(z="p", gamma="p", beta="p", rm="p", rv="p", out="p", ws="p", M=16, C=2 * V, ld=2 * V, eps=1e-5, momentum=0.1,
             ws_bytes=None):
        pick = lambda v: p if v == "p" else v
        if ws_bytes is None:
            ws_bytes = lib.step_bn_stats_workspace_bytes(M, C)
        return fn(pick(z), ld, M, C, pick(gamma), pick(beta), eps, momentum, pick(rm), pick(rv), pick(out), p, p, p, pick(ws),
                  ws_bytes, None)
    for kw in (dict(z=None), dict(gamma=None), dict(beta=None), dict(out=None), dict(ws=None), dict(C=0, ws_bytes=64)):
        expect(lib, call(**kw), "bn_stats: bad arguments")
    for M in (1, 0):
        expect(lib, call(M=M, ws_bytes=64), "Expected more than 1 value per channel when training")
    expect(lib, call(rm=None), "both running statistics or neither")
    for kw in (dict(C=V + V // 2, ld=2 * V), dict(ld=2 * V + 2), dict(C=2 * V, ld=V)):
        expect(lib, call(**kw), "bn_stats", "multiples of %d" % V)
    expect(lib, call(z=ctypes.c_void_p(p.value + 4)), "16-byte aligned")
    expect(lib, call(eps=0.0), "eps")
    expect(lib, call(momentum=1.5), "momentum")
    need = lib.step_bn_stats_workspace_bytes(16, 2 * V)
    assert need == 3 * 2 * V * 4                               # one chunk of (count, mean, M2) per channel
    from step_b200 import _lib as L
    expect(lib, call(ws_bytes=need - 4), "workspace", code=L.E_WORKSPACE)
    assert call(rm=None, rv=None, ws_bytes=need - 4) == L.E_WORKSPACE   # the running statistics are optional


@pytest.mark.parametrize("dtype", ["f16", "f32"])
def test_bn_apply_refuses_bad_arguments(lib, buf, dtype):
    _, p = buf
    V = 8 if dtype == "f16" else 4
    fn = getattr(lib, "step_bn_apply_" + dtype)

    def call(z="p", scale="p", shift="p", y="p", y1=None, y2=None, M=16, C=3 * V, z_ld=3 * V, y_ld=3 * V, s1=3 * V, s2=3 * V,
             y1_ld=0, y2_ld=0):
        pick = lambda v: p if v == "p" else v
        return fn(pick(z), z_ld, M, C, pick(scale), pick(shift), 1, pick(y), y_ld, s1, pick(y1), y1_ld, s2, pick(y2), y2_ld, None)
    for kw in (dict(z=None), dict(scale=None), dict(shift=None), dict(y=None), dict(M=0)):
        expect(lib, call(**kw), "bn_apply: bad arguments")
    for kw in (dict(s1=V, s2=2 * V), dict(s1=V, s2=2 * V, y1="p", y1_ld=V), dict(s1=0, s2=0), dict(s1=2 * V, s2=V)):
        expect(lib, call(**kw), "need a destination each")
    for kw in (dict(z_ld=2 * V), dict(y_ld=3 * V + 2), dict(s1=V // 2, s2=3 * V, y1="p", y1_ld=3 * V),
               dict(s1=V, s2=2 * V, y1="p", y1_ld=V, y2="p", y2_ld=V // 2)):
        expect(lib, call(**kw), "bn_apply", "multiples of %d" % V)
    expect(lib, call(s1=V, s2=2 * V, y1="p", y1_ld=V, y2=ctypes.c_void_p(p.value + 4), y2_ld=V), "16-byte aligned")


@pytest.mark.parametrize("dtype", ["f16", "f32"])
def test_bn_bwd_refuses_bad_arguments(lib, buf, dtype):
    _, p = buf
    V = 8 if dtype == "f16" else 4
    fn = getattr(lib, "step_bn_bwd_" + dtype)

    def call(dy="p", y="p", z="p", mean="p", rstd="p", gamma="p", dz="p", ws="p", M=16, C=2 * V, ld=2 * V, relu=1,
             ws_bytes=None):
        pick = lambda v: p if v == "p" else v
        if ws_bytes is None:
            ws_bytes = lib.step_bn_bwd_workspace_bytes(M, C)
        return fn(pick(dy), ld, pick(y), ld, pick(z), ld, M, C, pick(mean), pick(rstd), pick(gamma), relu, 1.0, pick(dz), ld,
                  None, None, pick(ws), ws_bytes, None)
    for kw in (dict(dy=None), dict(y=None), dict(z=None), dict(mean=None), dict(rstd=None), dict(gamma=None), dict(dz=None),
               dict(ws=None)):
        expect(lib, call(**kw), "bn_bwd: bad arguments")
    expect(lib, call(M=1, ws_bytes=64), "Expected more than 1 value per channel when training")
    for kw in (dict(C=V + V // 2, ld=2 * V), dict(ld=2 * V + 2), dict(C=2 * V, ld=V)):
        expect(lib, call(**kw), "bn_bwd", "multiples of %d" % V)
    expect(lib, call(z=ctypes.c_void_p(p.value + 8)), "16-byte aligned")
    need = lib.step_bn_bwd_workspace_bytes(16, 2 * V)
    assert need == (2 + 3) * 2 * V * 4                         # one chunk of (sum g, sum g xhat) and three coefficients
    from step_b200 import _lib as L
    expect(lib, call(ws_bytes=need - 4), "workspace", code=L.E_WORKSPACE)
    assert call(y=None, relu=0, ws_bytes=need - 4) == L.E_WORKSPACE   # no ReLU: y is not read


def test_bn_workspaces_follow_the_pixel_count_only(lib):
    for fn, per in ((lib.step_bn_stats_workspace_bytes, 3), (lib.step_bn_bwd_workspace_bytes, None)):
        assert fn(0, 64) == 0 and fn(100, 0) == 0
        big = 2 * 36 * 200 * 200 // 2
        assert fn(big, 64) == fn(10 * big, 64)
    assert lib.step_bn_stats_workspace_bytes(257, 64) == 2 * 3 * 64 * 4
    assert lib.step_bn_bwd_workspace_bytes(2 * 36 * 200 * 200, 64) == (512 * 2 + 3) * 64 * 4
