"""CPU: the pieces of the modules' autograd path that need no GPU.

* step_head_outputs_bwd_f32 (the head's tail backward from upstream gradients) is exported and refuses bad arguments with
  STEP_E_ARG before any launch (host addresses that are never dereferenced).
* The parameters each autograd Function takes (step_b200.autograd.trainable) are, module by module, the tensors train_step
  trains: the reference's get_params groups of the shipped configuration (freeze_affine True and False) and of the
  class-only stage (freeze_affine True; with False, those plus every BatchNorm gamma and beta)."""
import ctypes
import os

import numpy as np
import pytest

from step_b200 import synth
from step_b200 import _lib as L

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SHIPPED_CFG = synth.WORKLOADS["shipped"].cfg
CLS_CFG = synth.WORKLOADS["cls"].cfg


@pytest.fixture(scope="module")
def lib():
    return L.lib()


@pytest.fixture(scope="module")
def buf():
    b = (ctypes.c_char * (1 << 16))()
    addr = (ctypes.addressof(b) + 15) & ~15
    return b, ctypes.c_void_p(addr)


def test_head_outputs_bwd_is_exported():
    assert "step_head_outputs_bwd_f32" in L.exported_symbols()


def test_head_outputs_bwd_rejects_bad_arguments(lib, buf):
    _, p = buf

    def call(N=4, cls=60, T_len=9, T=3, Tc=3, cls_only=0, logits="p", loc="p", first="p", last="p", tubes="p", targets="p",
             dlogits="p", dloc="p", dfirst="p", dlast="p"):
        pick = lambda v: p if v == "p" else v
        return lib.step_head_outputs_bwd_f32(pick(logits), pick(loc), pick(first), pick(last), pick(tubes), pick(targets), N, cls,
                                             T_len, T, Tc, cls_only, None, None, None, None, None, None, None, pick(dlogits),
                                             pick(dloc), pick(dfirst), pick(dlast), None)

    def expect(rc, *words):
        assert rc == L.E_ARG
        msg = lib.step_last_error().decode()
        for w in ("head_outputs_bwd",) + words:
            assert w in msg, (w, msg)

    for kw in (dict(N=0), dict(cls=0), dict(T=0), dict(T_len=2), dict(T_len=8), dict(N=0, cls_only=1), dict(cls=-1, cls_only=1)):
        expect(call(**kw), "bad shape")
    for kw in (dict(Tc=1), dict(Tc=4, T_len=3)):
        expect(call(**kw), "chunk slices out of range")
    for kw in (dict(loc=None), dict(first=None), dict(last=None), dict(tubes=None), dict(dloc=None), dict(dfirst=None),
               dict(dlast=None)):
        expect(call(**kw), "null pointer")
    for kw in (dict(logits=None), dict(targets=None), dict(dlogits=None), dict(cls_only=1, logits=None), dict(cls_only=1, dlogits=None)):
        expect(call(**kw), "null pointer")


def _function_params(nets):
    """{(module key, parameter name)} of the parameters each module's Function takes."""
    from step_b200 import autograd
    out = []
    for k, net in nets.items():
        names = {id(p): n for n, p in net.named_parameters()}
        out += [(k, names[id(p)]) for p in autograd.trainable(net)]
    assert len(out) == len(set(out))
    return out


def _fixture(name):
    g = np.load(os.path.join(GOLDEN, name))
    return {(str(m), str(n)) for m, n in zip(g["module"], g["name"])}


def _shipped(freeze_affine):
    import step_b200
    cfg = synth.make_cfg(fp16=True, **SHIPPED_CFG, image_size=(64, 64), freeze_affine=freeze_affine)
    nets = {"base_net": step_b200.BaseNet(cfg), "context_net": step_b200.ContextNet(cfg)}
    for i in range(3):
        nets["det_net%d" % i] = step_b200.TwoBranchNet(cfg)
    return nets


def _cls(freeze_affine):
    import step_b200
    cfg = synth.make_cfg(fp16=False, **CLS_CFG, image_size=(64, 64), freeze_affine=freeze_affine)
    return {"base_net": step_b200.BaseNet(cfg), "context_net": step_b200.ContextNet(cfg),
            "det_net0": step_b200.TwoBranchNet(cfg, cls_only=True)}


@pytest.mark.parametrize("freeze_affine,fixture,count", [(True, "shipped_param_groups.npz", 159),
                                                         (False, "bn_affine_param_groups.npz", 345)])
def test_full_head_functions_take_the_trained_parameters(freeze_affine, fixture, count):
    got = _function_params(_shipped(freeze_affine))
    assert len(got) == count
    assert set(got) == _fixture(fixture)


@pytest.mark.parametrize("freeze_affine", [True, False])
def test_class_only_functions_take_the_trained_parameters(freeze_affine):
    nets = _cls(freeze_affine)
    got = set(_function_params(nets))
    want = _fixture("cls_param_groups.npz")
    assert len(want) == 73
    if not freeze_affine:   # every BatchNorm's gamma and beta trains too
        want |= {(k, n) for k, net in nets.items() for n, _ in net.named_parameters() if "batch3d" in n}
        assert len(want) > 73
    assert got == want
