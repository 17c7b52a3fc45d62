"""CPU: BatchNorm batch statistics over several ranks (train_step with freeze_stats=False and world_size > 1).

* The DataParallel oracle (_bn_sync_case.py: the trunk and ContextNet per rank chunk with rank 0's running-statistic update,
  the heads over every rank's rows) reproduces the reference's losses, gradients, outputs and running statistics
  (tests/golden/bn_sync_cases.npz: the trunk, ContextNet with the shipped temporal heads, and the class-only stage, each
  with freeze_affine True and False).  Once pinned here it is the checker of the device's synchronised training.
* freeze_stats=True and world_size=1 never take the synchronised path.
* The split entries (step_bn_stats_local_* / step_bn_stats_merge / step_bn_bwd_sums_* / step_bn_bwd_merge_dz_*) refuse bad
  arguments before any launch."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from step_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _bn_stats_case as bc  # noqa: E402
import _bn_sync_case as sc  # noqa: E402
from test_bn_stats_cpu import expect  # noqa: E402


def check_case(g, c, sds, outs):
    """test_bn_stats_cpu.check_case with looser gradient bounds: norms to 1e-3 (not 1e-4) and the leading values ("gh") to
    1e-2 of the tensor's largest leading value (not 1e-3 of each).  With one clip per ContextNet replica, the batch
    statistics of each replica come from 13 x 13 x 9 / 2 pixels, and the ContextNet's smallest gradients (a BatchNorm gamma
    of norm 1.4e-5, leading weight values of 1e-6) differ by up to 2.4e-4 in norm and 1% in value between the reference's
    and the oracle's summation orders."""
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
            assert np.allclose(p.grad.double().norm().numpy(), g[key], rtol=1e-3, atol=1e-12), key
            gh = g["gh:" + c + ":" + rest]
            assert np.allclose(p.grad.reshape(-1)[:8].numpy(), gh, rtol=1e-3, atol=1e-2 * float(np.abs(gh).max())), key
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
def test_trunk_sync_oracle_matches_reference(golden, fa):
    g = golden("bn_sync_cases")
    c = "trunk:fa%d" % fa
    sd = bc.trainable_sd(synth.base_net_state_dict(), fa, convs_too=False)
    loss, cfs = sc.trunk_sync_objective(sd, sc.trunk_inputs())
    loss.backward()
    assert np.allclose(loss.detach().numpy(), g["loss:" + c], rtol=1e-4, atol=1e-8)
    n = check_case(g, c, {"base": sd}, {"conv_feat": torch.cat(cfs)})
    assert n == {"gn": 45 + (0 if fa else 90), "rm": 45, "out": 1}
    assert all(int(v) == 1 for k, v in sd.items() if k.endswith("num_batches_tracked"))


@pytest.mark.parametrize("fa", [1, 0], ids=["freeze_affine", "train_affine"])
@pytest.mark.parametrize("name", ["ctx", "cls"])
def test_heads_sync_oracle_matches_reference(golden, name, fa):
    g = golden("bn_sync_cases")
    c = "%s:fa%d" % (name, fa)
    cfg, cf, step_tubes, step_targets = sc.feat_case(name, bool(fa))
    sds = sc.oracle_sds(name, cfg, fa)
    ranks = sc.split_rows(cfg, cf, step_tubes, step_targets)
    assert all(t.shape[0] == 3 for _, tubes_r, _ in ranks for t in tubes_r)
    loss, losses, named = sc.sync_objective(cfg, sds, ranks, cls_only=name == "cls", from_feat=True)
    loss.backward()
    assert np.allclose(loss.detach().numpy(), g["loss:" + c], rtol=1e-5)
    outs = {"ctx": torch.cat([named["ctx0"], named["ctx1"]])}
    outs.update({k: v for k, v in named.items() if k.endswith(":prob")})
    tags = {"ctx": sds["context_net"]}
    tags.update({"h%d" % i: sds["det_net%d" % i] for i in range(len(step_tubes))})
    n = check_case(g, c, tags, outs)
    assert n["rm"] == 12 * len(tags) and n["out"] == 1 + len(step_tubes)


# ---- which steps synchronise -----------------------------------------------------------------------------------------------
class _Recorder:
    def __init__(self):
        self.calls = []

    def __call__(self, group, rows_total):
        import contextlib
        self.calls.append(rows_total)
        return contextlib.nullcontext()


def test_frozen_statistics_and_one_rank_never_synchronise(monkeypatch):
    """With freeze_stats=True (any world_size) and with world_size=1, train_step reaches the trunk (whose first device use
    fails on CPU nets) without the up-front plan or the sync context; batch statistics with world_size > 1 and no process
    group still raise NotImplementedError."""
    from step_b200 import engine as E, training
    import torch.distributed as dist
    rec = _Recorder()
    monkeypatch.setattr(E, "batch_stats_sync", rec)
    assert E.SYNC_STATS is None
    gathered = []
    monkeypatch.setattr(training, "_sync_plan", lambda *a, **k: gathered.append(a) or [])
    cfg = synth.make_cfg(fp16=False, T=3, max_iter=1, NUM_CHUNKS={1: 1}, no_context=True, image_size=(64, 64),
                         freeze_stats=True)
    nets = synth.device_nets(cfg, [synth.head_state_dict(100, cfg)], "align", device="cpu")
    for k in ("base_net", "det_net0"):
        nets[k].train()
    from step_b200.i3d import Unit3Dpy
    assert not any(m.batch_stats() for net in nets.values() if net is not None for m in net.modules() if isinstance(m, Unit3Dpy))
    assert not dist.is_initialized()
    x = torch.zeros(1, 3, 12, 64, 64)
    tubes, targets = synth.make_train_case(cfg, 1, 2, 64, 64)
    for world in (1, 2):
        # frozen statistics: train_step goes on to the trunk, which needs a GPU; neither the plan nor the context runs
        with pytest.raises(ValueError, match="Expected a cuda device"):
            training.train_step(cfg, nets, x, tubes, targets, world_size=world)
    assert not gathered and not rec.calls
    cfg.freeze_stats = False
    nets = synth.device_nets(cfg, [synth.head_state_dict(100, cfg)], "align", device="cpu")
    for k in ("base_net", "det_net0"):
        nets[k].train()
    with pytest.raises(ValueError, match="Expected a cuda device"):
        training.train_step(cfg, nets, x, tubes, targets, world_size=1)
    assert not gathered and not rec.calls
    with pytest.raises(NotImplementedError, match="world_size"):       # no process group
        training.train_step(cfg, nets, x, tubes, targets, world_size=2)
    assert not gathered and not rec.calls


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


@pytest.mark.parametrize("dtype", ["f16", "f32"])
def test_bn_stats_local_and_merge_refuse_bad_arguments(lib, buf, dtype):
    from step_b200 import _lib as L
    _, p = buf
    V = 8 if dtype == "f16" else 4
    local = getattr(lib, "step_bn_stats_local_" + dtype)

    def call_local(z="p", stats="p", ws="p", M=16, C=2 * V, ld=2 * V, stats_ld=2 * V, ws_bytes=None):
        pick = lambda v: p if v == "p" else v
        if ws_bytes is None:
            ws_bytes = lib.step_bn_stats_workspace_bytes(M, C)
        return local(pick(z), ld, M, C, pick(stats), stats_ld, pick(ws), ws_bytes, None)
    for kw in (dict(z=None), dict(stats=None), dict(ws=None), dict(M=0, ws_bytes=64), dict(C=0, ws_bytes=64),
               dict(stats_ld=V)):
        expect(lib, call_local(**kw), "bn_stats_local: bad arguments")
    for kw in (dict(C=V + V // 2, ld=2 * V), dict(ld=2 * V + 2), dict(C=2 * V, ld=V)):
        expect(lib, call_local(**kw), "bn_stats_local", "multiples of %d" % V)
    expect(lib, call_local(z=ctypes.c_void_p(p.value + 4)), "16-byte aligned")
    expect(lib, call_local(ws_bytes=lib.step_bn_stats_workspace_bytes(16, 2 * V) - 4), "workspace", code=L.E_WORKSPACE)
    # one pixel is a rank's share, not an error: the argument checks pass and only the workspace is short
    assert call_local(M=1, ws_bytes=0) == L.E_WORKSPACE

    def call_merge(stats="p", ranks=2, stats_ld=2 * V, M=16, C=2 * V, rm="p", rv="p", out="p", eps=1e-5, momentum=0.1):
        pick = lambda v: p if v == "p" else v
        return lib.step_bn_stats_merge(pick(stats), ranks, stats_ld, M, C, p, p, eps, momentum, pick(rm), pick(rv), pick(out),
                                       p, p, p, None)
    for kw in (dict(stats=None), dict(out=None), dict(ranks=0), dict(C=0), dict(stats_ld=V)):
        expect(lib, call_merge(**kw), "bn_stats_merge: bad arguments")
    for M in (1, 0):
        expect(lib, call_merge(M=M), "Expected more than 1 value per channel when training")
    expect(lib, call_merge(rm=None), "both running statistics or neither")
    expect(lib, call_merge(eps=0.0), "eps")
    expect(lib, call_merge(momentum=1.5), "momentum")


@pytest.mark.parametrize("dtype", ["f16", "f32"])
def test_bn_bwd_sums_and_merge_dz_refuse_bad_arguments(lib, buf, dtype):
    from step_b200 import _lib as L
    _, p = buf
    V = 8 if dtype == "f16" else 4
    sums_fn = getattr(lib, "step_bn_bwd_sums_" + dtype)
    merge = getattr(lib, "step_bn_bwd_merge_dz_" + dtype)

    def call_sums(dy="p", y="p", z="p", mean="p", rstd="p", sums="p", ws="p", M=16, C=2 * V, ld=2 * V, sums_ld=2 * V, relu=1,
                  ws_bytes=None):
        pick = lambda v: p if v == "p" else v
        if ws_bytes is None:
            ws_bytes = lib.step_bn_bwd_sums_workspace_bytes(M, C)
        return sums_fn(pick(dy), ld, pick(y), ld, pick(z), ld, M, C, pick(mean), pick(rstd), relu, 1.0, pick(sums), sums_ld, None,
                       None, pick(ws), ws_bytes, None)
    for kw in (dict(dy=None), dict(y=None), dict(z=None), dict(mean=None), dict(rstd=None), dict(sums=None), dict(ws=None),
               dict(M=0, ws_bytes=64), dict(sums_ld=V)):
        expect(lib, call_sums(**kw), "bn_bwd_sums: bad arguments")
    for kw in (dict(C=V + V // 2, ld=2 * V), dict(ld=2 * V + 2), dict(C=2 * V, ld=V)):
        expect(lib, call_sums(**kw), "bn_bwd_sums", "multiples of %d" % V)
    expect(lib, call_sums(z=ctypes.c_void_p(p.value + 8)), "16-byte aligned")
    need = lib.step_bn_bwd_sums_workspace_bytes(16, 2 * V)
    assert need == 2 * 2 * V * 4                              # one chunk of (sum g, sum g xhat)
    expect(lib, call_sums(ws_bytes=need - 4), "workspace", code=L.E_WORKSPACE)
    assert call_sums(M=1, ws_bytes=0) == L.E_WORKSPACE        # one pixel is a rank's share
    assert call_sums(y=None, relu=0, ws_bytes=need - 4) == L.E_WORKSPACE

    def call_merge(sums="p", ranks=2, sums_ld=2 * V, M_total=32, dy="p", y="p", z="p", mean="p", rstd="p", gamma="p", dz="p",
                   ws="p", M=16, C=2 * V, ld=2 * V, relu=1, ws_bytes=None):
        pick = lambda v: p if v == "p" else v
        if ws_bytes is None:
            ws_bytes = lib.step_bn_bwd_merge_dz_workspace_bytes(C)
        return merge(pick(sums), ranks, sums_ld, M_total, pick(dy), ld, pick(y), ld, pick(z), ld, M, C, pick(mean), pick(rstd),
                     pick(gamma), relu, pick(dz), ld, pick(ws), ws_bytes, None)
    for kw in (dict(sums=None), dict(dy=None), dict(y=None), dict(z=None), dict(mean=None), dict(rstd=None), dict(gamma=None),
               dict(dz=None), dict(ws=None), dict(ranks=0), dict(M=0), dict(sums_ld=V)):
        expect(lib, call_merge(**kw), "bn_bwd_merge_dz: bad arguments")
    for kw in (dict(M_total=1, M=1), dict(M_total=8)):
        expect(lib, call_merge(**kw), "Expected more than 1 value per channel when training")
    for kw in (dict(C=V + V // 2, ld=2 * V), dict(ld=2 * V + 2)):
        expect(lib, call_merge(**kw), "bn_bwd_merge_dz", "multiples of %d" % V)
    expect(lib, call_merge(dz=ctypes.c_void_p(p.value + 8)), "16-byte aligned")
    assert lib.step_bn_bwd_merge_dz_workspace_bytes(2 * V) == 3 * 2 * V * 4 and lib.step_bn_bwd_merge_dz_workspace_bytes(0) == 0
    expect(lib, call_merge(ws_bytes=3 * 2 * V * 4 - 4), "workspace", code=L.E_WORKSPACE)
