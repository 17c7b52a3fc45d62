"""The heads' dropout without a GPU:
  * the masked oracle (tests/_dropout_oracle.py) against the reference's own TwoBranchNet in training mode, its nn.Dropout
    replaced by the same fixed masks (two_branch.py:244, 261): forward outputs and autograd gradients, full and class-only
    heads, with and without the context columns.  This pins where the masks apply, their element order, and that the local
    branch reads the undropped downsample output;
  * the argument checks of the step_dropout_* entries, which refuse before any device work (the pointers are 16-byte
    aligned host addresses that are never dereferenced)."""
import ctypes
import os
import sys

import pytest
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _dropout_oracle as DO  # noqa: E402
from _train_case import trainable  # noqa: E402
from oracle import refload  # noqa: E402
from step_b200 import _lib as L  # noqa: E402
from step_b200 import synth  # noqa: E402

P = 0.3


class FixedMasks(nn.Module):
    """nn.Dropout(p) in training mode with the given masks, one per call in call order."""

    def __init__(self, masks, p):
        super().__init__()
        self.masks, self.p, self.calls = list(masks), p, 0

    def forward(self, x):
        m = self.masks[self.calls].view(x.shape)
        self.calls += 1
        return x * m.to(x.dtype) * DO.scale_of(self.p)


def _case(context, cls_only, seed=5):
    cfg = synth.make_cfg(T=3, max_iter=1, NUM_CHUNKS={1: 1}, no_context=not context, image_size=(112, 112), dropout=P)
    N, Tl = 2, 3
    g = torch.Generator().manual_seed(seed)
    feat = torch.randn((N, Tl, 832, 7, 7), generator=g).relu()
    ctx = torch.randn((N, 1024, Tl, 1, 1), generator=g).relu() if context else None
    sizes = DO.head_draw_sizes(N, Tl, cfg.fc_dim, cfg.pool_size, context, cls_only)
    masks = [torch.rand((n,), generator=g) >= P for n in sizes]
    sd = synth.cls_head_state_dict(100, cfg) if cls_only else synth.head_state_dict(100, cfg)
    return cfg, feat, ctx, masks, sd


@pytest.mark.skipif(not refload.available(), reason="needs the reference tree")
@pytest.mark.parametrize("context", [False, True])
@pytest.mark.parametrize("cls_only", [False, True])
def test_masked_oracle_matches_reference_train_mode_dropout(context, cls_only):
    ref = refload.load()
    cfg, feat, ctx, masks, sd = _case(context, cls_only)
    net = ref.models.TwoBranchNet(cfg, cls_only=cls_only) if cls_only else ref.models.TwoBranchNet(cfg)
    net.load_state_dict(sd, strict=True)
    net.train()
    net.device = torch.device("cpu")
    net.dropout = FixedMasks(masks, P)
    f_ref = feat.clone().requires_grad_(True)
    c_ref = ctx.clone().requires_grad_(True) if context else None
    out = net(f_ref, c_ref)
    assert net.dropout.calls == len(masks)
    prob, loc, first, last = out[:4]
    obj = prob.square().sum() + (0 if cls_only else loc.square().sum() + first.sum() + 2.0 * last.sum())
    obj.backward()

    sdo = trainable(sd)
    f_o = feat.clone().requires_grad_(True)
    c_o = ctx.clone().requires_grad_(True) if context else None
    mo = (masks[0], None if cls_only else masks[1])
    prob_o, loc_o, first_o, last_o = DO.two_branch(f_o, sdo, cfg.T, c_o, cfg.fc_dim, cfg.pool_size, cls_only, dropout_masks=mo, p=P)
    obj_o = prob_o.square().sum() + (0 if cls_only else loc_o.square().sum() + first_o.sum() + 2.0 * last_o.sum())
    obj_o.backward()

    tol = dict(rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(prob_o, prob, **tol)
    if not cls_only:
        for a, b in ((loc_o, loc), (first_o, first), (last_o, last)):
            torch.testing.assert_close(a, b, **tol)
    params = dict(net.named_parameters())
    checked = 0
    for k, v in sdo.items():
        if v.grad is None or k not in params or params[k].grad is None:
            continue
        torch.testing.assert_close(v.grad, params[k].grad, rtol=1e-3, atol=1e-7 * float(params[k].grad.abs().max()) + 1e-12)
        checked += 1
    assert checked == (16 if cls_only else 34)
    torch.testing.assert_close(f_o.grad, f_ref.grad, rtol=1e-3, atol=1e-6 * float(f_ref.grad.abs().max()))
    if context:
        torch.testing.assert_close(c_o.grad, c_ref.grad, rtol=1e-3, atol=1e-6 * float(c_ref.grad.abs().max()))
    # the masks matter: the undropped model gives other outputs
    assert not torch.allclose(om_prob(f_o.detach(), sd, cfg, ctx, cls_only), prob.detach(), rtol=1e-4, atol=1e-6)


def om_prob(feat, sd, cfg, ctx, cls_only):
    from oracle import model as om
    return om.two_branch(feat, sd, cfg.T, ctx, cfg.fc_dim, cfg.pool_size, cls_only)[0]


# ---- argument checks ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    return L.lib()


@pytest.fixture(scope="module")
def buf():
    b = (ctypes.c_char * (4096 + 16))()
    addr = (ctypes.addressof(b) + 15) & ~15
    return b, ctypes.c_void_p(addr)


def draw(p=P, **kw):
    d = dict(seed=1234, offset=0, keep=1.0 - p, sm_count=132, threads_per_sm=2048)
    d.update(kw)
    return L.step_dropout_draw(**d)


def expect(lib, rc, *words, code=L.E_ARG):
    assert rc == code, rc
    msg = lib.step_last_error().decode()
    for w in words:
        assert w in msg, (w, msg)


def calls(lib, p, d, n4=True):
    """Every dropout entry with draw d, on shapes whose draw has 4 * k elements (n4) or not."""
    R, T, P_, C = (1, 3, 7, 4) if n4 else (1, 1, 1, 3)
    ctx_cols = 0
    return {
        "mask_u8": lambda: lib.step_dropout_mask_u8(d, 12 if n4 else 6, p, None),
        "global_fwd": lambda: lib.step_dropout_global_fwd(d, p, L.F32, C, R, T, P_, C, ctx_cols, p, C, None),
        "local_fwd": lambda: lib.step_dropout_local_fwd(d, p, L.F32, C, R * T, P_, C, p, C, None),
        "ctx_mean": lambda: lib.step_dropout_ctx_mean_f32(d, P_, C, p, None, 4 * T, 1, T, R, T, 4 if n4 else 3, p, None),
        "mean_mid_bwd": lambda: lib.step_mean_mid_bwd_dropout(d, ctx_cols, p, R, T, P_, C, 1.0, p, L.F32, C, None),
        "f32_accum": lambda: lib.step_f32_accum_dropout(d, p, R * T, P_, C, 1.0, p, L.F16, C, None),
        "ctx_reduce": lambda: lib.step_ctx_grad_reduce_dropout_f32(d, P_, C, p, 4, p, R, T, 1, T, 0, 4 if n4 else 3, p, None),
    }


def test_dropout_entries_refuse_p_thread_counts_and_null_draws(lib, buf):
    _, p = buf
    for bad in (dict(p=0.0), dict(p=1.0), dict(p=-0.5), dict(p=1.5), dict(p=float("nan"))):
        for name, call in calls(lib, p, draw(**bad)).items():
            expect(lib, call(), "outside (0, 1)")
    for bad in (dict(sm_count=0), dict(sm_count=-1), dict(threads_per_sm=0), dict(threads_per_sm=128)):
        for name, call in calls(lib, p, draw(**bad)).items():
            expect(lib, call(), "sm_count")
    for name, call in calls(lib, p, None).items():
        expect(lib, call(), "null draw")
    expect(lib, lib.step_dropout_check(None, 8, None), "null draw")


def test_dropout_entries_refuse_sizes_off_the_vectorised_path(lib, buf):
    _, p = buf
    for name, call in calls(lib, p, draw(), n4=False).items():
        expect(lib, call(), "n % 4 == 0", code=L.E_UNSUPPORTED)
    for n in (0, -4, 6, 1 << 31):
        expect(lib, lib.step_dropout_check(draw(), n, None), "elements", code=L.E_UNSUPPORTED)


def test_dropout_entries_refuse_null_pointers(lib, buf):
    _, p = buf
    d = draw()
    expect(lib, lib.step_dropout_mask_u8(d, 12, None, None), "null pointer")
    expect(lib, lib.step_dropout_global_fwd(d, None, L.F32, 4, 1, 3, 7, 4, 0, p, 4, None), "null pointer")
    expect(lib, lib.step_dropout_global_fwd(d, p, L.F32, 4, 1, 3, 7, 4, 0, None, 4, None), "null pointer")
    expect(lib, lib.step_dropout_local_fwd(d, None, L.F32, 4, 3, 7, 4, p, 4, None), "null pointer")
    expect(lib, lib.step_dropout_ctx_mean_f32(d, 7, 4, None, None, 12, 1, 3, 1, 3, 4, p, None), "null pointer")
    expect(lib, lib.step_dropout_ctx_mean_f32(d, 7, 4, p, None, 12, 1, 3, 1, 3, 4, None, None), "null pointer")
    expect(lib, lib.step_mean_mid_bwd_dropout(d, 0, None, 1, 3, 7, 4, 1.0, p, L.F32, 4, None), "null pointer")
    expect(lib, lib.step_f32_accum_dropout(d, p, 3, 7, 4, 1.0, None, L.F32, 4, None), "null pointer")
    expect(lib, lib.step_ctx_grad_reduce_dropout_f32(d, 7, 4, p, 4, None, 1, 3, 1, 3, 0, 4, p, None), "null pointer")


def test_dropout_offset_step_follows_torchs_launch_geometry(lib):
    """((n - 1) / (4 * n_threads) + 1) * 4 with n_threads = 256 * min(ceil(n / 256), sm_count * threads_per_sm / 256)."""
    s = ctypes.c_uint64()
    nt = 132 * 2048
    for n, want in ((4, 4), (1020, 4), (4 * nt, 4), (4 * nt + 4, 8), (8 * nt + 4, 12), (68 * 12544 * 9, 32)):
        assert lib.step_dropout_check(draw(), n, ctypes.byref(s)) == 0
        assert s.value == want, (n, s.value, want)
    assert lib.step_dropout_check(draw(sm_count=1, threads_per_sm=256), 4 * 256 + 4, ctypes.byref(s)) == 0 and s.value == 8
