"""Argument checks of the fp32 training entry points (step_conv_wgrad_f32 and the fp32 siblings of the fp16 backward
entries), without a GPU: every refused call returns STEP_E_ARG (or STEP_E_WORKSPACE) with its reason before any launch.
The pointers are 16-byte aligned host addresses that are never dereferenced."""
import ctypes
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from step_b200 import _lib as L  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    return L.lib()


@pytest.fixture(scope="module")
def buf():
    b = (ctypes.c_char * (4096 + 16))()
    addr = (ctypes.addressof(b) + 15) & ~15
    return b, ctypes.c_void_p(addr)


def expect(lib, rc, *words, code=L.E_ARG):
    assert rc == code
    msg = lib.step_last_error().decode()
    for w in words:
        assert w in msg, (w, msg)


def wgrad(lib, p, dz="p", x="p", dw="p", ws="p", dz_ld=8, x_ld=4, N=1, dims=(6, 10, 10), out=(3, 5, 5), Cout=8, Cin=4,
          k=(7, 7, 7), s=(2, 2, 2), pad=(2, 2, 2), dw_ld=4, ws_bytes=None):
    pick = lambda v: p if v == "p" else v
    taps = k[0] * k[1] * k[2]
    if ws_bytes is None:
        ws_bytes = lib.step_conv_wgrad_f32_workspace_bytes(N * out[0] * out[1] * out[2], Cout, Cin, taps)
    return lib.step_conv_wgrad_f32(pick(dz), dz_ld, pick(x), x_ld, N, *dims, *out, Cout, Cin, *k, *s, *pad, 1.0, pick(dw), dw_ld, 0,
                                   pick(ws), ws_bytes, None)


def test_conv_wgrad_f32_rejects_bad_shapes_channels_padding_extent_and_workspace(lib, buf):
    _, p = buf
    for kw in (dict(N=0), dict(out=(0, 5, 5)), dict(Cin=0), dict(k=(0, 7, 7)), dict(s=(2, 0, 2)), dict(dz=None), dict(x=None),
               dict(dw=None), dict(ws=None)):
        expect(lib, wgrad(lib, p, **kw), "conv_wgrad_f32: bad arguments")
    for kw in (dict(Cin=3, x_ld=4, dw_ld=4), dict(Cout=6, dz_ld=8), dict(dz_ld=10), dict(x_ld=6, Cin=4), dict(dz_ld=4),
               dict(dw_ld=3)):
        expect(lib, wgrad(lib, p, **kw), "conv_wgrad_f32", "multiples of 4")
    expect(lib, wgrad(lib, p, x=ctypes.c_void_p(p.value + 4)), "16-byte aligned")
    for pad in ((7, 2, 2), (2, -1, 2), (2, 2, 7)):
        expect(lib, wgrad(lib, p, pad=pad), "conv_wgrad_f32: bad padding")
    expect(lib, wgrad(lib, p, k=(1, 1, 1), s=(1, 1, 1), pad=(0, 0, 1)), "conv_wgrad_f32: bad padding")
    # an output pixel whose first tap starts past the padded input
    expect(lib, wgrad(lib, p, out=(6, 5, 5)), "inconsistent")
    expect(lib, wgrad(lib, p, N=1 << 20, dims=(64, 64, 64), out=(32, 32, 32)), "exceed 2^31")
    need = lib.step_conv_wgrad_f32_workspace_bytes(75, 8, 4, 343)
    assert need > 0
    expect(lib, wgrad(lib, p, ws_bytes=need - 4), "workspace", code=L.E_WORKSPACE)


def test_conv_wgrad_f32_workspace_follows_the_shape_only():
    lib = L.lib()
    assert lib.step_conv_wgrad_f32_workspace_bytes(0, 8, 4, 1) == 0
    assert lib.step_conv_wgrad_f32_workspace_bytes(100, 8, 4, 0) == 0
    # one 64 x 64 fp32 tile per (chunk, co tile, column tile); at least one chunk; columns are taps * Cin
    tile = 64 * 64 * 4
    assert lib.step_conv_wgrad_f32_workspace_bytes(10, 8, 4, 1) == tile
    assert lib.step_conv_wgrad_f32_workspace_bytes(10, 68, 4, 343) == tile * 2 * 22
    big = lib.step_conv_wgrad_f32_workspace_bytes(1 << 24, 64, 4, 343)
    assert big % (tile * 22) == 0 and big // (tile * 22) <= 2048 // 22 + 1


def test_fp32_backward_siblings_reject_bad_arguments(lib, buf):
    _, p = buf
    pick = lambda v: p if v == "p" else v

    def act(dy="p", y="p", dz="p", dres="p", C=16, dy_ld=16, y_ld=16, dz_ld=16, dres_ld=16, relu=1, M=10):
        return lib.step_act_bwd_f32(pick(dy), dy_ld, pick(y), y_ld, None, relu, M, C, pick(dz), dz_ld, pick(dres), dres_ld, None)
    assert act(M=0) == L.E_ARG
    for kw in (dict(C=6, dy_ld=6, y_ld=6, dz_ld=6, dres_ld=6), dict(dy_ld=18), dict(dz_ld=14), dict(dres_ld=10), dict(y=None),
               dict(dy=None), dict(dz=None)):
        expect(lib, act(**kw), "act_bwd: bad arguments")
    assert act(C=4, dy_ld=4, y_ld=4, dz_ld=4, dres_ld=4, M=0) == L.E_ARG        # 4 channels are a whole fp32 vector
    for which in ("dy", "y", "dz", "dres"):
        expect(lib, act(**{which: ctypes.c_void_p(p.value + 4)}), "16-byte aligned")
    expect(lib, lib.step_colsum_f32(None, 4, 10, 4, 1.0, p, p, None), "colsum: bad arguments")
    expect(lib, lib.step_colsum_f32(p, 4, 0, 4, 1.0, p, p, None), "colsum: bad arguments")
    expect(lib, lib.step_colsum_f32(p, 4, 10, 4, 1.0, p, None, None), "colsum: bad arguments")
    expect(lib, lib.step_mean_mid_bwd_f32(p, 2, 3, 4, 8, 1.0, p, 7, None), "mean_mid_bwd: bad arguments")
    expect(lib, lib.step_mean_mid_bwd_f32(None, 2, 3, 4, 8, 1.0, p, 8, None), "mean_mid_bwd: bad arguments")
    expect(lib, lib.step_f32_accum_f32(p, 10, 8, 1.0, p, 4, None), "f32_accum_f32: bad arguments")
    expect(lib, lib.step_f32_accum_f32(p, 0, 8, 1.0, p, 8, None), "f32_accum_f32: bad arguments")
    expect(lib, lib.step_f32_accum_f32(p, 10, 8, 1.0, None, 8, None), "f32_accum_f32: bad arguments")

    def pool(k=(3, 3, 3), s=(1, 1, 1), lo=(1, 1, 1), hi=(1, 1, 1), x="p", ws="p", dims=(4, 6, 6)):
        return lib.step_maxpool3d_bwd_f32(pick(x), 8, p, 8, 1, *dims, 8, *k, *s, *lo, *hi, *dims, p, 8, pick(ws), None)
    expect(lib, pool(k=(1, 1, 254), lo=(0, 0, 1)), "maxpool3d_bwd: bad arguments")
    expect(lib, pool(x=None), "maxpool3d_bwd: bad arguments")
    expect(lib, pool(ws=None), "maxpool3d_bwd: bad arguments")
    expect(lib, pool(s=(1, 0, 1)), "maxpool3d_bwd", "must be positive")
    expect(lib, pool(lo=(3, 1, 1)), "maxpool3d_bwd: bad padding")
    expect(lib, pool(hi=(1, -1, 1)), "maxpool3d_bwd: bad padding")

