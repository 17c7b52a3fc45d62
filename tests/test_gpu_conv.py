"""GPU: the convolution kernels.
  * SIMT fp32 (parity mode) vs torch-CPU conv3d (the reference's arithmetic, i3dpt.py:103-111);
  * TMA addressing (box / im2col) checked byte-for-byte through the debug tile dump;
  * wgmma fp16 kernel vs the SIMT kernel on identical fp16 inputs (fp32 accumulate both:
    differences are accumulation order only -> tolerance 2e-3 of max|ref| + 1 fp16 ulp).
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from step_b200 import _lib as L
from step_b200 import engine as E
from step_b200.engine import Act

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _tape_reference as R  # noqa: E402

pytestmark = pytest.mark.gpu


def check_f64(got, x, wp, scale, shift, res, k, pad, out_dims, relu, what, widths=None):
    """got (list of fp16 outputs) against conv_fwd with the bound derived in tests/test_gpu_forward_layers.py."""
    ys, xws, epis = R.conv_fwd(x, wp, scale, shift, res, k, (1, 1, 1), pad, out_dims, relu, widths)
    for g, y, xw, epi in zip(got, ys, xws, epis):
        R.check_fwd(g, y, xw, epi, R.conv_steps(k, x.shape[-1]), what)


def ref_conv(x_ndhwc, w, k, stride, scale, shift, relu, residual):
    """torch-CPU fp32 reference: TF-SAME padded conv3d + affine + residual + relu, NDHWC in/out."""
    x = x_ndhwc.permute(0, 4, 1, 2, 3).float().cpu()
    pads = [E.same_pad(k[i], stride[i]) for i in range(3)]
    x = F.pad(x, (pads[2][0], pads[2][1], pads[1][0], pads[1][1], pads[0][0], pads[0][1]))
    y = F.conv3d(x, w.float().cpu(), stride=stride)
    if scale is not None:
        y = y * scale.cpu().view(1, -1, 1, 1, 1)
    if shift is not None:
        y = y + shift.cpu().view(1, -1, 1, 1, 1)
    y = y.permute(0, 2, 3, 4, 1)
    if residual is not None:
        y = y + residual.float().cpu()
    return F.relu(y) if relu else y


def run_conv(x, w, code, k, stride, scale, shift, relu, residual, a_mode, coff=0, extra=0):
    Cout = w.shape[0]
    wp = E.pack_conv_weight(w.cuda(), code)
    xa = Act(x.contiguous())
    od = tuple(-(-d // s) for d, s in zip((xa.T, xa.H, xa.W), stride))
    buf = torch.zeros((xa.N,) + od + (Cout + coff + extra,), dtype=E.torch_dtype(code), device="cuda")
    out = Act(buf, Cout, coff)
    res = Act(residual.contiguous()) if residual is not None else None
    E.conv(xa, wp, scale, shift, out, k, stride, None, relu, res, a_mode=a_mode)
    torch.cuda.synchronize()
    return buf


CASES_F32 = [
    # N, T, H, W, Cin, Cout, k, stride
    (2, 4, 9, 7, 8, 24, (1, 1, 1), (1, 1, 1)),
    (1, 5, 9, 11, 12, 20, (3, 3, 3), (1, 1, 1)),
    (1, 8, 20, 18, 4, 16, (7, 7, 7), (2, 2, 2)),
    (3, 1, 7, 7, 16, 8, (1, 3, 3), (1, 1, 1)),
]


@pytest.mark.parametrize("case", CASES_F32)
def test_simt_fp32_matches_torch_cpu(case):
    N, T, H, W, Cin, Cout, k, stride = case
    g = torch.Generator().manual_seed(1)
    x = torch.randn(N, T, H, W, Cin, generator=g)
    w = torch.randn(Cout, Cin, *k, generator=g) / (Cin * k[0] * k[1] * k[2]) ** 0.5
    scale = torch.rand(Cout, generator=g) + 0.5
    shift = torch.randn(Cout, generator=g)
    od = tuple(-(-d // s) for d, s in zip((T, H, W), stride))
    res = torch.randn((N,) + od + (Cout,), generator=g)
    y = run_conv(x.cuda(), w, L.F32, k, stride, scale.cuda(), shift.cuda(), True, res.cuda(), L.A_AUTO, coff=8, extra=4)
    ref = ref_conv(x, w, k, stride, scale, shift, True, res)
    got = y[..., 8:8 + Cout].cpu()
    assert torch.allclose(got, ref, rtol=1e-4, atol=1e-4 * float(ref.abs().max()))
    assert float(y[..., :8].abs().max()) == 0 and float(y[..., 8 + Cout:].abs().max()) == 0   # slice only


# ---- TMA tile dump ---------------------------------------------------------------------------
def unswizzle(raw_u16, BK):
    """raw stage bytes (as uint16) -> [128, BK] logical tile, undoing the TMA swizzle (the layout wgmma reads)."""
    row_bytes = BK * 2
    tile = np.zeros((128, BK), np.uint16)
    raw = raw_u16.view(np.uint8)
    for r in range(128):
        for ch in range(row_bytes // 16):
            if row_bytes == 128:
                pch = ch ^ (r % 8)
            elif row_bytes == 64:
                pch = ch ^ ((r >> 1) & 3)
            else:
                pch = ch ^ ((r >> 2) & 1)
            off = r * row_bytes + pch * 16
            tile[r, ch * 8:(ch + 1) * 8] = raw[off:off + 16].view(np.uint16)
    return tile


def id_tensor(N, T, H, W, C):
    ids = (np.arange(N * T * H * W * C, dtype=np.int64) % 65521 + 1).astype(np.uint16).reshape(N, T, H, W, C)
    return ids


def conv_params(x, Cin, Cout, k, pad_lo, out_dims, a_mode, w):
    p = L.step_conv_params()
    p.dtype = L.F16
    p.N, p.T, p.H, p.W = x.shape[:4]
    p.Cin, p.in_ld = Cin, x.shape[4]
    p.Cout, p.out_ld, p.out_coff = Cout, Cout, 0
    p.KT, p.KH, p.KW = k
    p.ST = p.SH = p.SW = 1
    p.PT, p.PH, p.PW = pad_lo
    p.OT, p.OH, p.OW = out_dims
    p.w_ld = w.shape[2]
    p.x, p.w, p.y = x.data_ptr(), w.data_ptr(), x.data_ptr()
    p.a_mode = a_mode
    return p


@pytest.mark.parametrize("a_mode", [L.A_BOX, L.A_IM2COL])
@pytest.mark.parametrize("shape", [(2, 3, 5, 6, 64), (1, 4, 14, 14, 32), (2, 8, 7, 7, 16), (1, 2, 9, 10, 96)])
def test_tma_tile_addressing(a_mode, shape):
    N, T, H, W, C = shape
    ids = id_tensor(N, T, H, W, C)
    x = torch.from_numpy(ids.view(np.int16)).cuda().view(torch.float16)
    k, pad = (3, 3, 3), (1, 1, 1)
    w = torch.zeros((16, 27, C), dtype=torch.float16, device="cuda")
    p = conv_params(x, C, 16, k, pad, (T, H, W), a_mode, w)
    bk = ctypes.c_int(0)
    box = (ctypes.c_int * 3)()
    out = torch.zeros(128 * 64 * 2, dtype=torch.uint8, device="cuda")
    M = N * T * H * W
    checked = 0
    for (kt, kh, kw) in [(0, 0, 0), (1, 1, 1), (2, 2, 2), (0, 2, 1)]:
        n_tiles = None
        for m_tile in range(64):
            L.check(L.lib().step_debug_tma_tile(p, m_tile, kt, kh, kw, 0, L.ptr(out), ctypes.byref(bk), box, L.stream()))
            torch.cuda.synchronize()
            BK = bk.value
            raw = out.cpu().numpy()[:128 * BK * 2].view(np.uint16)
            tile = unswizzle(raw, BK)
            bw, bh, bt = box[0], box[1], box[2]
            if a_mode == L.A_BOX:
                tw, th, tt = -(-W // bw), -(-H // bh), -(-T // bt)
                n_tiles = N * tt * th * tw
                if m_tile >= n_tiles:
                    break
                r = m_tile
                w0 = (r % tw) * bw; r //= tw
                h0 = (r % th) * bh; r //= th
                t0 = (r % tt) * bt; n = r // tt
                rows = [(n, t0 + dt, h0 + dh, w0 + dw) for dt in range(bt) for dh in range(bh) for dw in range(bw)]
            else:
                n_tiles = -(-M // 128)
                if m_tile >= n_tiles:
                    break
                rows = []
                for m in range(m_tile * 128, m_tile * 128 + 128):
                    if m >= M:
                        rows.append(None); continue
                    ww = m % W; hh = (m // W) % H; tt_ = (m // (W * H)) % T; nn = m // (W * H * T)
                    rows.append((nn, tt_, hh, ww))
            for ri, pix in enumerate(rows):
                if pix is None:
                    continue
                n, t, h, ww = pix
                if a_mode == L.A_BOX and (t >= T or h >= H or ww >= W):
                    continue  # box overhang rows: never stored by the epilogue
                it, ih, iw = t + kt - 1, h + kh - 1, ww + kw - 1
                exp = ids[n, it, ih, iw, :BK] if (0 <= it < T and 0 <= ih < H and 0 <= iw < W) else np.zeros(BK, np.uint16)
                assert np.array_equal(tile[ri], exp), (a_mode, shape, (kt, kh, kw), m_tile, ri, pix)
                checked += 1
    assert checked > 100


CASES_F16 = [
    # N, T, H, W, Cin, Cout, k
    (2, 4, 14, 14, 64, 64, (1, 1, 1)),
    (1, 3, 9, 11, 192, 96, (1, 1, 1)),
    (2, 8, 7, 7, 160, 320, (3, 3, 3)),
    (1, 8, 14, 14, 96, 208, (3, 3, 3)),
    (1, 4, 12, 12, 16, 48, (3, 3, 3)),
    (1, 4, 10, 9, 24, 64, (3, 3, 3)),
    (5, 1, 7, 7, 256, 256, (1, 3, 3)),
    (1, 2, 28, 28, 32, 32, (3, 3, 3)),
]


@pytest.mark.parametrize("a_mode", [L.A_BOX, L.A_IM2COL])
@pytest.mark.parametrize("case", CASES_F16)
def test_umma_fp16_matches_simt(case, a_mode):
    N, T, H, W, Cin, Cout, k = case
    g = torch.Generator().manual_seed(3)
    x = torch.randn(N, T, H, W, Cin, generator=g).half().cuda()
    w = (torch.randn(Cout, Cin, *k, generator=g) / (Cin * k[0] * k[1] * k[2]) ** 0.5).half()
    scale = (torch.rand(Cout, generator=g) + 0.5).cuda()
    shift = torch.randn(Cout, generator=g).cuda()
    res = torch.randn(N, T, H, W, Cout, generator=g).half().cuda()
    mode = L.A_AUTO if k == (1, 1, 1) else a_mode
    ref = run_conv(x, w, L.F16, k, (1, 1, 1), scale, shift, True, res, L.A_SIMT, coff=8, extra=8).float()
    got = run_conv(x, w, L.F16, k, (1, 1, 1), scale, shift, True, res, mode, coff=8, extra=8).float()
    tol = 2e-3 * float(ref.abs().max()) + 2e-3
    err = float((got - ref).abs().max())
    assert err <= tol, "max err %g > %g" % (err, tol)
    assert float(got[..., :8].abs().max()) == 0 and float(got[..., 8 + Cout:].abs().max()) == 0
    pad = tuple(E.same_pad(kk, 1)[0] for kk in k)
    check_f64([got[..., 8:8 + Cout]], x, E.pack_conv_weight(w.cuda(), L.F16), scale, shift, res, k, pad, (T, H, W), True,
              (case, a_mode))


def test_stem_s2d_fp16_vs_fp32_simt():
    """the space-to-depth stem (fp16, wgmma) against the stride-2 fp32 SIMT conv of the same layer."""
    from step_b200 import synth
    import step_b200
    cfg16, cfg32 = synth.make_cfg(fp16=True), synth.make_cfg(fp16=False)
    sd = synth.base_net_state_dict()
    x = synth.make_clips(1, 8, 32, 32).cuda()
    outs = []
    for cfg in (cfg16, cfg32):
        net = step_b200.BaseNet(cfg).cuda()
        net.load_state_dict(sd)
        stem = net.base_model[0]
        code = E.dtype_code(cfg.fp16)
        src = x.contiguous()
        if code == L.F16:
            s2d = Act.empty(1, 4, 16, 16, 32, L.F16, x.device)
            L.check(L.lib().step_clip_to_s2d_f16(L.ptr(src), 1, 8, 3, 32, 32, L.ptr(s2d.buf), 32, L.stream()))
            outs.append(stem.forward_s2d(s2d).buf.float())
        else:
            a = Act.empty(1, 8, 32, 32, 4, L.F32, x.device)
            L.check(L.lib().step_clip_to_ndhwc(L.ptr(src), 1, 8, 3, 32, 32, L.ptr(a.buf), L.F32, 4, L.stream()))
            outs.append(stem(a).buf)
    torch.cuda.synchronize()
    err = float((outs[0] - outs[1]).abs().max())
    assert err <= 2e-2 * float(outs[1].abs().max()), err


POOL_CASES = [
    # N, T, H, W, C, k, s
    (2, 4, 7, 7, 64, (3, 3, 3), (1, 1, 1)),      # specialised 3x3x3 kernel (W % 7 == 0)
    (1, 3, 14, 28, 32, (3, 3, 3), (1, 1, 1)),
    (1, 7, 7, 14, 16, (3, 3, 3), (1, 1, 1)),     # t segments of 2 with a 1-plane tail
    (1, 1, 7, 7, 8, (3, 3, 3), (1, 1, 1)),       # a single plane
    (1, 4, 9, 10, 16, (3, 3, 3), (1, 1, 1)),     # generic kernel
    (1, 4, 12, 14, 24, (1, 3, 3), (1, 2, 2)),
    (2, 5, 13, 25, 8, (3, 3, 3), (2, 2, 2)),     # odd sizes: ceil_mode overhang + TF padding
    (1, 2, 25, 25, 16, (1, 3, 3), (1, 2, 2)),    # the ContextNet pool at 400x400 (25 -> 13)
]


@pytest.mark.parametrize("code", [L.F32, L.F16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("case", POOL_CASES)
def test_maxpool_tf_padding_matches_torch(case, code):
    N, T, H, W, C, k, s = case
    g = torch.Generator().manual_seed(5)
    x = torch.randn(N, T, H, W, C, generator=g)          # negative values exercise the zero padding
    xd = x.to(E.torch_dtype(code)).cuda()
    out = E.maxpool(Act(xd), k, s)
    torch.cuda.synchronize()
    xr = xd.float().cpu().permute(0, 4, 1, 2, 3)
    pads = [E.same_pad(k[i], s[i]) for i in range(3)]
    xr = F.pad(xr, (pads[2][0], pads[2][1], pads[1][0], pads[1][1], pads[0][0], pads[0][1]))
    ref = F.max_pool3d(xr, k, s, ceil_mode=True).permute(0, 2, 3, 4, 1)
    assert tuple(out.buf.shape) == tuple(ref.shape)
    assert torch.equal(out.buf.float().cpu(), ref)        # max is exact in either storage type


@pytest.mark.parametrize("Cin,outs", [(832, (256, 160, 32)), (192, (64, 96, 16)), (512, (160, 112, 24)),
                                      (512, (112, 144, 32))])
def test_fused_1x1_multi_destination_matches_separate_convs(Cin, outs):
    """Mixed's three 1x1x1 branches as one GEMM whose epilogue scatters column ranges (i3dpt.py:133-147);
    mixed_3b / 4c / 4e have destination boundaries that are not multiples of 32 columns."""
    g = torch.Generator().manual_seed(11)
    N, T, H, W = 2, 4, 7, 7
    x = torch.randn(N, T, H, W, Cin, generator=g).half().cuda()
    ws = [(torch.randn(c, Cin, 1, 1, 1, generator=g) / Cin ** 0.5).half() for c in outs]
    scale = (torch.rand(sum(outs), generator=g) + 0.5).cuda()
    shift = torch.randn(sum(outs), generator=g).cuda()
    xa = Act(x.contiguous())
    wp = torch.cat([E.pack_conv_weight(w.cuda(), L.F16) for w in ws], 0).contiguous()
    big = torch.zeros((N, T, H, W, 512), dtype=torch.float16, device="cuda")       # branch_0 lands in a slice
    t1 = torch.zeros((N, T, H, W, outs[1]), dtype=torch.float16, device="cuda")
    t2 = torch.zeros((N, T, H, W, outs[2] + 8), dtype=torch.float16, device="cuda")
    E.conv(xa, wp, scale, shift, Act(big, outs[0], 64), (1, 1, 1), extra_outs=[Act(t1), Act(t2, outs[2], 8)])
    torch.cuda.synchronize()
    off = 0
    for w, dst in zip(ws, (big[..., 64:64 + outs[0]], t1, t2[..., 8:])):
        c = w.shape[0]
        ref = run_conv(x, w, L.F16, (1, 1, 1), (1, 1, 1), scale[off:off + c].contiguous(), shift[off:off + c].contiguous(),
                       True, None, L.A_SIMT).float()
        err = float((dst.float() - ref).abs().max())
        assert err <= 2e-3 * float(ref.abs().max()) + 2e-3, (c, err)
        off += c
    assert float(big[..., :64].abs().max()) == 0 and float(big[..., 64 + outs[0]:].abs().max()) == 0
    assert float(t2[..., :8].abs().max()) == 0
    check_f64([big[..., 64:64 + outs[0]], t1, t2[..., 8:]], x, wp, scale, shift, None, (1, 1, 1), (0, 0, 0), (T, H, W), True,
              (Cin, outs), list(outs))


# ---- small-N linear layers / temporal mean of the head (two_branch.py:246-270) -------------------------------------
@pytest.mark.parametrize("code", [L.F32, L.F16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("M,K,N", [(100, 12544, 12), (37, 1000, 4), (88, 1024, 60), (5, 520, 33)])
def test_linear_small_n_matches_torch(M, K, N, code):
    g = torch.Generator().manual_seed(3)
    dt = E.torch_dtype(code)
    x = torch.randn(M + 3, K, generator=g).to(dt).cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dt).cuda()
    b = torch.randn(N, generator=g).cuda()
    rows = torch.randperm(M + 3, generator=g)[:M].to(torch.int32).cuda()
    y = E.linear_small_n(x, M, K, K, w, b, N, row_map=rows)
    ref = x.float()[rows.long()] @ w.float().t() + b
    tol = 1e-4 if code == L.F32 else 1e-3
    assert float((y - ref).abs().max()) <= tol * float(ref.abs().max()) + tol
    # accumulate + sigmoid on top of an existing y, no bias, identity rows
    y2 = E.linear_small_n(x, M, K, K, w, None, N, y=y.clone(), act=1, accumulate=True)
    ref2 = torch.sigmoid(y + x.float()[:M] @ w.float().t())
    assert float((y2 - ref2).abs().max()) <= 2e-3
    # bit-for-bit repeatable (fixed reduction order over the K split)
    assert torch.equal(E.linear_small_n(x, M, K, K, w, b, N, row_map=rows), y)


@pytest.mark.parametrize("out_code", [L.F32, L.F16], ids=["to_fp32", "to_fp16"])
def test_mean_mid_fp16_matches_torch(out_code):
    g = torch.Generator().manual_seed(4)
    A, B, P, C, ld = 5, 8, 49, 256, 1088
    buf = torch.randn(A, B, P, ld, generator=g).half().cuda()
    view = buf[..., 832:832 + C]
    y = E.mean_mid(view.data_ptr(), L.F16, A, B, P, C, ld, buf.device, out_code)
    ref = view.float().mean(1).reshape(A, P * C)
    tol = 1e-6 if out_code == L.F32 else 2e-3
    assert float((y.float() - ref).abs().max()) <= tol * float(ref.abs().max()) + tol


# ---- patch-in-shared-memory kernel (csrc/conv_halo.cu) against the TMA-im2col kernel ---------------------------------
HALO_CASES = [
    # N, T, H, W, Cin, Cout, k, pad_lo
    (2, 4, 32, 24, 32, 64, (4, 4, 4), (1, 1, 1)),     # the s2d stem shape (even tiles)
    (1, 3, 20, 13, 32, 64, (4, 4, 4), (1, 1, 1)),     # ragged in t, h and w
    (1, 5, 17, 9, 16, 32, (3, 3, 3), None),           # 32-byte rows
    (1, 4, 14, 14, 64, 128, (3, 3, 3), None),         # 128-byte rows, one accumulator set per CTA
    (2, 1, 7, 7, 32, 40, (1, 3, 3), None),            # 2-D filter, Cout not a multiple of 32
    (1, 3, 18, 16, 64, 192, (3, 3, 3), None),         # conv3d_2c_3x3 shape: two column tiles (128 + 64)
    (1, 9, 25, 25, 16, 48, (3, 3, 3), None),          # Mixed_4b's 3x3x3 at the shipped 400 x 400 clip: TT = 4, last group 1 plane
    (1, 18, 20, 22, 16, 32, (3, 3, 3), None),         # Mixed_3b's (T 18): TT = 4, a last group of 2 planes
]


@pytest.mark.parametrize("case", HALO_CASES)
def test_halo_kernel_matches_im2col_kernel(case):
    N, T, H, W, Cin, Cout, k, pad = case
    g = torch.Generator().manual_seed(31)
    x = torch.randn(N, T, H, W, Cin, generator=g).half().cuda()
    w = (torch.randn(Cout, Cin, *k, generator=g) / (Cin * k[0] * k[1] * k[2]) ** 0.5).half()
    scale = (torch.rand(Cout, generator=g) + 0.5).cuda()
    shift = torch.randn(Cout, generator=g).cuda()
    wp = E.pack_conv_weight(w.cuda(), L.F16)
    outs = []
    for mode in (L.A_HALO, L.A_IM2COL):
        buf = torch.zeros((N, T, H, W, Cout + 16), dtype=torch.float16, device="cuda")
        E.conv(Act(x), wp, scale, shift, Act(buf, Cout, 8), k, (1, 1, 1), pad, True, None, a_mode=mode, out_dims=(T, H, W))
        torch.cuda.synchronize()
        outs.append(buf)
    assert float(outs[0][..., :8].abs().max()) == 0 and float(outs[0][..., 8 + Cout:].abs().max()) == 0
    # both kernels against the float64 convolution of the same fp16 operands
    pad_lo = pad if pad is not None else tuple(E.same_pad(kk, 1)[0] for kk in k)
    for o, mode in zip(outs, ("halo", "im2col")):
        check_f64([o[..., 8:8 + Cout]], x, wp, scale, shift, None, k, pad_lo, (T, H, W), True, (case, mode))


# ---- fused bottleneck exit (step_bottleneck_exit_f16) -------------------------------------------------------------------
def _exit_inputs(M, seed, x_pad=0):
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(M, 256, generator=g).half().cuda()
    w3 = (torch.randn(1024, 256, generator=g) / 16).half().cuda()
    xbuf = torch.randn(M, 1024 + x_pad, generator=g).half().cuda()
    w1 = (torch.randn(256, 1024, generator=g) / 32).half().cuda()
    b = torch.randn(256, generator=g).float().cuda()
    return h, w3, xbuf, w1, b


def _frames(t2d, C, coff=0):
    return Act(t2d.view(t2d.shape[0], 1, 1, 1, t2d.shape[1]), C, coff)


@pytest.mark.parametrize("M", [1, 200, 256, 1000, 7 * 7 * 88 * 8])
@pytest.mark.parametrize("variant", ["next_conv1", "downsample2"])
def test_bottleneck_exit_equals_two_launches(M, variant):
    """y = relu(h w3^T + x), z = act(y w1^T + b): one launch == the two step_conv3d_fwd launches it replaces, bit for bit
    (same fp16 rounding of y, same K order), and within the derived bound of the float64 exit_fwd."""
    x_pad = 64 if M == 1000 else 0                       # residual read out of a wider buffer (row pitch > channels)
    h, w3, xbuf, w1, b = _exit_inputs(M, 7 + M, x_pad)
    relu2, bias = (True, None) if variant == "next_conv1" else (False, b)
    ha, xa = _frames(h, 256), _frames(xbuf, 1024)
    w3p, w1p = w3.view(1024, 1, 256), w1.view(256, 1, 1024)
    # two launches
    y_ref = _frames(torch.empty(M, 1024, dtype=torch.float16, device="cuda"), 1024)
    z_ref = _frames(torch.empty(M, 256, dtype=torch.float16, device="cuda"), 256)
    E.conv(ha, w3p, None, None, y_ref, (1, 1, 1), relu=True, residual=xa)
    E.conv(y_ref, w1p, None, bias, z_ref, (1, 1, 1), relu=relu2)
    # one launch
    store_y = variant == "next_conv1"
    y = _frames(torch.zeros(M, 1024, dtype=torch.float16, device="cuda"), 1024) if store_y else None
    z = _frames(torch.zeros(M, 256, dtype=torch.float16, device="cuda"), 256)
    E.bottleneck_exit(ha, w3p, xa, w1p, bias, relu2, z, y)
    torch.cuda.synchronize()
    if store_y:
        assert torch.equal(y.buf, y_ref.buf)
    assert torch.equal(z.buf, z_ref.buf)
    ref = R.exit_fwd(h, w3p, xbuf[:, :1024], w1p, bias, relu2)
    R.check_fwd(z.buf.view(M, 256), ref["z"], ref["z_xw"], ref["z_epi"], 1024 // 16, (M, variant, "z"), extra=ref["z_carry"])
    if store_y:
        R.check_fwd(y.buf.view(M, 1024), ref["y"], ref["y_xw"], ref["y_epi"], 256 // 16, (M, variant, "y"))


def test_bottleneck_exit_rejects_other_widths():
    h = _frames(torch.zeros(64, 128, dtype=torch.float16, device="cuda"), 128)
    x = _frames(torch.zeros(64, 1024, dtype=torch.float16, device="cuda"), 1024)
    z = _frames(torch.zeros(64, 256, dtype=torch.float16, device="cuda"), 256)
    w3 = torch.zeros(1024, 1, 128, dtype=torch.float16, device="cuda")
    w1 = torch.zeros(256, 1, 1024, dtype=torch.float16, device="cuda")
    with pytest.raises(RuntimeError, match="planes 256"):
        E.bottleneck_exit(h, w3, x, w1, None, True, z)
