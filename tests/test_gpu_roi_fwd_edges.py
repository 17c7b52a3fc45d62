"""GPU: the channels-last ROIAlign forward (step_roi_align_fwd_nhwc) on its own, at the bins, sampling grids, channel counts
and layouts where its kernels and their branches can go wrong, each against a reference of the same operation.

Kernels and branches (csrc/roi.cu):
  * exact=1, roi_align_fwd_nhwc_kernel<float, true> and <__half, true>: the reference's operation order, so fp32 is
    bit-identical to the C oracle (oracle.ops.roi_align_fwd, pinned to the reference's compiled op) and fp16 equals
    fp16(that on the fp16 inputs);
  * exact=2, roi_align_fwd_nhwc_kernel<__half, false>: fp32 FMAs, within R.roi_align_fma_tol of float64.  exact=0 takes
    it too when the packed table (ph pw x 136 B) exceeds 48 KB: 20 x 20 bins (19 x 19 is the largest table, 49 096 B);
  * exact=0, roi_align_fwd_nhwc_f16_packed_kernel: a per-ROI table of at most 16 merged pixels per bin, half2 FMAs,
    roi_gather_items<2> or <1> by the parity of C / 8, within R.roi_align_tol.  ROIs whose bins may not fit the table
    take its direct form, the fmaf chain of exact=2, bit-identical to exact=2 on those rows: sampling grids > 3 x 3, and
    bins wider than a fixed sampling grid g, whose samples touch up to 2 g pixels per axis (sampling_ratio 3 reaches 36);
  * the exact kernels' sample table of 784 taps: cached when ph pw gh gw <= 784, recomputed per use otherwise.
Which ROI takes which path is derived from R.roi_align_terms (bin sizes, grids, distinct pixels and samples per bin), so a
ROI the packed kernel kept in its table against that rule fails the tighter FMA bound, and every ROI with a bin of more
than 16 distinct pixels must be one the rule sends to the direct form.

Cases: 28 x 28 maps at C 8 and 24 (odd C / 8) and 64, and the shipped 25 x 25 x 832; bins 7x7, 5x3, 1x1, 19x19, 20x20;
sampling_ratio 0..4; the ROIs of the ROIAlign backward's edge test (the whole image: grid exactly 4 x 4 at 7 x 7, a full
784-tap table; grids 5 x 5 and 10 x 10; degenerate; corners in [-16, 0) and below -16; touching and passing the far
edges), 40 overlapping ROIs on one frame and 200 random ones.  The strided layout reads a channel slice at an offset of a
wider feature row, writes rows of pitch C + 8 into a canary-filled buffer (the columns past C and the rows of other ROIs
stay bit-identical) and maps ROI frames through (roi_T, feat_T, t_start), with NaN in the frames it must never read.
Every exact=0 launch is repeated with STEP_B200_ROI_PARTS=2 and 4 (a row split over 2 or 4 CTAs): bit-identical.
"""
import json
import os
import re
import subprocess
import sys

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [HERE, ROOT]
import _tape_reference as R  # noqa: E402
from oracle import ops as oops  # noqa: E402
from test_gpu_train_launches import EDGE_ROIS  # noqa: E402

pytestmark = pytest.mark.gpu
SCALE = 1.0 / 16.0
TAPS = 784                                  # the exact kernels' shared sample table (csrc/roi.cu kMaxTaps)
MERGED_BIN = 8 + 8 * R.ROI_MERGED           # bytes per bin of the packed table (csrc/roi.cu MergedBin)
PACKED_SMEM = 48 * 1024                     # largest packed table
FMAP = (2, 4, 1)                            # roi_T, feat_T, t_start: ROI frames 0..3 read frames 1, 2, 5, 6 of 8
WORST = {}                                  # path -> largest |err| / bound seen (printed at the end of the module)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nlargest |err| / bound per ROIAlign forward path: %s" % json.dumps(WORST, sort_keys=True))


def _note(kind, ratio):
    WORST[kind] = max(WORST.get(kind, 0.0), ratio)


def _rois(n_random=200, seed=51):
    """The edge ROIs (frames 0 and 3), 40 overlapping ROIs on frame 1, n_random ROIs on frames 0..3 from 1 px (degenerate
    ones included) to 37 px, up to 60 px (4 px of map) outside the 448 px image.  CPU float32 [R, 5]."""
    g = torch.Generator().manual_seed(seed)
    xy = torch.rand(40, 2, generator=g) * 200.0
    many = torch.cat([torch.ones(40, 1), xy, xy + 16.0 + torch.rand(40, 2, generator=g) * 200.0], 1)
    f = torch.randint(0, 4, (n_random, 1), generator=g).float()
    xy = torch.rand(n_random, 2, generator=g) * 560.0 - 60.0
    rand = torch.cat([f, xy, xy + torch.rand(n_random, 2, generator=g) * 600.0 - 20.0], 1)
    return torch.cat([torch.tensor(EDGE_ROIS, dtype=torch.float32), many, rand])


def _paths(rois, ph, pw, H, W, sr):
    """Per ROI row, from roi_align_terms: samples per bin; whether the packed kernel takes its direct form, by its rule
    (per axis g + 1 distinct pixels when the fp32 bin is no wider than the grid g, else 2 g; direct when the product
    exceeds 16), split into big_grid (g + 1 pixels per axis already exceed the table: grids > 3 x 3) and wide (bins wider
    than a fixed grid); and overflow, the rows with a bin of more than 16 distinct pixels, which the rule must send to the
    direct form."""
    groups = R.roi_align_terms(rois, SCALE, ph, pw, H, W, sr)
    n = rois.shape[0]
    spb = R.roi_samples_per_bin(groups, n)
    big_grid = torch.zeros(n, dtype=torch.bool)
    direct = torch.zeros(n, dtype=torch.bool)
    most = torch.zeros(n, dtype=torch.int64)
    for gr in groups:
        idx = gr["idx"].cpu()
        gh, gw = gr["grid"]
        bh, bw = (b.cpu() for b in gr["bin_hw"])
        nh = torch.where(bh <= float(gh), gh + 1, 2 * gh)
        nw = torch.where(bw <= float(gw), gw + 1, 2 * gw)
        direct[idx] = nh * nw > R.ROI_MERGED
        big_grid[idx] = (gh + 1) * (gw + 1) > R.ROI_MERGED
        most[idx] = R.roi_distinct_pixels(gr, ph * pw).max(1).values.cpu()
    overflow = most > R.ROI_MERGED
    assert not bool((overflow & ~direct).any()), ("a ROI with more distinct pixels per bin than the table holds keeps it",
                                                 (overflow & ~direct).nonzero().view(-1)[:8].tolist())
    return spb, big_grid, direct & ~big_grid, overflow


def _launch(feat, K, H, W, C, ld, rois, ph, pw, sr, out, out_ld, fmap, exact):
    from step_b200 import _lib as L
    code = L.F16 if feat.dtype == torch.float16 else L.F32
    L.check(L.lib().step_roi_align_fwd_nhwc(L.ptr(feat), code, K, H, W, C, ld, L.ptr(rois), rois.shape[0], SCALE, ph, pw, sr,
                                            L.ptr(out), out_ld, fmap[0], fmap[1], fmap[2], exact, L.stream()))


class Layout:
    """A feature map and an output buffer for one case.  plain: feat [K, H, W, C] dense, out [R, ph, pw, C], ROI frames
    index feat directly.  strided: feat the channels [8, 8 + C) of rows of C + 16, out rows 1..R of an [R + 2, ph, pw, C + 8]
    buffer filled with a canary, ROI frames mapped by FMAP, frames never read filled with NaN."""

    def __init__(self, strided, feat32, R_, ph, pw):
        self.strided = strided
        K, H, W, C = feat32.shape
        self.K, self.H, self.W, self.C = K, H, W, C
        self.R, self.ph, self.pw = R_, ph, pw
        if strided:
            buf = torch.randn(K, H, W, C + 16, device="cuda")
            buf[..., 8:8 + C] = feat32
            unread = [f for f in range(K) if not (FMAP[2] <= f % FMAP[1] < FMAP[2] + FMAP[0])]
            buf[unread] = float("nan")
            self.buf32, self.ld, self.fmap = buf, C + 16, FMAP
        else:
            self.buf32, self.ld, self.fmap = feat32, C, (0, 0, 0)

    def feat(self, dtype):
        b = self.buf32.to(dtype)
        return b[..., 8:8 + self.C] if self.strided else b

    def run(self, dtype, rois, sr, exact):
        """Launch into a fresh canary-filled buffer; check the canary; return the [R, ph, pw, C] result."""
        ld = self.C + 8 if self.strided else self.C
        rows = self.R + 2 if self.strided else self.R
        canary = torch.full((rows, self.ph, self.pw, ld), -3.0e4, dtype=dtype, device="cuda")
        obuf = canary.clone()
        out = obuf[1:] if self.strided else obuf
        _launch(self.feat(dtype), self.K, self.H, self.W, self.C, self.ld, rois, self.ph, self.pw, sr, out, ld, self.fmap, exact)
        torch.cuda.synchronize()
        if self.strided:
            assert torch.equal(obuf[0], canary[0]) and torch.equal(obuf[-1], canary[-1]), "rows of other ROIs written"
            assert torch.equal(obuf[..., self.C:], canary[..., self.C:]), "columns past C written"
        return out[:self.R, ..., :self.C].clone()

    def frames(self, rois):
        return R.roi_frames(rois, *self.fmap) if self.strided else R.roi_frames(rois)


def _check(feat32, rois_cpu, ph, pw, sr, strided, monkeypatch, what):
    K, H, W, C = feat32.shape
    n = rois_cpu.shape[0]
    rois = rois_cpu.cuda()
    lay = Layout(strided, feat32, n, ph, pw)
    monkeypatch.delenv("STEP_B200_ROI_PARTS", raising=False)

    # exact=1: the C oracle on the mapped frames, fp32 bit for bit, fp16 = fp16(exact fp32) on the fp16 inputs
    direct_rois = rois_cpu.clone()
    direct_rois[:, 0] = lay.frames(rois_cpu).float()
    nchw = feat32.permute(0, 3, 1, 2).contiguous().cpu().numpy()
    ora = torch.from_numpy(oops.roi_align_fwd(nchw, direct_rois.numpy(), SCALE, ph, pw, sr)).permute(0, 2, 3, 1)
    got32 = lay.run(torch.float32, rois, sr, 1).cpu()
    assert torch.equal(got32, ora), (what, "exact fp32 != oracle", int((got32 != ora).sum()))
    got16 = lay.run(torch.float16, rois, sr, 1).cpu()
    assert torch.equal(got16, ora.half()), (what, "exact fp16 != fp16(oracle)", int((got16 != ora.half()).sum()))

    # float64 reference on the frames the kernels read
    ref, out_abs = R.roi_align(feat32, rois, SCALE, ph, pw, *lay.fmap, sampling_ratio=sr) if strided else \
        R.roi_align(feat32, rois, SCALE, ph, pw, sampling_ratio=sr)
    spb, big_grid, wide, overflow = _paths(rois_cpu, ph, pw, H, W, sr)
    fma_tol = R.roi_align_fma_tol(out_abs, spb)
    fma = lay.run(torch.float16, rois, sr, 2).cpu()
    _note("fma (exact=2)", R._check_within(fma, ref, fma_tol, what + ("exact=2",)))

    # exact=0
    packed = lay.run(torch.float16, rois, sr, 0).cpu()
    fits = ph * pw * MERGED_BIN <= PACKED_SMEM
    if not fits:
        assert torch.equal(packed, fma), (what, "exact=0 without a packed table is the FMA kernel")
        return dict(spb=spb, big_grid=big_grid, wide=wide, overflow=overflow, table=torch.zeros(n, dtype=torch.bool))
    direct = big_grid | wide
    table = ~direct
    if bool(direct.any()):
        _note("packed direct (grid > 3x3)" if not bool(wide.any()) else "packed direct (incl. bins wider than the grid)",
              R._check_within(packed[direct], ref[direct], fma_tol[direct], what + ("exact=0 direct",)))
        same = (packed[direct] == fma[direct]).flatten(1).all(1)
        assert bool(same.all()), (what, "packed direct form != the FMA kernel", direct.nonzero().view(-1)[~same][:8].tolist())
    if bool(table.any()):
        tol = R.roi_align_tol(out_abs[table], float(feat32.abs().max()))
        _note("packed table", R._check_within(packed[table], ref[table], tol, what + ("exact=0 table",)))
    nvec = C // 8
    hv = nvec // 2 if nvec % 2 == 0 else nvec
    for parts in (2, 4):
        monkeypatch.setenv("STEP_B200_ROI_PARTS", str(parts))
        split = lay.run(torch.float16, rois, sr, 0).cpu()
        monkeypatch.delenv("STEP_B200_ROI_PARTS")
        assert torch.equal(split, packed), (what, "STEP_B200_ROI_PARTS=%d" % parts, hv % parts == 0)
    return dict(spb=spb, big_grid=big_grid, wide=wide, overflow=overflow, table=table)


def _feat(K, H, W, C, seed):
    """fp16-representable values, so that one fp32 oracle run serves the fp32 and the fp16 kernels."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(K, H, W, C, device="cuda", generator=g).half().float()


BINS = [(7, 7), (5, 3), (1, 1), (19, 19), (20, 20)]


@pytest.mark.parametrize("C,strided", [(8, False), (24, True), (64, False), (64, True)])
@pytest.mark.parametrize("bins", BINS, ids=["%dx%d" % b for b in BINS])
@pytest.mark.parametrize("sr", [0, 1, 2, 3, 4])
def test_roi_align_fwd_edges(C, strided, bins, sr, monkeypatch):
    ph, pw = bins
    H = W = 28
    rois = _rois()
    feat = _feat(8 if strided else 4, H, W, C, 52 + C + sr)
    p = _check(feat, rois, ph, pw, sr, strided, monkeypatch, ("edges", C, strided, bins, sr))
    # the dispatch this sweep relies on, so that a change to a threshold is noticed
    if bins == (7, 7) and sr == 0:
        assert int(p["spb"][0]) * 49 == TAPS and int(p["spb"][2]) == 25   # a full cached table and an uncached one
        assert bool(p["table"].any()) and bool(p["big_grid"].any()) and not bool(p["wide"].any())
    if bins == (7, 7) and sr == 3:
        assert bool(p["overflow"][2]) and bool(p["overflow"][3])          # bins of 5 and 10 px: 36 distinct pixels
        assert bool(p["wide"][2]) and bool(p["wide"][3]) and bool(p["table"].any())
    if sr == 4:
        assert not bool(p["table"].any())                                 # grid 4 x 4: (4 + 1)^2 > 16
    if bins == (19, 19) and sr != 4:
        assert bool(p["table"].any())                                     # 361 x 136 B = 49 096 B fit
    if bins == (20, 20):
        assert not bool(p["table"].any())


@pytest.mark.parametrize("sr", [0, 1, 2, 3, 4])
def test_roi_align_fwd_shipped_map(sr, monkeypatch):
    """The shipped map, 25 x 25 x 832 (C / 8 = 104: roi_gather_items<2>), 7 x 7 bins, with the strided layout."""
    rois = _rois(100, seed=53)
    feat = _feat(8, 25, 25, 832, 54 + sr)
    _check(feat, rois, 7, 7, sr, True, monkeypatch, ("shipped", sr))


REACH = [r"roi_align_fwd_nhwc_f16_packed_kernel", r"roi_align_fwd_nhwc_kernel<__half, ?false>",
         r"roi_align_fwd_nhwc_kernel<__half, ?true>", r"roi_align_fwd_nhwc_kernel<float, ?true>"]


def profiled_kernel_names():
    """Kernel names of the four kinds of launch (exact 1 fp32, 1 fp16, 2, 0 at 7 x 7 and at 20 x 20) under torch.profiler,
    in a child process (see test_gpu_forward_layers.profiled_kernel_names)."""
    rois = _rois(20).cuda()
    feat = _feat(4, 28, 28, 64, 55)
    runs = [(torch.float32, 1, 7), (torch.float16, 1, 7), (torch.float16, 2, 7), (torch.float16, 0, 7), (torch.float16, 0, 20)]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for dtype, exact, ps in runs:
            out = torch.empty(rois.shape[0], ps, ps, 64, dtype=dtype, device="cuda")
            _launch(feat.to(dtype), 4, 28, 28, 64, 64, rois, ps, ps, 0, out, 64, (0, 0, 0), exact)
        torch.cuda.synchronize()
    return sorted({e.key for e in prof.key_averages()})


def test_every_forward_kernel_is_reached():
    child = subprocess.run([sys.executable, os.path.abspath(__file__)], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert child.returncode == 0, child.stderr[-4000:]
    names = json.loads(child.stdout.strip().splitlines()[-1])
    missing = [p for p in REACH if not any(re.search(p, n) for n in names)]
    assert not missing, (missing, [n for n in names if "roi" in n])


if __name__ == "__main__":                                     # test_every_forward_kernel_is_reached's child process
    print(json.dumps(profiled_kernel_names()))
