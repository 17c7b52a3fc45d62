"""Generates tests/golden/roi_bwd_bits.npz: the exact bits of the deterministic channels-last ROI backward entries
(step_roi_align_bwd_nhwc, step_roi_align_bwd_slice_nhwc, step_roi_pool_bwd_slice_nhwc), so that a later build of these
kernels can be held to the same summation order, bit for bit.  Run once on a GPU with the build whose bits are pinned:

    python tests/golden/make_roi_bwd_golden.py

Every operand is drawn from numpy.random.default_rng(seed) (`operands`), so any machine rebuilds it from CASES; `run`
calls the entry on it and returns the output bytes.  The ROIPool backward is fed the argmax that
step_roi_pool_fwd_argmax_nhwc records on a drawn feature map.  Cases cover the shipped step's operands (2 clips, 9 frames
of 25 x 25 x 832, 34 tubes per clip, steps of 3 and 9 frames), the classification stage's (4 clips, 20 tubes, 9 frames)
and small edge cases, whose outputs are also stored in full.

Keys, per case <name> and grad_out dtype <dt> (f32, f16; ROIPool: f32 and f16 too):
  <name>_<dt>_sha     SHA-256 of the grad_in bytes after the call
  <name>_<dt>_out     grad_in itself (edge cases only)
  <name>_argmax_sha   SHA-256 of the argmax feeding a ROIPool case
  cases               CASES as JSON
"""
import hashlib
import json
import os
import sys

import numpy as np

OUT = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(OUT))

SCALE = 1.0 / 16.0
PH = PW = 7

# kind: align (step_roi_align_bwd_nhwc), align_slice, pool_slice.  K frames of H x W x C (grad_in channel stride in_ld),
# R rows (grad_out channel stride out_ld) on `frames` ROI frames; roi_T / feat_T / t_start: the slice frame map.
# oob: rows whose frame index lies outside [0, frames) (the entries ignore them).  neg0: grad_in starts with -0.0 entries.
_SHIP = dict(K=18, H=25, W=25, C=832, in_ld=832, out_ld=832, sr=0, oob=0, neg0=0)
CASES = [
    dict(name="shipped_whole", kind="align", R=204, frames=18, roi_T=0, feat_T=0, t_start=0, seed=11, **_SHIP),
    dict(name="shipped_step3", kind="align_slice", R=204, frames=6, roi_T=3, feat_T=9, t_start=3, seed=12, **_SHIP),
    dict(name="shipped_step9", kind="align_slice", R=612, frames=18, roi_T=9, feat_T=9, t_start=0, seed=13, **_SHIP),
    dict(name="cls_step9", kind="align_slice", R=720, frames=36, roi_T=9, feat_T=9, t_start=0, seed=14,
         **dict(_SHIP, K=36)),
    dict(name="pool_shipped_step3", kind="pool_slice", R=204, frames=6, roi_T=3, feat_T=9, t_start=6, seed=15, **_SHIP),
    dict(name="pool_shipped_step9", kind="pool_slice", R=612, frames=18, roi_T=9, feat_T=9, t_start=0, seed=16, **_SHIP),
    dict(name="pool_cls_step9", kind="pool_slice", R=720, frames=36, roi_T=9, feat_T=9, t_start=0, seed=17,
         **dict(_SHIP, K=36)),
    # edges: strided operands, sampling ratio 2, ROIs across / outside the map and of zero area, unsorted frames,
    # frames without a row, rows outside the frame range, -0.0 in grad_in, R = 0, a 100 x 100 plane
    dict(name="edge_sr2", kind="align", K=4, H=7, W=9, C=12, in_ld=16, out_ld=20, R=11, frames=4, roi_T=0, feat_T=0,
         t_start=0, sr=2, oob=2, neg0=1, seed=21),
    dict(name="edge_sr0", kind="align", K=3, H=11, W=6, C=4, in_ld=4, out_ld=8, R=9, frames=3, roi_T=0, feat_T=0,
         t_start=0, sr=0, oob=1, neg0=1, seed=22),
    dict(name="edge_slice", kind="align_slice", K=6, H=8, W=5, C=8, in_ld=12, out_ld=8, R=7, frames=4, roi_T=2,
         feat_T=3, t_start=1, sr=0, oob=2, neg0=1, seed=23),
    dict(name="edge_slice_r0", kind="align_slice", K=4, H=5, W=5, C=4, in_ld=4, out_ld=4, R=0, frames=2, roi_T=1,
         feat_T=2, t_start=1, sr=0, oob=0, neg0=1, seed=24),
    dict(name="edge_r0", kind="align", K=2, H=5, W=5, C=4, in_ld=8, out_ld=4, R=0, frames=2, roi_T=0, feat_T=0,
         t_start=0, sr=0, oob=0, neg0=1, seed=25),
    dict(name="edge_plane100", kind="align", K=2, H=100, W=100, C=8, in_ld=8, out_ld=8, R=6, frames=2, roi_T=0,
         feat_T=0, t_start=0, sr=0, oob=0, neg0=0, seed=26),
    dict(name="edge_pool", kind="pool_slice", K=6, H=9, W=7, C=8, in_ld=12, out_ld=12, R=9, frames=4, roi_T=2,
         feat_T=3, t_start=0, sr=0, oob=0, neg0=1, seed=27),
    dict(name="edge_pool_r0", kind="pool_slice", K=2, H=4, W=4, C=8, in_ld=8, out_ld=8, R=0, frames=2, roi_T=1,
         feat_T=1, t_start=0, sr=0, oob=0, neg0=1, seed=28),
]
EDGE = [c["name"] for c in CASES if c["name"].startswith("edge_")]


def operands(c):
    """numpy operands of case c: rois [R,5], grad_out [R,PH,PW,out_ld] fp32, grad_in (initial) [K,H,W,in_ld] fp32,
    feat [K,H,W,C] fp32 (the ROIPool forward's input)."""
    rng = np.random.default_rng(c["seed"])
    R, K, H, W, C = c["R"], c["K"], c["H"], c["W"], c["C"]
    img_w, img_h = W / SCALE, H / SCALE
    f = rng.integers(0, c["frames"], R).astype(np.float32)        # unsorted; some frames may have no row
    x1 = rng.uniform(-0.15, 0.95, R) * img_w
    y1 = rng.uniform(-0.15, 0.95, R) * img_h
    x2 = x1 + rng.uniform(0.0, 0.7, R) * img_w
    y2 = y1 + rng.uniform(0.0, 0.7, R) * img_h
    rois = np.stack([f, x1, y1, x2, y2], 1).astype(np.float32)
    if R >= 4:
        rois[1, 3] = rois[1, 1]                                  # zero width
        rois[2, 1:] = [img_w * 1.2, img_h * 1.1, img_w * 1.5, img_h * 1.4]   # wholly outside the map
        rois[3, 1:] = [-img_w, -img_h, img_w * 2, img_h * 2]      # larger than the map on every side
    for i in range(c["oob"]):
        rois[R - 1 - i, 0] = -1 if i % 2 == 0 else c["frames"]
    go = np.zeros((R, PH, PW, c["out_ld"]), np.float32)
    go[..., :C] = rng.standard_normal((R, PH, PW, C), np.float32)
    gin = rng.standard_normal((K, H, W, c["in_ld"]), np.float32)
    if c["neg0"]:
        gin[rng.random(gin.shape) < 0.3] = -0.0
    feat = rng.standard_normal((K, H, W, C), np.float32)
    return rois, go, gin, feat


def _cu(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def pool_argmax(c, rois, feat):
    """argmax [R,PH,PW,C] of step_roi_pool_fwd_argmax_nhwc on feat with the case's frame map."""
    import torch
    from step_b200 import _lib as L
    R, C = c["R"], c["C"]
    am = torch.full((max(R, 1), PH, PW, C), -7, dtype=torch.int32, device="cuda")
    out = torch.empty((max(R, 1), PH, PW, C), dtype=torch.float32, device="cuda")
    ft, r = _cu(feat), _cu(rois)
    L.check(L.lib().step_roi_pool_fwd_argmax_nhwc(L.ptr(ft), L.F32, c["K"], c["H"], c["W"], C, C, L.ptr(r), R, SCALE, PH, PW,
                                                  L.ptr(out), C, c["roi_T"], c["feat_T"], c["t_start"], L.ptr(am), L.stream()))
    return am


def run(c, dt, stream=None):
    """grad_in after the case's entry on grad_out stored as dt (torch.float32 | torch.float16), as a CUDA tensor; on
    `stream` (torch.cuda.Stream) when given.  Returns (grad_in, argmax or None)."""
    import torch
    from step_b200 import _lib as L
    rois, go, gin, feat = operands(c)
    am = pool_argmax(c, rois, feat) if c["kind"] == "pool_slice" else None
    r, g, out = _cu(rois), _cu(go).to(dt), _cu(gin)
    R, K, H, W, C = c["R"], c["K"], c["H"], c["W"], c["C"]
    s = stream or torch.cuda.current_stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        code = L.dt(g)
        if c["kind"] == "align":
            L.check(L.lib().step_roi_align_bwd_nhwc(L.ptr(g), code, c["out_ld"], L.ptr(r), R, SCALE, PH, PW, K, H, W, C, c["sr"],
                                                    L.ptr(out), c["in_ld"], L.stream()))
        elif c["kind"] == "align_slice":
            nb = L.lib().step_roi_align_bwd_slice_workspace_bytes(K, H, W, C, c["roi_T"], c["feat_T"])
            ws = torch.full((max(nb, 16) // 4,), float("nan"), dtype=torch.float32, device="cuda")
            L.check(L.lib().step_roi_align_bwd_slice_nhwc(L.ptr(g), code, c["out_ld"], L.ptr(r), R, SCALE, PH, PW, K, H, W, C,
                                                          c["sr"], c["roi_T"], c["feat_T"], c["t_start"], L.ptr(out), c["in_ld"],
                                                          L.ptr(ws), ws.numel() * 4, L.stream()))
        else:
            L.check(L.lib().step_roi_pool_bwd_slice_nhwc(L.ptr(g), code, c["out_ld"], L.ptr(am), L.ptr(r), R, PH, PW, K, H, W, C,
                                                         c["roi_T"], c["feat_T"], c["t_start"], L.ptr(out), c["in_ld"],
                                                         L.stream()))
    torch.cuda.synchronize()
    return out, am


def sha(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def main():
    import torch
    sys.path.insert(0, ROOT)
    out = {"cases": np.array(json.dumps(CASES))}
    for c in CASES:
        for tag, dt in (("f32", torch.float32), ("f16", torch.float16)):
            gin, am = run(c, dt)
            out["%s_%s_sha" % (c["name"], tag)] = np.array(sha(gin))
            if c["name"] in EDGE:
                out["%s_%s_out" % (c["name"], tag)] = gin.cpu().numpy()
            if am is not None:
                out["%s_argmax_sha" % c["name"]] = np.array(sha(am))
    path = os.path.join(OUT, "roi_bwd_bits.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d keys)" % (path, len(out)))


if __name__ == "__main__":
    main()
