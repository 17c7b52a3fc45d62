"""BASELINE.json configs 2 and 3 on one H100 (CUDA events, >= 5 warm-ups, inputs larger than L2 or L2 flushed).

  C2  I3D trunk only, batch 4, T=32, 224x224, fp16 storage / fp32 accumulate      -> clips/s, TFLOP/s, frac of bf16 peak
  C3a ROIAlign, 10 000 tubes x T'=8 = 80 000 ROI rows over a [64,14,14,832] map     -> GB/s of algorithmic bytes, frac of HBM peak
  C3b NMS, the 10 000 tube boxes, thr 0.4 (bit-exact vs the oracle)                 -> ms, boxes/s
Prints one JSON object; `python tools/microbench.py > microbench.json`."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import step_b200
from _bench import card
from step_b200 import _lib as L, engine as E, synth
from step_b200.engine import Act
from step_b200.roi_layers import nms

PEAKS = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json"))) \
    if os.path.exists(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")) else \
    {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0}   # H100 SXM data sheet (700 W)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def timeit(fn, reps=20, warm=5, flush_l2=False):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(reps):
        if flush_l2:
            flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / reps


out = {"card": card(0), "peaks": {"hbm_gbs": PEAKS["hbm_gbs"], "bf16_tflops_burst": PEAKS["bf16_tflops"], "bf16_tflops_sustained": PEAKS["bf16_tflops_sustained"]}}

# ---- C2: trunk only ---------------------------------------------------------------------------
cfg = synth.make_cfg(fp16=True)
base = step_b200.BaseNet(cfg); base.load_state_dict(synth.base_net_state_dict()); base = base.cuda().eval()
x = synth.make_clips(4, 32, 224, 224).cuda()
with torch.no_grad():
    ms_eager = timeit(lambda: base.forward_act(x), reps=20, warm=5)
    # the same launches as one CUDA graph (how StepRunner / bench.py run them): no Python between kernels
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        base.forward_act(x)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        feat_static = base.forward_act(x)
    ms = timeit(graph.replay, reps=20, warm=5)
gflop = 109.29 * 4
out["C2_trunk_b4_fp16"] = {"ms": round(ms, 3), "ms_eager": round(ms_eager, 3), "clips_per_s": round(4 / ms * 1e3, 1),
                           "tflops": round(gflop / ms, 1),
                           "frac_of_bf16_sustained": round(gflop / ms / PEAKS["bf16_tflops_sustained"], 3),
                           "algorithmic_gflop": gflop,
                           "note": "one CUDA graph per forward (ms_eager: Python-launched), inputs 77 MB fp32 (> L2 with activations)"}

# ---- C3a: ROIAlign ----------------------------------------------------------------------------
rois_np, boxes_np, scores_np = synth.make_c3_rois()
rois = torch.from_numpy(rois_np).cuda()
R = rois.shape[0]
g = torch.Generator().manual_seed(1234)
feat32 = torch.randn(64, 14, 14, 832, generator=g).cuda()
for name, code, feat, exact in (("fp32", L.F32, feat32, 1), ("fp16", L.F16, feat32.half(), 1), ("fp16_fma", L.F16, feat32.half(), 2), ("fp16_packed", L.F16, feat32.half(), 0)):
    o = torch.empty((R, 7, 7, 832), dtype=feat.dtype, device="cuda")

    def run():
        L.check(L.lib().step_roi_align_fwd_nhwc(L.ptr(feat), code, 64, 14, 14, 832, 832, L.ptr(rois), R, 1 / 16., 7, 7, 0,
                                                L.ptr(o), 832, 0, 0, 0, exact, L.stream()))
    ms = timeit(run, reps=10, warm=5)  # output 6.5 / 13 GB >> L2
    es = feat.element_size()
    bytes_alg = R * 832 * 49 * es + feat.numel() * es + R * 20
    # bit-exactness spot check against the oracle on 64 random rows (fp32) / round-to-half (fp16)
    from oracle import ops as oops
    idx = np.random.RandomState(0).choice(R, 64, replace=False)
    ref = oops.roi_align_fwd(feat.float().cpu().numpy().transpose(0, 3, 1, 2), rois_np[idx], 1 / 16., 7, 7, 0)
    got = o[torch.from_numpy(idx).cuda()].float().cpu().numpy().transpose(0, 3, 1, 2)
    refq = ref if code == L.F32 else ref.astype(np.float16).astype(np.float32)
    is_exact = bool(np.array_equal(got, refq))
    max_ulp_err = float(np.abs(got - refq).max() / max(np.abs(refq).max(), 1e-9))
    out["C3_roi_align_%s" % name] = {"ms": round(ms, 3), "gbytes_algorithmic": round(bytes_alg / 1e9, 3),
                                     "gb_per_s": round(bytes_alg / ms / 1e6, 1),
                                     "frac_of_hbm_peak": round(bytes_alg / ms / 1e6 / PEAKS["hbm_gbs"], 3),
                                     "rows": R, "bit_exact_vs_oracle_on_64_rows": is_exact, "max_rel_err": max_ulp_err}
    del o

# ---- C3b: NMS ---------------------------------------------------------------------------------
b, s = torch.from_numpy(boxes_np).cuda(), torch.from_numpy(scores_np).cuda()
keep = nms(b, s, 0.4)
ms = timeit(lambda: nms(b, s, 0.4), reps=20, warm=5)
from oracle import ops as oops
exact = bool(np.array_equal(keep.cpu().numpy(), oops.nms(boxes_np, scores_np, 0.4)))
out["C3_nms_10k"] = {"ms": round(ms, 3), "boxes_per_s": round(10000 / ms * 1e3), "kept": int(keep.numel()),
                     "bit_exact_vs_oracle": exact, "note": "includes the one D2H of the keep count (python wrapper)"}
print(json.dumps(out, indent=1))
