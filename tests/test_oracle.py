"""CPU: pins oracle/ (C restatement + torch-CPU restatement) against the committed golden vectors
that tests/golden/make_golden.py produced by running the unmodified reference."""
import numpy as np
import pytest
import torch

from oracle import model as om
from oracle import ops, tubes
from step_b200 import synth

NMS_CASES = ["iou_eq_thr", "four", "third", "empty", "single", "rand63", "rand64", "rand65", "rand129",
             "rand1000", "intgrid"]


@pytest.mark.parametrize("name", NMS_CASES)
def test_nms_oracle_matches_reference(golden, name):
    g = golden("nms_cases")
    keep = ops.nms(g[name + "_boxes"], g[name + "_scores"], float(g[name + "_thr"]))
    assert keep.dtype == np.int64
    assert np.array_equal(keep, g[name + "_keep"])


def test_nms_known_answers():
    # SURVEY.md appendix A probes of the reference
    b = np.array([[0, 0, 10, 10], [1, 1, 11, 11], [50, 50, 60, 60], [0, 0, 10, 10]], np.float32)
    assert ops.nms(b, np.array([.9, .8, .7, .95], np.float32), 0.4).tolist() == [2, 3]
    b = np.array([[0, 0, 9, 9], [0, 0, 9, 4]], np.float32)
    s = np.array([.9, .8], np.float32)
    assert ops.nms(b, s, 0.5, ge=True).tolist() == [0]       # cpu/nms_cpu.cpp:84  '>='
    assert ops.nms(b, s, 0.5, ge=False).tolist() == [0, 1]   # cuda/nms.cu:84      '>'
    # tie on scores: our contract is (score desc, index asc); torch.sort is unstable for n > 16
    b = np.array([[0, 0, 9, 9], [1, 1, 10, 10], [100, 100, 110, 110]], np.float32)
    assert ops.nms(b, np.full(3, .5, np.float32), 0.4).tolist() == [0, 2]


def test_roi_align_oracle_bit_exact(golden):
    g = golden("roi_align_cases")
    for sr in (0, 2):
        out = ops.roi_align_fwd(g["feat"], g["rois"], 1.0 / 16.0, 7, 7, sr)
        assert np.array_equal(out, g["out_sr%d" % sr])
    rois = g["rois"] * np.array([1, .1, .1, .1, .1], np.float32)
    assert np.array_equal(ops.roi_align_fwd(g["feat"], rois, 0.5, 3, 5, 0), g["out_3x5_s0p5"])


def test_roi_align_bwd_is_adjoint_of_fwd(golden):
    g = golden("roi_align_cases")
    feat, rois = g["feat"], g["rois"]
    K, C, H, W = feat.shape
    rs = np.random.RandomState(0)
    gout = rs.randn(rois.shape[0], C, 7, 7).astype(np.float32)
    gin = ops.roi_align_bwd(gout, rois, 1 / 16., 7, 7, K, C, H, W, 0)
    lhs = float((ops.roi_align_fwd(feat, rois, 1 / 16., 7, 7, 0).astype(np.float64) * gout).sum())
    rhs = float((feat.astype(np.float64) * gin).sum())
    assert abs(lhs - rhs) <= 1e-4 * max(1.0, abs(lhs))


def test_roi_pool_properties():
    rs = np.random.RandomState(1)
    feat = rs.randn(2, 3, 14, 14).astype(np.float32)
    rois = np.array([[0, 0, 0, 223, 223], [1, 16, 16, 47, 47], [1, 500, 500, 600, 600]], np.float32)
    out, arg = ops.roi_pool_fwd(feat, rois, 1 / 16., 7, 7)
    # whole-map ROI: rounded to [0,14] -> 15 wide, bins cover every cell; global max is present
    assert np.isclose(out[0].max(axis=(1, 2)), feat[0].max(axis=(1, 2))).all()
    # argmax indexes the value it reports
    flat = feat[1].reshape(3, -1)
    for c in range(3):
        assert np.array_equal(out[1, c].ravel(), flat[c][arg[1, c].ravel()])
    # empty region -> 0 and argmax -1  (ROIPool_cuda.cu:78-84)
    assert (out[2] == 0).all() and (arg[2] == -1).all()
    gin = ops.roi_pool_bwd(np.ones_like(out), arg, rois, 7, 7, 2, 3, 14, 14)
    assert gin.sum() == (arg != -1).sum()


def test_tube_ops_match_reference(golden):
    g = golden("tubes_cases")
    dec = tubes.decode_coef(g["dec_anchors"], g["dec_deltas"],
                            exp=lambda v: torch.exp(torch.from_numpy(np.ascontiguousarray(v))).numpy())
    assert np.array_equal(dec, g["dec_out"])
    assert np.allclose(tubes.encode_coef(g["enc_gt"], g["dec_anchors"]), g["enc_out"], rtol=1e-6, atol=1e-6)
    assert np.array_equal(tubes.valid_tubes(g["val_in"], 224, 224), g["val_out_224"])
    assert np.array_equal(tubes.valid_tubes(g["val_in"]), g["val_out_400"])
    for T in (2, 3, 4):
        assert np.array_equal(tubes.extrapolate_tubes(g["ext_in_T%d" % T], T), g["ext_out_T%d" % T])
    lst = [g["val_in"][:2], np.zeros((0, 4, 4), np.float32), g["val_in"][2:5]]
    flat, nums = tubes.flatten_tubes(lst, batch_idx=True)
    assert np.array_equal(flat, g["flat_out"]) and nums == g["flat_nums"].tolist()
    assert np.array_equal(tubes.extend_tubes(flat, 1.2, 224, 224), g["extend_out"])


PIPES = {
    "pipe_c1": dict(cfg=dict(T=2, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(112, 112))),
    "pipe_spatial": dict(cfg=dict(T=4, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 1}, image_size=(112, 112))),
    "pipe_temporal_predict": dict(cfg=dict(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3},
                                           temporal_mode="predict", image_size=(112, 112))),
    "pipe_temporal_extrapolate": dict(cfg=dict(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3},
                                               temporal_mode="extrapolate", image_size=(112, 112))),
    "pipe_temporal_mean": dict(cfg=dict(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3},
                                        temporal_mode="mean", image_size=(112, 112))),
}


@pytest.mark.parametrize("name", list(PIPES))
def test_pipeline_oracle_matches_reference(golden, name):
    """Same torch CPU backend + same thread count => the restatement must be bit-identical to the
    reference modules; allow 1e-5 rel for a different host thread count (SURVEY.md section 8c)."""
    g = golden(name)
    cfg = synth.make_cfg(**PIPES[name]["cfg"])
    B, T_in, HW, N = int(g["B"]), int(g["T_in"]), int(g["HW"]), int(g["N"])
    x = synth.make_clips(B, T_in, HW, HW)
    with torch.no_grad():
        cf = om.base_net(x, synth.base_net_state_dict())
        tol = dict(rtol=1e-4, atol=1e-4)
        if "conv_feat" in g:
            assert np.allclose(cf.numpy(), g["conv_feat"], **tol)
        heads = [synth.head_state_dict(100 + i, cfg) for i in range(cfg.max_iter)]
        tb = synth.make_proposals(B, N, cfg.T * cfg.NUM_CHUNKS[1], HW, HW)
        hist, traj = om.inference(cfg, cf, None, heads, cfg.max_iter, tb)
    for i, h in enumerate(hist):
        assert np.allclose(h["pred_prob"][:, 0].numpy(), g["prob%d" % i], rtol=1e-4, atol=1e-5)
        # the reference's CPU history['pred_loc'] is aliased and mutated by valid_tubes
        # (utils.py:107-121) except at a step that extends the tubes (cat/extrapolate make a copy)
        extends = i + 1 < cfg.max_iter and cfg.NUM_CHUNKS[i + 2] == cfg.NUM_CHUNKS[i + 1] + 2
        v = h["pred_loc"].numpy() if extends else tubes.valid_tubes(h["pred_loc"].numpy(), HW, HW)
        assert np.allclose(v, g["loc_valid%d" % i], rtol=1e-4, atol=1e-3)
        assert h["tubes_nums"] == g["nums%d" % i].tolist()
        assert np.allclose(np.concatenate([t[0] for t in traj[i]], 0), g["traj%d" % i], rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("name", list(synth.LOSS_CASES))
def test_head_losses_oracle_matches_reference(golden, name):
    """Training-time outputs of TwoBranchNet.forward(targets=...) (two_branch.py:276-341): BCE-with-logits on the
    centre chunk, masked smooth-L1 on encode_coef targets, neighbour smooth-L1.  Pins the oracle restatement the
    round-2 training path will be checked against; inputs are regenerated from the seed (checksum stored)."""
    g = golden("losses_cases")
    T_, chunks, _, _ = synth.LOSS_CASES[name]
    cfg = synth.make_cfg(T=T_, max_iter=1, NUM_CHUNKS={1: chunks}, image_size=(112, 112))
    _, _, feat, tb, tg = synth.make_loss_case(name, cfg.num_classes)
    assert abs(float(feat.double().sum()) - float(g[name + "_feat_checksum"][0])) < 1e-6   # same seeded inputs
    with torch.no_grad():
        prob, loc, first, last, logits = om.two_branch(feat, synth.head_state_dict(100, cfg), cfg.T, None, cfg.fc_dim,
                                                       cfg.pool_size, return_logits=True)
        lc, ll, ln = om.two_branch_losses(logits, loc, first, last, tb, tg, cfg.T)
    assert np.allclose(prob.numpy(), g[name + "_prob"], rtol=1e-4, atol=1e-5)
    assert np.allclose(loc.numpy(), g[name + "_loc"], rtol=1e-4, atol=1e-5)
    assert lc.shape == tuple(g[name + "_loss_cls"].shape)
    assert np.allclose(lc.numpy(), g[name + "_loss_cls"], rtol=1e-4, atol=1e-6)
    assert np.allclose(ll.numpy(), g[name + "_loss_loc"], rtol=1e-4, atol=1e-6)
    assert np.allclose(ln.numpy(), g[name + "_loss_nb"], rtol=1e-4, atol=1e-6)
    if name == "nomask":   # no positive sample: the three losses are the scalar 0 (two_branch.py:278-280)
        assert lc.numel() == 1 and float(lc) == 0.0 and float(ll) == 0.0 and float(ln) == 0.0


def test_head_gradients_oracle_matches_reference(golden):
    """Backward of the head's training objective (train.py:323-347 with train_step.sh's lambdas) through the oracle's
    functional model equals the reference's autograd result: per-parameter gradient norms and leading values.
    This is the checker for the round-2 dgrad / wgrad kernels."""
    g = golden("head_grads")
    name = "c1"
    T_, chunks, _, _ = synth.LOSS_CASES[name]
    cfg = synth.make_cfg(T=T_, max_iter=1, NUM_CHUNKS={1: chunks}, image_size=(112, 112))
    sd = {k: v.clone().requires_grad_(v.is_floating_point() and "running_" not in k)
          for k, v in synth.head_state_dict(100, cfg).items()}
    _, _, feat, tb, tg = synth.make_loss_case(name, cfg.num_classes)
    feat = feat.clone().requires_grad_(True)
    prob, loc, first, last, logits = om.two_branch(feat, sd, cfg.T, None, cfg.fc_dim, cfg.pool_size, return_logits=True)
    lc, ll, ln = om.two_branch_losses(logits, loc, first, last, tb, tg, cfg.T)
    loss = lc.mean() + ll.mean() * 5.0 + ln.mean() * 1.0
    loss.backward()
    assert np.allclose(loss.detach().numpy(), g["loss"], rtol=1e-5)
    assert np.allclose(feat.grad.double().norm().numpy(), g["feat_grad_norm"], rtol=1e-4)
    assert np.allclose(feat.grad.reshape(-1)[:16].numpy(), g["feat_grad_head"], rtol=1e-3, atol=1e-7)
    checked = 0
    for k in g.files:
        if not k.startswith("gn:"):
            continue
        p = sd[k[3:]]
        assert p.grad is not None, k
        assert np.allclose(p.grad.double().norm().numpy(), g[k], rtol=1e-4, atol=1e-9), k
        assert np.allclose(p.grad.reshape(-1)[:8].numpy(), g["gh:" + k[3:]], rtol=1e-3, atol=1e-7), k
        checked += 1
    assert checked >= 50   # every trainable tensor of the head (BatchNorm statistics excluded)


def test_trunk_gradients_oracle_matches_reference(golden):
    """Backward of the I3D trunk (45 Unit3D convolutions, BatchNorm eval + frozen affine) through the oracle's
    functional model equals the reference's autograd result.  Checker for the round-2 conv dgrad / wgrad kernels."""
    g = golden("trunk_grads")
    sd = {k: v.clone().requires_grad_(k.endswith("conv3d.weight")) for k, v in synth.base_net_state_dict().items()}
    x = synth.make_clips(1, 8, 64, 64, seed=4321).requires_grad_(True)
    cf = om.base_net(x, sd)
    proj = torch.randn(cf.shape, generator=torch.Generator().manual_seed(99))
    loss = (cf * proj).sum() / cf.numel()
    loss.backward()
    assert np.allclose(loss.detach().numpy(), g["loss"], rtol=1e-4, atol=1e-8)
    assert np.allclose(x.grad.double().norm().numpy(), g["x_grad_norm"], rtol=1e-3)
    checked = 0
    for k in g.files:
        if not k.startswith("gn:"):
            continue
        p = sd[k[3:]]
        assert p.grad is not None, k
        assert np.allclose(p.grad.double().norm().numpy(), g[k], rtol=1e-3, atol=1e-10), k
        assert np.allclose(p.grad.reshape(-1)[:8].numpy(), g["gh:" + k[3:]], rtol=2e-3, atol=1e-8), k
        checked += 1
    assert checked == 45   # one weight per Unit3D of the trunk (i3dpt.py:184-226); BN affine is frozen


def _det_key(rows):
    """(clip, class, score to 4 significant digits) multiset of detection rows, plus the boxes in that order."""
    fmt = lambda v: float("{:.4}".format(float(v)))   # the reference writes rows with '{:.4}' (test.py:211-218)
    keyed = sorted(((int(r[0]), int(r[1]), fmt(r[2])) + tuple(fmt(v) for v in r[3:7])) for r in rows)
    return keyed


@pytest.mark.parametrize("name", ["synth", "synth_topk", "c4"])
def test_postprocess_oracle_matches_reference_loop(golden, name):
    """oracle/postprocess.py against the rows the reference's OWN evaluation loop (test.py:156-218, executed from the
    file where it lies by tests/golden/make_golden.py::gen_postprocess) wrote for the same history."""
    from oracle import postprocess as opp
    g = golden("postprocess_cases")
    conf, thr, topk, width, height = g[name + "_cfg"].tolist()
    prob, loc, nums = g[name + "_prob"], g[name + "_loc"], g[name + "_nums"].tolist()
    dets = opp.detections(prob, loc[:, loc.shape[1] // 2].copy(), nums, conf, thr, width, height, topk=int(topk))
    rows = [(b, c, s) + tuple(bx) for b, d in enumerate(dets) for (bx, c, s) in d]
    ref = g[name + "_rows"]
    assert len(rows) == ref.shape[0]
    if int(topk) > 0:
        # ties at the k-th score are broken by (class, index) descending in the reference's tuple sort; the synthetic
        # scores are distinct, so the kept multiset is well defined
        assert len(set(np.round(ref[:, 2], 6))) == ref.shape[0]
    assert _det_key(rows) == _det_key(ref)


def _rows4(rows):
    """Detection rows (clip, class, score, box) as the reference writes them, 4 significant digits ('{:.4}'), in order."""
    fmt = lambda v: float("{:.4}".format(float(v)))
    return [(int(r[0]), int(r[1])) + tuple(fmt(v) for v in r[2:7]) for r in rows]


@pytest.mark.parametrize("name", ["ties", "ties_topk", "ties_topk_all"])
def test_postprocess_oracle_row_order_matches_reference_loop(golden, name):
    """oracle/postprocess.py writes the same rows in the same order as the reference's own loop
    (tests/golden/make_golden.py::gen_detect_edges) on scores with exact ties across and within classes, at the top-k cut
    and away from it, scores equal to conf_thresh and degenerate boxes: file order for topk 0, tied scores in reverse file
    order under a top-k sort."""
    from oracle import postprocess as opp
    g = golden("detect_edge_cases")
    conf, thr, topk, width, height = g[name + "_cfg"].tolist()
    prob, loc, nums = g[name + "_prob"], g[name + "_loc"], g[name + "_nums"].tolist()
    dets = opp.detections(prob, loc[:, loc.shape[1] // 2].copy(), nums, conf, thr, width, height, topk=int(topk))
    rows = [(b, c, s) + tuple(bx) for b, d in enumerate(dets) for (bx, c, s) in d]
    ref = g[name + "_rows"]
    assert _rows4(rows) == _rows4(ref)
    # the case exercises what it is for: tied scores next to each other in the output, and at the cut
    s = ref[:, 2]
    assert bool((s[1:] == s[:-1]).any())
    assert not bool((prob == np.float32(conf)).all()) and bool((prob == np.float32(conf)).any())
    if name == "ties_topk":
        full = opp.detections(prob, loc[:, loc.shape[1] // 2].copy(), nums, conf, thr, width, height, topk=10 ** 6)
        cut = [d for d in full if len(d) > int(topk)]
        assert cut and all(d[int(topk) - 1][2] == d[int(topk)][2] for d in cut)      # the cut splits a run of ties


def test_roi_pool_and_align_backward_match_torchvision(golden):
    """ROIPool fwd/bwd and ROIAlign bwd have no CPU implementation in the reference (ROIPool.h:47, ROIAlign.h:66), so
    the C restatement (cuda/ROIPool_cuda.cu:40-132, cuda/ROIAlign_cuda.cu:201-278) is cross-checked against
    torchvision's CPU ops -- a second implementation of the same Caffe2 lineage whose roi_align(aligned=False) forward
    is bit-identical to the reference's (asserted when the fixture was generated)."""
    g, a = golden("roi_cross_cases"), golden("roi_align_cases")
    feat, rois = a["feat"], a["rois"]
    K, C, H, W = feat.shape
    for sr in (0, 2):
        gin = ops.roi_align_bwd(g["align_gy_sr%d" % sr], rois, 1 / 16., 7, 7, K, C, H, W, sr)
        ref = g["align_gx_sr%d" % sr]
        assert np.abs(gin - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max())   # summation order differs
    out, arg = ops.roi_pool_fwd(feat, rois, 1 / 16., 7, 7)
    assert np.array_equal(out, g["pool_out"])
    gin = ops.roi_pool_bwd(g["pool_gy"], arg, rois, 7, 7, K, C, H, W)
    assert np.abs(gin - g["pool_gx"]).max() <= 2e-5 * max(1.0, np.abs(g["pool_gx"]).max())


def test_oracle_matches_reference_at_the_measured_c4_shape(golden):
    """The CPU pass bench.py times (and uses as its same-run parity reference) is this oracle at the C4 shape: pin it to
    the reference's outputs for clip 0 of the bench batch (tests/golden/pipe_c4.npz)."""
    g = golden("pipe_c4")
    cfg = synth.make_cfg(fp16=False, T=8, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 1}, image_size=(224, 224))
    sd = synth.base_net_state_dict()
    heads = [synth.head_state_dict(100 + i, cfg) for i in range(cfg.max_iter)]
    x = synth.make_clips(1, 32, 224, 224)
    tb = synth.make_proposals(1, 11, cfg.T, 224, 224)
    with torch.no_grad():
        cf = om.base_net(x, sd)
        hist, traj = om.inference(cfg, cf, None, heads, cfg.max_iter, [t.copy() for t in tb])
    ref = g["feat_sub_c0"]
    assert np.allclose(cf.numpy()[:, :, ::4], ref, rtol=1e-4, atol=1e-4 * np.abs(ref).max())
    for i, h in enumerate(hist):
        assert np.allclose(h["pred_prob"][:, 0].numpy(), g["prob%d_c0" % i], rtol=1e-4, atol=1e-5)
        loc = tubes.valid_tubes(h["pred_loc"].numpy().copy(), 224, 224)   # the reference's CPU aliasing (DESIGN.md section 5)
        assert np.allclose(loc, g["loc_valid%d_c0" % i], rtol=1e-4, atol=2e-3)
        assert np.allclose(h["pred_first_loc"].numpy(), g["first%d_c0" % i], rtol=1e-4, atol=2e-3)
        assert np.allclose(np.concatenate([t[0] for t in traj[i]], 0), g["traj%d_c0" % i], rtol=1e-4, atol=2e-3)
