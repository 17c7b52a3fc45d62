"""Generates tests/golden/*.npz by running the UNMODIFIED reference (imported from /root/reference,
native ops compiled from its own sources by oracle/build_ref.py) on seeded synthetic inputs.
Only runnable in the build container; the fixtures it writes are committed.

    python tests/golden/make_golden.py
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refload  # noqa: E402
from step_b200 import synth  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
R = refload.load()
T = torch.from_numpy


def quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def gen_nms():
    rs = np.random.RandomState(7)
    cases = {}
    def add(name, b, s, thr):
        b = np.asarray(b, np.float32).reshape(-1, 4); s = np.asarray(s, np.float32)
        keep = R._C.nms(T(b), T(s), float(thr)).numpy()
        cases[name + "_boxes"] = b; cases[name + "_scores"] = s
        cases[name + "_thr"] = np.float32(thr); cases[name + "_keep"] = keep.astype(np.int64)
    add("iou_eq_thr", [[0, 0, 9, 9], [0, 0, 9, 4]], [.9, .8], 0.5)           # IoU == thr -> suppressed (>=)
    add("four", [[0, 0, 10, 10], [1, 1, 11, 11], [50, 50, 60, 60], [0, 0, 10, 10]], [.9, .8, .7, .95], 0.4)
    add("third", [[0, 0, 2, 0], [0, 0, 0, 0]], [.9, .8], 1.0 / 3.0)          # IoU = 1/3 vs float32(1/3)
    add("empty", np.zeros((0, 4)), np.zeros((0,)), 0.4)
    add("single", [[3, 4, 50, 60]], [.1], 0.4)
    for n in (63, 64, 65, 129, 1000):
        x1 = rs.uniform(0, 150, n); y1 = rs.uniform(0, 150, n)
        w = rs.uniform(20, 120, n); h = rs.uniform(20, 120, n)
        b = np.stack([x1, y1, np.minimum(x1 + w, 223), np.minimum(y1 + h, 223)], 1)
        s = rs.permutation(n).astype(np.float32) / n   # unique scores: torch.sort is not stable on ties
        add("rand%d" % n, b, s, 0.4)
    # integer-coordinate boxes produce many exact IoU ties at the threshold
    b = rs.randint(0, 40, (300, 2)); wh = rs.randint(1, 30, (300, 2))
    add("intgrid", np.concatenate([b, b + wh], 1), rs.permutation(300).astype(np.float32), 0.5)
    np.savez_compressed(os.path.join(OUT, "nms_cases.npz"), **cases)
    print("nms cases:", len(cases) // 4)


def gen_roi_align():
    rs = np.random.RandomState(11)
    K, C, H, W = 3, 5, 14, 14
    feat = rs.randn(K, C, H, W).astype(np.float32)
    rois = [
        [0, 10, 10, 10.5, 10.2],          # < 1 px after scaling: forced 1x1
        [1, -40, -40, 60, 60],            # partly outside (samples < -1 -> 0)
        [2, 100, 100, 400, 400],          # runs past the far edge
        [2, 0, 0, 223, 223],              # whole map, grid 2x2
        [0, 0, 0, 111, 55],               # non-integer bin, adaptive grid 1..
        [1, 30.3, 17.7, 199.1, 222.9],
        [2, 223, 223, 223, 223],          # last pixel
        [0, 5, 5, 5, 5],
    ]
    for _ in range(40):
        x1, y1 = rs.uniform(-30, 200, 2); w, h = rs.uniform(0, 220, 2)
        rois.append([rs.randint(0, K), x1, y1, x1 + w, y1 + h])
    rois = np.asarray(rois, np.float32)
    out = {"feat": feat, "rois": rois}
    for sr in (0, 2):
        out["out_sr%d" % sr] = R._C.roi_align_forward(T(feat), T(rois), 1.0 / 16.0, 7, 7, sr).numpy()
    out["out_3x5_s0p5"] = R._C.roi_align_forward(T(feat), T(rois * np.array([1, .1, .1, .1, .1], np.float32)),
                                                 0.5, 3, 5, 0).numpy()
    np.savez_compressed(os.path.join(OUT, "roi_align_cases.npz"), **out)
    print("roi_align rois:", rois.shape[0])


def gen_tubes():
    rs = np.random.RandomState(3)
    tu = R.tube_utils
    out = {}
    anchors = np.concatenate([rs.uniform(0, 150, (64, 2)), rs.uniform(150, 223, (64, 2))], 1).astype(np.float32)
    deltas = (rs.randn(64, 4) * np.array([.2, .2, .5, .5])).astype(np.float32)
    deltas[0, 2:] = [6.0, -6.0]; deltas[1, 2:] = [20.0, 0.0]   # large dw
    out["dec_anchors"], out["dec_deltas"] = anchors, deltas
    out["dec_out"] = tu.decode_coef(T(anchors), T(deltas)).numpy()
    gt = anchors + rs.uniform(-5, 5, anchors.shape).astype(np.float32)
    out["enc_gt"] = gt; out["enc_out"] = tu.encode_coef(T(gt), T(anchors)).numpy()
    tubes = (rs.uniform(-20, 260, (9, 4, 2))).astype(np.float32)
    tubes = np.concatenate([tubes, tubes + rs.uniform(-3, 120, (9, 4, 2)).astype(np.float32)], 2)
    tubes[0, 0] = [10, 10, 12, 40]; tubes[1, 1] = [50, 50, 40, 90]   # degenerate -> whole image
    out["val_in"] = tubes
    out["val_out_224"] = tu.valid_tubes(tubes.copy(), width=224, height=224)
    out["val_out_400"] = tu.valid_tubes(tubes.copy())
    for Tt in (2, 3, 4):
        t = tubes[:, :Tt].copy()
        out["ext_in_T%d" % Tt] = t
        out["ext_out_T%d" % Tt] = tu.extrapolate_tubes(t.copy(), Tt)
    lst = [tubes[:2].copy(), np.zeros((0, 4, 4), np.float32), tubes[2:5].copy()]
    flat, nums = tu.flatten_tubes(lst, batch_idx=True)
    out["flat_out"], out["flat_nums"] = flat, np.asarray(nums)
    out["extend_out"] = tu.extend_tubes(T(flat), 1.2, 224, 224).numpy()
    np.savez_compressed(os.path.join(OUT, "tubes_cases.npz"), **out)
    print("tubes ok")


def build_nets(cfg, n_heads, context=False):
    nets = {"base_net": quiet(R.models.BaseNet, cfg), "roi_net": R.models.ROINet(cfg.pool_mode, cfg.pool_size)}
    nets["base_net"].load_state_dict(synth.base_net_state_dict()); nets["base_net"].eval()
    for i in range(n_heads):
        h = quiet(R.models.TwoBranchNet, cfg)
        h.load_state_dict(synth.head_state_dict(100 + i, cfg), strict=True)
        h.eval(); h.set_device("cpu")
        nets["det_net%d" % i] = h
    if context:
        c = quiet(R.models.ContextNet, cfg)
        c.load_state_dict(synth.context_net_state_dict(), strict=True); c.eval()
        nets["context_net"] = c
    return nets


def run_pipeline(name, cfg, B, T_in, HW, N, context=False, store_feat=True):
    nets = build_nets(cfg, cfg.max_iter, context)
    x = synth.make_clips(B, T_in, HW, HW)
    tubes = synth.make_proposals(B, N, cfg.T * cfg.NUM_CHUNKS[1], HW, HW)
    out = {"B": B, "T_in": T_in, "HW": HW, "N": N}
    with torch.no_grad():
        cf = nets["base_net"](x)
        ctx = nets["context_net"](cf) if context else None
        # .clone(): on CPU the reference's valid_tubes mutates history['pred_loc'] in place through
        # the shared numpy view (utils.py:107-121); the GPU path (.cpu() copies) does not.  We
        # record the un-mutated GPU semantics by re-running decode below from the trajectory.
        hist, traj = R.utils.inference(cfg, cf, ctx, nets, cfg.max_iter, [t.copy() for t in tubes])
    if store_feat:
        out["conv_feat"] = cf.numpy()
    else:
        out["conv_feat_sub"] = cf.numpy()[:, ::4, ::13, ::6, ::6].copy()
    out["conv_feat_absmean"] = np.float64(cf.abs().double().mean().item())
    if context:
        out["context_feat"] = ctx.numpy()
    for i, h in enumerate(hist):
        out["prob%d" % i] = h["pred_prob"][:, 0].numpy().copy()
        out["loc_valid%d" % i] = h["pred_loc"].numpy().copy()     # == valid_tubes(pred_loc) (CPU aliasing)
        if h["pred_first_loc"] is not None:
            out["first%d" % i] = h["pred_first_loc"].numpy().copy()
            out["last%d" % i] = h["pred_last_loc"].numpy().copy()
        out["nums%d" % i] = np.asarray(h["tubes_nums"])
        out["traj%d" % i] = np.concatenate([t[0] for t in traj[i]], 0)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **out)
    print(name, "conv_feat", tuple(cf.shape), "absmean %.4f" % cf.abs().mean().item())


def gen_pipelines():
    # C1 (BASELINE.json configs[0]): 1 clip, T=8, 112x112, 1 proposal, max_iter=1
    run_pipeline("pipe_c1", synth.make_cfg(T=2, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(112, 112)),
                 B=1, T_in=8, HW=112, N=1)
    # spatial mode, 3 steps, 2 clips x 5 proposals, T'=4
    run_pipeline("pipe_spatial", synth.make_cfg(T=4, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 1}, image_size=(112, 112)),
                 B=2, T_in=16, HW=112, N=5)
    # temporal mode (tube extension 1 -> 3 chunks at step 3), T=3, T'=9.  The reference's slicing
    # (two_branch.py:265-270) only works for odd T when chunks > 1; its shipped config is T=3.
    for mode in ("predict", "extrapolate", "mean"):
        run_pipeline("pipe_temporal_" + mode,
                     synth.make_cfg(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, temporal_mode=mode,
                                    image_size=(112, 112)),
                     B=2, T_in=36, HW=112, N=4, store_feat=(mode == "predict"))
    # native AVA shape with ContextNet (only valid at 400x400, two_branch.py:127): 1 clip, 3 proposals
    run_pipeline("pipe_ava_context",
                 synth.make_cfg(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False,
                                image_size=(400, 400)),
                 B=1, T_in=36, HW=400, N=3, context=True, store_feat=False)


def gen_losses():
    """TwoBranchNet.forward(targets=...) of the reference (two_branch.py:276-341): the training-time outputs.
    Inputs are regenerated from the seed by synth.make_loss_case, so only the outputs are stored."""
    out = {}
    for name in synth.LOSS_CASES:
        T_, chunks, _, _ = synth.LOSS_CASES[name]
        cfg = synth.make_cfg(T=T_, max_iter=1, NUM_CHUNKS={1: chunks}, image_size=(112, 112))
        net = quiet(R.models.TwoBranchNet, cfg)
        net.load_state_dict(synth.head_state_dict(100, cfg), strict=True)
        net.eval(); net.set_device("cpu")
        _, _, feat, tubes, tg = synth.make_loss_case(name, cfg.num_classes)
        with torch.no_grad():
            prob, loc, first, last, lc, ll, ln = net(feat, None, tubes=tubes, targets=tg)
        for k, v in (("prob", prob), ("loc", loc), ("first", first), ("last", last), ("loss_cls", lc), ("loss_loc", ll),
                     ("loss_nb", ln), ("feat_checksum", feat.double().sum().view(1))):
            out["%s_%s" % (name, k)] = v.numpy()
        print("losses", name, tuple(lc.shape), float(ll), float(ln))
    np.savez_compressed(os.path.join(OUT, "losses_cases.npz"), **out)


def gen_head_grads():
    """Gradients of the head's training objective (train.py:323-347, train_step.sh:43-44: lambda_reg 5,
    lambda_neighbor 1) in the reference, eval-mode dropout so that the result is deterministic: the checker the
    round-2 dgrad / wgrad kernels will be held to.  Stores per-parameter gradient norms and leading values."""
    out = {}
    name = "c1"
    T_, chunks, _, _ = synth.LOSS_CASES[name]
    cfg = synth.make_cfg(T=T_, max_iter=1, NUM_CHUNKS={1: chunks}, image_size=(112, 112))
    net = quiet(R.models.TwoBranchNet, cfg)
    net.load_state_dict(synth.head_state_dict(100, cfg), strict=True)
    net.eval(); net.set_device("cpu")
    for p_ in net.parameters():
        p_.requires_grad_(True)
    _, _, feat, tubes, tg = synth.make_loss_case(name, cfg.num_classes)
    feat = feat.clone().requires_grad_(True)
    prob, loc, first, last, lc, ll, ln = net(feat, None, tubes=tubes, targets=tg)
    loss = lc.mean() + ll.mean() * 5.0 + ln.mean() * 1.0
    loss.backward()
    out["loss"] = loss.detach().numpy().reshape(1)
    out["feat_grad_norm"] = feat.grad.double().norm().numpy().reshape(1)
    out["feat_grad_head"] = feat.grad.reshape(-1)[:16].numpy().copy()
    for k, p_ in net.named_parameters():
        if p_.grad is None:
            continue
        out["gn:" + k] = p_.grad.double().norm().numpy().reshape(1)
        out["gh:" + k] = p_.grad.reshape(-1)[:8].numpy().copy()
    np.savez_compressed(os.path.join(OUT, "head_grads.npz"), **out)
    print("head grads:", float(loss), len([k for k in out if k.startswith("gn:")]), "parameters")


def gen_trunk_grads():
    """Backward of the I3D trunk (BatchNorm in eval, affine frozen as build_base_i3d does, networks.py:136-142) for
    a seeded clip and a seeded linear functional of conv_feat: per-parameter gradient norms -- the checker for the
    round-2 Unit3D dgrad / wgrad kernels."""
    cfg = synth.make_cfg(T=2, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(64, 64))
    net = quiet(R.models.BaseNet, cfg)
    net.load_state_dict(synth.base_net_state_dict()); net.eval()
    x = synth.make_clips(1, 8, 64, 64, seed=4321).requires_grad_(True)
    cf = net(x)
    proj = torch.randn(cf.shape, generator=torch.Generator().manual_seed(99))
    loss = (cf * proj).sum() / cf.numel()
    loss.backward()
    out = {"loss": loss.detach().numpy().reshape(1), "x_grad_norm": x.grad.double().norm().numpy().reshape(1),
           "x_grad_head": x.grad.reshape(-1)[:16].numpy().copy()}
    n = 0
    for k, p_ in net.named_parameters():
        if p_.grad is None:
            continue
        out["gn:" + k] = p_.grad.double().norm().numpy().reshape(1)
        out["gh:" + k] = p_.grad.reshape(-1)[:8].numpy().copy()
        n += 1
    np.savez_compressed(os.path.join(OUT, "trunk_grads.npz"), **out)
    print("trunk grads:", float(loss), n, "parameters with gradients")


def gen_c4():
    """BASELINE.json configs[3] (C4) at the measured shape: T_in=32, 224x224, 11 proposals, max_iter=3, spatial mode.
    The reference runs one clip at a time here (clips are independent units; BatchNorm is in eval mode): clips 0 and 7
    of the seeded 8-clip bench batch, i.e. the first and the last M tiles of every layer at B=8.  The GPU test runs the
    whole 8-clip batch, so every dispatch branch the benchmark takes is checked against these rows."""
    cfg = synth.make_cfg(T=8, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 1}, image_size=(224, 224))
    nets = build_nets(cfg, cfg.max_iter)
    xs = synth.make_clips(8, 32, 224, 224)
    tubes = synth.make_proposals(1, 11, cfg.T, 224, 224)
    out = {"clips": np.asarray([0, 7]), "B": 8, "T_in": 32, "HW": 224, "N": 11}
    for c in (0, 7):
        with torch.no_grad():
            cf = nets["base_net"](xs[c:c + 1].clone())
            hist, traj = R.utils.inference(cfg, cf, None, nets, cfg.max_iter, [t.copy() for t in tubes])
        out["feat_sub_c%d" % c] = cf.numpy()[:, :, ::4].copy()         # every 4th channel, all positions
        out["feat_absmax_c%d" % c] = np.float32(cf.abs().max().item())
        out["feat_absmean_c%d" % c] = np.float64(cf.abs().double().mean().item())
        for i, h in enumerate(hist):
            out["prob%d_c%d" % (i, c)] = h["pred_prob"][:, 0].numpy().copy()
            out["loc_valid%d_c%d" % (i, c)] = h["pred_loc"].numpy().copy()
            out["first%d_c%d" % (i, c)] = h["pred_first_loc"].numpy().copy()
            out["last%d_c%d" % (i, c)] = h["pred_last_loc"].numpy().copy()
            out["traj%d_c%d" % (i, c)] = np.concatenate([t[0] for t in traj[i]], 0)
        print("c4 clip", c, "feat absmax %.3f" % cf.abs().max().item())
    np.savez_compressed(os.path.join(OUT, "pipe_c4.npz"), **out)


def gen_c2():
    """BASELINE.json configs[1] (C2): I3D trunk only, batch 4, T=32, 224x224.  Reference output for clip 3 of the
    seeded 4-clip batch (the last M tiles at B=4), every 4th channel."""
    cfg = synth.make_cfg(T=8, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(224, 224))
    net = quiet(R.models.BaseNet, cfg)
    net.load_state_dict(synth.base_net_state_dict()); net.eval()
    xs = synth.make_clips(4, 32, 224, 224)
    out = {"B": 4, "T_in": 32, "HW": 224}
    for c in (0, 3):
        with torch.no_grad():
            cf = net(xs[c:c + 1].clone())
        out["feat_sub_c%d" % c] = cf.numpy()[:, :, ::4].copy()
        out["feat_absmax_c%d" % c] = np.float32(cf.abs().max().item())
        out["feat_absmean_c%d" % c] = np.float64(cf.abs().double().mean().item())
    np.savez_compressed(os.path.join(OUT, "trunk_c2.npz"), **out)
    print("c2 trunk ok")


def _reference_eval_loop_source():
    """The evaluation loop body of the reference's test.py (the `for i in range(len(history))` block,
    test.py:156-218), read from the file where it lies and dedented -- executed, never stored."""
    import textwrap
    lines = open(os.path.join(refload.REF, "test.py")).read().split("\n")
    start = next(i for i, l in enumerate(lines) if l.strip() == "for i in range(len(history)):")
    end = next(i for i in range(start, len(lines)) if lines[i].startswith("    fout.close()"))
    return textwrap.dedent("\n".join(lines[start:end]))


def run_reference_eval_loop(history, n_clips, num_classes, conf_thresh, nms_thresh, topk, width, height):
    """Executes the reference's own loop body on `history` (CPU tensors) and parses the rows it writes
    (test.py:211-218 format) back into per-step, per-clip lists of (box[4], class, score) -- in file order."""
    from types import SimpleNamespace
    bufs = [io.StringIO() for _ in history]
    env = {"history": history, "args": SimpleNamespace(num_classes=num_classes, conf_thresh=conf_thresh,
                                                       nms_thresh=nms_thresh, evaluate_topk=topk, topk=topk),
           "infos": [{"video_name": "clip%d" % b, "fid": b} for b in range(n_clips)], "fouts": bufs,
           "label_dict": list(range(num_classes)), "width": width, "height": height, "np": np, "torch": torch,
           "valid_tubes": R.tube_utils.valid_tubes, "nms": R.roi_layers.nms}
    exec(compile(_reference_eval_loop_source(), "reference test.py:156-218", "exec"), env)
    out = []
    for buf in bufs:
        per_clip = [[] for _ in range(n_clips)]
        for row in buf.getvalue().strip().split("\n"):
            if not row:
                continue
            f = row.split(",")
            per_clip[int(f[1])].append((np.asarray([float(v) for v in f[2:6]], np.float32), int(f[6]), float(f[7])))
        out.append(per_clip)
    return out


def gen_postprocess():
    """Detection post-processing (test.py:156-218) by the reference's own code, on (a) a synthetic history with
    heavy overlaps, ragged / empty clips and scores straddling conf_thresh, (b) the reference's own C4 outputs
    (pipe_c4.npz, clip 0 and 7 as a 2-clip batch).  The file rows carry 4 significant digits; the raw inputs are
    stored so the checker re-derives full-precision values and compares sets."""
    rs = np.random.RandomState(5)
    out = {}

    def case(name, prob, loc, nums, conf, thr, topk, width, height):
        T_ = loc.shape[1]
        hist = [{"pred_prob": T(prob[:, None, :].repeat(T_, 1).copy()), "pred_loc": T(loc.copy()), "tubes_nums": list(nums)}]
        dets = run_reference_eval_loop(hist, len(nums), prob.shape[1], conf, thr, topk, width, height)[0]
        out[name + "_prob"], out[name + "_loc"], out[name + "_nums"] = prob, loc, np.asarray(nums)
        out[name + "_cfg"] = np.asarray([conf, thr, topk, width, height], np.float64)
        rows = [(b, c, s) + tuple(bx) for b, d in enumerate(dets) for (bx, c, s) in d]
        out[name + "_rows"] = np.asarray(rows, np.float64).reshape(-1, 7)
        print("postprocess", name, "detections per clip:", [len(d) for d in dets])

    nums = [6, 0, 9, 3]
    n = sum(nums)
    ctr = rs.uniform(40, 180, (n, 1, 2)); wh = rs.uniform(20, 90, (n, 1, 2))
    jit = rs.uniform(-6, 6, (n, 4, 4))
    loc = (np.concatenate([ctr - wh / 2, ctr + wh / 2], 2) + jit).astype(np.float32)
    loc[2] = loc[3] + 1.0          # near-duplicates -> suppressed
    loc[7, :, 2] = loc[7, :, 0] + 1.0   # degenerate -> valid_tubes replaces it by the 400x400 default box
    prob = rs.uniform(0, 1, (n, 12)).astype(np.float32) ** 3
    prob[:, 5] = 0.0
    prob[4, 3] = np.float32(0.2)   # == conf_thresh: not strictly greater -> dropped
    case("synth", prob, loc, nums, 0.2, 0.4, 0, 224, 224)
    case("synth_topk", prob, loc, nums, 0.05, 0.5, 5, 224, 224)
    g = np.load(os.path.join(OUT, "pipe_c4.npz"))
    prob = np.concatenate([g["prob2_c0"], g["prob2_c7"]], 0)
    loc = np.concatenate([g["loc_valid2_c0"], g["loc_valid2_c7"]], 0)
    # threshold in the middle of the widest score gap of the upper half, so that fp16-vs-fp32 score noise
    # (<= 5e-3) cannot move a candidate across it: the detection SET is then a meaningful fp16-vs-fp32 comparison
    sp = np.sort(prob.reshape(-1))
    band = sp[int(0.50 * sp.size):int(0.95 * sp.size)]
    k = int(np.argmax(np.diff(band)))
    conf = float(np.float32(0.5 * (band[k] + band[k + 1])))
    print("c4 conf_thresh %.5f (gap %.4f)" % (conf, band[k + 1] - band[k]))
    case("c4", prob, loc, [11, 11], conf, 0.4, 0, 224, 224)
    np.savez_compressed(os.path.join(OUT, "postprocess_cases.npz"), **out)


def gen_detect_edges():
    """Detection post-processing by the reference's own loop (test.py:156-218) where the order of the rows matters: scores
    on five levels, so that exact ties fall across classes and within a class, at and away from the top-k cut; the lowest
    level equal to conf_thresh (not strictly greater: dropped); a degenerate box in two clips (valid_tubes replaces it by
    the 400x400 default box); an empty clip.  Boxes of a clip lie in distinct grid cells, so that no NMS decision depends
    on how torch.sort orders tied scores, except one near-duplicate pair with distinct scores (suppressed).  Rows carry 4
    significant digits; the boxes differ at that precision, so the row order identifies the tubes."""
    rs = np.random.RandomState(13)
    out = {}
    nums, ncls, T_ = [10, 0, 7, 1], 6, 3
    n = sum(nums)
    cell = np.concatenate([np.arange(nums[0]), np.arange(nums[2]), np.arange(nums[3])])
    x1 = (cell % 5) * 44.0 + rs.uniform(0, 4, n)
    y1 = (cell // 5) * 44.0 + rs.uniform(0, 4, n)
    box = np.stack([x1, y1, x1 + rs.uniform(30, 38, n), y1 + rs.uniform(30, 38, n)], 1)
    loc = (box[:, None, :] + rs.uniform(-3, 3, (n, T_, 4))).astype(np.float32)
    loc[:, T_ // 2] = box
    loc[4, :, 2] = loc[4, :, 0] + 1.0              # degenerate (clip 0)
    loc[12, :, 3] = loc[12, :, 1]                  # degenerate (clip 2)
    loc[1] = loc[0] + 1.0                          # near-duplicate of tube 0
    levels = np.float32([0.2, 0.25, 0.5, 0.75, 0.875])
    prob = levels[rs.randint(0, 5, (n, ncls))]
    prob[1] = prob[0] * np.float32(0.75)          # distinct from tube 0's scores in every class
    for name, topk in (("ties", 0), ("ties_topk", 7), ("ties_topk_all", 100)):
        hist = [{"pred_prob": T(prob[:, None, :].repeat(T_, 1).copy()), "pred_loc": T(loc.copy()), "tubes_nums": list(nums)}]
        dets = run_reference_eval_loop(hist, len(nums), ncls, 0.2, 0.4, topk, 224, 224)[0]
        out[name + "_prob"], out[name + "_loc"], out[name + "_nums"] = prob, loc, np.asarray(nums)
        out[name + "_cfg"] = np.asarray([0.2, 0.4, topk, 224, 224], np.float64)
        rows = [(b, c, s) + tuple(bx) for b, d in enumerate(dets) for (bx, c, s) in d]
        out[name + "_rows"] = np.asarray(rows, np.float64).reshape(-1, 7)
        print("detect edges", name, "detections per clip:", [len(d) for d in dets])
    np.savez_compressed(os.path.join(OUT, "detect_edge_cases.npz"), **out)


def gen_roi_cross():
    """ROIPool forward/backward and ROIAlign backward have no CPU implementation in the reference
    (csrc/ROIPool.h:47, ROIAlign.h:66 raise on CPU tensors) -> cross-checked against torchvision 0.26's CPU ops,
    which descend from the same Caffe2 / maskrcnn-benchmark kernels (roi_align(aligned=False) is bit-identical to
    the reference's forward, SURVEY.md Appendix A).  A second independent implementation, not the reference."""
    import torchvision
    from torchvision.ops import roi_align as tv_align, roi_pool as tv_pool
    g = np.load(os.path.join(OUT, "roi_align_cases.npz"))
    feat, rois = T(g["feat"]), T(g["rois"])
    out = {"torchvision": np.asarray([int(v) for v in torchvision.__version__.split("+")[0].split(".")[:2]])}
    gen = torch.Generator().manual_seed(21)
    for sr in (0, 2):
        x = feat.clone().requires_grad_(True)
        y = tv_align(x, rois, (7, 7), 1.0 / 16.0, sr, aligned=False)
        assert torch.equal(y.detach(), T(g["out_sr%d" % sr])), "torchvision roi_align != reference forward"
        gy = torch.randn(y.shape, generator=gen)
        y.backward(gy)
        out["align_gy_sr%d" % sr] = gy.numpy(); out["align_gx_sr%d" % sr] = x.grad.numpy().copy()
    x = feat.clone().requires_grad_(True)
    y = tv_pool(x, rois, (7, 7), 1.0 / 16.0)
    gy = torch.randn(y.shape, generator=gen)
    y.backward(gy)
    out["pool_out"] = y.detach().numpy(); out["pool_gy"] = gy.numpy(); out["pool_gx"] = x.grad.numpy().copy()
    np.savez_compressed(os.path.join(OUT, "roi_cross_cases.npz"), **out)
    print("roi cross-check cases ok")


if __name__ == "__main__":
    which = sys.argv[1:] or ["nms", "roi_align", "tubes", "pipelines", "losses", "head_grads", "trunk_grads", "c4", "c2",
                             "postprocess", "detect_edges", "roi_cross"]
    for w_ in which:
        {"nms": gen_nms, "roi_align": gen_roi_align, "tubes": gen_tubes, "pipelines": gen_pipelines, "losses": gen_losses,
         "head_grads": gen_head_grads, "trunk_grads": gen_trunk_grads, "c4": gen_c4, "c2": gen_c2,
         "postprocess": gen_postprocess, "detect_edges": gen_detect_edges, "roi_cross": gen_roi_cross}[w_]()
