"""Generates tests/golden/select_cases.npz by running the reference's own `train_select` (utils/utils.py:135-340, imported
unmodified through oracle/refload) for every refinement step, each followed by the two `flatten_tubes` calls of
train.py:307-310, on seeded histories, targets and proposals.  Only runnable where the reference checkout exists; the
fixture it writes is committed.

    python tests/golden/make_select_golden.py

Each step's per-clip lists are flattened as train.py:307-310 does (oracle/select.py's `_flat`, flatten_tubes with one
convention added): when every clip of a step selects no row -- the `empty_rows` case, max_pos_num=0 -- the reference's
flatten_tubes raises in np.concatenate, and the fixture records zero rows instead, the result select_samples returns.

A seed is kept only when oracle/select.py gives the reference's result under the same generator states: that rejects the
seeds whose result depends on a tie (numpy's argsort orders equal values its own way) or on numpy's float32 exp, which
is not correctly rounded on its AVX-512 path (oracle/select.py states both contracts).

Per case <name>: <name>_cfg (JSON of the cfg fields), <name>_prob<i> / _loc<i> / _first<i> / _last<i> (history[i]:
pred_prob [R, C] before the expand to [R, L, C], pred_loc [R, L, 4], first / last [R, T, 4] in predict mode),
<name>_nums (tubes per clip), <name>_ngt (ground truths per clip), <name>_targets (the clips' targets concatenated,
float32 [sum G, max_chunks, 4 + C]), <name>_props (proposals concatenated, float64 [sum n, L_1, 4]), <name>_np_key /
_np_pos / _py_state (numpy's and Python's generator states before the call), <name>_tubes<i> / <name>_targets_out<i>
(the flat outputs of step i + 1) and <name>_np_key_after / _np_pos_after / _py_state_after.
"""
import json
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refload  # noqa: E402
from oracle import select as osel  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "select_cases.npz")

# scripts/train_step.sh: T=3, NUM_CHUNKS {1:1, 2:1, 3:3, 4:3}, max_iter 3, predict mode, topk 300, 60 classes
SHIPPED = dict(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3, 4: 3}, cls_thresh=[0.2, 0.35, 0.5], reg_thresh=[0.2, 0.35, 0.5],
               num_classes=60, topk=300, temporal_mode="predict", image_size=[400, 400], max_pos_num=5,
               selection_sampling="softmax", neg_ratio=2)


def make_cfg(**kw):
    d = dict(SHIPPED)
    d.update(kw)
    return SimpleNamespace(**d)


def cfg_json(cfg):
    d = dict(vars(cfg))
    d["NUM_CHUNKS"] = {str(k): v for k, v in d["NUM_CHUNKS"].items()}
    return json.dumps(d, sort_keys=True)


def make_inputs(cfg, rs, nums, ngt, zero_gt=False):
    """Ground truths, float64 proposals around them (tiled over the first step's frames) and a history whose boxes
    jitter around the proposals, so that every IoU range occurs."""
    W, H = cfg.image_size
    C, T = cfg.num_classes, cfg.T
    mc = cfg.NUM_CHUNKS[cfg.max_iter]
    targets, props = [], []
    for n, g in zip(nums, ngt):
        x1 = rs.uniform(0, 0.6 * W, (g, 1)); y1 = rs.uniform(0, 0.6 * H, (g, 1))
        w = rs.uniform(0.15 * W, 0.4 * W, (g, 1)); h = rs.uniform(0.15 * H, 0.4 * H, (g, 1))
        box = np.concatenate([x1, y1, x1 + w, y1 + h], 1)
        tg = np.zeros((g, mc, 4 + C), np.float32)
        tg[:, :, :4] = box[:, None] + rs.uniform(-4, 4, (g, mc, 4))
        tg[:, :, 4:] = rs.uniform(0, 1, (g, mc, C)) > 0.9
        tg[:, rs.randint(0, mc), :4] *= rs.randint(0, 2)     # a chunk without the person, sometimes
        if zero_gt:
            tg[0, int(mc / 2), :4] = 0
        targets.append(tg)
        src = box[rs.randint(0, g, n)] + rs.normal(0, 0.12 * W, (n, 4))
        src[:, 2:] = np.maximum(src[:, 2:], src[:, :2] + 8)
        props.append(np.tile(src[:, None], (1, cfg.NUM_CHUNKS[1] * T, 1)))
    R = sum(nums)
    flat = np.concatenate(props).astype(np.float32)
    history = []
    for i in range(1, cfg.max_iter):
        L = cfg.NUM_CHUNKS[i] * T
        base = np.concatenate([flat[:, :1]] * (L // flat.shape[1] + 1), 1)[:, :L] if flat.shape[1] < L else flat[:, :L]
        loc = (base + rs.normal(0, 6, (R, L, 4))).astype(np.float32)
        h = {"pred_prob": rs.uniform(0, 1, (R, C)).astype(np.float32), "pred_loc": loc, "tubes_nums": list(nums)}
        if cfg.temporal_mode == "predict":
            h["pred_first_loc"] = (loc[:, :T] + rs.normal(0, 6, (R, T, 4))).astype(np.float32)
            h["pred_last_loc"] = (loc[:, -T:] + rs.normal(0, 6, (R, T, 4))).astype(np.float32)
        history.append(h)
        nxt = L + 2 * T if cfg.NUM_CHUNKS.get(i + 1) == cfg.NUM_CHUNKS[i] + 2 else L
        flat = np.concatenate([loc[:, :1]] * nxt, 1) if nxt != L else loc
    return targets, props, history


def torch_history(cfg, history):
    """The history as step_b200.inference hands it over, on the CPU: pred_prob an expand view of [R, C]."""
    out = []
    for i, h in enumerate(history):
        L = h["pred_loc"].shape[1]
        d = {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in h.items()}
        d["pred_prob"] = d["pred_prob"].view(-1, 1, cfg.num_classes).expand(-1, L, -1)
        d.setdefault("pred_first_loc", None); d.setdefault("pred_last_loc", None)
        out.append(d)
    return out


def run_reference(ref, cfg, history, targets, props):
    th = torch_history(cfg, history)
    tubes = [p.copy() for p in props]
    outs = []
    for i in range(1, cfg.max_iter + 1):
        st, sg = ref.utils.train_select(i, th[i - 2] if i > 1 else None, targets, tubes, cfg)
        outs.append((osel._flat([np.asarray(s, np.float32) for s in st], True),
                     osel._flat([np.asarray(s, np.float32) for s in sg], False)))
    return outs


def run_oracle(cfg, history, targets, props):
    hist = [dict(h, pred_prob=np.broadcast_to(h["pred_prob"][:, None], (h["pred_prob"].shape[0], h["pred_loc"].shape[1],
                                                                         cfg.num_classes))) for h in history]
    st, sg = osel.select_samples(cfg, hist, targets, [p.copy() for p in props])
    return list(zip(st, sg))


def same(a, b):
    return all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(a, b))


def find_case(ref, cfg, nums, ngt, seed0, zero_gt=False, want=None):
    for seed in range(seed0, seed0 + 200):
        rs = np.random.RandomState(seed)
        targets, props, history = make_inputs(cfg, rs, nums, ngt, zero_gt)
        np.random.seed(seed + 7); random.seed(seed + 11)
        np_before, py_before = np.random.get_state(), random.getstate()
        out = run_reference(ref, cfg, history, targets, props)
        np_after, py_after = np.random.get_state(), random.getstate()
        np.random.set_state(np_before); random.setstate(py_before)
        mine = run_oracle(cfg, history, targets, props)
        if not same(out, mine) or random.getstate() != py_after or not np.array_equal(np.random.get_state()[1], np_after[1]):
            print("  seed %d rejected" % seed)
            continue
        if want is not None and not want(out, py_before, py_after):
            continue
        return seed, targets, props, history, out, (np_before, py_before), (np_after, py_after)
    raise RuntimeError("no seed found")


def main():
    assert refload.available(), "reference checkout not present"
    ref = refload.load()
    spatial = dict(NUM_CHUNKS={1: 1, 2: 1, 3: 1}, temporal_mode="extrapolate")
    cases = [  # name, cfg, proposals per clip, ground truths per clip, zero gt box, extra condition
        ("shipped_b2", make_cfg(), [34, 34], [3, 3], False, None),
        ("shipped_b8", make_cfg(), [34] * 8, [3] * 8, False, None),
        ("spatial_extrapolate_uniform", make_cfg(**spatial, selection_sampling="uniform"), [20, 26], [2, 3], False, None),
        ("mean_tubes", make_cfg(temporal_mode="mean"), [30, 18], [3, 2], False, None),
        ("extrapolate_temporal", make_cfg(temporal_mode="extrapolate"), [24, 24], [2, 4], False, None),
        ("random_sampling", make_cfg(selection_sampling="random"), [34, 28], [3, 2], False, None),
        ("topk_all", make_cfg(topk=-1, num_classes=12), [22, 30], [2, 3], False, None),
        ("many_gt_shuffle", make_cfg(), [34, 34], [8, 2], False, lambda o, a, b: a != b),
        ("few_negatives", make_cfg(), [6, 34], [3, 3], False, None),
        ("zero_gt_box", make_cfg(), [34, 20], [3, 2], True, None),
        ("empty_rows", make_cfg(max_pos_num=0), [12, 10], [3, 1], False, None),
    ]
    rec = {"numpy_version": np.array(np.__version__), "torch_version": np.array(torch.__version__),
           "cases": np.array([c[0] for c in cases])}
    for k, (name, cfg, nums, ngt, zero_gt, want) in enumerate(cases):
        seed, targets, props, history, out, before, after = find_case(ref, cfg, nums, ngt, 100 * k, zero_gt, want)
        rec[name + "_cfg"] = np.array(cfg_json(cfg))
        rec[name + "_nums"] = np.array(nums); rec[name + "_ngt"] = np.array(ngt)
        rec[name + "_targets"] = np.concatenate(targets); rec[name + "_props"] = np.concatenate(props)
        for i, h in enumerate(history):
            rec["%s_prob%d" % (name, i)] = h["pred_prob"]; rec["%s_loc%d" % (name, i)] = h["pred_loc"]
            if "pred_first_loc" in h:
                rec["%s_first%d" % (name, i)] = h["pred_first_loc"]; rec["%s_last%d" % (name, i)] = h["pred_last_loc"]
        for i, (t, g) in enumerate(out):
            rec["%s_tubes%d" % (name, i)] = t; rec["%s_targets_out%d" % (name, i)] = g
        for tag, (np_state, py_state) in (("", before), ("_after", after)):
            rec[name + "_np_key" + tag] = np_state[1]; rec[name + "_np_pos" + tag] = np.array(np_state[2])
            rec[name + "_py_state" + tag] = np.array(py_state[1], dtype=np.int64)
        print("%-28s seed %d rows %s" % (name, seed, [t.shape[0] for t, _ in out]))
    np.savez_compressed(OUT, **rec)
    print("wrote %s (%.2f MB)" % (OUT, os.path.getsize(OUT) / 1e6))


if __name__ == "__main__":
    main()
