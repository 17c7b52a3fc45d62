"""`select_samples()` -- the training-sample selection of train.py:291-310 on the device: for every refinement step
`train_select` (utils/utils.py:135-340, `select_proposals` at :342-423) and the two `flatten_tubes` calls after it.
`select_cls_samples()` -- the same for the classification pre-training stage (train_cls.py:260-297): `select_proposals`
with that stage's rows, one launch of the same kernel in its train_cls row mode.

The reference copies the history to the host at every step, ranks the candidates with numpy and Python sorts, draws
with `random.shuffle` and `np.random.choice`, and uploads the result.  Here one host-to-device copy carries the targets,
the step-1 proposals and the two generators' states (numpy's global RandomState and Python's `random`, both MT19937);
each step is one launch of step_select_step_f32 (select.cu), enqueued without a synchronisation; one device-to-host copy
brings back the rows of every step and clip and the advanced states, which are written back to the two generators.  The
draws are the reference's, in its order (step-major, then clip-major).

Two parity contracts, the ones README.md states: every `np.argsort(x)[::-1]` is a stable ascending argsort
reversed, which equals the reference whenever no tie decides a choice; and the softmax weights use the correctly rounded
float32(exp(float64(x))), where numpy's AVX-512 float32 exp can differ in the last bit.
"""
import ctypes
import random

import numpy as np
import torch

from . import _lib as L

SAMPLING = {"uniform": L.SAMPLING_UNIFORM, "random": L.SAMPLING_RANDOM, "softmax": L.SAMPLING_SOFTMAX}
SelectParams = L.step_select_params   # the struct's name before it was read from the header


def _ext_mode(cfg, i):
    """utils.py:283: the selected tubes of step i grow by one chunk on each side when NUM_CHUNKS grows by two."""
    if i - 1 in cfg.NUM_CHUNKS and cfg.NUM_CHUNKS[i] == cfg.NUM_CHUNKS[i - 1] + 2:
        if i == 1:
            raise ValueError("select_samples: NUM_CHUNKS[0] extends step 1, which has no history to extend from")
        return {"predict": L.EXT_PREDICT, "extrapolate": L.EXT_EXTRAPOLATE}.get(cfg.temporal_mode, L.EXT_MEAN)
    return L.EXT_NONE


def _check(cfg, targets, tubes):
    if len(targets) != len(tubes) or len(targets) == 0:
        raise ValueError("select_samples: %d target lists for %d proposal lists" % (len(targets), len(tubes)))
    for b, (g, t) in enumerate(zip(targets, tubes)):
        if np.asarray(g).shape[0] == 0:
            raise ValueError("select_samples: clip %d has no ground truth" % b)
        if np.asarray(t).shape[0] == 0:
            raise ValueError("select_samples: clip %d has no proposals" % b)
    if 0 < cfg.topk < cfg.num_classes:
        raise ValueError("select_samples: 0 < topk=%d < num_classes=%d keeps int(topk / num_classes) * 2 == 0 candidates "
                         "per class" % (cfg.topk, cfg.num_classes))
    if cfg.selection_sampling not in SAMPLING:
        raise ValueError("select_samples: selection_sampling %r is not one of %s" % (cfg.selection_sampling, tuple(SAMPLING)))
    if cfg.max_pos_num < 0 or cfg.neg_ratio < 0:
        raise ValueError("select_samples: max_pos_num and neg_ratio must be >= 0")


class _Blob:
    """Sections of one byte buffer, each 16-byte aligned, copied to the device in one transfer."""

    def __init__(self):
        self.parts, self.offsets, self.size = [], {}, 0

    def add(self, name, arr):
        arr = np.ascontiguousarray(arr)
        self.offsets[name] = self.size
        self.parts.append((self.size, arr))
        self.size += (arr.nbytes + 15) & ~15

    def pack(self):
        buf = np.zeros(max(self.size, 16), dtype=np.uint8)
        for o, a in self.parts:
            buf[o:o + a.nbytes] = a.reshape(-1).view(np.uint8)
        return buf


def _add_states(blob):
    """numpy's global RandomState, then Python's `random`, as the kernel's two MT19937 words ("mt"); returns the states
    for _restore_states."""
    np_state, py_state = np.random.get_state(), random.getstate()
    blob.add("mt", np.concatenate([np.asarray(np_state[1], np.uint32), [np.uint32(np_state[2])],
                                   np.asarray(py_state[1], np.uint32)]))
    return np_state, py_state


def _restore_states(words, np_state, py_state):
    """Leaves both generators where the kernel left its copies (words: the read-back "mt" section)."""
    np.random.set_state(("MT19937", words[:624].copy(), int(words[624]), np_state[3], np_state[4]))
    random.setstate((py_state[0], tuple(int(v) for v in words[L.SELECT_MT_WORDS:2 * L.SELECT_MT_WORDS]), py_state[2]))


def select_samples(cfg, history, targets, tubes):
    """Same result as train.py:291-310: for i in 1..cfg.max_iter, train_select(i, history[i-2], targets, tubes, cfg)
    followed by flatten_tubes of its targets and (with the frame index first) of its tubes.

    history: step_b200.inference(cfg, conv_feat, context_feat, nets, cfg.max_iter - 1, tubes)[0], on the device
    (pred_prob is read through its strides: the expand view inference returns, or any [R, L, C] tensor).
    targets / tubes: the loader's numpy lists, [n_gt_b, max_chunks, 4 + C] and [n_b, T_length_1, 4] per clip.
    Consumes numpy's global RandomState and Python's `random` as the reference does, and leaves them where it leaves them.
    Returns (step_tubes, step_targets): step_tubes[i-1] [R_i, T_length_i, 5] and step_targets[i-1] [R_i, 3, 6 + C], fp32
    on the device -- what training.train_step takes."""
    _check(cfg, targets, tubes)
    B, C, T = len(targets), cfg.num_classes, cfg.T
    n_steps = cfg.max_iter
    if len(history) < n_steps - 1:
        raise ValueError("select_samples: %d steps need %d history entries, got %d" % (n_steps, n_steps - 1, len(history)))
    max_chunks = cfg.NUM_CHUNKS[cfg.max_iter]
    tg = [np.asarray(g, dtype=np.float32) for g in targets]
    for b, g in enumerate(tg):
        if g.ndim != 3 or g.shape[1:] != (max_chunks, 4 + C):
            raise ValueError("select_samples: targets[%d] has shape %s, expected [n_gt, %d, %d]"
                             % (b, g.shape, max_chunks, 4 + C))
    props = [np.asarray(t) for t in tubes]
    prop_f64 = any(p.dtype == np.float64 for p in props)
    L1 = props[0].shape[1]
    for b, p in enumerate(props):
        if p.ndim != 3 or p.shape[1:] != (L1, 4):
            raise ValueError("select_samples: tubes[%d] has shape %s, expected [n, %d, 4]" % (b, p.shape, L1))
    nums = [p.shape[0] for p in props]
    ngt = [g.shape[0] for g in tg]
    for i, h in enumerate(history[:n_steps - 1]):
        if list(h["tubes_nums"]) != nums:
            raise ValueError("select_samples: history[%d] has tubes_nums %s for %s proposals" % (i, h["tubes_nums"], nums))
    max_rows = cfg.max_pos_num * (1 + cfg.neg_ratio)

    # every step's arguments, checked before anything is uploaded or launched
    steps, tensors = [], []
    for i in range(1, n_steps + 1):
        chunks = cfg.NUM_CHUNKS[i]
        T_start = int((max_chunks - chunks) / 2) * T
        T_length = chunks * T
        ext = _ext_mode(cfg, i)
        predict_nb = cfg.temporal_mode == "predict" and i < cfg.max_iter and cfg.NUM_CHUNKS[i + 1] == chunks + 2
        nb_first, nb_last = int((T_start - T) / T), int((T_start + T_length) / T)
        if predict_nb:   # utils.py:322-330 index the targets' chunks with these, Python's negative indices included
            if not (-max_chunks <= nb_first < max_chunks and -max_chunks <= nb_last < max_chunks):
                raise ValueError("select_samples: step %d's neighbour chunks %d / %d are outside the targets' %d chunks"
                                 % (i, nb_first, nb_last, max_chunks))
            nb_first, nb_last = nb_first % max_chunks, nb_last % max_chunks
        p = L.step_select_params(step=i, B=B, C=C, T=T, Lout=T_length, ext_mode=ext, max_chunks=max_chunks,
                                 gt_mid=int(max_chunks / 2), predict_nb=int(predict_nb), nb_first=nb_first, nb_last=nb_last,
                                 topk=cfg.topk, max_pos=cfg.max_pos_num, neg_ratio=cfg.neg_ratio,
                                 sampling=SAMPLING[cfg.selection_sampling], max_rows=max_rows, n_max=max(nums),
                                 g_max=max(ngt), prop_f64=int(prop_f64), cls_thresh=cfg.cls_thresh[i - 1],
                                 reg_thresh=cfg.reg_thresh[i - 1], width=float(cfg.image_size[0]),
                                 height=float(cfg.image_size[1]), L=L1)
        if i > 1:
            h = history[i - 2]
            prob, loc = h["pred_prob"], h["pred_loc"]
            R = sum(nums)
            ok = torch.is_tensor(prob) and torch.is_tensor(loc) and loc.dim() == 3 and loc.shape[0] == R and loc.shape[2] == 4
            ok = ok and prob.shape[0] == R and prob.shape[-1] == C and (prob.dim() == 2 or (prob.dim() == 3 and prob.shape[1] == loc.shape[1]))
            if not ok:
                raise ValueError("select_samples: history[%d] pred_prob %s / pred_loc %s for %d tubes and %d classes"
                                 % (i - 2, tuple(getattr(prob, "shape", ())), tuple(getattr(loc, "shape", ())), R, C))
            tensors += [prob, loc]
            p.L = loc.shape[1]
            if ext == L.EXT_PREDICT:
                for k in ("pred_first_loc", "pred_last_loc"):
                    v = h[k]
                    if not torch.is_tensor(v) or tuple(v.shape) != (R, T, 4):
                        raise ValueError("select_samples: history[%d] %s is %s, expected [%d, %d, 4]"
                                         % (i - 2, k, tuple(getattr(v, "shape", ())), R, T))
                    tensors.append(v)
        L.check(L.lib().step_select_check_f32(ctypes.byref(p)))
        steps.append(p)
    L.need_cuda(*tensors)
    dev = history[0]["pred_loc"].device if n_steps > 1 else torch.device("cuda", torch.cuda.current_device())

    blob = _Blob()
    np_state, py_state = _add_states(blob)
    blob.add("counts", np.zeros(n_steps * B, np.int32))
    blob.add("tube_off", np.concatenate([[0], np.cumsum(nums)]).astype(np.int32))
    blob.add("gt_off", np.concatenate([[0], np.cumsum(ngt)]).astype(np.int32))
    blob.add("targets", np.concatenate(tg))
    blob.add("props", np.concatenate([p.astype(np.float64) for p in props]))
    dbuf = torch.from_numpy(blob.pack()).to(dev)
    base = dbuf.data_ptr()
    at = lambda name: base + blob.offsets[name]
    head = blob.offsets["counts"] + 4 * n_steps * B          # the states and the counts: what comes back

    outs = []
    with torch.cuda.device(dev):
        stream = L.stream()
        for i, p in enumerate(steps, start=1):
            keep = []
            if i == 1:
                p.props = at("props")
            else:
                h = history[i - 2]
                prob, loc = h["pred_prob"], h["pred_loc"].float().contiguous()
                if prob.dim() == 2:
                    prob = prob.unsqueeze(1).expand(-1, loc.shape[1], -1)
                prob = prob.float()
                p.prob, p.loc = prob.data_ptr(), loc.data_ptr()
                p.prob_sr, p.prob_sl, p.prob_sc = prob.stride()
                keep += [prob, loc]
                if p.ext_mode == L.EXT_PREDICT:
                    first = h["pred_first_loc"].float().contiguous()
                    last = h["pred_last_loc"].float().contiguous()
                    p.first, p.last = first.data_ptr(), last.data_ptr()
                    keep += [first, last]
            rows = max(B * max_rows, 1)
            out_t = torch.empty((rows, p.Lout, 5), dtype=torch.float32, device=dev)
            out_g = torch.empty((rows, 3, 6 + C), dtype=torch.float32, device=dev)
            p.tube_off, p.gt_off, p.targets, p.mt = at("tube_off"), at("gt_off"), at("targets"), at("mt")
            p.out_tubes, p.out_targets = out_t.data_ptr(), out_g.data_ptr()
            p.counts = at("counts") + 4 * (i - 1) * B
            L.check(L.lib().step_select_step_f32(ctypes.byref(p), stream))
            outs.append((out_t, out_g, keep))
        back = dbuf[:head].cpu().numpy()                 # the one synchronisation
    words = back[:blob.offsets["counts"]].view(np.uint32)
    counts = back[blob.offsets["counts"]:head].view(np.int32).reshape(n_steps, B)
    _restore_states(words, np_state, py_state)
    step_tubes = [o[0][:int(c.sum())] for o, c in zip(outs, counts)]
    step_targets = [o[1][:int(c.sum())] for o, c in zip(outs, counts)]
    return step_tubes, step_targets


def select_cls_samples(targets, tubes, num_classes, cls_thresh=0.75, max_pos_num=5, sampling="uniform", neg_ratio=3):
    """Same result as train_cls.py:260-297: per clip select_proposals(targets[b][:, 0], tubes[b][:, T // 2], None,
    cls_thresh, max_pos_num, sampling, neg_ratio) with the stage's rows, then flatten_tubes of the targets and (with the
    frame index first) of the selected tubes.  The defaults are train_cls.py's literals.

    targets / tubes: the loader's numpy lists, [n_gt_b, chunks, 4 + C] (chunk 0 is read: the stage's max_chunks is 1) and
    [n_b, T, 4] per clip (float64, as its sample_anchors makes them, or float32).
    Rows: a positive carries its ground truth's box, classification flag 1 and labels; a negative classification flag 1
    only; the regression flag is 0, and the three target rows of a sample are the same.
    Consumes numpy's global RandomState and Python's `random` as the reference does, and leaves them where it leaves them.
    Returns (flat_tubes [R, T, 5], flat_targets [R, 3, 6 + C]), fp32 on the current CUDA device -- what
    training.train_step takes for the class-only heads."""
    if len(targets) != len(tubes) or len(targets) == 0:
        raise ValueError("select_cls_samples: %d target lists for %d proposal lists" % (len(targets), len(tubes)))
    for b, (g, t) in enumerate(zip(targets, tubes)):
        if np.asarray(g).shape[0] == 0:
            raise ValueError("select_cls_samples: clip %d has no ground truth" % b)
        if np.asarray(t).shape[0] == 0:
            raise ValueError("select_cls_samples: clip %d has no proposals" % b)
    if sampling not in SAMPLING:
        raise ValueError("select_cls_samples: sampling %r is not one of %s" % (sampling, tuple(SAMPLING)))
    if max_pos_num < 0 or neg_ratio < 0:
        raise ValueError("select_cls_samples: max_pos_num and neg_ratio must be >= 0")
    B, C = len(targets), int(num_classes)
    tg = [np.asarray(g, dtype=np.float32) for g in targets]
    chunks = tg[0].shape[1] if tg[0].ndim == 3 else 0
    for b, g in enumerate(tg):
        if g.ndim != 3 or g.shape[1] < 1 or g.shape[1:] != (chunks, 4 + C):
            raise ValueError("select_cls_samples: targets[%d] has shape %s, expected [n_gt, %d, %d]"
                             % (b, g.shape, max(chunks, 1), 4 + C))
    props = [np.asarray(t) for t in tubes]
    T = props[0].shape[1] if props[0].ndim == 3 else 0
    for b, p in enumerate(props):
        if p.ndim != 3 or T < 1 or p.shape[1:] != (T, 4):
            raise ValueError("select_cls_samples: tubes[%d] has shape %s, expected [n, %d, 4]" % (b, p.shape, max(T, 1)))
    nums, ngt = [p.shape[0] for p in props], [g.shape[0] for g in tg]
    max_rows = max_pos_num * (1 + neg_ratio)
    p = L.step_select_params(step=1, B=B, C=C, L=T, T=T, Lout=T, ext_mode=L.EXT_NONE, max_chunks=chunks, gt_mid=0,
                             max_pos=max_pos_num, neg_ratio=neg_ratio, sampling=SAMPLING[sampling], max_rows=max_rows,
                             n_max=max(nums), g_max=max(ngt), prop_f64=int(any(q.dtype == np.float64 for q in props)),
                             cls_thresh=float(cls_thresh), target_mode=L.TARGETS_CLS)
    L.check(L.lib().step_select_check_f32(ctypes.byref(p)))
    dev = torch.device("cuda", torch.cuda.current_device())

    blob = _Blob()
    np_state, py_state = _add_states(blob)
    blob.add("counts", np.zeros(B, np.int32))
    blob.add("tube_off", np.concatenate([[0], np.cumsum(nums)]).astype(np.int32))
    blob.add("gt_off", np.concatenate([[0], np.cumsum(ngt)]).astype(np.int32))
    blob.add("targets", np.concatenate(tg))
    blob.add("props", np.concatenate([q.astype(np.float64) for q in props]))
    dbuf = torch.from_numpy(blob.pack()).to(dev)
    at = lambda name: dbuf.data_ptr() + blob.offsets[name]
    head = blob.offsets["counts"] + 4 * B                    # the states and the counts: what comes back
    rows = max(B * max_rows, 1)
    out_t = torch.empty((rows, T, 5), dtype=torch.float32, device=dev)
    out_g = torch.empty((rows, 3, 6 + C), dtype=torch.float32, device=dev)
    p.tube_off, p.gt_off, p.targets, p.props, p.mt = at("tube_off"), at("gt_off"), at("targets"), at("props"), at("mt")
    p.out_tubes, p.out_targets, p.counts = out_t.data_ptr(), out_g.data_ptr(), at("counts")
    L.check(L.lib().step_select_step_f32(ctypes.byref(p), L.stream()))
    back = dbuf[:head].cpu().numpy()                         # the one synchronisation
    _restore_states(back[:blob.offsets["counts"]].view(np.uint32), np_state, py_state)
    R = int(back[blob.offsets["counts"]:head].view(np.int32).sum())
    return out_t[:R], out_g[:R]
