"""Device implementation of the reference's tube arithmetic (utils/tube_utils.py) with the same
function names and argument meaning: `get_center_size`, `decode_coef`, `encode_coef`,
`extrapolate_tubes`, `valid_tubes`, `flatten_tubes`, `extend_tubes`.

CUDA tensors are processed in place on their device.  numpy arrays (what the reference drivers pass,
e.g. test.py:191, utils/utils.py:112,121) are staged through the current CUDA device and handed
back as numpy, preserving `valid_tubes`' in-place mutation (tube_utils.py:70-90).  The fused
per-step kernel used by `step_b200.inference` is `tube_update`.
"""
import numpy as np
import torch

from . import _lib as L


def _dev():
    if not torch.cuda.is_available():
        raise RuntimeError("step_b200.tube_utils: no CUDA device (there is no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _to_dev(a):
    if isinstance(a, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(_dev())
    L.need_cuda(a)
    return a.detach().to(torch.float32).contiguous()


def get_center_size(boxes):
    """tube_utils.py:127-141 (pure tensor expression; kept for API completeness)."""
    w = boxes[:, 2] - boxes[:, 0] + 1.0
    h = boxes[:, 3] - boxes[:, 1] + 1.0
    return boxes[:, 0] + 0.5 * w, boxes[:, 1] + 0.5 * h, w, h


def decode_coef(anchors, deltas):
    """tube_utils.py:165-189: [n,4] anchors + [n,4] deltas -> [n,4] boxes."""
    a, d = _to_dev(anchors), _to_dev(deltas)
    if a.shape != d.shape or a.dim() != 2 or a.shape[1] != 4:
        raise RuntimeError("decode_coef: expected two [n,4] tensors")
    out = torch.empty_like(d)
    L.check(L.lib().step_tube_decode_f32(L.ptr(a), 4, L.ptr(d), a.shape[0], L.ptr(out), L.stream()))
    return out


def encode_coef(gt_tubes, tubes):
    """tube_utils.py:143-163."""
    g, t = _to_dev(gt_tubes), _to_dev(tubes)
    out = torch.empty_like(g)
    L.check(L.lib().step_tube_encode_f32(L.ptr(g), L.ptr(t), 4, g.shape[0], L.ptr(out), L.stream()))
    return out


def valid_tubes(tubes, width=400, height=400):
    """tube_utils.py:59-92: clamp to the image, degenerate boxes -> whole image; mutates its input."""
    is_np = isinstance(tubes, np.ndarray)
    t = _to_dev(tubes)
    n = t.numel() // 4
    L.check(L.lib().step_tube_valid_f32(L.ptr(t), n, float(width), float(height), L.stream()))
    if is_np:
        res = t.cpu().numpy().reshape(tubes.shape)
        tubes[...] = res  # the reference mutates the caller's array through a reshape view
        return tubes
    if t.data_ptr() != tubes.data_ptr():
        tubes.copy_(t.view_as(tubes))
    return tubes


def extrapolate_tubes(tubes, T=6, height=400, width=400):
    """tube_utils.py:10-27: [n,L,4] -> [n,L+2T,4].  T = 1 raises ZeroDivisionError, as the reference's T/(T-1) does."""
    if T == 1:
        raise ZeroDivisionError("extrapolate_tubes: T/(T-1) with T = 1")
    is_np = isinstance(tubes, np.ndarray)
    t = _to_dev(tubes)
    n, Lf, _ = t.shape
    out = torch.empty((n, Lf + 2 * T, 4), dtype=torch.float32, device=t.device)
    L.check(L.lib().step_tube_extrapolate_f32(L.ptr(t), n, Lf, int(T), float(width), float(height), L.ptr(out),
                                              L.stream()))
    return out.cpu().numpy() if is_np else out


def extend_tubes(tubes, ratio=1.2, width=400, height=400):
    """tube_utils.py:248-266: tubes [-1,T,5] (frame index first)."""
    t = _to_dev(tubes)
    out = torch.empty_like(t)
    L.check(L.lib().step_tube_extend_f32(L.ptr(t), t.numel() // 5, float(ratio), float(width), float(height),
                                         L.ptr(out), L.stream()))
    return out


def flatten_tubes(tubes, batch_idx=False):
    """tube_utils.py:214-246 -- host-side list bookkeeping only (no arithmetic): returns
    (flat [sum n_i, T, dim(+1)], tubes_nums)."""
    _, T, dim = tubes[0].shape
    flat, nums = [], []
    for i, t in enumerate(tubes):
        nums.append(t.shape[0])
        if t.shape[0] == 0:
            continue
        t = np.asarray(t)
        if batch_idx:
            idx = np.tile((np.arange(T) + i * T).reshape(1, T, 1), (t.shape[0], 1, 1)).astype(t.dtype)
            flat.append(np.concatenate((idx, t), axis=2))
        else:
            flat.append(t.copy())
    return np.concatenate(flat, axis=0), nums


def tube_update(flat_in, loc, first, last, clip_of_tube, T, decode_neighbors, ext_mode, width, height):
    """The fused between-steps kernel (utils/utils.py:61-129): returns
    (pred_loc, pred_first, pred_last, flat_out)."""
    R, Lf, _ = flat_in.shape
    dev = flat_in.device
    pred_loc = torch.empty((R, Lf, 4), dtype=torch.float32, device=dev)
    pf = torch.empty((R, T, 4), dtype=torch.float32, device=dev) if decode_neighbors else None
    pl = torch.empty((R, T, 4), dtype=torch.float32, device=dev) if decode_neighbors else None
    L_out = Lf + 2 * T if ext_mode != L.EXT_NONE else Lf
    flat_out = torch.empty((R, L_out, 5), dtype=torch.float32, device=dev)
    L.check(L.lib().step_tube_update_f32(L.ptr(flat_in), L.ptr(loc), L.ptr(first), L.ptr(last), L.ptr(clip_of_tube),
                                         R, Lf, int(T), 1 if decode_neighbors else 0, int(ext_mode), float(width),
                                         float(height), L.ptr(pred_loc), L.ptr(pf), L.ptr(pl), L.ptr(flat_out),
                                         L.stream()))
    return pred_loc, pf, pl, flat_out
