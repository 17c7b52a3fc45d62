"""The reference's input transform on the device: `BaseTransform` (data/augmentations.py:601-615) from uint8 frames.

The reference builds every clip on the host, in DataLoader workers: ConvertFromInts(scale), cv2.resize (INTER_LINEAR) on the
float frames, SubtractMeans, DivideStds, then the dataset's BGR->RGB swap and permute to [T, 3, H, W]
(data/ava.py:328-338, data/customize.py:122-127).  Here the workers pass the uint8 frames through unchanged and the main
process turns the collated batch into the fp32 clip [B, T, 3, H, W] with one kernel launch (step_frames_to_clip_u8),
bit-identical to cv2's generic (non-IPP) resize:

    transform = BaseTransform((400, 400), scale=2)                 # the reference's constructor, size = (width, height)
    dataset = CustomizedDataset(..., transform=transform)          # host stage: the identity on the uint8 frames
    loader = DataLoader(dataset, collate_fn=keep_frames(detection_collate), pin_memory=True, ...)
    for images, tubes, infos in loader:
        images = transform.apply(images)                           # device stage: fp32 CUDA clip [B, T, 3, 400, 400]
"""
import ctypes

import numpy as np
import torch

from . import _lib as L

# The kernel stages the source columns of a 128-column output tile in shared memory: W0 <= 48 W always fits.
MAX_WIDTH_RATIO = 48


def frame_entry(clip, W):
    """The step_frame_src entry of one clip: a uint8 CUDA tensor [T, 3, H0, W0] with any strides (a view of a stacked batch,
    a permuted HWC frame array, ...), for an output width W."""
    L.need_cuda(clip)
    if clip.dtype != torch.uint8 or clip.dim() != 4 or clip.shape[1] != 3:
        raise ValueError("step_b200: expected uint8 frames [T, 3, H0, W0], got %s %s" % (clip.dtype, tuple(clip.shape)))
    T, _, H0, W0 = clip.shape
    if T < 1 or H0 < 1 or W0 < 1:
        raise ValueError("step_b200: empty source clip %s" % (tuple(clip.shape),))
    if W0 > MAX_WIDTH_RATIO * W:
        raise ValueError("step_b200: source width %d exceeds %d x the output width %d" % (W0, MAX_WIDTH_RATIO, W))
    st = clip.stride()
    return L.FrameSrc(clip.data_ptr(), H0, W0, st[0], st[1], st[2], st[3])


def frame_table(entries, device):
    """Uploads step_frame_src entries (one per clip) to `device` on the current stream; the returned tensor is the kernel's
    `table`.  The host copy is pinned, so the upload does not wait for the stream (torch keeps the pinned block until the
    copy has run)."""
    arr = bytes((L.FrameSrc * len(entries))(*entries))
    host = torch.empty(len(arr), dtype=torch.uint8, pin_memory=True)
    host.numpy()[:] = np.frombuffer(arr, dtype=np.uint8)
    return host.to(device, non_blocking=True)


class BaseTransform:
    """The reference's BaseTransform(size, mean, stds, scale), with `size = (width, height)` and `mean` / `stds` in the
    source's BGR order as there.  `__call__` is the host stage, `apply` the device stage."""

    def __init__(self, size=(400, 320), mean=(0, 0, 0), stds=(1, 1, 1), scale=1):
        if scale not in (0, 1, 2):
            raise ValueError("step_b200: BaseTransform scale must be 0, 1 or 2, got %r" % (scale,))
        self.size = (int(size[0]), int(size[1]))
        self.mean = np.array(mean, dtype=np.float32)
        self.stds = np.array(stds, dtype=np.float32)
        if self.mean.shape != (3,) or self.stds.shape != (3,):
            raise ValueError("step_b200: BaseTransform takes 3 means and 3 stds")
        self.scale = scale
        # the reference subtracts in BGR order before its dataset swaps to RGB: output channel c uses mean[2 - c]
        self._mean_rgb = (ctypes.c_float * 3)(*self.mean[::-1].tolist())
        self._std_rgb = (ctypes.c_float * 3)(*self.stds[::-1].tolist())

    def __call__(self, images, tubes=None, proposals=None):
        """Host stage (the DataLoader workers): the frames stay uint8, so the arguments are returned unchanged."""
        return images, tubes, proposals

    def launch(self, table, B, T, out):
        """Enqueues the kernel on the current stream: B clips of T frames described by `table` (frame_table) into `out`,
        a contiguous fp32 CUDA tensor [B, T, 3, H, W]."""
        W, H = self.size
        if out.dtype != torch.float32 or not out.is_contiguous() or tuple(out.shape) != (B, T, 3, H, W):
            raise ValueError("step_b200: out must be contiguous fp32 %s, got %s %s" % ((B, T, 3, H, W), out.dtype,
                                                                                         tuple(out.shape)))
        dev = L.same_device(table, out)
        with torch.cuda.device(dev):
            L.check(L.lib().step_frames_to_clip_u8(L.ptr(table), B, T, H, W, self.scale, self._mean_rgb, self._std_rgb,
                                                   L.ptr(out), L.stream(dev)))
        return out

    def apply(self, images, device=None):
        """Device stage: the collated uint8 RGB frames -> the fp32 CUDA clip [B, T, 3, H, W] the reference's dataset and
        collate produce.  `images` is a [B, T, 3, H0, W0] tensor or a list of [T, 3, H0_i, W0_i] tensors (keep_frames), on
        a CUDA device or in (pinned) host memory, which is copied in asynchronously on the current stream."""
        if device is None:
            first = images[0]
            device = first.device if first.is_cuda else torch.device("cuda", torch.cuda.current_device())
        device = torch.device(device)
        if isinstance(images, (list, tuple)):
            clips = [c.to(device, non_blocking=True) for c in images]
        else:
            if images.dim() != 5:
                raise ValueError("step_b200: expected frames [B, T, 3, H0, W0], got %s" % (tuple(images.shape),))
            stacked = images.to(device, non_blocking=True)
            clips = [stacked[b] for b in range(stacked.shape[0])]
        if not clips:
            raise ValueError("step_b200: empty batch")
        T = clips[0].shape[0]
        if any(c.dim() != 4 or c.shape[0] != T for c in clips):
            raise ValueError("step_b200: every clip of a batch needs the same number of frames [T, 3, H0, W0]")
        W, H = self.size
        table = frame_table([frame_entry(c, W) for c in clips], device)
        out = torch.empty((len(clips), T, 3, H, W), dtype=torch.float32, device=device)
        return self.launch(table, len(clips), T, out)

    def __str__(self):
        return "BaseTransform(size=%s, mean=%s, stds=%s, scale=%d)\n" % (self.size, self.mean.tolist(), self.stds.tolist(),
                                                                          self.scale)


def keep_frames(collate):
    """Wraps a reference `detection_collate` so the images come back as the list of per-clip tensors instead of one stacked
    tensor: frames of different videos may differ in width (extract_clips.py scales to 360 rows only), and
    `BaseTransform.apply` takes the list.  The other fields are exactly what `collate` returns."""
    def wrapped(batch):
        frames = [sample[0] for sample in batch]
        out = collate([(None,) + tuple(sample[1:]) for sample in batch])
        return (frames,) + tuple(out[1:])
    return wrapped
