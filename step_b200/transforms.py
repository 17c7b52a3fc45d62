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
    return L.step_frame_src(clip.data_ptr(), H0, W0, st[0], st[1], st[2], st[3])


def frame_table(entries, device):
    """Uploads step_frame_src entries (one per clip) to `device` on the current stream; the returned tensor is the kernel's
    `table`.  The host copy is pinned, so the upload does not wait for the stream (torch keeps the pinned block until the
    copy has run)."""
    return upload(bytes((L.step_frame_src * len(entries))(*entries)), device)


def upload(data, device):
    """Copies the bytes `data` to `device` on the current stream through a pinned host block, so the copy does not wait
    for the stream (torch keeps the pinned block until the copy has run).  Returns the uint8 device tensor."""
    host = torch.empty(len(data), dtype=torch.uint8, pin_memory=True)
    host.numpy()[:] = np.frombuffer(data, dtype=np.uint8)
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


# --------------------------------------------------------------------------------------------------- TubeAugmentation --
# The reference's RandomSampleCrop modes: the whole frame, a minimum IoU with the boxes, or unconstrained.
CROP_MODES = (None, (0.1, None), (0.3, None), (0.5, None), (0.7, None), (0.9, None), (None, None))
# RandomLightingNoise's channel permutations: channel k of the result is channel perm[k] of its input
PERMS = ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0))
# RandomErase's noise range per ConvertFromInts scale
ERASE_RANGE = {0: (0, 255), 1: (0, 1), 2: (-1, 1)}


class AugRecipe:
    """What TubeAugmentation's host stage drew for one clip, in the order the device stage applies it.

    src_hw: (H0, W0) of the frames it was drawn for.  crop: (x0, y0, w, h), the source pixels kept (the whole frame when
    there is no crop).  flip: mirror the crop.  photometric: whether PhotometricDistort ran; then brightness, contrast,
    saturation and hue are the fp32 values applied (None where the op's gate was off), contrast_first says whether the
    contrast came before the HSV round trip, and perm is the lighting noise's channel permutation (BGR order).  erase: the
    (x1, y1, x2, y2) regions in crop-and-mirror coordinates, later ones on top; noise: their fp32 values, region after
    region, each [y2 - y1, x2 - x1, 3] in BGR order."""

    def __init__(self, src_hw):
        self.src_hw = tuple(src_hw)
        self.crop = (0, 0, src_hw[1], src_hw[0])
        self.flip = False
        self.photometric = False
        self.brightness = self.contrast = self.saturation = self.hue = None
        self.contrast_first = False
        self.perm = PERMS[0]
        self.erase = []
        self.noise = np.zeros(0, np.float32)
        # the crop's bookkeeping: the mode accepted (None: the whole frame) and the trials each test rejected
        self.crop_mode = None
        self.crop_rejects = dict(aspect=0, overlap=0, centre=0, modes=0)

    def __repr__(self):
        return "AugRecipe(src_hw=%s, crop=%s, flip=%s, photometric=%s, brightness=%s, contrast=%s%s, saturation=%s, " \
               "hue=%s, perm=%s, erase=%s)" % (self.src_hw, self.crop, self.flip, self.photometric, self.brightness,
                                               self.contrast, " first" if self.contrast_first else "", self.saturation,
                                               self.hue, self.perm, self.erase)


def _f32_or_none(x):
    return None if x is None else np.float32(x)


class TubeAugmentation:
    """The reference's TubeAugmentation(size, mean, stds, do_flip, do_crop, do_photometric, do_erase, scale) with
    `size = (width, height)` and `mean` / `stds` in BGR order, as there.

    `__call__(images, tubes, proposals)` is the host stage, run in the DataLoader workers.  It does no per-pixel work: it
    draws every random decision from the global numpy RandomState in the reference's order and count, returns the uint8
    frames unchanged and the tubes and proposals the reference returns (bit for bit), and keeps what it drew for the
    clip in `last_recipe`.  `with_recipes` and `keep_recipes` carry that recipe to the main process beside the clip's
    frames, and `apply` builds the fp32 clip from both in one CUDA launch (step_frames_to_clip_aug_u8):

        transform = TubeAugmentation((400, 400), do_flip=True, do_crop=True, do_photometric=True, do_erase=True, scale=2)
        dataset = with_recipes(AVADataset(..., transform), transform)
        loader = DataLoader(dataset, collate_fn=keep_recipes(detection_collate), pin_memory=True, ...)
        for images, targets, tubes, infos in loader:
            images = transform.apply(images)                       # fp32 CUDA clip [B, T, 3, 400, 400]
    """

    def __init__(self, size=300, mean=(0, 0, 0), stds=(1, 1, 1), do_flip=False, do_crop=False, do_photometric=False,
                 do_erase=False, scale=1):
        if isinstance(size, (int, np.integer)):
            size = (size, size)
        self.base = BaseTransform(size, mean, stds, scale)
        self.size, self.mean, self.stds, self.scale = self.base.size, self.base.mean, self.base.stds, scale
        self.do_flip, self.do_crop, self.do_photometric, self.do_erase = do_flip, do_crop, do_photometric, do_erase
        self.last_recipe = None

    # ---------------------------------------------------------------------------------------------- host stage ----
    def __call__(self, images, tubes, proposals=None):
        T, height, width, _ = images.shape
        rec = AugRecipe((height, width))
        if self.do_photometric:
            self._draw_photometric(rec)
        tubes = tubes.copy()
        self._scale_boxes(tubes, width, height, np.multiply)
        if proposals is not None:
            proposals = proposals.copy()
            self._scale_boxes(proposals, width, height, np.multiply)
        if self.do_crop:
            tubes, proposals = self._crop(rec, tubes, proposals, width, height)
        w, h = rec.crop[2], rec.crop[3]
        if self.do_flip:
            tubes, proposals = self._mirror(rec, tubes, proposals, w)
        if self.do_erase:
            self._draw_erase(rec, tubes, w, h)
        self._scale_boxes(tubes, w, h, np.divide)
        if proposals is not None:
            self._scale_boxes(proposals, w, h, np.divide)
        self.last_recipe = rec
        return images, tubes, proposals

    @staticmethod
    def _scale_boxes(boxes, width, height, op):
        """ToAbsoluteCoords (np.multiply) / ToPercentCoords (np.divide), in place and in the boxes' dtype."""
        for k, s in ((0, width), (2, width), (1, height), (3, height)):
            op(boxes[:, :, k], s, out=boxes[:, :, k])

    @staticmethod
    def _draw_photometric(rec):
        """PhotometricDistort's draws.  The ops act on fp32 frames with a Python float, which numpy rounds to fp32 first,
        so the recipe keeps the fp32 values."""
        rnd = np.random
        rec.photometric = True
        rec.brightness = _f32_or_none(rnd.uniform(-32, 32) if rnd.randint(2) else None)
        rec.contrast_first = bool(rnd.randint(2))
        if rec.contrast_first:
            rec.contrast = _f32_or_none(rnd.uniform(0.5, 1.5) if rnd.randint(2) else None)
        rec.saturation = _f32_or_none(rnd.uniform(0.5, 1.5) if rnd.randint(2) else None)
        rec.hue = _f32_or_none(rnd.uniform(-18.0, 18.0) if rnd.randint(2) else None)
        if not rec.contrast_first:
            rec.contrast = _f32_or_none(rnd.uniform(0.5, 1.5) if rnd.randint(2) else None)
        if rnd.randint(2):
            rec.perm = PERMS[rnd.randint(len(PERMS))]

    @staticmethod
    def _iou(boxes, rect):
        """IoU of boxes [N, 4] with the integer rect, with numpy's type promotion of the reference's jaccard_numpy."""
        inter = np.clip(np.minimum(boxes[:, 2:], rect[2:]) - np.maximum(boxes[:, :2], rect[:2]), 0, np.inf)
        inter = inter[:, 0] * inter[:, 1]
        area = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1])
        return inter / (area + (rect[2] - rect[0]) * (rect[3] - rect[1]) - inter)

    def _crop(self, rec, tubes, proposals, width, height):
        """RandomSampleCrop.  The reference draws the mode with random.choice over its tuple of modes, which numpy >= 1.24
        rejects (the tuple is an inhomogeneous array).  Drawing the index instead, choice(len(modes)), takes the same
        value from the legacy stream as numpy 1.x's choice over the object array did, so the mode sequence is the same."""
        rnd = np.random
        boxes = tubes[:, tubes.shape[1] // 2, :4]
        while True:
            mode = CROP_MODES[rnd.choice(len(CROP_MODES))]
            if mode is None:
                return tubes, proposals
            min_iou = -np.inf if mode[0] is None else mode[0]
            max_iou = np.inf if mode[1] is None else mode[1]
            for _ in range(50):
                w = rnd.uniform(0.3 * width, width)
                h = rnd.uniform(0.3 * height, height)
                if h / w < 0.5 or h / w > 2:
                    rec.crop_rejects["aspect"] += 1
                    continue
                # one argument is `low` (high stays 1.0): the reference's draw, kept for its stream and its values
                left = rnd.uniform(width - w)
                top = rnd.uniform(height - h)
                rect = np.array([int(left), int(top), int(left + w), int(top + h)])
                iou = self._iou(boxes, rect)
                if iou.min() < min_iou or iou.max() > max_iou:
                    rec.crop_rejects["overlap"] += 1
                    continue
                centre = (boxes[:, :2] + boxes[:, 2:]) / 2.0
                keep = (rect[0] < centre[:, 0]) & (rect[1] < centre[:, 1]) & \
                       (rect[2] > centre[:, 0]) & (rect[3] > centre[:, 1])
                if not keep.any():
                    rec.crop_rejects["centre"] += 1
                    continue
                rec.crop_mode = mode
                rec.crop = (int(rect[0]), int(rect[1]), int(rect[2] - rect[0]), int(rect[3] - rect[1]))
                kept = tubes[keep]
                self._clamp_shift(kept, rect)
                kept[:, :, :4] = np.maximum(kept[:, :, :4], 0.)
                if proposals is not None:
                    proposals = proposals.copy()
                    self._clamp_shift(proposals, rect)
                    self._valid_tubes(proposals, w, h)
                return kept, proposals
            rec.crop_rejects["modes"] += 1

    @staticmethod
    def _clamp_shift(boxes, rect):
        boxes[:, :, :2] = np.maximum(boxes[:, :, :2], rect[:2])
        boxes[:, :, :2] -= rect[:2]
        boxes[:, :, 2:4] = np.minimum(boxes[:, :, 2:4], rect[2:])
        boxes[:, :, 2:4] -= rect[:2]

    @staticmethod
    def _valid_tubes(proposals, width, height):
        """utils.tube_utils.valid_tubes on the crop's drawn (fractional) size, in place: clamp to the frame, and boxes
        not at least 2 pixels wide and high become the whole frame."""
        b = proposals.reshape(-1, 4)
        b[:, 0] = np.maximum(0, b[:, 0])
        b[:, 1] = np.maximum(0, b[:, 1])
        b[:, 2] = np.minimum(width, b[:, 2])
        b[:, 3] = np.minimum(height, b[:, 3])
        bad = ~((b[:, 0] < b[:, 2] - 2) & (b[:, 1] < b[:, 3] - 2))
        b[bad, :2] = 0
        b[bad, 2] = width
        b[bad, 3] = height
        if not np.shares_memory(b, proposals):
            proposals[...] = b.reshape(proposals.shape)

    @staticmethod
    def _mirror(rec, tubes, proposals, width):
        """RandomMirror: tube boxes flip only where their coordinates sum to more than 0 (all-zero boxes stay)."""
        if not np.random.randint(2):
            return tubes, proposals
        rec.flip = True
        out = tubes.copy()
        b = tubes[:, :, :4]
        flip = ((b[..., 0] + b[..., 1]) + b[..., 2]) + b[..., 3] > 0
        out[..., 0] = np.where(flip, width - tubes[..., 2], tubes[..., 0])
        out[..., 2] = np.where(flip, width - tubes[..., 0], tubes[..., 2])
        if proposals is not None:
            p = proposals.copy()
            p[..., 0] = width - proposals[..., 2]
            p[..., 2] = width - proposals[..., 0]
            proposals = p
        return out, proposals

    def _draw_erase(self, rec, tubes, width, height):
        """RandomErase: one region per tube, from its middle frame's box, filled with uniform noise (drawn as float64,
        stored as the fp32 the frames hold)."""
        rnd = np.random
        if not rnd.randint(2):
            return
        lo, hi = ERASE_RANGE[self.scale]
        noise = []
        for box in tubes[:, tubes.shape[1] // 2, :4]:
            x1, y1, x2, y2 = self._erase_region(box)
            if not (0 <= x1 <= x2 <= width and 0 <= y1 <= y2 <= height):
                raise ValueError("step_b200: erase region %s leaves the %dx%d frame" % ((x1, y1, x2, y2), width, height))
            rec.erase.append((x1, y1, x2, y2))
            noise.append(rnd.uniform(lo, hi, (y2 - y1, x2 - x1, 3)).astype(np.float32).ravel())
        rec.noise = np.concatenate(noise) if noise else rec.noise

    @staticmethod
    def _erase_region(box):
        """RandomErase.get_region: redraw until the region fits the box.  The box's coordinates are np.float32, so the
        products with the Python floats drawn stay fp32, as numpy computes them there."""
        rnd = np.random
        x1, y1, x2, y2 = box
        area = (x2 - x1) * (y2 - y1)
        while True:
            se = rnd.uniform(0.02, 0.2) * area
            ratio = rnd.uniform(0.3, 10 / 3.)
            he, we = np.sqrt(se * ratio), np.sqrt(se / ratio)
            xe = rnd.uniform(x1, x2 - we)
            ye = rnd.uniform(y1, y2 - he)
            if xe + we <= x2 and ye + he <= y2:
                return int(xe), int(ye), int(xe + we), int(ye + he)

    # -------------------------------------------------------------------------------------------- device stage ----
    def apply(self, batch, device=None):
        """Device stage: `batch` is the list of (frames, recipe) pairs keep_recipes collates, frames a uint8 RGB
        [T, 3, H0, W0] tensor on a CUDA device or in (pinned) host memory.  Returns the fp32 CUDA clip [B, T, 3, H, W]
        the reference's TubeAugmentation, dataset and collate produce."""
        if not batch:
            raise ValueError("step_b200: empty batch")
        if device is None:
            first = batch[0][0]
            device = first.device if first.is_cuda else torch.device("cuda", torch.cuda.current_device())
        device = torch.device(device)
        clips = [f.to(device, non_blocking=True) for f, _ in batch]
        T = clips[0].shape[0]
        if any(c.dim() != 4 or c.shape[0] != T for c in clips):
            raise ValueError("step_b200: every clip of a batch needs the same number of frames [T, 3, H0, W0]")
        W, H = self.size
        params, erase, noise = [], [], []
        n_noise = 0
        for c, (_, rec) in zip(clips, batch):
            if not isinstance(rec, AugRecipe) or tuple(c.shape[2:]) != rec.src_hw:
                raise ValueError("step_b200: clip %s does not match its recipe %r" % (tuple(c.shape), rec))
            if rec.crop[2] > MAX_WIDTH_RATIO * W:
                raise ValueError("step_b200: crop width %d exceeds %d x the output width %d" % (rec.crop[2],
                                                                                               MAX_WIDTH_RATIO, W))
            p = L.step_clip_aug(*rec.crop, int(rec.flip), int(rec.photometric))
            for gate, name in (("brightness", "brightness_delta"), ("contrast", "contrast_alpha"),
                               ("saturation", "saturation_alpha"), ("hue", "hue_delta")):
                v = getattr(rec, gate)
                setattr(p, gate, int(v is not None))
                setattr(p, name, 0.0 if v is None else float(v))
            p.contrast_first = int(rec.contrast_first)
            p.perm[:] = list(rec.perm)
            p.erase_begin, p.erase_count = len(erase), len(rec.erase)
            for x1, y1, x2, y2 in rec.erase:
                erase.append(L.step_aug_erase(x1, y1, x2, y2, n_noise))
                n_noise += (x2 - x1) * (y2 - y1) * 3
            if len(rec.noise) != sum((x2 - x1) * (y2 - y1) * 3 for x1, y1, x2, y2 in rec.erase):
                raise ValueError("step_b200: recipe noise does not match its erase regions")
            noise.append(rec.noise)
            params.append(p)
        table = frame_table([frame_entry(c, W) for c in clips], device)
        params_d = upload(bytes((L.step_clip_aug * len(params))(*params)), device)
        erase_d = upload(bytes((L.step_aug_erase * len(erase))(*erase)), device) if erase else None
        noise_d = None
        if n_noise:
            noise_d = torch.from_numpy(np.concatenate(noise).astype(np.float32)).pin_memory().to(device,
                                                                                             non_blocking=True)
        out = torch.empty((len(clips), T, 3, H, W), dtype=torch.float32, device=device)
        return self.launch(table, params_d, erase_d, noise_d, len(clips), T, out)

    def launch(self, table, params, erase, noise, B, T, out):
        """Enqueues the kernel on the current stream: B clips of T frames (frame_table), their step_clip_aug records
        (`params`), erase regions and noise (None when no clip erases) into `out`, contiguous fp32 [B, T, 3, H, W]."""
        W, H = self.size
        if out.dtype != torch.float32 or not out.is_contiguous() or tuple(out.shape) != (B, T, 3, H, W):
            raise ValueError("step_b200: out must be contiguous fp32 %s, got %s %s" % ((B, T, 3, H, W), out.dtype,
                                                                                         tuple(out.shape)))
        dev = L.same_device(table, params, erase, noise, out)
        with torch.cuda.device(dev):
            L.check(L.lib().step_frames_to_clip_aug_u8(
                L.ptr(table), L.ptr(params), None if erase is None else L.ptr(erase),
                None if noise is None else L.ptr(noise), B, T, H, W, self.scale, self.base._mean_rgb,
                self.base._std_rgb, L.ptr(out), L.stream(dev)))
        return out

    def __str__(self):
        return "TubeAugmentation(size=%s, mean=%s, stds=%s, do_flip=%s, do_crop=%s, do_photometric=%s, do_erase=%s, " \
               "scale=%d)\n" % (self.size, self.mean.tolist(), self.stds.tolist(), self.do_flip, self.do_crop,
                                self.do_photometric, self.do_erase, self.scale)


class with_recipes(torch.utils.data.Dataset):
    """Wraps a reference dataset built with `transform` (a TubeAugmentation): each sample gets the recipe the transform
    drew for it appended as its last element.  A worker runs __getitem__ one sample at a time, so the transform's
    per-process `last_recipe` belongs to the sample just produced."""

    def __init__(self, dataset, transform):
        self.dataset, self.transform = dataset, transform

    def __len__(self):
        return len(self.dataset)

    def __getitem__(self, index):
        self.transform.last_recipe = None
        sample = self.dataset[index]
        rec, self.transform.last_recipe = self.transform.last_recipe, None
        if rec is None:
            raise RuntimeError("step_b200: the dataset did not call its TubeAugmentation for sample %r" % (index,))
        return tuple(sample) + (rec,)

    def __getattr__(self, name):  # the wrapped dataset's attributes (name, num_classes, ...)
        if name in ("dataset", "transform"):
            raise AttributeError(name)
        return getattr(self.dataset, name)


def keep_recipes(collate):
    """Wraps a reference `detection_collate` for a `with_recipes` dataset: the images come back as the list of
    (uint8 frames, recipe) pairs TubeAugmentation.apply takes, the other fields exactly as `collate` returns them."""
    def wrapped(batch):
        pairs = [(sample[0], sample[-1]) for sample in batch]
        out = collate([(None,) + tuple(sample[1:-1]) for sample in batch])
        return (pairs,) + tuple(out[1:])
    return wrapped
