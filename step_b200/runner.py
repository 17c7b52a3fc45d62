"""`StepRunner` -- one CUDA graph for the whole batch step.

The reference runs ~600 PyTorch kernels per batch from Python with B*max_iter host round trips
(SURVEY.md section 3.1).  Our step is ~155 launches with no host dependency, so the entire
trunk -> (ROIAlign -> head -> tube update) x max_iter chain is captured ONCE per (B, T, H, W, N) shape into
a CUDA graph (TMA descriptors and buffer addresses are baked at capture) and replayed with a single
`cudaGraphLaunch`: launch latency and Python overhead disappear from the timed path.

    runner = StepRunner(cfg, nets, B, T_in, H, W, tubes)     # captures
    hist = runner(clips)          # clips: [B,T_in,3,H,W] fp32, CUDA or pinned host (copied in asynchronously)
`hist` is the same structure `inference()` returns (tensors are static graph outputs: copy them out
before the next call if they must survive it).
"""
import torch

from . import _lib as L
from . import engine as E
from .inference import inference_device, stage_tubes
from .postprocess import Detector, Merger
from .transforms import frame_entry, frame_table


class StepRunner:
    def __init__(self, cfg, nets, B, T_in, H, W, tubes, device=None, context=False, use_graph=True, warmup=2,
                 detect=None, transform=None, source_hw=None):
        """detect: None, or dict(conf_thresh, nms_thresh, topk[, steps]) -- the reference drivers' detection
        post-processing (test.py:156-218: confidence threshold, valid_tubes, per-class NMS, top-k) appended to the
        captured step for the listed refinement steps (default: the last one); results in `self.detections`.
        transform: None, or a transforms.BaseTransform of output size (W, H) with source_hw = (H0, W0): the runner then
        takes the uint8 RGB frames [B, T_in, 3, H0, W0] (or a list of B [T_in, 3, H0, W0] clips) and the step starts
        with the transform's kernel writing the clip.  The graph bakes the source size: other sizes raise."""
        self.cfg, self.nets = cfg, nets
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        self.context = context and not cfg.no_context
        self.x = torch.zeros((B, T_in, 3, H, W), dtype=torch.float32, device=self.device)
        self.transform = transform
        if transform is not None:
            if source_hw is None:
                raise ValueError("StepRunner: a transform needs source_hw = (H0, W0)")
            if tuple(transform.size) != (W, H):
                raise ValueError("StepRunner: transform size %s is not the clip's (W, H) = %s" % (transform.size, (W, H)))
            self.src = torch.zeros((B, T_in, 3) + tuple(source_hw), dtype=torch.uint8, device=self.device)
            self.table = frame_table([frame_entry(self.src[b], W) for b in range(B)], self.device)
        self.flat, self.clip_of_tube, self.tubes_nums = stage_tubes(tubes, self.device)
        self.graph = None
        self.history = None
        self.detections = None
        self.detectors = {}
        self.merged = None
        self.mergers = {}
        if detect is not None:
            for i in detect.get("steps", [cfg.max_iter - 1]):
                self.detectors[i] = Detector(self.tubes_nums, cfg.num_classes, self.device, detect["conf_thresh"],
                                             detect["nms_thresh"], W, H, topk=detect.get("topk", 0))
                if detect.get("merge") is not None:
                    self.mergers[i] = Merger(self.detectors[i], detect["merge"])
        if not use_graph:
            return
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(warmup):  # packs weights, sets kernel attributes, warms the allocator
                self._body()
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.history = self._body()
        self.graph = g

    def _body(self):
        with torch.no_grad():
            if self.transform is not None:
                self.transform.launch(self.table, self.x.shape[0], self.x.shape[1], self.x)
            feat = self.nets["base_net"].forward_act(self.x)
            ctx_all = self.nets["context_net"].forward_act(feat) if self.context else None
            hist, _ = inference_device(self.cfg, feat, ctx_all, self.nets, self.cfg.max_iter, self.flat,
                                       self.clip_of_tube, self.tubes_nums)
            if self.detectors:
                self.detections = {i: d.run(hist[i]["pred_prob"], hist[i]["pred_loc"]) for i, d in self.detectors.items()}
            if self.mergers:
                self.merged = {i: m.run(self.detections[i]) for i, m in self.mergers.items()}
        return hist

    def __call__(self, clips=None):
        """clips: the fp32 clip [B,T_in,3,H,W], or with a transform the uint8 frames (see __init__); None replays on
        what the static input already holds."""
        if self.transform is not None:
            if clips is not None:
                self._stage_frames(clips)
        elif clips is not None and clips.data_ptr() != self.x.data_ptr():
            self.x.copy_(clips, non_blocking=True)
        if self.graph is None:
            return self._body()
        self.graph.replay()
        return self.history

    def _stage_frames(self, frames):
        """Copies uint8 frames into the static source buffer (asynchronously from pinned host memory)."""
        clips = list(frames) if isinstance(frames, (list, tuple)) else [frames[b] for b in range(frames.shape[0])]
        want = tuple(self.src.shape[1:])
        if len(clips) != self.src.shape[0] or any(tuple(c.shape) != want or c.dtype != torch.uint8 for c in clips):
            raise ValueError("StepRunner: expected %d uint8 clips %s (the captured source size), got %s" % (
                self.src.shape[0], want, [(c.dtype, tuple(c.shape)) for c in clips]))
        if isinstance(frames, torch.Tensor):
            self.src.copy_(frames, non_blocking=True)
        else:
            for dst, c in zip(self.src, clips):
                dst.copy_(c, non_blocking=True)
