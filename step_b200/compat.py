"""Run the reference's own drivers (test.py / demo.py, and train.py / train_cls.py on one GPU without apex) of
NVlabs/STEP on step_b200 without editing them.  The training drivers then run their fp32 path (the reference forces
args.fp16 = False without apex) and back-propagate with `loss.backward()` through the modules' torch.autograd Functions
(step_b200/autograd.py), whose backward is train_step's; their gradients repeat bit for bit from run to run (the NCHW
ROI backward has no atomics).  What differs from step_b200.training.train_step: the optimizer is torch's unless the
driver builds it from step_b200.optim (INTEGRATION.md).  nn.DataParallel over several GPUs and apex O1
are not covered.

    import step_b200.compat as compat
    compat.patch("/path/to/STEP")        # before the driver's own imports run
    runpy.run_path("/path/to/STEP/test.py", run_name="__main__")

What gets substituted (the drop-in boundary of SURVEY.md section 8b):
  * `external.maskrcnn_benchmark.roi_layers`  -> step_b200.roi_layers  (nms, roi_align, ROIAlign,
    roi_pool, ROIPool; the reference's `_C` extension is not needed at all);
  * `models.BaseNet / ROINet / TwoBranchNet / ContextNet` -> the step_b200 classes (same
    constructor, forward signature and state_dict keys, so `load_state_dict(checkpoint[...])` and
    `nn.DataParallel(...)` in test.py:79-95 keep working);
  * `utils.utils.inference` -> step_b200.inference (same signature and history/trajectory structure).
Everything else in the reference tree (datasets, config, evaluation, the numpy helpers the drivers
call on host arrays) is left as is.
"""
import importlib
import sys
import types


def _namespace(name):
    m = sys.modules.get(name)
    if m is None:
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules[name] = m
    return m


def patch(reference_root=None):
    import step_b200
    from step_b200 import roi_layers

    if reference_root and reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    # 1. native ops: the package the reference imports resolves to ours
    _namespace("external")
    _namespace("external.maskrcnn_benchmark")
    sys.modules["external.maskrcnn_benchmark.roi_layers"] = roi_layers
    sys.modules["external.maskrcnn_benchmark"].roi_layers = roi_layers
    # 2. model classes
    models = types.ModuleType("models")
    models.__path__ = []
    for n in ("BaseNet", "ROINet", "TwoBranchNet", "ContextNet"):
        setattr(models, n, getattr(step_b200, n))
    models.__all__ = ["BaseNet", "ROINet", "TwoBranchNet", "ContextNet"]
    sys.modules["models"] = models
    # 3. the progressive loop: keep the rest of the reference's utils.utils, swap `inference`
    if reference_root:
        ru = importlib.import_module("utils.utils")
        ru.inference = step_b200.inference
    return step_b200
