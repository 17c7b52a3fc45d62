"""step_b200 -- the STEP (NVlabs/STEP) inference hot path on H100 (sm_90a).

Public surface mirrors the reference (SURVEY.md section 8b):
    from step_b200 import BaseNet, ROINet, TwoBranchNet, ContextNet      # models/__init__.py:6-7
    from step_b200 import inference                                       # utils/utils.py:15
    from step_b200 import select_samples                                  # utils/utils.py:135 train_select, per step
    from step_b200 import select_cls_samples                              # train_cls.py:260-297 select_proposals
    from step_b200 import FrameAP                                         # utils/eval_utils.py ava_evaluation
    from step_b200.roi_layers import nms, roi_align, ROIAlign, roi_pool, ROIPool
    from step_b200 import tube_utils                                      # utils/tube_utils.py
All compute goes through libstep_b200.so (include/step_b200.h); there is no CPU/PyTorch fallback.
"""
from .networks import BaseNet, ROINet  # noqa: F401
from .two_branch import ContextNet, TwoBranchNet  # noqa: F401
from .inference import inference  # noqa: F401
from .runner import StepRunner  # noqa: F401
from .select import select_cls_samples, select_samples  # noqa: F401
from .evaluation import FrameAP  # noqa: F401
from . import optim, postprocess, roi_layers, tube_utils  # noqa: F401

__all__ = ["BaseNet", "ROINet", "TwoBranchNet", "ContextNet", "inference", "select_samples", "select_cls_samples", "FrameAP", "StepRunner", "roi_layers",
           "tube_utils", "postprocess"]
