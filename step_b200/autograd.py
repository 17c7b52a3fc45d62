"""torch.autograd Functions behind BaseNet.forward, ContextNet.forward and TwoBranchNet.forward, so that the reference's own
training drivers back-propagate with `loss.backward()` (train.py:345-347, train_cls.py:318-321).

Each Function runs the forward half of the module's explicit backward in step_b200/training.py (trunk_forward,
context_forward, head_forward) and, in its backward, the matching backward half (trunk_backward, context_backward,
head_outputs_backward then head_backward) on the upstream gradients autograd hands over: the same code train_step runs.
The module's trainable parameters (those that require grad, in module.parameters() order) are inputs of the Function,
so their gradients reach p.grad through autograd's own accumulation; a trainable parameter the backward finds no
gradient for is an error.  The halves run with loss_scale=1.0: the upstream gradients carry whatever scale the loss was
multiplied by, and the parameter gradients come back with it (as torch.amp's GradScaler expects).

The path is taken only when grad mode is on and a trainable parameter or a tensor input requires grad (`wanted`);
otherwise the modules run their forward exactly as before.  The saved tape is released by the first backward: a second
backward through the same forward (retain_graph=True) raises.  Double backward is not supported.
What the driver computes around the modules (the conv_feat slices' .contiguous(), the per-tube context copies, autograd's
sums of several gradients of one tensor) is torch's; the ROI pooling of those slices is roi_layers.py's, whose NCHW
backward has no atomics.  The path repeats bit for bit: two train.py / train_cls.py iterations from the same nets, clips
and generator state give identical gradients and identical parameters after step_b200.optim.Adam (fp32 ROIAlign and
ROIPool, fp16 with a loss scale of 1024, the class-only stage; tests/test_gpu_roi_bwd_det.py)."""
import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import training


def trainable(module):
    """The parameters a module's Function takes: those that require grad, in module.parameters() order."""
    return [p for p in module.parameters() if p.requires_grad]


def wanted(params, *tensors):
    """Whether a forward builds the autograd graph: grad mode is on and a trainable parameter or a tensor input requires
    grad."""
    if not torch.is_grad_enabled():
        return False
    return any(p.requires_grad for p in params) or any(t is not None and t.requires_grad for t in tensors)


def _take_state(ctx, who):
    state = ctx.state
    if state is None:
        raise RuntimeError("%s: a second backward through the same forward; its saved tape was released by the first backward "
                           "(retain_graph=True is not supported here): run the forward again" % who)
    ctx.state = None
    return state


def _param_grads(who, module, params, grads):
    """The gradients of params (a Function's inputs) from {parameter: gradient}; a missing one raises."""
    missing = [p for p in params if p not in grads]
    if missing:
        names = {id(p): n for n, p in module.named_parameters()}
        raise RuntimeError("%s: the backward produced no gradient for the trainable parameter(s) %s"
                           % (who, ", ".join(names.get(id(p), "?") for p in missing)))
    return tuple(grads[p].to(p.dtype).view(p.shape) for p in params)


class BaseNetFunction(Function):
    """conv_feat = BaseNet(clips) (networks.py:69-83) with the trunk's backward.  The clip has no gradient."""

    @staticmethod
    def forward(ctx, net, clips, *params):
        feat, ctx.state = training.trunk_forward(net, clips)
        ctx.net, ctx.params = net, params
        return feat.logical()

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        state = _take_state(ctx, "BaseNet")
        # [N, T', 832, H', W'] in whatever layout autograd hands over -> the channels-last gradient of the trunk's output
        grads = training.trunk_backward(state, g.permute(0, 1, 3, 4, 2), loss_scale=1.0)
        return (None, None) + _param_grads("BaseNet", ctx.net, ctx.params, grads)


class ContextNetFunction(Function):
    """context_feat = ContextNet(conv_feat) (two_branch.py:132-138), with the gradient of conv_feat."""

    @staticmethod
    def forward(ctx, net, feat_act, conv_feat, *params):
        c, ctx.state = training.context_forward(net, feat_act)
        ctx.net, ctx.params, ctx.feat_dtype = net, params, conv_feat.dtype
        return c.permute(0, 2, 1).unsqueeze(-1).unsqueeze(-1)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        state = _take_state(ctx, "ContextNet")
        B, K, Tp = g.shape[:3]
        grads, gfeat = training.context_backward(state, g.reshape(B, K, Tp).permute(0, 2, 1), loss_scale=1.0)
        dfeat = gfeat.permute(0, 1, 4, 2, 3).to(ctx.feat_dtype)           # [B, T', 832, H', W'] view of the channels-last buffer
        return (None, None, dfeat) + _param_grads("ContextNet", ctx.net, ctx.params, grads)


class TwoBranchNetFunction(Function):
    """The seven outputs of TwoBranchNet.forward(global_feat, context_feat, tubes, targets) (two_branch.py:213-342), with
    the gradients of global_feat and context_feat.  In training mode the head draws the reference's dropout masks."""

    @staticmethod
    def forward(ctx, net, global_feat, context_feat, tubes, targets, *params):
        ctx.set_materialize_grads(False)
        dev = global_feat.device
        N, Tl = global_feat.shape[0], global_feat.shape[1]
        has_targets = targets is not None
        if not has_targets:   # no losses: all-zero masks make the kernel ignore them
            targets = torch.zeros((N, 3, 6 + net.num_classes), dtype=torch.float32, device=dev)
            tubes = torch.zeros((N, Tl, 5), dtype=torch.float32, device=dev) if tubes is None else tubes
        fwd, ctx.state = training.head_forward(net, global_feat, tubes, targets, context_feat=context_feat, dropout=True)
        prob, loc, first, last, logits = fwd["prob"], fwd["loc"], fwd["first"], fwd["last"], fwd["logits"]
        zero = lambda: torch.zeros((1,), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            if not has_targets:
                lc, ll, ln = zero(), zero(), zero()
            elif net.cls_only:
                lc, ll, ln = training.cls_loss(logits, targets), zero(), zero()
            else:
                lc, ll, ln = training.head_losses(logits, loc, first, last, tubes, targets, net.T)
        if net.cls_only:   # the reference's constant [0.] regression outputs (two_branch.py:252)
            loc, first, last = zero(), zero(), zero()
            ctx.mark_non_differentiable(loc, first, last, ll, ln)
        if not has_targets:
            ctx.mark_non_differentiable(lc, ll, ln)
        ctx.net, ctx.params, ctx.logits = net, params, logits
        ctx.feat_dtype = global_feat.dtype
        ctx.ctx_dtype = None if context_feat is None else context_feat.dtype
        ctx.save_for_backward(loc, first, last, tubes, targets)
        return prob, loc, first, last, lc, ll, ln

    @staticmethod
    @once_differentiable
    def backward(ctx, g_prob, g_loc, g_first, g_last, g_lc, g_ll, g_ln):
        state = _take_state(ctx, "TwoBranchNet")
        net = ctx.net
        loc, first, last, tubes, targets = ctx.saved_tensors
        g = training.head_outputs_backward(ctx.logits, loc, first, last, tubes, targets, net.T, net.cls_only, g_prob, g_loc,
                                           g_first, g_last, g_lc, g_ll, g_ln)
        r = training.head_backward(state, g, loss_scale=1.0)
        ctx.logits = None
        dfeat = r["feat_grad"].to(ctx.feat_dtype)
        dctx = None if ctx.ctx_dtype is None else r["ctx_grad"].to(ctx.ctx_dtype)
        return (None, dfeat, dctx, None, None) + _param_grads("TwoBranchNet", net, ctx.params, r["grads"])
