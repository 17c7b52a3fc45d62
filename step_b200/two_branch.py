"""`TwoBranchNet` and `ContextNet` with the reference's constructor / forward signatures and
state_dict keys (models/two_branch.py:113-373), running on libstep_b200.so.

TwoBranchNet.forward(global_feat[R,T',832,7,7], context_feat=None|[R,1024,T',1,1], tubes, targets)
  -> (global_prob[R,cls], local_loc[R,T',4], first_loc[R,T,4], last_loc[R,T,4], loss x3)
With targets=None the three losses are returned as zeros exactly as the reference does
(two_branch.py:278-280, 338-340); with targets they are computed on the device (step_b200/training.py::head_losses,
eval-mode dropout; heads built with cls_only=True compute the classification loss alone, training.cls_loss).  The outputs
carry no grad_fn: the backward of the head (with or without the context columns) and of ContextNet runs explicitly on the
forward's tape (step_b200/training.py: head_forward_backward, context_backward, train_step).

Layout tricks (none changes results beyond fp rounding):
  * ROI features and the 1x1x1 `downsample` output share one [R*T',7,7,1088] buffer, so the concat
    of two_branch.py:256 is free;
  * the classifier is linear, so the temporal mean (two_branch.py:249) is taken on the features
    before `global_cls` instead of on the logits (T' times less work);
  * Linear / global_cls weights are permuted once from the reference's (c*49 + h*7 + w) flattening
    (two_branch.py:239,261) to channels-last ((h*7 + w)*256 + c).
"""
import torch
import torch.nn as nn

from . import _lib as L
from . import engine as E
from .engine import Act
from .i3d import I3D_head
from .networks import to_act, weights_init

__all__ = ['ContextNet', 'TwoBranchNet']


def build_conv(base_name='i3d', kinetics_pretrain=None, mode='global', freeze_affine=True):
    """two_branch.py:20-57"""
    if base_name != "i3d":
        raise NotImplementedError
    i3d = I3D_head()
    if kinetics_pretrain is not None:
        import os
        if not os.path.isfile(kinetics_pretrain):
            raise ValueError("Kinetics_pretrain doesn't exist: {}".format(kinetics_pretrain))
        model_dict = i3d.state_dict()
        pre = torch.load(kinetics_pretrain, map_location="cpu")
        model_dict.update({k: v for k, v in pre.items() if k in model_dict})
        i3d.load_state_dict(model_dict)
    if mode == 'context':
        model = nn.Sequential(i3d.maxPool3d, i3d.mixed_5b, i3d.mixed_5c)
    else:
        model = nn.Sequential(i3d.mixed_5b, i3d.mixed_5c)
    if freeze_affine:
        for m in model.modules():
            if m.__class__.__name__.find('BatchNorm') != -1:
                for p in m.parameters():
                    p.requires_grad = False
    return model


def _packed(mod, code, kind="conv"):
    """Pack (and cache on the module) the weights of an nn.Conv2d / nn.Conv3d / nn.Linear container."""
    key = (code, kind) + E.params_key(mod.weight, mod.bias)
    c = mod.__dict__.get("_step_cache")
    if c is None or c[0] != key:
        if kind == "conv":
            w = E.pack_conv_weight(mod.weight, code)
            bias = mod.bias.detach().float().contiguous() if mod.bias is not None else None
            val = (w, bias)
        else:
            raise AssertionError(kind)
        mod.__dict__["_step_cache"] = (key, val)
        c = mod.__dict__["_step_cache"]
    return c[1]


def _perm_flat(w2d, fc, ps):
    """[n, fc*ps*ps] with column c*ps*ps + p  ->  column p*fc + c."""
    n = w2d.shape[0]
    return w2d.detach().float().view(n, fc, ps * ps).permute(0, 2, 1).reshape(n, fc * ps * ps).contiguous()


def conv2d(mod, x, relu, residual=None, out=None):
    """nn.Conv2d container (kernel 1 or 3, stride 1, pad k//2) on frames Act [F,1,H,W,*]."""
    w, bias = _packed(mod, x.code)
    kh, kw = mod.kernel_size
    if out is None:
        out = Act.empty(x.N, 1, x.H, x.W, mod.out_channels, x.code, x.device)
    return E.conv(x, w, None, bias, out, (1, kh, kw), (1, 1, 1), (0, kh // 2, kw // 2), relu, residual, tag=mod)


class Bottleneck(nn.Module):
    """two_branch.py:60-84"""

    def __init__(self, inplanes, planes, stride=1):
        super(Bottleneck, self).__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=1, bias=False)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, stride=stride, padding=1, bias=False)
        self.conv3 = nn.Conv2d(planes, inplanes, kernel_size=1, bias=False)
        self.relu = nn.ReLU(inplace=True)
        self.stride = stride

    def forward(self, x):
        o = conv2d(self.conv1, x, True)
        o = conv2d(self.conv2, o, True)
        return conv2d(self.conv3, o, True, residual=x)  # out += residual; relu  (two_branch.py:79-82)


class Bottleneck_resample(nn.Module):
    """two_branch.py:86-111"""

    def __init__(self, inplanes, outplanes, planes, stride=1):
        super(Bottleneck_resample, self).__init__()
        self.conv1 = nn.Conv2d(inplanes, outplanes, kernel_size=1, bias=False)
        self.conv2 = nn.Conv2d(inplanes, planes, kernel_size=1, bias=False)
        self.conv3 = nn.Conv2d(planes, planes, kernel_size=3, stride=stride, padding=1, bias=False)
        self.conv4 = nn.Conv2d(planes, outplanes, kernel_size=1, bias=False)
        self.relu = nn.ReLU(inplace=True)
        self.stride = stride

    def forward(self, x):
        box = {}
        # the residual projection (conv1) is independent of the conv2 -> conv3 chain
        E.run_parallel(x.device,
                       lambda: box.__setitem__("o", conv2d(self.conv3, conv2d(self.conv2, x, True), True)),
                       [lambda: box.__setitem__("res", conv2d(self.conv1, x, False))])
        return conv2d(self.conv4, box["o"], True, residual=box["res"])


class ContextNet(nn.Module):
    """two_branch.py:113-161.  forward(conv_feat[N,T',832,H',W']) -> [N,1024,T',1,1].

    The reference hard-codes AvgPool3d((1,13,13)) and therefore only accepts 400x400 inputs
    (25 -> 13 after the pool); here the average is taken over the whole map, which is the same
    number at 400x400 and well defined elsewhere."""

    def __init__(self, cfg):
        super(ContextNet, self).__init__()
        self.T = cfg.T
        self.freeze_stats = cfg.freeze_stats
        self.freeze_affine = cfg.freeze_affine
        self.fp16 = cfg.fp16
        self.i3d_conv_context = build_conv(cfg.base_net, cfg.kinetics_pretrain, 'context', self.freeze_affine)
        self.avg_pool = nn.AvgPool3d((1, 13, 13), (1, 1, 1))  # kept for repr / state parity; not called
        self._init_net()

    def forward(self, conv_feat):
        L.need_cuda(conv_feat)
        with torch.cuda.device(conv_feat.device):
            ctx = self.forward_act(to_act(conv_feat, E.dtype_code(self.fp16)))  # [N, T', 1024] fp32
        return ctx.permute(0, 2, 1).unsqueeze(-1).unsqueeze(-1)

    def forward_act(self, a, keep=None):
        """Act [N,T',H',W',832] -> fp32 tensor [N, T', 1024] (spatial mean).  keep: dict that receives Mixed_5c's output
        Act under "mixed_5c" (the input of the spatial mean, for the backward in step_b200/training.py)."""
        x = self.i3d_conv_context[0](a)
        x = self.i3d_conv_context[1](x)
        x = self.i3d_conv_context[2](x)
        if keep is not None:
            keep["mixed_5c"] = x
        # mean over the H*W pixels of every (n, t): [A = N*T', B = H*W, P = 1, C]
        y = E.mean_mid(x.data_ptr(), x.code, x.N * x.T, x.H * x.W, 1, x.C, x.ld, x.device)
        return y.view(x.N, x.T, x.C)

    def _init_net(self):
        pass

    def set_device(self, device):
        self.device = device

    def train(self, mode=True):
        nn.Module.train(self, mode)
        return self


class TwoBranchNet(nn.Module):
    """two_branch.py:164-373"""

    def __init__(self, cfg, cls_only=False):
        super(TwoBranchNet, self).__init__()
        self.num_classes = cfg.num_classes
        self.T = cfg.T
        self.base_net = cfg.base_net
        self.freeze_stats = cfg.freeze_stats
        self.freeze_affine = cfg.freeze_affine
        self.fc_dim = cfg.fc_dim
        self.dropout_prob = cfg.dropout
        self.pool_size = cfg.pool_size
        self.no_context = cfg.no_context
        self.fp16 = cfg.fp16
        self.cls_only = cls_only

        self.i3d_conv = build_conv(cfg.base_net, cfg.kinetics_pretrain, 'global', self.freeze_affine)
        self.downsample = nn.Conv3d(1024, self.fc_dim, kernel_size=1, stride=1, bias=True)
        self.dropout = nn.Dropout(self.dropout_prob)
        self.global_cls = nn.Conv3d(self.fc_dim * self.pool_size ** 2 + (1024 if not self.no_context else 0),
                                    self.num_classes, (1, 1, 1), bias=True)
        if not self.cls_only:
            self.local_conv = nn.Sequential(Bottleneck_resample(832 + self.fc_dim, 1024, 256),
                                            Bottleneck(1024, 256), Bottleneck(1024, 256))
            self.downsample2 = nn.Conv2d(1024, self.fc_dim, kernel_size=1, stride=1, bias=True)
            self.local_reg = nn.Linear(self.fc_dim * self.pool_size ** 2, 4)
            self.neighbor_reg1 = nn.Linear(self.fc_dim * self.pool_size ** 2, 4)  # for tube t-1
            self.neighbor_reg2 = nn.Linear(self.fc_dim * self.pool_size ** 2, 4)  # for tube t+1
        self.device = None
        self._init_net()

    # ---- weights ------------------------------------------------------------------------------
    def _head_weights(self):
        """fp32 permuted copies of global_cls / local_reg / neighbor_reg (cached per version)."""
        mods = [self.global_cls] + ([self.local_reg, self.neighbor_reg1, self.neighbor_reg2] if not self.cls_only else [])
        key = E.params_key(*[t for m in mods for t in (m.weight, m.bias)])
        c = self.__dict__.get("_hw")
        if c is None or c[0] != key:
            D = self.fc_dim * self.pool_size ** 2
            gw = self.global_cls.weight.detach().float().view(self.num_classes, -1)
            val = {"cls_w": _perm_flat(gw[:, :D], self.fc_dim, self.pool_size),
                   "cls_b": self.global_cls.bias.detach().float().contiguous(),
                   "ctx_w": gw[:, D:].contiguous() if gw.shape[1] > D else None}
            if not self.cls_only:
                for name in ("local_reg", "neighbor_reg1", "neighbor_reg2"):
                    m = getattr(self, name)
                    val[name + "_w32"] = _perm_flat(m.weight, self.fc_dim, self.pool_size)
                    val[name + "_b"] = m.bias.detach().float().contiguous()
            self.__dict__["_hw"] = (key, val)
            c = self.__dict__["_hw"]
        return c[1]

    def _reg_weight(self, name, code):
        hw = self._head_weights()
        k = name + ("_w16" if code == L.F16 else "_w32")
        if k not in hw:
            hw[k] = hw[name + "_w32"].to(torch.float16).contiguous()
        return hw[k], hw[name + "_b"]

    # ---- forward ------------------------------------------------------------------------------
    def forward(self, global_feat, context_feat=None, tubes=None, targets=None):
        dev = self.device
        if dev is not None and str(dev) != "cpu":
            global_feat = global_feat.to(dev)
            if context_feat is not None:
                context_feat = context_feat.to(dev)
        L.same_device(global_feat, context_feat)
        code = E.dtype_code(self.fp16)
        N, T, C, W, H = global_feat.shape
        with torch.cuda.device(global_feat.device):   # kernels run on the device (and its stream) that owns the tensors
            # stage [ROI features | downsample output] in one [N*T,7,7,1088] buffer (two_branch.py:256)
            cat = Act.empty(N, T, W, H, C + self.fc_dim, code, global_feat.device)
            src = to_act(global_feat, code)
            cat.buf[..., :C].copy_(src.buf[..., src.coff:src.coff + C])
            ctx_mean = None
            if context_feat is not None:
                cf = context_feat.detach().float().contiguous().view(N * context_feat.shape[1], T)
                # mean over T' of [N*1024, T', 1] -> [N, 1024]
                ctx_mean = E.mean_mid(cf.data_ptr(), L.F32, N * context_feat.shape[1], T, 1, 1, 1, cf.device).view(N, -1)
            if targets is None:
                prob, loc, first, last = self.forward_act(cat, ctx_mean, None)
            else:
                prob, loc, first, last, logits = self.forward_act(cat, ctx_mean, None, want_logits=True)
        z = torch.tensor(0., device=prob.device)
        if targets is None:
            return prob, loc, first, last, z.view(-1), z.view(-1), z.view(-1)
        # training-time outputs (two_branch.py:276-341), eval-mode dropout; the losses are computed on the device.
        # NOTE: the outputs carry no grad_fn -- the backward runs explicitly (step_b200/training.py::head_forward_backward).
        from . import training
        if tubes is None:
            raise RuntimeError("TwoBranchNet.forward: targets need tubes")
        tb, tg = tubes.to(prob.device), targets.to(prob.device)
        if self.cls_only:
            # train_cls.py:310: only the classification loss; the regression losses are zeros (two_branch.py:276-280)
            return prob, loc, first, last, training.cls_loss(logits, tg), z.view(-1), z.view(-1)
        lc, ll, ln = training.head_losses(logits, loc, first, last, tb, tg, self.T)
        return prob, loc, first, last, lc, ll, ln

    def forward_act(self, cat, ctx_mean=None, ctx_row_map=None, want_logits=False, keep=None, dropout=None):
        """cat: Act [R, T', 7, 7, ld >= 832 + fc] whose first 832 channels hold the ROI features.
        ctx_mean: fp32 [rows, 1024] temporal mean of the context feature; ctx_row_map: int32 [R]
        row of ctx_mean for each tube (None = identity).  Returns fp32 tensors.
        dropout: None (eval-mode dropout, the identity), or the head's two training-mode draws (global, local) of
        step_b200.training.dropout_draw (local None for class-only heads): the classifier then reads the dropped copy of the
        downsample output (two_branch.py:244; the concat into the local branch stays undropped, :256) and the regressors the
        dropped downsample2 output (:261).  The context columns' draw is the caller's: ctx_mean is then already the mean of
        the dropped context (training.head_forward_backward)."""
        R, T, ps = cat.N, cat.T, self.pool_size
        code = cat.code
        roi = cat.slice(0, 832)
        g = self.i3d_conv[0](roi)
        g = self.i3d_conv[1](g)
        # downsample: 1x1x1, bias, no activation (two_branch.py:236) -> channels [832, 832+fc) of cat
        w, bias = _packed(self.downsample, code)
        gconv = cat.slice(832, self.fc_dim)
        E.conv(g, w, None, bias, gconv, (1, 1, 1), relu=False, tag=self.downsample)
        hw = self._head_weights()
        D = self.fc_dim * ps * ps
        gsrc = gconv
        if dropout is not None:
            gsrc = Act.empty(R, T, ps, ps, self.fc_dim, code, cat.device)
            ctx_cols = 0 if hw["ctx_w"] is None else hw["ctx_w"].shape[1]
            L.check(L.lib().step_dropout_global_fwd(dropout[0], L.c_void_p(gconv.data_ptr()), code, cat.ld, R, T, ps * ps, self.fc_dim,
                                                    ctx_cols, L.c_void_p(gsrc.data_ptr()), gsrc.ld, L.stream()))
        # temporal mean then classifier (+ context columns) then sigmoid (two_branch.py:246-249,337)
        xbar = E.mean_mid(gsrc.data_ptr(), code, R, T, ps * ps, self.fc_dim, gsrc.ld, cat.device)
        has_ctx = ctx_mean is not None and hw["ctx_w"] is not None
        logits = E.linear_small_n(xbar, R, D, D, hw["cls_w"], hw["cls_b"], self.num_classes,
                                  act=0 if has_ctx else 1)
        if has_ctx:
            E.linear_small_n(ctx_mean, R, 1024, 1024, hw["ctx_w"], None, self.num_classes, y=logits, act=1,
                             accumulate=True, row_map=ctx_row_map)
        prob = logits
        raw = None
        if want_logits:   # the losses take the pre-sigmoid class scores (two_branch.py:296): same GEMV without the sigmoid
            raw = E.linear_small_n(xbar, R, D, D, hw["cls_w"], hw["cls_b"], self.num_classes, act=0)
            if has_ctx:
                E.linear_small_n(ctx_mean, R, 1024, 1024, hw["ctx_w"], None, self.num_classes, y=raw, act=0,
                                 accumulate=True, row_map=ctx_row_map)
        if self.cls_only:
            if keep is not None:
                keep.update(xbar=xbar)
            z = torch.tensor([0.], device=prob.device)
            return (prob, z, z, z, raw) if want_logits else (prob, z, z, z)
        # local branch on frames (two_branch.py:253-262)
        lf, lf2 = self._local_branch(cat.frames(), want_lf=keep is not None)
        lf2d = lf2
        if dropout is not None:
            lf2d = Act.empty(R * T, 1, ps, ps, self.fc_dim, code, cat.device)
            L.check(L.lib().step_dropout_local_fwd(dropout[1], L.c_void_p(lf2.data_ptr()), code, lf2.ld, R * T, ps * ps, self.fc_dim,
                                                   L.c_void_p(lf2d.data_ptr()), lf2d.ld, L.stream()))
        # the three regressors share their input: one pass with the twelve weight rows (two_branch.py:261-270)
        Tc = self.T
        chunks = int(T / Tc)
        half = int(Tc / 2)
        s0, s1 = max(int(Tc / 2) - half, 0), min(int(Tc / 2) + half + 1, T)
        e0 = max((chunks - 1) * Tc + int(Tc / 2) - half, 0)
        e1 = min((chunks - 1) * Tc + int(Tc / 2) + half + 1, T)
        w12, b12 = self._reg12(code)
        local_loc = torch.empty((R, T, 4), dtype=torch.float32, device=cat.device)
        first = torch.empty((R, s1 - s0, 4), dtype=torch.float32, device=cat.device)
        last = torch.empty((R, e1 - e0, 4), dtype=torch.float32, device=cat.device)
        nbytes = L.lib().step_linear_small_n_workspace_bytes(R * T, D, 12)
        ws = torch.empty((max(nbytes, 4) // 4,), dtype=torch.float32, device=cat.device)
        L.check(L.lib().step_head_regress(L.ptr(lf2d.buf), code, R, T, D, D, L.ptr(w12), L.ptr(b12), s0, s1, e0, e1,
                                          L.ptr(local_loc), L.ptr(first), L.ptr(last), L.ptr(ws), nbytes, L.stream()))
        if keep is not None:   # activations the training pieces need (step_b200/training.py): channels-last layouts
            keep.update(xbar=xbar, local_feat=lf, local_feat2=lf2, local_feat2_dropped=lf2d, slices=(s0, s1, e0, e1))
        return (prob, local_loc, first, last, raw) if want_logits else (prob, local_loc, first, last)

    def _local_branch(self, frames, want_lf=False):
        """local_conv (Bottleneck_resample + 2 Bottlenecks) and downsample2 on frames (two_branch.py:258-259).  Returns
        (local_feat or None, local_feat2).  On the fp16 inference path the exit of every block (1x1 conv + residual + ReLU)
        runs in one launch with the 1x1 convolution that consumes it (engine.bottleneck_exit); otherwise layer by layer."""
        code = frames.code
        F, ps = frames.N, self.pool_size
        blocks = list(self.local_conv)
        w2, b2 = _packed(self.downsample2, code)
        lf2 = Act.empty(F, 1, ps, ps, self.fc_dim, code, frames.device)
        rs = blocks[0]
        fuse = (len(blocks) == 3 and isinstance(rs, Bottleneck_resample) and all(isinstance(b, Bottleneck) for b in blocks[1:])
                and E.can_fuse_exit(code, rs.conv4.in_channels, rs.conv4.out_channels, self.fc_dim)
                and all(b.conv1.in_channels == 1024 and b.conv1.out_channels == 256 and b.conv3.in_channels == 256
                        and b.conv3.out_channels == 1024 for b in blocks[1:]))
        if not fuse:
            lf = self.local_conv(frames)
            E.conv(lf, w2, None, b2, lf2, (1, 1, 1), relu=False, tag=self.downsample2)
            return lf, lf2
        # block 0: conv2 -> conv3 chain beside the residual projection conv1 (two_branch.py:100-110)
        box = {}
        E.run_parallel(frames.device,
                       lambda: box.__setitem__("o", conv2d(rs.conv3, conv2d(rs.conv2, frames, True), True)),
                       [lambda: box.__setitem__("res", conv2d(rs.conv1, frames, False))])
        h, x = box["o"], box["res"]
        w3 = _packed(rs.conv4, code)[0]
        for nxt in blocks[1:]:
            # y = relu(conv_exit(h) + x) is the block's output and the next block's residual; z = relu(next.conv1(y))
            y = Act.empty(F, 1, ps, ps, 1024, code, frames.device)
            z = Act.empty(F, 1, ps, ps, 256, code, frames.device)
            E.bottleneck_exit(h, w3, x, _packed(nxt.conv1, code)[0], None, True, z, y)
            h = conv2d(nxt.conv2, z, True)
            x = y
            w3 = _packed(nxt.conv3, code)[0]
        # last block's exit + downsample2 (bias, no activation); its output is only materialised when a caller keeps it
        lf = Act.empty(F, 1, ps, ps, 1024, code, frames.device) if want_lf else None
        E.bottleneck_exit(h, w3, x, w2, b2, False, lf2, lf)
        return lf, lf2

    def _reg12(self, code):
        """[W_local | W_nb1 | W_nb2] (12 x D, permuted to channels-last) in the compute dtype + fp32 biases."""
        hw = self._head_weights()
        k = "w12_%d" % code
        if k not in hw:
            w = torch.cat([hw[n + "_w32"] for n in ("local_reg", "neighbor_reg1", "neighbor_reg2")], 0)
            hw[k] = w.to(E.torch_dtype(code)).contiguous()
            hw["b12"] = torch.cat([hw[n + "_b"] for n in ("local_reg", "neighbor_reg1", "neighbor_reg2")]).contiguous()
        return hw[k], hw["b12"]

    def _init_net(self):
        self.global_cls.apply(weights_init)
        self.downsample.apply(weights_init)
        if not self.cls_only:
            self.local_conv.apply(weights_init)
            self.local_reg.apply(weights_init)
            self.downsample2.apply(weights_init)
            self.neighbor_reg1.apply(weights_init)
            self.neighbor_reg2.apply(weights_init)

    def set_device(self, device):
        self.device = device

    def train(self, mode=True):
        nn.Module.train(self, mode)
        return self
