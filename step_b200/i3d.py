"""Inception-I3D building blocks with the reference's class names, constructor signatures and
state_dict keys (models/i3dpt.py:43-173), executing on libstep_b200.so.

The torch.nn.Conv3d / BatchNorm3d children are *parameter containers only* (so that
`load_state_dict`, `.cuda()`, DataParallel replication and checkpoints keep the reference's key
names, SURVEY.md section 5); their forward is never called.  `forward` takes and returns
`engine.Act` handles (channels-last, possibly a channel slice of a wider buffer).
"""
import torch

from . import _lib as L
from . import engine as E
from .engine import Act


def get_padding_shape(filter_shape, stride):
    """i3dpt.py:14-31, same return convention (h_lo, h_hi, w_lo, w_hi, t_lo, t_hi)."""
    pads = [E.same_pad(k, s) for k, s in zip(filter_shape, stride)]
    return pads[1] + pads[2] + pads[0]


class Unit3Dpy(torch.nn.Module):
    """i3dpt.py:43-111: [zero pad] -> Conv3d -> BatchNorm3d -> ReLU.  With the running statistics (eval mode, or a net built
    with cfg.freeze_stats, the default) one fused kernel; with batch statistics (`batch_stats`) the convolution, then
    step_bn_stats and step_bn_apply (engine.conv's `bn`)."""

    # cfg.freeze_stats of the net that owns the unit (set_freeze_stats); a unit outside such a net keeps its statistics
    freeze_stats = True

    def __init__(self, in_channels, out_channels, kernel_size=(1, 1, 1), stride=(1, 1, 1), activation='relu',
                 padding='SAME', use_bias=False, use_bn=True):
        super(Unit3Dpy, self).__init__()
        if padding not in ('SAME', 'VALID'):
            raise ValueError('padding should be in [VALID|SAME] but got {}'.format(padding))
        self.padding = padding
        self.activation = activation
        self.use_bn = use_bn
        self.kernel_size = tuple(kernel_size)
        self.stride = tuple(stride)
        self.conv3d = torch.nn.Conv3d(in_channels, out_channels, kernel_size, stride=stride, bias=use_bias)
        if use_bn:
            self.batch3d = torch.nn.BatchNorm3d(out_channels)
        self._cache = {}

    def batch_stats(self):
        """Whether the BatchNorm normalises with the batch's statistics: the owning net was built with cfg.freeze_stats =
        False and batch3d is in training mode (models/networks.py:85-99).  With freeze_stats the mode is never read."""
        return not self.freeze_stats and self.use_bn and self.batch3d.training

    # -- weight preparation (cached per parameter version / device / dtype) --------------------
    def packed(self, code, s2d=False):
        """(packed weight, scale, shift): the BatchNorm folded with its running statistics, or with batch statistics
        (scale None, shift the conv bias) the weight alone, whose cache then does not follow the running statistics."""
        bn = self.batch3d if self.use_bn else None
        stats = self.batch_stats()
        tens = [self.conv3d.weight, self.conv3d.bias]
        if bn is not None and not stats:
            tens += [bn.weight, bn.bias, bn.running_mean, bn.running_var]
        key = (code, s2d, stats) + E.params_key(*tens)
        hit = self._cache.get("k")
        if hit != key:
            w = E.pack_stem_s2d(self.conv3d.weight) if s2d else E.pack_conv_weight(self.conv3d.weight, code)
            scale, shift = E.fold_bn(None if stats else bn, self.conv3d.bias, self.conv3d.out_channels, w.device)
            self._cache = {"k": key, "v": (w, scale, shift)}
        return self._cache["v"]

    def _bn_kw(self):
        """engine.conv's `bn` keyword with batch statistics; none otherwise, so the frozen-statistics call is unchanged."""
        return {"bn": [self.batch3d]} if self.batch_stats() else {}

    def out_channels(self):
        return self.conv3d.out_channels

    def forward(self, x, out=None, residual=None):
        if not isinstance(x, Act):
            raise RuntimeError("step_b200.Unit3Dpy runs on engine.Act handles; use BaseNet / TwoBranchNet")
        relu = self.activation is not None
        if self.padding == 'VALID':
            pad_lo = (0, 0, 0)
            dims = tuple((d - k) // s + 1 for d, k, s in zip((x.T, x.H, x.W), self.kernel_size, self.stride))
        else:
            pad_lo, dims = None, None
        w, scale, shift = self.packed(x.code)
        if out is None:
            od = dims or E.same_out_dims((x.T, x.H, x.W), self.kernel_size, self.stride)
            out = Act.empty(x.N, od[0], od[1], od[2], self.conv3d.out_channels, x.code, x.device)
        return E.conv(x, w, scale, shift, out, self.kernel_size, self.stride, pad_lo, relu, residual, out_dims=dims, tag=self,
                      **self._bn_kw())

    def forward_s2d(self, x_s2d):
        """fp16 stem: x_s2d is the space-to-depth clip [N, T/2, H/2, W/2, 32]; 4x4x4 filter, pad 1."""
        w, scale, shift = self.packed(L.F16, s2d=True)
        out = Act.empty(x_s2d.N, x_s2d.T, x_s2d.H, x_s2d.W, self.conv3d.out_channels, L.F16, x_s2d.device)
        # only the 8 * Cin live channels of the s2d buffer are convolved (the rest of its row is padding)
        x = x_s2d.slice(0, 8 * self.conv3d.in_channels)
        # the stem's patch-in-shared-memory kernel (csrc/conv_stem.cu) unless STEP_B200_STEM_HALO=0
        # tap plane qt = 2 is k_t = 6 + rt: only the rt = 0 sub-position (channels [0, 4 Cin)) has weights there, the
        # rt = 1 half is structurally zero (engine.pack_stem_s2d) -> the stem kernel skips its channel group 16..23
        return E.conv(x, w, scale, shift, out, (4, 4, 4), (1, 1, 1), (1, 1, 1), self.activation is not None,
                      a_mode=L.A_HALO if E.STEM_HALO else None, out_dims=(x_s2d.T, x_s2d.H, x_s2d.W),
                      zero_cin_last_kt=4 * self.conv3d.in_channels, tag=("s2d", self), **self._bn_kw())


def set_freeze_stats(module, freeze_stats):
    """Give every Unit3Dpy under module its net's cfg.freeze_stats (Unit3Dpy.batch_stats)."""
    for m in module.modules():
        if isinstance(m, Unit3Dpy):
            m.freeze_stats = bool(freeze_stats)


def set_bn_eval(module):
    """The reference's train() overrides with freeze_stats (networks.py:85-99, two_branch.py:146-161, 358-373): every
    BatchNorm under module back in eval mode.  (Their fp16 `.half()` of the BatchNorm does not apply here: the folded
    scale and shift are fp32 on both precision paths.)"""
    for m in module.modules():
        if m.__class__.__name__.find('BatchNorm') != -1:
            m.eval()


class MaxPool3dTFPadding(torch.nn.Module):
    """i3dpt.py:114-126."""

    def __init__(self, kernel_size, stride=None, padding='SAME'):
        super(MaxPool3dTFPadding, self).__init__()
        self.kernel_size = tuple(kernel_size)
        self.stride = tuple(stride if stride is not None else kernel_size)
        if padding == 'SAME':
            self.padding_shape = get_padding_shape(self.kernel_size, self.stride)

    def forward(self, x, out=None):
        return E.maxpool(x, self.kernel_size, self.stride, out)


class Mixed(torch.nn.Module):
    """i3dpt.py:129-163.  The four branches write straight into channel slices of one output
    buffer, so torch.cat (i3dpt.py:162) and its extra read+write disappear."""

    def __init__(self, in_channels, out_channels):
        super(Mixed, self).__init__()
        o = out_channels
        self.branch_0 = Unit3Dpy(in_channels, o[0], kernel_size=(1, 1, 1))
        self.branch_1 = torch.nn.Sequential(Unit3Dpy(in_channels, o[1], kernel_size=(1, 1, 1)),
                                            Unit3Dpy(o[1], o[2], kernel_size=(3, 3, 3)))
        self.branch_2 = torch.nn.Sequential(Unit3Dpy(in_channels, o[3], kernel_size=(1, 1, 1)),
                                            Unit3Dpy(o[3], o[4], kernel_size=(3, 3, 3)))
        self.branch_3 = torch.nn.Sequential(MaxPool3dTFPadding(kernel_size=(3, 3, 3), stride=(1, 1, 1), padding='SAME'),
                                            Unit3Dpy(in_channels, o[5], kernel_size=(1, 1, 1)))
        self.out_plan = (o[0], o[2], o[4], o[5])

    def out_channels(self):
        return sum(self.out_plan)

    def forward(self, x, out=None):
        c0, c1, c2, c3 = self.out_plan
        if out is None:
            out = Act.empty(x.N, x.T, x.H, x.W, c0 + c1 + c2 + c3, x.code, x.device)
        if x.code == L.F16 and E.FUSE_1X1:
            return self._forward_fused(x, out)
        # the heaviest branch (1x1 -> 3x3x3) stays on the caller's stream, the other three fork off
        E.run_parallel(
            x.device,
            lambda: self.branch_1[1](self.branch_1[0](x), out=out.slice(c0, c1)),
            [lambda: self.branch_0(x, out=out.slice(0, c0)),
             lambda: self.branch_2[1](self.branch_2[0](x), out=out.slice(c0 + c1, c2)),
             lambda: self.branch_3[1](self.branch_3[0](x), out=out.slice(c0 + c1 + c2, c3))])
        return out


    def _fused_weights(self):
        """branch_0 | branch_1[0] | branch_2[0] read the same input (i3dpt.py:133-147): one GEMM with
        N = o0 + o1 + o3 whose epilogue scatters the three column ranges to their destinations."""
        units = (self.branch_0, self.branch_1[0], self.branch_2[0])
        parts = [u.packed(L.F16) for u in units]
        key = tuple(id(p[0]) for p in parts)
        c = self.__dict__.get("_fused")
        if c is None or c[0] != key:
            w = torch.cat([p[0] for p in parts], 0).contiguous()
            # batch statistics: no folded scale, and no shift (I3D's Unit3D convolutions have no bias)
            scale = torch.cat([p[1] for p in parts]).contiguous() if parts[0][1] is not None else None
            shift = torch.cat([p[2] for p in parts]).contiguous() if parts[0][2] is not None else None
            self.__dict__["_fused"] = (key, (w, scale, shift))
            c = self.__dict__["_fused"]
        return c[1]

    def _forward_fused(self, x, out):
        c0, c1, c2, c3 = self.out_plan
        w, scale, shift = self._fused_weights()
        m1 = self.branch_1[0].conv3d.out_channels
        m2 = self.branch_2[0].conv3d.out_channels
        t1 = Act.empty(x.N, x.T, x.H, x.W, m1, x.code, x.device)
        t2 = Act.empty(x.N, x.T, x.H, x.W, m2, x.code, x.device)

        units = [self.branch_0, self.branch_1[0], self.branch_2[0]]
        bn = {"bn": [u.batch3d for u in units]} if self.branch_0.batch_stats() else {}

        def trunk():
            E.conv(x, w, scale, shift, out.slice(0, c0), (1, 1, 1), extra_outs=[t1, t2], tag=units, **bn)

        def tail():
            E.run_parallel(x.device,
                           lambda: self.branch_1[1](t1, out=out.slice(c0, c1)),
                           [lambda: self.branch_2[1](t2, out=out.slice(c0 + c1, c2))])
        # the pool -> 1x1 branch only needs x: it overlaps the fused GEMM and the 3x3x3 convs
        E.run_parallel(x.device, lambda: (trunk(), tail()),
                       [lambda: self.branch_3[1](self.branch_3[0](x), out=out.slice(c0 + c1 + c2, c3))],
                       first_side=2)
        return out


class I3D_head(torch.nn.Module):
    """i3dpt.py:165-173."""

    def __init__(self):
        super(I3D_head, self).__init__()
        self.maxPool3d = MaxPool3dTFPadding(kernel_size=(1, 3, 3), stride=(1, 2, 2), padding='SAME')
        self.mixed_5b = Mixed(832, [256, 160, 320, 32, 128, 128])
        self.mixed_5c = Mixed(832, [384, 192, 384, 48, 128, 128])


def build_trunk_stages():
    """The 13 stages BaseNet keeps (networks.py:120-132), i.e. I3D up to mixed_4f (i3dpt.py:184-226)."""
    return [
        Unit3Dpy(out_channels=64, in_channels=3, kernel_size=(7, 7, 7), stride=(2, 2, 2), padding='SAME'),
        MaxPool3dTFPadding(kernel_size=(1, 3, 3), stride=(1, 2, 2), padding='SAME'),
        Unit3Dpy(out_channels=64, in_channels=64, kernel_size=(1, 1, 1), padding='SAME'),
        Unit3Dpy(out_channels=192, in_channels=64, kernel_size=(3, 3, 3), padding='SAME'),
        MaxPool3dTFPadding(kernel_size=(1, 3, 3), stride=(1, 2, 2), padding='SAME'),
        Mixed(192, [64, 96, 128, 16, 32, 32]),
        Mixed(256, [128, 128, 192, 32, 96, 64]),
        MaxPool3dTFPadding(kernel_size=(3, 3, 3), stride=(2, 2, 2), padding='SAME'),
        Mixed(480, [192, 96, 208, 16, 48, 64]),
        Mixed(512, [160, 112, 224, 24, 64, 64]),
        Mixed(512, [128, 128, 256, 24, 64, 64]),
        Mixed(512, [112, 144, 288, 32, 64, 64]),
        Mixed(528, [256, 160, 320, 32, 128, 128]),
    ]
