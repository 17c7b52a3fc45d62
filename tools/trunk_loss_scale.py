"""Per-layer error of the trunk's weight gradients against the oracle's fp32 torch-CPU autograd at two static loss
scales, and how much of each layer's fp16 activation gradient sits in the fp16 subnormal range (|g| < 2^-14).

The case is tests/test_gpu_train.py::test_trunk_backward_matches_reference_autograd (one 8x64x64 clip, loss =
<conv_feat, proj> / numel).  One JSON line per (loss_scale, layer):
    python tools/trunk_loss_scale.py [--scales 1024 65536]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=float, nargs="+", default=[1024.0, 65536.0])
    args = ap.parse_args()
    import step_b200
    from oracle import model as om
    from step_b200 import synth, training
    cfg = synth.make_cfg(fp16=True, T=2, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(64, 64))
    net = step_b200.BaseNet(cfg)
    net.load_state_dict(synth.base_net_state_dict(), strict=True)
    net = net.cuda().eval()
    x = synth.make_clips(1, 8, 64, 64, seed=4321)
    proj = torch.randn((1, 2, 832, 4, 4), generator=torch.Generator().manual_seed(99))
    numel = proj.numel()
    sd = {k: v.clone().requires_grad_(k.endswith("conv3d.weight")) for k, v in synth.base_net_state_dict().items()}
    cf = om.base_net(x.clone(), sd)
    ((cf * proj).sum() / cf.numel()).backward()
    names = {p: k for k, p in net.named_parameters()}
    print(json.dumps({"gpu": torch.cuda.get_device_name(0)}))
    for scale in args.scales:
        calls, orig = [], training.tape_backward

        def spy(tape, grads, loss_scale=1.0, need_input_grad=None):
            out = orig(tape, grads, loss_scale, need_input_grad)
            calls.append((tape, grads))
            return out
        training.tape_backward = spy
        try:
            _, grads = training.trunk_forward_backward(net, x.cuda(), lambda f: (proj / numel).permute(0, 1, 3, 4, 2).contiguous().cuda(),
                                                       loss_scale=scale)
        finally:
            training.tape_backward = orig
        torch.cuda.synchronize()
        tape, store = calls[0]
        sub = {}
        for e in tape:
            if e["kind"] != "conv":
                continue
            tags = e["tag"] if isinstance(e["tag"], list) else [e["tag"]]
            for tg, o in zip(tags, [e["out"]] + e["extra_outs"]):
                unit = tg[1] if isinstance(tg, tuple) else tg
                g = store.of(o).buf[..., o.coff:o.coff + o.C].float().abs()
                nz = g[g > 0]
                sub[unit.conv3d.weight] = (float((nz < 2.0 ** -14).float().mean()) if nz.numel() else 0.0,
                                           float((g == 0).float().mean()))
        for p, gdev in grads.items():
            k = names[p]
            ref = sd[k].grad.double()
            rel = float((gdev.cpu().double() - ref).norm() / ref.norm())
            s, z = sub.get(p, (None, None))
            print(json.dumps({"loss_scale": scale, "layer": k, "rel_l2": round(rel, 5),
                              "norm_ratio": round(float(gdev.double().norm()) / float(ref.norm()), 5),
                              "out_grad_subnormal_frac": s, "out_grad_zero_frac": z}))


if __name__ == "__main__":
    main()
