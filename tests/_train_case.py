"""Set-up shared by the train_step tests: the seeded two-step spatial case, which state-dict entries the oracle trains,
and the comparison of train_step's gradients with the oracle's autograd."""
import torch

from step_b200 import synth

SHIPPED = synth.WORKLOADS["shipped"].cfg


def rel_l2(got, ref):
    return float((got.detach().cpu().double() - ref.double()).norm() / ref.double().norm())


def trainable(sd):
    """A copy of the state dict sd whose trained entries require grad: every float tensor but BatchNorm's (frozen)."""
    return {k: v.clone().requires_grad_(v.is_floating_point() and "running_" not in k and "batch3d" not in k) for k, v in sd.items()}


def spatial_case():
    """Two spatial refinement steps (T=2, NUM_CHUNKS {1:1, 2:1}) over 2 clips of 8x64x64 with 3 seeded tubes per clip and
    targets with mixed flags: (cfg, clips, step_tubes, step_targets) on the CPU."""
    B, N = 2, 3
    cfg = synth.make_cfg(fp16=True, T=2, max_iter=2, NUM_CHUNKS={1: 1, 2: 1}, image_size=(64, 64))
    x = synth.make_clips(B, 8, 64, 64, seed=11)
    gen = torch.Generator().manual_seed(3)
    step_tubes, step_targets = [], []
    for i in range(2):
        R = B * N
        x1 = torch.rand(R, 1, generator=gen) * 20; y1 = torch.rand(R, 1, generator=gen) * 20
        w = 20 + torch.rand(R, 1, generator=gen) * 20; hh = 20 + torch.rand(R, 1, generator=gen) * 20
        box = torch.cat([x1, y1, x1 + w, y1 + hh], 1)
        frame = (torch.arange(R) // N).view(R, 1, 1) * 2 + torch.arange(2).view(1, 2, 1)
        tubes = torch.cat([frame.float(), box.view(R, 1, 4).expand(R, 2, 4) + torch.rand(R, 2, 4, generator=gen)], 2)
        tg = torch.zeros(R, 3, 66)
        tg[:, :, :4] = box.view(R, 1, 4) + torch.rand(R, 3, 4, generator=gen) * 4
        tg[:, :, 4] = (torch.rand(R, 3, generator=gen) > 0.3).float(); tg[:, :, 5] = (torch.rand(R, 3, generator=gen) > 0.3).float()
        tg[0, :, 4:6] = 1.0
        tg[:, :, 6:] = (torch.rand(R, 3, 60, generator=gen) > 0.9).float()
        step_tubes.append(tubes); step_targets.append(tg)
    return cfg, x, step_tubes, step_targets


def compare_grads(r, module, sd_ref, ntol, ttol):
    """train_step's gradients (r["grads"]) of module's parameters against the oracle's autograd (the .grad of sd_ref[name]):
    the norm within ntol and the difference within ttol of the reference's norm.  Returns the number of tensors compared."""
    names = {p: k for k, p in module.named_parameters()}
    n = 0
    for p, gdev in r["grads"].items():
        if p not in names:
            continue
        ref = sd_ref[names[p]].grad
        rn = float(ref.double().norm())
        assert abs(float(gdev.double().norm()) - rn) <= ntol * rn, (names[p], float(gdev.double().norm()), rn)
        assert float((gdev.cpu().double() - ref.double()).norm()) <= ttol * rn, (names[p], rel_l2(gdev, ref))
        n += 1
    return n
