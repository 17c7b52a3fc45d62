"""torchrun worker for tests/test_gpu_multi.py: rank r runs clips [r*B, (r+1)*B) of a seeded 2B-clip stream through the
captured step (trunk -> 3 refinement steps -> device post-processing) and the fixed-shape detections are gathered with ONE
NCCL all_gather_into_tensor (DESIGN.md section 6).  Rank 0 saves what it gathered."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import step_b200  # noqa: E402
from step_b200 import synth  # noqa: E402


def build(cfg, dev):
    heads = [synth.head_state_dict(100 + i, cfg) for i in range(cfg.max_iter)]
    return synth.device_nets(cfg, heads, cfg.pool_mode, device=dev)


def run_shard(dev, clips, B, T_in, HW, N, detect):
    cfg = synth.make_cfg(fp16=True, T=T_in // 4, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 1}, image_size=(HW, HW))
    nets = build(cfg, dev)
    tubes = synth.make_proposals(B, N, cfg.T, HW, HW)
    runner = step_b200.StepRunner(cfg, nets, B, T_in, HW, HW, tubes, device=dev, detect=detect)
    with torch.no_grad():
        runner(clips.to(dev))
    d = runner.detections[cfg.max_iter - 1]
    return torch.cat([d["det"].view(B, -1), d["count"].view(B, 1).float()], dim=1).contiguous()


def train_inputs(rank, B=1, N=3):
    """Seeded clips / tubes / targets of one rank for the training-step test (one refinement step, T' = 2, 64 x 64)."""
    gen = torch.Generator().manual_seed(100 + rank)
    x = synth.make_clips(B, 8, 64, 64, seed=50 + rank)
    R = B * N
    x1 = torch.rand(R, 1, generator=gen) * 20; y1 = torch.rand(R, 1, generator=gen) * 20
    w = 20 + torch.rand(R, 1, generator=gen) * 20; hh = 20 + torch.rand(R, 1, generator=gen) * 20
    box = torch.cat([x1, y1, x1 + w, y1 + hh], 1)
    frame = (torch.arange(R) // N).view(R, 1, 1) * 2 + torch.arange(2).view(1, 2, 1)
    tubes = torch.cat([frame.float(), box.view(R, 1, 4).expand(R, 2, 4) + torch.rand(R, 2, 4, generator=gen)], 2)
    tg = torch.zeros(R, 3, 66)
    tg[:, :, :4] = box.view(R, 1, 4) + torch.rand(R, 3, 4, generator=gen) * 4
    tg[:, :, 4:6] = 1.0
    tg[:, :, 6:] = (torch.rand(R, 3, 60, generator=gen) > 0.9).float()
    return x, tubes, tg


def train_nets(dev):
    cfg = synth.make_cfg(fp16=True, T=2, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(64, 64))
    return cfg, build(cfg, dev)


WATCH = ("base_net:base_model.12.branch_0.conv3d.weight", "base_net:base_model.3.conv3d.weight", "det_net0:downsample2.weight",
         "det_net0:local_reg.weight")


def watched(nets):
    out = {}
    for key in WATCH:
        net, name = key.split(":")
        out[key] = dict(nets[net].named_parameters())[name].detach().float().cpu().numpy().copy()
    return out


def main_train(out_path):
    """Each rank: gradients of its own clip (training.train_step, no update), then ONE sgd_step with the gradient
    all-reduce over NCCL (mean over ranks, train_step.sh's SGD).  Rank 0 saves the updated watched parameters."""
    from step_b200 import training
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    cfg, nets = train_nets(dev)
    x, tubes, tg = train_inputs(rank)
    r = training.train_step(cfg, nets, x.to(dev), [tubes.to(dev)], [tg.to(dev)], lr=None)
    training.sgd_step(r["grads"], lr=0.05, momentum=0.9, weight_decay=1e-4, world_size=world)
    torch.cuda.synchronize()
    if rank == 0:
        np.savez(out_path, **watched(nets))
    dist.barrier()
    dist.destroy_process_group()


def main():
    if sys.argv[1] == "train":
        return main_train(sys.argv[2])
    out_path, B, T_in, HW, N = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5])
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    clips = synth.make_clips(world * B, T_in, HW, HW, seed=77)[rank * B:(rank + 1) * B].contiguous()
    det = run_shard(dev, clips, B, T_in, HW, N, dict(conf_thresh=0.01, nms_thresh=0.4, topk=50))
    gathered = torch.empty((world,) + tuple(det.shape), dtype=det.dtype, device=dev)
    dist.all_gather_into_tensor(gathered.view(-1, det.shape[1]), det)
    torch.cuda.synchronize()
    if rank == 0:
        np.save(out_path, gathered.cpu().numpy())
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
