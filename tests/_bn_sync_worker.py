"""torch.distributed.run worker for tests/test_gpu_bn_sync.py: train_step with batch statistics on two ranks.

    python -m torch.distributed.run --standalone --nproc-per-node=2 tests/_bn_sync_worker.py <gloo|nccl> <out_dir>

gloo runs both ranks on cuda:0, nccl rank r on cuda:r.  Each rank saves out_dir/rank<r>.pt: per scenario its loss, the
averaged gradients and the running statistics (CPU tensors keyed "<net>.<name>"), and the outcome of each refusal; rank 0
also saves the nets' state after the first shipped step, for the oracle's second step."""
import os
import sys

import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from step_b200 import optim, synth, training  # noqa: E402
import _bn_sync_case as sc  # noqa: E402

NETS = ("base_net", "context_net", "det_net0", "det_net1", "det_net2")


def build(name, fp16, fa, dev):
    cfg = sc.case_cfg(name, fp16, bool(fa))
    heads = [synth.cls_head_state_dict(100, cfg)] if name == "cls" else [synth.head_state_dict(100 + i, cfg) for i in range(3)]
    nets = synth.device_nets(cfg, heads, "pool", context=True, cls_only=name == "cls", device=dev)
    for k in NETS:
        if nets.get(k) is not None:
            nets[k].train()
    return cfg, nets


def adam(nets):
    return optim.Adam([p for m in NETS if nets.get(m) is not None for p in nets[m].parameters() if p.requires_grad], lr=1e-4)


def state(nets):
    return {"%s.%s" % (m, k): v.detach().cpu().clone() for m in NETS if nets.get(m) is not None
            for k, v in nets[m].state_dict().items()}


def buffers(nets):
    return {k: v for k, v in state(nets).items() if "running_" in k or "num_batches" in k}


def grads(nets, g):
    names = {p: "%s.%s" % (m, k) for m in NETS if nets.get(m) is not None for k, p in nets[m].named_parameters()}
    return {names[p]: v.detach().cpu().clone() for p, v in g.items()}


def step(cfg, nets, rank_case, dev, **kw):
    x, tubes, targets = rank_case
    r = training.train_step(cfg, nets, x.to(dev), [t.to(dev) for t in tubes], [t.to(dev) for t in targets],
                            world_size=dist.get_world_size(), **kw)
    torch.cuda.synchronize(dev)
    return dict(loss=float(r["loss"]), skipped=bool(r["skipped"]), loss_scale=float(r["loss_scale"]), grads=grads(nets, r["grads"]),
                buffers=buffers(nets))


def unequal_case(cfg, rank):
    """Rank r's clip of the shipped case with 3 (rank 0) or 5 (rank 1) rows per step."""
    x = synth.make_clips(2, 36, 64, 64, seed=11)[rank:rank + 1].contiguous()
    tubes, targets = synth.make_train_case(cfg, 1, (3, 5)[rank], 64, 64, seed=20 + rank)
    return x, tubes, targets


def refusals(rank, dev):
    """Each refusal of train_step's up-front plan on both ranks; nothing changes (parameters, running statistics, the
    device generator)."""
    cfg, nets = build("ctx", False, 1, dev)
    x, tubes, targets = sc.split_rows(cfg, *sc.whole_case("ctx", cfg))[rank]
    gen = torch.cuda.default_generators[dev.index]
    before, offset = state(nets), gen.get_offset()
    out = {}
    zero = [t if i != 1 or rank == 0 else t[:0] for i, t in enumerate(tubes)]
    cases = {"steps": dict(tubes=tubes[:2] if rank else tubes, targets=targets[:2] if rank else targets, kw={}),
             "loss_scale": dict(tubes=tubes, targets=targets, kw=dict(loss_scale=2.0 if rank else 1.0)),
             "zero_rows": dict(tubes=zero, targets=[t[:z.shape[0]] for t, z in zip(targets, zero)], kw={}),
             "world_size": dict(tubes=tubes, targets=targets, kw=dict(world_size=3))}
    for name, c in cases.items():
        kw = dict(loss_scale=1.0, world_size=dist.get_world_size())
        kw.update(c["kw"])
        try:
            training.train_step(cfg, nets, x.to(dev), [t.to(dev) for t in c["tubes"]], [t.to(dev) for t in c["targets"]], **kw)
            out[name] = "no error"
        except ValueError as e:
            out[name] = "ValueError: %s" % e
        now = state(nets)
        out[name + ":unchanged"] = all(torch.equal(now[k], v) for k, v in before.items()) and gen.get_offset() == offset
    return out


def main():
    backend, out_dir = sys.argv[1], sys.argv[2]
    rank, local = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", 0 if backend == "gloo" else local)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, device_id=dev if backend == "nccl" else None)
    res = {}
    # the shipped case, fp32, equal rows: two Adam steps
    cfg, nets = build("ctx", False, 0, dev)
    mine = sc.split_rows(cfg, *sc.whole_case("ctx", cfg))[rank]
    opt = adam(nets)
    res["ship1"] = step(cfg, nets, mine, dev, loss_scale=1.0, optimizer=opt)
    if rank == 0:
        res["ship1_state"] = state(nets)
    res["ship2"] = step(cfg, nets, mine, dev, loss_scale=1.0, optimizer=opt)
    # trunk_stats_updated=True after the caller's own training-mode forward of its chunk
    cfg, nets = build("ctx", False, 0, dev)
    with torch.no_grad():
        nets["context_net"](nets["base_net"](mine[0].to(dev)))
    torch.cuda.synchronize(dev)
    res["prepass_buffers"] = buffers(nets)
    res["prepass"] = step(cfg, nets, mine, dev, loss_scale=1.0, optimizer=adam(nets),
                          trunk_stats_updated=True)
    # unequal rows: 3 and 5 per step
    cfg, nets = build("ctx", False, 1, dev)
    res["unequal"] = step(cfg, nets, unequal_case(cfg, rank), dev, loss_scale=1.0,
                          optimizer=adam(nets))
    # one fp16 step with a LossScaler
    cfg, nets = build("ctx", True, 0, dev)
    res["fp16_before"] = buffers(nets)
    res["fp16"] = step(cfg, nets, mine, dev, optimizer=adam(nets),
                       scaler=optim.LossScaler(init_scale=1024.0))
    # the class-only stage
    cfg, nets = build("cls", False, 0, dev)
    res["cls"] = step(cfg, nets, sc.split_rows(cfg, *sc.whole_case("cls", cfg))[rank], dev, loss_scale=1.0,
                      optimizer=adam(nets))
    res["refusals"] = refusals(rank, dev)
    torch.save(res, os.path.join(out_dir, "rank%d.pt" % rank))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
