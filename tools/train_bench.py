"""Time one training step (step_b200.training.train_step: train.py:263-348 for already selected samples).

    python tools/train_bench.py [B]              C4 shape: B clips of T=32 x 224 x 224, 11 tubes per clip, 3 spatial steps
    python tools/train_bench.py --shipped [B]    the reference's shipped configuration (scripts/train_step.sh): B clips of
                                                 36 x 400 x 400, 34 tubes per clip, 3 temporal steps (NUM_CHUNKS {1:1, 2:1,
                                                 3:3}: frames [3, 6), [3, 6), [0, 9) of T'=9), ContextNet on
    python tools/train_bench.py --cls [B]        the classification pre-training stage (scripts/train_cls.sh): B clips of
                                                 36 x 400 x 400, 20 tubes per clip (5 positives; the last clip negatives
                                                 only), one class-only head over T=9 frames, ContextNet on, Adam with a
                                                 LossScaler
    --pool (with any of the above)               ROINet("pool", 7), the reference's default pool_mode (config.py:67): ROIPool
                                                 forward with argmax and its deterministic backward instead of ROIAlign
    --fp32 (with any of the above)               the fp32 path (cfg.fp16=False, the reference's default precision): fp32
                                                 activations and gradients, SIMT convolutions and step_conv_wgrad_f32;
                                                 loss_scale 1.0 and, with --cls, no LossScaler
Correctness is covered by tests/test_gpu_train.py, tests/test_gpu_train_context.py, tests/test_gpu_train_cls.py and
tests/test_gpu_train_pool.py; this only
reports where the (not yet optimised) step stands."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import step_b200
from step_b200 import optim, synth, training
shipped = "--shipped" in sys.argv
cls = "--cls" in sys.argv
pool_mode = "pool" if "--pool" in sys.argv else "align"
fp16 = "--fp32" not in sys.argv
pos = [a for a in sys.argv[1:] if not a.startswith("--")]
if cls:
    B = int(pos[0]) if pos else 4
    N, T_in, HW = 20, 36, 400
    cfg = synth.make_cfg(fp16=fp16, T=9, max_iter=1, NUM_CHUNKS={1: 1}, no_context=False, image_size=(HW, HW))
elif shipped:
    B = int(pos[0]) if pos else 2
    N, T_in, HW = 34, 36, 400
    cfg = synth.make_cfg(fp16=fp16, T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False, image_size=(HW, HW))
else:
    B = int(pos[0]) if pos else 8
    N, T_in, HW = 11, 32, 224
    cfg = synth.make_cfg(fp16=fp16, T=8, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 1}, image_size=(HW, HW))
nets = {"base_net": step_b200.BaseNet(cfg), "roi_net": step_b200.ROINet(pool_mode, 7)}
nets["base_net"].load_state_dict(synth.base_net_state_dict())
if shipped or cls:
    nets["context_net"] = step_b200.ContextNet(cfg)
    nets["context_net"].load_state_dict(synth.context_net_state_dict())
if cls:
    h = step_b200.TwoBranchNet(cfg, cls_only=True); h.load_state_dict(synth.cls_head_state_dict(100, cfg)); nets["det_net0"] = h
else:
    for i in range(3):
        h = step_b200.TwoBranchNet(cfg); h.load_state_dict(synth.head_state_dict(100 + i, cfg)); nets["det_net%d" % i] = h
for k in nets:
    nets[k] = nets[k].cuda().eval()
    if hasattr(nets[k], "set_device"):
        nets[k].set_device("cuda:0")
x = synth.make_clips(B, T_in, HW, HW).cuda()
if cls:
    ft, fg = synth.make_cls_case(cfg, B, N, HW, HW)
    step_tubes, step_targets = [ft.cuda()], [fg.cuda()]
elif shipped:
    st, sg = synth.make_train_case(cfg, B, N, HW, HW)
    step_tubes, step_targets = [t.cuda() for t in st], [t.cuda() for t in sg]
else:
    props = synth.make_proposals(B, N, cfg.T, 224, 224)
    flat, _ = step_b200.tube_utils.flatten_tubes(props, batch_idx=True)
    tubes = torch.from_numpy(flat).cuda()
    gen = torch.Generator().manual_seed(0)
    tg = torch.zeros(B * N, 3, 66)
    tg[:, :, :4] = tubes[:, 4:5, 1:].cpu() + torch.rand(B * N, 3, 4, generator=gen) * 6
    tg[:, :, 4:6] = (torch.rand(B * N, 3, 2, generator=gen) > 0.3).float(); tg[0, :, 4:6] = 1
    tg[:, :, 6:] = (torch.rand(B * N, 3, 60, generator=gen) > 0.9).float()
    step_tubes, step_targets = [tubes] * 3, [tg.cuda()] * 3
# --cls: the step with train_cls.py's optimizer, Adam with dynamic loss scaling (one rate for all tensors: it does not change
# the time of the single multi-tensor launch)
opt = optim.Adam([p for n in nets.values() for p in n.parameters() if p.requires_grad], lr=5e-8) if cls else None
scaler = optim.LossScaler() if cls and fp16 else None
loss_scale = 1024.0 if fp16 else 1.0
# Otherwise timing of the full step incl. an SGD update.  The update is layer-wise normalised (every tensor moves by 3e-4 of its own norm):
# the synthetic nets pair regressor weights of std 5e-5 with convolution weights of O(0.05), one global rate cannot suit both
for it in range(4):
    training.TIMING = {} if it == 3 else None
    torch.cuda.synchronize(); t0 = time.perf_counter()
    if cls:
        r = training.train_step(cfg, nets, x, step_tubes, step_targets, optimizer=opt, scaler=scaler, loss_scale=loss_scale)
    else:
        r = training.train_step(cfg, nets, x, step_tubes, step_targets, lr=None, loss_scale=loss_scale)
        for p, g in r["grads"].items():
            pn, gn = float(p.detach().norm()), float(g.norm())
            if pn > 0 and gn > 0:
                training.sgd_step({p: g}, lr=3e-4 * pn / gn, momentum=0.0)
    torch.cuda.synchronize(); dt = time.perf_counter() - t0
    print(json.dumps({"iter": it, "config": "cls" if cls else "shipped" if shipped else "c4", "pool_mode": pool_mode, "precision": "fp16" if fp16 else "fp32", "B": B, "train_step_ms": round(dt * 1e3, 1), "loss": round(float(r["loss"]), 5),
                      "clips_per_s": round(B / dt, 1), "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 2)}), flush=True)
phases = training.timing_summary()
wgrad = round(sum(v for k, v in phases.items() if k.startswith("wgrad_")), 2)
print(json.dumps({"device_ms_by_phase_of_the_backward_tape": phases, "wgrad_ms": wgrad,
                  "wgrad_share_of_step": round(wgrad / (dt * 1e3), 3)}))
