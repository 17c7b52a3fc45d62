"""Generates tests/golden/shipped_param_groups.npz by running the reference's own `get_params` (utils/solver.py) over the
reference's modules, built by the module builders of tests/golden/make_golden.py with the values of scripts/train_step.sh
(base_lr 7.5e-5, det_lr0 1.5e-4, det_lr 7.5e-4, rgb input, context on, max_iter 3) and config.py's default weight_decay
1e-7.  Records, in group order, each group's (module key, parameter name, lr, weight_decay).  Only runnable in the build
container; the fixture it writes is committed.

    python tests/golden/make_optim_golden.py
"""
import os
import sys
from types import SimpleNamespace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, build_nets  # noqa: E402  (loads the reference once, as make_golden.py does)
from step_b200 import synth  # noqa: E402

from utils import solver  # noqa: E402  (the reference tree is on sys.path once make_golden has loaded it)

SHIPPED_ARGS = dict(base_lr=7.5e-5, det_lr0=1.5e-4, det_lr=7.5e-4, weight_decay=1e-7, input_type="rgb", no_context=False,
                    max_iter=3)


def shipped_args():
    return SimpleNamespace(**SHIPPED_ARGS)


def gen_shipped_param_groups():
    args = shipped_args()
    cfg = synth.make_cfg(T=3, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 3}, no_context=False, image_size=(400, 400))
    nets = build_nets(cfg, args.max_iter, context=True)
    owner = {id(p): (key, name) for key, net in nets.items() for name, p in net.named_parameters()}
    groups = solver.get_params(nets, args)
    keys, names, lrs, wds = [], [], [], []
    for g in groups:
        assert len(g["params"]) == 1
        key, name = owner[id(g["params"][0])]
        keys.append(key)
        names.append(name)
        lrs.append(g["lr"])
        wds.append(g["weight_decay"])
    np.savez_compressed(os.path.join(OUT, "shipped_param_groups.npz"), module=np.array(keys), name=np.array(names),
                        lr=np.array(lrs, np.float64), weight_decay=np.array(wds, np.float64),
                        numel=np.array([g["params"][0].numel() for g in groups], np.int64))
    print("shipped param groups:", len(groups), "tensors,", sum(g["params"][0].numel() for g in groups), "parameters")


if __name__ == "__main__":
    gen_shipped_param_groups()
