"""Writes tests/golden/lr_schedules.npz: the learning rate of the reference's cosine schedulers (Deraining/basicsr/models/
lr_scheduler.py: CosineAnnealingRestartCyclicLR for the four Deraining recipes, CosineAnnealingRestartLR on a made-up schedule) at
sampled iterations: around every restart, and across each run.  Iteration `it` runs at last_epoch it - 1 (base_model.py:183-193).

The reference's lr_scheduler.py is imported from a checkout of the reference project at generation time only:
    python tests/golden/make_golden_lr.py /path/to/reference
Each schedule is stored as <name>/it (int64) and <name>/lr (float64, the reference's Python float)."""
import importlib.util
import os
import sys
import warnings

import numpy as np
import torch

# name -> (scheduler class, base lr, keyword arguments, total_iter); the Deraining entries restate the recipes'
# train.scheduler / optim_g.lr / total_iter
SCHEDULES = {
    "mamber28": ("CosineAnnealingRestartCyclicLR", 3e-4,
                 {"periods": [92000, 208000], "restart_weights": [1, 1], "eta_mins": [0.0003, 0.000001]}, 300000),
    "mamber32": ("CosineAnnealingRestartCyclicLR", 1e-4,
                 {"periods": [48000, 96000], "restart_weights": [1, 1], "eta_mins": [0.000285, 0.000001]}, 144001),
    "mamber33": ("CosineAnnealingRestartCyclicLR", 3e-4,
                 {"periods": [144000, 288000], "restart_weights": [1, 1], "eta_mins": [0.0003, 0.000001]}, 396000),
    "mamber34": ("CosineAnnealingRestartCyclicLR", 3e-4,
                 {"periods": [144000, 288000], "restart_weights": [1, 1], "eta_mins": [0.0003, 0.000001]}, 396000),
    "restart": ("CosineAnnealingRestartLR", 2e-4,
                {"periods": [10, 20, 30, 40], "restart_weights": [1, 0.5, 0.5, 0.25], "eta_min": 1e-7}, 100),
}


def iterations(periods, total):
    """every iteration within 3 of a restart (last_epoch at a cumulative period), 1 and `total`, and a sweep of ~400 across"""
    its = {1, 2, total}
    c = 0
    for p in periods:
        c += p
        its.update(range(c - 2, c + 5))
    its.update(range(1, total + 1, max(1, total // 400)))
    return sorted(i for i in its if 1 <= i <= total)


def main(ref_root):
    spec = importlib.util.spec_from_file_location("ref_lr_scheduler",
                                                  os.path.join(ref_root, "Deraining", "basicsr", "models", "lr_scheduler.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    out = {}
    for name, (cls, base, kw, total) in SCHEDULES.items():
        opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=base)
        sched = getattr(mod, cls)(opt, **kw)
        its = iterations(kw["periods"], total)
        lrs = []
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")  # get_lr() outside step(): the closed form at last_epoch
            for it in its:
                sched.last_epoch = it - 1
                lrs.append(sched.get_lr()[0])
        out[f"{name}/it"] = np.asarray(its, dtype=np.int64)
        out[f"{name}/lr"] = np.asarray(lrs, dtype=np.float64)
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "lr_schedules.npz"), **out)


if __name__ == "__main__":
    main(sys.argv[1])
