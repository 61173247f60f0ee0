"""Torch restatement of the Deraining recipes' batch preparation (test infrastructure): Restormer's progressive patch / batch schedule
(Deraining/basicsr/train.py:213-262) and ImageCleanModel's mixup (Deraining/basicsr/models/image_restoration_model.py:22-49,
136-143), on any device, for vmambair_b200.restore_train to be checked against.

It works on the tensors the way the reference loop does -- advanced indexing for the subset, slicing for the crop, a torch expression
for the mix -- and draws from the same host streams in the same order: Python's `random` for the subset, the crop origin and the
identity choice; torch's default CPU generator for lam (Beta(b, b).rsample) and the permutation (torch.randperm).
"""
from __future__ import annotations

import random

import numpy as np
import torch


def phase(opt, current_iter):
    """the phase index the loop uses at `current_iter`: the first cumulative `iters` entry >= current_iter, else the last"""
    iters = opt["datasets"]["train"]["iters"]
    cumulative = np.cumsum(np.asarray(iters, dtype=np.int64))
    hits = np.flatnonzero(current_iter <= cumulative)
    return int(hits[0]) if hits.size else len(cumulative) - 1


def progressive(opt, current_iter, lq, gt):
    """the loop's subset and crop for `current_iter` -> (lq, gt, phase); gt is cropped at scale x the lq window, x0 offsets rows"""
    d = opt["datasets"]["train"]
    j = phase(opt, current_iter)
    patch, batch, full = d["gt_sizes"][j], d["mini_batch_sizes"][j], d["gt_size"]
    scale = opt["scale"]
    if batch < d["batch_size_per_gpu"]:
        chosen = random.sample(range(d["batch_size_per_gpu"]), k=batch)
        lq, gt = lq[chosen], gt[chosen]
    if patch < full:
        x0 = int((full - patch) * random.random())
        y0 = int((full - patch) * random.random())
        lq = lq[:, :, x0:x0 + patch, y0:y0 + patch]
        gt = gt[:, :, x0 * scale:(x0 + patch) * scale, y0 * scale:(y0 + patch) * scale]
    return lq, gt, j


class Mixup:
    """ImageCleanModel's mixing augmentation (train.mixing_augs): one augment, mixup, optionally next to the identity"""

    def __init__(self, beta, use_identity):
        self.dist = torch.distributions.Beta(torch.tensor([float(beta)]), torch.tensor([float(beta)]))
        self.use_identity = use_identity

    def __call__(self, gt, lq):
        pick = random.randint(0, 1) if self.use_identity else random.randint(0, 0)
        if pick == 1:  # the identity
            return gt, lq
        lam = self.dist.rsample((1, 1)).item()
        r = torch.randperm(gt.shape[0]).to(gt.device)
        return lam * gt + (1 - lam) * gt[r, :], lam * lq + (1 - lam) * lq[r, :]


def prepare(opt, current_iter, lq, gt, mixup=None):
    """one iteration's batch as the reference loop feeds optimize_parameters: progressive subset and crop, then the mixup (a Mixup,
    or None when train.mixing_augs.mixup is off) -> (lq, gt, phase)"""
    if ((opt.get("datasets") or {}).get("train") or {}).get("iters") is not None:
        lq, gt, j = progressive(opt, current_iter, lq, gt)
    else:
        j = 0
    if mixup is not None:
        gt, lq = mixup(gt, lq)
    return lq, gt, j
