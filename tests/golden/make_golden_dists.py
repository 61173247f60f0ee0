#!/usr/bin/env python
"""Generate tests/golden/dists_ref.npz from the REAL reference's DISTS (RealSR/Metric/dists.py), in float64 on the CPU.  Runs on a
development machine with the reference checkout (../reference or $VMB_REFERENCE_DIR); no test imports it.

  python tests/golden/make_golden_dists.py

Nothing is copied from the reference: its module is imported at run time, with `models.vgg16` replaced by
torchvision.models.vgg16(weights=None) (the pretrained download is not available).  The trunk then gets the seeded weights of
oracle.lpips_ref.seeded_vgg16_convs(VGG_SEED); only the seed and a checksum per tensor are stored.
  keys, shapes             the state_dict key list and shapes of DISTS(load_weights=False)
  seed_alpha, seed_beta    alpha and beta of DISTS(load_weights=False) constructed after torch.manual_seed(SEED) (float32)
  real_alpha, real_beta    the reference's Metric/DISTS/DISTS_pytorch/weights.pt (float32)
  vgg_seed, vgg_checksums  VGG_SEED and oracle.lpips_ref.checksums of the trunk
  x_<s>, y_<s>             the input pairs (float32 in [0, 1], upcast for the run), s = a (2 x 3 x 40 x 56), b (1 x 3 x 33 x 47)
  score_<w>_<s>            the reference's forward(x, y) (batch_average=False) with the <w> = real / seed alpha and beta
  feat_<s>                 per feature of forward_once(x_<s>): (sum, sum of squares), to localise a trunk mismatch
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch
import torchvision

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.lpips_ref import checksums, seeded_vgg16_convs  # noqa: E402

REF = os.environ.get("VMB_REFERENCE_DIR") or os.path.join(os.path.dirname(ROOT), "reference")
SEED, VGG_SEED, INPUT_SEED = 5, 11, 3
SHAPES = {"a": (2, 3, 40, 56), "b": (1, 3, 33, 47)}
CONV_INDEX = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
STAGE_STARTS = (0, 4, 9, 16, 23, 30)


def load_reference():
    spec = importlib.util.spec_from_file_location("vmb_ref_dists", f"{REF}/RealSR/Metric/dists.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.models = types.SimpleNamespace(vgg16=lambda pretrained=True: torchvision.models.vgg16(weights=None))
    return mod


def main():
    ref = load_reference()
    torch.manual_seed(SEED)
    net = ref.DISTS(load_weights=False)
    sd = net.state_dict()
    out = {"keys": np.array(list(sd)), "shapes": np.array([str(tuple(v.shape)) for v in sd.values()]),
           "seed_alpha": net.alpha.detach().numpy().copy(), "seed_beta": net.beta.detach().numpy().copy()}
    real = torch.load(f"{REF}/RealSR/Metric/DISTS/DISTS_pytorch/weights.pt", map_location="cpu", weights_only=True)
    out["real_alpha"], out["real_beta"] = real["alpha"].numpy(), real["beta"].numpy()
    convs = seeded_vgg16_convs(VGG_SEED)
    out["vgg_seed"], out["vgg_checksums"] = np.int64(VGG_SEED), checksums(convs).numpy()
    with torch.no_grad():
        for i, (w, b) in zip(CONV_INDEX, convs):
            k = next(k for k in range(5) if STAGE_STARTS[k] <= i < STAGE_STARTS[k + 1]) + 1
            getattr(net, f"stage{k}")[i - STAGE_STARTS[k - 1]].weight.copy_(w)
            getattr(net, f"stage{k}")[i - STAGE_STARTS[k - 1]].bias.copy_(b)
    net = net.double().eval()
    g = torch.Generator().manual_seed(INPUT_SEED)
    for s, shape in SHAPES.items():
        x, y = torch.rand(shape, generator=g), torch.rand(shape, generator=g)
        out[f"x_{s}"], out[f"y_{s}"] = x.numpy(), y.numpy()
        for w in ("real", "seed"):
            with torch.no_grad():
                net.alpha.copy_(torch.from_numpy(out[f"{w}_alpha"]).double())
                net.beta.copy_(torch.from_numpy(out[f"{w}_beta"]).double())
            out[f"score_{w}_{s}"] = net(x.double(), y.double()).detach().numpy()
        with torch.no_grad():
            out[f"feat_{s}"] = np.array([[f.sum().item(), (f * f).sum().item()] for f in net.forward_once(x.double())])
    path = os.path.join(HERE, "dists_ref.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
