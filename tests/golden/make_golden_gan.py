#!/usr/bin/env python
"""Generate tests/golden/gan_ref.npz from the REAL reference's UNetDiscriminatorSN (RealSR/VmambaIR/archs/discriminator_arch.py),
in float64 on the CPU, under a seed.  Runs on a development machine with the reference checkout (../reference or
$VMB_REFERENCE_DIR); no test imports it.

  python tests/golden/make_golden_gan.py

Nothing is copied from the reference: its module is imported at run time with the basicsr registry stubbed (make_golden.py).  The
loss is F.binary_cross_entropy_with_logits, which is what basicsr's vanilla GANLoss computes.  At B = 2, 3 x 24 x 40, num_feat 4:
  init.<key>        the seeded initial state_dict, as constructed (float32; skip_connection does not change it)
  x, gt             the generator output and the ground truth
and per skip_connection value (prefix skip0. / skip1.):
  c<i>.<what>       the three calls of the recipe iteration (oracle/gan_ref.recipe_iteration): logits, dfake (call 0), the
                    parameter gradients so far (calls 1, 2), the u / v of every SN layer after the call
  eval.logits       an eval-mode forward afterwards (u / v unchanged)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import make_golden as mg  # noqa: E402
from oracle import gan_ref  # noqa: E402

SEED, B, H, W, NF = 7, 2, 24, 40, 4


def main():
    mg.install_stubs()
    ref = mg.load_file("vmb_ref_discriminator_arch", f"{mg.REF}/RealSR/VmambaIR/archs/discriminator_arch.py")
    g = torch.Generator().manual_seed(SEED + 1)
    x = torch.randn(B, 3, H, W, generator=g, dtype=torch.float64)
    gt = torch.rand(B, 3, H, W, generator=g, dtype=torch.float64)
    out = {"x": x.numpy(), "gt": gt.numpy()}
    for skip in (True, False):
        tag = f"skip{int(skip)}"
        torch.manual_seed(SEED)
        net = ref.UNetDiscriminatorSN(3, num_feat=NF, skip_connection=skip)
        init = {f"init.{k}": v.detach().numpy().copy() for k, v in net.state_dict().items()}
        assert all(np.array_equal(v, out.get(k, v)) for k, v in init.items())
        out.update(init)
        net = net.double()
        for i, call in enumerate(gan_ref.recipe_iteration(net, x, gt)):
            out.update({f"{tag}.c{i}.{k}": v.numpy() for k, v in call.items()})
        net.eval()
        with torch.no_grad():
            out[f"{tag}.eval.logits"] = net(x).numpy()
    path = os.path.join(HERE, "gan_ref.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
