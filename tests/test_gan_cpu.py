"""The GAN stage on the CPU: the torch restatement (oracle/gan_ref.py) against float64 outputs of the reference's UNetDiscriminatorSN
(tests/golden/gan_ref.npz, make_golden_gan.py), state_dict compatibility of the drop-in, and the vanilla GAN loss."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import gan_ref
from vmambair_b200 import checkpoint, gan

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gan_ref.npz")
SEED, NF = 7, 4  # make_golden_gan.py


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as f:
        return {k: f[k] for k in f.files}


def _init(golden):
    return {k[5:]: torch.from_numpy(v) for k, v in golden.items() if k.startswith("init.")}


@pytest.mark.parametrize("cls", [gan.UNetDiscriminatorSN, gan_ref.UNetDiscriminatorSNRef])
@pytest.mark.parametrize("skip", [True, False])
def test_seeded_construction_is_the_references(golden, cls, skip):
    torch.manual_seed(SEED)
    sd = cls(3, num_feat=NF, skip_connection=skip).state_dict()
    init = _init(golden)
    assert list(sd) == list(init)
    for k, v in init.items():
        assert sd[k].shape == v.shape and torch.equal(sd[k], v), k


@pytest.mark.parametrize("skip", [True, False])
def test_restatement_reproduces_the_reference(golden, skip):
    net = gan_ref.UNetDiscriminatorSNRef(3, num_feat=NF, skip_connection=skip)
    net.load_state_dict(_init(golden))
    net = net.double()
    x, gt = torch.from_numpy(golden["x"]), torch.from_numpy(golden["gt"])
    tag = f"skip{int(skip)}"
    calls = gan_ref.recipe_iteration(net, x, gt)
    n = 0
    for i, call in enumerate(calls):
        for k, v in call.items():
            ref = torch.from_numpy(golden[f"{tag}.c{i}.{k}"])
            err = (v - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)
            assert err <= 1e-12, (i, k, err)
            n += 1
    assert n == len([k for k in golden if k.startswith(tag + ".c")])
    net.eval()
    with torch.no_grad():
        y = net(x)
    ref = torch.from_numpy(golden[f"{tag}.eval.logits"])
    assert (y - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()
    for name in gan_ref.SN_LAYERS:  # eval mode: no power iteration
        for b in "uv":
            assert torch.equal(getattr(net, name).get_buffer(f"weight_{b}"), torch.from_numpy(golden[f"{tag}.c2.{name}.{b}"]))


def test_state_dict_round_trips_with_strict_loading(tmp_path):
    torch.manual_seed(1)
    ours = gan.UNetDiscriminatorSN(3, num_feat=8)
    torch.manual_seed(2)
    theirs = gan_ref.UNetDiscriminatorSNRef(3, num_feat=8)
    p1, p2 = str(tmp_path / "net_d_ours.pth"), str(tmp_path / "net_d_ref.pth")
    checkpoint.save_network(ours, p1)
    checkpoint.save_network(theirs, p2)
    a = gan_ref.UNetDiscriminatorSNRef(3, num_feat=8)
    checkpoint.load_network(a, p1, strict=True)
    b = gan.UNetDiscriminatorSN(3, num_feat=8)
    checkpoint.load_network(b, p2, strict=True)
    for k, v in ours.state_dict().items():
        assert torch.equal(a.state_dict()[k], v), k
    for k, v in theirs.state_dict().items():
        assert torch.equal(b.state_dict()[k], v), k
    keys = set(ours.state_dict())
    want = {"conv0.weight", "conv0.bias", "conv9.weight", "conv9.bias"} | \
        {f"conv{k}.weight_{s}" for k in range(1, 9) for s in ("orig", "u", "v")}
    assert keys == want


@pytest.mark.parametrize("real", [True, False])
@pytest.mark.parametrize("is_disc", [True, False])
def test_vanilla_gan_loss_restates_bce_with_logits(real, is_disc):
    x = torch.randn(2, 1, 8, 8, dtype=torch.float64) * 5
    x[0, 0, 0, :2] = torch.tensor([80.0, -80.0])
    t = 0.9 if real else 0.1
    y = gan_ref.gan_loss(x, real, is_disc, real_label_val=0.9, fake_label_val=0.1, loss_weight=0.5)
    per = torch.clamp(x, min=0) - x * t + torch.log1p(torch.exp(-x.abs()))
    want = per.mean() * (1.0 if is_disc else 0.5)
    assert torch.isfinite(y) and abs(y.item() - want.item()) <= 1e-14
    assert torch.allclose(y, F.binary_cross_entropy_with_logits(x, torch.full_like(x, t)) * (1.0 if is_disc else 0.5))


def test_gan_loss_types_and_devices():
    with pytest.raises(NotImplementedError):
        gan.GANLoss("lsgan")
    with pytest.raises(ValueError):
        gan.GANLoss("vanilla")(torch.zeros(1, 1, 8, 8), True)


def test_discriminator_rejects_cpu_input():
    with pytest.raises(ValueError):
        gan.UNetDiscriminatorSN(3, num_feat=4)(torch.zeros(1, 3, 16, 16))
