"""Torch restatement of the GAN stage (test infrastructure): the U-Net discriminator with spectral normalisation of Real-ESRGAN and
basicsr's vanilla GANLoss, in any dtype and on any device, for vmambair_b200.gan to be checked against.

The discriminator is built from a layer table in the construction order the reference uses (conv0 .. conv9, each nn.Conv2d, conv1 ..
conv8 wrapped in torch.nn.utils.spectral_norm), so a seeded construction and the state_dict are the reference's.  Its forward is
composed from F.leaky_relu(0.2) and F.interpolate(scale_factor=2, mode='bilinear', align_corners=False); torch's bilinear backward
has no deterministic CUDA implementation, so this module cannot run backward under torch.use_deterministic_algorithms(True).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn
from torch.nn.utils import spectral_norm

# name -> (in, out) in units of (num_in_ch | num_feat), kernel, stride, bias, spectral norm; the encoder halves the size three times
_TABLE = [
    ("conv0", ("in", 1), 3, 1, True, False),
    ("conv1", (1, 2), 4, 2, False, True),
    ("conv2", (2, 4), 4, 2, False, True),
    ("conv3", (4, 8), 4, 2, False, True),
    ("conv4", (8, 4), 3, 1, False, True),
    ("conv5", (4, 2), 3, 1, False, True),
    ("conv6", (2, 1), 3, 1, False, True),
    ("conv7", (1, 1), 3, 1, False, True),
    ("conv8", (1, 1), 3, 1, False, True),
    ("conv9", (1, "out"), 3, 1, True, False),
]


class UNetDiscriminatorSNRef(nn.Module):
    def __init__(self, num_in_ch, num_feat=64, skip_connection=True):
        super().__init__()
        self.skip_connection = skip_connection
        width = lambda m: num_in_ch if m == "in" else 1 if m == "out" else m * num_feat
        for name, (ci, co), k, s, bias, sn in _TABLE:
            conv = nn.Conv2d(width(ci), width(co), k, s, 1, bias=bias)
            setattr(self, name, spectral_norm(conv) if sn else conv)

    def forward(self, x):
        act = lambda t: F.leaky_relu(t, negative_slope=0.2)
        up = lambda t: F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=False)
        join = lambda t, s: t + s if self.skip_connection else t
        e0 = act(self.conv0(x))
        e1 = act(self.conv1(e0))
        e2 = act(self.conv2(e1))
        e3 = act(self.conv3(e2))
        d4 = join(act(self.conv4(up(e3))), e2)
        d5 = join(act(self.conv5(up(d4))), e1)
        d6 = join(act(self.conv6(up(d5))), e0)
        return self.conv9(act(self.conv8(act(self.conv7(d6)))))


SN_LAYERS = [name for name, *_, sn in _TABLE if sn]


def sn_state(net):
    """{layer: (u, v, sigma)} of the spectral-normalised layers as they stand (sigma = u . (W_orig v), no power iteration)"""
    out = {}
    for name in SN_LAYERS:
        m = getattr(net, name)
        w = m.weight_orig.detach().reshape(m.weight_orig.shape[0], -1)
        out[name] = (m.weight_u.clone(), m.weight_v.clone(), torch.dot(m.weight_u, w @ m.weight_v))
    return out


def gan_loss(input, target_is_real, is_disc=False, real_label_val=1.0, fake_label_val=0.0, loss_weight=1.0):
    """basicsr GANLoss(gan_type='vanilla').forward"""
    label = real_label_val if target_is_real else fake_label_val
    loss = F.binary_cross_entropy_with_logits(input, torch.full_like(input, label))
    return loss if is_disc else loss * loss_weight


def recipe_iteration(net_d, fake, real, loss_weight=1.0, loss=gan_loss):
    """The discriminator's part of one MambaRealSRGAN iteration (RealSR/VmambaIR/models/MambaRealSRGAN_model.py:289-359), three
    train-mode calls: (1) on G's output with D frozen, l_g_gan backpropagated into the output only; (2) on the GT and (3) on the
    detached output, both backpropagated into D's parameters, which accumulate.  -> a list of three dicts with the call's logits,
    the fake's gradient (call 1), the parameter gradients so far (calls 2, 3) and every SN layer's u / v after the call.  `loss`
    takes gan_loss's (input, target_is_real, is_disc, loss_weight=...) arguments."""
    calls = []
    uv = lambda: {f"{n}.{b}": getattr(net_d, n).get_buffer(f"weight_{b}").detach().clone() for n in SN_LAYERS for b in "uv"}
    net_d.train()
    for p in net_d.parameters():
        p.requires_grad_(False)
    fake = fake.detach().requires_grad_()
    pred = net_d(fake)
    loss(pred, True, is_disc=False, loss_weight=loss_weight).backward()
    calls.append({"logits": pred.detach(), "dfake": fake.grad.detach().clone(), **uv()})
    for p in net_d.parameters():
        p.requires_grad_(True)
    for inp, is_real in ((real, True), (fake.detach(), False)):
        pred = net_d(inp)
        loss(pred, is_real, is_disc=True).backward()
        grads = {f"grad.{n}": p.grad.detach().clone() for n, p in net_d.named_parameters()}
        calls.append({"logits": pred.detach(), **grads, **uv()})
    return calls
