"""The GAN recipes' perceptual loss: a drop-in for basicsr's `PerceptualLoss` (basicsr/losses/basic_loss.py) on its
`VGGFeatureExtractor` (basicsr/archs/vgg_arch.py), the generator step's `perceptual_opt` in RealSR/options/mambaSR11GAN_x4.yml and
SRGAN/options/MambaSISR15GAN_x4.yml.

The module holds basicsr's state (`vgg.mean`, `vgg.std`, `vgg.vgg_net.<layer name>.weight|bias`, torchvision's VGG `features` cut
after the deepest requested layer, frozen), and its forward never calls the sub-modules: the whole loss is one autograd Function.
Output and ground truth run as one 2B batch.  Each convolution is one cuDNN call over the batch; everything between them is
csrc/perceptual.cu: the input normalisation, per convolution one stage kernel (in-place ReLU fused with the following max-pool, the
criterion's per-CTA partials at the feature layers, and for the output half a byte per 2 x 2 cell of ReLU mask and pool argmax plus
the sign (l1) or the difference (l2, fro) at the feature layers), and the loss in one CTA.  The backward computes data gradients only,
down to the output: per stage one kernel builds the gradient at the convolution's output from those bits and injects the loss
gradient, then cuDNN's data gradient of the convolution.  No atomics and no host synchronisation: a forward + backward is bitwise
reproducible and can be captured in a CUDA graph.
"""
from __future__ import annotations

import os
from collections import OrderedDict

import torch
from torch import nn

from . import ops

_BLOCKS = {"vgg11": (1, 1, 2, 2, 2), "vgg13": (2, 2, 2, 2, 2), "vgg16": (2, 2, 3, 3, 3), "vgg19": (2, 2, 4, 4, 4)}


def layer_names(vgg_type):
    """basicsr's names of torchvision's VGG `features`, in index order: conv{i}_{j}, relu{i}_{j}, ..., pool{i}"""
    names = []
    for i, n in enumerate(_BLOCKS[vgg_type], 1):
        for j in range(1, n + 1):
            names += [f"conv{i}_{j}", f"relu{i}_{j}"]
        names.append(f"pool{i}")
    return names


def weights_file_name(vgg_type):
    """torchvision's file name of the ImageNet weights, e.g. vgg19-dcbb9e9d.pth"""
    import torchvision
    return os.path.basename(torchvision.models.get_model_weights(vgg_type).IMAGENET1K_V1.url)


def find_weights(vgg_type, who="PerceptualLoss"):
    """basicsr's lookup of the pretrained weights, without the download: experiments/pretrained_models/<file>, then the torch hub
    cache's checkpoints/<file>; `who` names the caller in the error"""
    name = weights_file_name(vgg_type)
    paths = [os.path.join("experiments", "pretrained_models", name), os.path.join(torch.hub.get_dir(), "checkpoints", name)]
    for p in paths:
        if os.path.isfile(p):
            return p
    raise FileNotFoundError(f"{who}: the {vgg_type} weights are in neither {paths[0]} nor {paths[1]}; place "
                            f"torchvision's {name} there, or pass weights=<path> (nothing is downloaded)")


class _VGGFeatureExtractor(nn.Module):
    """basicsr's VGGFeatureExtractor state: the VGG `features` up to the deepest requested layer under basicsr's layer names, frozen
    and in eval mode, and the ImageNet mean / std buffers when use_input_norm"""

    def __init__(self, layer_name_list, vgg_type, use_input_norm, range_norm, weights):
        super().__init__()
        import torchvision
        self.layer_name_list = list(layer_name_list)
        self.use_input_norm, self.range_norm = use_input_norm, range_norm
        self.names = layer_names(vgg_type)
        for v in self.layer_name_list:
            if v not in self.names:
                raise ValueError(f"PerceptualLoss: {v!r} is not a layer of {vgg_type} ({', '.join(self.names)})")
        max_idx = max(self.names.index(v) for v in self.layer_name_list)
        features = getattr(torchvision.models, vgg_type)(weights=None).features[:max_idx + 1]
        if weights == "auto":
            weights = find_weights(vgg_type)
        if weights is not None:
            sd = torch.load(weights, map_location="cpu", weights_only=True)
            sub = {k[len("features."):]: v for k, v in sd.items() if k.startswith("features.")}
            missing = [k for k in features.state_dict() if k not in sub]
            if missing:
                raise KeyError(f"PerceptualLoss: {weights} lacks {', '.join('features.' + k for k in missing)}")
            features.load_state_dict({k: sub[k] for k in features.state_dict()})
        net = OrderedDict()
        for k, v in zip(self.names, features):
            net[k] = nn.MaxPool2d(kernel_size=2, stride=2) if k.startswith("pool") else v
        self.vgg_net = nn.Sequential(net)
        self.vgg_net.eval()
        for p in self.parameters():
            p.requires_grad = False
        if use_input_norm:
            self.register_buffer("mean", torch.Tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1))
            self.register_buffer("std", torch.Tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1))

    def stages(self):
        """per convolution: (conv module, relu follows, pool follows, (conv, relu, pool) site names) within the cut network"""
        names = list(self.vgg_net._modules)
        out = []
        for i, k in enumerate(names):
            if not k.startswith("conv"):
                continue
            relu = i + 1 < len(names) and names[i + 1].startswith("relu")
            pool = relu and i + 2 < len(names) and names[i + 2].startswith("pool")
            out.append((self.vgg_net[i], relu, pool, (k, names[i + 1] if relu else None, names[i + 2] if pool else None)))
        return out


def _conv(h, w, b):
    return torch.ops.aten.convolution(h, w, b, [1, 1], [1, 1], [1, 1], False, [0, 0], 1).contiguous()


class _Perceptual(torch.autograd.Function):
    """(plan, x, gt) -> perceptual loss (0-dim fp32); the gradient reaches x only"""

    @staticmethod
    def forward(ctx, plan, x, gt):
        dt, crit, save = plan["dtype"], plan["crit"], plan["save"]
        with torch.autocast("cuda", enabled=False):
            h = ops.percep_norm(x, gt, plan["mean"], plan["std"], plan["range_norm"], dt)
            partial = torch.empty(plan["parts"], dtype=torch.float32, device=x.device)
            kept = []
            for st, (w, b) in zip(plan["stages"], plan["weights"]):
                y = _conv(h, w, b)
                parts = [partial[o:o + st["ctas"]] if f else None for f, o in zip(st["feat"], st["offset"])]
                pooled, code, saves = ops.percep_stage(y, st["relu"], st["pool"], st["feat"], parts, crit, save)
                kept += [code, *saves]
                h = pooled if st["pool"] else y
            loss, value = ops.percep_loss(partial, plan["offsets"], plan["numels"], plan["layer_weights"], crit,
                                          plan["perceptual_weight"])
        ctx.plan = plan
        ctx.save_for_backward(value, *kept)
        return loss

    @staticmethod
    def backward(ctx, g):
        plan = ctx.plan
        dt = plan["dtype"]
        value, *kept = ctx.saved_tensors
        g = g.float().contiguous()
        with torch.autocast("cuda", enabled=False):
            gin = None
            for i in reversed(range(len(plan["stages"]))):
                st, (w, _) = plan["stages"][i], plan["weights"][i]
                code, saves = kept[4 * i], kept[4 * i + 1:4 * i + 4]
                gout = ops.percep_stage_bwd(gin, code, saves, st["feat"], st["feat_index"], st["scale"], g, value, st["out_shape"],
                                            st["relu"], st["pool"], plan["crit"], dt)
                empty = gout.new_empty(1).expand(st["in_shape"])
                gin = torch.ops.aten.convolution_backward(gout, empty, w, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1,
                                                          [True, False, False])[0].contiguous()
            dx = ops.percep_norm_bwd(gin, plan["std"], plan["range_norm"])
        return None, dx, None


class PerceptualLoss(nn.Module):
    """basicsr's PerceptualLoss: perceptual_weight * sum_k layer_weights[k] * criterion(vgg_k(x), vgg_k(gt)), gt detached.

    Args:
        layer_weights (dict): basicsr layer name (conv*_*, relu*_*, pool*) -> weight.  A conv feature is taken before its ReLU.
        vgg_type (str): 'vgg11', 'vgg13', 'vgg16' or 'vgg19' ('_bn' types raise NotImplementedError).
        use_input_norm (bool): normalise by the ImageNet mean / std.  range_norm (bool): map [-1, 1] to [0, 1] first.
        perceptual_weight (float): 0 returns None as the perceptual loss.
        style_weight (float): must be 0 (the Gram-matrix style loss raises NotImplementedError).
        criterion (str): 'l1', 'l2' (means over each feature) or 'fro' (Frobenius norm of each feature's difference).
        weights: 'auto' (experiments/pretrained_models/<torchvision file>, then the torch hub cache's checkpoints/<file>; never
            downloaded), a path to a torchvision VGG state_dict, or None for torchvision's random initialisation.

    forward(x, gt) -> (percep_loss, style_loss): 0-dim fp32 tensors or None.  x and gt are CUDA float32 (B, 3, H, W) of one shape,
    H and W at least 2 ** (pools up to the deepest layer); under torch.autocast("cuda", torch.bfloat16) the activations are bf16."""

    def __init__(self, layer_weights, vgg_type="vgg19", use_input_norm=True, range_norm=False, perceptual_weight=1.0,
                 style_weight=0.0, criterion="l1", weights="auto"):
        super().__init__()
        if style_weight > 0:
            raise NotImplementedError("PerceptualLoss: style_weight > 0 (the Gram-matrix style loss) is not implemented; no recipe "
                                      "uses it")
        if vgg_type.endswith("_bn"):
            raise NotImplementedError(f"PerceptualLoss: {vgg_type} (VGG with batch norm) is not implemented; no recipe uses it")
        if vgg_type not in _BLOCKS:
            raise ValueError(f"PerceptualLoss: unknown vgg_type {vgg_type!r}")
        if criterion not in ops.PERCEP_CRIT:
            raise NotImplementedError(f"{criterion} criterion has not been supported.")
        self.perceptual_weight, self.style_weight = perceptual_weight, style_weight
        self.layer_weights = dict(layer_weights)
        self.criterion_type = criterion
        self.vgg = _VGGFeatureExtractor(list(layer_weights.keys()), vgg_type, use_input_norm, range_norm, weights)
        self._cache = None

    def _weights(self, dt, dev):
        """the convolutions' (weight, bias) in the conv dtype; the bf16 copies are cached by parameter version"""
        convs = [m for m, *_ in self.vgg.stages()]
        if dt == torch.float32:
            return [(m.weight, m.bias) for m in convs]
        ps = [p for m in convs for p in (m.weight, m.bias)]
        ver = (dt, dev, tuple(p._version for p in ps), tuple(p.data_ptr() for p in ps))
        if self._cache is None or self._cache[0] != ver:
            self._cache = (ver, [(m.weight.detach().to(dt), m.bias.detach().to(dt)) for m in convs])
        return self._cache[1]

    def _plan(self, x, dt, save):
        B, _, H, W = x.shape
        pw = float(self.perceptual_weight)
        stages, offsets, numels, lw, parts = [], [0], [], [], 0
        h, w, cin = H, W, 3
        for m, relu, pool, sites in self.vgg.stages():
            c = m.out_channels
            ctas = ops.percep_stage_ctas(B, c, h, w)
            st = dict(relu=relu, pool=pool, ctas=ctas, in_shape=(B, cin, h, w), out_shape=(B, c, h, w), feat=[0, 0, 0],
                      feat_index=[-1, -1, -1], scale=[0.0, 0.0, 0.0], offset=[0, 0, 0])
            for k, name in enumerate(sites):
                if name is None or name not in self.layer_weights:
                    continue
                n = B * c * (h // 2) * (w // 2) if k == 2 else B * c * h * w
                wk = float(self.layer_weights[name])
                st["feat"][k], st["feat_index"][k], st["offset"][k] = 1, len(numels), parts
                st["scale"][k] = pw * wk if self.criterion_type == "fro" else (2.0 if self.criterion_type == "l2" else 1.0) * pw * wk / n
                parts += ctas
                offsets.append(parts)
                numels.append(n)
                lw.append(wk)
            stages.append(st)
            if pool:
                h, w = h // 2, w // 2
            cin = c
        return dict(dtype=dt, crit=self.criterion_type, save=save, range_norm=self.vgg.range_norm,
                    mean=getattr(self.vgg, "mean", None), std=getattr(self.vgg, "std", None), stages=stages,
                    weights=self._weights(dt, x.device), parts=parts, offsets=offsets, numels=numels, layer_weights=lw,
                    perceptual_weight=pw)

    def forward(self, x, gt):
        if self.perceptual_weight == 0:
            return None, None
        pools = sum(1 for k in self.vgg.vgg_net._modules if k.startswith("pool"))
        for name, t in (("x", x), ("gt", gt)):
            if not isinstance(t, torch.Tensor) or t.dim() != 4 or t.shape[1] != 3:
                raise ValueError(f"PerceptualLoss: {name} must be a (B, 3, H, W) tensor, got {getattr(t, 'shape', type(t))}")
            if t.dtype != torch.float32:
                raise ValueError(f"PerceptualLoss: {name} must be float32, got {t.dtype}")
        if x.shape != gt.shape:
            raise ValueError(f"PerceptualLoss: x {tuple(x.shape)} and gt {tuple(gt.shape)} differ")
        if x.shape[0] == 0 or min(x.shape[2], x.shape[3]) < 2 ** pools:
            raise ValueError(f"PerceptualLoss: H and W must be at least {2 ** pools} for {pools} pools (and B at least 1), got "
                             f"{tuple(x.shape)}")
        dev = self.vgg.vgg_net[0].weight.device
        if not x.is_cuda or x.device != gt.device or x.device != dev:
            raise ValueError(f"PerceptualLoss runs on CUDA: x on {x.device}, gt on {gt.device}, the VGG on {dev}")
        dt = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else torch.float32
        if dt != torch.float32 and dt != torch.bfloat16:
            raise ValueError(f"PerceptualLoss runs in float32 or under bfloat16 autocast, not {dt}")
        plan = self._plan(x, dt, torch.is_grad_enabled() and x.requires_grad)
        return _Perceptual.apply(plan, x, gt.detach()), None


__all__ = ["PerceptualLoss", "layer_names"]
