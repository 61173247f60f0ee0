"""Drop-in OSS modules and networks (same class names, ctor kwargs, forward() signatures and
state_dict keys/shapes as the reference archs), running on the sm_90a kernels of this repo.

Reference classes mirrored (file:line in the reference project):
  LayerNorm / WithBias_LayerNorm / BiasFree_LayerNorm   SRGAN/VmambaIR/archs/MambaSISR6_arch.py:149-195
  FeedForward (EFFN)                                     MambaSISR6_arch.py:201-218
  SS2D_1 (OSS module)                                    MambaSISR6_arch.py:222-498 (SISR)
                                                         Deraining/basicsr/models/archs/mamber32_arch.py:219-494 (additive channel gate)
                                                         Deraining/basicsr/models/archs/mamber33_arch.py (dc_inner=2)
                                                         RealSR/VmambaIR/archs/MambaRealSR11_arch.py:547-832 (dc_inner=1, rank=dt_rank)
  MamberBlock                                            MambaSISR6_arch.py:502-515
  MambaSISR6 / MambaRealSR11 / Mamber32 / Mamber33       MambaSISR6_arch.py:557-643, MambaRealSR11_arch.py:891-974,
                                                         mamber32_arch.py:554-649, mamber33_arch.py
  Upsampler / default_conv (SR tail)                     SRGAN/VmambaIR/archs/common.py:7-8,45-60

Two execution paths share the parameters:
  * `fused`  (CUDA, no-grad calls): the hand-written kernels (vmambair_b200.fused) -- if the CUDA library is missing a
    RuntimeError is raised; shapes outside the kernels' limits (fused.unsupported_reason) take `compose` with a warning;
  * `fused_train` (CUDA, grad enabled; default): the fused stages with their hand-written backward kernels
    (vmambair_b200.fused_train);
  * `compose`: the same math composed from torch ops + this repo's selective-scan operator with autograd
    (VMB_TRAIN_PATH=compose / set_train_path; the module-level cross-check and the fallback for unsupported shapes).
"""
from __future__ import annotations

import math
import numbers
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from .selective_scan import selective_scan_fn

# training path: "fused" = fused_train (native forward + backward kernels); "compose" = torch ops + the scan operator (round 1)
_TRAIN_PATH = os.environ.get("VMB_TRAIN_PATH", "fused")


def set_train_path(path: str) -> None:
    global _TRAIN_PATH
    assert path in ("fused", "compose")
    _TRAIN_PATH = path


VARIANTS = {
    # name: (dc_inner, channel rank ("dt_rank" -> same as dt_rank), has conv_cin/cout, gate)
    "sisr": (4, 6, True, "mul"),       # MambaSISR6_arch.py:263-267,494-496
    "mamber32": (4, 6, True, "add"),   # mamber32_arch.py:260,490-492
    "mamber33": (2, 6, True, "mul"),   # mamber33_arch.py:257,487-490
    "realsr": (1, "dt_rank", False, "mul"),  # MambaRealSR11_arch.py:589,628,645,806-817
}


# ----------------------------------------------------------------------------- LayerNorm
class BiasFree_LayerNorm(nn.Module):
    def __init__(self, normalized_shape):
        super().__init__()
        if isinstance(normalized_shape, numbers.Integral):
            normalized_shape = (normalized_shape,)
        assert len(normalized_shape) == 1
        self.weight = nn.Parameter(torch.ones(normalized_shape))
        self.normalized_shape = torch.Size(normalized_shape)

    def forward(self, x):  # x: (b, hw, c)
        sigma = x.var(-1, keepdim=True, unbiased=False)
        return x / torch.sqrt(sigma + 1e-5) * self.weight


class WithBias_LayerNorm(nn.Module):
    def __init__(self, normalized_shape):
        super().__init__()
        if isinstance(normalized_shape, numbers.Integral):
            normalized_shape = (normalized_shape,)
        assert len(normalized_shape) == 1
        self.weight = nn.Parameter(torch.ones(normalized_shape))
        self.bias = nn.Parameter(torch.zeros(normalized_shape))
        self.normalized_shape = torch.Size(normalized_shape)

    def forward(self, x):
        mu = x.mean(-1, keepdim=True)
        sigma = x.var(-1, keepdim=True, unbiased=False)
        return (x - mu) / torch.sqrt(sigma + 1e-5) * self.weight + self.bias


class LayerNorm(nn.Module):
    """Per-pixel LayerNorm over channels of a (b,c,h,w) tensor."""

    def __init__(self, dim, LayerNorm_type):
        super().__init__()
        self.body = BiasFree_LayerNorm(dim) if LayerNorm_type == "BiasFree" else WithBias_LayerNorm(dim)

    def forward(self, x):
        b, c, h, w = x.shape
        y = self.body(x.flatten(2).transpose(1, 2))
        return y.transpose(1, 2).reshape(b, c, h, w).to(x.dtype)


# ----------------------------------------------------------------------------- EFFN
class FeedForward(nn.Module):
    def __init__(self, dim, ffn_expansion_factor, bias):
        super().__init__()
        hidden = int(dim * ffn_expansion_factor)
        self.project_in = nn.Conv2d(dim, hidden * 2, kernel_size=1, bias=bias)
        self.dwconv = nn.Conv2d(hidden * 2, hidden * 2, kernel_size=3, stride=1, padding=1, groups=hidden * 2, bias=bias)
        self.project_out = nn.Conv2d(hidden, dim, kernel_size=1, bias=bias)

    def forward(self, x):
        x = self.project_in(x)
        x1, x2 = self.dwconv(x).chunk(2, dim=1)
        return self.project_out(F.gelu(x1) * x2)


# ----------------------------------------------------------------------------- OSS module
class SS2D_1(nn.Module):
    def __init__(self, d_model=96, d_state=16, ssm_ratio=2.0, ssm_rank_ratio=2.0, dt_rank="auto", act_layer=nn.SiLU,
                 d_conv=3, conv_bias=True, dropout=0.0, bias=False, dt_min=0.001, dt_max=0.1, dt_init="random",
                 dt_scale=1.0, dt_init_floor=1e-4, simple_init=False, softmax_version=False, forward_type="v2",
                 variant="sisr", **kwargs):
        super().__init__()
        if softmax_version or forward_type != "v2" or d_conv != 3:
            raise NotImplementedError("only the configuration every VmambaIR arch uses is built: "
                                      "softmax_version=False, forward_type='v2', d_conv=3")
        self.variant = variant
        dc_inner, rankc, has_cio, self.gate = VARIANTS[variant]
        d_expand = int(ssm_ratio * d_model)
        d_inner = int(min(ssm_rank_ratio, ssm_ratio) * d_model) if ssm_rank_ratio > 0 else d_expand
        if d_inner != d_expand:
            raise NotImplementedError("ssm_low_rank (d_inner < d_expand) is not used by any VmambaIR arch")
        self.d_model, self.d_inner = d_model, d_inner
        self.dt_rank = math.ceil(d_model / 16) if dt_rank == "auto" else dt_rank
        self.d_state = math.ceil(d_model / 6) if d_state == "auto" else d_state
        self.d_conv = d_conv
        self.dc_inner = dc_inner
        self.dtc_rank = self.dt_rank if rankc == "dt_rank" else rankc
        self.dc_state = 16 if variant != "realsr" else self.d_state
        self.K, self.KC = 4, 2
        self.softmax_version = False

        if has_cio:
            self.conv_cin = nn.Conv2d(1, dc_inner, kernel_size=1)
            self.conv_cout = nn.Conv2d(dc_inner, 1, kernel_size=1)
        self.pooling = nn.AdaptiveAvgPool2d(1)
        self.channel_norm = LayerNorm(d_inner, LayerNorm_type="WithBias")
        self.in_conv = nn.Conv2d(d_model, d_expand * 2, kernel_size=1)
        self.act = act_layer()
        self.conv2d = nn.Conv2d(d_expand, d_expand, groups=d_expand, bias=conv_bias, kernel_size=d_conv,
                                padding=(d_conv - 1) // 2)
        self.out_norm = LayerNorm(d_inner, LayerNorm_type="WithBias")

        R, N = self.dt_rank, self.d_state
        self.x_proj_weight = nn.Parameter(torch.stack(
            [nn.Linear(d_inner, R + 2 * N, bias=False).weight for _ in range(self.K)], dim=0))
        self.xc_proj_weight = nn.Parameter(torch.stack(
            [nn.Linear(dc_inner, self.dtc_rank + 2 * self.dc_state, bias=False).weight for _ in range(self.KC)], dim=0))
        dts = [self.dt_init(R, d_inner, dt_scale, dt_init, dt_min, dt_max, dt_init_floor) for _ in range(self.K)]
        self.dt_projs_weight = nn.Parameter(torch.stack([t.weight for t in dts], dim=0))
        self.dt_projs_bias = nn.Parameter(torch.stack([t.bias for t in dts], dim=0))
        self.A_logs = self.A_log_init(N, d_inner, copies=self.K)
        self.Ds = self.D_init(d_inner, copies=self.K)
        self.out_conv = nn.Conv2d(d_expand, d_model, kernel_size=1)
        self.dropout = nn.Dropout(dropout) if dropout > 0.0 else nn.Identity()
        if variant == "realsr":  # MambaRealSR11_arch.py:645-657
            dtc = [self.dt_init(R, 1, dt_scale, dt_init, dt_min, dt_max, dt_init_floor) for _ in range(self.KC)]
            self.dtc_projs_weight = nn.Parameter(torch.stack([t.weight for t in dtc], dim=0))
            self.dtc_projs_bias = nn.Parameter(torch.stack([t.bias for t in dtc], dim=0))
            self.Ac_logs = self.A_log_init(N, 1, copies=self.KC)
            self.Dsc = self.D_init(1, copies=self.KC)
        else:  # MambaSISR6_arch.py:332-335
            self.Dsc = nn.Parameter(torch.ones(self.KC * dc_inner))
            self.Ac_logs = nn.Parameter(torch.randn(self.KC * dc_inner, self.dc_state))
            self.dtc_projs_weight = nn.Parameter(torch.randn(self.KC, dc_inner, self.dtc_rank))
            self.dtc_projs_bias = nn.Parameter(torch.randn(self.KC, dc_inner))

    # -- parameter initialisers (reference :337-391) --------------------------------------
    @staticmethod
    def dt_init(dt_rank, d_inner, dt_scale=1.0, dt_init="random", dt_min=0.001, dt_max=0.1, dt_init_floor=1e-4):
        proj = nn.Linear(dt_rank, d_inner, bias=True)
        std = dt_rank ** -0.5 * dt_scale
        if dt_init == "constant":
            nn.init.constant_(proj.weight, std)
        elif dt_init == "random":
            nn.init.uniform_(proj.weight, -std, std)
        else:
            raise NotImplementedError
        dt = torch.exp(torch.rand(d_inner) * (math.log(dt_max) - math.log(dt_min)) + math.log(dt_min)).clamp(min=dt_init_floor)
        with torch.no_grad():
            proj.bias.copy_(dt + torch.log(-torch.expm1(-dt)))  # softplus^-1(dt)
        return proj

    @staticmethod
    def A_log_init(d_state, d_inner, copies=-1):
        A_log = torch.log(torch.arange(1, d_state + 1, dtype=torch.float32)).repeat(d_inner, 1)
        if copies > 0:
            A_log = A_log.repeat(copies, 1)
        p = nn.Parameter(A_log.contiguous())
        p._no_weight_decay = True
        return p

    @staticmethod
    def D_init(d_inner, copies=-1):
        p = nn.Parameter(torch.ones(d_inner * max(copies, 1)))
        p._no_weight_decay = True
        return p

    # -- composed path: torch ops + this repo's scan operator (autograd) ------------------
    def forward_core(self, x):
        B, C, H, W = x.shape
        L = H * W
        x_hwwh = torch.stack([x.flatten(2), x.transpose(2, 3).contiguous().flatten(2)], dim=1)
        xs = torch.cat([x_hwwh, x_hwwh.flip(-1)], dim=1)  # (B,4,C,L): row-major, col-major, and both reversed
        # the two per-direction projections as grouped 1x1 conv1d (same contraction as the reference einsums :409-411,
        # but cuDNN grouped kernels in forward and backward instead of strided batched GEMMs)
        K, RN = 4, self.dt_rank + 2 * self.d_state
        x_dbl = F.conv1d(xs.reshape(B, K * C, L), self.x_proj_weight.reshape(K * RN, C, 1), groups=K).view(B, K, RN, L)
        dts, Bs, Cs = torch.split(x_dbl, [self.dt_rank, self.d_state, self.d_state], dim=2)
        dts = F.conv1d(dts.reshape(B, K * self.dt_rank, L), self.dt_projs_weight.reshape(K * C, self.dt_rank, 1),
                       groups=K).view(B, K, C, L)
        out_y = selective_scan_fn(xs.reshape(B, -1, L), dts.reshape(B, -1, L), -torch.exp(self.A_logs.float()),
                                  Bs.contiguous(), Cs.contiguous(), self.Ds.float(),
                                  delta_bias=self.dt_projs_bias.reshape(-1).float(), delta_softplus=True).view(B, 4, C, L)
        inv_y = out_y[:, 2:4].flip(-1)
        wh_y = out_y[:, 1].view(B, C, W, H).transpose(2, 3).reshape(B, C, L)
        invwh_y = inv_y[:, 1].view(B, C, W, H).transpose(2, 3).reshape(B, C, L)
        y = out_y[:, 0].float() + inv_y[:, 0].float() + wh_y.float() + invwh_y.float()
        return self.out_norm(y.view(B, C, H, W)).to(x.dtype)

    def cforward_pooled(self, pooled):
        """channel-direction OSS on the pooled descriptor: pooled (b, d) channel means -> channel_norm output (b, d)
        (reference cforward_corev1, MambaSISR6_arch.py:438-483, after its AdaptiveAvgPool2d)"""
        if hasattr(self, "conv_cin"):
            wci = self.conv_cin.weight.view(-1, 1)
            seq = pooled[:, None, :] * wci[None] + self.conv_cin.bias.view(1, -1, 1)  # (b, dc, L=d)
        else:
            seq = pooled[:, None, :]  # (b, 1, L=d)
        Bn, Dc, L = seq.shape
        xsc = torch.stack([seq, seq.flip(-1)], dim=1)  # (b,2,dc,L)
        xc_dbl = torch.einsum("bkdl,kcd->bkcl", xsc, self.xc_proj_weight)
        dts, Bs, Cs = torch.split(xc_dbl, [self.dtc_rank, self.dc_state, self.dc_state], dim=2)
        dts = torch.einsum("bkrl,kdr->bkdl", dts, self.dtc_projs_weight)
        out_y = selective_scan_fn(xsc.reshape(Bn, -1, L), dts.reshape(Bn, -1, L).contiguous(),
                                  -torch.exp(self.Ac_logs.float()), Bs.contiguous(), Cs.contiguous(), self.Dsc.float(),
                                  delta_bias=self.dtc_projs_bias.reshape(-1).float(), delta_softplus=True).view(Bn, 2, -1, L)
        y = out_y[:, 0].float() + out_y[:, 1].flip(-1).float()  # (b, dc, L)
        if hasattr(self, "conv_cout"):
            y = (y * self.conv_cout.weight.view(1, -1, 1).float()).sum(1, keepdim=True) + self.conv_cout.bias.float().view(1, 1, 1)
        y = y.transpose(1, 2).unsqueeze(-1)  # (b, L=d, 1, 1)
        return self.channel_norm(y).view(Bn, L)

    def cforward_core(self, xc):
        b, d, h, w = xc.shape
        pooled = xc.float().mean(dim=(2, 3)).to(xc.dtype)  # AdaptiveAvgPool2d(1) -> (b, d)
        return self.cforward_pooled(pooled).view(b, d, 1, 1).to(xc.dtype)

    def forward_compose(self, x):
        xz = self.in_conv(x)
        x, z = xz.chunk(2, dim=1)
        z = self.act(z)
        x = self.act(self.conv2d(x))
        y2 = self.forward_core(x) * z
        c = self.cforward_core(y2)
        y2 = y2 * c + y2 if self.gate == "mul" else y2 + c
        return self.out_conv(y2)

    def forward(self, x: torch.Tensor, **kwargs):
        return self.forward_compose(x)


class MamberBlock(nn.Module):
    def __init__(self, dim, num_heads, ffn_expansion_factor, bias, LayerNorm_type, variant="sisr"):
        super().__init__()
        self.norm1 = LayerNorm(dim, LayerNorm_type)
        self.attn = SS2D_1(d_model=dim, ssm_ratio=1, variant=variant)
        self.norm2 = LayerNorm(dim, LayerNorm_type)
        self.ffn = FeedForward(dim, ffn_expansion_factor, bias)
        self.ln_type = LayerNorm_type

    def forward_compose(self, x):
        x = x + self.attn.forward_compose(self.norm1(x))
        return x + self.ffn(self.norm2(x))

    def forward(self, x, out=None):
        """out (inference only, vmambair_b200.unet): optional destination view (a channel slice of a concatenation buffer)"""
        if x.is_cuda:
            from . import fused
            if not torch.is_grad_enabled():
                if fused.available(self, x):
                    return fused.block_forward(self, x, out)
            elif _TRAIN_PATH == "fused" and fused.available(self, x):
                from . import fused_train
                return fused_train.block_forward(self, x)  # forward + backward of every stage on this library's kernels
        y = self.forward_compose(x)
        if out is not None:
            out.copy_(y)
            return out
        return y


# ----------------------------------------------------------------------------- U-Net pieces
class OverlapPatchEmbed(nn.Module):
    def __init__(self, in_c=3, embed_dim=48, bias=False):
        super().__init__()
        self.proj = nn.Conv2d(in_c, embed_dim, kernel_size=3, stride=1, padding=1, bias=bias)

    def forward(self, x):
        return self.proj(x)


class Downsample(nn.Module):
    def __init__(self, n_feat):
        super().__init__()
        self.body = nn.Sequential(nn.Conv2d(n_feat, n_feat // 2, 3, 1, 1, bias=False), nn.PixelUnshuffle(2))

    def forward(self, x):
        return self.body(x)


class Upsample(nn.Module):
    def __init__(self, n_feat):
        super().__init__()
        self.body = nn.Sequential(nn.Conv2d(n_feat, n_feat * 2, 3, 1, 1, bias=False), nn.PixelShuffle(2))

    def forward(self, x):
        return self.body(x)


def default_conv(in_channels, out_channels, kernel_size, bias=True):
    return nn.Conv2d(in_channels, out_channels, kernel_size, padding=kernel_size // 2, bias=bias)


class Upsampler(nn.Sequential):
    def __init__(self, conv, scale, n_feat, act=False, bias=True):
        m = []
        if (int(scale) & (int(scale) - 1)) == 0:
            for _ in range(int(math.log(scale, 2))):
                m += [conv(n_feat, 4 * n_feat, 3, bias), nn.PixelShuffle(2)]
                if act:
                    m.append(act())
        elif scale == 3:
            m += [conv(n_feat, 9 * n_feat, 3, bias), nn.PixelShuffle(3)]
            if act:
                m.append(act())
        else:
            raise NotImplementedError
        super().__init__(*m)


_DEFER_TAIL_BIAS = os.environ.get("VMB_TAIL_BIAS", "deferred") == "deferred"


def fused_f32(t):
    from . import fused
    return fused._f32(t)


def ops_mod():
    from . import ops
    return ops


class _MamberUNet(nn.Module):
    """Shared 4-level encoder/decoder wiring (reference forward :610-638)."""
    VARIANT = "sisr"

    def _build_trunk(self, inp_channels, dim, num_blocks, num_refinement_blocks, heads, ffn_expansion_factor, bias,
                     LayerNorm_type):
        def stage(d, n, h):
            return nn.Sequential(*[MamberBlock(dim=d, num_heads=h, ffn_expansion_factor=ffn_expansion_factor, bias=bias,
                                               LayerNorm_type=LayerNorm_type, variant=self.VARIANT) for _ in range(n)])
        self.patch_embed = OverlapPatchEmbed(inp_channels, dim)
        self.encoder_level1 = stage(dim, num_blocks[0], heads[0])
        self.down1_2 = Downsample(dim)
        self.encoder_level2 = stage(dim * 2, num_blocks[1], heads[1])
        self.down2_3 = Downsample(dim * 2)
        self.encoder_level3 = stage(dim * 4, num_blocks[2], heads[2])
        self.down3_4 = Downsample(dim * 4)
        self.latent = stage(dim * 8, num_blocks[3], heads[3])
        self.up4_3 = Upsample(dim * 8)
        self.reduce_chan_level3 = nn.Conv2d(dim * 8, dim * 4, kernel_size=1, bias=bias)
        self.decoder_level3 = stage(dim * 4, num_blocks[2], heads[2])
        self.up3_2 = Upsample(dim * 4)
        self.reduce_chan_level2 = nn.Conv2d(dim * 4, dim * 2, kernel_size=1, bias=bias)
        self.decoder_level2 = stage(dim * 2, num_blocks[1], heads[1])
        self.up2_1 = Upsample(dim * 2)
        self.decoder_level1 = stage(dim * 2, num_blocks[0], heads[0])
        self.refinement = stage(dim * 2, num_refinement_blocks, heads[0])

    _lowres_chains = 1
    _lowres_streams = ()

    def set_lowres_chains(self, chains: int, streams) -> None:
        """inference only (vmambair_b200.engine): evaluate the levels below full resolution on `chains` sub-batches in
        parallel streams -- images are independent, so the result does not change"""
        self._lowres_chains, self._lowres_streams = int(chains), tuple(streams)

    def _lowres(self, e1):
        """everything below full resolution: e1 -> up2_1(d2)  (reference forward :612-633)"""
        e2 = self.encoder_level2(self.down1_2(e1))
        e3 = self.encoder_level3(self.down2_3(e2))
        lat = self.latent(self.down3_4(e3))
        d3 = self.decoder_level3(self.reduce_chan_level3(torch.cat([self.up4_3(lat), e3], 1)))
        d2 = self.decoder_level2(self.reduce_chan_level2(torch.cat([self.up3_2(d3), e2], 1)))
        return self.up2_1(d2)

    def _trunk(self, inp_img):
        from . import unet
        if unet.enabled(inp_img) and inp_img.shape[2] % 8 == 0 and inp_img.shape[3] % 8 == 0:
            return unet.trunk(self, inp_img)  # inference: the non-OSS convs / shuffles / concatenations on this library's kernels
        e1_in = self.patch_embed(inp_img)
        e1 = self.encoder_level1(e1_in)
        if self._lowres_chains > 1 and e1.is_cuda and not torch.is_grad_enabled():
            from .engine import fork_join_batch
            up = fork_join_batch(self._lowres, e1, self._lowres_chains, self._lowres_streams)
        else:
            up = self._lowres(e1)
        d1 = self.decoder_level1(torch.cat([up, e1], 1))
        return self.refinement(d1), e1_in


class MambaSISR6(_MamberUNet):
    VARIANT = "sisr"

    def __init__(self, inp_channels=3, out_channels=3, scale=4, dim=48, num_blocks=[6, 2, 2, 1], num_refinement_blocks=6,
                 heads=[1, 2, 4, 8], ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias"):
        super().__init__()
        self.scale = scale
        self._build_trunk(inp_channels, dim, num_blocks, num_refinement_blocks, heads, ffn_expansion_factor, bias, LayerNorm_type)
        self.tail = nn.Sequential(Upsampler(default_conv, 4, dim * 2, act=False), default_conv(dim * 2, out_channels, 3))

    def forward(self, inp_img):
        feat, _ = self._trunk(inp_img)
        if feat.is_cuda and not torch.is_grad_enabled() and feat.dtype in (torch.float32, torch.bfloat16, torch.float16):
            from . import unet
            if unet.enabled(feat) and float(self.scale).is_integer() and feat.shape[1] % 8 == 0:
                return self._tail_channels_last(feat, inp_img)  # "+ nearest-upsampled input" inside the last conv's store
            return self._tail_channels_last(feat) + F.interpolate(inp_img, scale_factor=self.scale, mode="nearest")
        return self.tail(feat) + F.interpolate(inp_img, scale_factor=self.scale, mode="nearest")

    def _tail_channels_last(self, feat, inp_img=None):
        """inference: the SR tail (conv 3x3 -> PixelShuffle(2), twice, conv 3x3; reference common.py:45-60 and
        MambaSISR6_arch.py:607,640) on NHWC storage end to end -- the convs run on cuDNN's native layout and the pixel
        shuffles are this library's permutation kernel, instead of an NCHW<->NHWC transform either side of every conv
        plus an un-vectorised strided copy per shuffle (together ~9 % of the round-1 step).  Same values as self.tail."""
        from . import ops
        cache = getattr(self, "_tail_cl", None)
        ver = tuple((p.data_ptr(), p._version, p.dtype) for p in self.tail.parameters())
        if cache is None or cache[0] != ver:
            cache = (ver, {id(m): m.weight.detach().contiguous(memory_format=torch.channels_last)
                           for m in self.tail.modules() if isinstance(m, nn.Conv2d)})
            self._tail_cl = cache
        wcl = cache[1]
        x = feat.contiguous(memory_format=torch.channels_last)
        mods = list(self.tail[0]) + [self.tail[1]]
        pending_bias = None
        for i, m in enumerate(mods):
            if inp_img is not None and i == len(mods) - 1 and x.shape[1] % 8 == 0:
                # conv_last + F.interpolate(inp_img, nearest) + add + NHWC -> NCHW: one kernel of this library (unet.py)
                from . import unet
                return unet.conv3x3(m, x.contiguous(memory_format=torch.channels_last), ops.CONV_ADD_NEAREST,
                                    add=inp_img.to(x.dtype), add_scale=int(self.scale), nhwc=True)
            if isinstance(m, nn.Conv2d):
                nxt = mods[i + 1] if i + 1 < len(mods) else None
                # a conv followed by PixelShuffle(2) runs without its bias: the permutation kernel adds it (the library conv would
                # otherwise spend a separate elementwise pass over its (B,4C,H,W) output on the bias)
                defer = (m.bias is not None and isinstance(nxt, nn.PixelShuffle) and nxt.upscale_factor == 2 and
                         m.out_channels % 8 == 0 and _DEFER_TAIL_BIAS)
                x = F.conv2d(x, wcl[id(m)], None if defer else m.bias, m.stride, m.padding)
                pending_bias = fused_f32(m.bias) if defer else None
            elif isinstance(m, nn.PixelShuffle) and m.upscale_factor == 2 and x.shape[1] % 8 == 0:
                x = ops.pixel_shuffle2_nhwc(x.contiguous(memory_format=torch.channels_last), pending_bias)
                pending_bias = None
            else:
                x = m(x)
        if inp_img is not None:
            return x.contiguous() + F.interpolate(inp_img, scale_factor=self.scale, mode="nearest")
        return x.contiguous()


class MambaRealSR11(MambaSISR6):
    VARIANT = "realsr"


class Mamber32(_MamberUNet):
    VARIANT = "mamber32"

    def __init__(self, inp_channels=3, out_channels=3, dim=48, num_blocks=[6, 6, 7, 8], num_refinement_blocks=2,
                 heads=[1, 2, 4, 8], ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias", dual_pixel_task=False):
        super().__init__()
        self._build_trunk(inp_channels, dim, num_blocks, num_refinement_blocks, heads, ffn_expansion_factor, bias, LayerNorm_type)
        self.dual_pixel_task = dual_pixel_task
        if dual_pixel_task:
            self.skip_conv = nn.Conv2d(dim, dim * 2, kernel_size=1, bias=bias)
        self.output = nn.Conv2d(dim * 2, out_channels, kernel_size=3, stride=1, padding=1, bias=bias)

    def forward(self, inp_img):
        feat, e1_in = self._trunk(inp_img)
        if self.dual_pixel_task:
            return self.output(feat + self.skip_conv(e1_in))
        from . import unet
        if unet.enabled(feat):  # output conv + inp_img in one kernel
            return unet.conv3x3(self.output, feat, ops_mod().CONV_ADD_NEAREST, add=inp_img.to(feat.dtype), add_scale=1)
        return self.output(feat) + inp_img


class Mamber33(Mamber32):
    VARIANT = "mamber33"
