"""Padded and tiled inference around the fused networks -- the deployment-side callers of the hot path (SURVEY.md 8f rank 4).

Reference behaviour mirrored:
  * pad_to_multiple / padded_inference: reflect-pad H, W up to a multiple of `window_size` (SR: MambaSISRModel.pad_test + test,
    SRGAN/VmambaIR/models/MambaSISR_model.py:87-118) or of 8 (deraining: Deraining/basicsr/test_deraining.py:73-85 -- note its
    `((h+factor)//factor)*factor` only pads when h % factor != 0), run the net, crop the output back to (h*scale, w*scale);
  * tile_process: RealESRGANer.tile_process (RealSR/VmambaIR/utils.py:97-160): tiles of `tile_size` with `tile_pad` pixels of
    context on every side that exists, each upscaled on its own, the un-padded centre written into the output.

GPU-first difference: tiles of equal shape are independent units of the path, so they are stacked on the batch axis and go through
the network in batches of `max_batch` tiles instead of one forward per tile; the stitched result is the reference's.
"""
from __future__ import annotations

import math
from collections import defaultdict
from typing import Callable, Tuple

import torch
import torch.nn.functional as F


def pad_to_multiple(x: torch.Tensor, multiple: int) -> Tuple[torch.Tensor, int, int]:
    """reflect-pad the bottom / right of (B,C,H,W) so that H and W are multiples of `multiple` -> (padded, pad_h, pad_w)"""
    _, _, h, w = x.shape
    pad_h = (multiple - h % multiple) % multiple
    pad_w = (multiple - w % multiple) % multiple
    if pad_h == 0 and pad_w == 0:
        return x, 0, 0
    return F.pad(x, (0, pad_w, 0, pad_h), "reflect"), pad_h, pad_w


def padded_inference(net_fn: Callable[[torch.Tensor], torch.Tensor], x: torch.Tensor, multiple: int = 8, scale: int = 1) -> torch.Tensor:
    """net_fn on the reflect-padded input, output cropped to the original extent times `scale`"""
    _, _, h, w = x.shape
    xp, _, _ = pad_to_multiple(x, multiple)
    y = net_fn(xp)
    return y[:, :, :h * scale, :w * scale]


def tile_plan(height: int, width: int, tile_size: int, tile_pad: int):
    """the reference's tile loop as data: per tile the padded input window, the output window and the centre inside the tile output"""
    tiles = []
    for ty in range(math.ceil(height / tile_size)):
        for tx in range(math.ceil(width / tile_size)):
            x0, y0 = tx * tile_size, ty * tile_size
            x1, y1 = min(x0 + tile_size, width), min(y0 + tile_size, height)
            x0p, y0p = max(x0 - tile_pad, 0), max(y0 - tile_pad, 0)
            x1p, y1p = min(x1 + tile_pad, width), min(y1 + tile_pad, height)
            tiles.append(dict(inp=(y0p, y1p, x0p, x1p), out=(y0, y1, x0, x1), ctr=(y0 - y0p, x0 - x0p)))
    return tiles


def tile_process(net_fn: Callable[[torch.Tensor], torch.Tensor], img: torch.Tensor, tile_size: int, tile_pad: int = 10, scale: int = 4,
                 max_batch: int = 8) -> torch.Tensor:
    """RealESRGANer.tile_process on (B,C,H,W): equal-shape tiles are batched (max_batch tiles x B images per forward)."""
    b, c, height, width = img.shape
    plan = tile_plan(height, width, tile_size, tile_pad)
    groups = defaultdict(list)
    for i, t in enumerate(plan):
        y0p, y1p, x0p, x1p = t["inp"]
        groups[(y1p - y0p, x1p - x0p)].append(i)
    out = None
    for (_th, _tw), idxs in groups.items():
        for s in range(0, len(idxs), max_batch):
            chunk = idxs[s:s + max_batch]
            stack = torch.cat([img[:, :, plan[i]["inp"][0]:plan[i]["inp"][1], plan[i]["inp"][2]:plan[i]["inp"][3]] for i in chunk], 0)
            res = net_fn(stack.contiguous())
            if out is None:
                out = res.new_zeros((b, res.shape[1], height * scale, width * scale))
            for j, i in enumerate(chunk):
                y0, y1, x0, x1 = plan[i]["out"]
                cy, cx = plan[i]["ctr"]
                tile = res[j * b:(j + 1) * b]
                out[:, :, y0 * scale:y1 * scale, x0 * scale:x1 * scale] = \
                    tile[:, :, cy * scale:(cy + y1 - y0) * scale, cx * scale:(cx + x1 - x0) * scale]
    return out


class TiledInference:
    """Public entry for arbitrary-size images on the fused networks: mod-pad (reflect) -> optional tiling -> crop.
    net: a vmambair_b200.archs network; dtype: compute dtype (the module is cast on a private copy, like InferenceEngine)."""

    def __init__(self, net: torch.nn.Module, scale: int = 1, multiple: int = 8, tile_size: int = 0, tile_pad: int = 10,
                 dtype=torch.bfloat16, device="cuda", max_batch: int = 8):
        import copy
        from .engine import cast_for_inference
        self.net = cast_for_inference(copy.deepcopy(net).to(device).eval(), dtype)
        self.scale, self.multiple, self.tile_size, self.tile_pad = scale, multiple, tile_size, tile_pad
        self.dtype, self.device, self.max_batch = dtype, torch.device(device), max_batch

    @torch.no_grad()
    def _fwd(self, x):
        return self.net(x)

    @torch.no_grad()
    def __call__(self, img: torch.Tensor) -> torch.Tensor:
        """img: (B,C,H,W) host or device tensor -> (B,C,H*scale,W*scale) on the device, in the compute dtype"""
        x = img.to(self.device, self.dtype)
        _, _, h, w = x.shape
        xp, _, _ = pad_to_multiple(x, self.multiple)
        if self.tile_size and (xp.shape[2] > self.tile_size or xp.shape[3] > self.tile_size):
            y = tile_process(self._fwd, xp, self.tile_size, self.tile_pad, self.scale, self.max_batch)
        else:
            y = self._fwd(xp)
        return y[:, :, :h * self.scale, :w * self.scale]
