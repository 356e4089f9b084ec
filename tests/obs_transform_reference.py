"""A short restatement, in torch ops on the CPU, of what the reference's ResizeShortestEdge and CenterCropper compute
for channels-last images (habitat_baselines/common/obs_transformers.py, utils/common.py image_resize_shortest_edge /
center_crop).  The GPU tests compare the fused kernel with it bit for bit; test_obs_transforms_cpu.py shows it is
bit-identical to the reference classes themselves."""
from __future__ import annotations

import torch
import torch.nn.functional as F


def resized_hw(h, w, size):
    """The reference's float64 shape rule (not integer arithmetic)."""
    return int(h * (size / min(h, w))), int(w * (size / min(h, w)))


def resize(img: torch.Tensor, size: int, mode: str) -> torch.Tensor:
    """[B,] H, W, C -> [B,] Hr, Wr, C: resampled through float32 and converted back with truncation."""
    x = img if img.dim() == 4 else img[None]
    hr, wr = resized_hw(x.shape[1], x.shape[2], size)
    y = F.interpolate(x.cpu().permute(0, 3, 1, 2).float(), size=(hr, wr), mode=mode)
    y = y.to(img.dtype).permute(0, 2, 3, 1).contiguous()
    return y if img.dim() == 4 else y[0]


def crop(img: torch.Tensor, hw) -> torch.Tensor:
    h, w = img.shape[-3], img.shape[-2]
    y0, x0 = h // 2 - hw[0] // 2, w // 2 - hw[1] // 2
    return img[..., y0:y0 + hw[0], x0:x0 + hw[1], :]


def mode_for(key: str, semantic_key: str = "semantic") -> str:
    return "nearest" if semantic_key in key else "area"


def transform(obs: dict, size=None, crop_hw=None, keys=("rgb", "depth", "semantic"), semantic_key="semantic"):
    """ResizeShortestEdge(size) then CenterCropper(crop_hw) on the `keys` of a dict of CPU tensors (either may be
    None); other keys pass through."""
    out = dict(obs)
    for k in keys:
        if k not in out:
            continue
        v = out[k].cpu()
        if size is not None:
            v = resize(v, size, mode_for(k, semantic_key))
        if crop_hw is not None:
            v = crop(v, crop_hw)
        out[k] = v.contiguous()
    return out
