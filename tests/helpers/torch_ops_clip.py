"""TEST INFRASTRUCTURE: helpers.torch_ops plus a torch-CPU stand-in for the CLIP encoder's input kernel
(yb_resize_bicubic_normalize, include/yume_b200_clip.h), so the CPU suite can drive yume_b200/clip.py's host logic."""
import torch.nn.functional as F

from helpers.torch_ops import *  # noqa: F401,F403


def resize_bicubic_normalize(x, out, mean, std):
    """x f32 [C, H, W] -> out f32 [C, S, S]: F.interpolate(bicubic, align_corners=False), * 0.5 + 0.5, - mean, / std."""
    y = F.interpolate(x[None].float(), size=tuple(out.shape[-2:]), mode="bicubic", align_corners=False)[0]
    out.copy_(y.mul_(0.5).add_(0.5).sub_(mean.view(-1, 1, 1)).div_(std.view(-1, 1, 1)))
    return out
