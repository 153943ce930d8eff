"""float64 restatements of GIMM's splatting weights shared by the stage tests (test_stages_gpu.py, test_motion_stages_gpu.py), and the
per-pixel bound of an fp32 implementation's distance from them.  Layouts: the engine's NHWC, both directions as 2B samples."""
import torch
import torch.nn.functional as F

import gimmvfi_r_oracle as O


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def splat_w_float64(sd, flows):
    """flows (B, 2, 2, H, W): [f01 | f10] on dim 2 -> the splatting weights of both directions, (2B, H, W, 1) float64"""
    sd64 = {k: sd[k].to(flows.device, torch.float64) for k in ("g_filter", "alpha_fe", "alpha_v")}
    w1, w2 = O.splatting_weights(sd64, flows[:, :, 0].double(), flows[:, :, 1].double())
    return torch.cat([nhwc(w1), nhwc(w2)], 0)


def splat_w_bound(sd, flows):
    """per-pixel bound of |fp32 - float64| of the splatting weights, (2B, H, W, 1).  The variance term: E[f^2] - E[f]^2 over the 3x3
    gaussian carries an fp32 rounding e <= 16 * 2^-24 * E[f^2] (nine products and sums, a square, a difference), which moves its square
    root by at most min(sqrt(e), e / (2 sqrt(d))) - unbounded conditioning where d -> 0; the 1e-9 clamp adds up to 3.2e-5; the weight
    takes a_v / 2 of the channels' sum.  The consistency term is a bilinear tap and an absolute difference: ~1e-6 * |f| * a_fe, plus the
    tap's sample position, which backwarp rounds on its way through [-1, 1] (<= 4 * 2^-24 * (W + H + |f|) px), times the warped flow's
    slope in the sampled cell (a 3x3 max of its finite differences, itself sampled there): the term that dominates where a large flow
    field is steep (GIMM-VFI-F's 544 x 1024 network resolution)."""
    fl = torch.cat([flows[:, :, 0], flows[:, :, 1]], 0).double()
    g = sd["g_filter"].to(fl.device, torch.float64)
    blur = F.conv3d(F.pad(torch.cat([fl ** 2, fl], 1), (1, 1, 1, 1), mode="reflect").unsqueeze(1), g).squeeze(1)
    sq, m = torch.split(blur, 2, dim=1)
    d = (sq - m ** 2).clamp(min=0.0)
    e = 16 * 2.0 ** -24 * sq
    dsqrt = torch.minimum(e.sqrt(), e / (2 * d.sqrt()).clamp(min=1e-30)) + 3.2e-5
    B, H, W = flows.shape[0], fl.shape[-2], fl.shape[-1]
    dx = F.max_pool2d(F.pad((fl[..., :, 1:] - fl[..., :, :-1]).abs(), (0, 1, 0, 0)), 3, 1, 1)
    dy = F.max_pool2d(F.pad((fl[..., 1:, :] - fl[..., :-1, :]).abs(), (0, 0, 0, 1)), 3, 1, 1)
    slope = dx + dy
    pos = 4 * 2.0 ** -24 * (W + H + fl.abs().sum(1, keepdim=True))
    # err01 warps f10 along f01 and vice versa (gimmvfi_r.py:476-477)
    tap = pos * O.backwarp(torch.cat([slope[B:], slope[:B]], 0), fl).mean(1, keepdim=True)
    return (nhwc(0.5 * float(sd["alpha_v"]) * dsqrt.sum(1, keepdim=True) + float(sd["alpha_fe"]) * tap)
            + 2e-6 * float(fl.abs().max()) * float(sd["alpha_fe"]) + 1e-6)
