"""RAFT-style correlation lookups in float64 without the volume, and the per-entry bound of an fp32 implementation's distance from them.
Shared by the stage tests of the flow estimator (test_raft_stages_gpu.py) and of the motion stage (test_motion_stages_gpu.py)."""
import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24   # fp32 unit roundoff
# the fp32-class constant of a 256-term dot product: the recursive-summation bound K u of the fp32 CUDA-core GEMM (mode 0), the host
# simulation's sequential FMAs and the volume-free warp dot, which also covers the 3xF16 GEMM (operand split 2^-22 per operand, the
# dropped lo x lo product 2^-22, and the fp32 accumulation of 16 segments of K = 16); plus 16 u for the pooling (fp32 averages of up to
# 64 values), the bilinear weights' products and the four-tap blend
GAMMA_DOT = (256 + 16) * U
HALF = 2.0 ** -11   # IEEE half unit roundoff: the volume-free lookup's target features


def _pool_levels(ftgt, levels=4):
    pyr = [ftgt]
    for _ in range(levels - 1):
        pyr.append(F.avg_pool2d(pyr[-1], 2, stride=2))
    return pyr


def corr_direct64(fsrc, ftgt, coords, r=4, chunk=2048):
    """BidirCorrBlock's / RAFT's CorrBlock lookup (raft/corr.py:23-93, :120-165 == oracle.BidirCorr / corr_lookup) without the volume:
    at level l the 2r+2 x 2r+2 integer neighbours of each window on the 2^l-average-pooled target features (pooling the volume's target
    dims is pooling the features: the dot product is linear), zero outside the frame, then the bilinear weights.  fsrc / ftgt (N, C, h, w),
    coords (N, 2, h, w) (x, y) at level 0 -> (N, 4 (2r+1)^2, h, w); channel i (2r+1) + j of a level samples (Δx, Δy) = (i - r, j - r)."""
    return corr_lookup64(fsrc, ftgt, coords, r, chunk)[0]


def corr_lookup64(fsrc, ftgt, coords, r=4, chunk=2048, bound=None):
    """corr_direct64, and with bound = "volume" or "direct" also the per-entry bound (same shape) of an fp32 lookup's distance from it:
    - the dot products: GAMMA_DOT times the bilinear blend of sum_c |s_c| |t_c| / sqrt(C), i.e. this lookup on |fsrc| and |ftgt|
      (with the pooled |t| at levels 1-3, which bounds |pooled t|);
    - the coordinates: the fp32 normalise / un-normalise round trip of bilinear_sampler (raft/utils/utils.py:66-80), which both the volume
      lookup (corr.cu CorrLookupK) and the volume-free one (corr_axis) evaluate: pc = c / 2^l + d, g = 2 pc / (S - 1) - 1,
      ((g + 1) / 2) (S - 1) rounds five times, |error| <= u (6 |pc| + S) along an axis of S pixels, times the largest slope of the
      bilinear interpolant next to the sample (the differences of neighbouring dots in x or y over the cells a rounding can move it to);
    - "direct" only: HALF times the same absolute-value blend (the target features enter as IEEE half at every level; subnormal halves'
      absolute error 2^-25 is far below it for O(1) features), and its 10 x 10 dot grid, which folds a tap that rounding moves one cell
      past the grid onto the grid's edge with zero weight: the slopes there are taken against 0."""
    N, C, h, w = fsrc.shape
    k = 2 * r + 1
    pyr = _pool_levels(ftgt)
    src = fsrc.permute(0, 2, 3, 1).reshape(N, h * w, C)
    cen0 = coords.permute(0, 2, 3, 1).reshape(N, h * w, 2)
    e = 1 if bound else 0                                                  # the bound's grid reaches one more neighbour on each side
    offs = torch.arange(-r - e, r + 2 + e, device=fsrc.device)
    out = torch.empty(N, h * w, 4 * k * k, device=fsrc.device, dtype=fsrc.dtype)
    bnd = torch.empty_like(out) if bound else None
    if bound:
        pyra = _pool_levels(ftgt.abs())
        srca = src.abs()
    for l, ft in enumerate(pyr):
        hl, wl = ft.shape[-2:]
        tgt = ft.permute(0, 2, 3, 1).reshape(N, hl * wl, C)
        tgta = pyra[l].permute(0, 2, 3, 1).reshape(N, hl * wl, C) if bound else None
        cen = cen0 / 2 ** l
        for n in range(N):
            for p0 in range(0, h * w, chunk):
                c = cen[n, p0:p0 + chunk]
                x0, y0 = torch.floor(c[:, 0]), torch.floor(c[:, 1])
                fx, fy = (c[:, 0] - x0).view(-1, 1, 1), (c[:, 1] - y0).view(-1, 1, 1)
                xs = x0.long().view(-1, 1) + offs                                  # (P, 2r+2 (+2))
                ys = y0.long().view(-1, 1) + offs
                valid = ((ys >= 0) & (ys < hl)).unsqueeze(2) & ((xs >= 0) & (xs < wl)).unsqueeze(1)   # (P, y, x)
                idx = ys.clamp(0, hl - 1).unsqueeze(2) * wl + xs.clamp(0, wl - 1).unsqueeze(1)
                blend = lambda d: ((1 - fx) * (1 - fy) * d[:, :k, :k] + fx * (1 - fy) * d[:, :k, 1:] + (1 - fx) * fy * d[:, 1:, :k]
                                   + fx * fy * d[:, 1:, 1:])                      # (P, Δy, Δx)
                dg = torch.einsum("pabc,pc->pab", tgt[n][idx], src[n, p0:p0 + chunk]) / math.sqrt(C) * valid
                d = dg[:, e:dg.shape[1] - e, e:dg.shape[2] - e]
                out[n, p0:p0 + chunk, l * k * k:(l + 1) * k * k] = blend(d).transpose(1, 2).reshape(-1, k * k)
                if not bound:
                    continue
                da = torch.einsum("pabc,pc->pab", tgta[n][idx[:, 1:-1, 1:-1]], srca[n, p0:p0 + chunk]) / math.sqrt(C) * valid[:, 1:-1, 1:-1]
                ab = blend(da)
                if bound == "direct":
                    dg = dg.clone()
                    dg[:, 0], dg[:, -1], dg[:, :, 0], dg[:, :, -1] = 0, 0, 0, 0
                # slope of cell (row y, cells x..x+1) of the (2r+4)^2 grid; window sample (Δy = b, Δx = a) sits in cell (b + 1, a + 1):
                # the largest over the neighbouring cells a..a+2 and rows b..b+3 (resp. the transpose for y)
                sx = F.max_pool2d((dg[:, :, 1:] - dg[:, :, :-1]).abs().unsqueeze(1), (4, 3), stride=1)[:, 0]   # (P, k, k)
                sy = F.max_pool2d((dg[:, 1:, :] - dg[:, :-1, :]).abs().unsqueeze(1), (3, 4), stride=1)[:, 0]
                dd = torch.arange(-r, r + 1, device=fsrc.device, dtype=fsrc.dtype)
                ex = U * (6 * (c[:, :1] + dd).abs() + wl)                             # (P, Δx)
                ey = U * (6 * (c[:, 1:] + dd).abs() + hl)                             # (P, Δy)
                b = (GAMMA_DOT + (HALF if bound == "direct" else 0.0)) * ab + ex.unsqueeze(1) * sx + ey.unsqueeze(2) * sy
                bnd[n, p0:p0 + chunk, l * k * k:(l + 1) * k * k] = b.transpose(1, 2).reshape(-1, k * k)
    shape = lambda t: t.view(N, h, w, -1).permute(0, 3, 1, 2)
    return shape(out), (shape(bnd) if bound else None)


def windows_outside(coords, h, w, r=4):
    """per pyramid level, how many lookup windows straddle or leave the frame (the zero padding is read); r = 0: how many window
    centres lie outside the frame (the flow, not only the window's reach, takes the lookup past the border)"""
    out = []
    for l in range(4):
        hl, wl = h >> l, w >> l
        cx, cy = coords[:, 0] / 2 ** l, coords[:, 1] / 2 ** l
        out.append(int(((cx - r < 0) | (cx + r > wl - 1) | (cy - r < 0) | (cy + r > hl - 1)).sum().item()))
    return out
