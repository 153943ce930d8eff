"""GPU kernels at the edges the model-level tests do not reach, against float64 references of the same operation.

* RAFT FlowHead.conv2 (3x3, 256 -> 1/2 channels) at output widths that are not multiples of four: conv_narrow3x3_c256_kernel computes
  four horizontally adjacent pixels per warp, so the last quad of every row is partial (frame widths 136 / 200 give RAFT widths 17 / 25).
* The three-pass forward splat's warp-shuffle merge (softsplat_acc_v4_kernel): lane l hands its east column of target cells to lane
  l+1 when that pixel lands exactly one cell further east in the same row - what smooth flows produce, and what i.i.d. random flows
  almost never do.  Rows of 17 / 25 / 33 pixels straddle warps; landings at x0 = -1 and x1 = W; integer landings; a discontinuity in
  the middle of a warp.
* The one-pass splat (softsplat_tile_kernel) with a reach R larger than its 32 x 32 target tile, at t = 0 and t = 1.

Every kernel launch is confirmed by name with torch.profiler, so a change of dispatch cannot silently move a case to another kernel."""
import pytest
import torch
import torch.nn.functional as F
from torch.profiler import ProfilerActivity, profile

import gimmvfi_r_oracle as O
import gpu_ops as K

pytestmark = pytest.mark.gpu
DEV = "cuda"


def launched_kernels(fn):
    """runs fn() under torch.profiler and returns (fn's result, names of the CUDA kernels it launched)"""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = fn()
        torch.cuda.synchronize()
    return res, {e.key for e in prof.key_averages()}


def assert_launched(names, kernel):
    assert any(kernel in n for n in names), "expected a launch of %s, got %s" % (kernel, sorted(names))


# --------------------------------------------------------------------------- FlowHead.conv2 on partial quads
@pytest.mark.parametrize("use_res", [False, True])
@pytest.mark.parametrize("cout", [2, 1])
@pytest.mark.parametrize("W", [17, 25, 23])
def test_flow_head_conv2_partial_quads(W, cout, use_res):
    """gimmvfi_op_conv2d with 3x3, cin 256, cout <= 2, stride 1, pad 1, no activation, fp32 NHWC with 16-byte pixels: conv_narrow_ok
    holds and the 3x3 / 256-channel branch takes conv_narrow3x3_c256_kernel.  W = 17, 25, 23 leave 1, 1 and 3 pixels in the last quad.
    Exact fp32 FMAs over K = 2304 products of |x| ~ 1 and |w| ~ 1/48: the float64 sum is met within ~1e-6 (bar 1e-5)."""
    n, cin, H = 2, 256, 9
    g = torch.Generator().manual_seed(100 + W + 10 * cout)
    x = torch.randn(n, cin, H, W, generator=g).to(DEV)
    w = (torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9) ** 0.5).to(DEV)
    b = (0.1 * torch.randn(cout, generator=g)).to(DEV)
    res = torch.randn(n, cout, H, W, generator=g).to(DEV) if use_res else None
    got, names = launched_kernels(lambda: K.conv2d(K.nhwc(x), w, b, pad=(1, 1), residual=K.nhwc(res) if use_res else None))
    assert_launched(names, "conv_narrow3x3_c256_kernel")
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    if use_res:
        ref = ref + res.double()
    err = (K.nchw(got).double() - ref).abs()
    print("conv_narrow3x3 W=%d cout=%d res=%d: max %.3e, last column max %.3e" % (W, cout, use_res, err.max().item(), err[..., -1].max().item()))
    assert err.max().item() <= 1e-5
    assert err[..., W - W % 4:].max().item() <= 1e-5   # the partial quad itself (a skipped or misplaced store is O(1))


# --------------------------------------------------------------------------- three-pass splat: the x-neighbour merge
Q = 64.0   # flows on a 1/64 grid and t in {1/4, 1/2, 3/4}: x + f * s is exact in fp32, so kernel and float64 reference land identically


def q(f):
    return torch.round(f * Q) / Q


def splat_flow(kind, n, H, W):
    """(n, 2, H, W) float64 flows whose neighbouring pixels land in neighbouring cells"""
    y = torch.arange(H, dtype=torch.float64).view(1, H, 1).expand(n, H, W)
    x = torch.arange(W, dtype=torch.float64).view(1, 1, W).expand(n, H, W)
    if kind == "constant_subpixel":        # every lane of a row merges with its east neighbour
        fx, fy = torch.full((n, H, W), 1.3125, dtype=torch.float64), torch.full((n, H, W), -0.5625, dtype=torch.float64)
    elif kind == "smooth_with_jump":       # smooth field, jump of +6.4 px at column W // 2 (the middle of a warp on every row)
        fx = 0.6 + 0.02 * y + 0.03 * torch.sin(x / 3.0) + torch.where(x >= W // 2, 6.4, 0.0)
        fy = -0.35 + 0.05 * torch.cos(x / 5.0 + y / 4.0)
    elif kind == "integer":                # integer landings (f * t is 1 or 3 cells): three of the four corner weights are exactly 0
        fx, fy = torch.full((n, H, W), 4.0, dtype=torch.float64), torch.full((n, H, W), -4.0, dtype=torch.float64)
        fx[:, :, W // 3:] = -4.0           # (and a row segment landing west)
    elif kind == "edges":                  # column 0 lands at x = -0.5 (x0 = -1), column W-1 at W - 0.5 (x1 = W)
        fx = -0.5 + x / (W - 1)
        fy = 0.25 + 0.0 * y
    else:
        raise ValueError(kind)
    return q(torch.stack([fx, fy], 1))


def merge_pairs(flow_sc):
    """number of pixels whose east neighbour (same row) lands one cell east in the same row: where the kernel's merge runs"""
    n, _, H, W = flow_sc.shape
    x = torch.arange(W, dtype=flow_sc.dtype).view(1, 1, W)
    y = torch.arange(H, dtype=flow_sc.dtype).view(1, H, 1)
    x0, y0 = torch.floor(x + flow_sc[:, 0]), torch.floor(y + flow_sc[:, 1])
    return int(((x0[..., 1:] == x0[..., :-1] + 1) & (y0[..., 1:] == y0[..., :-1])).sum())


def splat_inputs(kind, n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(n, 16, H, W, generator=g, dtype=torch.float64)
    metric = 0.5 + torch.rand(n, 1, H, W, generator=g, dtype=torch.float64)
    return lat.float().double(), splat_flow(kind, n, H, W), metric.float().double()


def splat_ref(lat, flow, metric, t, mode):
    sc = (t if mode == 0 else 1 - t).view(-1, 1, 1, 1).double()
    return O.softsplat_linear_zeroeps(lat, flow * sc, metric), flow * sc


SPLAT_BAR = 1e-5   # out = sum(lat * m * w) / sum(m * w) over positive weights: each term carries a few fp32 roundings (~1e-7 relative),
                   # so the quotient stays within ~1e-6 of float64 for |lat| <= 5, however small the accumulated weight


@pytest.mark.parametrize("W", [17, 25, 33])
@pytest.mark.parametrize("kind", ["constant_subpixel", "smooth_with_jump", "integer", "edges"])
def test_softsplat_three_pass_merge(kind, W):
    """gimmvfi_op_softsplat (memset + softsplat_acc_v4_kernel + normalise) against float64 "linear-zeroeps" (softsplat.py:286-352), two
    samples with different t, both t_modes (mode 0 scales the flow by t, mode 1 by 1 - t)."""
    n, H = 2, 11
    lat, flow, metric = splat_inputs(kind, n, H, W, seed=W)
    t = torch.tensor([0.25, 0.75], dtype=torch.float64)
    for mode in (0, 1):
        ref, fsc = splat_ref(lat, flow, metric, t, mode)
        pairs = merge_pairs(fsc)
        assert pairs >= n * H * (W - 1) // 2, (kind, pairs)   # the case really exercises the merge
        args = (K.nhwc(lat.float().to(DEV)), K.nhwc(flow.float().to(DEV)), K.nhwc(metric.float().to(DEV)), t.float().to(DEV), mode)
        got, names = launched_kernels(lambda: K.softsplat(*args))
        assert_launched(names, "softsplat_acc_v4_kernel")
        err = (K.nchw(got).double().cpu() - ref).abs()
        print("softsplat v4 %s W=%d mode %d: %d merging pairs, max %.3e" % (kind, W, mode, pairs, err.max().item()))
        assert err.max().item() <= SPLAT_BAR


def test_softsplat_three_pass_edge_landings_reach_the_border():
    """The `edges` field puts real weight on the first and last columns through the x0 = -1 / x1 = W cases: those columns must
    not be holes, and the cells outside the frame must not leak into them."""
    n, H, W = 1, 9, 33
    lat, flow, metric = splat_inputs("edges", n, H, W, seed=3)
    t = torch.tensor([1.0], dtype=torch.float64)
    ref, fsc = splat_ref(lat, flow, metric, t, 0)
    assert float(torch.floor(fsc[0, 0, 0, 0])) == -1.0 and float(torch.floor(W - 1 + fsc[0, 0, 0, -1])) + 1 == W
    got = K.nchw(K.softsplat(K.nhwc(lat.float().to(DEV)), K.nhwc(flow.float().to(DEV)), K.nhwc(metric.float().to(DEV)), t.float().to(DEV), 0))
    assert (ref[..., 0].abs().amax() > 0.1) and (ref[..., -1].abs().amax() > 0.1)
    assert (got.double().cpu() - ref).abs().max().item() <= SPLAT_BAR


# --------------------------------------------------------------------------- one-pass splat: reach beyond one tile, t = 0 and t = 1
@pytest.mark.parametrize("shape", [(2, 70, 100), (2, 45, 77)])
def test_softsplat_fused_long_reach(shape):
    """gimmvfi_op_softsplat_fused: a smooth ~38 px motion, so R = ceil(max|flow| * s) + 1 > 32 and every tile scans sources from beyond
    its neighbouring tiles; sample 0 at t = 0 and sample 1 at t = 1 (mode 0: s = 0 splats every pixel onto itself, s = 1 moves it the
    whole flow; mode 1 swaps them)."""
    n, H, W = shape
    y = torch.arange(H, dtype=torch.float64).view(1, H, 1).expand(n, H, W)
    x = torch.arange(W, dtype=torch.float64).view(1, 1, W).expand(n, H, W)
    flow = q(torch.stack([-37.5 + 0.05 * y + 0.5 * torch.sin(x / 7.0), 12.25 + 0.3 * torch.cos(y / 9.0 + x / 11.0)], 1))
    g = torch.Generator().manual_seed(7)
    lat = torch.randn(n, 16, H, W, generator=g).double()
    metric = (0.5 + torch.rand(n, 1, H, W, generator=g)).double()
    t = torch.tensor([0.0, 1.0], dtype=torch.float64)
    absmax = flow.abs().amax(dim=(1, 2, 3)).float().to(DEV).contiguous()
    assert absmax.min().item() > 32.0
    for mode in (0, 1):
        ref, _ = splat_ref(lat, flow, metric, t, mode)
        args = (K.nhwc(lat.float().to(DEV)), K.nhwc(flow.float().to(DEV)), K.nhwc(metric.float().to(DEV)), t.float().to(DEV), mode, absmax)
        got, names = launched_kernels(lambda: K.softsplat_fused(*args))
        assert_launched(names, "softsplat_tile_kernel")
        got = K.nchw(got).double().cpu()
        still = 0 if mode == 0 else 1                               # the sample whose scale is 0: the identity
        assert (got[still] - lat[still]).abs().max().item() <= 1e-6  # m * lat * 1 / (m * 1): two roundings
        err = (got - ref).abs()
        print("softsplat fused %s mode %d: max %.3e" % (shape, mode, err.max().item()))
        assert err.max().item() <= SPLAT_BAR
