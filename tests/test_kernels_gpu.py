"""GPU parity tests of every C-ABI kernel entry point against the oracle / plain
PyTorch fp32 of the same op.  Tolerances are written next to each check."""
import pytest
import torch
import torch.nn.functional as F

import gimmvfi_r_oracle as O
import gpu_ops as K

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rnd(*s, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*s, generator=g) * scale).to(DEV)


CONV_CASES = [
    # cin, cout, kh, kw, stride, pad, reflect, act, H, W, n
    (64, 64, 3, 3, 1, (1, 1), False, 0, 24, 40, 2),
    (273, 256, 3, 3, 1, (1, 1), False, 3, 16, 24, 1),     # final-decoder stem: odd cin, PReLU
    (3, 64, 7, 7, 2, (3, 3), False, 1, 64, 96, 2),        # RAFT stem: tiny cin, stride 2
    (384, 128, 1, 5, 1, (0, 2), False, 4, 16, 20, 2),     # SepConvGRU horizontal, sigmoid
    (384, 128, 5, 1, 1, (2, 0), False, 5, 16, 20, 1),     # vertical, tanh
    (256, 2, 3, 3, 1, (1, 1), False, 0, 16, 20, 2),       # flow head: tiny cout
    (9, 18, 7, 7, 1, (3, 3), False, 3, 32, 48, 1),        # comb block
    (32, 16, 3, 3, 1, (1, 1), True, 0, 20, 28, 2),        # reflect padding
    (324, 256, 1, 1, 1, (0, 0), False, 1, 16, 20, 2),     # 1x1 on the lookup
    (35, 128, 1, 1, 1, (0, 0), False, 6, 24, 24, 1),      # HypoNet layer 0: sin
    (64, 96, 1, 1, 2, (0, 0), False, 0, 32, 48, 2),       # 1x1 stride-2 downsample
    (256, 126, 3, 3, 1, (1, 1), False, 1, 16, 20, 1),     # cout not a multiple of 4... 126
    (128, 133, 3, 3, 1, (1, 1), False, 0, 16, 24, 1),
    (8, 32, 5, 5, 1, (2, 2), False, 3, 32, 32, 1),
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv2d(case):
    cin, cout, kh, kw, stride, pad, reflect, act, H, W, n = case
    x = rnd(n, cin, H, W, seed=1)
    w = rnd(cout, cin, kh, kw, seed=2, scale=1.0 / (cin * kh * kw) ** 0.5)
    b = rnd(cout, seed=3, scale=0.1)
    slope = (0.25 + 0.1 * rnd(cout, seed=4)) if act == 3 else None
    got = K.nchw(K.conv2d(K.nhwc(x), w, b, stride, pad, reflect, act, slope))
    xp = F.pad(x, (pad[1], pad[1], pad[0], pad[0]), mode="reflect") if reflect else x
    ref = F.conv2d(xp.double(), w.double(), b.double(), stride=stride, padding=(0, 0) if reflect else pad)
    ref = {0: lambda v: v, 1: F.relu, 2: lambda v: F.leaky_relu(v, 0.1), 3: lambda v: F.prelu(v, slope.double()),
           4: torch.sigmoid, 5: torch.tanh, 6: torch.sin}[act](ref).float()
    assert got.shape == ref.shape
    assert (got - ref).abs().max().item() <= 2e-5  # fp32 accumulate vs fp64 reference


def test_conv2d_two_segments_and_residual():
    """cat([a[:, :192], s]) input (ResBlock splice) + residual epilogue."""
    a = rnd(1, 256, 16, 24, seed=1)
    s = rnd(1, 64, 16, 24, seed=2)
    w = rnd(256, 256, 3, 3, seed=3, scale=0.02)
    b = rnd(256, seed=4, scale=0.1)
    res = rnd(1, 256, 16, 24, seed=5)
    a_nhwc, s_nhwc = K.nhwc(a), K.nhwc(s)
    got = K.nchw(K.conv2d(a_nhwc, w, b, 1, (1, 1), residual=K.nhwc(res), x1_nhwc=s_nhwc, in_view=K.view_of(a_nhwc, channels=192)))
    ref = F.conv2d(torch.cat([a[:, :192], s], 1).double(), w.double(), b.double(), padding=1).float() + res
    assert (got - ref).abs().max().item() <= 2e-5


def test_softsplat_vs_oracle():
    n, h, w = 2, 40, 56
    lat = rnd(n, 16, h, w, seed=1)
    flow = rnd(n, 2, h, w, seed=2, scale=4.0)
    flow[0, 0, 3, 3] = float("nan")
    flow[1, 1, 5, 7] = float("inf")
    flow[0, :, 0, 0] = torch.tensor([2.0, 1.0], device=DEV)   # integer landing
    flow[0, :, 10:14, 10:14] = 100.0                           # leaves the frame -> holes stay 0
    metric = 0.5 + rnd(n, 1, h, w, seed=3).abs()
    t = torch.tensor([0.5, 0.25], device=DEV)
    for mode in (0, 1):
        got = K.nchw(K.softsplat(K.nhwc(lat), K.nhwc(flow), K.nhwc(metric), t, mode))
        sc = (t if mode == 0 else (1 - t)).view(n, 1, 1, 1)
        ref = O.softsplat_linear_zeroeps(lat.cpu(), (flow * sc).cpu(), metric.cpu()).to(DEV)
        err = (got - ref).abs()
        # atomics order + the division by a small accumulated weight amplify fp32 rounding
        assert err.max().item() <= 3e-4 and err.mean().item() <= 1e-6


@pytest.mark.parametrize("shape", [(2, 40, 56), (1, 70, 100)])   # < one 32 x 32 tile row / ragged tiles
def test_softsplat_fused_vs_oracle(shape):
    """the one-pass splat (32 x 32 target tiles in shared memory, scan region bounded by the per-sample max |flow|): NaN / inf flows,
    flows that leave the frame (holes stay 0), an infinite bound (sample with an inf flow: the scan degrades to the whole frame)"""
    n, h, w = shape
    lat = rnd(n, 16, h, w, seed=1)
    flow = rnd(n, 2, h, w, seed=2, scale=4.0)
    flow[0, 0, 3, 3] = float("nan")
    flow[n - 1, 1, 5, 7] = float("inf")
    flow[0, :, 0, 0] = torch.tensor([2.0, 1.0], device=DEV)
    flow[0, :, 10:14, 10:14] = 100.0
    metric = 0.5 + rnd(n, 1, h, w, seed=3).abs()
    t = torch.tensor([0.5, 0.25][:n], device=DEV)
    absmax = torch.nan_to_num(flow.abs(), nan=0.0, posinf=float("inf")).amax(dim=(1, 2, 3)).contiguous()   # what absmax_per_sample yields (fmaxf drops NaN)
    for mode in (0, 1):
        got = K.nchw(K.softsplat_fused(K.nhwc(lat), K.nhwc(flow), K.nhwc(metric), t, mode, absmax))
        sc = (t if mode == 0 else (1 - t)).view(n, 1, 1, 1)
        ref = O.softsplat_linear_zeroeps(lat.cpu(), (flow * sc).cpu(), metric.cpu()).to(DEV)
        err = (got - ref).abs()
        assert err.max().item() <= 3e-4 and err.mean().item() <= 1e-6


def test_backwarp_vs_oracle():
    src = rnd(2, 19, 24, 40, seed=1)
    flow = rnd(2, 2, 24, 40, seed=2, scale=6.0)   # includes out-of-frame targets (border clamp)
    got = K.nchw(K.backwarp(K.nhwc(src), K.nhwc(flow)))
    ref = O.backwarp(src.cpu(), flow.cpu()).to(DEV)
    assert (got - ref).abs().max().item() <= 1e-4  # coordinate round trip differs by ~1 ulp of 40 px


@pytest.mark.parametrize("scale", [0.25, 0.5, 2.0, 4.0])
def test_resize_vs_interpolate(scale):
    x = rnd(2, 5, 24, 40, seed=1)
    got = K.nchw(K.resize(K.nhwc(x), scale, 1.5))
    ref = 1.5 * F.interpolate(x, scale_factor=scale, mode="bilinear", align_corners=False)
    assert got.shape == ref.shape
    assert (got - ref).abs().max().item() <= 1e-5


def test_corr_volume_pyramid_lookup():
    n, h, w, C = 2, 16, 20, 256
    fa, fb = rnd(n, C, h, w, seed=1), rnd(n, C, h, w, seed=2)
    lv = K.corr_pyramid(K.nhwc(fa), K.nhwc(fb))
    vol = O.all_pairs_corr(fa.cpu(), fb.cpu())
    pyr = O.corr_pyramid(vol.reshape(n * h * w, 1, h, w))
    for a, b in zip(lv, pyr):
        assert a.shape == b[:, 0].shape
        assert (a.cpu() - b[:, 0]).abs().max().item() <= 1e-4   # K=256 fp32 dot products, |v| ~ 16
    coords = O.coords_grid(n, h, w) + 3.0 * torch.randn(n, 2, h, w, generator=torch.Generator().manual_seed(3))
    coords[0, :, 0, 0] = torch.tensor([-20.0, 50.0])  # far outside: zero padding
    got = K.nchw(K.corr_lookup(lv, K.nhwc(coords.to(DEV))))
    ref = O.corr_lookup(pyr, coords)
    assert (got.cpu() - ref).abs().max().item() <= 2e-3  # bilinear weights after a float normalise round trip x |v|~16
    # the transposed-window quirk (raft/corr.py:152-158): channel a*9+b <-> (dx, dy) = (a-4, b-4)
    c0 = O.coords_grid(1, h, w)
    g2 = K.nchw(K.corr_lookup([l[: h * w] for l in lv], K.nhwc(c0.to(DEV))))
    v0 = lv[0][: h * w].view(h, w, h, w)
    y, x = 8, 9
    assert abs(g2[0, 5 * 9 + 3, y, x].item() - v0[y, x, y - 1, x + 1].item()) <= 1e-4  # a=5 -> dx=+1, b=3 -> dy=-1


@pytest.mark.parametrize("h,w", [(16, 20), (34, 61), (17, 24)])
def test_corr_lookup_direct_vs_oracle(h, w):
    """volume-free BidirCorrBlock lookup (raft/corr.py:23-93): same 324 channels as the oracle's volume -> pyramid -> lookup.
    Target features are rounded to half in the kernel (11-bit significand, the plain-TF32 volume GEMM's operand precision):
    |corr| ~ 16, 256 products -> ~1e-2 absolute."""
    n, C = 2, 256
    fa, fb = rnd(n, C, h, w, seed=1), rnd(n, C, h, w, seed=2)
    vol = O.all_pairs_corr(fa.cpu(), fb.cpu())
    pyr = O.corr_pyramid(vol.reshape(n * h * w, 1, h, w))
    coords = O.coords_grid(n, h, w) + 3.0 * torch.randn(n, 2, h, w, generator=torch.Generator().manual_seed(3))
    coords[0, :, 0, 0] = torch.tensor([-20.0, 50.0])     # far outside: zero padding
    coords[0, :, 1, 1] = torch.tensor([3.0, 5.0])        # exactly integral coordinates
    coords[1, :, 2, 3] = torch.tensor([-0.5, h - 0.5])   # straddling the border
    got = K.nchw(K.corr_lookup_direct(K.nhwc(fa), K.nhwc(fb), K.nhwc(coords.to(DEV))))
    ref = O.corr_lookup(pyr, coords)
    d = (got.cpu() - ref).abs()
    assert d.max().item() <= 3e-2 and d.mean().item() <= 2e-3
    # with targets that are exactly representable in half the only difference is the fp32 summation order
    fbh = fb.half().float()
    vol = O.all_pairs_corr(fa.cpu(), fbh.cpu())
    pyr0 = O.corr_pyramid(vol.reshape(n * h * w, 1, h, w))
    got = K.nchw(K.corr_lookup_direct(K.nhwc(fa), K.nhwc(fbh), K.nhwc(coords.to(DEV))))
    ref = O.corr_lookup(pyr0[:1] + pyr[1:], coords)
    assert (got.cpu() - ref)[:, :81].abs().max().item() <= 2e-3   # level 0 (the pooled levels round their pooled features again)


def test_instnorm():
    x = rnd(2, 96, 20, 28, seed=1, scale=3.0) + 2.0
    got = K.nchw(K.instnorm(K.nhwc(x), True))
    ref = F.relu(F.instance_norm(x.double(), eps=1e-5)).float()
    assert (got - ref).abs().max().item() <= 2e-5


def test_convex_upsample():
    flow = rnd(2, 2, 16, 20, seed=1, scale=2.0)
    mask = rnd(2, 576, 16, 20, seed=2)
    got = K.nchw(K.convex_upsample(K.nhwc(flow), K.nhwc(mask)))
    ref = O.convex_upsample(flow.cpu(), mask.cpu()).to(DEV)
    assert (got - ref).abs().max().item() <= 2e-5


@pytest.mark.parametrize("times", [1, 2])
def test_pixel_shuffle(times):
    x = rnd(2, 128, 8, 12, seed=1)
    got = K.nchw(K.pixel_shuffle(K.nhwc(x), times))
    ref = x
    for _ in range(times):
        ref = F.pixel_shuffle(ref, 2)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("h,w", [(16, 20), (34, 60), (17, 31)])
def test_corr_pool_pyramid_matches_levelwise(h, w):
    """the fused three-level pooling is bit-identical to three corr_pool passes (raft/corr.py:139-142)"""
    import ctypes as C
    lib = K.default_lib()
    rows = 300
    l0 = torch.randn(rows, h, w, device="cuda")
    ref = [l0]
    hh, ww = h, w
    for _ in range(3):
        nxt = torch.empty(rows, hh // 2, ww // 2, device="cuda")
        lib.check(lib.dll.gimmvfi_op_corr_pool(C.c_void_p(ref[-1].data_ptr()), C.c_void_p(nxt.data_ptr()), rows, hh, ww, K._stream(l0)))
        ref.append(nxt); hh, ww = hh // 2, ww // 2
    got = [torch.empty_like(r) for r in ref[1:]]
    lib.check(lib.dll.gimmvfi_op_corr_pool_pyramid(C.c_void_p(l0.data_ptr()), *[C.c_void_p(g.data_ptr()) for g in got], rows, h, w, K._stream(l0)))
    torch.cuda.synchronize()
    for g, r in zip(got, ref[1:]):
        assert torch.equal(g, r)
    assert torch.allclose(got[0], torch.nn.functional.avg_pool2d(l0[:, None], 2, 2)[:, 0], atol=1e-6)


@pytest.mark.parametrize("case", [(256, 2, 3, 24, 40, 2, True), (128, 1, 3, 17, 23, 1, False), (256, 2, 5, 16, 20, 1, True)])
def test_conv_narrow_cout(case):
    """1-2 output channels over a wide input (RAFT FlowHead.conv2, raft/update.py:6-14): warp-per-pixel fp32 kernel, + residual"""
    cin, cout, k, H, W, n, use_res = case
    g = torch.Generator().manual_seed(5)
    x = torch.randn(n, cin, H, W, generator=g).cuda()
    w = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).cuda()
    b = (0.1 * torch.randn(cout, generator=g)).cuda()
    res = torch.randn(n, cout, H, W, generator=g).cuda() if use_res else None
    got = K.nchw(K.conv2d(K.nhwc(x), w, b, pad=(k // 2, k // 2), residual=K.nhwc(res) if use_res else None))
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=k // 2)
    if use_res:
        ref = ref + res.double()
    assert (got.double() - ref).abs().max().item() <= 2e-5


@pytest.mark.parametrize("case", [(2, 16, 3, 40, 56, 2, 0), (3, 16, 3, 17, 23, 1, 2), (4, 16, 5, 16, 20, 1, 1)])
def test_conv_thin_cin(case):
    """very few input channels, 16 outputs (GIMM cnn_encoder.0: 3x3 2 -> 16, gimmvfi_r.py:86-88): thread-per-pixel fp32 kernel"""
    cin, cout, k, H, W, n, act = case
    g = torch.Generator().manual_seed(9)
    x = torch.randn(n, cin, H, W, generator=g).cuda()
    w = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).cuda()
    b = (0.1 * torch.randn(cout, generator=g)).cuda()
    got = K.nchw(K.conv2d(K.nhwc(x), w, b, pad=(k // 2, k // 2), act=act))
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=k // 2)
    ref = {0: lambda v: v, 1: F.relu, 2: lambda v: F.leaky_relu(v, 0.1)}[act](ref)
    assert (got.double() - ref).abs().max().item() <= 2e-5


@pytest.mark.parametrize("fp32_class", [1, 0])
@pytest.mark.parametrize("shape", [(1, 24, 40), (2, 50, 37), (1, 128, 160)])   # incl. pixel counts that are not a multiple of the 64-pixel tile
def test_hyponet_fused_vs_oracle(shape, fp32_class, weights0):
    """The fused wgmma HypoNet kernels (csrc/hyponet.cu) against the oracle's hyponet_forward (modules/hyponet.py:71-146) in fp32.
    fp32_class = 1 (the forward pass's default): fp16 hi/lo operand pairs in layers 1-3, CUDA-core fp32 layers 0 and 4 -> fp32-level
    agreement (the output feeds (2 o - 1) * max|flow|: 1e-5 here is 1e-3 px at 40 px motion).  fp32_class = 0: TF32 layer 0 + half
    hidden activations -> operand rounding at 2^-11."""
    import ctypes as C

    from gimmvfi_b200 import EngineHandle
    from gimmvfi_b200._lib import view_of

    n, h, w = shape
    eng = EngineHandle(DEV)
    eng.load_state_dict(weights0)
    g = torch.Generator().manual_seed(5)
    lat = (torch.randn(n, h, w, 32, generator=g) * 0.7)
    coord = torch.cat([O.sample_coord_input(1, (h, w), [0.25 + 0.5 * i]) for i in range(n)], 0)   # (n,1,h,w,3), a different t per sample
    lat = K.tf32_rn(lat)   # the producing conv stores TF32-representable values (conv_tc.cu round_out): both kernels see them exactly
    ref = O.hyponet_forward({k: v.double() for k, v in weights0.items() if k.startswith("hyponet.")}, coord.double(), lat.double()).float()   # (n,1,h,w,2)
    lat_d = lat.to(DEV)
    out = torch.empty(n, h, w, 2, device=DEV)
    cd = coord.to(DEV).contiguous()
    eng.lib.check(eng.lib.dll.gimmvfi_op_hyponet(eng._h, C.byref(view_of(lat_d)), C.c_void_p(cd.data_ptr()), C.byref(view_of(out)), fp32_class,
                                                 C.c_void_p(torch.cuda.current_stream().cuda_stream)), eng._h)
    torch.cuda.synchronize()
    d = (out.cpu() - ref[:, 0]).abs()
    print("hyponet fused", shape, "fp32_class", fp32_class, "max %.3e mean %.3e" % (d.max().item(), d.mean().item()))
    assert torch.isfinite(out).all()
    if fp32_class:
        assert d.max().item() <= 2e-5 and d.mean().item() <= 2e-6   # MUFU sin (~1e-6 per activation) is the largest term
    else:
        assert d.max().item() <= 4e-3 and d.mean().item() <= 5e-4
