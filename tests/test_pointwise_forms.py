"""The synthesis tail's pointwise ops (resize_bilinear, backwarp, copy_channels in csrc/ops_pointwise.cu) in every storage form Engine::run
uses, through gimmvfi_op_tail_pointwise, against float64 — on the GPU (`gpu` marker) and on the CPU build of the same sources (tests/hostsim;
not a product path), which runs the same functors.  The forms are instances of one functor template per op, K<L, Any>: L = 4 channels
per item (16-byte fp32 / 8-byte half accesses) or 1, Any = half-aware storage; resize's half-aware form is ResizeAnyK4.  Tolerances are
written next to each check."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim"))
import gimmvfi_r_oracle as O
import gpu_ops as K
from gimmvfi_b200._lib import Lib, default_lib

BACKENDS = [pytest.param("hostsim", id="hostsim"), pytest.param("gpu", id="b200", marks=pytest.mark.gpu)]


@pytest.fixture(scope="module", params=BACKENDS)
def be(request):
    if request.param == "gpu":
        return default_lib(), "cuda"
    import harness
    return Lib(harness.build_hostsim()), "cpu"


def rnd(dev, *s, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*s, generator=g) * scale).to(dev)


def half_ulp(v):
    """spacing of IEEE half around |v| (subnormal spacing below 2^-14)"""
    return torch.pow(2.0, torch.floor(torch.log2(v.abs().clamp(min=2.0 ** -14))) - 10)


def interp64(x_nhwc, scale):
    return K.nhwc(F.interpolate(K.nchw(x_nhwc.double()), scale_factor=scale, mode="bilinear", align_corners=False))


@pytest.mark.parametrize("scale", [2, 4])
@pytest.mark.parametrize("c,ld,mult", [(6, 8, "inv"), (3, 4, 1.0), (9, 12, 1.0)])
@pytest.mark.parametrize("widened", [True, False])
def test_resize_widened_lane_views(be, scale, c, ld, mult, widened):
    """The ds_factor resize of the four heads (F0 / F1 6-of-8, Mk 3-of-4, Rs 9-of-12 lanes, flows x 1/ds): the engine widens the views to
    the pixel stride so that ResizeK<4, false> runs and the padding lanes ride along; the narrow view runs ResizeK<1, false>.  Both must
    give the real channels of mult * interpolate(src) in fp32 (exact bilinear weights at power-of-two scales: a few ulps of |src|)."""
    lib, dev = be
    n, h, w = 2, 20, 36
    mult = float(scale) if mult == "inv" else mult
    src = rnd(dev, n, h, w, ld, seed=7, scale=40.0)
    dst = torch.full((n, h * scale, w * scale, ld), 7.0, device=dev)
    K.tail_op(K.TAIL_RESIZE, src, dst, scale=scale, mult=mult, src_ch=ld if widened else c, dst_ch=ld if widened else c, lib=lib)
    ref = mult * interp64(src, scale)
    d = (dst[..., :c].double() - ref[..., :c]).abs().max().item()
    print("resize %d-of-%d x%d mult %g widened %s: max |d| %.3e of |ref| <= %.1f" % (c, ld, scale, mult, widened, d, ref.abs().max().item()))
    assert d <= 4 * 2.0 ** -24 * ref[..., :c].abs().max().item()
    if not widened:
        assert (dst[..., c:] == 7.0).all()   # the scalar form leaves the padding lanes alone


@pytest.mark.parametrize("src_half", [False, True])
def test_resize_into_half_concat_slice(be, src_half):
    """ResizeAnyK4: the x4 resize of ft_4 / the flows into the half-precision 273-of-280 concat of precision mode 4 (and the
    half-source form).  The result is the fp32 value rounded to half: within one half ulp of float64 rounded to half, and every channel
    outside the slice untouched."""
    lib, dev = be
    n, h, w = 2, 10, 18
    src = rnd(dev, n, h, w, 128, seed=8, scale=3.0)
    if src_half:
        src = src.half()
    dst = torch.full((n, 4 * h, 4 * w, 280), 5.0, device=dev, dtype=torch.float16 if not src_half else torch.float32)
    K.tail_op(K.TAIL_RESIZE, src, dst, scale=4.0, mult=0.5, dst_ch=128, dst_off=128, lib=lib)
    ref = 0.5 * interp64(src.float(), 4.0)
    got = dst[..., 128:256].double()
    if src_half:
        assert (got - ref).abs().max().item() <= 4 * 2.0 ** -24 * ref.abs().max().item()
    else:
        ratio = ((got - ref.half().double()).abs() / half_ulp(ref)).max().item()
        print("resize fp32 -> half slice: max |d| %.3f half ulps" % ratio)
        assert ratio <= 1.0 + 1e-9
    assert (dst[..., :128] == 5.0).all() and (dst[..., 256:] == 5.0).all()


@pytest.mark.parametrize("c", [1, 2, 4])
@pytest.mark.parametrize("form", ["accumulate", "sigmoid"])
def test_resize_accumulate_and_sigmoid(be, c, form):
    """The update blocks add 2 * resize(dflow, 2) to the flows in place (accumulate); img_warp_4 takes sigmoid(resize(mask4, 4)).  c = 4
    runs ResizeK<4, false>, 1 and 2 ResizeK<1, false>."""
    lib, dev = be
    n, h, w = 2, 12, 20
    src = rnd(dev, n, h, w, c, seed=9, scale=2.0)
    scale, mult = (2.0, 2.0) if form == "accumulate" else (4.0, 1.0)
    old = rnd(dev, n, int(h * scale), int(w * scale), c, seed=10, scale=5.0)
    dst = old.clone()
    K.tail_op(K.TAIL_RESIZE, src, dst, scale=scale, mult=mult, accumulate=form == "accumulate", act=0 if form == "accumulate" else 4, lib=lib)
    r = mult * interp64(src, scale)
    ref = old.double() + r if form == "accumulate" else torch.sigmoid(r)
    d = (dst.double() - ref).abs().max().item()
    print("resize %s c=%d: max |d| %.3e" % (form, c, d))
    assert d <= (4e-6 if form == "accumulate" else 4e-7)


@pytest.mark.parametrize("src_half", [False, True])
def test_backwarp_features_into_half_concat(be, src_half):
    """BackwarpK<4, true>: the warps of the 64-channel up-sampled features (half in mode 4) into the half concat, flows reaching past the
    border.  Within half a half ulp of float64 plus the fp32 coordinate round trip of border_tap (~1 ulp of 40 px times the gradient)."""
    lib, dev = be
    n, h, w = 2, 24, 40
    src = rnd(dev, n, h, w, 64, seed=11)
    flow = rnd(dev, n, h, w, 2, seed=12, scale=8.0)
    if src_half:
        src = src.half()
    dst = torch.full((n, h, w, 280), 5.0, device=dev, dtype=torch.float16)
    K.tail_op(K.TAIL_BACKWARP, src, dst, flow=flow, dst_ch=64, dst_off=128, lib=lib)
    ref = K.nhwc(O.backwarp(K.nchw(src.double()), K.nchw(flow.double())))
    got = dst[..., 128:192].double()
    d = ((got - ref).abs() - 0.5 * half_ulp(ref)).max().item()
    exact = (got == ref.half().double()).double().mean().item()
    print("backwarp -> half (src half %s): max excess over half an ulp %.3e, %.4f of the values equal to float64 rounded" % (src_half, d, exact))
    assert d <= 1e-4 and exact >= 0.98
    assert (dst[..., :128] == 5.0).all() and (dst[..., 192:] == 5.0).all()


def test_backwarp_frames_into_half_concat(be):
    """BackwarpK<1, true>: the 3-channel frame warps (ld 4) into channels 267-269 of the half concat - an offset that is not 4-aligned,
    so the scalar form runs; the padding lane of the frames is never read."""
    lib, dev = be
    n, h, w = 2, 24, 40
    src = rnd(dev, n, h, w, 4, seed=13)
    src[..., 3] = float("nan")
    flow = rnd(dev, n, h, w, 2, seed=14, scale=8.0)
    dst = torch.full((n, h, w, 280), 5.0, device=dev, dtype=torch.float16)
    K.tail_op(K.TAIL_BACKWARP, src, dst, flow=flow, src_ch=3, dst_ch=3, dst_off=267, lib=lib)
    ref = K.nhwc(O.backwarp(K.nchw(src[..., :3].double()), K.nchw(flow.double())))
    got = dst[..., 267:270].double()
    assert torch.isfinite(got).all()
    assert ((got - ref).abs() - 0.5 * half_ulp(ref)).max().item() <= 1e-4
    assert (got == ref.half().double()).double().mean().item() >= 0.98
    assert (dst[..., :267] == 5.0).all() and (dst[..., 270:] == 5.0).all()


@pytest.mark.parametrize("c,ld,off", [(3, 4, 261), (5, 8, 256)])
def test_copy_channels_into_half_slice(be, c, ld, off):
    """CopyK<1, true>: the frames (3 of 4 lanes) and mode 4's fp32 flows / mask (aux5, 5 of 8) into their half concat slices: exactly the
    fp32 values rounded to nearest even, nothing else written."""
    lib, dev = be
    n, h, w = 2, 9, 13
    src = rnd(dev, n, h, w, ld, seed=15, scale=30.0)
    src[0, 0, 0, 0] = 1e5   # saturates to the largest half
    dst = torch.full((n, h, w, 280), 5.0, device=dev, dtype=torch.float16)
    K.tail_op(K.TAIL_COPY, src, dst, src_ch=c, dst_ch=c, dst_off=off, lib=lib)
    want = src[..., :c].clamp(-65504, 65504).half()
    assert torch.equal(dst[..., off:off + c], want)
    assert (dst[..., :off] == 5.0).all() and (dst[..., off + c:] == 5.0).all()
