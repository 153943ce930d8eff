"""csrc/conv_wide.cu: the final decoder trunk's 3x3 f16 convolution with each 64-channel K block's tile + halo loaded once.

The three trunk forms of a ResBlock (fi_components.py:97-154): conv1 on one 256-channel input; conv3 on two segments (192 channels of a
256-wide tensor + the 64-channel side output); conv5 on two segments with the half residual updated in place and PReLU after the add.
Against float64 F.conv2d on the half-rounded operands (the bar of test_conv_tc_wide_gpu.py), and against conv2d_tc_f16 on the same
inputs: the two kernels sum K in a different order, so a stored half may differ by one rounding step."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

import gpu_ops as K
from gimmvfi_b200._lib import View, default_lib

pytestmark = pytest.mark.gpu
DEV = "cuda"
PRELU = 3


def rnd(*s, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*s, generator=g) * scale).to(DEV)


def conv2d_wide(x_nhwc, w, b, act1=0, slope1=None, residual=None, act2=0, slope2=None, x1_nhwc=None, in_view=None, out=None,
                out_view=None):
    """gimmvfi_op_conv2d_wide on half NHWC tensors; in_view / out_view: channel-slice views of x / out (out given: written in place,
    e.g. the residual's own buffer)"""
    lib = default_lib()
    cout, cin, kh, kw = w.shape
    assert (kh, kw) == (3, 3) and x_nhwc.dtype == torch.float16
    pw_h = K.pack_weight_tc_f16(w)
    bb = torch.zeros((K.tc_cout_pad(cout) + 31) // 32 * 32 + 128, device=w.device)
    bb[:cout] = b
    n, h, wd, _ = x_nhwc.shape
    if out is None:
        out = torch.empty(n, h, wd, cout, device=w.device, dtype=torch.float16)
    mask = 1 | (2 if out.dtype == torch.float16 else 0) | (4 if (residual is not None and residual.dtype == torch.float16) else 0)
    V = lambda t: C.byref(K.view_of(t)) if t is not None else None
    P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    v0 = in_view if in_view is not None else K.view_of(x_nhwc)
    vo = out_view if out_view is not None else K.view_of(out)
    stream = C.c_void_p(torch.cuda.current_stream(out.device).cuda_stream)
    lib.check(lib.dll.gimmvfi_op_conv2d_wide(C.byref(v0), V(x1_nhwc), P(pw_h), P(bb), cin, cout, act1, P(slope1), V(residual), act2,
                                             P(slope2), mask, C.byref(vo), stream))
    return out


def layer(seed):
    w = rnd(256, 256, 3, 3, seed=seed, scale=1.0 / (256 * 9) ** 0.5)
    b = rnd(256, seed=seed + 1, scale=0.1)
    slope = 0.25 + 0.1 * rnd(256, seed=seed + 2)
    return w, b, slope


def ref_conv(xin, w, b):
    return F.conv2d(xin.half().double(), w.half().double(), b.double(), padding=1)


def check(got, ref, tag):
    err = (K.nchw(got.float()) - ref.float()).abs().max().item()
    amax = ref.abs().max().item()
    print("%s err %.3e ref absmax %.3e" % (tag, err, amax))
    assert err <= 1e-3 * max(1.0, amax)


def check_agree(a, b, tag):
    d = (a.float() - b.float()).abs().max().item()
    amax = b.float().abs().max().item()
    print("%s max|wide - tc| %.3e" % (tag, d))
    assert d <= 2.0 ** -10 * max(1.0, amax)


SIZES = [(1, 1088, 1920), (1, 37, 45), (2, 50, 70), (1, 168, 232)]   # pair1080; ragged (H % 16, W % 8 != 0); n = 2; 319 pixel tiles


@pytest.mark.parametrize("n,h,w", SIZES)
def test_conv_wide_one_input(n, h, w):
    x = rnd(n, 256, h, w, seed=1)
    wt, b, slope = layer(10)
    xh = K.nhwc(x).half()
    got = conv2d_wide(xh, wt, b, PRELU, slope)
    check(got, F.prelu(ref_conv(x, wt, b), slope.double()), "conv1 %dx%dx%d" % (n, h, w))
    check_agree(got, K.conv2d_tc_f16(xh, wt, b, PRELU, slope), "conv1 %dx%dx%d" % (n, h, w))


@pytest.mark.parametrize("n,h,w", SIZES)
def test_conv_wide_two_segments(n, h, w):
    a = rnd(n, 256, h, w, seed=2); s1 = rnd(n, 64, h, w, seed=3)
    wt, b, slope = layer(20)
    ah, sh = K.nhwc(a).half(), K.nhwc(s1).half()
    got = conv2d_wide(ah, wt, b, PRELU, slope, x1_nhwc=sh, in_view=K.view_of(ah, channels=192))
    ref = F.prelu(ref_conv(torch.cat([a[:, :192], s1], 1), wt, b), slope.double())
    check(got, ref, "conv3 %dx%dx%d" % (n, h, w))
    tc = K.conv2d_tc_f16(ah[..., :192].contiguous(), wt, b, PRELU, slope, x1_nhwc=sh)
    check_agree(got, tc, "conv3 %dx%dx%d" % (n, h, w))


@pytest.mark.parametrize("n,h,w", SIZES)
def test_conv_wide_residual_in_place(n, h, w):
    bt = rnd(n, 256, h, w, seed=4); s2 = rnd(n, 64, h, w, seed=5); x = rnd(n, 256, h, w, seed=6)
    wt, b, slope = layer(30)
    bh, sh, xh = K.nhwc(bt).half(), K.nhwc(s2).half(), K.nhwc(x).half()
    xin = torch.cat([bt[:, :192], s2], 1)
    ref = F.prelu(ref_conv(xin, wt, b) + K.nchw(xh).double(), slope.double())
    tc = K.conv2d_tc_f16(bh[..., :192].contiguous(), wt, b, 0, None, residual=xh, act2=PRELU, slope2=slope, x1_nhwc=sh)
    got = conv2d_wide(bh, wt, b, 0, None, residual=xh, act2=PRELU, slope2=slope, x1_nhwc=sh, in_view=K.view_of(bh, channels=192), out=xh)
    assert got.data_ptr() == xh.data_ptr()
    check(got, ref, "conv5 in place %dx%dx%d" % (n, h, w))
    check_agree(got, tc, "conv5 in place %dx%dx%d" % (n, h, w))


@pytest.mark.parametrize("out_half", [True, False])
def test_conv_wide_output_slice_keeps_other_channels(out_half):
    """the output is channels [32, 288) of a 320-wide buffer filled with a sentinel: nothing outside the slice is written"""
    n, h, w = 1, 40, 56
    x = rnd(n, 256, h, w, seed=7)
    wt, b, slope = layer(40)
    xh = K.nhwc(x).half()
    dt = torch.float16 if out_half else torch.float32
    buf = torch.full((n, h, w, 320), 7.0, dtype=dt, device=DEV)
    vo = View(buf.data_ptr() + buf.element_size() * 32, n, h, w, 256, 320, h * w * 320)
    conv2d_wide(xh, wt, b, PRELU, slope, out=buf, out_view=vo)
    assert bool((buf[..., :32] == 7.0).all()) and bool((buf[..., 288:] == 7.0).all())
    check(buf[..., 32:288], F.prelu(ref_conv(x, wt, b), slope.double()), "slice out_half=%s" % out_half)


def test_conv_wide_rejects_unaligned_segments():
    """a segment whose channels are not whole 64-channel blocks is not this kernel's (conv_tc keeps it)"""
    x = rnd(1, 256, 16, 16, seed=8)
    wt, b, slope = layer(50)
    xh = K.nhwc(x).half()
    w2 = wt[:, :224]
    with pytest.raises(RuntimeError, match="unsupported"):
        conv2d_wide(xh, w2, b, PRELU, slope, in_view=K.view_of(xh, channels=224))
