"""f16 tensor-core convolution (csrc/conv_tc.cu) at a size with several pixel tiles per persistent CTA.

168 x 240 = 21 x 15 = 315 pixel tiles of 8 x 16 (an odd count): the CTAs loop over tiles with the producer running ahead
by several stages, at the final decoder trunk's width (cout 256), with the half residual and two
half input segments of ResBlock conv5."""
import pytest
import torch
import torch.nn.functional as F

import gpu_ops as K

pytestmark = pytest.mark.gpu
DEV = "cuda"
H, W = 168, 240


def rnd(*s, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*s, generator=g) * scale).to(DEV)


@pytest.mark.parametrize("out_half", [True, False])
def test_conv2d_tc_f16_operands_many_tiles(out_half):
    cin, cout, k, n = 256, 256, 3, 1
    x = rnd(n, cin, H, W, seed=1)
    w = rnd(cout, cin, k, k, seed=2, scale=1.0 / (cin * k * k) ** 0.5)
    b = rnd(cout, seed=3, scale=0.1)
    slope = 0.25 + 0.1 * rnd(cout, seed=4)
    got = K.conv2d_tc_f16(K.nhwc(x).half(), w, b, 3, slope, out_half=out_half)
    ref = F.prelu(F.conv2d(x.half().double(), w.half().double(), b.double(), padding=k // 2), slope.double()).float()
    err = (K.nchw(got.float()) - ref).abs().max().item()
    print("f16 168x240", out_half, "err %.3e ref absmax %.3e" % (err, ref.abs().max().item()))
    assert err <= 1e-3 * max(1.0, ref.abs().max().item())


def test_conv2d_tc_f16_resblock_tail_many_tiles():
    n = 1
    a = rnd(n, 192, H, W, seed=1); s2 = rnd(n, 64, H, W, seed=2); res = rnd(n, 256, H, W, seed=3)
    w = rnd(256, 256, 3, 3, seed=4, scale=1.0 / (256 * 9) ** 0.5)
    b = rnd(256, seed=5, scale=0.1)
    slope = 0.25 + 0.1 * rnd(256, seed=6)
    ah, sh, rh = K.nhwc(a).half(), K.nhwc(s2).half(), K.nhwc(res).half()
    got = K.conv2d_tc_f16(ah, w, b, 0, None, residual=rh, act2=3, slope2=slope, x1_nhwc=sh, out_half=True)
    xin = torch.cat([a.half().double(), s2.half().double()], 1)
    ref = F.prelu(F.conv2d(xin, w.half().double(), b.double(), padding=1) + res.half().double(), slope.double()).float()
    err = (K.nchw(got.float()) - ref).abs().max().item()
    print("f16 resblock tail 168x240 err %.3e" % err)
    assert err <= 1e-3 * max(1.0, ref.abs().max().item())


def test_conv2d_tc_tf32_two_segments_residual_many_tiles():
    """the TF32 form of the trunk width over many tiles: two fp32 input segments (192 + 64 channels), residual, PReLU after the add"""
    a = rnd(1, 256, H, W, seed=1); s = rnd(1, 64, H, W, seed=2); res = rnd(1, 256, H, W, seed=5)
    w = rnd(256, 256, 3, 3, seed=3, scale=0.02)
    b = rnd(256, seed=4, scale=0.1)
    slope = 0.25 + 0.1 * rnd(256, seed=6)
    a_nhwc = K.nhwc(a)
    got = K.nchw(K.conv2d_tc(a_nhwc, w, b, 0, None, K.nhwc(res), 3, slope, x1_nhwc=K.nhwc(s), in_view=K.view_of(a_nhwc, channels=192)))
    xin = torch.cat([a[:, :192], s], 1)
    ref = F.prelu(res.double() + F.conv2d(K.tf32_trunc(xin).double(), K.tf32_rn(w).double(), b.double(), padding=1), slope.double()).float()
    err = (got - ref).abs().max().item()
    print("tf32 two segments + residual 168x240 err %.3e" % err)
    assert err <= 5e-5 + 2.0 ** -11 * ref.abs().max().item()
