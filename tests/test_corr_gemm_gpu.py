"""The all-pairs correlation GEMM in the 3xF16 form (corr_gemm.cu) through gimmvfi_op_corr_volume_tc(split=1): against float64 at ragged
shapes (M, N not multiples of 128, N < 128, RAFT's pooled level sizes 17x30 and 34x60, whose row pitch of 510 targets takes the plain
stores and of 2040 the TMA stores), K = 64 / 128 / 256; run-to-run bit equality; and a RAFT pair alone against the same pair inside
a pair list, whose pyramid reads the pre-split planes of every frame at the pair's offsets.

Past one raster group (groups of 32 M tiles): FlowFormer's 68 x 128 grid at the 2K / 4K settings (8704 pixels: groups of 32, 32 and 4
M tiles, ~35 tiles per CTA) and 4200 pixels (a last group of one M tile); K = 320 / 384 / 512, which fold segments inside the tile's K
loop (an odd number of segments at 320 and 448).  These are held per entry to the fp32-class bound of tests/corr_ref.py."""
import ctypes as C
import math

import pytest
import torch

import gpu_ops as K
from corr_ref import U

pytestmark = pytest.mark.gpu
DEV = "cuda"


def corr_tc(fa, fb):
    h, w, c = fa.shape[1:]
    n = h * w
    vol = torch.full((n, n), float("nan"), device=DEV)
    scratch = torch.empty(2 * n * c + n + 2048, device=DEV)
    lib = K.default_lib()
    lib.check(lib.dll.gimmvfi_op_corr_volume_tc(C.byref(K.view_of(fa)), C.byref(K.view_of(fb)), C.c_void_p(scratch.data_ptr()),
                                                C.c_void_p(vol.data_ptr()), 1, K._stream(vol)))
    torch.cuda.synchronize()
    return vol


@pytest.mark.parametrize("hw", [(5, 7), (9, 14), (17, 30), (34, 60), (24, 40)])
@pytest.mark.parametrize("c", [64, 128, 256])
def test_corr_gemm_3xf16(hw, c):
    h, w = hw
    g = torch.Generator().manual_seed(7 + c)
    fa = torch.randn(1, h, w, c, generator=g).to(DEV)
    fb = torch.randn(1, h, w, c, generator=g).to(DEV)
    vol = corr_tc(fa, fb)
    n = h * w
    ref = (fa.view(n, c).double() @ fb.view(n, c).double().t() / c ** 0.5).float()
    err = (vol - ref).abs().max().item()
    print("corr_gemm_3xf16", hw, "C", c, "err %.3e" % err, "absmax %.2f" % ref.abs().max().item())
    assert torch.isfinite(vol).all()
    assert err <= 3e-5
    assert torch.equal(vol, corr_tc(fa, fb))


def test_corr_gemm_pair_in_list():
    """RAFT.flows: pair (2, 1) alone equals the same pair as the second sample of [(0, 1), (2, 1)], bit for bit; 272x480 frames give
    pyramid levels of 34x60, 17x30, 8x15 and 4x7 targets"""
    from gimmvfi_b200.raft import RAFT

    g = torch.Generator().manual_seed(5)
    frames = (torch.rand(3, 3, 272, 480, generator=g) * 255).to(DEV)
    model = RAFT(seed=0).to(DEV).eval()
    both = model.flows(frames, [(0, 1), (2, 1)], iters=4)
    alone = model.flows(frames, [(2, 1)], iters=4)
    torch.cuda.synchronize()
    assert torch.isfinite(both).all()
    assert torch.equal(both[1:2], alone)


def gemm_bound64(fa, fb):
    """float64 volume and the per-entry bound of an fp32-class K-term dot product's distance from it (corr_ref.GAMMA_DOT at K = 256):
    (K + 16) u sum_k |a_k b_k| / sqrt(K) - recursive summation K u (the GEMM sums segments of 128 terms in fp32), the 3xF16 operand split
    2^-22 per operand and the dropped lo x lo product 2^-22 per term, and the scale"""
    h, w, c = fa.shape[1:]
    a, b = fa.view(h * w, c).double(), fb.view(h * w, c).double()
    ref = a @ b.t() / math.sqrt(c)
    bnd = (c + 16) * U * (a.abs() @ b.abs().t()) / math.sqrt(c)
    return ref, bnd


def ratio(vol, ref, bnd):
    d = (vol.double() - ref).abs()
    return torch.where(d == 0, torch.zeros_like(d), d / bnd).max().item()


@pytest.mark.parametrize("hw,c", [((68, 128), 256), ((42, 100), 256), ((30, 70), 320), ((30, 70), 384), ((20, 56), 448), ((30, 70), 512)],
                         ids=["8704px-K256", "4200px-K256", "2100px-K320", "2100px-K384", "1120px-K448", "2100px-K512"])
def test_corr_gemm_3xf16_raster_groups_and_long_k(hw, c):
    """every entry within the fp32-class bound at shapes past one raster group and at K >= 320; bit equal across two runs; a 1xF16 GEMM
    of the same operands (the lo planes dropped) breaks the bound, so the bound would catch a lost correction term"""
    h, w = hw
    n = h * w
    tiles_m = (n + 127) // 128
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    groups = [min(32, tiles_m - g) for g in range(0, tiles_m, 32)]
    g = torch.Generator().manual_seed(3 + c + n)
    fa = torch.randn(1, h, w, c, generator=g).to(DEV)
    fb = torch.randn(1, h, w, c, generator=g).to(DEV)
    vol = corr_tc(fa, fb)
    ref, bnd = gemm_bound64(fa, fb)
    r = ratio(vol, ref, bnd)
    half = (fa.view(n, c).half().double() @ fb.view(n, c).half().double().t() / math.sqrt(c)).float()
    r_half = ratio(half, ref, bnd)
    print("\ncorr_gemm_3xf16 %dx%d (%d px, M tile groups %s, %.1f tiles per CTA) K %d: max |d| / bound %.3f, max |d| %.3e; 1xF16 %.1f"
          % (h, w, n, groups, tiles_m * tiles_m / sms, c, r, (vol.double() - ref).abs().max().item(), r_half))
    assert torch.isfinite(vol).all()
    assert r <= 1.0 < r_half
    assert torch.equal(vol, corr_tc(fa, fb))
