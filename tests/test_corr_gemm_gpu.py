"""The all-pairs correlation GEMM in the 3xF16 form (corr_gemm.cu) through gimmvfi_op_corr_volume_tc(split=1): against float64 at ragged
shapes (M, N not multiples of 128, N < 128, RAFT's pooled level sizes 17x30 and 34x60, whose row pitch of 510 targets takes the plain
stores and of 2040 the TMA stores), K = 64 / 128 / 256; run-to-run bit equality; and a RAFT pair alone against the same pair inside
a pair list, whose pyramid reads the pre-split planes of every frame at the pair's offsets."""
import ctypes as C

import pytest
import torch

import gpu_ops as K

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
