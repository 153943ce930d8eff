"""GIMM.forward on coordinate grids of another size than the flows, on the GPU: the model against the unmodified reference's
outputs (tests/golden/manifest_gimm_grid.json), the resampling HypoNet kernel (hyponet_fused3_resample) against the oracle and
against the composed form (resize, then the equal-size kernel)."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gimmvfi_r_oracle as O
import gpu_ops as K
from conftest import GOLDEN_DIR
from gimmvfi_b200.gimm import GIMM, GIMM_KEY_PREFIXES
from gimmvfi_b200.synth import synth_flow_pair
from golden import load as load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"

with open(os.path.join(GOLDEN_DIR, "manifest_gimm_grid.json")) as _f:
    MANIFEST = json.load(_f)


def _gimm(weights0, mode):
    m = GIMM(seed=0).to(DEV).eval()
    m.load_state_dict({k: v for k, v in weights0.items() if k.startswith(GIMM_KEY_PREFIXES)}, strict=True)
    m.tensor_cores = mode
    return m


def _run_fixture(m, meta):
    B, H, W, ts = meta["B"], meta["H"], meta["W"], meta["timesteps"]
    ori = synth_flow_pair(B, H, W, seed=meta["flow_seed"])
    xs, _ = O.normalize_flow(ori)
    coord = [m.sample_coord_input(B, (H, W), [t], upsample_ratio=meta["upsample_ratio"], device=DEV) for t in ts]
    return m(xs.to(DEV), coord, True, ori.to(DEV), [t * torch.ones(B, device=DEV) for t in ts]), (xs, ori, coord)


@pytest.mark.parametrize("mode", [1, 0])
@pytest.mark.parametrize("name", sorted(MANIFEST))
def test_gimm_on_grid_matches_reference_golden(name, mode, weights0):
    meta = MANIFEST[name]
    g = load_golden(name)
    m = _gimm(weights0, mode)
    out, (xs, ori, coord) = _run_fixture(m, meta)
    B, Hc, Wc = meta["B"], meta["Hc"], meta["Wc"]
    tol = 2e-5 if mode == 0 else 5e-3   # as tests/test_gimm_gpu.py: fp32 CUDA cores / TF32 convolutions before the fp32-class HypoNet
    for i in range(len(meta["timesteps"])):
        assert out[i].shape == (B, 2, 1, Hc, Wc)
        err = np.abs(out[i].cpu().numpy() - g["out_%d" % i]).max()
        print(name, "mode", mode, "max err %.3e" % err)
        assert err <= tol
    one = m(xs.to(DEV), coord[0], False, ori.to(DEV), meta["timesteps"][0] * torch.ones(B, device=DEV))   # tensor form
    assert one.shape == (B, 1, Hc, Wc, 2)


def test_gimm_list_form_with_two_grid_sizes(weights0):
    B, H, W = 1, 64, 96
    m = _gimm(weights0, 0)
    ori = synth_flow_pair(B, H, W, seed=5)
    xs, _ = O.normalize_flow(ori)
    spec = [(0.25, 2.0), (0.5, 1.0), (0.75, 2.0)]
    coord = [m.sample_coord_input(B, (H, W), [t], upsample_ratio=r, device=DEV) for t, r in spec]
    tt = [t * torch.ones(B, device=DEV) for t, _ in spec]
    out = m(xs.to(DEV), coord, True, ori.to(DEV), tt)
    with torch.no_grad():
        ref = O.gimm_forward(weights0, xs, [c.cpu() for c in coord], ori, [t.cpu() for t in tt])
    for o, r in zip(out, ref):
        assert o.shape == r.shape
        assert (o.cpu() - r).abs().max().item() <= 2e-5


def test_gimm_larger_resolution_on_grid_matches_oracle(weights0):
    """448x256 flows queried at r = 2 (896x512), the default tensor-core mode vs the CPU oracle"""
    B, H, W = 1, 256, 448
    m = _gimm(weights0, 1)
    ori = synth_flow_pair(B, H, W, seed=9)
    xs, _ = O.normalize_flow(ori)
    coord = [m.sample_coord_input(B, (H, W), [0.5], upsample_ratio=2.0, device=DEV)]
    out = m(xs.to(DEV), coord, True, ori.to(DEV), [0.5 * torch.ones(B, device=DEV)])[0].cpu()
    assert out.shape == (B, 2, 1, 2 * H, 2 * W)
    with torch.no_grad():
        ref = O.gimm_forward(weights0, xs, [c.cpu() for c in coord], ori, [0.5 * torch.ones(B)])[0]
    d = (out - ref).abs()
    print("256x448 r=2 max %.3e mean %.3e" % (d.max().item(), d.mean().item()))
    assert d.max().item() <= 5e-3 and d.mean().item() <= 5e-4


def _op_hyponet(eng, lat_d, coord_d, out, fp32_class=1):
    from gimmvfi_b200._lib import view_of

    eng.lib.check(eng.lib.dll.gimmvfi_op_hyponet(eng._h, C.byref(view_of(lat_d)), C.c_void_p(coord_d.data_ptr()), C.byref(view_of(out)),
                                                 fp32_class, C.c_void_p(torch.cuda.current_stream().cuda_stream)), eng._h)


def _latent_and_grid(n, h, w, r, seed=5):
    g = torch.Generator().manual_seed(seed)
    lat = K.tf32_rn(torch.randn(n, h, w, 32, generator=g) * 0.7)
    coord = torch.cat([O.sample_coord_input(1, (h, w), [0.25 + 0.5 * i], r) for i in range(n)], 0)   # (n,1,hc,wc,3)
    return lat, coord


@pytest.mark.parametrize("shape,r", [((2, 25, 37), 2.0), ((1, 50, 37), 0.5), ((1, 36, 40), 1.7)])   # grids of 2x50x74, 25x18, 61x68 px
def test_hyponet_resample_vs_oracle(shape, r, weights0):
    """hyponet_fused3_resample against the oracle's hyponet_forward (F.interpolate to the grid, then the MLP) in fp64; pixel counts
    that are not a multiple of the 64-pixel tile, and a grid smaller than the latent."""
    from gimmvfi_b200 import EngineHandle

    n, h, w = shape
    eng = EngineHandle(DEV)
    eng.load_state_dict(weights0)
    lat, coord = _latent_and_grid(n, h, w, r)
    hc, wc = coord.shape[2], coord.shape[3]
    ref = O.hyponet_forward({k: v.double() for k, v in weights0.items() if k.startswith("hyponet.")}, coord.double(), lat.double()).float()
    out = torch.empty(n, hc, wc, 2, device=DEV)
    _op_hyponet(eng, lat.to(DEV), coord.to(DEV).contiguous(), out)
    torch.cuda.synchronize()
    d = (out.cpu() - ref[:, 0]).abs()
    print("hyponet resample", shape, "->", (hc, wc), "max %.3e mean %.3e" % (d.max().item(), d.mean().item()))
    assert torch.isfinite(out).all()
    assert d.max().item() <= 2e-5 and d.mean().item() <= 2e-6   # the fp32-class bar of test_hyponet_fused_vs_oracle
    with pytest.raises(Exception):   # the TF32 kernel has no resampling form
        _op_hyponet(eng, lat.to(DEV), coord.to(DEV).contiguous(), out, fp32_class=0)


@pytest.mark.parametrize("r", [2.0, 0.5, 1.7])
def test_hyponet_resample_equals_composed_form(r, weights0):
    """The resampling kernel against resize-into-a-buffer + the equal-size kernel on the same inputs.  r = 2 and 0.5 resize with
    the engine's resize_bilinear (its scale 1 / r is then exactly h / hc); r = 1.7 has different y and x scales, so the buffer
    comes from PyTorch's upsample_bilinear2d (the same formulas).  Layers 1-4 are the same code: the forms differ only by the
    rounding of the interpolated latent."""
    from gimmvfi_b200 import EngineHandle

    eng = EngineHandle(DEV)
    eng.load_state_dict(weights0)
    lat, coord = _latent_and_grid(2, 68, 120, r, seed=6)
    lat_d, coord_d = lat.to(DEV), coord.to(DEV).contiguous()
    hc, wc = coord.shape[2], coord.shape[3]
    if r != 1.7:
        big = K.resize(lat_d, r)
    else:
        big = F.interpolate(lat_d.permute(0, 3, 1, 2), size=(hc, wc), mode="bilinear", align_corners=False).permute(0, 2, 3, 1).contiguous()
    assert big.shape == (2, hc, wc, 32)
    composed = torch.empty(2, hc, wc, 2, device=DEV)
    fused = torch.empty(2, hc, wc, 2, device=DEV)
    _op_hyponet(eng, big, coord_d, composed)
    _op_hyponet(eng, lat_d, coord_d, fused)
    torch.cuda.synchronize()
    d = (fused - composed).abs().max().item()
    print("resample vs composed r=%g: max|d| %.3e, identical pixels %.4f" % (r, d, (fused == composed).all(-1).float().mean().item()))
    assert d <= 1e-6
