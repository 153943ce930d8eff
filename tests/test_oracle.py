"""CPU tests of the oracle (oracle/gimmvfi_r_oracle.py) against the golden
fixtures, which are outputs of the UNMODIFIED reference (oracle/make_golden.py).
This is the oracle's pin: the reference itself ships no tests (SURVEY.md §4)."""
import os

import numpy as np
import pytest
import torch

import gimmvfi_r_oracle as O
from conftest import GOLDEN_DIR
from gimmvfi_b200.synth import synth_batch
from golden import load as load_golden

# oracle == reference bit-for-bit in the build container (manifest records 0.0);
# allow for a different BLAS/oneDNN thread split on another host.
TOL = 2e-5


def run_case(name, meta, sd):
    torch.set_grad_enabled(False)
    B, H, W, ts, ds = meta["B"], meta["H"], meta["W"], meta["timesteps"], meta["ds_factor"]
    xs = synth_batch(B, H, W, seed=meta["input_seed"])
    ratio = 1.0 if ds is None else ds
    coord = [(O.sample_coord_input(B, (H, W), [t], ratio), None) for t in ts]
    tt = [t * torch.ones(B) for t in ts]
    return O.gimmvfi_r_forward(sd, xs, coord, tt, ds_factor=ds)


@pytest.mark.parametrize("name", ["r_128x160_t0.5", "r_b2_128x192_t0.25_0.75", "r_ds0.5_256x320_t0.5"])
def test_oracle_matches_reference_golden(name, golden_manifest, weights0):
    meta = golden_manifest[name]
    assert meta["oracle_vs_reference_max_abs"] <= 2e-6
    g = load_golden(name)
    s = int(g["stride"])
    out = run_case(name, meta, weights0)
    for i in range(len(meta["timesteps"])):
        a = out["imgt_pred"][i][..., ::s, ::s].numpy()
        assert a.shape == g["imgt_pred_%d" % i].shape
        assert np.abs(a - g["imgt_pred_%d" % i]).max() <= TOL
        f = out["flowt"][i][..., ::s, ::s].numpy()
        assert np.abs(f - g["flowt_%d" % i]).max() <= 50 * TOL
        w4 = out["other_pred"][i][0][..., :: 2 * s, :: 2 * s].numpy()
        assert np.abs(w4 - g["img_warp_4_%d" % i]).max() <= TOL
    rf = out["raft_flow"][..., :: 2 * s, :: 2 * s].numpy()
    assert np.abs(rf - g["raft_flow"]).max() <= 50 * TOL


@pytest.mark.parametrize("name", ["r8_136x200_t0.5", "r8_b2_128x136_t0.25_0.75", "r8_ds0.5_272x400_t0.5"])
def test_oracle_matches_reference_golden_r8(name, weights0):
    """Frame sizes that are multiples of 8 but not of 32 (oracle/make_golden_r8.py): RAFT on odd h/8 x w/8 grids, a correlation
    pyramid that floors odd levels.  Full-resolution fixtures (stride 1)."""
    import json

    with open(os.path.join(GOLDEN_DIR, "manifest_r8.json")) as f:
        meta = json.load(f)[name]
    assert meta["oracle_vs_reference_max_abs"] <= 2e-6
    g = load_golden(name)
    s = int(g["stride"])
    out = run_case(name, meta, weights0)
    for i in range(len(meta["timesteps"])):
        a = out["imgt_pred"][i][..., ::s, ::s].numpy()
        assert a.shape == g["imgt_pred_%d" % i].shape
        assert np.abs(a - g["imgt_pred_%d" % i]).max() <= TOL
        f = out["flowt"][i][..., ::s, ::s].numpy()
        assert f.shape == g["flowt_%d" % i].shape
        assert np.abs(f - g["flowt_%d" % i]).max() <= 50 * TOL
        w4 = out["other_pred"][i][0][..., :: 2 * s, :: 2 * s].numpy()
        assert np.abs(w4 - g["img_warp_4_%d" % i]).max() <= TOL
        assert np.abs(out["flowt0_pred"][i][1][..., ::s, ::s].numpy() - g["flowt0_4_%d" % i]).max() <= 50 * TOL
    rf = out["raft_flow"][..., :: 2 * s, :: 2 * s].numpy()
    assert np.abs(rf - g["raft_flow"]).max() <= 50 * TOL


def test_output_contract(golden_manifest, weights0):
    """Keys / shapes of the returned dict (gimmvfi_r.py:398-407), incl. the B=1 flowt squeeze."""
    meta = golden_manifest["r_128x160_t0.5"]
    out = run_case("r_128x160_t0.5", meta, weights0)
    assert set(out) == {"imgt_pred", "other_pred", "flowt0_pred", "flowt1_pred", "raft_flow", "ninrflow", "nflow", "flowt"}
    assert out["imgt_pred"][0].shape == (1, 3, 128, 160)
    assert out["flowt"][0].shape == (2, 128, 160)
    assert out["ninrflow"][0].shape == (1, 2, 1, 128, 160)
    assert out["raft_flow"].shape == (1, 2, 2, 128, 160)
    assert out["flowt0_pred"][0][0].shape == (1, 3, 2, 128, 160)
    assert out["flowt0_pred"][0][1].shape == (1, 2, 32, 40)


def test_splat_restatement_vs_bruteforce():
    """forward_splat_sum vs a literal double loop over the kernel body
    (modules/softsplat.py:384-420) incl. out-of-frame targets and non-finite flow."""
    torch.manual_seed(0)
    N, C, H, W = 1, 3, 6, 7
    inp = torch.randn(N, C, H, W)
    flow = torch.randn(N, 2, H, W) * 3
    flow[0, 0, 1, 1] = float("nan")
    flow[0, 1, 2, 3] = float("inf")
    flow[0, :, 0, 0] = torch.tensor([2.0, 1.0])  # integer landing: three zero-weight corners
    got = O.forward_splat_sum(inp, flow)
    exp = torch.zeros_like(inp)
    for y in range(H):
        for x in range(W):
            fx = x + flow[0, 0, y, x].item()
            fy = y + flow[0, 1, y, x].item()
            if not (np.isfinite(fx) and np.isfinite(fy)):
                continue
            x0, y0 = int(np.floor(fx)), int(np.floor(fy))
            for xx, yy, w in ((x0, y0, (x0 + 1 - fx) * (y0 + 1 - fy)), (x0 + 1, y0, (fx - x0) * (y0 + 1 - fy)),
                              (x0, y0 + 1, (x0 + 1 - fx) * (fy - y0)), (x0 + 1, y0 + 1, (fx - x0) * (fy - y0))):
                if 0 <= xx < W and 0 <= yy < H:
                    exp[0, :, yy, xx] += inp[0, :, y, x] * w
    assert torch.allclose(got, exp, atol=1e-5)


def test_zeroeps_holes():
    """'zeroeps': a target that receives no weight outputs 0 (softsplat.py:333-344)."""
    inp = torch.ones(1, 2, 4, 4)
    flow = torch.full((1, 2, 4, 4), 10.0)  # everything leaves the frame
    out = O.softsplat_linear_zeroeps(inp, flow, torch.ones(1, 1, 4, 4))
    assert torch.count_nonzero(out) == 0


@pytest.mark.parametrize("name", ["gimm_64x96_t0.25_0.75", "gimm_b2_72x80_t0.5"])
def test_oracle_gimm_matches_reference_golden(name, golden_manifest, weights0):
    """GIMM standalone (gimm.py:129-214): the oracle's gimm_forward vs outputs of the unmodified reference GIMM"""
    from gimmvfi_b200.synth import synth_flow_pair

    torch.set_grad_enabled(False)
    meta = golden_manifest[name]
    assert meta["kind"] == "gimm" and meta["oracle_vs_reference_max_abs"] <= 2e-6
    g = load_golden(name)
    B, H, W, ts = meta["B"], meta["H"], meta["W"], meta["timesteps"]
    ori = synth_flow_pair(B, H, W, seed=meta["flow_seed"])
    xs, _ = O.normalize_flow(ori)
    coord = [O.sample_coord_input(B, (H, W), [t], 1.0) for t in ts]
    out = O.gimm_forward(weights0, xs, coord, ori, [t * torch.ones(B) for t in ts])
    for i in range(len(ts)):
        assert out[i].shape == (B, 2, 1, H, W)
        assert np.abs(out[i].numpy() - g["out_%d" % i]).max() <= TOL
    one = O.gimm_forward(weights0, xs, coord[0], ori, ts[0] * torch.ones(B), keep_xs_shape=False)   # tensor form
    assert one.shape == (B, 1, H, W, 2) and torch.equal(one.permute(0, 4, 1, 2, 3), out[0])


def test_oracle_matches_reference_on_demo_frames(weights0):
    """The reference's own demo frames (demo/input_frames, 720x844 -> InputPadder 736x864): the fixture holds the uint8 frames and
    the UNMODIFIED reference's output at this size (oracle/make_golden_big.py) — the oracle restatement must reproduce it."""
    import json

    import torch.nn.functional as F

    name = "big_r_demo_736x864_t0.5"
    with open(os.path.join(GOLDEN_DIR, "manifest_big.json")) as f:
        meta = json.load(f)[name]
    g = load_golden(name)
    torch.set_grad_enabled(False)
    x = torch.from_numpy(g["frames_u8"].copy()).permute(0, 3, 1, 2).float() / 255.0
    ht, wd = x.shape[-2:]
    ph, pw = (((ht // 32) + 1) * 32 - ht) % 32, (((wd // 32) + 1) * 32 - wd) % 32
    x = F.pad(x, [pw // 2, pw - pw // 2, ph // 2, ph - ph // 2], mode="replicate")
    xs = torch.stack([x[0], x[1]], 1).unsqueeze(0).contiguous()
    H, W = meta["H"], meta["W"]
    assert tuple(xs.shape) == (1, 3, 2, H, W)
    out = O.gimmvfi_r_forward(weights0, xs, [(O.sample_coord_input(1, (H, W), [0.5]), None)], [0.5 * torch.ones(1)])
    s = int(g["stride"])
    assert np.abs(out["imgt_pred"][0][..., ::s, ::s].numpy() - g["imgt_pred_0"]).max() <= TOL
    assert np.abs(out["raft_flow"][..., ::s, ::s].numpy() - g["raft_flow"]).max() <= 50 * TOL


@pytest.mark.parametrize("name", ["ff_128x160_t0.5", "ff_b2_128x128_t0.5"])
def test_flowformer_oracle_matches_reference(name):
    """oracle/flowformer_oracle.py (the restatement of GIMM-VFI-F's FlowFormer estimator) against the outputs of the UNMODIFIED reference
    FlowFormer on the same seeded weights and inputs (oracle/make_golden_ff.py): flows, context features, fnet maps, both directions."""
    import json

    import flowformer_oracle as FO
    from gimmvfi_b200.weights import random_state_dict_f

    torch.set_grad_enabled(False)
    meta = json.load(open(os.path.join(GOLDEN_DIR, "manifest_ff.json")))[name]
    assert meta["oracle_vs_reference"]["flow"] <= 1e-4
    g = load_golden(name)
    sd = random_state_dict_f(0)
    xs = synth_batch(meta["B"], meta["H"], meta["W"], seed=meta["input_seed"])
    im = [255 * xs[:, :, 0], 255 * xs[:, :, 1]]
    for d in range(2):
        (fu, fl), cf, ff = FO.flowformer_forward(sd, im[d], im[1 - d])
        assert np.abs(fu.numpy() - g["flows"][:, :, d]).max() <= 2e-4        # px; |flow| up to ~25
        assert np.abs(fl.numpy() - g["flow_low_%s" % ("01" if d == 0 else "10")]).max() <= 5e-5
        assert np.abs(cf[0].numpy() - g["feat4_%d" % d]).max() <= 2e-5 and np.abs(cf[1].numpy() - g["feat8_%d" % d]).max() <= 2e-5
        assert np.abs(ff.numpy() - g["fnet_%d" % d]).max() <= 2e-5
