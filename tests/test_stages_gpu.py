"""GIMM-VFI-R stage by stage: the engine's debug taps (Engine::tap, EngineHandle.tap) against the matching entries of the oracle's
trace (oracle/gimmvfi_r_oracle.py), at 136 x 200 - RAFT on a 17 x 25 grid, H/4 = 34 x 50 - with T = 1.

Each stage is compared on the inputs the engine itself used wherever the oracle allows it, so that RAFT's 20-iteration amplification
does not reach the downstream bounds: GIMM's stages come from predict_flow fed with the engine's raft_flow, the synthesis stages from
frame_synthesize fed with the engine's flowt.  (The context features and correlation maps the synthesis reads come from the oracle's
own RAFT encoders: the encoders are not iterated.)

Layouts: the engine stores NHWC and batches both RAFT directions as 2B samples [I0 -> I1 ; I1 -> I0]; the oracle stores NCHW, per call.

Backends: the CPU build of the same sources (tests/hostsim, fp32 arithmetic; runs without a GPU), and the H100 in precision modes 0
(fp32 CUDA cores) and 4 (the default).  Mode 0 on the GPU has the same bars as the host simulation."""
import os
import sys

import pytest
import torch

import gimmvfi_r_oracle as O
from gimmvfi_b200.synth import synth_batch
from splat_ref import splat_w_bound, splat_w_float64

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim"))

B, H, W, T_VAL, SEED = 1, 136, 200, 0.5, 41     # the r8_136x200_t0.5 case (oracle/make_golden_r8.py)
BACKENDS = [pytest.param(("hostsim", 0), id="hostsim-mode0"),
            pytest.param(("gpu", 0), id="h100-mode0", marks=pytest.mark.gpu),
            pytest.param(("gpu", 4), id="h100-mode4", marks=pytest.mark.gpu)]
TAPS = ["raft.fmap", "raft.corr_it0", "raft.lowres_flow_it0", "raft.lowres_flow_it4", "raft.lowres_flow_final", "raft.net_final",
        "gimm.splat_w", "gimm.lat0", "gimm.splat0", "gimm.latent", "syn.ft_4", "syn.fl4", "syn.corr_4_hi"]


def nhwc(t):
    return t.permute(0, 2, 3, 1)


@pytest.fixture(scope="module")
def inputs():
    xs = synth_batch(B, H, W, seed=SEED)
    coords = O.sample_coord_input(B, (H, W), [T_VAL], 1.0).unsqueeze(0).contiguous()   # (T, B, 1, H, W, 3)
    tt = T_VAL * torch.ones(1, B)
    return xs, coords, tt


@pytest.fixture(scope="module")
def oracle_raft(inputs, weights0):
    """both RAFT directions with their traces, and the context features / bidirectional correlation the synthesis reads"""
    torch.set_grad_enabled(False)
    xs = inputs[0]
    I0, I1 = 255 * xs[:, :, 0], 255 * xs[:, :, 1]
    tr = [{}, {}]
    _, feats0, fnet0 = O.raft_forward(weights0, "flow_estimator", I0, I1, 20, tr[0])
    _, feats1, fnet1 = O.raft_forward(weights0, "flow_estimator", I1, I0, 20, tr[1])
    # gimmvfi_r_forward's plumbing between RAFT and frame_synthesize (gimmvfi_r.py:126-156)
    corr_fn = O.BidirCorr(O._conv(weights0, "amt_fproj", fnet0), O._conv(weights0, "amt_fproj", fnet1))
    proj = lambda f: [O._conv(weights0, "amt_second_last_cproj", f[0]), O._conv(weights0, "amt_last_cproj", f[1])]
    return tr, proj(feats0), proj(feats1), corr_fn


@pytest.fixture(scope="module", params=BACKENDS)
def engine_run(request, inputs, weights0):
    """one forward with debug taps on; returns (backend, precision mode, {tap: NHWC tensor}, {output: tensor}), all on the CPU"""
    kind, mode = request.param
    torch.set_grad_enabled(False)
    if kind == "gpu":
        from gimmvfi_b200.engine import EngineHandle
        eng, dev = EngineHandle("cuda"), "cuda"
    else:
        from harness import hostsim_engine
        eng, dev = hostsim_engine(), "cpu"
    eng.load_state_dict(weights0)
    eng.set_tensor_cores(mode)
    eng.set_debug(True)
    xs, coords, tt = inputs
    out = eng.forward(xs.to(dev), coords.to(dev), tt.to(dev), None)
    if dev == "cuda":
        torch.cuda.synchronize()
    taps = {k: eng.tap(k).cpu() for k in TAPS}
    return kind, mode, taps, {k: v.cpu() for k, v in out.items()}


def maxdiff(got, ref):
    assert got.shape == ref.shape, (tuple(got.shape), tuple(ref.shape))
    return (got.double() - ref.double()).abs().max().item()


def check(engine_run, rows):
    """rows: (stage, engine NHWC tensor, reference NHWC tensor, {mode: bar}) compared by max |d|, or (stage, measured value, None,
    {mode: bar}); reports every stage, then asserts them all"""
    kind, mode, _, _ = engine_run
    lines, bad = [], []
    for stage, got, ref, bars in rows:
        err = maxdiff(got, ref) if ref is not None else got
        lines.append("%-34s %.3e (bar %.1e)" % (stage, err, bars[mode]))
        if not err <= bars[mode]:
            bad.append(stage)
    print("\n%s mode %d\n  " % (kind, mode) + "\n  ".join(lines))
    assert not bad, "stages over their bar: %s\n%s" % (bad, "\n".join(lines))


def both(trace, key):
    """oracle trace entries of the two RAFT calls -> the engine's 2B NHWC layout [direction 0 ; direction 1]"""
    return torch.cat([nhwc(trace[0][key]), nhwc(trace[1][key])], 0)


def test_raft_stages(engine_run, oracle_raft):
    """fnet features, the first lookup and the recurrence at iterations 0, 4 and 19.  The iteration amplifies operand rounding: an
    fp32 reassociation (~1e-7) in the encoders becomes ~1e-5 px after 20 GRU updates; mode 4 runs RAFT on 3xTF32 (fp32-class)."""
    _, _, taps, _ = engine_run
    tr = oracle_raft[0]
    check(engine_run, [
        # RAFT is fp32-class in both modes (mode 4: 3xTF32 operands, ~fp32 products), so the bars are shared.
        # Instance-normalised features, |f| <= 8.3, after ~20 convolutions with K up to 2304: fp32 reassociation ~1e-5 (measured
        # 1.5e-5 on the host simulation and on both GPU modes)
        ("raft.fmap", taps["raft.fmap"], both(tr, "fmap1"), {0: 1e-4, 4: 1e-4}),
        # 256-channel dot products / 16 of those features + bilinear taps, |corr| <= 68: ~1e-4 (measured 6.5e-5 / 9.2e-5 / 1.2e-4)
        ("raft.corr_it0", taps["raft.corr_it0"], both(tr, "corr_it0"), {0: 4e-4, 4: 4e-4}),
        # the recurrence: 1.9e-6 px after one update, ~4e-6 after five, ~1e-5 after twenty (|flow| <= 2.7 px)
        ("raft.lowres_flow_it0", taps["raft.lowres_flow_it0"], both(tr, "lowres_flow_it0"), {0: 2e-5, 4: 2e-5}),
        ("raft.lowres_flow_it4", taps["raft.lowres_flow_it4"], both(tr, "lowres_flow_it4"), {0: 5e-5, 4: 5e-5}),
        ("raft.lowres_flow_final", taps["raft.lowres_flow_final"], both(tr, "lowres_flow_it19"), {0: 1e-4, 4: 1e-4}),
        # tanh-bounded GRU state after twenty updates
        ("raft.net_final", taps["raft.net_final"], both(tr, "net_final"), {0: 2e-5, 4: 2e-5}),
    ])


def test_gimm_stages(engine_run, inputs, weights0):
    """splatting weights, motion latents, forward splat and refined latent, from the oracle's predict_flow on the engine's own
    raft_flow (so the comparison starts from identical flows)."""
    _, _, taps, out = engine_run
    _, coords, tt = inputs
    flows = out["raft_flow"]                                     # (B, 2, 2, H, W): [f01 | f10] on dim 2, like predict_flow's `flows`
    nflow, _ = O.normalize_flow(torch.stack([flows[:, :, 0], -flows[:, :, 1]], 2))
    tr = {}
    O.predict_flow(weights0, nflow, [coords[0]], [tt[0]], flows, tr)
    # splatting weights 1/(1+err*a_fe) + 1/(1+var*a_v) against float64 (gimmvfi_r.py:444-492 on the same flows), per pixel within
    # splat_w_bound: var = sqrt(E[f^2] - E[f]^2) cancels wherever the flow is locally near constant, so fp32 (the oracle's as much as
    # the engine's) is there off float64 by up to ~4e-3 - and by ~1e-5 where the flow varies.  Measured max |d| / bound: 0.68 for the
    # host simulation and the oracle, 0.49 / 0.58 on the GPU in modes 0 / 4 (whose FMA contraction rounds the difference once instead of
    # twice: ~1.5e-3 away from the oracle's fp32, not from float64); 3.4 with var scaled by 1.001
    w64 = splat_w_float64(weights0, flows)
    bound = splat_w_bound(weights0, flows)
    sw = taps["gimm.splat_w"].double()
    w32 = torch.cat([nhwc(tr["splat_w1"]), nhwc(tr["splat_w2"])], 0).double()
    print("\noracle fp32 splat_w vs float64: max %.3e, max |d| / bound %.3f" % (maxdiff(w32, w64), ((w32 - w64).abs() / bound).max().item()))
    check(engine_run, [
        ("gimm.splat_w max |d| / bound", ((sw - w64).abs() / bound).max().item(), None, {0: 1.0, 4: 1.0}),
        # motion latents |lat| <= 0.31: fp32 convolutions (measured ~3e-7 in mode 0).  Mode 4 stores the 32-channel full-resolution
        # chain of cnn_encoder / res_conv in half (2^-11 relative, ~1.5e-4 here per rounding) on TF32 / f16 operands (measured 3.6e-4)
        ("gimm.lat0", taps["gimm.lat0"], nhwc(tr["lat0"]), {0: 5e-6, 4: 1.5e-3}),
        # the forward splat normalises a weighted average of those latents: no amplification with identical flows and weights
        ("gimm.splat0", taps["gimm.splat0"], nhwc(tr["splat0"]), {0: 5e-6, 4: 1.5e-3}),
        ("gimm.latent", taps["gimm.latent"], nhwc(tr["latent"]), {0: 5e-6, 4: 1.5e-3}),
    ])


def test_synthesis_stages(engine_run, inputs, weights0, oracle_raft):
    """the init decoder + both AMT update blocks at H/4, from the oracle's frame_synthesize fed with the engine's flowt"""
    _, _, taps, out = engine_run
    xs, _, tt = inputs
    _, feats0, feats1, corr_fn = oracle_raft
    tr = {}
    flow_t = out["flowt"][0]                                     # (B, 2, H, W)
    _, _, ft1s, _ = O.frame_synthesize(weights0, xs, flow_t, feats0, feats1, corr_fn, tt[0].reshape(-1, 1, 1, 1), None, tr)
    fl4 = taps["syn.fl4"]
    check(engine_run, [
        # bidirectional correlation at the init decoder's flows, |corr| <= 19.4.  Mode 0: the fp32 volume (256-term dot products,
        # measured 2e-5).  Mode 4 (T = 1): no volume - the lookup rounds the other frame's features to half (11-bit significand), as
        # in test_corr_lookup_direct_vs_oracle: ~1e-2 (measured 1.4e-2)
        ("syn.corr_4_hi", taps["syn.corr_4_hi"], nhwc(tr["corr_4_hi"]), {0: 2e-4, 4: 5e-2}),
        # init decoder + two AMT update blocks.  Mode 0: fp32 (measured ~3e-7).  Mode 4: TF32 operands (2^-11 relative) over K up to
        # 272 x 9, the H/4 residual trunk stored in half, and the correlation above as input (measured 1.4e-4 on |ft_4| <= 0.17,
        # 1.6e-4 px on |flow| <= 1.5 px)
        ("syn.ft_4", taps["syn.ft_4"], nhwc(tr["ft_4"]), {0: 5e-6, 4: 1e-3}),
        ("syn.fl4 (flowt0_4)", fl4[..., :2], nhwc(tr["flowt0_4"]), {0: 5e-6, 4: 1e-3}),
        ("syn.fl4 (flowt1_4)", fl4[..., 2:], nhwc(ft1s[1]), {0: 5e-6, 4: 1e-3}),
    ])
