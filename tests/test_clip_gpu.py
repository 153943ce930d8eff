"""The clip form (GIMMVFI_R / GIMMVFI_F.interpolate, gimmvfi_forward_clip) on the GPU: pair p of a clip call against forward() with B = 1 on
(frames[src], frames[tgt]); the reference fixtures through a 2-frame clip; the per-frame stages really running once per frame; and
VideoInterpolator with pairs_per_call > 1 against the per-pair loop.

Equivalence bar: the outputs upstream of GIMM's forward splat - the estimator's flows and nflow - must be bit-identical in the clip, and so
are the splat's inputs (the latents and splat weights, debug taps).  The outputs behind the splat, which sums with float
atomics, may differ by the run-to-run noise of both sides: what three per-pair runs differ by among themselves plus what two clip runs
differ by (the summation order follows the launch geometry, so B = 1 runs resemble each other more than a clip run), with a floor of
1e-5."""
import json
import os

import pytest
import torch

from conftest import GOLDEN_DIR
from gimmvfi_b200 import GIMMVFI_R
from gimmvfi_b200.model_f import GIMMVFI_F
from gimmvfi_b200.synth import synth_batch
from gimmvfi_b200.weights import random_state_dict, random_state_dict_f
from golden import load as load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module", params=["R", "F"])
def model(request):
    if request.param == "R":
        m = GIMMVFI_R(seed=0).to(DEV).eval()
        m.load_state_dict(random_state_dict(0), strict=True)
    else:
        m = GIMMVFI_F(seed=0).to(DEV).eval()
        m.load_state_dict(random_state_dict_f(0), strict=True)
    m.kind = request.param
    yield m
    m.tensor_cores = 4
    m.aux_outputs = True


def clip_frames(n, H, W, seed):
    """n distinct frames (F,3,H,W) in [0,1] from the synthetic pair generator"""
    xs = synth_batch((n + 1) // 2, H, W, seed=seed)           # (B,3,2,H,W)
    return xs.permute(0, 2, 1, 3, 4).reshape(-1, 3, H, W)[:n].contiguous().to(DEV)


def per_pair(model, frames, a, b, ts, ds):
    H, W = frames.shape[-2:]
    xs = torch.stack([frames[a], frames[b]], 1).unsqueeze(0).contiguous()
    ratio = 1.0 if ds is None else ds
    coord = [(model.sample_coord_input(1, (H, W), [t], device=DEV, upsample_ratio=ratio), None) for t in ts]
    tt = [t * torch.ones(1, device=DEV) for t in ts]
    return model(xs, coord, t=tt, ds_factor=ds)


def flat(out, p=None):
    """the returned dict as {name: tensor}, pair p's slice of the clip form (pair axis first after the timestep)"""
    r = {"raft_flow": out["raft_flow"], "nflow": out["nflow"]}
    T = len(out["imgt_pred"])
    for i in range(T):
        r["imgt_pred_%d" % i] = out["imgt_pred"][i]
        r["ninrflow_%d" % i] = out["ninrflow"][i]
        r["img_warp_4_%d" % i] = out["other_pred"][i][0]
        r["flowt0_1_%d" % i] = out["flowt0_pred"][i][0]
        r["flowt1_4_%d" % i] = out["flowt1_pred"][i][1]
        f = out["flowt"][i]
        r["flowt_%d" % i] = f if p is None else (f.unsqueeze(0) if f.dim() == 3 else f)
    if p is not None:
        r = {k: v[p:p + 1] for k, v in r.items()}
    else:
        r = {k: (v.unsqueeze(0) if k.startswith("flowt_") else v) for k, v in r.items()}
    return {k: v.float() for k, v in r.items()}


EXACT = ("raft_flow", "nflow")   # upstream of the splat

CASES = {
    "2f_128x160_T1": (2, (128, 160), [(0, 1)], [0.5], None),
    "3f_128x160_T3": (3, (128, 160), [(0, 1), (1, 2)], [0.25, 0.5, 0.75], None),
    "2f_ds0.5": (2, None, [(0, 1), (1, 0)], [0.5], 0.5),
    "5f_mixed": (5, (128, 160), [(0, 1), (1, 2), (3, 1), (0, 4), (2, 2), (0, 1)], [0.5], None),
}


@pytest.mark.parametrize("mode", [4, 0], ids=["mode4", "mode0"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_clip_matches_per_pair_forwards(model, case, mode):
    n, size, pairs, ts, ds = CASES[case]
    if size is None:   # F's network resolution must be a multiple of 32
        size = (272, 400) if model.kind == "R" else (256, 320)
    H, W = size
    model.tensor_cores = mode
    model.aux_outputs = True
    frames = clip_frames(n, H, W, seed=40 + n)
    clip = model.interpolate(frames, pairs, ts, ds)
    torch.cuda.synchronize()
    # Upstream of GIMM's forward splat every stage is per sample: the estimator's flows and nflow must be bit-identical (the splat's own
    # inputs have a test of their own below).  Every output behind the splat is bounded by the splat's atomic-order noise on either side:
    # what three per-pair runs (B = 1) differ by among themselves, pooled over the pairs, plus what two clip runs differ by (the clip's
    # launch geometry, whose summation orders differ from B = 1's), with a floor of 1e-5.
    R = 3
    runs = [[flat(per_pair(model, frames, a, b, ts, ds)) for _ in range(R)] for a, b in pairs]
    clip2 = model.interpolate(frames, pairs, ts, ds)
    noisy, spread = {}, {}
    for k in runs[0][0]:
        if k not in EXACT:
            s1 = max((rs[i][k] - rs[j][k]).abs().max().item() for rs in runs for i in range(R) for j in range(i + 1, R))
            s2 = max((flat(clip, p)[k] - flat(clip2, p)[k]).abs().max().item() for p in range(len(pairs)))
            spread[k] = s1 + s2
    for p, (a, b) in enumerate(pairs):
        got = flat(clip, p)
        for k, ref in runs[p][0].items():
            assert got[k].shape == ref.shape, (k, got[k].shape, ref.shape)
            if k in EXACT:
                assert torch.equal(got[k], ref), "%s pair %d (%d,%d): max diff %.3e in the clip" % (k, p, a, b, (got[k] - ref).abs().max().item())
            else:
                d = min((got[k] - r[k]).abs().max().item() for r in runs[p])
                noisy[k] = max(noisy.get(k, 0.0), d)
                assert d <= max(spread[k], 1e-5), "%s pair %d: clip differs by %.3e, the runs' noise %.3e" % (k, p, d, spread[k])
    print(model.kind, case, "mode", mode, "within the splat noise:", {k: "%.1e" % v for k, v in noisy.items()})


def test_clip_splat_inputs_are_bit_identical(model):
    """everything before GIMM's forward splat - the latents of both directions and the splat weights - equals the per-pair forward bit
    for bit (5 frames, reversed, repeated and self pairs, mode 4); only the splat's float-atomic sums can tell the two apart"""
    H, W = 128, 160
    pairs = [(0, 1), (3, 1), (2, 2), (0, 1)]
    model.tensor_cores = 4
    model.aux_outputs = False
    frames = clip_frames(5, H, W, seed=45)
    eng = model._ready(frames)
    names = ("gimm.lat0", "gimm.lat1", "gimm.splat_w")
    eng.set_debug(True)
    try:
        model.interpolate(frames, pairs, [0.5])
        torch.cuda.synchronize()
        clip = {n: eng.tap(n) for n in names}
        P = len(pairs)
        for p, (a, b) in enumerate(pairs):
            per_pair(model, frames, a, b, [0.5], None)
            torch.cuda.synchronize()
            one = {n: eng.tap(n) for n in names}
            for n in ("gimm.lat0", "gimm.lat1"):
                assert torch.equal(clip[n][p:p + 1], one[n]), (n, p)
            w = clip["gimm.splat_w"]   # [both directions' pairs]: sample p and P + p
            assert torch.equal(w[p:p + 1], one["gimm.splat_w"][0:1]) and torch.equal(w[P + p:P + p + 1], one["gimm.splat_w"][1:2]), p
    finally:
        eng.set_debug(False)


def test_clip_keeps_the_per_pair_raft_lookup(monkeypatch):
    """RAFT's lookup path (all-pairs volume or volume-free) is chosen as a one-pair forward chooses it, not from the clip's 2P directions:
    with the volume budget set between one pair's pyramid (1.1 MB at 128x160) and three pairs' (3.3 MB), the clip keeps the volume and
    its flows stay bit-identical to forward() with B = 1"""
    monkeypatch.setenv("GIMMVFI_RAFT_CORR_DIRECT_GB", "0.002")   # read when the model's engine is made
    m = GIMMVFI_R(seed=0).to(DEV).eval()
    m.load_state_dict(random_state_dict(0), strict=True)
    m.aux_outputs = ("raft_flow",)
    frames = clip_frames(4, 128, 160, seed=12)
    pairs, ts = [(0, 1), (1, 2), (3, 2)], [0.25, 0.5, 0.75]   # (T = 3: GIMM's own correlation uses its volume, not the direct lookup)
    eng = m._ready(frames)
    eng.set_profile(True)
    try:
        clip = m.interpolate(frames, pairs, ts)
        prof = eng.profile()
    finally:
        eng.set_profile(False)
    assert "corr_lookup_direct" not in prof and "corr_lookup" in prof, sorted(prof)
    for p, (a, b) in enumerate(pairs):
        assert torch.equal(clip["raft_flow"][p:p + 1], per_pair(m, frames, a, b, ts, None)["raft_flow"]), p


@pytest.mark.parametrize("mode", [4, 0], ids=["mode4", "mode0"])
def test_clip_meets_the_reference_fixture(model, mode):
    """the fixture of one pair at 128x160 (made by the unmodified reference) through interpolate as a 2-frame clip"""
    name = "r_128x160_t0.5" if model.kind == "R" else "ff_128x160_t0.5"
    manifest = "manifest.json" if model.kind == "R" else "manifest_ff.json"
    with open(os.path.join(GOLDEN_DIR, manifest)) as f:
        meta = json.load(f)[name]
    g = load_golden(name)
    H, W = meta["H"], meta["W"]
    xs = synth_batch(1, H, W, seed=meta["input_seed"])
    frames = xs[0].permute(1, 0, 2, 3).contiguous().to(DEV)    # (2,3,H,W)
    model.tensor_cores = mode
    model.aux_outputs = False
    out = model.interpolate(frames, [(0, 1)], meta["timesteps"], meta["ds_factor"])
    s = int(g["stride"]) if "stride" in g else 1
    for i in range(len(meta["timesteps"])):
        d = (out["imgt_pred"][i][..., ::s, ::s].cpu() - torch.from_numpy(g["imgt_pred_%d" % i])).abs().max().item()
        print(model.kind, name, "mode", mode, "imgt_pred[%d] max %.3e" % (i, d))
        assert d <= 1e-3


def test_clip_encodes_each_frame_once(model):
    """5 frames, 4 consecutive pairs at 128x160: the estimator's encoders run over 5 frames, not 8 - RAFT's fnet / cnet stems and first
    layers (the only layers at H/2 = 64x80), FlowFormer's two Twins stacks (at H/4 = 32x40 per frame, where the synthesis runs per pair:
    4).  GIMM's cnn_encoder encodes each pair's normalised flows, so it runs per pair and direction: 8 at full resolution."""
    H, W = 128, 160
    model.tensor_cores = 4
    model.aux_outputs = False
    frames = clip_frames(5, H, W, seed=7)
    eng = model._ready(frames)
    eng.set_profile(True)
    try:
        model.interpolate(frames, [(0, 1), (1, 2), (2, 3), (3, 4)], [0.5])
        prof = eng.profile()
    finally:
        eng.set_profile(False)
    if model.kind == "R":
        enc = sorted(k for k in prof if "x64x80" in k)
        assert enc and all("@5x64x80" in k for k in enc), enc
    else:
        enc = sorted(k for k in prof if "@5x32x40" in k)
        assert enc and not [k for k in prof if "@8x32x40" in k or "@10x32x40" in k], sorted(prof)
    print(model.kind, "per-frame encoder layers:", enc)
    assert any(k.startswith("clip_gather") for k in prof), sorted(prof)
    assert any("@8x128x160" in k for k in prof), sorted(prof)   # cnn_encoder, per pair direction


def test_video_interpolator_pairs_per_call_matches_per_pair(model):
    """a 9-frame synthetic clip through VideoInterpolator with pairs_per_call 4 and 1: the same uint8 frames and flow pictures, up to
    one level where the splat noise crosses a rounding boundary"""
    from gimmvfi_b200.video import VideoInterpolator

    if model.kind == "F":
        H, W = 128, 160
    else:
        H, W = 120, 150   # padded to 128 x 160 by the driver
    model.tensor_cores = 4
    fr = clip_frames(9, 128, 160, seed=9)[..., :H, :W]
    u8 = [(f.permute(1, 2, 0) * 255).to(torch.uint8).contiguous() for f in fr]
    res = {}
    for K in (1, 4):
        vi = VideoInterpolator(model, N=3, with_flow=True, pairs_per_call=K)
        frames, flows = [], []
        for f in u8:
            a, b = vi.push(f)
            frames += a
            flows += b
        a, b = vi.flush()
        frames += a
        flows += b
        res[K] = (frames, flows)
    assert len(res[1][0]) == len(res[4][0]) == 8 * 2 and len(res[1][1]) == len(res[4][1]) == 16
    for x, y in zip(res[1][0] + res[1][1], res[4][0] + res[4][1]):
        assert x.shape == y.shape
        assert (x.int() - y.int()).abs().max().item() <= 1
