"""The query form (GIMMVFI_R / GIMMVFI_F.interpolate_at, gimmvfi_forward_queries) on the GPU: query q against forward() with B = 1 on
(frames[src], frames[tgt]) at its pair's own timestep list; both of GIMM's correlation lookups in one call; encoders over the used frames
only; the device coordinate grid against sample_coord_input; the reference fixtures; and FrameRateConverter's batching.

Equivalence bar, as tests/test_clip_gpu.py: the estimator's outputs (raft_flow, nflow) must be bit-identical; the outputs behind GIMM's
forward splat, which sums with float atomics, may differ by what three per-pair runs differ by among themselves plus what two query runs
differ by, with a floor of 1e-5."""
import json
import os

import pytest
import torch

from conftest import GOLDEN_DIR
from gimmvfi_b200 import GIMMVFI_R
from gimmvfi_b200.config import default_arch_config
from gimmvfi_b200.model_f import GIMMVFI_F
from gimmvfi_b200.synth import synth_batch
from gimmvfi_b200.weights import random_state_dict, random_state_dict_f
from golden import load as load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"


def make_model(kind, config=None):
    if kind == "R":
        m = GIMMVFI_R(config, seed=0).to(DEV).eval()
        m.load_state_dict(random_state_dict(0), strict=True)
    else:
        m = GIMMVFI_F(config).to(DEV).eval()
        m.load_state_dict(random_state_dict_f(0), strict=True)
    m.kind = kind
    return m


@pytest.fixture(scope="module", params=["R", "F"])
def model(request):
    m = make_model(request.param)
    yield m
    m.tensor_cores = 4
    m.aux_outputs = True


def clip_frames(n, H, W, seed):
    """n distinct frames (F,3,H,W) in [0,1] from the synthetic pair generator"""
    xs = synth_batch((n + 1) // 2, H, W, seed=seed)
    return xs.permute(0, 2, 1, 3, 4).reshape(-1, 3, H, W)[:n].contiguous().to(DEV)


def per_pair(model, frames, a, b, ts, ds):
    H, W = frames.shape[-2:]
    xs = torch.stack([frames[a], frames[b]], 1).unsqueeze(0).contiguous()
    ratio = 1.0 if ds is None else ds
    coord = [(model.sample_coord_input(1, (H, W), [t], device=DEV, upsample_ratio=ratio), None) for t in ts]
    tt = [t * torch.ones(1, device=DEV) for t in ts]
    return model(xs, coord, t=tt, ds_factor=ds)


def flat_forward(out):
    """forward()'s dict (B = 1) as {name: (T, ...)} per-timestep tensors, plus the per-pair ones"""
    T = len(out["imgt_pred"])
    r = {"raft_flow": out["raft_flow"], "nflow": out["nflow"]}
    r["imgt_pred"] = torch.cat([out["imgt_pred"][i] for i in range(T)], 0)
    r["ninrflow"] = torch.cat([out["ninrflow"][i] for i in range(T)], 0)
    r["img_warp_4"] = torch.cat([out["other_pred"][i][0] for i in range(T)], 0)
    r["flowt0_1"] = torch.cat([out["flowt0_pred"][i][0] for i in range(T)], 0)
    r["flowt1_4"] = torch.cat([out["flowt1_pred"][i][1] for i in range(T)], 0)
    r["flowt"] = torch.stack([out["flowt"][i].reshape(out["flowt"][i].shape[-3:]) for i in range(T)], 0)
    return r


EXACT = ("raft_flow", "nflow")   # upstream of the splat
SPLAT = ("imgt_pred", "ninrflow", "img_warp_4", "flowt0_1", "flowt1_4", "flowt")

# (frames, size, queries, ds): counts {3, 2, 1, 1}, a reversed and a self pair, an unused frame, interleaved queries
MIXED = [(0, 1, 0.2), (2, 2, 0.3), (1, 0, 0.6), (0, 1, 0.5), (4, 2, 0.25), (2, 2, 0.7), (0, 1, 0.8)]
CASES = {
    "5f_mixed": (5, (128, 160), MIXED, None),
    "3f_ds0.5": (3, None, [(0, 1, 0.4), (1, 2, 0.2), (0, 1, 0.8), (1, 2, 0.6), (2, 1, 0.5)], 0.5),
}


def check_against_per_pair(model, frames, queries, ds, R=3):
    q = model.interpolate_at(frames, queries, ds)
    torch.cuda.synchronize()
    pairs, index = q["pairs"], q["pair_index"].tolist()
    mine = {p: [i for i, x in enumerate(index) if x == p] for p in range(len(pairs))}
    runs = {p: [flat_forward(per_pair(model, frames, a, b, [queries[i][2] for i in mine[p]], ds)) for _ in range(R)]
            for p, (a, b) in enumerate(pairs)}
    q2 = model.interpolate_at(frames, queries, ds)
    spread = {}
    for k in SPLAT:
        s1 = max((rs[i][k] - rs[j][k]).abs().max().item() for rs in runs.values() for i in range(R) for j in range(i + 1, R))
        s2 = (q[k] - q2[k]).abs().max().item()
        spread[k] = s1 + s2
    noisy = {}
    for p, (a, b) in enumerate(pairs):
        for k in EXACT:
            ref = runs[p][0][k]
            assert torch.equal(q[k][p:p + 1], ref), "%s pair (%d,%d): max diff %.3e" % (k, a, b, (q[k][p:p + 1] - ref).abs().max().item())
        for i, qi in enumerate(mine[p]):
            for k in SPLAT:
                got = q[k][qi]
                d = min((got - r[k][i].reshape(got.shape)).abs().max().item() for r in runs[p])
                noisy[k] = max(noisy.get(k, 0.0), d)
                assert d <= max(spread[k], 1e-5), "%s query %d (%d,%d): differs by %.3e, the runs' noise %.3e" % (k, qi, a, b, d, spread[k])
    return noisy


def gimm_lookups(counts):
    """GIMM's correlation lookup launches of one query call in a tensor-core mode, (pyramid, volume-free), from its pairs' timestep
    counts: pairs with more than 2 timesteps take the pyramid; slot k runs the B_k pairs with more than k timesteps, sorted by count,
    so each slot launches each lookup kind once per direction when it has pairs of that kind"""
    c = sorted(counts, reverse=True)
    Bp = sum(1 for x in c if x > 2)
    p = d = 0
    for k in range(c[0]):
        Bk = sum(1 for x in c if x > k)
        p += 2 if min(Bp, Bk) > 0 else 0
        d += 2 if Bk > min(Bp, Bk) else 0
    return p, d


def check_gimm_lookups(model, frames, queries, ds=None):
    """GIMM's lookup launches in a query call, net of the flow estimator's own (RAFT's lookups are the same kernels): a second call
    over the same pairs with one timestep each runs the estimator alike and GIMM's volume-free lookup once per direction"""
    eng = model._ready(frames)
    pairs = list(dict.fromkeys((a, b) for a, b, _ in queries))
    counts = [sum(1 for q in queries if (q[0], q[1]) == pr) for pr in pairs]
    n = lambda prof, k: prof.get(k, {}).get("launches", 0)
    eng.set_profile(True)
    try:
        model.interpolate_at(frames, queries, ds)
        prof = eng.profile()
        model.interpolate_at(frames, [(a, b, 0.5) for a, b in pairs], ds)
        ref = eng.profile()
    finally:
        eng.set_profile(False)
    est_p, est_d = n(ref, "corr_lookup"), n(ref, "corr_lookup_direct") - 2
    got = (n(prof, "corr_lookup") - est_p, n(prof, "corr_lookup_direct") - est_d)
    want = gimm_lookups(counts)
    assert want[0] > 0 and want[1] > 0
    assert got == want, "GIMM's (pyramid, volume-free) lookups %s, want %s; estimator's %s" % (got, want, (est_p, est_d))
    return prof


@pytest.mark.parametrize("mode", [4, 0], ids=["mode4", "mode0"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_queries_match_per_pair_forwards(model, case, mode):
    n, size, queries, ds = CASES[case]
    if size is None:   # F's network resolution must be a multiple of 32
        size = (272, 400) if model.kind == "R" else (256, 320)
    model.tensor_cores = mode
    model.aux_outputs = True
    frames = clip_frames(n, *size, seed=60 + n)
    noisy = check_against_per_pair(model, frames, queries, ds)
    print(model.kind, case, "mode", mode, "within the splat noise:", {k: "%.1e" % v for k, v in noisy.items()})


def test_queries_mixed_lookups_at_1080p():
    """GIMM-VFI-R at 1088x1920 with timestep counts {3, 2, 1}: the 3-timestep pair takes the all-pairs pyramid, the others the
    volume-free lookup, in one call; every pair matches its own forward"""
    m = make_model("R")
    m.aux_outputs = True
    frames = clip_frames(4, 1088, 1920, seed=81)
    queries = [(0, 1, 0.25), (1, 2, 0.4), (0, 1, 0.5), (3, 2, 0.5), (1, 2, 0.8), (0, 1, 0.75)]
    check_gimm_lookups(m, frames, queries)
    noisy = check_against_per_pair(m, frames, queries, None, R=2)
    print("R 1088x1920 {3,2,1} within the splat noise:", {k: "%.1e" % v for k, v in noisy.items()})


def test_queries_encode_only_the_used_frames(model):
    """5 frames of which 3 are used, at 128x160: the estimator's encoders run over 3 frames (RAFT's H/2 stems at 64x80; FlowFormer's
    Twins at 32x40), and GIMM's correlation takes the pyramid for the 3-timestep pair and the volume-free lookup for the other"""
    model.tensor_cores = 4
    model.aux_outputs = False
    frames = clip_frames(5, 128, 160, seed=7)
    prof = check_gimm_lookups(model, frames, [(0, 2, 0.5), (4, 2, 0.3), (0, 2, 0.25), (0, 2, 0.75), (4, 2, 0.6)])
    if model.kind == "R":
        enc = sorted(k for k in prof if "x64x80" in k)
        assert enc and all("@3x64x80" in k for k in enc), enc
    else:
        enc = sorted(k for k in prof if "@3x32x40" in k)
        assert enc and not [k for k in prof if "@5x32x40" in k], sorted(prof)
    assert any(k.startswith("combine_output_rows") for k in prof), sorted(prof)


@pytest.mark.parametrize("coord_range", [(-1.0, 1.0), (0.0, 1.0), (-0.3, 0.7)])
@pytest.mark.parametrize("size,ds", [((1088, 360), None), ((272, 400), 0.5)])
def test_device_coordinates_equal_sample_coord_input(coord_range, size, ds):
    """the engine's grid of every query, bit for bit against the model's sample_coord_input on the device, for the shipped coord_range
    and ranges set in an edited arch block (one timestep per pair: a single slot holds every query, in query order)"""
    cfg = default_arch_config()
    cfg.coord_range = list(coord_range)
    m = make_model("R", cfg)
    m.aux_outputs = False
    frames = clip_frames(3, *size, seed=3)
    queries = [(0, 1, 0.1), (1, 2, 0.37), (2, 0, 0.9)]
    eng = m._ready(frames)
    eng.set_debug(True)
    try:
        m.interpolate_at(frames, queries, ds)
        torch.cuda.synchronize()
        grid = eng.tap("query.coords")
    finally:
        eng.set_debug(False)
    ratio = 1.0 if ds is None else ds
    want = torch.cat([m.sample_coord_input(1, size, [t], device=DEV, upsample_ratio=ratio)[0] for _, _, t in queries], 0)
    assert grid.shape == want.shape, (grid.shape, want.shape)
    assert torch.equal(grid, want), (grid - want).abs().max().item()


@pytest.mark.parametrize("mode", [4, 0], ids=["mode4", "mode0"])
def test_queries_meet_the_reference_fixture(model, mode):
    """the fixture of one pair at 128x160 (made by the unmodified reference) through interpolate_at"""
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
    out = model.interpolate_at(frames, [(0, 1, t) for t in meta["timesteps"]], meta["ds_factor"])
    s = int(g["stride"]) if "stride" in g else 1
    for i in range(len(meta["timesteps"])):
        d = (out["imgt_pred"][i][..., ::s, ::s].cpu() - torch.from_numpy(g["imgt_pred_%d" % i])).abs().max().item()
        print(model.kind, name, "mode", mode, "imgt_pred[%d] max %.3e" % (i, d))
        assert d <= 1e-3


def test_frame_rate_converter_pairs_per_call(model):
    """24 -> 60 over 9 frames with K = 1 and K = 4: the same uint8 frames up to one level where the splat noise crosses a rounding
    boundary; the integral instants are the input frames, BGR-flipped, byte for byte"""
    from gimmvfi_b200.video import FrameRateConverter

    H, W = (128, 160) if model.kind == "F" else (120, 150)   # (R's frames are padded to 128 x 160 by the converter)
    model.tensor_cores = 4
    fr = clip_frames(9, 128, 160, seed=9)[..., :H, :W]
    u8 = [(f.permute(1, 2, 0) * 255).to(torch.uint8).contiguous() for f in fr]
    res = {}
    for K in (1, 4):
        conv = FrameRateConverter(model, 24, 60, pairs_per_call=K)
        out = []
        for f in u8:
            out += conv.push(f)
        out += conv.flush()
        res[K] = out
    assert len(res[1]) == len(res[4]) == 8 * 60 // 24 + 1
    for k, (x, y) in enumerate(zip(res[1], res[4])):
        assert x.shape == y.shape == (H, W, 3)
        assert (x.int() - y.int()).abs().max().item() <= 1, k
        if (k * 24) % 60 == 0:
            j = k * 24 // 60
            assert torch.equal(x, u8[j].flip(-1)) and torch.equal(y, u8[j].flip(-1)), k
