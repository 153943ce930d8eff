"""GIMM-VFI-R's flow estimator (RAFT) stage by stage against float64, at the benchmarked sizes: the feature and context encoders, the
correlation lookup at the first and the last iteration, the update block (motion encoder, GRU, flow head, mask head), the convex
upsampling, and 20 float64 iterations composed from the engine's own encoder outputs.

Each stage is fed the engine's own stored input (its debug taps, EngineHandle.tap), so that no upstream difference reaches its bar; the
reference is the oracle (oracle/gimmvfi_r_oracle.py) in float64 with the weights cast to double, and the lookups are the chunked
float64 restatement of CorrBlock in tests/corr_ref.py, held to a per-entry bound of an fp32 lookup's distance from it (|corr| grows with
the features and the coordinates' rounding with |x|, so a flat bar does not carry from one size to another).

Cases: a small GIMM-VFI-R batch with ds_factor 0.5 (the host simulation and the H100); on the H100 bench.py's pair1080, the RAFT of its
batch720 forward with 8 distinct pairs (16 RAFT samples, a 13.9 GB level-0 volume, per-sample offsets past 2^31 floats, pyramid levels
that floor at odd sizes), GIMM-VFI-R at 2K with ds_factor 0.5, and EngineHandle.raft_forward on a 4K pair in both directions, whose
volume pyramid (179 GB) does not fit: the volume-free lookup.  batch720 runs through EngineHandle.raft_forward with GIMM-VFI-R's 16
(source, target) pairs - the same in-order batch, route and arithmetic as the forward's RAFT: a debug forward keeps RAFT's workspace
for its taps, which at B = 8 would take a 90 GB plan.  The forward with the taps off is held bit for bit to that raft_forward's flow,
and to each of its pairs run alone.  Backends: the CPU build of the same sources (tests/hostsim, fp32, mode 0) and the H100 in precision modes 0 (fp32 CUDA cores) and 4 (the default; RAFT runs 3xTF32 / 3xF16, fp32-class).  Layouts: the engine
stores NHWC and batches the RAFT samples [I0 -> I1 ; I1 -> I0]; the oracle NCHW."""
import gc
import math
import os
import sys
import time

import pytest
import torch
import torch.nn.functional as F

import gimmvfi_r_oracle as O
from corr_ref import U, corr_direct64, corr_lookup64, windows_outside
from gimmvfi_b200.synth import synth_batch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim"))

ITERS = 20
P = "flow_estimator"
# name: entry ("R": GIMM-VFI-R forward, "raft": EngineHandle.raft_forward on GIMM-VFI-R's pairs of frames [I0 batch ; I1 batch], sample s
# from frame s to frame (s + B) mod 2B), pairs B, full size, ds_factor, seed
CASES = {
    "small": ("R", 2, 272, 400, 0.5, 41),          # 17 x 25 grid
    "pair1080": ("R", 1, 1088, 1920, None, 100),   # bench.py's pair: 136 x 240, an 11.4 GB volume pyramid
    "batch720": ("raft", 8, 736, 1280, None, 100),  # bench.py --micro-batch 8 with 8 distinct pairs: 92 x 160 ... 11 x 20, 18.5 GB
    "r2k": ("R", 1, 1088, 2048, 0.5, 100),         # GIMM-VFI-R at 2K, ds_factor 0.5: 68 x 128
    "raft4k": ("raft", 1, 2160, 3840, None, 100),  # 270 x 480 ... 33 x 60: no volume (179 GB), the volume-free lookup
}
ENCODE_ENDS = ("batch720", "raft4k")   # float64 encoders on the first and last sample only (they carry the largest offsets)
RUNS = [pytest.param(("small", "hostsim", 0), id="small-hostsim-mode0")]
RUNS += [pytest.param((c, "gpu", m), id="%s-h100-mode%d" % (c, m), marks=pytest.mark.gpu) for c in CASES for m in (0, 4)]
TAPS = ["raft.fmap", "raft.cnet", "raft.corr_it0", "raft.lowres_flow_it0", "raft.lowres_flow_it4", "raft.coords_last", "raft.net_last",
        "raft.corr_last", "raft.motion_last", "raft.mask", "raft.lowres_flow_final", "raft.net_final"]


def nchw(t, dev):
    return t.permute(0, 3, 1, 2).to(dev, torch.float64)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


@pytest.fixture(autouse=True)
def _no_grad():
    """the float64 restatements build no autograd graph; scoped to each test, so the process's grad mode is left as it was found"""
    with torch.no_grad():
        yield


def _forward(eng, entry, xs, frames, ds, debug):
    """one forward -> the per-sample RAFT flow (2B, 2, H, W) and the engine's outputs"""
    eng.set_debug(debug)
    if entry == "raft":
        nf = frames.shape[0]
        out = eng.raft_forward(frames, [(s, (s + nf // 2) % nf) for s in range(nf)], iters=ITERS, outputs=("flow_up", "flow_low"))
        return out["flow_up"], out
    B, H, W = xs.shape[0], xs.shape[-2], xs.shape[-1]
    coords = O.sample_coord_input(B, (H, W), [0.5], ds or 1.0).unsqueeze(0).contiguous().to(xs.device)   # at the network resolution
    out = eng.forward(xs, coords, torch.full((1, B), 0.5, device=xs.device), ds)
    rf = out["raft_flow"]
    return torch.cat([rf[:, :, 0], rf[:, :, 1]], 0), out


def _one_pair_matches(eng, xs, frames, taps, flow, B):
    """pair b alone against its place in the B-pair batch: RAFT has no atomics, so its flow and every raft.* tap agree bit for bit (samples
    b and B + b; frames likewise); the GIMM-VFI-R forward (taps off) gives the same raft_flow bit for bit, and a frame that moves by the
    splat's summation-order jitter only"""
    res = []
    fw, outB = _forward(eng, "R", xs, None, None, False)
    fw, img = fw.clone(), outB["imgt_pred"][0].clone()
    del outB
    for b in range(B):
        pick = lambda t: torch.cat([t[b:b + 1], t[B + b:B + b + 1]], 0)
        f1, _ = _forward(eng, "raft", None, pick(frames).contiguous(), None, True)
        bad = [k for k in TAPS if not torch.equal(eng.tap(k), pick(taps[k]))]
        r1, out1 = _forward(eng, "R", xs[b:b + 1].contiguous(), None, None, False)
        res.append(dict(flow=torch.equal(f1, pick(flow)), taps=bad, fwd=torch.equal(r1, pick(fw)),
                        img=(out1["imgt_pred"][0] - img[b:b + 1]).abs().max().item()))
    res.append(dict(same_as_forward=torch.equal(fw, flow)))
    return res


@pytest.fixture(scope="module", params=RUNS)
def run(request):
    """one forward with debug taps (and the engine profiler on the H100), then the engine freed; everything on the reference device"""
    case, kind, mode = request.param
    entry, B, H, W, ds, seed = CASES[case]
    from gimmvfi_b200.weights import random_state_dict
    sd = random_state_dict(0)
    if kind == "gpu":
        from gimmvfi_b200.engine import EngineHandle
        eng, dev = EngineHandle("cuda"), "cuda"
    else:
        from harness import hostsim_engine
        eng, dev = hostsim_engine(), "cpu"
    eng.load_state_dict(sd)
    eng.set_tensor_cores(mode)
    xs = synth_batch(B, H, W, seed=seed).to(dev)
    frames = (255 * torch.cat([xs[:, :, 0], xs[:, :, 1]], 0)).contiguous() if entry == "raft" else None
    t0 = time.time()
    if kind == "gpu":
        eng.set_profile(True)
    flow, out = _forward(eng, entry, xs, frames, ds, True)
    prof = None
    if kind == "gpu":
        torch.cuda.synchronize()
        prof = eng.profile()
        eng.set_profile(False)
    taps = {k: eng.tap(k) for k in TAPS}
    flow = flow.clone()
    del out
    bitwise = {}
    if kind == "gpu" and mode == 4 and case == "batch720":
        bitwise["one pair"] = _one_pair_matches(eng, xs, frames, taps, flow, B)
    if kind == "gpu" and mode == 4 and case == "pair1080":
        bitwise["taps off"] = torch.equal(_forward(eng, entry, xs, frames, ds, False)[0], flow)
    engine_s = time.time() - t0
    del eng
    gc.collect()
    if dev == "cuda":
        torch.cuda.empty_cache()
    sd64 = {k: (v.to(dev, torch.float64) if v.is_floating_point() else v) for k, v in sd.items()}
    if entry == "raft":
        img64 = 2 * (frames.double() / 255.0) - 1.0                                         # raft.py:111-112
    else:
        x64 = xs.double()
        net = torch.stack([O.resize(x64[:, :, 0], ds), O.resize(x64[:, :, 1], ds)], 2) if ds else x64   # gimmvfi_r.py:329-337
        img64 = 2 * torch.cat([net[:, :, 0], net[:, :, 1]], 0) - 1.0                       # gimmvfi_r.py:349 + raft.py:111-112
    S = 2 * B
    h, w = img64.shape[-2] // 8, img64.shape[-1] // 8
    pyr_gb = S * (h * w) ** 2 * 4 * 4 / 3 / 1e9
    route = "direct" if case == "raft4k" and kind == "gpu" else "volume"   # (the engine picks it when the pyramid exceeds 0.4 x 80 GB)
    yield dict(case=case, kind=kind, mode=mode, dev=dev, entry=entry, taps=taps, flow=flow, sd64=sd64, img64=img64, B=B, S=S, h=h, w=w,
               tgt=[(s + B) % S for s in range(S)], grid=O.coords_grid(S, h, w, img64), prof=prof, bitwise=bitwise, route=route,
               pyr_gb=pyr_gb, engine_s=engine_s)
    del taps, sd64
    gc.collect()
    if dev == "cuda":
        torch.cuda.empty_cache()


def maxdiff(got, ref):
    assert got.shape == ref.shape, (tuple(got.shape), tuple(ref.shape))
    return (got.to(ref.device, torch.float64) - ref).abs().max().item()


def check(run, rows):
    """rows: (stage, measured, bar); reports every stage, then asserts them all"""
    lines, bad = [], []
    for stage, err, bar in rows:
        lines.append("%-52s %.3e (bar %.1e)" % (stage, err, bar))
        if not err <= bar:
            bad.append(stage)
    print("\n%s %s mode %d (%s lookup, %dx%d grid, S = %d)\n  " % (run["case"], run["kind"], run["mode"], run["route"], run["h"], run["w"],
                                                                 run["S"]) + "\n  ".join(lines))
    assert not bad, "stages over their bar: %s\n%s" % (bad, "\n".join(lines))


def encoded_samples(run):
    return [0, run["S"] - 1] if run["case"] in ENCODE_ENDS else list(range(run["S"]))


def lookup_ratio(run, tap, coords):
    """max |engine - float64| / bound over every entry of a lookup, with the float64 lookup of the engine's own fmap at `coords`"""
    fm, dev = nchw(run["taps"]["raft.fmap"], run["dev"]), run["dev"]
    got = nchw(run["taps"][tap], dev)
    worst = 0.0
    for s in range(run["S"]):   # (one sample at a time: the float64 gathers of a 4K sample take ~1 GB)
        ref, bnd = corr_lookup64(fm[s:s + 1], fm[run["tgt"][s]:run["tgt"][s] + 1], coords[s:s + 1], chunk=1024, bound=run["route"])
        d = (got[s:s + 1] - ref).abs()
        worst = max(worst, torch.where(d == 0, torch.zeros_like(d), d / bnd).max().item())
    return worst


# The SepConvGRU's gates are convolutions over [h | inp | motion], K = 384 x 5 = 1920 terms t_k = w_k x_k.  Summed in fp32, each partial
# sum s_k is rounded once (|d_k| <= u), so the error is sum_k d_k s_k; with independent roundings its standard deviation is
# u sqrt(sum_k s_k^2 / 3), and for partial sums of terms of either sign sum_k s_k^2 ~ K |t|_2^2 / 2, i.e. sigma ~ u sqrt(K / 6) |t|_2.
# Blocked and tensor-core accumulation only shortens the chains.  The 3xTF32 / 3xF16 operand split leaves a relative error of at
# most 2^-22 per operand and the dropped lo x lo product (12 u per term, also of either sign): 12 u |t|_2 more.  The bound takes
# LAMBDA = 8 of the larger sigma sqrt(K / 3) (twice the variance of the model): a per-entry tail below 1e-15 for a Gaussian, and below
# 1e-7 over the 6.6e7 gate entries of a 4K pair.  The worst case over every sign pattern (Higham & Mary, SIAM J. Sci. Comput. 41
# (2019) A2815: lambda sqrt(K) u sum |t|) sits ~500x above the measured errors: it would let a 1e-4 mistake in the GRU state through.
LAMBDA = 8.0
GAMMA_GRU = LAMBDA * (math.sqrt(1920 / 3) + 12) * U


def gru_bound64(sd, net, inp, motion):
    """SepConvGRU (raft/update.py:35-73) in float64 from the engine's own input - net, inp and the motion features | flow of the same
    iteration - and the per-entry bound of an fp32-class GRU's distance from it, propagated to first order through both halves:
    each gate's pre-activation carries GAMMA_GRU |t|_2 (the square root of the convolution of W^2 with [h, x]^2, plus bias^2) and |W_h|
    applied to the error already in h; sigmoid' <= 1/4, tanh' <= 1, each activation adds 8 u (MUFU.EX2 / RCP, ~2 ulp), r h adds one
    rounding and the blend (1 - z) h + z q four of |h| + |q|"""
    g = P + ".update_block.gru"
    x = torch.cat([inp, motion], 1)
    h, eh = net, torch.zeros_like(net)
    zx = torch.zeros_like(x)
    for sfx, pad in (("1", (0, 2)), ("2", (2, 0))):
        wb = lambda n: (sd[g + n + sfx + ".weight"], sd[g + n + sfx + ".bias"])
        conv = lambda n, t: F.conv2d(t, *wb(n), padding=pad)
        rms = lambda n, t: F.conv2d(t * t, wb(n)[0] ** 2, wb(n)[1] ** 2, padding=pad).sqrt()      # |t|_2 of each output's terms
        prop = lambda n, e: F.conv2d(e, wb(n)[0].abs(), padding=pad)                              # |W| applied to an input error
        hx, ehx = torch.cat([h, x], 1), torch.cat([eh, zx], 1)
        z, r = torch.sigmoid(conv(".convz", hx)), torch.sigmoid(conv(".convr", hx))
        ez = 0.25 * (GAMMA_GRU * rms(".convz", hx) + prop(".convz", ehx)) + 8 * U
        er = 0.25 * (GAMMA_GRU * rms(".convr", hx) + prop(".convr", ehx)) + 8 * U
        rh = r * h
        erh = er * h.abs() + r * eh + U * rh.abs()
        rx = torch.cat([rh, x], 1)
        q = torch.tanh(conv(".convq", rx))
        eq = GAMMA_GRU * rms(".convq", rx) + prop(".convq", torch.cat([erh, zx], 1)) + 8 * U
        hn = (1 - z) * h + z * q
        eh = (1 - z) * eh + z * eq + ez * (q - h).abs() + 4 * U * (h.abs() + q.abs())
        h = hn
    return h, eh


def coord_rounding(run, coords):
    """fp32 rounding of a coordinate update and of coords - grid: 2 u (|coords| + |grid|), in pixels"""
    return 2 * U * (coords.abs().max().item() + max(run["h"], run["w"]))


# ---------------------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("h,w", [(23, 40), (34, 60)])
def test_corr_direct64_matches_corrblock(h, w):
    """the chunked float64 lookup against RAFT's own CorrBlock in float64 (all-pairs volume, the VOLUME average-pooled, grid_sample), at
    grids whose levels floor at odd sizes (23 x 40 -> 11 x 20 -> 5 x 10 -> 2 x 5; 34 x 60 -> 17 x 30 -> 8 x 15 -> 4 x 7), with windows
    inside, across and outside the frame"""
    g = torch.Generator().manual_seed(h)
    f0, f1 = torch.randn(2, 256, h, w, generator=g, dtype=torch.float64), torch.randn(2, 256, h, w, generator=g, dtype=torch.float64)
    base = O.coords_grid(2, h, w, f0)
    c = base + torch.cat([3 * torch.randn(1, 2, h, w, generator=g, dtype=torch.float64),
                          40 * torch.randn(1, 2, h, w, generator=g, dtype=torch.float64)], 0)
    ref = O.corr_lookup(O.corr_pyramid(O.all_pairs_corr(f0, f1).reshape(2 * h * w, 1, h, w)), c)
    got = corr_direct64(f0, f1, c, chunk=300)
    err = (got - ref).abs().max().item()
    print("\ncorr_direct64 vs CorrBlock (float64) at %dx%d: %.3e, |corr| <= %.1f; windows outside the frame per level: %s"
          % (h, w, err, ref.abs().max().item(), windows_outside(c, h, w)))
    assert ref.dtype == torch.float64 and ref.abs().max() > 1.0
    inside = windows_outside(c[:1], h, w)   # (sample 0: small displacements; every level-2 / 3 window reaches past those small frames)
    assert all(n > 0 for n in inside) and inside[0] < h * w
    assert err <= 1e-12


@pytest.mark.parametrize("route", ["volume", "direct"])
def test_lookup_bound_holds_fp32_and_rejects_a_shift(route):
    """the per-entry bound against an fp32 lookup of the same inputs: RAFT's CorrBlock in fp32 (volume), resp. that lookup on targets
    rounded to half (direct) lie within it; the same lookup at coordinates moved by 1e-3 px does not"""
    h, w = 34, 60
    g = torch.Generator().manual_seed(7)
    f0, f1 = torch.randn(1, 256, h, w, generator=g, dtype=torch.float64), torch.randn(1, 256, h, w, generator=g, dtype=torch.float64)
    c = O.coords_grid(1, h, w, f0) + 30 * torch.randn(1, 2, h, w, generator=g, dtype=torch.float64)
    c = c.float().double()   # coordinates the fp32 lookup holds exactly
    ref, bnd = corr_lookup64(f0, f1, c, chunk=500, bound=route)
    t32 = f1.float().half().float() if route == "direct" else f1.float()
    lk = lambda cc: O.corr_lookup(O.corr_pyramid(O.all_pairs_corr(f0.float(), t32).reshape(h * w, 1, h, w)), cc.float()).double()
    r32 = ((lk(c) - ref).abs() / bnd).nan_to_num(0.0).max().item()
    rsh = ((lk(c + 1e-3) - ref).abs() / bnd).nan_to_num(0.0).max().item()
    print("\n%s: fp32 lookup max |d| / bound %.3f; with the coordinates moved by 1e-3 px %.3f" % (route, r32, rsh))
    assert r32 <= 1.0 < rsh


def test_raft_stages(run):
    """Each stage from the engine's stored inputs against float64.  RAFT is fp32-class in every mode (mode 4: 3xTF32 / 3xF16 operands),
    so the bars are shared: each is derived next to it; the lookups are held to corr_ref's per-entry bound"""
    tp, dev, sd, S, B = run["taps"], run["dev"], run["sd64"], run["S"], run["B"]
    img, grid = run["img64"], run["grid"]
    rows = []
    # 1-2. the encoders on the prepared frames.  Instance-normalised features |f| <= ~10 after ~20 convolutions with K <= 2304: fp32
    #      reassociation ~1e-5.  The context: BatchNorm encoder -> tanh | relu, the same class.  Measured on an H100 80GB HBM3 (700 W)
    #      over the cases and modes: fmap 1.4e-5 (small) - 3.4e-5 (raft4k, mode 0); cnet 6.7e-6 - 2.7e-5 (raft4k, mode 4); the host
    #      simulation 1.6e-5 / 5.8e-6
    e_f, e_c = 0.0, 0.0
    for s in encoded_samples(run):
        f64 = O.basic_encoder(sd, P + ".fnet", img[s:s + 1], "instance")[0]
        e_f = max(e_f, maxdiff(tp["raft.fmap"][s:s + 1], nhwc(f64)))
        c64 = O.basic_encoder(sd, P + ".cnet", img[s:s + 1], "batch")[0]        # sample s's source is frame s
        e_c = max(e_c, maxdiff(tp["raft.cnet"][s:s + 1], nhwc(torch.cat([torch.tanh(c64[:, :128]), torch.relu(c64[:, 128:])], 1))))
    rows += [("1 raft.fmap (samples %s)" % encoded_samples(run), e_f, 1e-4), ("2 raft.cnet", e_c, 1e-4)]

    # 3-4. the lookups at iteration 0 (the integer grid: the volume's own entries) and at the last iteration, per entry within the bound
    #      (measured max |d| / bound: 0.075 - 0.40 on the H100, largest at r2k / batch720; 0.22 / 0.35 volume-free at 4K; hostsim 0.23)
    rows.append(("3 raft.corr_it0 max |d| / bound", lookup_ratio(run, "raft.corr_it0", grid), 1.0))
    cl = nchw(tp["raft.coords_last"], dev)
    rows.append(("4 raft.corr_last max |d| / bound", lookup_ratio(run, "raft.corr_last", cl), 1.0))
    out, cen = windows_outside(cl, run["h"], run["w"]), windows_outside(cl, run["h"], run["w"], r=0)
    print("\n%s: last-iteration windows straddling or leaving the frame per level: %s, window centres outside it: %s, of %d"
          % (run["case"], out, cen, cl[:, 0].numel()))
    # (every border pixel's window straddles the frame whatever the flow; a centre outside it is the flow's doing)
    assert all(n > 0 for n in cen), "no last-iteration window centre lies outside the frame at some level: the flow never leaves it"

    # 5. the update block at iteration 0 (net | inp = raft.cnet, flow 0) and at the last iteration (raft.net_last, raft.corr_last,
    #    raft.coords_last).  Chains of up to three convolutions with K <= 2304 (fp32-class): the sqrt(K)-scale reassociation of each, about
    #    2^-17 (128 u) of the largest output, is the bar for the motion features and the mask logits; the GRU alone, on the engine's own
    #    motion features, is held per entry to gru_bound64; the flow update adds the fp32 rounding of coords1 + delta and of
    #    coords1 - grid, 2 u (|coords| + |grid|): 1.2e-7 px per pixel of grid width.  Measured (H100, both modes): flow updates
    #    1.0e-6 (small) - 1.6e-5 px (raft4k), 0.13 of their bars; motion 6.9e-6 - 4.3e-5 (0.2 of the bar); GRU state 0.016 - 0.047 of
    #    gru_bound64 (0.031 small - 0.047 raft4k in mode 0, 0.016 - 0.018 in mode 4; hostsim 0.032);
    #    mask 7.3e-8 - 2.8e-7
    cn = nchw(tp["raft.cnet"], dev)
    _, _, d0 = O.raft_update_block(sd, P + ".update_block", cn[:, :128], cn[:, 128:], nchw(tp["raft.corr_it0"], dev), torch.zeros_like(grid))
    rows.append(("5 it 0: raft.lowres_flow_it0", maxdiff(tp["raft.lowres_flow_it0"], nhwc(d0)), 1e-5 + coord_rounding(run, grid)))
    fl = cl - grid
    corr_l = nchw(tp["raft.corr_last"], dev)
    mot = O.raft_motion_encoder(sd, P + ".update_block", corr_l, fl)
    rel = lambda ref: 2.0 ** -17 * max(1.0, ref.abs().max().item())
    rows.append(("5 last: raft.motion_last", maxdiff(tp["raft.motion_last"], nhwc(mot)), rel(mot)))
    hN, mask, dN = O.raft_update_block(sd, P + ".update_block", nchw(tp["raft.net_last"], dev), cn[:, 128:], corr_l, fl)
    # the GRU alone, on the engine's own motion features, per entry within gru_bound64
    hG, eG = gru_bound64(sd, nchw(tp["raft.net_last"], dev), cn[:, 128:], nchw(tp["raft.motion_last"], dev))
    rows.append(("5 last: raft.net_final (GRU) max |d| / bound", (nchw(tp["raft.net_final"], dev) - hG).abs().div(eG).max().item(), 1.0))
    rows.append(("5 last: raft.mask", maxdiff(tp["raft.mask"], nhwc(mask)), rel(mask)))
    upd = nchw(tp["raft.lowres_flow_final"], dev) + grid - cl
    rows.append(("5 last: lowres_flow_final - coords_last", maxdiff(nhwc(upd), nhwc(dN)), 1e-5 + coord_rounding(run, cl)))

    # 6. convex upsampling of the engine's final low-resolution flow with its mask, at every pixel: a 9-way softmax (expf) and a 9-term
    #    sum of 8 flow, ~16 roundings of 8 |flow| (measured 3.2e-6 small - 1.3e-5 raft4k, 0.15 - 0.3 of the bar)
    low = nchw(tp["raft.lowres_flow_final"], dev)
    up = O.convex_upsample(low, nchw(tp["raft.mask"], dev))
    rows.append(("6 convex upsampling (every pixel)", maxdiff(run["flow"], up), 1e-6 + 16 * U * 8 * low.abs().max().item()))
    check(run, rows)


def test_raft_composed(run):
    """20 float64 iterations from the engine's raft.fmap and raft.cnet, every lookup in float64, against the engine's flows at EVERY pixel:
    test_raft_gpu.py's flow_low / flow_up bars (2e-3 / 1e-2 px), which it applies on a stride-8 subsample"""
    tp, dev, sd, S = run["taps"], run["dev"], run["sd64"], run["S"]
    grid = run["grid"]
    fm, cn = nchw(tp["raft.fmap"], dev), nchw(tp["raft.cnet"], dev)
    ftgt = fm[run["tgt"]]
    net, inp, coords = cn[:, :128], cn[:, 128:], grid.clone()
    for _ in range(ITERS):
        corr = corr_direct64(fm, ftgt, coords, chunk=1024)
        net, mask, dflow = O.raft_update_block(sd, P + ".update_block", net, inp, corr, coords - grid)
        coords = coords + dflow
    low = coords - grid
    up = O.convex_upsample(low, mask)
    # measured on the H100 (modes 0 / 4): flow_low 7.2e-6 / 1.0e-5 (small), 7.8e-5 / 7.6e-5 (pair1080), 8.8e-5 / 8.4e-5 (batch720),
    # 3.7e-5 / 4.1e-5 (r2k), 1.9e-4 / 2.0e-4 (raft4k); the upsampled flow 2.2e-5 - 8.9e-4 px (raft4k); the host simulation 8.9e-6 / 2.3e-5
    check(run, [("7 composed: raft.lowres_flow_final (every pixel)", maxdiff(tp["raft.lowres_flow_final"], nhwc(low)), 2e-3),
                ("7 composed: raft flow (every pixel)", maxdiff(run["flow"], up), 1e-2)])


def test_raft_route(run):
    """the route each case claims ran, by the engine profiler's kernel names (the automatic choice depends on the device's memory: a
    silent change of route must fail here)"""
    if run["kind"] != "gpu":
        pytest.skip("the profiler and the routes are the H100's")
    prof, mode = run["prof"], run["mode"]
    n = lambda k: prof.get(k, {}).get("launches", 0)
    gemm = "corr_gemm_nt" if mode == 0 else "corr_gemm_tc_3xf16"
    names = ("corr_gemm_nt", "corr_gemm_tc_3xf16", "corr_gemm_tc_3xtf32", "corr_gemm_tc_tf32", "corr_lookup", "corr_lookup_direct")
    print("\n%s mode %d (%s, a %.1f GB pyramid): %s" % (run["case"], mode, run["route"], run["pyr_gb"], {k: n(k) for k in names}))
    if run["route"] == "direct":
        # pairs (0, 1), (1, 0) are two runs of the pair list: one launch each per iteration; no volume at all
        assert n("corr_lookup_direct") == 2 * ITERS and not any(n(k) for k in names[:5]), sorted(prof)
    elif run["entry"] == "raft":
        assert n(gemm) >= 1 and n("corr_lookup") == ITERS and not n("corr_lookup_direct"), sorted(prof)
    else:
        # GIMM-VFI-R at T = 1: the bidirectional lookup after RAFT is volume-free in mode 4 (2 launches) and looks up the fp32 volume
        # in mode 0 (2 launches of corr_lookup)
        assert n(gemm) >= 1 and n("corr_lookup") == ITERS + (2 if mode == 0 else 0), sorted(prof)
        assert n("corr_lookup_direct") == (2 if mode == 4 else 0), sorted(prof)


def test_raft_bitwise(run):
    """batch720, mode 4: each of the 8 pairs alone equals its place in the batch (raft_flow and every raft.* tap bit for bit, the frame
    within test_forward_gpu's repeat jitter, 6e-4); pair1080, mode 4: the taps do not change the flow (bit for bit)"""
    if not run["bitwise"]:
        pytest.skip("batch720 and pair1080 in mode 4 only")
    print("\n%s: engine wall time %.1f s (forwards and taps)" % (run["case"], run["engine_s"]))
    if "one pair" in run["bitwise"]:
        res, last = run["bitwise"]["one pair"][:-1], run["bitwise"]["one pair"][-1]
        for b, r in enumerate(res):
            print("pair %d alone: RAFT flow torch.equal %s, raft.* taps differing %s; GIMM-VFI-R forward: raft_flow torch.equal %s, imgt_pred "
                  "max |d| %.3e" % (b, r["flow"], r["taps"], r["fwd"], r["img"]))
        print("the B = 8 forward's raft_flow torch.equal raft_forward's flow of its 16 pairs: %s" % last["same_as_forward"])
        assert all(r["flow"] and not r["taps"] and r["fwd"] and r["img"] <= 6e-4 for r in res)
        # the forward's own RAFT is the one checked above against float64: raft_forward on its 16 pairs gives the same flow bit for bit
        assert last["same_as_forward"]
    if "taps off" in run["bitwise"]:
        print("raft_flow with the taps off torch.equal the forward with them on: %s" % run["bitwise"]["taps off"])
        assert run["bitwise"]["taps off"]
