"""GIMM's motion stage and the H/4 decoders stage by stage against float64: normalize_flow, the splatting weights, cnn_encoder, the
forward splat to time t, res_conv, HypoNet, unnormalize_flow, the init decoder, the bidirectional correlation lookup and both AMT update
blocks - everything Engine::run does between the flow estimator and the synthesis tail (tests/test_synthesis_tail_gpu.py).

Each stage is fed the engine's own stored input (its debug taps, EngineHandle.tap, and its aux outputs), so that no upstream difference
reaches its bar; the reference is the oracle (oracle/gimmvfi_r_oracle.py) in float64 with the weights cast to double.  The per-timestep
taps are taken at the last timestep, so the timestep a case inspects is put last; the others only set the route the engine takes (T > 2:
the all-pairs correlation pyramid instead of the volume-free lookup).

The forward splat is discontinuous where its normaliser D -> 0, so it is held to a per-pixel bound of its fp32 rounding instead of a flat
bar.  Everything after it is continuous (convolutions, sin, bilinear lookups with zero padding, border-clamped warps, sigmoid, clamp), so
the composed check - float64 from the engine's splat outputs to the frame - is held per pixel at every size.

Cases: a small GIMM-VFI-R batch with per-sample t and ds_factor 0.5 (the host simulation and the H100), the same size at T = 3 with
t = 1/8 last, and on the H100 the three benchmarked configurations at bench.py's inputs: pair1080 (GIMM-VFI-R, T = 1), f2k and f4k
(GIMM-VFI-F, native FlowFormer, T = 7) with t = 1/8 or t = 7/8 last.  Backends: the CPU build of the same sources (tests/hostsim, fp32,
mode 0) and the H100 in precision modes 0 (fp32 CUDA cores) and 4 (the default).  Layouts: the engine stores NHWC, the oracle NCHW."""
import gc
import math
import os
import sys

import pytest
import torch

import gimmvfi_r_oracle as O
from gimmvfi_b200.synth import synth_batch
from corr_ref import corr_direct64
from splat_ref import splat_w_bound, splat_w_float64

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim"))

U = 2.0 ** -24   # fp32 unit roundoff
_F8 = [(i / 8,) for i in range(1, 8)]   # bench.py's f2k / f4k timesteps, t = i / 8
# name: model, full size, ds_factor, per-timestep per-sample t (the last timestep is the one inspected), input seed
CASES = {
    "small": ("R", 272, 400, 0.5, [(0.25, 0.75)], 41),
    "small-T3": ("R", 272, 400, None, [(0.5,), (0.875,), (0.125,)], 41),
    "pair1080": ("R", 1088, 1920, None, [(0.5,)], 100),
    "f2k-t1of8": ("F", 1088, 2048, 0.5, _F8[1:] + _F8[:1], 100),
    "f2k-t7of8": ("F", 1088, 2048, 0.5, _F8, 100),
    "f4k-t1of8": ("F", 2176, 4096, 0.25, _F8[1:] + _F8[:1], 100),
    "f4k-t7of8": ("F", 2176, 4096, 0.25, _F8, 100),
}
RUNS = [pytest.param(("small", "hostsim", 0), id="small-hostsim-mode0")]
RUNS += [pytest.param((c, "gpu", m), id="%s-h100-mode%d" % (c, m), marks=pytest.mark.gpu) for c in CASES for m in (0, 4)]
TAPS = ["gimm.splat_w", "gimm.lat0", "gimm.lat1", "gimm.splat0", "gimm.splat1", "gimm.latent", "syn.feat4", "syn.feat8", "syn.fup4",
        "syn.fproj", "syn.fin4", "syn.ft4_init", "syn.fl4_init", "syn.mask4_init", "syn.corr648", "syn.ft4_low", "syn.fl4_low",
        "syn.ft_4", "syn.fl4", "syn.mask4"]
OUTS = ["raft_flow", "nflow", "ninrflow", "flowt", "imgt_pred"]


def nchw(t, dev):
    return t.permute(0, 3, 1, 2).to(dev, torch.float64)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def route(kind, mode, T):
    """which bidirectional correlation the engine runs (Engine::run: corr_direct_max_t_ = 2; mode 0 always builds the fp32 volume)"""
    return "direct" if kind == "gpu" and mode >= 1 and T <= 2 else "volume"


@pytest.fixture(autouse=True)
def _no_grad():
    """the float64 restatements build no autograd graph; scoped to each test, so the process's grad mode is left as it was found"""
    with torch.no_grad():
        yield


@pytest.fixture(scope="module", params=RUNS)
def run(request):
    """one eager forward with debug taps (and the engine profiler on the H100); everything on the reference device.  Nothing here
    requires grad, so no graph is built without switching the process's grad mode"""
    case, kind, mode = request.param
    model, H, W, ds, tss, seed = CASES[case]
    if model == "R":
        from gimmvfi_b200.weights import random_state_dict
        sd = random_state_dict(0)
    else:
        from gimmvfi_b200.weights import random_state_dict_f
        sd = random_state_dict_f(0)
    if kind == "gpu":
        from gimmvfi_b200.engine import EngineHandle
        eng, dev = EngineHandle("cuda"), "cuda"
    else:
        from harness import hostsim_engine
        eng, dev = hostsim_engine(), "cpu"
    eng.load_state_dict(sd, full_f=model == "F")
    eng.set_tensor_cores(mode)
    B, T = len(tss[0]), len(tss)
    xs = synth_batch(B, H, W, seed=seed).to(dev)

    def inputs(order):
        c = torch.stack([torch.cat([O.sample_coord_input(1, (H, W), [t], ds or 1.0) for t in ts], 0) for ts in order], 0)
        return c.contiguous().to(dev), torch.tensor(order, dtype=torch.float32).to(dev)

    coords, tt = inputs(tss)
    eng.set_debug(True)   # (no CUDA-graph replay with taps on)
    if kind == "gpu":
        eng.set_profile(True)
    out = eng.forward(xs, coords, tt, ds)
    prof = None
    if kind == "gpu":
        torch.cuda.synchronize()
        prof = eng.profile()
        eng.set_profile(False)
    taps = {k: eng.tap(k) for k in TAPS}
    res = {k: out[k] for k in OUTS}
    res.update(ninrflow=out["ninrflow"][T - 1], flowt=out["flowt"][T - 1], img=out["imgt_pred"][T - 1].clone())
    bench = None
    if tss != sorted(tss) and model == "F":
        # the same frame in two forwards with bench.py's timestep order (t = i / 8 ascending: the inspected t = 1/8 comes first); the
        # second measures how much two identical forwards differ
        eng.set_debug(False)
        cb, tb = inputs(sorted(tss))
        bench = [{k: v[0].clone() if k == "imgt_pred" else v.clone() for k, v in eng.forward(xs, cb, tb, ds, aux_outputs=("raft_flow",)).items()}
                 for _ in range(2)]
    del eng, out
    gc.collect()
    if dev == "cuda":
        torch.cuda.empty_cache()
    sd64 = {k: (v.to(dev, torch.float64) if v.is_floating_point() else v) for k, v in sd.items()}
    x64 = xs.double()
    net = torch.stack([O.resize(x64[:, :, 0], ds), O.resize(x64[:, :, 1], ds)], 2) if ds else x64   # gimmvfi_r.py:329-337
    yield dict(case=case, kind=kind, mode=mode, dev=dev, taps=taps, out=res, sd64=sd64, full=x64 if ds else None, B=B, T=T,
               img0=2 * net[:, :, 0] - 1.0, img1=2 * net[:, :, 1] - 1.0, coords=coords[T - 1].double(),
               t=tt[T - 1].double().view(B, 1, 1, 1), prof=prof, bench=bench, route=route(kind, mode, T))
    del taps, sd64, res
    gc.collect()
    if dev == "cuda":
        torch.cuda.empty_cache()


def maxdiff(got, ref):
    assert got.shape == ref.shape, (tuple(got.shape), tuple(ref.shape))
    return (got.to(ref.device, torch.float64) - ref).abs().max().item()


def check(run, rows):
    """rows: (stage, measured, {key: bar}) with key "hostsim" or the H100 precision mode; reports every stage, then asserts them all"""
    key = "hostsim" if run["kind"] == "hostsim" else run["mode"]
    lines, bad = [], []
    for stage, err, bars in rows:
        lines.append("%-46s %.3e (bar %.1e)" % (stage, err, bars[key]))
        if not err <= bars[key]:
            bad.append(stage)
    print("\n%s %s mode %d (%s correlation)\n  " % (run["case"], run["kind"], run["mode"], run["route"]) + "\n  ".join(lines))
    assert not bad, "stages over their bar: %s\n%s" % (bad, "\n".join(lines))


# ----------------------------------------------------------------------------------------------------------- float64 restatements
def _corners(flow):
    """the forward splat's targets (oracle.forward_splat_sum): per corner (flat target index, in-frame mask, bilinear weight), and the
    landing position x + f, y + f"""
    N, _, H, W = flow.shape
    kw = dict(device=flow.device, dtype=flow.dtype)
    gx = torch.arange(W, **kw).view(1, 1, W).expand(N, H, W)
    gy = torch.arange(H, **kw).view(1, H, 1).expand(N, H, W)
    fx, fy = gx + flow[:, 0], gy + flow[:, 1]
    x0, y0 = torch.floor(fx).long(), torch.floor(fy).long()
    nidx = torch.arange(N, device=flow.device).view(N, 1, 1).expand(N, H, W)
    out = []
    for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
        xx, yy = x0 + dx, y0 + dy
        wx = (fx - x0) if dx else (x0 + 1 - fx)
        wy = (fy - y0) if dy else (y0 + 1 - fy)
        ok = ((xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)).reshape(-1)
        lin = ((nidx * H + yy.clamp(0, H - 1)) * W + xx.clamp(0, W - 1)).reshape(-1)
        out.append((lin[ok], ok, (wx * wy).reshape(-1)[ok]))
    return out, fx, fy


def splat64(lat, flow, metric):
    """softsplat "linear-zeroeps" of the engine's latents in float64 and the per-pixel bound of an fp32 implementation's distance from it,
    both (N, C, H, W).  fp32 rounds the landing position x + f·s once or twice: δ <= 2^-24 (|f·s| + |x + f·s|) per axis, which moves each
    bilinear weight by at most δx + δy (unit slope); through the normalisation out = Σ w b lat / Σ w b that is Σ_i w_i δ_i |lat_i - out| / D.
    The re-associated (atomic) sums of n terms and the products w·b·lat add (n + 4) 2^-24 (Σ w b |lat| + D |out|) / D.  Both are divided by
    the smallest D the perturbed weights allow; where that reaches 0 the bound is infinite (an ill-conditioned pixel)."""
    N, C, H, W = lat.shape
    corners, fx, fy = _corners(flow)
    delta = 2 * U * ((fx - torch.arange(W, device=lat.device)).abs() + fx.abs() + (fy - torch.arange(H, device=lat.device).view(H, 1)).abs()
                     + fy.abs()).reshape(-1, 1)
    src = lat.permute(0, 2, 3, 1).reshape(N * H * W, C)
    w = metric.permute(0, 2, 3, 1).reshape(N * H * W, 1)
    z = lambda c: torch.zeros(N * H * W, c, device=lat.device, dtype=torch.float64)
    num, den, absn, wd, cnt = z(C), z(1), z(C), z(1), z(1)
    for lin, ok, b in corners:
        wb = w[ok] * b.view(-1, 1)
        num.index_add_(0, lin, wb * src[ok])
        den.index_add_(0, lin, wb)
        absn.index_add_(0, lin, wb * src[ok].abs())
        wd.index_add_(0, lin, w[ok] * delta[ok])
        cnt.index_add_(0, lin, torch.ones_like(wb))
    out = num / torch.where(den == 0, torch.ones_like(den), den)
    spread = z(C)
    for lin, ok, b in corners:
        spread.index_add_(0, lin, (w[ok] * delta[ok]) * (src[ok] - out[lin]).abs())
    dlo = den - wd
    bound = (spread + (cnt + 4) * U * (absn + den * out.abs())) / dlo.clamp(min=1e-300)
    bound = torch.where(dlo > 0, bound, torch.full_like(bound, math.inf))
    bound = torch.where(cnt == 0, torch.zeros_like(bound), bound)   # no source reaches the pixel: both give exactly 0
    shape = lambda t: t.view(N, H, W, -1).permute(0, 3, 1, 2)
    return shape(out), shape(bound)


def lookup_coords64(fl4, t):
    """_amt_corr_scale_lookup (gimmvfi_r.py:494-507): the H/4 flows at H/8 and the two lookup positions"""
    fl0, fl1 = 0.5 * O.resize(fl4[:, :2], 0.5), 0.5 * O.resize(fl4[:, 2:], 0.5)
    B, _, h, w = fl0.shape
    coord = O.coords_grid(B, h, w, fl0)
    return fl0, fl1, coord + fl1 * (1.0 / (1.0 - t)), coord + fl0 * (1.0 / t)


def bidir_lookup64(fproj, fl4, t):
    """corr648 = [frame 0's pixels against frame 1's features | the transposed volume's counterpart] at lookup_coords(fl4, t)"""
    B = fl4.shape[0]
    fl0, fl1, cA, cB = lookup_coords64(fl4, t)
    return torch.cat([corr_direct64(fproj[:B], fproj[B:], cA), corr_direct64(fproj[B:], fproj[:B], cB)], 1), fl0, fl1, cA, cB


def flow_scale(run):
    """normalize_flow's per-sample scale: max |flow| over both directions (B, 1, 1, 1)"""
    f = run["out"]["raft_flow"].double()
    return f.abs().flatten(1).max(1)[0].view(-1, 1, 1, 1)


def chain64(run, lat0, lat1, sp0, sp1, fup4, fup1):
    """float64 from the splat outputs to the frame: res_conv, HypoNet, unnormalize_flow, the init decoder, the bidirectional lookup on
    the engine's syn.fproj, both update blocks and synthesis_tail"""
    sd, B, t, dev = run["sd64"], run["B"], run["t"], run["dev"]
    sp = torch.cat([sp0, sp1], 1)
    lat = sp + O.res_conv(sd, torch.cat([lat0, lat1, sp], 1))
    ninr = O.hyponet_forward(sd, run["coords"], lat.permute(0, 2, 3, 1))[:, 0].permute(0, 3, 1, 2)   # (B, 2, Hc, Wc)
    flowt = (ninr * 2.0 - 1.0) * flow_scale(run)
    ft0, ft1 = 0.25 * O.resize(flowt * (-t), 0.25), 0.25 * O.resize(flowt * (1.0 - t), 0.25)
    f0, f1, rest = O.init_convblock(sd, O.init_decoder_concat(fup4[:B], fup4[B:], ft0, ft1, run["img0"], run["img1"]), ft0, ft1)
    mask4, ft = rest[:, :1], rest[:, 1:]
    fl4 = torch.cat([f0, f1], 1)
    corr, fl0, fl1, _, _ = bidir_lookup64(nchw(run["taps"]["syn.fproj"], dev), fl4, t)
    dft, dfl = O.amt_update_block(sd, "amt_update4_low", ft, torch.cat([fl0, fl1], 1), corr, 2.0)
    ft, fl4 = ft + dft, fl4 + dfl
    dft, dfl = O.amt_update_block(sd, "amt_update4_high", ft, fl4, O.resize(corr, 2.0), None)
    ft, fl4 = ft + dft, fl4 + dfl
    pred, _, _ = O.synthesis_tail(sd, ft, fl4[:, :2], fl4[:, 2:], mask4, fup1[:B], fup1[B:], run["img0"], run["img1"], run["full"])
    return pred


# ---------------------------------------------------------------------------------------------------------------------------- tests
def test_corr_direct64_matches_bidircorr():
    """the chunked float64 lookup against the oracle's BidirCorr (all-pairs volume, avg-pooled pyramid, grid_sample) in float64, at odd
    level sizes (17 x 25 -> 8 x 12 -> 4 x 6 -> 2 x 3) and with windows inside, across and outside the frame"""
    g = torch.Generator().manual_seed(3)
    f0, f1 = torch.randn(2, 256, 17, 25, generator=g, dtype=torch.float64), torch.randn(2, 256, 17, 25, generator=g, dtype=torch.float64)
    base = O.coords_grid(2, 17, 25, f0)
    c0 = base + 6 * torch.randn(2, 2, 17, 25, generator=g, dtype=torch.float64)
    c1 = base + 30 * torch.randn(2, 2, 17, 25, generator=g, dtype=torch.float64)
    r0, r1 = O.BidirCorr(f0, f1)(c0, c1)
    d0, d1 = corr_direct64(f0, f1, c0, chunk=100), corr_direct64(f1, f0, c1, chunk=100)
    err = max((d0 - r0).abs().max().item(), (d1 - r1).abs().max().item())
    print("\ncorr_direct64 vs BidirCorr (float64): %.3e, |corr| <= %.1f" % (err, r0.abs().max().item()))
    assert r0.dtype == torch.float64 and r0.abs().max() > 1.0
    assert err <= 1e-12


def test_motion_stages(run):
    """Each stage from the engine's stored input against float64.  Bars: about 2-4x the measured value on an H100 80GB HBM3 (700 W) and
    on the host simulation, the largest over the cases, written next to each bar; fp32 stages share the host simulation's bars."""
    tp, out, dev, sd, B, mode, t = run["taps"], run["out"], run["dev"], run["sd64"], run["B"], run["mode"], run["t"]
    fp32 = lambda b: {"hostsim": b, 0: b, 4: b}
    rows = []
    flows = out["raft_flow"].to(dev, torch.float64)                                    # (B, 2, 2, H, W): [f01 | f10] on dim 2
    # 1. normalize_flow: (f / max|f| + 1) / 2 in fp32, values in [0, 1] (measured 4.5e-8 everywhere: < 1 ulp of 1)
    nflow_ref, _ = O.normalize_flow(torch.stack([flows[:, :, 0], -flows[:, :, 1]], 2))
    rows.append(("1 nflow", maxdiff(out["nflow"], nflow_ref), fp32(1.5e-7)))

    # 2. splatting weights, per pixel within test_stages_gpu's conditioning bound (var = sqrt(E[f^2] - E[f]^2) cancels where the flow is
    #    locally constant, and backwarp rounds its sample position where the flow is steep).  Measured max |d| / bound: 0.57 hostsim,
    #    0.45 - 0.85 on the H100 over the cases and modes (without the sample-position term: up to 1.7 at f2k)
    w64 = splat_w_float64(sd, flows)
    rows.append(("2 gimm.splat_w max |d| / bound", ((tp["gimm.splat_w"].double().to(dev) - w64).abs() / splat_w_bound(sd, flows)).max().item(),
                 fp32(1.0)))

    # 3. motion latents from the engine's nflow.  fp32: reassociation over K <= 32 x 9 (measured ...).  Mode 4: the 32-channel
    #    full-resolution chain stored in half on TF32 / f16 operands (measured 3.3e-7 / 3.7e-4, |lat| <= 0.3)
    nflow_e = out["nflow"].to(dev, torch.float64)
    for j in (0, 1):
        lat = O.cnn_encoder(sd, nflow_e[:, :, j])
        rows.append(("3 gimm.lat%d" % j, maxdiff(tp["gimm.lat%d" % j], nhwc(lat)), {"hostsim": 1e-6, 0: 1e-6, 4: 1e-3}))

    # 4. the forward splat to t from the engine's latents, flows and weights, per pixel within splat64's bound
    lat0, lat1 = nchw(tp["gimm.lat0"], dev), nchw(tp["gimm.lat1"], dev)
    wts = nchw(tp["gimm.splat_w"], dev)
    sps = []
    for j, (lat, f, s, w) in enumerate(((lat0, flows[:, :, 0], t, wts[:B]), (lat1, flows[:, :, 1], 1.0 - t, wts[B:]))):
        ref, bound = splat64(lat, f * s, w)
        d = (nchw(tp["gimm.splat%d" % j], dev) - ref).abs()
        ratio = torch.where(d == 0, torch.zeros_like(d), d / bound).max().item()
        ill = (bound > 1e-4).any(1)
        print("\n%s: gimm.splat%d max |d| %.3e; %d of %d pixels have a bound above 1e-4 (%d unbounded: D can reach 0)"
              % (run["case"], j, d.max().item(), int(ill.sum()), ill.numel(), int(torch.isinf(bound).any(1).sum())))
        rows.append(("4 gimm.splat%d max |d| / bound" % j, ratio, fp32(1.0)))
        sps.append(ref)

    # 5. res_conv from the engine's [lat0 | lat1 | splat0 | splat1]: as stage 3 (64 -> 32 channels, K <= 64 x 9; measured 1.3e-7 / 1.6e-4)
    X = torch.cat([lat0, lat1, nchw(tp["gimm.splat0"], dev), nchw(tp["gimm.splat1"], dev)], 1)
    latent = X[:, 32:] + O.res_conv(sd, X)
    rows.append(("5 gimm.latent", maxdiff(tp["gimm.latent"], nhwc(latent)), {"hostsim": 5e-7, 0: 5e-7, 4: 5e-4}))

    # 6. HypoNet on the network-resolution grid from the engine's latent: fp32-class in both modes (hyponet_fused3 / five 1x1 convs),
    #    sin layers of 128, output in [0, 1] (measured 6.3e-7 mode 0; 1.5e-6 mode 4, whose 3xTF32 split rounds once more per layer)
    ninr = O.hyponet_forward(sd, run["coords"], tp["gimm.latent"].to(dev, torch.float64))           # (B, 1, Hc, Wc, 2)
    rows.append(("6 ninrflow", maxdiff(out["ninrflow"], ninr.permute(0, 4, 1, 2, 3)), {"hostsim": 2e-6, 0: 2e-6, 4: 4e-6}))

    # 7. unnormalize_flow: (2 o - 1) * max|flow|, |flow| up to ~38 px (measured 1.9e-6 pair1080: one ulp of 16-32 px)
    flowt_e = out["flowt"].to(dev, torch.float64)
    ref = (out["ninrflow"][:, :, 0].to(dev, torch.float64) * 2.0 - 1.0) * flow_scale(run)
    rows.append(("7 flowt", maxdiff(out["flowt"], ref), fp32(5e-6)))

    # 8. init decoder: the upsample branch from syn.feat8 (fp32 in both modes, TF32 operands in mode 4), the 272-channel concat from the
    #    engine's flowt and fup4 (fp32 pointwise: the warps carry the sample position's float round trip times the source's gradient),
    #    and the trunk + head from the engine's concat (H/4 trunk stored in half in mode 4).  Measured (the largest over the cases):
    #    fup4 8.7e-8 / 1.6e-4; warped features 1.4e-6, flows 5.8e-7, frames 1.0e-7, warped frames 6.3e-6 in both modes;
    #    ft4 / fl4 / mask4 6.5e-7 / 4.5e-7 / 4.7e-7 in mode 0, 3.7e-4 / 2.6e-4 / 3.0e-4 in mode 4
    fup4 = O._decoder_upsample(sd, "amt_init_decoder.upsample", nchw(tp["syn.feat8"], dev), 1)
    rows.append(("8 syn.fup4", maxdiff(tp["syn.fup4"], nhwc(fup4)), {"hostsim": 3e-7, 0: 3e-7, 4: 5e-4}))
    ft0, ft1 = 0.25 * O.resize(flowt_e * (-t), 0.25), 0.25 * O.resize(flowt_e * (1.0 - t), 0.25)
    fup4_e = nchw(tp["syn.fup4"], dev)
    fin = nhwc(O.init_decoder_concat(fup4_e[:B], fup4_e[B:], ft0, ft1, run["img0"], run["img1"]))
    for g, c0, c1, a in (("backwarp(fup4 frame 0)", 0, 128, 4e-6), ("backwarp(fup4 frame 1)", 128, 256, 4e-6),
                         ("flows", 256, 260, 2e-6), ("frames", 260, 266, 4e-7), ("backwarp(frames)", 266, 272, 2e-5)):
        rows.append(("8 syn.fin4 %s" % g, maxdiff(tp["syn.fin4"][..., c0:c1], fin[..., c0:c1]), fp32(a)))
    fin_e = nchw(tp["syn.fin4"], dev)
    f0, f1, rest = O.init_convblock(sd, fin_e, fin_e[:, 256:258], fin_e[:, 258:260])
    rows.append(("8 syn.ft4_init", maxdiff(tp["syn.ft4_init"], nhwc(rest[:, 1:])), {"hostsim": 2e-6, 0: 2e-6, 4: 1e-3}))
    rows.append(("8 syn.fl4_init", maxdiff(tp["syn.fl4_init"], nhwc(torch.cat([f0, f1], 1))), {"hostsim": 1.5e-6, 0: 1.5e-6, 4: 1e-3}))
    rows.append(("8 syn.mask4_init", maxdiff(tp["syn.mask4_init"], nhwc(rest[:, :1])), {"hostsim": 1.5e-6, 0: 1.5e-6, 4: 1e-3}))

    # 9. the bidirectional lookup at lookup_coords(fl4_init, t), against the float64 lookup of the engine's syn.fproj.  Mode 0: the fp32
    #    volume (256-term dot products).  Mode 4: the volume-free lookup rounds the target features to half (T <= 2); the volume route
    #    (T > 2) runs plain TF32 GEMMs.  Measured: 5.7e-4 mode 0 (pair1080, |corr| of R's projected features is largest there),
    #    3.2e-3 direct (pair1080), 8.8e-3 volume (small-T3), on |corr| up to ~20
    fl4i = nchw(tp["syn.fl4_init"], dev)
    corr, fl0, fl1, cA, cB = bidir_lookup64(nchw(tp["syn.fproj"], dev), fl4i, t)
    b4 = 1e-2 if run["route"] == "direct" else 2.5e-2
    rows.append(("9 syn.corr648 (%s)" % run["route"], maxdiff(tp["syn.corr648"], nhwc(corr)), {"hostsim": 1.5e-3, 0: 1.5e-3, 4: b4}))
    h, w = fl0.shape[-2:]
    outside = []
    for l in range(4):
        hl, wl = h >> l, w >> l
        cnt = 0
        for c in (cA, cB):
            cx, cy = c[:, 0] / 2 ** l, c[:, 1] / 2 ** l
            cnt += int(((cx - 4 < 0) | (cx + 4 > wl - 1) | (cy - 4 < 0) | (cy + 4 > hl - 1)).sum().item())
        outside.append(cnt)
    print("\n%s: lookup windows reaching outside the frame per level: %s of %d" % (run["case"], outside, 2 * cA[:, 0].numel()))
    assert all(n > 0 for n in outside), "a pyramid level never looks outside its frame: the zero padding is not exercised"

    # 10. amt_update4_low from the engine's init state and lookup; amt_update4_high from the engine's low state and resize(corr648, 2).
    #     fp32: reassociation over K <= 648 / 320 x 9 (measured 3.2e-7 / 5.2e-7 / 7.0e-7 / 6.1e-7); mode 4: TF32 operands (measured
    #     1.7e-4 / 2.4e-4 / 2.4e-4 / 2.3e-4, pair1080)
    corr_e = nchw(tp["syn.corr648"], dev)
    ft4i = nchw(tp["syn.ft4_init"], dev)
    dft, dfl = O.amt_update_block(sd, "amt_update4_low", ft4i, torch.cat([fl0, fl1], 1), corr_e, 2.0)
    rows.append(("10 syn.ft4_low", maxdiff(tp["syn.ft4_low"], nhwc(ft4i + dft)), {"hostsim": 1e-6, 0: 1e-6, 4: 5e-4}))
    rows.append(("10 syn.fl4_low", maxdiff(tp["syn.fl4_low"], nhwc(fl4i + dfl)), {"hostsim": 1.5e-6, 0: 1.5e-6, 4: 7e-4}))
    ftl, fll = nchw(tp["syn.ft4_low"], dev), nchw(tp["syn.fl4_low"], dev)
    dft, dfl = O.amt_update_block(sd, "amt_update4_high", ftl, fll, O.resize(corr_e, 2.0), None)
    rows.append(("10 syn.ft_4", maxdiff(tp["syn.ft_4"], nhwc(ftl + dft)), {"hostsim": 2e-6, 0: 2e-6, 4: 7e-4}))
    rows.append(("10 syn.fl4", maxdiff(tp["syn.fl4"], nhwc(fll + dfl)), {"hostsim": 2e-6, 0: 2e-6, 4: 7e-4}))
    check(run, rows)


def test_motion_route(run):
    """the benchmarked route ran (by the engine profiler's kernel names), and the inspected frame does not depend on the timestep order"""
    if run["kind"] != "gpu":
        pytest.skip("the profiler and the routes are the H100's")
    prof, B, T = run["prof"], run["B"], run["T"]
    n = lambda k: prof.get(k, {}).get("launches", 0)
    # (corr_lookup and the pooling kernels also serve the flow estimators' own correlations: counted, not excluded)
    if run["route"] == "direct":
        want, absent = {"corr_lookup_direct": 2 * T}, ("corr_gemm_tc_tf32",)
    elif run["mode"] == 4:   # the volume as plain-TF32 GEMMs, levels 1-3 against the 2^l average-pooled target features
        want, absent = {"corr_gemm_tc_tf32": 4 * 2 * B, "corr_lookup": 2 * T}, ("corr_lookup_direct",)
    else:                    # the fp32 volume and its pooled pyramid
        want, absent = {"corr_gemm_nt": 1, "corr_pool_pyramid": 1, "corr_lookup": 2 * T}, ("corr_lookup_direct",)
    print("\n%s mode %d (%s): %s" % (run["case"], run["mode"], run["route"], {k: n(k) for k in list(want) + list(absent)}))
    assert all(n(k) >= c for k, c in want.items()) and not any(n(k) for k in absent), sorted(prof)
    if run["bench"] is not None:
        # the inspected frame (t = 1/8 last) against bench.py's order (t = 1/8 first) differs no more than two identical forwards do
        b0, b1 = run["bench"]
        md = lambda a, b: (a.double() - b.double()).abs().max().item()
        d_order, d_rep = md(b0["imgt_pred"], run["out"]["img"]), md(b0["imgt_pred"], b1["imgt_pred"])
        print("%s: frame t = 1/8 last vs first: max |d| %.3e; two forwards in bench order: %.3e (their flows: %.3e px; the inspected "
              "forward's: %.3e px)" % (run["case"], d_order, d_rep, md(b0["raft_flow"], b1["raft_flow"]),
                                       md(b0["raft_flow"], run["out"]["raft_flow"])))
        assert d_order <= 2 * d_rep + 1e-5


def test_motion_composed(run):
    """float64 from the engine's splat outputs to the frame, against the engine's frame per pixel; and, reported only, the same chain
    from the engine's latents through a float64 splat (the splat's conditioning included)"""
    tp, dev, sd, B, t = run["taps"], run["dev"], run["sd64"], run["B"], run["t"]
    fup4 = O._decoder_upsample(sd, "amt_init_decoder.upsample", nchw(tp["syn.feat8"], dev), 1)
    fup1 = O._decoder_upsample(sd, "amt_final_decoder.upsample", nchw(tp["syn.feat4"], dev), 2)
    lat0, lat1 = nchw(tp["gimm.lat0"], dev), nchw(tp["gimm.lat1"], dev)
    img = run["out"]["img"].to(dev, torch.float64)
    pred = chain64(run, lat0, lat1, nchw(tp["gimm.splat0"], dev), nchw(tp["gimm.splat1"], dev), fup4, fup1)
    d = (img - pred).abs()
    flows = run["out"]["raft_flow"].to(dev, torch.float64)
    wts = nchw(tp["gimm.splat_w"], dev)
    sp0, _ = splat64(lat0, flows[:, :, 0] * t, wts[:B])
    sp1, _ = splat64(lat1, flows[:, :, 1] * (1.0 - t), wts[B:])
    d2 = (img - chain64(run, lat0, lat1, sp0, sp1, fup4, fup1)).abs()
    p = lambda x: x.flatten().topk(max(1, x.numel() // 10000)).values[-1].item()
    print("\n%s %s mode %d: frame from the engine's splat: max %.3e p99.99 %.3e; from its latents through a float64 splat: max %.3e "
          "p99.99 %.3e" % (run["case"], run["kind"], run["mode"], d.max().item(), p(d), d2.max().item(), p(d2)))
    # mode 4: BASELINE.json's per-pixel contract (measured 9.7e-5 small, 1.9e-4 small-T3, 3.2e-4 pair1080, 2.9e-4 f2k, 3.2e-4 f4k).
    # fp32: reassociation through the chain and the warps' sample position round trip (measured 9.2e-7 hostsim, 3.5e-6 pair1080,
    # 2.6e-6 f2k, 7.7e-6 f4k).  The chain from the latents through the float64 splat differs by up to 1.5e-2 at f2k in both modes: the
    # splat's conditioning, which the engine's fp32 shares with the reference's own
    check(run, [("splat -> imgt_pred", d.max().item(), {"hostsim": 2e-5, 0: 2e-5, 4: 1e-3})])
