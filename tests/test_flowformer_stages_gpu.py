"""GIMM-VFI-F's flow estimator (the native FlowFormer, csrc/flowformer.cu) stage by stage against float64: the encoders, the cost volume,
the cost perceiver layer by layer, the GMA attention rows, the first decoder iteration, every piece of the last one (lookup, motion
encoder, aggregation, GRU, flow head, mask, convex upsampling), and the full decoder depth composed in float64 from the engine's own
encoder outputs.

Each stage is fed the engine's own stored input (its debug taps, EngineHandle.tap), so that no upstream difference reaches its bar; the
reference is the oracle (oracle/flowformer_oracle.py) in float64 with the weights cast to double.  The long contractions are held per
entry to a bound of an fp32-class implementation's distance from float64, not to a flat bar: the cost volume (K = 256), the GMA logits
(K = 128), the aggregation attn @ v (K = N) and the GRU gates; test_bounds_reject_planted_errors shows that each bound rejects a small
planted error.

Cases (GIMM-VFI-F's own pair layout unless stated), each in precision modes 0 (fp32 CUDA cores) and 4 (the default: 3xF16 tensor cores):
  small   128x160, B = 2 pairs in both directions, 2 pairs per reference call (the vertical blocks read the call's contexts): 16 x 20 grid
  ragged  160x224: a 20 x 28 grid, N = 560 (N % 64 != 0: mode 4 aggregates through gemm_nn), cost maps padded to 24 x 32
  gather  256x320 through the pair list [(2, 0), (0, 1), (2, 1)]: out-of-order and repeated sources, the gathering path (32 x 40 grid)
  f2k     bench.py's f2k pair (2K, seed 100) at ds_factor 0.5: FlowFormer at 544x1024, a 68 x 128 grid, N = 8704 - the estimator size
          f4k shares: cost maps through the patch embedding in 6 chunks per volume, the shared-K/V attention kernels, a GMA softmax over
          rows of 8704, the tensor-core aggregation and corr_gemm_3xf16 past one raster group
The engine profile confirms each case's route.  Layouts: the engine stores NHWC and the latent tokens token-major [(pair, token)][h][w];
the oracle NCHW and (maps, 8, 128).

Measured on an H100 80GB HBM3 (700 W), over the four cases and both modes (max |d| / bound for the bounded stages): cost volume
0.054 - 0.070; GMA rows 5.6e-4 - 2.2e-3 (row sums within 2.0e-7 of att_mul); lookup 0.14 - 0.19 at iteration 0 and 0.18 - 0.32 at the
last; aggregation 8.4e-3 - 0.038; GRU 0.011 - 0.036.  Flat-bar stages: encoders <= 7.3e-6, cost perceiver layers <= 3.2e-6, the 64
global channels <= 5.8e-5, motion features <= 3.6e-5, flow head <= 7.6e-6 px, convex upsampling <= 8.7e-6 px; composed, flow_low
1.2e-5 (small) - 6.9e-5 px (f2k), flow_up 2.8e-5 - 2.3e-4 px.  The whole file (8 engine runs and every float64 restatement) takes
~40 s there."""
import gc
import math
import time

import pytest
import torch
import torch.nn.functional as F

import flowformer_oracle as FO
import gimmvfi_r_oracle as O
from corr_ref import U
from gimmvfi_b200.synth import synth_batch

ITERS = 32
P = FO.P
ME, MD = P + "memory_encoder", P + "memory_decoder"
CP, UB = ME + ".cost_perceiver_encoder", MD + ".update_block"
# name: H, W, frames ("pairs": B pairs of synth_batch as [I0 ; I1]; "three": 3 frames), pairs, pairs per call, seed, ds_factor
CASES = {
    "small": (128, 160, "pairs", [(0, 2), (1, 3), (2, 0), (3, 1)], 2, 41, None),
    "ragged": (160, 224, "pairs", [(0, 1), (1, 0)], 1, 43, None),
    "gather": (256, 320, "three", [(2, 0), (0, 1), (2, 1)], 1, 47, None),
    "f2k": (1088, 2048, "pairs", [(0, 1), (1, 0)], 1, 100, 0.5),
}
RUNS = [pytest.param((c, m), id="%s-h100-mode%d" % (c, m), marks=pytest.mark.gpu) for c in CASES for m in (0, 4)]
TAPS = ["ff.feat4", "ff.feat8", "ff.fproj", "ff.cost_volume", "ff.latent_in", "ff.latent_0", "ff.latent_1", "ff.latent_2", "ff.cost_memory",
        "ff.cnet", "ff.gma_attn", "ff.dec_corr_0", "ff.dec_net_0", "ff.coords_last", "ff.net_last", "ff.corr_last", "ff.motion_last",
        "ff.mg_last", "ff.net_final", "ff.mask", "ff.lowres_flow"]
DEV = "cuda"


def nchw(t):
    return t.permute(0, 3, 1, 2).to(DEV, torch.float64)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def tokens(t, S, h, w):
    """engine latent maps (S*8, h, w, 128) token-major -> the oracle's (S*h*w, 8, 128)"""
    return t.to(DEV, torch.float64).reshape(S, 8, h * w, -1).permute(0, 2, 1, 3).reshape(S * h * w, 8, -1)


@pytest.fixture(autouse=True)
def _no_grad():
    with torch.no_grad():
        yield


def frames_of(case):
    H, W, kind, pairs, per_call, seed, ds = CASES[case]
    if kind == "three":
        xs = synth_batch(2, H, W, seed=seed)
        return 255 * torch.stack([xs[0, :, 0], xs[0, :, 1], xs[1, :, 1]], 0)
    B = len(pairs) // 2
    xs = synth_batch(B, H, W, seed=seed).double()
    if ds:
        xs = torch.stack([O.resize(xs[:, :, 0], ds), O.resize(xs[:, :, 1], ds)], 2)
    return (255 * torch.cat([xs[:, :, 0], xs[:, :, 1]], 0)).float()


@pytest.fixture(scope="module", params=RUNS)
def run(request):
    """one forward with the debug taps and the profiler, one with both off; then the engine is freed"""
    case, mode = request.param
    H, W, kind, pairs, per_call, seed, ds = CASES[case]
    from gimmvfi_b200.engine import EngineHandle
    from gimmvfi_b200.weights import random_state_dict_f

    sd = random_state_dict_f(0)
    eng = EngineHandle(DEV)
    eng.load_state_dict(sd, full_f=True)
    eng.set_tensor_cores(mode)
    frames = frames_of(case).to(DEV).contiguous()
    t0 = time.time()
    eng.set_debug(True)
    eng.set_profile(True)
    up, low = eng.flowformer_forward(frames, pairs, pairs_per_call=per_call, iters=ITERS, flow_low=True)
    torch.cuda.synchronize()
    prof = eng.profile()
    eng.set_profile(False)
    launches_dbg = eng.last_launches
    taps = {k: eng.tap(k).clone() for k in TAPS}
    up, low = up.clone(), low.clone()
    eng.set_debug(False)
    up0, low0 = eng.flowformer_forward(frames, pairs, pairs_per_call=per_call, iters=ITERS, flow_low=True)
    torch.cuda.synchronize()
    bitwise = dict(up=torch.equal(up0, up), low=torch.equal(low0, low), launches=(launches_dbg, eng.last_launches))
    engine_s = time.time() - t0
    del eng, up0, low0
    gc.collect()
    torch.cuda.empty_cache()
    sd64 = {k: (v.to(DEV, torch.float64) if v.is_floating_point() else v) for k, v in sd.items()}
    S, h, w = len(pairs), frames.shape[-2] // 8, frames.shape[-1] // 8
    src, tgt = [a for a, _ in pairs], [b for _, b in pairs]
    srcs = list(dict.fromkeys(src))                                                  # distinct sources in first-use order
    img64 = 2 * (frames.double() / 255.0) - 1.0                                      # transformer.py:49-50
    ctx = nchw(taps["ff.feat8"])[[srcs.index(s) for s in src]]                      # each pair's context (the engine's feat8)
    yield dict(case=case, mode=mode, taps=taps, up=up, low=low, sd=sd64, img=img64, S=S, h=h, w=w, N=h * w, src=src, tgt=tgt, srcs=srcs,
               per_call=per_call, ctx=ctx, grid=FO.coords_grid(S, h, w, img64), prof=prof, bitwise=bitwise, engine_s=engine_s,
               att_mul=2.0 ** min(15, math.ceil(math.log2(h * w))))
    del taps, sd64
    gc.collect()
    torch.cuda.empty_cache()


def maxdiff(got, ref):
    assert got.shape == ref.shape, (tuple(got.shape), tuple(ref.shape))
    return (got.to(ref.device, torch.float64) - ref).abs().max().item()


def ratio(got, ref, bnd):
    assert got.shape == ref.shape, (tuple(got.shape), tuple(ref.shape))
    d = (got.to(ref.device, torch.float64) - ref).abs()
    return torch.where(d == 0, torch.zeros_like(d), d / bnd).max().item()


def rel(ref, k=2.0 ** -13):
    return k * max(1.0, ref.abs().max().item())


def check(run, rows):
    lines, bad = [], []
    for stage, err, bar in rows:
        lines.append("%-56s %.3e (bar %.1e)" % (stage, err, bar))
        if not err <= bar:
            bad.append(stage)
    print("\n%s mode %d (%dx%d grid, S = %d)\n  " % (run["case"], run["mode"], run["h"], run["w"], run["S"]) + "\n  ".join(lines))
    assert not bad, "stages over their bar: %s\n%s" % (bad, "\n".join(lines))


# ---------------------------------------------------------------------------------------------------------------------------- bounds
# An fp32-class K-term dot product (recursive summation, the 3xF16 split's 2^-22 per operand and dropped lo x lo term, blocked or
# tensor-core accumulation only shortening the chains) lies within (K + 16) u sum_k |a_k b_k| of the float64 value: corr_ref.GAMMA_DOT.
def dot_bound(K):
    return (K + 16) * U


def volume64(fs, ft, rows=4096):
    """vol[i][j] = <fs_i, ft_j> (encoder.py:507-522, no scale) and its per-entry bound, in row chunks: fs / ft (N, 256)"""
    for p0 in range(0, fs.shape[0], rows):
        a = fs[p0:p0 + rows]
        yield p0, a @ ft.t(), dot_bound(fs.shape[1]) * (a.abs() @ ft.abs().t())


def softmax_bound(prob, dl, N):
    """per-entry bound of an fp32 row softmax's distance from float64 given per-logit errors dl (first order: dp_j = p_j (dl_j - sum_i p_i
    dl_i), so |dp_j| <= p_j (dl_j + max_i dl_i)), plus its own rounding: expf (2 ulp), the max subtraction, and the fp32 row sum of N
    terms (N u, recursive summation) and the division"""
    return prob * (dl + dl.amax(-1, keepdim=True) + (N + 16) * U)


def logits_bound(sd, inp):
    """the GMA logits l = q k^T / sqrt(128), q | k = to_qk(inp) (a 1x1 convolution, K = 128), and each logit's error bound: the K = 128
    product of the engine's q and k, and the q / k errors of the fp32-class convolution carried through it.  inp (S, 128, h, w) ->
    (q, k (S, N, 128), the bound (S, N, N))"""
    wq = sd[MD + ".att.to_qk.weight"]                                               # (no bias)
    qk = F.conv2d(inp, wq).flatten(2).transpose(1, 2)
    eqk = dot_bound(128) * (F.conv2d(inp.abs(), wq.abs()).flatten(2).transpose(1, 2))
    q, k, eq, ek = qk[..., :128], qk[..., 128:], eqk[..., :128], eqk[..., 128:]
    s = 128 ** -0.5
    return q, k, s * (dot_bound(128) * (q.abs() @ k.abs().transpose(1, 2)) + eq @ k.abs().transpose(1, 2) + q.abs() @ ek.transpose(1, 2))


def aggregate_bound(sd, mf, att):
    """Aggregate (gma.py:84-115) in float64 and the per-entry bound: v = to_v(mf) (K = 128) carries dot_bound(128) |W| |mf|; attn @ v
    (K = N) dot_bound(N) sum_j |a_ij| |v_j| plus sum_j |a_ij| |dv_j|; times |gamma|, plus the fp32 roundings of the axpy.  mf (S,128,h,w),
    att (S, N, N) -> (mg, bound)"""
    wv = sd[UB + ".aggregator.to_v.weight"]
    S, c, h, w = mf.shape
    v = F.conv2d(mf, wv).flatten(2).transpose(1, 2)
    ev = dot_bound(128) * F.conv2d(mf.abs(), wv.abs()).flatten(2).transpose(1, 2)
    g = sd[UB + ".aggregator.gamma"]
    av = att @ v
    e = dot_bound(att.shape[-1]) * (att.abs() @ v.abs()) + att.abs() @ ev
    shape = lambda t: t.transpose(1, 2).reshape(S, c, h, w)
    mg = mf + g * shape(av)
    return mg, g.abs() * shape(e) + 2 * U * (mf.abs() + (g * shape(av)).abs())


# The GRU's gates: convolutions over [h | inp | mf | mg], K = 512 x 5 = 2560.  As in test_raft_stages_gpu.py: with independent roundings
# the error of K partial sums has sigma ~ u sqrt(K / 6) |t|_2, plus the 3xF16 split's 12 u |t|_2; the bound takes 8 x the larger sigma
# sqrt(K / 3).  (The K u sum |t| worst case would let a 1e-4 mistake in the state through.)
GAMMA_GRU = 8.0 * (math.sqrt(2560 / 3) + 12) * U


def gru_bound64(sd, net, x):
    """SepConvGRU (gru.py:35-73) in float64 from the engine's own input and the per-entry bound, propagated to first order through both
    halves (sigmoid' <= 1/4, tanh' <= 1, 8 u per activation, one rounding of r h, four of the blend) - test_raft_stages_gpu.gru_bound64"""
    g = UB + ".gru"
    h, eh = net, torch.zeros_like(net)
    zx = torch.zeros_like(x)
    for sfx, pad in (("1", (0, 2)), ("2", (2, 0))):
        wb = lambda n: (sd[g + n + sfx + ".weight"], sd[g + n + sfx + ".bias"])
        conv = lambda n, t: F.conv2d(t, *wb(n), padding=pad)
        rms = lambda n, t: F.conv2d(t * t, wb(n)[0] ** 2, wb(n)[1] ** 2, padding=pad).sqrt()
        prop = lambda n, e: F.conv2d(e, wb(n)[0].abs(), padding=pad)
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


def lookup_bound64(maps, coords):
    """encode_flow_token (decoder.py:233-252) of the engine's own cost maps (maps (M, 1, h, w) float64) at coords (M / (h w), 2, h, w),
    and the per-entry bound of an fp32 lookup's distance from it: the coordinate rounding of bilinear_sampler's normalise / un-normalise
    round trip, u (6 |c| + S) along an axis of S pixels (corr_ref.corr_lookup64), times the largest slope of the interpolant near the
    sample, plus 8 u of the largest |value| there (the bilinear weights' products and the four-tap blend).  "Near": the differences of
    neighbouring values (zero outside the frame) max-pooled over 5 x 5, then sampled bilinearly - at least the largest of the 3 x 3
    cells around the sample"""
    h, w = maps.shape[-2:]
    ref = FO.encode_flow_token(maps, coords)
    pm = F.pad(maps, (2, 2, 2, 2))
    dx, dy = F.pad(pm.diff(dim=-1).abs(), (0, 1)), F.pad(pm.diff(dim=-2).abs(), (0, 0, 0, 1))
    pool = lambda t: F.max_pool2d(t, 5, stride=1, padding=2)
    slope, val = pool(torch.maximum(dx, dy)), pool(pm.abs())
    del pm, dx, dy
    b, _, hh, ww = coords.shape
    d = torch.linspace(-4, 4, 9, dtype=coords.dtype, device=coords.device)
    delta = torch.stack(torch.meshgrid(d, d, indexing="ij"), -1).view(1, 9, 9, 2)
    pc = coords.permute(0, 2, 3, 1).reshape(-1, 1, 1, 2) + delta                    # (x + dy[i], y + dx[j]): the transposed window
    e = U * (6 * pc[..., :1].abs() + w) + U * (6 * pc[..., 1:].abs() + h)
    shape = lambda t: t.reshape(b, hh, ww, -1).permute(0, 3, 1, 2)
    samp = lambda m: shape(FO.bilinear_sampler(m, pc + 2))
    return ref, shape(e) * samp(slope) + 8 * U * samp(val)


def patch_and_input_layer64(sd, maps, chunk=2048):
    """cost_patch_embed + the input layer in float64 over cost maps (M, 1, h, w), in chunks of maps -> (M, 8, 128)"""
    return torch.cat([FO.cost_input_layer(sd, CP, FO.cost_patch_embed(sd, CP + ".patch_embed", maps[m:m + chunk])[0])
                      for m in range(0, maps.shape[0], chunk)], 0)


def maps_of(run, s):
    """pair s's cost maps from the engine's volume: (N, 1, h, w) float64"""
    return run["taps"]["ff.cost_volume"][s].to(DEV, torch.float64).reshape(run["N"], 1, run["h"], run["w"])


def layer_by_call(run, i, x):
    """cost_perceiver_layer i over each reference call's pairs (the vertical blocks repeat that call's contexts)"""
    S, h, w, pc = run["S"], run["h"], run["w"], run["per_call"]
    n = h * w
    return torch.cat([FO.cost_perceiver_layer(run["sd"], CP, i, x[c * n:(c + pc) * n], (h, w), run["ctx"][c:c + pc])
                      for c in range(0, S, pc)], 0)


# ---------------------------------------------------------------------------------------------------------------------------- tests
def test_bounds_reject_planted_errors():
    """each per-entry bound holds for an fp32 evaluation of the same inputs and rejects a small planted error: the cost volume (K = 256)
    a 1xF16 product (the lo planes dropped); the GMA rows logits moved by 1e-3; the aggregation sample 0's attention for sample 1's; the
    GRU a state moved by 1e-4; the lookup coordinates moved by 1e-3 px"""
    g = torch.Generator().manual_seed(5)
    R = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    from gimmvfi_b200.weights import random_state_dict_f
    sd = {k: (v.double() if v.is_floating_point() else v) for k, v in random_state_dict_f(0).items()}
    res = {}
    # cost volume
    fs, ft = R(300, 256), R(280, 256)
    _, ref, bnd = next(volume64(fs, ft))
    res["volume fp32"] = ratio(fs.float() @ ft.float().t(), ref, bnd)
    res["volume 1xF16"] = ratio(fs.half().double() @ ft.half().double().t(), ref, bnd)
    # GMA rows
    inp = torch.relu(R(2, 128, 8, 12))
    q, k, dl = logits_bound(sd, inp)
    lg = q @ k.transpose(1, 2) * 128 ** -0.5
    pr = torch.softmax(lg, -1)
    pb = softmax_bound(pr, dl, lg.shape[-1])
    qk32 = F.conv2d(inp.float(), sd[MD + ".att.to_qk.weight"].float()).flatten(2).transpose(1, 2)
    res["GMA rows fp32"] = ratio(torch.softmax(qk32[..., :128] @ qk32[..., 128:].transpose(1, 2) * 128 ** -0.5, -1), pr, pb)
    res["GMA rows, logits + 1e-3"] = ratio(torch.softmax(lg + 1e-3 * R(*lg.shape).sign(), -1), pr, pb)
    # aggregation
    mf = torch.relu(R(2, 128, 8, 12))
    mg, mb = aggregate_bound(sd, mf, pr)
    wv = sd[UB + ".aggregator.to_v.weight"].float()
    agg32 = lambda a: mf.float() + sd[UB + ".aggregator.gamma"].float() * (a.float() @ F.conv2d(mf.float(), wv).flatten(2).transpose(1, 2)
                                                                          ).transpose(1, 2).reshape(mf.shape)
    res["aggregate fp32"] = ratio(agg32(pr), mg, mb)
    res["aggregate, sample 0's attention"] = ratio(agg32(pr[[0, 0]]), mg, mb)
    # GRU
    net, x = torch.tanh(R(2, 128, 8, 12)), torch.relu(R(2, 384, 8, 12))
    hG, eG = gru_bound64(sd, net, x)
    sd32 = {k: v.float() for k, v in sd.items() if k.startswith(UB + ".gru")}
    res["GRU fp32"] = ratio(FO.sep_conv_gru(sd32, UB, net.float(), x.float()), hG, eG)
    res["GRU, state + 1e-4"] = ratio(FO.sep_conv_gru(sd32, UB, net.float() + 1e-4, x.float()), hG, eG)
    # lookup
    maps = 30 * R(2 * 10 * 14, 1, 10, 14)
    co = (FO.coords_grid(2, 10, 14, maps) + 6 * R(2, 2, 10, 14)).float().double()
    ref, lb = lookup_bound64(maps, co)
    res["lookup fp32"] = ratio(FO.encode_flow_token(maps.float(), co.float()), ref, lb)
    res["lookup, coordinates + 1e-3 px"] = ratio(FO.encode_flow_token(maps.float(), co.float() + 1e-3), ref, lb)
    print("\n" + "\n".join("%-40s max |d| / bound %.3f" % kv for kv in res.items()))
    for name, r in res.items():
        assert (r <= 1.0) == ("fp32" in name), name


def test_flowformer_stages(run):
    """Each stage from the engine's stored inputs against float64 (see the module docstring); measured ratios and differences are in
    DESIGN.md (FlowFormer stage by stage)"""
    tp, sd, S, h, w, N = run["taps"], run["sd"], run["S"], run["h"], run["w"], run["N"]
    img, grid, src, tgt = run["img"], run["grid"], run["src"], run["tgt"]
    rows = []
    # 1. encoders.  Twins-SVT: LayerNorm'd tokens through 4 blocks a stage, linears with K <= 1024, fp32-class in both modes: 2^-13 of
    #    the largest value
    c4, c8 = FO.twins_svt(sd, P + "context_encoder", img[run["srcs"]])
    rows += [("1 ff.feat4", maxdiff(tp["ff.feat4"], nhwc(c4)), rel(c4)), ("1 ff.feat8", maxdiff(tp["ff.feat8"], nhwc(c8)), rel(c8))]
    fp = torch.cat([F.conv2d(FO.twins_svt(sd, ME + ".feat_encoder", img[f:f + 1])[1], sd[ME + ".channel_convertor.weight"])
                    for f in range(img.shape[0])], 0)
    rows.append(("1 ff.fproj", maxdiff(tp["ff.fproj"], nhwc(fp)), rel(fp)))
    del c4, c8, fp

    # 2. cost volume from the engine's fproj, every row, per entry within dot_bound(256)
    fpj = tp["ff.fproj"].to(DEV, torch.float64).reshape(-1, N, 256)
    worst = 0.0
    for s in range(S):
        vol = tp["ff.cost_volume"][s].reshape(N, N)
        for p0, ref, bnd in volume64(fpj[src[s]], fpj[tgt[s]]):
            worst = max(worst, ratio(vol[p0:p0 + ref.shape[0]], ref, bnd))
    rows.append(("2 ff.cost_volume max |d| / bound", worst, 1.0))

    # 3. cost perceiver: the patch embedding + input layer from the engine's volume (6x6 convolutions, K <= 1152, then LayerNorm),
    #    each layer from the engine's previous one, the residual sum exactly
    lat_in = torch.cat([patch_and_input_layer64(sd, maps_of(run, s)) for s in range(S)], 0)
    rows.append(("3 ff.latent_in", maxdiff(tokens(tp["ff.latent_in"], S, h, w), lat_in), rel(lat_in)))
    del lat_in
    prev = tokens(tp["ff.latent_in"], S, h, w)
    for i in range(3):
        ref = layer_by_call(run, i, prev)
        rows.append(("3 ff.latent_%d" % i, maxdiff(tokens(tp["ff.latent_%d" % i], S, h, w), ref), rel(ref)))
        prev = tokens(tp["ff.latent_%d" % i], S, h, w)
    mem = prev + tokens(tp["ff.latent_in"], S, h, w)
    rows.append(("3 ff.cost_memory (latent_2 + latent_in)", maxdiff(tokens(tp["ff.cost_memory"], S, h, w), mem), 2 * U * mem.abs().max().item()))

    # 4. GMA attention rows from the engine's cnet: per entry within softmax_bound of the logits' bound; each row sums to att_mul
    cn = nchw(tp["ff.cnet"])
    worst, sums = 0.0, 0.0
    for s in range(S):
        q, k, dl = logits_bound(sd, cn[s:s + 1, 128:])
        lg = q @ k.transpose(1, 2) * 128 ** -0.5
        del q, k
        pr = torch.softmax(lg, -1)
        del lg
        got = tp["ff.gma_attn"][s].reshape(1, N, N)
        worst = max(worst, ratio(got / run["att_mul"], pr, softmax_bound(pr, dl, N)))
        sums = max(sums, (got.double().sum(-1) / run["att_mul"] - 1).abs().max().item())
        del pr, dl
    rows += [("4 ff.gma_attn / att_mul max |d| / bound", worst, 1.0), ("4 rows sum to att_mul (|sum / att_mul - 1|)", sums, (N + 16) * U)]

    # 5. decoder iteration 0: the windowed channels are the lookup at the integer grid, per entry within lookup_bound64 (the fp32
    #    normalise / un-normalise round trip moves an integer coordinate off the grid by up to u (6 |c| + S)); the 64 global channels
    #    from the engine's cost memory (flow-token encoder, cross attention, ffn: fp32-class, 2^-13); the GRU state after iteration 0
    key, value = FO._lin(sd, MD + ".decoder_layer.cross_attend.k", mem), FO._lin(sd, MD + ".decoder_layer.cross_attend.v", mem)
    d0 = nchw(tp["ff.dec_corr_0"])
    worst = 0.0
    for s in range(S):
        ref, bnd = lookup_bound64(maps_of(run, s), grid[s:s + 1])
        worst = max(worst, ratio(d0[s:s + 1, 64:], ref, bnd))
        del ref, bnd
    rows.append(("5 it 0: dec_corr_0 windowed (81) max |d| / bound", worst, 1.0))
    cg0 = FO.cost_global(sd, d0[:, 64:], grid, key, value)
    rows.append(("5 it 0: dec_corr_0 global (64)", maxdiff(nhwc(d0[:, :64]), nhwc(cg0)), rel(cg0)))
    att = torch.cat([tp["ff.gma_attn"][s].to(DEV, torch.float64).reshape(1, 1, N, N) for s in range(S)], 0) / run["att_mul"]
    n0, _, _ = FO.gma_update_block(sd, UB, cn[:, :128], cn[:, 128:], d0, torch.zeros_like(grid), att, False)
    rows.append(("5 it 0: ff.dec_net_0", maxdiff(tp["ff.dec_net_0"], nhwc(n0)), 1e-4))
    del d0, cg0, n0

    # 6. the last iteration, each piece from the engine's own input
    cl = nchw(tp["ff.coords_last"])
    worst = 0.0
    for s in range(S):
        ref, bnd = lookup_bound64(maps_of(run, s), cl[s:s + 1])
        worst = max(worst, ratio(nchw(tp["ff.corr_last"][s:s + 1, :, :, 64:]), ref, bnd))
        del ref, bnd
    rows.append(("6 last: lookup at coords_last max |d| / bound", worst, 1.0))
    outside = int(((cl[:, 0] < 0) | (cl[:, 0] > w - 1) | (cl[:, 1] < 0) | (cl[:, 1] > h - 1)).sum().item())
    print("\n%s: last-iteration window centres outside the frame: %d of %d" % (run["case"], outside, S * N))
    assert outside > 0, "no last-iteration window centre lies outside the frame"
    fl = cl - grid
    mot = FO.motion_encoder(sd, UB, nchw(tp["ff.corr_last"]), fl)
    rows.append(("6 last: ff.motion_last", maxdiff(tp["ff.motion_last"], nhwc(mot)), 2.0 ** -17 * max(1.0, mot.abs().max().item())))
    mg, mb = aggregate_bound(sd, nchw(tp["ff.motion_last"]), att[:, 0])
    rows.append(("6 last: ff.mg_last (aggregation) max |d| / bound", ratio(nchw(tp["ff.mg_last"]), mg, mb), 1.0))
    del att
    x = torch.cat([cn[:, 128:], nchw(tp["ff.motion_last"]), nchw(tp["ff.mg_last"])], 1)
    hG, eG = gru_bound64(sd, nchw(tp["ff.net_last"]), x)
    rows.append(("6 last: ff.net_final (GRU) max |d| / bound", ratio(nchw(tp["ff.net_final"]), hG, eG), 1.0))
    nf = nchw(tp["ff.net_final"])
    dfl = FO.flow_head(sd, UB, nf)
    upd = nchw(tp["ff.lowres_flow"]) + grid - cl
    coord_round = 2 * U * (cl.abs().max().item() + max(h, w))
    rows.append(("6 last: flow head (lowres_flow - coords_last)", maxdiff(nhwc(upd), nhwc(dfl)), 1e-5 + coord_round))
    mk = FO.mask_head(sd, UB, nf)
    rows.append(("6 last: ff.mask", maxdiff(tp["ff.mask"], nhwc(mk)), 2.0 ** -17 * max(1.0, mk.abs().max().item())))
    low = nchw(tp["ff.lowres_flow"])
    up = FO.upsample_flow(low, nchw(tp["ff.mask"]))
    rows.append(("6 convex upsampling (every pixel)", maxdiff(run["up"], up), 1e-6 + 16 * U * 8 * low.abs().max().item()))
    rows.append(("6 flow_low output = ff.lowres_flow", maxdiff(run["low"], low), 0.0))
    check(run, rows)


def test_flowformer_composed(run):
    """the memory encoder and all 32 decoder iterations in float64 from the engine's context (feat8) and fproj, against the engine's
    flows at every pixel: flow_low to test_flowformer_gpu.py's bars (2e-4 px in mode 0, 2e-3 px in mode 4), flow_up to 8 times those
    (convex upsampling takes a convex combination of 8 flow_low: a flow_low error e reaches flow_up as up to 8 e)"""
    tp, sd, S, h, w, N = run["taps"], run["sd"], run["S"], run["h"], run["w"], run["N"]
    fpj = nchw(tp["ff.fproj"])
    ctx, grid = run["ctx"], run["grid"]
    mem, maps = [], []
    for c in range(0, S, run["per_call"]):
        ps = range(c, c + run["per_call"])
        vol = torch.stack([torch.einsum("id,jd->ij", fpj[run["src"][s]].flatten(1).t(), fpj[run["tgt"][s]].flatten(1).t()) for s in ps], 0)
        m = vol.reshape(-1, 1, h, w)
        del vol
        x = patch_and_input_layer64(sd, m)
        sc = x
        for i in range(3):
            x = FO.cost_perceiver_layer(sd, CP, i, x, (h, w), ctx[c:c + run["per_call"]])
        mem.append(x + sc)
        maps.append(m)
    mem, maps = torch.cat(mem, 0), torch.cat(maps, 0)
    cproj = FO._conv(sd, MD + ".proj", ctx)
    net, inp = torch.tanh(cproj[:, :128]), torch.relu(cproj[:, 128:])
    att = FO.gma_attention(sd, inp)
    key, value = FO._lin(sd, MD + ".decoder_layer.cross_attend.k", mem), FO._lin(sd, MD + ".decoder_layer.cross_attend.v", mem)
    coords = grid.clone()
    for it in range(ITERS):
        net, dflow, mask, _ = FO.decoder_iteration(sd, net, inp, grid, coords, maps, key, value, att, it == ITERS - 1)
        coords = coords + dflow
    low = coords - grid
    up = FO.upsample_flow(low, mask)
    bar = 2e-4 if run["mode"] == 0 else 2e-3
    check(run, [("7 composed: flow_low (every pixel)", maxdiff(run["low"], low), bar),
                ("7 composed: flow_up (every pixel)", maxdiff(run["up"], up), 8 * bar)])


def test_flowformer_route_and_taps(run):
    """the route each case claims, by the engine profiler's kernel names; the taps do not change the flows (bit for bit), and add only
    their 11 snapshot copies to the launches (ff.cnet, latent_0..2, dec_corr_0, dec_net_0 and the five *_last)"""
    prof, mode, S, N, case = run["prof"], run["mode"], run["S"], run["N"], run["case"]
    n = lambda k: prof.get(k, {}).get("launches", 0)
    h, w = run["h"], run["w"]
    oh1, ow1 = (h + 7) // 8 * 4, (w + 7) // 8 * 4
    oh2, ow2, oh3, ow3 = oh1 // 2, ow1 // 2, oh1 // 4, ow1 // 4
    per_map = ((oh1 + 4) * (ow1 + 4) * 16 + oh2 * ow2 * 32 + (oh2 + 4) * (ow2 + 4) * 32 + oh3 * ow3 * 128 * 5) * 4
    chunks = -(-N // min(N, max(1, (1 << 30) // per_map)))
    names = ("cost_conv1_6x6s2", "attention_shared_kv_d32", "attention_shared_kv_d16", "row_softmax", "corr_gemm_tc_3xf16", "gemm_nn_simt")
    print("\n%s mode %d: %d cost-map chunks per volume; %s; taps on / off: flows equal %s / %s, launches %s; engine %.1f s"
          % (case, mode, chunks, {k: n(k) for k in names}, run["bitwise"]["up"], run["bitwise"]["low"], run["bitwise"]["launches"],
             run["engine_s"]))
    assert run["bitwise"]["up"] and run["bitwise"]["low"]
    assert run["bitwise"]["launches"][0] - run["bitwise"]["launches"][1] == 11
    assert n("cost_conv1_6x6s2") == S * chunks
    if case == "f2k":
        assert chunks == 6 and n("attention_shared_kv_d32") > 0 and n("attention_shared_kv_d16") > 0
    agg_tc = mode == 4 and N % 64 == 0
    assert n("corr_gemm_tc_3xf16") == (2 * S + (S * ITERS if agg_tc else 0) if mode == 4 else 0), sorted(prof)
    assert n("gemm_nn_simt") == (0 if agg_tc else S * ITERS), sorted(prof)
