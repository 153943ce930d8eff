"""TEST INFRASTRUCTURE — CPU oracle for the GIMM-VFI-R per-pair interpolation path.

A plain-PyTorch fp32, functional restatement of ``GIMMVFI_R.forward``
(reference: src/models/generalizable_INR/gimmvfi_r.py:324-407) that works
directly on a flat ``state_dict`` (the reference's 414-key checkpoint layout).
It exists so that parity tests, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` have a checker
that travels to the GPU box, where /root/reference does not exist.

It is NOT product code: nothing under ``gimm-vfi_b200/`` imports it, and the
product path never falls back to it.

Pinning: the reference ships no tests / golden vectors (SURVEY.md §4), so this
restatement is pinned against the reference's own modules imported unmodified
in the build container (oracle/ref_shim.py) — see oracle/make_golden.py and
tests/test_oracle.py (max |Δ imgt_pred| vs the reference ≤ 2e-6 on every golden
case; the golden fixtures themselves are outputs of the *reference*).

Every function cites the reference file:line it follows (paths relative to
src/models/generalizable_INR/).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
SD = Dict[str, Tensor]


# --------------------------------------------------------------------------
# small helpers
# --------------------------------------------------------------------------
def _conv(sd: SD, name: str, x: Tensor, stride=1, padding=0, reflect=False) -> Tensor:
    w = sd[name + ".weight"]
    b = sd.get(name + ".bias")
    if reflect:
        ph, pw = (padding, padding) if isinstance(padding, int) else padding
        x = F.pad(x, (pw, pw, ph, ph), mode="reflect")
        padding = 0
    return F.conv2d(x, w, b, stride=stride, padding=padding)


def _bn_eval(sd: SD, name: str, x: Tensor, eps=1e-5) -> Tensor:
    """nn.BatchNorm2d in eval mode (running statistics)."""
    return F.batch_norm(
        x,
        sd[name + ".running_mean"],
        sd[name + ".running_var"],
        sd[name + ".weight"],
        sd[name + ".bias"],
        training=False,
        eps=eps,
    )


def _prelu(sd: SD, name: str, x: Tensor) -> Tensor:
    return F.prelu(x, sd[name + ".weight"])


def resize(x: Tensor, scale: float) -> Tensor:
    """modules/fi_utils.py:67-70 — bilinear, half-pixel centres."""
    return F.interpolate(x, scale_factor=scale, mode="bilinear", align_corners=False)


def backwarp(src: Tensor, flow: Tensor) -> Tensor:
    """modules/fi_utils.py:19-49 — sample ``src`` at (x+fx, y+fy), bilinear,
    border clamp, align_corners=True.  The base grid has the FLOW's size
    (linspace(-1,1,W_flow)); the flow is normalised by the SOURCE's size.
    The grid is built on the flow's device, in its dtype (float64 restatements)."""
    B, _, H, W = flow.shape
    kw = dict(device=flow.device, dtype=flow.dtype)
    gx = torch.linspace(-1.0, 1.0, W, **kw).view(1, 1, 1, W).expand(B, -1, H, -1)
    gy = torch.linspace(-1.0, 1.0, H, **kw).view(1, 1, H, 1).expand(B, -1, -1, W)
    base = torch.cat([gx, gy], 1)
    nf = torch.cat(
        [
            flow[:, 0:1] / ((src.shape[3] - 1.0) / 2.0),
            flow[:, 1:2] / ((src.shape[2] - 1.0) / 2.0),
        ],
        1,
    )
    g = (base + nf).permute(0, 2, 3, 1)
    return F.grid_sample(src, g, mode="bilinear", padding_mode="border", align_corners=True)


def coords_grid(B: int, h: int, w: int, like: Optional[Tensor] = None) -> Tensor:
    """raft/utils/utils.py:82-87 — (B,2,h,w), channel 0 = x, 1 = y.  With `like`: on its device, in its dtype (else fp32 on the CPU)."""
    dev = like.device if like is not None else None
    ys, xs = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
    return torch.stack([xs, ys], 0).to(like.dtype if like is not None else torch.float32)[None].repeat(B, 1, 1, 1)


# --------------------------------------------------------------------------
# RAFT  (raft/raft.py:99-169)
# --------------------------------------------------------------------------
def _norm(sd: SD, name: str, x: Tensor, kind: str) -> Tensor:
    if kind == "instance":  # nn.InstanceNorm2d(planes): no affine, no running stats
        return F.instance_norm(x, eps=1e-5)
    return _bn_eval(sd, name, x)


def _residual_block(sd: SD, p: str, x: Tensor, kind: str, stride: int) -> Tensor:
    """raft/extractor.py:6-58"""
    y = F.relu(_norm(sd, p + ".norm1", _conv(sd, p + ".conv1", x, stride=stride, padding=1), kind))
    y = F.relu(_norm(sd, p + ".norm2", _conv(sd, p + ".conv2", y, padding=1), kind))
    if stride != 1:
        # downsample = Sequential(conv1x1 stride, norm3): keys downsample.0 / downsample.1
        # (norm3 is the same module object as downsample.1, so both key sets exist).
        x = _norm(sd, p + ".downsample.1", _conv(sd, p + ".downsample.0", x, stride=stride), kind)
    return F.relu(x + y)


def basic_encoder(sd: SD, p: str, x: Tensor, kind: str):
    """raft/extractor.py:173-220 (the unused x_2/x_4 bilinear downsamples at
    :182-183 have no effect on the outputs and are omitted)."""
    feats = []
    x = F.relu(_norm(sd, p + ".norm1", _conv(sd, p + ".conv1", x, stride=2, padding=3), kind))
    x = _residual_block(sd, p + ".layer1.0", x, kind, 1)
    x = _residual_block(sd, p + ".layer1.1", x, kind, 1)
    feats.append(x)
    x = _residual_block(sd, p + ".layer2.0", x, kind, 2)
    x = _residual_block(sd, p + ".layer2.1", x, kind, 1)
    feats.append(x)
    x = _residual_block(sd, p + ".layer3.0", x, kind, 2)
    x = _residual_block(sd, p + ".layer3.1", x, kind, 1)
    feats.append(x)
    x = _conv(sd, p + ".conv2", x)
    return x, feats


def all_pairs_corr(f1: Tensor, f2: Tensor) -> Tensor:
    """raft/corr.py:167-175 / :85-93 → (B, h, w, 1, h, w)."""
    B, D, h, w = f1.shape
    c = torch.matmul(f1.view(B, D, h * w).transpose(1, 2), f2.view(B, D, h * w))
    return c.view(B, h, w, 1, h, w) / torch.sqrt(torch.tensor(D, device=c.device).to(c.dtype))


def corr_pyramid(vol: Tensor, levels=4) -> List[Tensor]:
    """raft/corr.py:135-142 — vol (B*N,1,h,w) + 3 × avg_pool2d(2)."""
    pyr = [vol]
    for _ in range(levels - 1):
        vol = F.avg_pool2d(vol, 2, stride=2)
        pyr.append(vol)
    return pyr


def _bilinear_sampler(img: Tensor, coords: Tensor) -> Tensor:
    """raft/utils/utils.py:66-80 — pixel coords → normalised → grid_sample
    (zeros padding, align_corners=True)."""
    H, W = img.shape[-2:]
    xg, yg = coords.split([1, 1], dim=-1)
    xg = 2 * xg / (W - 1) - 1
    yg = 2 * yg / (H - 1) - 1
    return F.grid_sample(img, torch.cat([xg, yg], dim=-1), align_corners=True)


def corr_lookup(pyr: List[Tensor], coords: Tensor, r=4) -> Tensor:
    """raft/corr.py:144-165.  ``delta = stack(meshgrid(dy, dx))`` is added to
    (x, y): output channel i*9+j of a level samples offset (Δx, Δy)=(i-4, j-4).
    On the coordinates' device, in the volume's dtype (float64 restatements)."""
    B, _, h1, w1 = coords.shape
    c = coords.permute(0, 2, 3, 1)
    d = torch.linspace(-r, r, 2 * r + 1, device=coords.device, dtype=coords.dtype)
    delta = torch.stack(torch.meshgrid(d, d, indexing="ij"), dim=-1).view(1, 2 * r + 1, 2 * r + 1, 2)
    out = []
    for i, vol in enumerate(pyr):
        cen = c.reshape(B * h1 * w1, 1, 1, 2) / 2**i
        s = _bilinear_sampler(vol, cen + delta)
        out.append(s.view(B, h1, w1, -1))
    return torch.cat(out, dim=-1).permute(0, 3, 1, 2).contiguous().to(pyr[0].dtype)


def raft_motion_encoder(sd: SD, p: str, corr: Tensor, flow: Tensor) -> Tensor:
    """raft/update.py:94-112 (BasicMotionEncoder) → 126 motion features | the 2 flow channels."""
    e = p + ".encoder"
    cor = F.relu(_conv(sd, e + ".convc1", corr))
    cor = F.relu(_conv(sd, e + ".convc2", cor, padding=1))
    flo = F.relu(_conv(sd, e + ".convf1", flow, padding=3))
    flo = F.relu(_conv(sd, e + ".convf2", flo, padding=1))
    out = F.relu(_conv(sd, e + ".conv", torch.cat([cor, flo], 1), padding=1))
    return torch.cat([out, flow], 1)


def raft_update_block(sd: SD, p: str, net: Tensor, inp: Tensor, corr: Tensor, flow: Tensor):
    """raft/update.py:131-154 (BasicMotionEncoder :94-112, SepConvGRU :35-73,
    FlowHead :6-14, mask head :139-143)."""
    motion = raft_motion_encoder(sd, p, corr, flow)
    x = torch.cat([inp, motion], 1)
    g = p + ".gru"
    h = net
    for sfx, pad in (("1", (0, 2)), ("2", (2, 0))):
        hx = torch.cat([h, x], 1)
        z = torch.sigmoid(_conv(sd, g + ".convz" + sfx, hx, padding=pad))
        rr = torch.sigmoid(_conv(sd, g + ".convr" + sfx, hx, padding=pad))
        q = torch.tanh(_conv(sd, g + ".convq" + sfx, torch.cat([rr * h, x], 1), padding=pad))
        h = (1 - z) * h + z * q
    dflow = _conv(sd, p + ".flow_head.conv2", F.relu(_conv(sd, p + ".flow_head.conv1", h, padding=1)), padding=1)
    mask = 0.25 * _conv(sd, p + ".mask.2", F.relu(_conv(sd, p + ".mask.0", h, padding=1)))
    return h, mask, dflow


def convex_upsample(flow: Tensor, mask: Tensor) -> Tensor:
    """raft/raft.py:86-97"""
    N, _, H, W = flow.shape
    mask = torch.softmax(mask.view(N, 1, 9, 8, 8, H, W), dim=2)
    up = F.unfold(8 * flow, [3, 3], padding=1).view(N, 2, 9, 1, 1, H, W)
    up = torch.sum(mask * up, dim=2).permute(0, 1, 4, 2, 5, 3)
    return up.reshape(N, 2, 8 * H, 8 * W)


def raft_forward(sd: SD, p: str, image1: Tensor, image2: Tensor, iters=20, trace: Optional[dict] = None):
    """raft/raft.py:99-169 with return_feat=True → (flow_up, feats[1:], fmap1)."""
    image1 = (2 * (image1 / 255.0) - 1.0).contiguous()
    image2 = (2 * (image2 / 255.0) - 1.0).contiguous()
    fmaps, _ = basic_encoder(sd, p + ".fnet", torch.cat([image1, image2], 0), "instance")
    B = image1.shape[0]
    fmap1, fmap2 = fmaps[:B].float(), fmaps[B:].float()
    vol = all_pairs_corr(fmap1, fmap2)
    b, h1, w1, d, h2, w2 = vol.shape
    pyr = corr_pyramid(vol.reshape(b * h1 * w1, d, h2, w2))
    cnet, feats = basic_encoder(sd, p + ".cnet", image1, "batch")
    net, inp = torch.split(cnet, [128, 128], dim=1)
    net, inp = torch.tanh(net), torch.relu(inp)
    coords0 = coords_grid(B, h1, w1)
    coords1 = coords_grid(B, h1, w1)
    flow_up = None
    for it in range(iters):
        corr = corr_lookup(pyr, coords1)
        flow = coords1 - coords0
        net, up_mask, dflow = raft_update_block(sd, p + ".update_block", net, inp, corr, flow)
        coords1 = coords1 + dflow
        if trace is not None and it in (0, 4, iters - 1):
            trace["lowres_flow_it%d" % it] = (coords1 - coords0).clone()
            if it == 0:
                trace["corr_it0"] = corr.clone()
        if it == iters - 1:  # only the last upsample is used (raft.py:159-167)
            flow_up = convex_upsample(coords1 - coords0, up_mask)
    if trace is not None:
        trace["fmap1"] = fmap1
        trace["net_final"] = net
    return flow_up, feats[1:], fmap1


# --------------------------------------------------------------------------
# bidirectional correlation (raft/corr.py:23-93)
# --------------------------------------------------------------------------
class BidirCorr:
    def __init__(self, f0: Tensor, f1: Tensor, levels=4, radius=4):
        vol = all_pairs_corr(f0, f1)
        b, h1, w1, d, h2, w2 = vol.shape
        vol_t = vol.clone().permute(0, 4, 5, 3, 1, 2)
        self.pyr = corr_pyramid(vol.reshape(b * h1 * w1, d, h2, w2), levels)
        self.pyr_t = corr_pyramid(vol_t.reshape(b * h2 * w2, d, h1, w1), levels)
        self.r = radius

    def __call__(self, coords0: Tensor, coords1: Tensor):
        return corr_lookup(self.pyr, coords0, self.r), corr_lookup(self.pyr_t, coords1, self.r)


# --------------------------------------------------------------------------
# GIMM: splat weights, latent encoders, forward splat, HypoNet
# --------------------------------------------------------------------------
def normalize_flow(flows: Tensor):
    """modules/fi_utils.py:52-60"""
    s = torch.max(torch.abs(flows).flatten(1), dim=-1)[0].reshape(-1, 1, 1, 1, 1)
    return (flows / s + 1.0) / 2.0, s


def splatting_weights(sd: SD, f01: Tensor, f10: Tensor):
    """gimmvfi_r.py:444-492"""
    B = f01.shape[0]
    fl = torch.cat([f01, f10], 0)
    x = F.pad(torch.cat([fl**2, fl], 1), (1, 1, 1, 1), mode="reflect").unsqueeze(1)
    blur = F.conv3d(x, sd["g_filter"]).squeeze(1)
    sq_mean, mean = torch.split(blur, 2, dim=1)
    var = (sq_mean - mean**2).clamp(1e-9, None).sqrt().mean(1).unsqueeze(1)
    var01, var10 = var[:B], var[B:]
    err01 = (-backwarp(f10, f01) - f01).abs().mean(1).unsqueeze(1)
    err10 = (-backwarp(f01, f10) - f10).abs().mean(1).unsqueeze(1)
    w1 = 1 / (1 + err01 * sd["alpha_fe"]) + 1 / (1 + var01 * sd["alpha_v"])
    w2 = 1 / (1 + err10 * sd["alpha_fe"]) + 1 / (1 + var10 * sd["alpha_v"])
    return w1, w2


def _lateral(sd: SD, p: str, x: Tensor) -> Tensor:
    """modules/fi_components.py:17-29"""
    y = _conv(sd, p + ".layers.0", x, padding=1)
    y = F.leaky_relu(y, 0.1)
    y = _conv(sd, p + ".layers.2", y, padding=1)
    return y + x


def cnn_encoder(sd: SD, x: Tensor) -> Tensor:
    """gimmvfi_r.py:86-97"""
    p = "cnn_encoder"
    x = _conv(sd, p + ".0", x, padding=1)
    x = F.leaky_relu(_conv(sd, p + ".1", x, padding=1), 0.1)
    for i in (3, 4, 5):
        x = _lateral(sd, "%s.%d" % (p, i), x)
    x = F.leaky_relu(x, 0.1)
    return _conv(sd, p + ".7", x, padding=1, reflect=True)


def res_conv(sd: SD, x: Tensor) -> Tensor:
    """gimmvfi_r.py:100-109"""
    p = "res_conv"
    x = _conv(sd, p + ".0", x, padding=1)
    x = F.leaky_relu(_conv(sd, p + ".1", x, padding=1), 0.1)
    x = F.leaky_relu(_lateral(sd, p + ".3", x), 0.1)
    return _conv(sd, p + ".5", x, padding=1, reflect=True)


def forward_splat_sum(inp: Tensor, flow: Tensor) -> Tensor:
    """The ``softsplat_out`` CUDA kernel (modules/softsplat.py:376-421) restated
    with index_add_: every source pixel adds ``in·w_corner`` to its ≤4 in-frame
    target corners; non-finite flow → pixel skipped.  On the input's device, in its dtype."""
    N, C, H, W = inp.shape
    kw = dict(device=inp.device, dtype=inp.dtype)
    gx = torch.arange(W, **kw).view(1, 1, W).expand(N, H, W)
    gy = torch.arange(H, **kw).view(1, H, 1).expand(N, H, W)
    fx, fy = gx + flow[:, 0], gy + flow[:, 1]
    finite = torch.isfinite(fx) & torch.isfinite(fy)
    fx = torch.where(finite, fx, torch.zeros_like(fx))
    fy = torch.where(finite, fy, torch.zeros_like(fy))
    x0, y0 = torch.floor(fx).long(), torch.floor(fy).long()
    x1, y1 = x0 + 1, y0 + 1
    x0f, y0f, x1f, y1f = x0.to(inp.dtype), y0.to(inp.dtype), x1.to(inp.dtype), y1.to(inp.dtype)
    corners = (
        (x0, y0, (x1f - fx) * (y1f - fy)),
        (x1, y0, (fx - x0f) * (y1f - fy)),
        (x0, y1, (x1f - fx) * (fy - y0f)),
        (x1, y1, (fx - x0f) * (fy - y0f)),
    )
    nidx = torch.arange(N, device=inp.device).view(N, 1, 1).expand(N, H, W)
    buf = torch.zeros(N * H * W, C, **kw)
    src = inp.permute(0, 2, 3, 1).reshape(N * H * W, C)
    for xx, yy, ww in corners:
        ok = (finite & (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)).reshape(-1)
        lin = ((nidx * H + yy.clamp(0, H - 1)) * W + xx.clamp(0, W - 1)).reshape(-1)
        buf.index_add_(0, lin[ok], src[ok] * ww.reshape(-1, 1)[ok])
    return buf.view(N, H, W, C).permute(0, 3, 1, 2).contiguous()


def softsplat_linear_zeroeps(inp: Tensor, flow: Tensor, metric: Tensor) -> Tensor:
    """modules/softsplat.py:286-352 for strMode == "linear-zeroeps"."""
    out = forward_splat_sum(torch.cat([inp * metric, metric], 1), flow)
    norm = out[:, -1:].clone()
    norm[norm == 0.0] = 1.0
    return out[:, :-1] / norm


def hyponet_weights(sd: SD, n_layer=5):
    """modules/hyponet.py:99-132 — per layer: fan-in-normalised weight columns
    (F.normalize over dim=1 of (B, fan_in, fan_out)) and the raw bias row."""
    ws = []
    for i in range(n_layer):
        wb = sd["hyponet.params_dict.linear_wb%d" % i]
        ws.append((F.normalize(wb[:-1], dim=0), wb[-1:]))
    return ws


def hyponet_forward(sd: SD, coord: Tensor, latent_bhwc: Tensor, output_bias=0.5, w0=1.0) -> Tensor:
    """modules/hyponet.py:71-146 (no modulation, no sub-sampling)."""
    B = coord.shape[0]
    cshape = coord.shape[1:-1]
    lat = F.interpolate(latent_bhwc.permute(0, 3, 1, 2), size=(cshape[1], cshape[2]), mode="bilinear").permute(0, 2, 3, 1)
    hid = torch.cat([lat.reshape(B, -1, lat.shape[-1]), coord.view(B, -1, coord.shape[-1])], dim=-1)
    ws = hyponet_weights(sd)
    for i, (w, b) in enumerate(ws):
        ones = torch.ones(*hid.shape[:-1], 1, device=hid.device, dtype=hid.dtype)
        hid = torch.bmm(torch.cat([hid, ones], -1), torch.cat([w, b], 0)[None].expand(B, -1, -1))
        if i < len(ws) - 1:
            hid = torch.sin(w0 * hid)
    return (hid + output_bias).view(B, *cshape, -1)


def predict_flow(sd: SD, nflow: Tensor, coords: List[Tensor], ts: List[Tensor], flows: Tensor, trace=None):
    """gimmvfi_r.py:158-211 → list of (B,2,1,Hc,Wc) normalised flows."""
    f01, f10 = flows[:, :, 0], flows[:, :, 1]
    w1, w2 = splatting_weights(sd, f01, f10)
    lat0 = cnn_encoder(sd, nflow[:, :, 0])
    lat1 = cnn_encoder(sd, nflow[:, :, 1])
    outs = []
    for c, t in zip(coords, ts):
        tt = t.reshape(-1, 1, 1, 1)
        s0 = softsplat_linear_zeroeps(lat0, f01 * tt, w1)
        s1 = softsplat_linear_zeroeps(lat1, f10 * (1 - tt), w2)
        sp = torch.cat([s0, s1], 1)
        lat = sp + res_conv(sd, torch.cat([lat0, lat1, sp], 1))
        if trace is not None and "latent" not in trace:
            trace.update(splat_w1=w1, splat_w2=w2, lat0=lat0, splat0=s0, latent=lat)
        o = hyponet_forward(sd, c, lat.permute(0, 2, 3, 1))  # (B,1,Hc,Wc,2)
        outs.append(o.permute(0, 4, 1, 2, 3))
    return outs


def gimm_forward(sd: SD, xs: Tensor, coord, ori_flow: Tensor, timesteps, keep_xs_shape: bool = True):
    """gimm.py:129-214 — GIMM.forward, the motion-modelling network alone (cal_splatting_weights :82-127, cnn_encoder,
    softsplat "linear-zeroeps", res_conv, HypoNet).  xs (B,2,2,H,W): normalised flows [f01 | f10] on dim 2; ori_flow: the raw
    flows.  List form: timesteps = [ (B,) ... ], coord = [ (B,1,Hc,Wc,3) ... ] -> list of outputs; tensor form -> one output.
    Output (B,2,1,Hc,Wc) with keep_xs_shape (the reference's `permute(0, -1, 1, 2, 3)`), else (B,1,Hc,Wc,2)."""
    is_list = isinstance(timesteps, list)
    if is_list:
        assert isinstance(coord, list) and len(coord) == len(timesteps)
    outs = predict_flow(sd, xs, coord if is_list else [coord], timesteps if is_list else [timesteps], ori_flow)
    if not keep_xs_shape:
        outs = [o.permute(0, 2, 3, 4, 1) for o in outs]
    return outs if is_list else outs[0]


# --------------------------------------------------------------------------
# AMT-style synthesis (modules/fi_components.py)
# --------------------------------------------------------------------------
def _convrelu(sd: SD, p: str, x: Tensor, padding=1) -> Tensor:
    """fi_components.py:32-54 — Sequential(Conv2d, PReLU(C))."""
    return _prelu(sd, p + ".1", _conv(sd, p + ".0", x, padding=padding))


def _resblock(sd: SD, p: str, x: Tensor, side: int) -> Tensor:
    """fi_components.py:97-154"""
    out = _convrelu(sd, p + ".conv1", x)
    out = torch.cat([out[:, :-side], _convrelu(sd, p + ".conv2", out[:, -side:])], 1)
    out = _convrelu(sd, p + ".conv3", out)
    out = torch.cat([out[:, :-side], _convrelu(sd, p + ".conv4", out[:, -side:])], 1)
    out = _conv(sd, p + ".conv5", out, padding=1)
    return _prelu(sd, p + ".prelu", x + out)


def _decoder_upsample(sd: SD, p: str, x: Tensor, n_shuffle: int) -> Tensor:
    """fi_components.py:234-244 (n_shuffle=1) / :284-295 (n_shuffle=2)."""
    for _ in range(n_shuffle):
        x = F.pixel_shuffle(x, 2)
    i = n_shuffle
    x = _convrelu(sd, "%s.%d" % (p, i), x, padding=2)
    for k in range(1, 5):
        x = _convrelu(sd, "%s.%d" % (p, i + k), x, padding=1)
    x = _conv(sd, "%s.%d" % (p, i + 5), x)
    return F.relu(_bn_eval(sd, "%s.%d" % (p, i + 6), x))


def init_decoder(sd: SD, f0, f1, flow0_in, flow1_in, img0, img1):
    """fi_components.py:229-276"""
    f0 = _decoder_upsample(sd, "amt_init_decoder.upsample", f0, 1)
    f1 = _decoder_upsample(sd, "amt_init_decoder.upsample", f1, 1)
    return init_convblock(sd, init_decoder_concat(f0, f1, flow0_in, flow1_in, img0, img1), flow0_in, flow1_in)


def init_decoder_concat(fup0, fup1, flow0_in, flow1_in, img0, img1):
    """fi_components.py:255-268: the 272-channel convblock input from the up-sampled features and the flows at H/4"""
    f_in = torch.cat([backwarp(fup0, flow0_in), backwarp(fup1, flow1_in), flow0_in, flow1_in], 1)
    sc = f_in.shape[2] / img0.shape[2]
    i0, i1 = resize(img0, sc), resize(img1, sc)
    return torch.cat([f_in, i0, i1, backwarp(i0, flow0_in), backwarp(i1, flow1_in)], 1)


def init_convblock(sd: SD, f_in, flow0_in, flow1_in):
    """fi_components.py:269-276 -> (flow0, flow1, [mask | ft_])"""
    c = "amt_init_decoder.convblock"
    x = _convrelu(sd, c + ".0", f_in, padding=0)
    for k in (1, 2, 3):
        x = _resblock(sd, "%s.%d" % (c, k), x, 64)
    out = _conv(sd, c + ".4", x, padding=1)
    return flow0_in + out[:, :2], flow1_in + out[:, 2:4], out[:, 4:]


def amt_update_block(sd: SD, p: str, net, flow, corr, scale_factor):
    """fi_components.py:157-222"""
    lr = lambda v: F.leaky_relu(v, 0.1)
    if scale_factor is not None:
        net = resize(net, 1 / scale_factor)
    cor = lr(_conv(sd, p + ".convc1", corr))
    cor = lr(_conv(sd, p + ".convc2", cor, padding=1))
    flo = lr(_conv(sd, p + ".convf1", flow, padding=3))
    flo = lr(_conv(sd, p + ".convf2", flo, padding=1))
    inp = lr(_conv(sd, p + ".conv", torch.cat([cor, flo], 1), padding=1))
    inp = torch.cat([inp, flow, net], 1)
    out = _conv(sd, p + ".gru.2", lr(_conv(sd, p + ".gru.0", inp, padding=1)), padding=1)
    dnet = _conv(sd, p + ".feat_head.2", lr(_conv(sd, p + ".feat_head.0", out, padding=1)), padding=1)
    dflow = _conv(sd, p + ".flow_head.2", lr(_conv(sd, p + ".flow_head.0", out, padding=1)), padding=1)
    if scale_factor is not None:
        dnet = resize(dnet, scale_factor)
        dflow = scale_factor * resize(dflow, scale_factor)
    return dnet, dflow


def final_decoder_concat(ft_, fup0, fup1, flow0, flow1, mask, img0, img1):
    """fi_components.py:318-326: the 273-channel input of the final decoder's convblock from the H/4 state and the up-sampled
    features -> (f_in, flow0, flow1, mask), the last three at full network resolution."""
    flow0 = 4.0 * resize(flow0, 4.0)
    flow1 = 4.0 * resize(flow1, 4.0)
    ft_ = resize(ft_, 4.0)
    mask = resize(mask, 4.0)
    f_in = torch.cat([ft_, backwarp(fup0, flow0), backwarp(fup1, flow1), flow0, flow1, mask], 1)
    f_in = torch.cat([f_in, img0, img1, backwarp(img0, flow0), backwarp(img1, flow1)], 1)
    return f_in, flow0, flow1, mask


def final_convblock(sd: SD, f_in):
    """fi_components.py:327-330: the 256-channel residual trunk and convblock.4 -> the 24-channel head input"""
    c = "amt_final_decoder.convblock"
    x = _convrelu(sd, c + ".0", f_in)
    for k in (1, 2, 3):
        x = _resblock(sd, "%s.%d" % (c, k), x, 64)
    return _conv(sd, c + ".4", x, padding=1)


def final_heads(out, flow0, flow1, mask, n=3):
    """fi_components.py:331-340"""
    dflow0, dflow1, dmask, img_res = torch.split(out, [2 * n, 2 * n, n, 3 * n], 1)
    mask = torch.sigmoid(dmask + mask.repeat(1, n, 1, 1))
    return dflow0 + flow0.repeat(1, n, 1, 1), dflow1 + flow1.repeat(1, n, 1, 1), mask, img_res


def final_decoder(sd: SD, ft_, f0, f1, flow0, flow1, mask, img0, img1, n=3):
    """fi_components.py:279-340"""
    p = "amt_final_decoder"
    f0 = _decoder_upsample(sd, p + ".upsample", f0, 2)
    f1 = _decoder_upsample(sd, p + ".upsample", f1, 2)
    f_in, flow0, flow1, mask = final_decoder_concat(ft_, f0, f1, flow0, flow1, mask, img0, img1)
    return final_heads(final_convblock(sd, f_in), flow0, flow1, mask, n)


def comb_block(sd: SD, warps):
    """gimmvfi_r.py:60-64: Conv2d(9, 18, 7) + PReLU + Conv2d(18, 3, 7) on the (b, 3n, h, w) blended warps"""
    x = _conv(sd, "amt_comb_block.0", warps, padding=3)
    x = _prelu(sd, "amt_comb_block.1", x)
    return _conv(sd, "amt_comb_block.2", x, padding=3)


def multi_flow_combine(sd: SD, img0, img1, flow0, flow1, mask, img_res, trace=None):
    """fi_components.py:57-94 with comb_block = amt_comb_block (gimmvfi_r.py:60-64).  trace: warps (b,3n,h,w), mean, comb."""
    b, c, h, w = flow0.shape
    n = c // 2
    flow0 = flow0.reshape(b * n, 2, h, w)
    flow1 = flow1.reshape(b * n, 2, h, w)
    mask = mask.reshape(b * n, 1, h, w)
    img_res = img_res.reshape(b * n, 3, h, w)
    i0 = torch.stack([img0] * n, 1).reshape(-1, 3, h, w)
    i1 = torch.stack([img1] * n, 1).reshape(-1, 3, h, w)
    warps = mask * backwarp(i0, flow0) + (1 - mask) * backwarp(i1, flow1) + img_res
    warps = warps.reshape(b, n, 3, h, w)
    x = comb_block(sd, warps.view(b, -1, h, w))
    if trace is not None:
        trace.update(warps=warps.view(b, -1, h, w), mean=warps.mean(1), comb=x)
    return (warps.mean(1) + x + 1.0) / 2


def synthesis_tail(sd: SD, ft_4, flowt0_4, flowt1_4, mask_4, fup0, fup1, img0, img1, full_img=None, trace=None, n=3):
    """gimmvfi_r.py:283-308 from the H/4 state on, starting at the final decoder's up-sampled features fup0 / fup1 (so that another
    implementation's own can be fed in): the concat, the residual trunk and heads (fi_components.py:318-340), the resize of the heads to
    full_img's resolution (gimmvfi_r.py:294-303), multi_flow_combine and the clamp -> (pred, flowt0_1, flowt1_1).  img0 / img1 in [-1, 1]
    at the network resolution, full_img (B,3,2,Hf,Wf) in [0, 1].  trace: fin, out24, F0 / F1 / Mk / Rs (the heads at the network
    resolution), F0f / F1f / Mkf / Rsf (at full resolution), warps, mean, comb, pred."""
    f_in, flow0, flow1, mask = final_decoder_concat(ft_4, fup0, fup1, flowt0_4, flowt1_4, mask_4, img0, img1)
    out = final_convblock(sd, f_in)
    flowt0_1, flowt1_1, mask, img_res = final_heads(out, flow0, flow1, mask, n)
    if trace is not None:
        trace.update(fin=f_in, out24=out, F0=flowt0_1, F1=flowt1_1, Mk=mask, Rs=img_res)
    if full_img is not None:
        img0 = 2 * full_img[:, :, 0] - 1.0
        img1 = 2 * full_img[:, :, 1] - 1.0
        inv = img1.shape[2] / flowt0_1.shape[2]
        flowt0_1 = inv * resize(flowt0_1, inv)
        flowt1_1 = inv * resize(flowt1_1, inv)
        mask = resize(mask, inv)
        img_res = resize(img_res, inv)
    if trace is not None:
        trace.update(F0f=flowt0_1, F1f=flowt1_1, Mkf=mask, Rsf=img_res)
    pred = torch.clamp(multi_flow_combine(sd, img0, img1, flowt0_1, flowt1_1, mask, img_res, trace), 0, 1)
    if trace is not None:
        trace["pred"] = pred
    return pred, flowt0_1, flowt1_1


def frame_synthesize(sd: SD, img_xs, flow_t, feats0, feats1, corr_fn: BidirCorr, cur_t, full_img=None, trace=None):
    """gimmvfi_r.py:222-322"""
    B = img_xs.shape[0]
    img0 = 2 * img_xs[:, :, 0] - 1.0
    img1 = 2 * img_xs[:, :, 1] - 1.0
    H, W = img0.shape[-2:]
    coord = coords_grid(B, H // 8, W // 8, flow_t)
    flow_t0_full = flow_t * (-cur_t)
    flow_t1_full = flow_t * (1.0 - cur_t)
    ft0_4 = 0.25 * resize(flow_t0_full, 0.25)
    ft1_4 = 0.25 * resize(flow_t1_full, 0.25)
    flowt0_4, flowt1_4, ft_4 = init_decoder(sd, feats0[-1], feats1[-1], ft0_4, ft1_4, img0, img1)
    mask_4, ft_4 = ft_4[:, :1], ft_4[:, 1:]
    # warp_w_mask (gimmvfi_r.py:213-220), scale=4 — aux output only
    a0 = 4 * resize(flowt0_4, 4)
    a1 = 4 * resize(flowt1_4, 4)
    am = resize(mask_4, 4).sigmoid()
    img_warp_4 = am * backwarp(img0, a0) + (1 - am) * backwarp(img1, a1)
    img_warp_4 = torch.clamp((img_warp_4 + 1.0) / 2, 0, 1)
    # _amt_corr_scale_lookup (gimmvfi_r.py:494-507), downsample=2
    fl0 = 0.5 * resize(flowt0_4, 0.5)
    fl1 = 0.5 * resize(flowt1_4, 0.5)
    c0, c1 = corr_fn(coord + fl1 * (1.0 / (1.0 - cur_t)), coord + fl0 * (1.0 / cur_t))
    corr_4 = torch.cat([c0, c1], 1)
    flow_4_lr = torch.cat([fl0, fl1], 1)
    dft, dfl = amt_update_block(sd, "amt_update4_low", ft_4, flow_4_lr, corr_4, 2.0)
    d0, d1 = torch.chunk(dfl, 2, 1)
    flowt0_4, flowt1_4, ft_4 = flowt0_4 + d0, flowt1_4 + d1, ft_4 + dft
    corr_4 = resize(corr_4, 2.0)
    dft, dfl = amt_update_block(sd, "amt_update4_high", ft_4, torch.cat([flowt0_4, flowt1_4], 1), corr_4, None)
    flowt0_4, flowt1_4, ft_4 = flowt0_4 + dfl[:, :2], flowt1_4 + dfl[:, 2:4], ft_4 + dft
    if trace is not None and "ft_4" not in trace:
        trace.update(ft_4=ft_4, flowt0_4=flowt0_4, corr_4_hi=corr_4)
    fup0 = _decoder_upsample(sd, "amt_final_decoder.upsample", feats0[0], 2)
    fup1 = _decoder_upsample(sd, "amt_final_decoder.upsample", feats1[0], 2)
    pred, flowt0_1, flowt1_1 = synthesis_tail(sd, ft_4, flowt0_4, flowt1_4, mask_4, fup0, fup1, img0, img1, full_img)
    Hf, Wf = pred.shape[-2:]
    return (
        pred,
        [flowt0_1.reshape(B, 3, 2, Hf, Wf), flowt0_4],
        [flowt1_1.reshape(B, 3, 2, Hf, Wf), flowt1_4],
        [img_warp_4],
    )


# --------------------------------------------------------------------------
# top level
# --------------------------------------------------------------------------
def sample_coord_input(B: int, shape, t_ids, upsample_ratio=1.0) -> Tensor:
    """modules/coord_sampler.py:21-43 — (B, T, Hc, Wc, 3) with last dim (t, y, x)."""
    cs = [torch.tensor(t_ids).to(torch.float32) / 1.0]
    for n in shape:
        n = int(n * upsample_ratio)
        cs.append(-1.0 + 2.0 * ((0.5 + torch.arange(n)) / n))
    g = torch.stack(torch.meshgrid(*cs, indexing="ij"), dim=-1)
    return g.unsqueeze(0).repeat(B, 1, 1, 1, 1)


def gimmvfi_r_forward(sd: SD, img_xs: Tensor, coord: list, t: list, ds_factor=None, iters=20, trace: Optional[dict] = None):
    """gimmvfi_r.py:324-407 (inference form: every coord[i][1] is None)."""
    assert isinstance(t, list) and isinstance(coord, list) and len(t) == len(coord)
    full = None
    if ds_factor is not None:
        full = img_xs.clone()
        img_xs = torch.stack([resize(img_xs[:, :, 0], ds_factor), resize(img_xs[:, :, 1], ds_factor)], 2)
    # cal_bidirection_flow (gimmvfi_r.py:126-156)
    I0, I1 = 255 * img_xs[:, :, 0], 255 * img_xs[:, :, 1]
    tr0 = {} if trace is not None else None
    f01, feats0, fnet0 = raft_forward(sd, "flow_estimator", I0, I1, iters, tr0)
    f10, feats1, fnet1 = raft_forward(sd, "flow_estimator", I1, I0, iters)
    corr_fn = BidirCorr(_conv(sd, "amt_fproj", fnet0), _conv(sd, "amt_fproj", fnet1))
    feats0 = [_conv(sd, "amt_second_last_cproj", feats0[0]), _conv(sd, "amt_last_cproj", feats0[1])]
    feats1 = [_conv(sd, "amt_second_last_cproj", feats1[0]), _conv(sd, "amt_last_cproj", feats1[1])]
    nflow, scaler = normalize_flow(torch.stack([f01, -f10], 2))
    flows = torch.stack([f01, f10], 2)
    if trace is not None:
        trace.update({"raft0." + k: v for k, v in tr0.items()})
        trace.update(feat0_4=feats0[0], feat0_8=feats0[1])
    ninr = predict_flow(sd, nflow, [c[0] for c in coord], t, flows, trace)
    flow_t = [((o * 2.0 - 1.0) * scaler).squeeze() for o in ninr]  # unnormalize_flow fi_utils.py:63-64
    preds, ft0s, ft1s, others = [], [], [], []
    for i in range(len(coord)):
        cur = flow_t[i]
        if cur.ndim != 4:
            cur = cur.unsqueeze(0)
        p, a, b, o = frame_synthesize(sd, img_xs, cur, feats0, feats1, corr_fn, t[i].reshape(-1, 1, 1, 1), full, trace)
        preds.append(p)
        ft0s.append(a)
        ft1s.append(b)
        others.append(o)
    return {
        "imgt_pred": preds,
        "other_pred": others,
        "flowt0_pred": ft0s,
        "flowt1_pred": ft1s,
        "raft_flow": flows,
        "ninrflow": ninr,
        "nflow": nflow,
        "flowt": flow_t,
    }
