"""TEST INFRASTRUCTURE — not product code.  CPU restatement (functional torch fp32 on a flat ``state_dict``) of the flow estimator of
GIMM-VFI-F: FlowFormer (LatentCostFormer) as the reference runs it at inference.  Only tests/, __graft_entry__.smoke() and the
bench's cpu_baseline / reference arm may import this file.

Pinned against the UNMODIFIED reference modules (oracle/ref_shim_f.py) by tests/test_oracle.py::test_flowformer_oracle_matches_reference
and oracle/make_golden_ff.py (max|Δ| = 0.0 on the flows / features of every fixture).  PARITY UNPINNED AT THE TIMM BOUNDARY: the Twins-SVT
arithmetic restated here follows the reference tree's vendored copy of timm 0.4.12's twins.py; timm itself is not available offline.

Citations are relative to /root/reference/src/models/generalizable_INR/flowformer/core/FlowFormer/ (LCF = LatentCostFormer/).
Configuration = configs/submission.py:19-50 (the only one GIMM-VFI-F builds, flowformer/__init__.py): twins encoders, 8 latent tokens of
128, cost_heads 1, patch 8, encoder_depth 3, vert_c_dim 64, GMA, decoder_depth 32, add_flow_token, query dim 64.
"""
import math

import torch
import torch.nn.functional as F

P = "flow_estimator."


def _lin(sd, k, x):
    return F.linear(x, sd[k + ".weight"], sd.get(k + ".bias"))


def _ln(sd, k, x, eps):
    return F.layer_norm(x, (x.shape[-1],), sd[k + ".weight"], sd[k + ".bias"], eps)


def coords_grid(b, h, w, like=None):
    """flowformer/core/utils/utils.py coords_grid: channel 0 = x, channel 1 = y.  With `like`: on its device, in its dtype (else fp32 on
    the CPU)."""
    dev = like.device if like is not None else None
    ys, xs = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
    return torch.stack([xs, ys], 0).to(like.dtype if like is not None else torch.float32)[None].repeat(b, 1, 1, 1)


def linear_pos_embedding_sine(x, dim=128):
    """LCF/attention.py:170-182 (the constant is 3.14, not pi)."""
    fb = torch.linspace(0, dim // 4 - 1, dim // 4, dtype=x.dtype, device=x.device)
    k = 1 / 200
    return torch.cat([torch.sin(3.14 * x[..., -2:-1] * fb * k), torch.cos(3.14 * x[..., -2:-1] * fb * k),
                      torch.sin(3.14 * x[..., -1:] * fb * k), torch.cos(3.14 * x[..., -1:] * fb * k)], -1)


def bilinear_sampler(img, coords):
    """flowformer/core/utils/utils.py bilinear_sampler: pixel coordinates -> grid_sample(align_corners=True), zeros padding."""
    H, W = img.shape[-2:]
    xg, yg = coords.split([1, 1], -1)
    xg = 2 * xg / (W - 1) - 1
    yg = 2 * yg / (H - 1) - 1
    return F.grid_sample(img, torch.cat([xg, yg], -1), align_corners=True)


def mha(q, k, v, heads):
    """LCF/attention.py:10-66 (MultiHeadAttention / BroadMultiHeadAttention): softmax(q k^T * (dim/heads)^-0.5) v per head."""
    B, Nq, D = q.shape
    d = D // heads
    qh = q.view(B, Nq, heads, d).transpose(1, 2)
    kh = k.view(k.shape[0], -1, heads, d).transpose(1, 2)
    vh = v.view(v.shape[0], -1, heads, d).transpose(1, 2)
    att = torch.softmax(qh @ kh.transpose(-1, -2) * d ** -0.5, -1)
    return (att @ vh).transpose(1, 2).reshape(max(B, k.shape[0]), Nq, D)


# ---------------------------------------------------------------------------------------------------------------------------
# Twins-SVT-L, stages 1-2 (encoders.py:7-48 wraps timm's twins_svt_large; arithmetic = LCF/twins.py:814-926,1100-1150 + timm Block)
# ---------------------------------------------------------------------------------------------------------------------------
def twins_lsa(sd, p, x, size, heads, ws=7):
    """LocallyGroupedAttn, LCF/twins.py:814-867: zero padding AFTER the norm, the padded tokens take part un-masked."""
    B, N, C = x.shape
    H, W = size
    x = x.view(B, H, W, C)
    pr, pb = (ws - W % ws) % ws, (ws - H % ws) % ws
    x = F.pad(x, (0, 0, 0, pr, 0, pb))
    Hp, Wp = x.shape[1:3]
    _h, _w = Hp // ws, Wp // ws
    x = x.reshape(B, _h, ws, _w, ws, C).transpose(2, 3)
    qkv = _lin(sd, p + ".qkv", x).reshape(B, _h * _w, ws * ws, 3, heads, C // heads).permute(3, 0, 1, 4, 2, 5)
    q, k, v = qkv[0], qkv[1], qkv[2]
    att = torch.softmax(q @ k.transpose(-2, -1) * (C // heads) ** -0.5, -1)
    o = (att @ v).transpose(2, 3).reshape(B, _h, _w, ws, ws, C).transpose(2, 3).reshape(B, Hp, Wp, C)[:, :H, :W].reshape(B, N, C)
    return _lin(sd, p + ".proj", o)


def twins_gsa(sd, p, x, size, heads, sr):
    """GlobalSubSampleAttn, LCF/twins.py:870-925: keys / values from a stride-sr conv of the tokens + LayerNorm (eps 1e-5)."""
    B, N, C = x.shape
    q = _lin(sd, p + ".q", x).reshape(B, N, heads, C // heads).permute(0, 2, 1, 3)
    xs = x.permute(0, 2, 1).reshape(B, C, *size)
    xs = F.conv2d(xs, sd[p + ".sr.weight"], sd[p + ".sr.bias"], stride=sr).reshape(B, C, -1).permute(0, 2, 1)
    xs = _ln(sd, p + ".norm", xs, 1e-5)
    kv = _lin(sd, p + ".kv", xs).reshape(B, -1, 2, heads, C // heads).permute(2, 0, 3, 1, 4)
    att = torch.softmax(q @ kv[0].transpose(-2, -1) * (C // heads) ** -0.5, -1)
    return _lin(sd, p + ".proj", (att @ kv[1]).transpose(1, 2).reshape(B, N, C))


def twins_svt(sd, p, x):
    """encoders.py:22-45: two stages (embed 128 / 256, heads 4 / 8, depth 2 each: LSA ws 7 then GSA sr 8 / 4), PEG after block 0.
    Returns the stage outputs as NCHW maps [(B,128,H/4,W/4), (B,256,H/8,W/8)]."""
    B = x.shape[0]
    feats = []
    for i, (patch, heads, sr) in enumerate([(4, 4, 8), (2, 8, 4)]):
        q = "%s.svt.patch_embeds.%d" % (p, i)
        x = F.conv2d(x, sd[q + ".proj.weight"], sd[q + ".proj.bias"], stride=patch)                 # LCF/twins.py:1142-1149
        size = x.shape[2:]
        x = _ln(sd, q + ".norm", x.flatten(2).transpose(1, 2), 1e-5)
        for j in range(2):
            b = "%s.svt.blocks.%d.%d" % (p, i, j)
            y = _ln(sd, b + ".norm1", x, 1e-6)                                                      # timm Block, norm eps 1e-6 (twins.py:1167)
            x = x + (twins_lsa(sd, b + ".attn", y, size, heads) if j == 0 else twins_gsa(sd, b + ".attn", y, size, heads, sr))
            y = _ln(sd, b + ".norm2", x, 1e-6)
            x = x + _lin(sd, b + ".mlp.fc2", F.gelu(_lin(sd, b + ".mlp.fc1", y)))
            if j == 0:                                                                              # PosConv, LCF/twins.py:1100-1116
                pw = "%s.svt.pos_block.%d.proj.0" % (p, i)
                m = x.transpose(1, 2).view(B, -1, *size)
                x = (F.conv2d(m, sd[pw + ".weight"], sd[pw + ".bias"], padding=1, groups=m.shape[1]) + m).flatten(2).transpose(1, 2)
        x = x.reshape(B, *size, -1).permute(0, 3, 1, 2).contiguous()
        feats.append(x)
    return feats


# ---------------------------------------------------------------------------------------------------------------------------
# Memory encoder (LCF/encoder.py)
# ---------------------------------------------------------------------------------------------------------------------------
def _mlp_block_tail(sd, b, x):
    y = _ln(sd, b + ".norm2", x, 1e-5)
    return x + _lin(sd, b + ".mlp.fc2", F.gelu(_lin(sd, b + ".mlp.fc1", y)))


def vertical_local(sd, b, x, size, context, heads=8, ws=7):
    """Block(ws=7, with_rpe, vert_c_dim=64) = LocallyGroupedAttnRPEContext, LCF/twins.py:331-427 + Block :1094-1097 (LayerNorm eps 1e-5)."""
    a = b + ".attn"
    y = _ln(sd, b + ".norm1", x, 1e-5)
    B, N, C = y.shape
    H, W = size
    ctx = context.repeat(B // context.shape[0], 1, 1, 1).view(B, -1, H * W).permute(0, 2, 1)
    ctx = _lin(sd, a + ".context_proj", ctx).view(B, H, W, -1)
    y = y.view(B, H, W, C)
    yqk = torch.cat([y, ctx], -1)
    Cqk = yqk.shape[-1]
    pr, pb = (ws - W % ws) % ws, (ws - H % ws) % ws
    y = F.pad(y, (0, 0, 0, pr, 0, pb))
    yqk = F.pad(yqk, (0, 0, 0, pr, 0, pb))
    Hp, Wp = y.shape[1:3]
    _h, _w = Hp // ws, Wp // ws
    y = y.reshape(B, _h, ws, _w, ws, C).transpose(2, 3)
    yqk = yqk.reshape(B, _h, ws, _w, ws, Cqk).transpose(2, 3)
    hd = C // heads
    v = _lin(sd, a + ".v", y).reshape(B, _h * _w, ws * ws, heads, hd).transpose(2, 3)
    pe = linear_pos_embedding_sine(coords_grid(B, ws, ws, y).view(B, 2, -1).permute(0, 2, 1), dim=Cqk).view(B, ws, ws, Cqk)
    yqk = yqk + pe[:, None, None]
    q = _lin(sd, a + ".q", yqk).reshape(B, _h * _w, ws * ws, heads, hd).transpose(2, 3)
    k = _lin(sd, a + ".k", yqk).reshape(B, _h * _w, ws * ws, heads, hd).transpose(2, 3)
    att = torch.softmax(q @ k.transpose(-2, -1) * hd ** -0.5, -1)
    o = (att @ v).transpose(2, 3).reshape(B, _h, _w, ws, ws, C).transpose(2, 3).reshape(B, Hp, Wp, C)[:, :H, :W].reshape(B, N, C)
    x = x + _lin(sd, a + ".proj", o)
    return _mlp_block_tail(sd, b, x)


def vertical_global(sd, b, x, size, context, heads=8, sr=4):
    """Block(ws=1, with_rpe, vert_c_dim=64) = GlobalSubSampleAttnRPEContext, LCF/twins.py:430-546."""
    a = b + ".attn"
    y = _ln(sd, b + ".norm1", x, 1e-5)
    B, N, C = y.shape
    H, W = size
    ctx = context.repeat(B // context.shape[0], 1, 1, 1).view(B, -1, H * W).permute(0, 2, 1)
    ctx = _lin(sd, a + ".context_proj", ctx).view(B, H, W, -1)
    y = y.view(B, H, W, C)
    yqk = torch.cat([y, ctx], -1)
    Cqk = yqk.shape[-1]
    pr, pb = (sr - W % sr) % sr, (sr - H % sr) % sr
    y = F.pad(y, (0, 0, 0, pr, 0, pb))
    yqk = F.pad(yqk, (0, 0, 0, pr, 0, pb))
    Hp, Wp = y.shape[1:3]
    hd = C // heads
    y = y.view(B, -1, C)
    yqk = yqk.view(B, -1, Cqk)
    pe = linear_pos_embedding_sine(coords_grid(B, Hp, Wp, y).view(B, 2, -1).permute(0, 2, 1), dim=Cqk)
    q = _lin(sd, a + ".q", yqk + pe).reshape(B, Hp * Wp, heads, hd).permute(0, 2, 1, 3)
    ys = F.conv2d(y.permute(0, 2, 1).reshape(B, C, Hp, Wp), sd[a + ".sr_value.weight"], sd[a + ".sr_value.bias"], stride=sr)
    yk = F.conv2d(yqk.permute(0, 2, 1).reshape(B, Cqk, Hp, Wp), sd[a + ".sr_key.weight"], sd[a + ".sr_key.bias"], stride=sr)
    ys = _ln(sd, a + ".norm", ys.reshape(B, C, -1).permute(0, 2, 1), 1e-5)
    yk = _ln(sd, a + ".norm", yk.reshape(B, C, -1).permute(0, 2, 1), 1e-5)
    pe2 = linear_pos_embedding_sine(coords_grid(B, Hp // sr, Wp // sr, y).view(B, 2, -1).permute(0, 2, 1) * sr, dim=C)
    k = _lin(sd, a + ".k", yk + pe2).reshape(B, -1, heads, hd).permute(0, 2, 1, 3)
    v = _lin(sd, a + ".v", ys).reshape(B, -1, heads, hd).permute(0, 2, 1, 3)
    att = torch.softmax(q @ k.transpose(-2, -1) * hd ** -0.5, -1)
    o = (att @ v).transpose(1, 2).reshape(B, Hp, Wp, C)[:, :H, :W].reshape(B, N, C)
    x = x + _lin(sd, a + ".proj", o)
    return _mlp_block_tail(sd, b, x)


def cost_patch_embed(sd, p, cost_maps, patch=8, dim=64):
    """PatchEmbed, LCF/encoder.py:30-99: three 6x6 stride-2 convs, patch-centre positional code, 1x1 ffn, LayerNorm."""
    B, _, H, W = cost_maps.shape
    x = F.pad(cost_maps, (0, (patch - W % patch) % patch, 0, (patch - H % patch) % patch))
    x = F.relu(F.conv2d(x, sd[p + ".proj.0.weight"], sd[p + ".proj.0.bias"], stride=2, padding=2))
    x = F.relu(F.conv2d(x, sd[p + ".proj.2.weight"], sd[p + ".proj.2.bias"], stride=2, padding=2))
    x = F.conv2d(x, sd[p + ".proj.4.weight"], sd[p + ".proj.4.bias"], stride=2, padding=2)
    size = x.shape[2:]
    pc = (coords_grid(B, *size, x) * patch + patch / 2).view(B, 2, -1).permute(0, 2, 1)
    pe = linear_pos_embedding_sine(pc, dim=dim).permute(0, 2, 1).view(B, -1, *size)
    x = torch.cat([x, pe], 1)
    x = F.conv2d(F.relu(F.conv2d(x, sd[p + ".ffn_with_coord.0.weight"], sd[p + ".ffn_with_coord.0.bias"])),
                 sd[p + ".ffn_with_coord.2.weight"], sd[p + ".ffn_with_coord.2.bias"])
    return _ln(sd, p + ".norm", x.flatten(2).transpose(1, 2), 1e-5), size


def _ffn(sd, p, x):
    return _lin(sd, p + ".ffn.3", F.gelu(_lin(sd, p + ".ffn.0", x)))


def cost_input_layer(sd, p, tokens):
    """input_layer: CrossAttentionLayer, LCF/encoder.py:275-343 (8 heads; the 8 latent queries are shared by every cost map).
    tokens (maps, n, 128) from cost_patch_embed -> (maps, 8, 128)"""
    il = p + ".input_layer"
    lat = sd[p + ".latent_tokens"]
    qn = _ln(sd, il + ".norm1", lat, 1e-5)
    o = mha(_lin(sd, il + ".q", qn), _lin(sd, il + ".k", tokens), _lin(sd, il + ".v", tokens), 8)
    x = lat + _lin(sd, il + ".proj", o)
    return x + _ffn(sd, il, _ln(sd, il + ".norm2", x, 1e-5))


def cost_perceiver_layer(sd, p, i, x, size, context):
    """Layer i of CostPerceiverEncoder's loop, LCF/encoder.py:477-492: the SelfAttentionLayer over the 8 latent tokens of every cost map
    (encoder.py:209-272), then the vertical Twins blocks over each token's map.  x (B*H1*W1, 8, 128) -> the same; context (B, 256, H1, W1)
    of the B pairs of one reference call (each block repeats it over the B*8 token maps)."""
    H1, W1 = size
    B = x.shape[0] // (H1 * W1)
    e = "%s.encoder_layers.%d" % (p, i)
    y = _ln(sd, e + ".norm1", x, 1e-5)
    o = mha(_lin(sd, e + ".q", y), _lin(sd, e + ".k", y), _lin(sd, e + ".v", y), 8)
    x = x + _lin(sd, e + ".proj", o)
    x = x + _ffn(sd, e, _ln(sd, e + ".norm2", x, 1e-5))
    x = x.view(B, H1 * W1, 8, -1).permute(0, 2, 1, 3).reshape(B * 8, H1 * W1, -1)                    # LCF/encoder.py:481-491
    v = "%s.vertical_encoder_layers.%d" % (p, i)
    x = vertical_local(sd, v + ".local_block", x, (H1, W1), context)
    x = vertical_global(sd, v + ".global_block", x, (H1, W1), context)
    return x.view(B, 8, H1 * W1, -1).permute(0, 2, 1, 3).reshape(B * H1 * W1, 8, -1)


def cost_perceiver_encoder(sd, p, cost_volume, context, taps=None):
    """CostPerceiverEncoder.forward, LCF/encoder.py:450-495.  cost_volume (B,1,H1,W1,H2,W2) -> cost memory (B*H1*W1, 8, 128)."""
    B, heads, H1, W1, H2, W2 = cost_volume.shape
    cost_maps = cost_volume.permute(0, 2, 3, 1, 4, 5).contiguous().view(B * H1 * W1, heads, H2, W2)
    x, size = cost_patch_embed(sd, p + ".patch_embed", cost_maps)
    if taps is not None:
        taps["patch_tokens"] = x
    x = cost_input_layer(sd, p, x)
    short_cut = x
    if taps is not None:
        taps["latent_in"] = x
    for i in range(3):
        x = cost_perceiver_layer(sd, p, i, x, (H1, W1), context)
        if taps is not None:
            taps["latent_%d" % i] = x
    return x + short_cut, cost_maps, size


def memory_encoder(sd, img1, img2, context, taps=None):
    """MemoryEncoder.forward, LCF/encoder.py:509-539: Twins on both frames, 1x1 channel_convertor, all-pairs dot products (no scale)."""
    p = P + "memory_encoder"
    feats = twins_svt(sd, p + ".feat_encoder", torch.cat([img1, img2], 0))[1]
    feats = F.conv2d(feats, sd[p + ".channel_convertor.weight"])
    B = feats.shape[0] // 2
    fs, ft = feats[:B], feats[B:]
    _, C, H, W = fs.shape
    corr = torch.einsum("bid,bjd->bij", fs.flatten(2).transpose(1, 2), ft.flatten(2).transpose(1, 2)).view(B, 1, H, W, H, W)
    mem, cost_maps, size = cost_perceiver_encoder(sd, p + ".cost_perceiver_encoder", corr, context, taps)
    return mem, cost_maps, size, fs


# ---------------------------------------------------------------------------------------------------------------------------
# Memory decoder (LCF/decoder.py, gru.py, gma.py)
# ---------------------------------------------------------------------------------------------------------------------------
def encode_flow_token(cost_maps, coords):
    """LCF/decoder.py:233-252: 9x9 bilinear window around coords in each pixel's own cost map (x + dy[i], y + dx[j]: the transposed window)."""
    coords = coords.permute(0, 2, 3, 1)
    b, h1, w1, _ = coords.shape
    d = torch.linspace(-4, 4, 9, dtype=coords.dtype, device=coords.device)
    delta = torch.stack(torch.meshgrid(d, d, indexing="ij"), -1).view(1, 9, 9, 2)
    corr = bilinear_sampler(cost_maps, coords.reshape(b * h1 * w1, 1, 1, 2) + delta)
    return corr.view(b, h1, w1, -1).permute(0, 3, 1, 2)


def _conv(sd, k, x, pad=0):
    return F.conv2d(x, sd[k + ".weight"], sd.get(k + ".bias"), padding=pad)


def motion_encoder(sd, u, corr, flow):
    """BasicMotionEncoder, LCF/gru.py:75-97: corr (B,145,h,w), flow (B,2,h,w) -> motion features | flow (B,128,h,w)"""
    e = u + ".encoder"
    cor = F.relu(_conv(sd, e + ".convc2", F.relu(_conv(sd, e + ".convc1", corr)), 1))
    flo = F.relu(_conv(sd, e + ".convf2", F.relu(_conv(sd, e + ".convf1", flow, 3)), 1))
    return torch.cat([F.relu(_conv(sd, e + ".conv", torch.cat([cor, flo], 1), 1)), flow], 1)


def aggregate(sd, u, mf, attention):
    """Aggregate, gma.py:84-115: mf + gamma * (attention @ to_v(mf)); attention (B,1,N,N)"""
    b, c, h, w = mf.shape
    v = _conv(sd, u + ".aggregator.to_v", mf).view(b, 1, c, h * w).transpose(2, 3)
    return mf + sd[u + ".aggregator.gamma"] * (attention @ v).transpose(2, 3).reshape(b, c, h, w)


def sep_conv_gru(sd, u, net, x):
    """SepConvGRU, LCF/gru.py:35-73: net (B,128,h,w), x = [inp | mf | mg] (B,384,h,w)"""
    g = u + ".gru"
    for s, pad in (("1", (0, 2)), ("2", (2, 0))):
        hx = torch.cat([net, x], 1)
        z = torch.sigmoid(_conv(sd, g + ".convz" + s, hx, pad))
        r = torch.sigmoid(_conv(sd, g + ".convr" + s, hx, pad))
        q = torch.tanh(_conv(sd, g + ".convq" + s, torch.cat([r * net, x], 1), pad))
        net = (1 - z) * net + z * q
    return net


def flow_head(sd, u, net):
    return _conv(sd, u + ".flow_head.conv2", F.relu(_conv(sd, u + ".flow_head.conv1", net, 1)), 1)


def mask_head(sd, u, net):
    """0.25 * mask(net), LCF/gru.py:158"""
    return 0.25 * _conv(sd, u + ".mask.2", F.relu(_conv(sd, u + ".mask.0", net, 1)))


def gma_update_block(sd, u, net, inp, corr, flow, attention, last):
    """GMAUpdateBlock.forward, LCF/gru.py:130-160 (+ BasicMotionEncoder :75-97, Aggregate gma.py:84-115, SepConvGRU :35-73)."""
    mf = motion_encoder(sd, u, corr, flow)
    mg = aggregate(sd, u, mf, attention)
    net = sep_conv_gru(sd, u, net, torch.cat([inp, mf, mg], 1))
    return net, (mask_head(sd, u, net) if last else None), flow_head(sd, u, net)


def upsample_flow(flow, mask):
    """LCF/decoder.py:220-231"""
    N, _, H, W = flow.shape
    mask = torch.softmax(mask.view(N, 1, 9, 8, 8, H, W), 2)
    up = F.unfold(8 * flow, [3, 3], padding=1).view(N, 2, 9, 1, 1, H, W)
    return torch.sum(mask * up, 2).permute(0, 1, 4, 2, 5, 3).reshape(N, 2, 8 * H, 8 * W)


def gma_attention(sd, inp):
    """Attention, gma.py:56-76 (its positional term is disabled there): softmax(q k^T / sqrt(128)) of to_qk(inp) -> (B,1,N,N)"""
    qk = _conv(sd, P + "memory_decoder.att.to_qk", inp)
    q, k = qk[:, :128].flatten(2).transpose(1, 2) * 128 ** -0.5, qk[:, 128:].flatten(2).transpose(1, 2)
    return torch.softmax(q @ k.transpose(1, 2), -1)[:, None]


def cost_global(sd, cost_forward, coords1, key, value):
    """flow_token_encoder + the decoder's CrossAttentionLayer (LCF/decoder.py:81-117, :295-305) for one query per pixel against its 8
    memory tokens: cost_forward (B,81,h,w), key / value (B*h*w, 8, 64) -> cost_global (B,64,h,w)"""
    p = P + "memory_decoder"
    ca = p + ".decoder_layer.cross_attend"
    B, _, H1, W1 = cost_forward.shape
    query = _conv(sd, p + ".flow_token_encoder.2", F.gelu(_conv(sd, p + ".flow_token_encoder.0", cost_forward)))
    query = query.permute(0, 2, 3, 1).contiguous().view(B * H1 * W1, 1, 64)
    qc = coords1.reshape(B, 2, -1).permute(0, 2, 1).reshape(B * H1 * W1, 1, 2)
    pe = linear_pos_embedding_sine(qc, dim=64)
    y = _ln(sd, ca + ".norm1", query, 1e-5)
    o = mha(_lin(sd, ca + ".q", y + pe), key, value, 8)
    x = query + _lin(sd, ca + ".proj", torch.cat([o, query], 2))
    x = x + _ffn(sd, ca, _ln(sd, ca + ".norm2", x, 1e-5))
    return x.view(B, H1, W1, 64).permute(0, 3, 1, 2)


def decoder_iteration(sd, net, inp, coords0, coords1, cost_maps, key, value, attention, last):
    """One iteration of MemoryDecoder.forward's loop, LCF/decoder.py:290-319 -> (net, the flow update, mask (last only), corr)"""
    cost_forward = encode_flow_token(cost_maps, coords1)
    corr = torch.cat([cost_global(sd, cost_forward, coords1, key, value), cost_forward], 1)
    net, up_mask, dflow = gma_update_block(sd, P + "memory_decoder.update_block", net, inp, corr, coords1 - coords0, attention, last)
    return net, dflow, up_mask, corr


def memory_decoder(sd, cost_memory, context, cost_maps, iters=32, taps=None):
    """MemoryDecoder.forward, LCF/decoder.py:254-321 (only the last iteration's up-sampled flow is returned / needed)."""
    p = P + "memory_decoder"
    B, _, H1, W1 = context.shape
    coords0 = coords_grid(B, H1, W1, context)
    coords1 = coords_grid(B, H1, W1, context)
    ctx = _conv(sd, p + ".proj", context)
    net, inp = torch.tanh(ctx[:, :128]), torch.relu(ctx[:, 128:])
    attention = gma_attention(sd, inp)
    ca = p + ".decoder_layer.cross_attend"
    key, value = _lin(sd, ca + ".k", cost_memory), _lin(sd, ca + ".v", cost_memory)                 # computed in iteration 0, re-used after
    flow_up = None
    for it in range(iters):
        net, dflow, up_mask, corr = decoder_iteration(sd, net, inp, coords0, coords1, cost_maps, key, value, attention, it == iters - 1)
        if taps is not None and it == 0:
            taps["dec_corr_0"] = corr
        coords1 = coords1 + dflow
        if taps is not None and it == 0:
            taps["dec_net_0"], taps["dec_dflow_0"] = net, dflow
        if up_mask is not None:
            flow_up = upsample_flow(coords1 - coords0, up_mask)
    return flow_up, coords1 - coords0


def flowformer_forward(sd, image1, image2, iters=32, taps=None):
    """FlowFormer.forward(image1, image2, return_feat=True), LCF/transformer.py:45-74.  Images in 0..255.
    -> (flow_up (B,2,H,W), flow_low (B,2,H/8,W/8)), cfeat [(B,128,H/4,W/4), (B,256,H/8,W/8)], ffeat (B,256,H/8,W/8)"""
    image1 = 2 * (image1 / 255.0) - 1.0
    image2 = 2 * (image2 / 255.0) - 1.0
    cfeat = twins_svt(sd, P + "context_encoder", image1)
    context = cfeat[1]
    mem, cost_maps, _, ffeat = memory_encoder(sd, image1, image2, context, taps)
    if taps is not None:
        taps["cost_memory"], taps["cost_maps"] = mem, cost_maps
    flows = memory_decoder(sd, mem, context, cost_maps, iters, taps)
    return flows, cfeat, ffeat
