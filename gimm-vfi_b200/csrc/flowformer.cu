// Native FlowFormer (LatentCostFormer) flow estimator of GIMM-VFI-F — SURVEY 8(a) row a24 / 8(f) row 1.
// Reference: flowformer/core/FlowFormer/LatentCostFormer/{transformer.py:45-74, encoder.py, decoder.py, gru.py, gma.py, twins.py,
// attention.py} + encoders.py:7-48, in the one configuration GIMM-VFI-F builds (configs/submission.py:19-50).
//
// Design (GPU-first, not a translation):
//  * a token sequence (B, H*W, C) IS an NHWC map, so every nn.Linear / MLP / 1x1 projection is a 1x1 convolution on the wgmma
//    implicit-GEMM kernel (conv_tc.cu, fp32-class 3xF16 form: the 32-iteration recurrence amplifies operand rounding like RAFT's);
//    stride-k patch / sub-sampling convolutions are space-to-depth + 1x1; GELU, residual adds and the GRU gates are conv epilogues;
//  * both flow directions and both frames run batched on the N axis: the feature Twins runs ONCE on [I0; I1] (the reference runs it
//    twice per direction = 4 times), direction 1's cost volume is the transposed GEMM of the same two feature maps;
//  * the 8 latent tokens of every cost map are stored token-major [(dir, sample, token)][h][w][128], so the "vertical" Twins blocks see
//    plain NHWC batches and the per-map attentions address the same buffer through strides (ops_tokens.cu strided_attention);
//  * the cost-map patch embedding (8704 maps of 68x128 at the 2K / 4K settings) streams over chunks of maps: 6x6 stride-2 layers as
//    x-packed tensor-core convolutions on pre-padded buffers, never more than ~1 GB of temporaries alive;
//  * GMA: the N x N attention matrix is built once per pair (tensor-core GEMM + row softmax, stored pre-scaled by a power of two) and
//    the per-iteration aggregate attn @ v is a tensor-core GEMM with v^T as the K-major operand.
#include "engine.h"
#include "net.h"

#include <algorithm>

namespace gv {

static const char* const FE = "flow_estimator.";

// ---------------------------------------------------------------------------------------------------------------------------
// weights
// ---------------------------------------------------------------------------------------------------------------------------
// k x k stride-k Conv2d (cout, cin, k, k) -> Linear over the space-to-depth channels (ky*k + kx)*cin + ci, stored as "<name>#p"
void Engine::pack_patch_conv(const std::string& name) {
  const HostTensor& W = raw(name + ".weight");
  const int cout = (int)W.shape[0], cin = (int)W.shape[1], k = (int)W.shape[2];
  if (W.shape.size() != 4 || W.shape[3] != k) throw std::runtime_error("pack_patch_conv: expected a square kernel");
  HostTensor L; L.shape = {cout, (int64_t)k * k * cin}; L.data.resize((size_t)cout * k * k * cin);
  for (int co = 0; co < cout; ++co)
    for (int ci = 0; ci < cin; ++ci)
      for (int t = 0; t < k * k; ++t) L.data[((size_t)co * k * k + t) * cin + ci] = W.data[((size_t)co * cin + ci) * k * k + t];
  raw_[name + "#p.weight"] = L;
  raw_[name + "#p.bias"] = raw(name + ".bias");
  pack_conv(name + "#p");
}

void Engine::pack_twins(const std::string& p) {
  for (int i = 0; i < 2; ++i) {
    const std::string pe = p + ".svt.patch_embeds." + std::to_string(i);
    pack_patch_conv(pe + ".proj"); vec(pe + ".norm.weight"); vec(pe + ".norm.bias");
    for (int j = 0; j < 2; ++j) {
      const std::string b = p + ".svt.blocks." + std::to_string(i) + "." + std::to_string(j);
      for (const char* n : {".norm1", ".norm2"}) { vec(b + n + ".weight"); vec(b + n + ".bias"); }
      if (j == 0) pack_conv(b + ".attn.qkv");
      else { pack_conv(b + ".attn.q"); pack_conv(b + ".attn.kv"); pack_patch_conv(b + ".attn.sr"); vec(b + ".attn.norm.weight"); vec(b + ".attn.norm.bias"); }
      pack_conv(b + ".attn.proj"); pack_conv(b + ".mlp.fc1"); pack_conv(b + ".mlp.fc2");
    }
    // PosConv: depthwise (C,1,3,3) -> [9][C]
    const std::string pw = p + ".svt.pos_block." + std::to_string(i) + ".proj.0";
    const HostTensor& W = raw(pw + ".weight");
    const int C = (int)W.shape[0];
    std::vector<float> w9((size_t)9 * C);
    for (int c = 0; c < C; ++c) for (int t = 0; t < 9; ++t) w9[(size_t)t * C + c] = W.data[(size_t)c * 9 + t];
    vec_[pw + ".weight#9c"] = upload(w9); vec(pw + ".bias");
  }
}

void Engine::finalize_flowformer() {
  const std::string me = std::string(FE) + "memory_encoder", md = std::string(FE) + "memory_decoder";
  pack_twins(me + ".feat_encoder");
  pack_twins(std::string(FE) + "context_encoder");
  pack_conv(me + ".channel_convertor");
  const std::string cp = me + ".cost_perceiver_encoder";
  {
    // first patch-embedding layer (1 -> 16, 6x6): [36][16] for cost_conv1; the next two as x-packed 6x1 kernels over 6 * cin lanes
    const HostTensor& W = raw(cp + ".patch_embed.proj.0.weight");
    if (W.shape[0] != 16 || W.shape[1] != 1 || W.shape[2] != 6) throw std::runtime_error("flowformer: unexpected cost patch embedding");
    std::vector<float> w((size_t)36 * 16);
    for (int co = 0; co < 16; ++co) for (int t = 0; t < 36; ++t) w[(size_t)t * 16 + co] = W.data[(size_t)co * 36 + t];
    ff_c1w_ = w; ff_c1b_ = raw(cp + ".patch_embed.proj.0.bias").data;   // kept on the host: cost_conv1 passes them in its kernel parameter block
    pack_xpacked(cp + ".patch_embed.proj.2", 16); pack_xpacked(cp + ".patch_embed.proj.4", 32);
    pack_conv(cp + ".patch_embed.ffn_with_coord.0"); pack_conv(cp + ".patch_embed.ffn_with_coord.2");
    vec(cp + ".patch_embed.norm.weight"); vec(cp + ".patch_embed.norm.bias");
  }
  vec(cp + ".latent_tokens");
  auto pack_attn_layer = [&](const std::string& l) {   // CrossAttentionLayer / SelfAttentionLayer (encoder.py:209-343, decoder.py:34-117)
    for (const char* n : {".norm1", ".norm2"}) { vec(l + n + ".weight"); vec(l + n + ".bias"); }
    for (const char* n : {".q", ".k", ".v", ".proj", ".ffn.0", ".ffn.3"}) pack_conv(l + n);
  };
  pack_attn_layer(cp + ".input_layer");
  for (int i = 0; i < 3; ++i) {
    pack_attn_layer(cp + ".encoder_layers." + std::to_string(i));
    for (const char* blk : {".local_block", ".global_block"}) {
      const std::string b = cp + ".vertical_encoder_layers." + std::to_string(i) + blk;
      for (const char* n : {".norm1", ".norm2"}) { vec(b + n + ".weight"); vec(b + n + ".bias"); }
      for (const char* n : {".attn.context_proj", ".attn.q", ".attn.k", ".attn.v", ".attn.proj", ".mlp.fc1", ".mlp.fc2"}) pack_conv(b + n);
      if (std::string(blk) == ".global_block") {
        pack_patch_conv(b + ".attn.sr_key"); pack_patch_conv(b + ".attn.sr_value");
        vec(b + ".attn.norm.weight"); vec(b + ".attn.norm.bias");
      }
    }
  }
  // memory decoder
  pack_conv(md + ".flow_token_encoder.0"); pack_conv(md + ".flow_token_encoder.2"); pack_conv(md + ".proj");
  pack_attn_layer(md + ".decoder_layer.cross_attend");
  pack_conv(md + ".att.to_qk");
  const std::string u = md + ".update_block";
  for (const char* n : {".encoder.convc1", ".encoder.convc2", ".encoder.convf1", ".encoder.convf2", ".encoder.conv", ".gru.convz1", ".gru.convr1",
                        ".gru.convq1", ".gru.convz2", ".gru.convr2", ".gru.convq2", ".flow_head.conv1", ".flow_head.conv2", ".mask.0", ".aggregator.to_v"})
    pack_conv(u + n);
  for (const char* sfx : {"1", "2"}) {   // z | r gates read the same input: one 512 -> 256 convolution (gru.py:56-58,64-66)
    const HostTensor& wz = raw(u + ".gru.convz" + sfx + ".weight"); const HostTensor& wr = raw(u + ".gru.convr" + sfx + ".weight");
    const HostTensor& bz = raw(u + ".gru.convz" + sfx + ".bias"); const HostTensor& br = raw(u + ".gru.convr" + sfx + ".bias");
    HostTensor w = wz, b = bz;
    w.shape[0] = wz.shape[0] + wr.shape[0]; w.data.insert(w.data.end(), wr.data.begin(), wr.data.end());
    b.shape[0] = bz.shape[0] + br.shape[0]; b.data.insert(b.data.end(), br.data.begin(), br.data.end());
    raw_[u + ".gru.convzr" + sfx + ".weight"] = w; raw_[u + ".gru.convzr" + sfx + ".bias"] = b;
    pack_conv(u + ".gru.convzr" + sfx);
    // The GRU input is [h | inp | mf | mg] (gru.py:147-151) and `inp` (the context half, decoder.py:270-273) does not change over the 32
    // iterations: its share of every gate convolution is computed once per pair ("_inp", carries the bias) and enters the per-iteration
    // convolutions over [h | mf | mg] ("_hm", K = 384 instead of 512) as a pre-activation term - the scheme of RAFT's update block (engine.cu).
    for (const char* gate : {"zr", "q"}) {
      const std::string g = u + ".gru.conv" + gate + sfx;
      const HostTensor& wf = raw(g + ".weight"); const HostTensor& bf = raw(g + ".bias");
      const int64_t co = wf.shape[0], ci = wf.shape[1], kk = wf.shape[2] * wf.shape[3];
      if (ci != 512) throw std::runtime_error("flowformer: SepConvGRU input width");
      HostTensor w_hm, w_in, b0 = bf;
      w_hm.shape = {co, 384, wf.shape[2], wf.shape[3]}; w_in.shape = {co, 128, wf.shape[2], wf.shape[3]};
      for (int64_t o = 0; o < co; ++o)
        for (int64_t c = 0; c < ci; ++c) {
          std::vector<float>& dst = (c >= 128 && c < 256) ? w_in.data : w_hm.data;
          dst.insert(dst.end(), wf.data.begin() + (o * ci + c) * kk, wf.data.begin() + (o * ci + c + 1) * kk);
        }
      std::fill(b0.data.begin(), b0.data.end(), 0.f);
      raw_[g + "_hm.weight"] = w_hm; raw_[g + "_hm.bias"] = b0;
      raw_[g + "_inp.weight"] = w_in; raw_[g + "_inp.bias"] = bf;
      pack_conv(g + "_hm"); pack_conv(g + "_inp");
    }
  }
  pack_conv(u + ".mask.2", "", 0.25f);   // mask = 0.25 * self.mask(net)  (gru.py:158)
  pack_xpacked(u + ".encoder.convf1", 4);
  vec(u + ".aggregator.gamma");
}

// ---------------------------------------------------------------------------------------------------------------------------
// forward pieces
// ---------------------------------------------------------------------------------------------------------------------------
namespace {

struct FF {
  Engine& E; Net& N; Ctx& cx; Arena& A;
  const float* V(const std::string& n) const { return N.V(n); }
  void ln(const std::string& name, const TV& x, const TV& out, float eps, float pe_scale = 0.f, int pe_dim = 0) {
    layernorm(cx, x, V(name + ".weight"), V(name + ".bias"), eps, out, pe_scale, pe_dim);
  }
  // 1x1 convolutions see a token map of arbitrary shape as rows of 16-pixel lines: a flat view keeps the 16 x 8 tiles of conv_tc full
  static TV flat(const TV& t) {
    if (t.sn != (int64_t)t.h * t.w * t.ld) return t;   // (not dense over the batch: leave as is)
    const int64_t px = t.pixels();
    int wv = 16;
    while (wv > 1 && px % wv) wv >>= 1;
    TV f = t; f.n = 1; f.w = wv; f.h = (int)(px / wv); f.sn = px * t.ld;
    return f;
  }
  void lin(const std::string& name, const TV& in, const TV& out, int act = ACT_NONE) { N.conv(name, flat(in), flat(out), act); }
  void lin_res(const std::string& name, const TV& in0, const TV& in1, const TV& res, const TV& out) {
    ConvEpi e; e.res = flat(res);
    N.conv_e(name, flat(in0), in1.p ? flat(in1) : TV(), flat(out), e);
  }
  // x + mlp(norm2(x)): Linear -> GELU -> Linear (timm Mlp; encoder.py:261-266 for the ffn form), result in `out` (may alias nothing)
  void mlp(const std::string& norm, float eps, const std::string& fc1, const std::string& fc2, const TV& x, const TV& out) {
    const size_t mk = A.mark();
    const int hidden = N.W(fc1).cout;
    TV y = A.tensor(x.n, x.h, x.w, x.c), hdn = A.tensor(x.n, x.h, x.w, hidden);
    ln(norm, x, y, eps);
    lin(fc1, y, hdn, ACT_GELU);
    lin_res(fc2, hdn, TV(), x, out);
    A.release(mk);
  }

  // ------------------------------------------------------------------ Twins-SVT-L stages 1-2 (encoders.py:22-45)
  // img (n,H,W,3) in [-1,1] -> f4 (n,H/4,W/4,128), f8 (n,H/8,W/8,256)
  void twins(const std::string& p, const TV& img, const TV& f4, const TV& f8) {
    const size_t mk0 = A.mark();
    TV cur = img;
    const int n = img.n;
    for (int i = 0; i < 2; ++i) {
      const int patch = i == 0 ? 4 : 2, C = i == 0 ? 128 : 256, heads = i == 0 ? 4 : 8, sr = i == 0 ? 8 : 4, ws = 7;
      const int H = cur.h / patch, W = cur.w / patch;
      const TV& stage_out = i == 0 ? f4 : f8;
      const std::string pe = p + ".svt.patch_embeds." + std::to_string(i);
      TV xa = A.tensor(n, H, W, C), xb = A.tensor(n, H, W, C);
      {
        const size_t mk = A.mark();
        TV pt = A.tensor(n, H, W, patch * patch * cur.c), t0 = A.tensor(n, H, W, C);
        patchify(cx, cur, pt, patch);
        lin(pe + ".proj#p", pt, t0);
        ln(pe + ".norm", t0, xa, 1e-5f);
        A.release(mk);
      }
      // block 0: locally-grouped attention (twins.py:814-867), zero padding after the norm
      {
        const std::string b = p + ".svt.blocks." + std::to_string(i) + ".0";
        const size_t mk = A.mark();
        const int Hp = (H + ws - 1) / ws * ws, Wp = (W + ws - 1) / ws * ws;
        TV yp = A.tensor(n, Hp, Wp, C), qkv = A.tensor(n, Hp, Wp, 3 * C), o = A.tensor(n, H, W, C);
        ln(b + ".norm1", xa, yp, 1e-6f);
        lin(b + ".attn.qkv", yp, qkv);
        window_attention(cx, qkv.slice(0, C), qkv.slice(C, C), qkv.slice(2 * C, C), o, heads, ws);
        lin_res(b + ".attn.proj", o, TV(), xa, xb);
        A.release(mk);
        mlp(b + ".norm2", 1e-6f, b + ".mlp.fc1", b + ".mlp.fc2", xb, xa);
        const std::string pw = p + ".svt.pos_block." + std::to_string(i) + ".proj.0";
        dwconv3x3_residual(cx, xa, V(pw + ".weight#9c"), V(pw + ".bias"), xb);   // PEG after the first block (encoders.py:39-40)
      }
      // block 1: global sub-sampled attention (twins.py:870-925)
      {
        const std::string b = p + ".svt.blocks." + std::to_string(i) + ".1";
        const size_t mk = A.mark();
        if (H % sr || W % sr) throw std::runtime_error("gimmvfi: FlowFormer needs a network resolution that is a multiple of 32");
        const int hk = H / sr, wk = W / sr;
        TV y = A.tensor(n, H, W, C), q = A.tensor(n, H, W, C), ys = A.tensor(n, hk, wk, sr * sr * C), s = A.tensor(n, hk, wk, C),
           sn = A.tensor(n, hk, wk, C), kv = A.tensor(n, hk, wk, 2 * C), o = A.tensor(n, H, W, C);
        ln(b + ".norm1", xb, y, 1e-6f);
        lin(b + ".attn.q", y, q);
        patchify(cx, y, ys, sr);
        lin(b + ".attn.sr#p", ys, s);
        ln(b + ".attn.norm", s, sn, 1e-5f);
        lin(b + ".attn.kv", sn, kv);
        AttnDims a{};
        a.nb1 = n; a.nb2 = 1; a.nq = (int64_t)H * W; a.nk = (int64_t)hk * wk; a.heads = heads;
        a.q_s1 = q.sn; a.q_si = q.ld; a.k_s1 = kv.sn; a.k_sj = kv.ld; a.v_s1 = kv.sn; a.v_sj = kv.ld; a.o_s1 = o.sn; a.o_si = o.ld;
        strided_attention(cx, q.p, kv.p, kv.p + C, o.p, a, C / heads);
        lin_res(b + ".attn.proj", o, TV(), xb, xa);
        A.release(mk);
        mlp(b + ".norm2", 1e-6f, b + ".mlp.fc1", b + ".mlp.fc2", xa, stage_out);
      }
      cur = stage_out;
    }
    A.release(mk0);
  }

  // ------------------------------------------------------------------ vertical Twins blocks over the latent maps (encoder.py:150-196)
  // x: (nb = S*8, h, w, 128) token-major latent maps, in place.  ctx8: (S, h, w, 256) in pair order; the pairs form reference calls of
  // `per_call` pairs each, and sample n reads the context the reference's context.repeat(...) hands it within its call (ops_tokens.cu
  // concat_pe): with per_call > 1 a token may read another pair's context, as in the reference.
  void vertical_local(const std::string& b, const TV& x, const TV& ctx8, int per_call) {
    const size_t mk = A.mark();
    const int n = x.n, H = x.h, W = x.w, C = 128, ws = 7, heads = 8;
    const int Hp = (H + ws - 1) / ws * ws, Wp = (W + ws - 1) / ws * ws;
    TV ctxp = A.tensor(ctx8.n, H, W, 64), yp = A.tensor(n, Hp, Wp, C), xqk = A.tensor(n, Hp, Wp, C + 64);
    TV q = A.tensor(n, Hp, Wp, C), k = A.tensor(n, Hp, Wp, C), v = A.tensor(n, Hp, Wp, C), o = A.tensor(n, H, W, C), x2 = A.tensor(n, H, W, C);
    lin(b + ".attn.context_proj", ctx8, ctxp);
    ln(b + ".norm1", x, yp, 1e-5f);
    concat_pe(cx, yp, ctxp, xqk, ws, true, per_call * 8, per_call);
    lin(b + ".attn.q", xqk, q); lin(b + ".attn.k", xqk, k); lin(b + ".attn.v", yp, v);
    window_attention(cx, q, k, v, o, heads, ws);
    lin_res(b + ".attn.proj", o, TV(), x, x2);
    mlp(b + ".norm2", 1e-5f, b + ".mlp.fc1", b + ".mlp.fc2", x2, x);
    A.release(mk);
  }
  void vertical_global(const std::string& b, const TV& x, const TV& ctx8, int per_call) {
    const size_t mk = A.mark();
    const int n = x.n, H = x.h, W = x.w, C = 128, sr = 4, heads = 8;
    if (H % sr || W % sr) throw std::runtime_error("gimmvfi: FlowFormer needs a network resolution that is a multiple of 32");
    const int hk = H / sr, wk = W / sr;
    TV ctxp = A.tensor(ctx8.n, H, W, 64), y = A.tensor(n, H, W, C), xqk = A.tensor(n, H, W, C + 64), xqp = A.tensor(n, H, W, C + 64);
    TV q = A.tensor(n, H, W, C), o = A.tensor(n, H, W, C), x2 = A.tensor(n, H, W, C);
    TV pk = A.tensor(n, hk, wk, sr * sr * (C + 64)), pv = A.tensor(n, hk, wk, sr * sr * C);
    TV sk = A.tensor(n, hk, wk, C), sv = A.tensor(n, hk, wk, C), skn = A.tensor(n, hk, wk, C), svn = A.tensor(n, hk, wk, C);
    TV k = A.tensor(n, hk, wk, C), v = A.tensor(n, hk, wk, C);
    lin(b + ".attn.context_proj", ctx8, ctxp);
    ln(b + ".norm1", x, y, 1e-5f);
    concat_pe(cx, y, ctxp, xqk, 0, false, per_call * 8, per_call);
    concat_pe(cx, y, ctxp, xqp, 0, true, per_call * 8, per_call);        // + code of the absolute position (twins.py:486-492)
    lin(b + ".attn.q", xqp, q);
    patchify(cx, xqk, pk, sr); lin(b + ".attn.sr_key#p", pk, sk);
    patchify(cx, y, pv, sr); lin(b + ".attn.sr_value#p", pv, sv);
    ln(b + ".attn.norm", sk, skn, 1e-5f, (float)sr, C);      // norm, then + code of coords * sr (twins.py:494-513)
    ln(b + ".attn.norm", sv, svn, 1e-5f);
    lin(b + ".attn.k", skn, k); lin(b + ".attn.v", svn, v);
    AttnDims a{};
    a.nb1 = n; a.nb2 = 1; a.nq = (int64_t)H * W; a.nk = (int64_t)hk * wk; a.heads = heads;
    a.q_s1 = q.sn; a.q_si = q.ld; a.k_s1 = k.sn; a.k_sj = k.ld; a.v_s1 = v.sn; a.v_sj = v.ld; a.o_s1 = o.sn; a.o_si = o.ld;
    strided_attention(cx, q.p, k.p, v.p, o.p, a, C / heads);
    lin_res(b + ".attn.proj", o, TV(), x, x2);
    mlp(b + ".norm2", 1e-5f, b + ".mlp.fc1", b + ".mlp.fc2", x2, x);
    A.release(mk);
  }

  // ------------------------------------------------------------------ all-pairs cost volume (encoder.py:507-522): no 1/sqrt(d) here
  // vol[s][i][j] = <F[src[s],i], F[tgt[s],j]> for every pair s
  void cost_volume(const TV& F, const std::vector<int>& src, const std::vector<int>& tgt, float* vol) {
    const int64_t Npx = (int64_t)F.h * F.w;
    const int S = (int)src.size();
    if (cx.tc && F.c % 64 == 0 && F.ld == F.c && corr_volume_tc_wants_f16_planes()) {   // every frame split once
      const size_t mk = A.mark();
      const int64_t plane = F.n * Npx * F.c;
      uint16_t* pl = reinterpret_cast<uint16_t*>(A.alloc_f((size_t)plane));
      split_planes_f16(cx, F, pl);
      for (int s = 0; s < S; ++s)
        if (!cx.dry) corr_gemm_3xf16(cx, pl + src[s] * Npx * F.c, plane, (int)Npx, pl + tgt[s] * Npx * F.c, plane, (int)Npx, F.c, 1.0f, vol + (int64_t)s * Npx * Npx);
      A.release(mk);
    } else if (cx.tc && F.c % 64 == 0 && F.ld == F.c) {
      const size_t mk = A.mark();
      float* planes = A.alloc_f((size_t)2 * Npx * F.c);
      const int64_t nz = ((Npx + 255) / 256) * 256 + 512;
      float* zeros = A.alloc_f((size_t)nz);
      if (!cx.dry) dev_memset(zeros, 0, (size_t)nz * sizeof(float), cx.stream);
      for (int s = 0; s < S; ++s) {
        if (corr_volume_tc_wants_f16_planes()) split_planes_f16(cx, F.batch(tgt[s], 1), planes);
        else split_planes(cx, F.batch(tgt[s], 1), planes);
        if (!cx.dry) corr_volume_tc(cx, F.batch(src[s], 1), planes, zeros, vol + (int64_t)s * Npx * Npx, 1.0f, true, (int)Npx);
      }
      A.release(mk);
    } else {
      for (int s = 0; s < S; ++s) corr_volume(cx, F.batch(src[s], 1), F.batch(tgt[s], 1), vol + (int64_t)s * Npx * Npx, 1.0f);
    }
  }

  // ------------------------------------------------------------------ CostPerceiverEncoder (encoder.py:450-495)
  // vol: [S][N][N]; latent: (S*8, h, w, 128) token-major (output: the cost memory)
  void cost_perceiver(const std::string& p, int S, int per_call, const float* vol, int h, int w, const TV& ctx8, const TV& latent) {
    const size_t mk0 = A.mark();
    const int64_t Npx = (int64_t)h * w;
    const int Hpad = (h + 7) / 8 * 8, Wpad = (w + 7) / 8 * 8;          // F.pad to a multiple of patch_size (encoder.py:68-71)
    const int oh1 = Hpad / 2, ow1 = Wpad / 2, oh2 = oh1 / 2, ow2 = ow1 / 2, oh3 = oh2 / 2, ow3 = ow2 / 2;
    const std::string pe = p + ".patch_embed", il = p + ".input_layer";
    TV att = A.tensor(S * 8, h, w, 128);      // input-layer attention output, token-major
    // the 8 latent queries are shared by every cost map (BroadMultiHeadAttention, attention.py:10-34)
    TV lat1 = make_tv(const_cast<float*>(V(p + ".latent_tokens")), 1, 1, 8, 128), qn = A.tensor(1, 1, 8, 128), q8 = A.tensor(1, 1, 8, 128);
    ln(il + ".norm1", lat1, qn, 1e-5f);
    N.conv(il + ".q", qn, q8);
    // stream the cost maps through the patch embedding in chunks (per direction-sample): bounded temporaries at any resolution
    const size_t per_map = ((size_t)(oh1 + 4) * (ow1 + 4) * 16 + (size_t)oh2 * ow2 * 32 + (size_t)(oh2 + 4) * (ow2 + 4) * 32 + (size_t)oh3 * ow3 * 128 * 5) * 4;
    int64_t chunk = std::max<int64_t>(1, (int64_t)(size_t(1) << 30) / (int64_t)per_map);
    if (chunk > Npx) chunk = Npx;
    const ConvW& w2 = N.W(pe + ".proj.2#xp"); const ConvW& w4 = N.W(pe + ".proj.4#xp");
    for (int s = 0; s < S; ++s)
      for (int64_t p0 = 0; p0 < Npx; p0 += chunk) {
        const size_t mk = A.mark();
        const int cm = (int)std::min<int64_t>(chunk, Npx - p0);
        TV c1 = A.tensor(cm, oh1 + 4, ow1 + 4, 16), c2 = A.tensor(cm, oh2, ow2, 32), c2p = A.tensor(cm, oh2 + 4, ow2 + 4, 32);
        TV xpe = A.tensor(cm, oh3, ow3, 128), t1 = A.tensor(cm, oh3, ow3, 128), t2 = A.tensor(cm, oh3, ow3, 128);
        TV kk = A.tensor(cm, oh3, ow3, 128), vv = A.tensor(cm, oh3, ow3, 128);
        cost_conv1(cx, vol + ((int64_t)s * Npx + p0) * Npx, cm, h, w, E.ff_c1w(), E.ff_c1b(), c1, oh1, ow1);
        ConvGeom g; g.stride = 2; g.ph = 0; g.pw = 0; g.loose_w = 1;   // pre-padded inputs: the taps index the buffer directly
        { TV v1 = c1; v1.c = w2.cin; ConvEpi e; e.act1 = ACT_RELU; conv2d(cx, v1, TV(), w2, g, e, c2); }
        pad_zero(cx, c2, c2p, 2);
        { TV v2 = c2p; v2.c = w4.cin; ConvEpi e; conv2d(cx, v2, TV(), w4, g, e, xpe.slice(0, 64)); }
        write_pe(cx, xpe.slice(64, 64), 8.f, 4.f);                       // patch centres, encoder.py:76-89
        lin(pe + ".ffn_with_coord.0", xpe, t1, ACT_RELU);
        lin(pe + ".ffn_with_coord.2", t1, t2);
        ln(pe + ".norm", t2, t1, 1e-5f);
        lin(il + ".k", t1, kk); lin(il + ".v", t1, vv);
        AttnDims a{};
        a.nb1 = 1; a.nb2 = cm; a.nq = 8; a.nk = (int64_t)oh3 * ow3; a.heads = 8;
        a.q_si = 128; a.k_s2 = kk.sn; a.k_sj = 128; a.v_s2 = vv.sn; a.v_sj = 128; a.o_s2 = 128; a.o_si = Npx * 128;
        strided_attention(cx, q8.p, kk.p, vv.p, att.p + ((int64_t)s * 8 * Npx + p0) * 128, a, 16);
        A.release(mk);
      }
    // x = latent_tokens + proj(attn); x = x + ffn(norm2(x))   (encoder.py:332-342)
    TV x = A.tensor(S * 8, h, w, 128), x2 = A.tensor(S * 8, h, w, 128), sc = A.tensor(S * 8, h, w, 128);
    broadcast_tokens(cx, V(p + ".latent_tokens"), x2, 8);
    lin_res(il + ".proj", att, TV(), x2, x);
    mlp(il + ".norm2", 1e-5f, il + ".ffn.0", il + ".ffn.3", x, sc);       // sc = short_cut (encoder.py:470)
    copy_channels(cx, sc, x);
    E.tap_pub("ff.latent_in", sc);                                        // (kept in debug mode: mk0 is not released then)
    for (int i = 0; i < 3; ++i) {
      const std::string e = p + ".encoder_layers." + std::to_string(i);
      {   // SelfAttentionLayer over the 8 tokens of every cost map (encoder.py:248-266)
        const size_t mk = A.mark();
        TV y = A.tensor(S * 8, h, w, 128), q = A.tensor(S * 8, h, w, 128), k = A.tensor(S * 8, h, w, 128), v = A.tensor(S * 8, h, w, 128), o = att;
        ln(e + ".norm1", x, y, 1e-5f);
        lin(e + ".q", y, q); lin(e + ".k", y, k); lin(e + ".v", y, v);
        AttnDims a{};
        a.nb1 = S; a.nb2 = Npx; a.nq = 8; a.nk = 8; a.heads = 8;
        a.q_s1 = a.k_s1 = a.v_s1 = a.o_s1 = 8 * Npx * 128; a.q_s2 = a.k_s2 = a.v_s2 = a.o_s2 = 128; a.q_si = a.k_sj = a.v_sj = a.o_si = Npx * 128;
        strided_attention(cx, q.p, k.p, v.p, o.p, a, 16);
        lin_res(e + ".proj", o, TV(), x, x2);
        A.release(mk);
        mlp(e + ".norm2", 1e-5f, e + ".ffn.0", e + ".ffn.3", x2, x);
      }
      const std::string vl = p + ".vertical_encoder_layers." + std::to_string(i);
      vertical_local(vl + ".local_block", x, ctx8, per_call);
      vertical_global(vl + ".global_block", x, ctx8, per_call);
      E.tap_copy(cx, "ff.latent_" + std::to_string(i), x);
    }
    axpby(cx, x, 1.f, sc, 1.f, latent);                                   // cost_encoder_res (encoder.py:493-494)
    if (!E.debug_on()) A.release(mk0);
  }
};

}  // namespace

// FlowFormer.forward (transformer.py:45-74) over a frame set and a list of (source, target) pairs, batched on the N axis:
// img (F,H,W,3 [ld 4]) in [-1,1]; pair s = (src[s], tgt[s]) -> flow_up (S,H,W,2) and, optionally, flow_low (S,H/8,W/8,2) = the last
// iteration's coords1 - coords0.  Consecutive pairs form reference calls of `per_call` pairs (the batch of one FlowFormer.forward;
// it decides which context the vertical Twins blocks read, see vertical_local).  The feature Twins + channel_convertor run once per
// frame (-> fproj, optional), the context Twins once per distinct source frame (-> feat4 / feat8 in first-use order, optional); the
// context is then gathered into pair order unless the sources are the frames in order, pair s from frame s (GIMM-VFI-F).
// flow_init (S,2,H/8,W/8) NCHW, optional, warm-starts coords1; `encoded` (optional) sees feat4 / feat8 / fproj once the encoders ran.
// gather: always take the gathering path (the planner's upper bound).  Memory per pair: the cost volume and the GMA attention matrix,
// N^2 floats each, N = (H/8)(W/8).
void Engine::run_flowformer(Ctx& cx, Net& N, const TV& img, const std::vector<int>& src, const std::vector<int>& tgt, int per_call, int iters,
                            bool gather, const TV& flow_up, const TV& flow_low, const TV& feat4_out, const TV& feat8_out, const TV& fproj_out,
                            const float* flow_init, const std::function<void(const TV&, const TV&, const TV&)>& encoded) {
  Arena& A = cx.arena;
  FF f{*this, N, cx, A};
  const int F = img.n, S = (int)src.size(), H = img.h, W = img.w, h = H / 8, w = W / 8;
  if (H % 32 || W % 32) throw std::runtime_error("gimmvfi: GIMM-VFI-F needs a network resolution that is a multiple of 32 (Twins-SVT sub-sampling)");
  if (S < 1 || (int)tgt.size() != S || per_call < 1 || S % per_call) throw std::runtime_error("flowformer: bad pair list");
  for (int s = 0; s < S; ++s)
    if (src[s] < 0 || src[s] >= F || tgt[s] < 0 || tgt[s] >= F) throw std::runtime_error("flowformer: pair index out of range");
  const int64_t Npx = (int64_t)h * w;
  const std::string me = std::string(FE) + "memory_encoder", md = std::string(FE) + "memory_decoder", u = md + ".update_block";
  std::vector<int> srcs, slot(F, -1);   // distinct sources in first-use order
  for (int s = 0; s < S; ++s)
    if (slot[src[s]] < 0) { slot[src[s]] = (int)srcs.size(); srcs.push_back(src[s]); }
  bool in_order = !gather && S == F;
  for (int s = 0; in_order && s < S; ++s) in_order = src[s] == s;
  const int ns = (int)srcs.size();
  if ((feat4_out.p && feat4_out.n != ns) || (feat8_out.p && feat8_out.n != ns) || (fproj_out.p && fproj_out.n != F))
    throw std::runtime_error("flowformer: feature outputs do not match the frame set");
  const size_t mk0 = A.mark();
  TV feat4 = feat4_out.p ? feat4_out : A.tensor(ns, H / 4, W / 4, 128);
  TV feat8 = feat8_out.p ? feat8_out : A.tensor(ns, h, w, 256);
  TV fproj = fproj_out.p ? fproj_out : A.tensor(F, h, w, 256);
  // ---- encoders: context Twins on the source frames -> feat4 / feat8; feature Twins once on all frames -> channel_convertor -> fproj
  {
    const size_t mk = A.mark();
    TV cimg = img;
    if (!in_order) {
      cimg = A.tensor(ns, H, W, 3, 4);
      for (int i = 0; i < ns; ++i) copy_channels(cx, img.batch(srcs[i], 1), cimg.batch(i, 1));
    }
    f.twins(std::string(FE) + "context_encoder", cimg, feat4, feat8);
    A.release(mk);
  }
  {
    const size_t mk = A.mark();
    TV t4 = A.tensor(F, H / 4, W / 4, 128), t8 = A.tensor(F, h, w, 256);
    f.twins(me + ".feat_encoder", img, t4, t8);
    f.lin(me + ".channel_convertor", t8, fproj);
    A.release(mk);
  }
  tap("ff.feat4", feat4); tap("ff.feat8", feat8); tap("ff.fproj", fproj);
  if (encoded) encoded(feat4, feat8, fproj);
  TV ctx8 = feat8;   // the context of every pair (decoder proj, GMA, the vertical blocks' concat_pe), in pair order
  if (!in_order) {
    ctx8 = A.tensor(S, h, w, 256);
    for (int s = 0; s < S; ++s) copy_channels(cx, feat8.batch(slot[src[s]], 1), ctx8.batch(s, 1));
  }
  // ---- memory encoder
  float* vol = A.alloc_f((size_t)S * Npx * Npx);
  f.cost_volume(fproj, src, tgt, vol);
  tap("ff.cost_volume", make_tv(vol, S, h, w, (int)Npx));   // [pair][source pixel][target pixel]
  TV latent = A.tensor(S * 8, h, w, 128);
  f.cost_perceiver(me + ".cost_perceiver_encoder", S, per_call, vol, h, w, ctx8, latent);
  tap("ff.cost_memory", latent);
  // ---- memory decoder (decoder.py:254-321)
  TV hx = A.tensor(S, h, w, 512);   // [net | inp | motion features | globally aggregated motion features] = the SepConvGRU's [h | x]
  TV hcur = hx.slice(0, 128), xin = hx.slice(128, 384), mf = hx.slice(256, 128), mg = hx.slice(384, 128);
  {
    const ConvW& wp = N.W(md + ".proj");
    ConvW wa = wp; wa.cout = 128; wa.w_tc = nullptr;
    ConvW wb = wp; wb.w = wp.w + 128; wb.b = wp.b + 128; wb.cout = 128; wb.w_tc = nullptr;
    ConvEpi e1; e1.act1 = ACT_TANH; conv2d(cx, ctx8, TV(), wa, ConvGeom(), e1, hcur);
    ConvEpi e2; e2.act1 = ACT_RELU; conv2d(cx, ctx8, TV(), wb, ConvGeom(), e2, hx.slice(128, 128));
  }
  tap_copy(cx, "ff.cnet", hx.slice(0, 256));   // tanh(net) | relu(inp) (the GRU overwrites net in place)
  // GMA attention (gma.py:56-76), once per pair: softmax(q k^T / sqrt(128)) stored * att_mul (a power of two)
  float att_mul = 1.f;
  while (att_mul < (float)Npx && att_mul < 32768.f) att_mul *= 2.f;   // (<= 2^15: a one-hot row stays below the largest half)
  float* att = A.alloc_f((size_t)S * Npx * Npx);
  float* zeros = nullptr;
  {
    const size_t mk = A.mark();
    const ConvW& wq = N.W(md + ".att.to_qk");
    ConvW wa = wq; wa.cout = 128; wa.w_tc = nullptr;
    ConvW wb = wq; wb.w = wq.w + 128; wb.b = wq.b + 128; wb.cout = 128; wb.w_tc = nullptr;
    TV q = A.tensor(S, h, w, 128), k = A.tensor(S, h, w, 128);
    conv2d(cx, hx.slice(128, 128), TV(), wa, ConvGeom(), ConvEpi(), q);
    conv2d(cx, hx.slice(128, 128), TV(), wb, ConvGeom(), ConvEpi(), k);
    const float scale = 1.0f / std::sqrt(128.f);
    if (cx.tc && corr_volume_tc_wants_f16_planes()) {
      const int64_t plane = (int64_t)S * Npx * 128;
      uint16_t* qp = reinterpret_cast<uint16_t*>(A.alloc_f((size_t)plane));
      uint16_t* kp = reinterpret_cast<uint16_t*>(A.alloc_f((size_t)plane));
      split_planes_f16(cx, q, qp); split_planes_f16(cx, k, kp);
      for (int s = 0; s < S; ++s)
        if (!cx.dry) corr_gemm_3xf16(cx, qp + s * Npx * 128, plane, (int)Npx, kp + s * Npx * 128, plane, (int)Npx, 128, scale, att + (int64_t)s * Npx * Npx);
    } else if (cx.tc) {
      float* planes = A.alloc_f((size_t)2 * Npx * 128);
      const int64_t nz = ((Npx + 255) / 256) * 256 + 512;
      float* zb = A.alloc_f((size_t)nz);
      if (!cx.dry) dev_memset(zb, 0, (size_t)nz * sizeof(float), cx.stream);
      for (int s = 0; s < S; ++s) {
        if (corr_volume_tc_wants_f16_planes()) split_planes_f16(cx, k.batch(s, 1), planes); else split_planes(cx, k.batch(s, 1), planes);
        if (!cx.dry) corr_volume_tc(cx, q.batch(s, 1), planes, zb, att + (int64_t)s * Npx * Npx, scale, true, (int)Npx);
      }
    } else {
      corr_volume(cx, q, k, att, scale);
    }
    row_softmax(cx, att, (int64_t)S * Npx, Npx, att_mul);
    A.release(mk);
  }
  tap("ff.gma_attn", make_tv(att, S, h, w, (int)Npx));   // softmax rows * att_mul
  const bool agg_tc = cx.tc && Npx % 64 == 0;
  float* vt_planes = nullptr; float* vT = nullptr;
  if (agg_tc) {
    vT = A.alloc_f((size_t)128 * Npx); vt_planes = A.alloc_f((size_t)2 * 128 * Npx);
    const int64_t nz = 1024;
    zeros = A.alloc_f((size_t)nz);
    if (!cx.dry) dev_memset(zeros, 0, (size_t)nz * sizeof(float), cx.stream);
  }
  const std::string ca = md + ".decoder_layer.cross_attend";
  TV k8 = A.tensor(S * 8, h, w, 64), v8 = A.tensor(S * 8, h, w, 64);   // computed in the first iteration, re-used after (decoder.py:86-88)
  f.lin(ca + ".k", latent, k8); f.lin(ca + ".v", latent, v8);
  TV coords1 = A.tensor(S, h, w, 2), flow = A.tensor(S, h, w, 2, 4);
  TV corr = A.tensor(S, h, w, 145, 148);     // [cost_global (64) | cost_forward (81)]  (decoder.py:305)
  TV cfw = corr.slice(64, 81), cgl = corr.slice(0, 64);
  TV ft1 = A.tensor(S, h, w, 64), qr = A.tensor(S, h, w, 64), y64 = A.tensor(S, h, w, 64), q64 = A.tensor(S, h, w, 64), o64 = A.tensor(S, h, w, 64),
     xg = A.tensor(S, h, w, 64);
  TV cor1 = A.tensor(S, h, w, 256), corflo = A.tensor(S, h, w, 256), flo1 = A.tensor(S, h, w, 128), vv = A.tensor(S, h, w, 128),
     agg = A.tensor(S, h, w, 128), zb = A.tensor(S, h, w, 128), rh = A.tensor(S, h, w, 128), fh = A.tensor(S, h, w, 256), mask = A.tensor(S, h, w, 576);
  init_coords(cx, coords1);
  if (flow_init) parallel_for(cx, (int64_t)S * 2 * h * w, FlowInitAddK{flow_init, coords1}, "flowformer_flow_init");   // decoder.py:265-267
  const bool hoist = cx.tc;
  TV Pzr[2], Pq[2];
  if (hoist)
    for (int sx = 0; sx < 2; ++sx) {
      const std::string sfx = sx == 0 ? "1" : "2";
      Pzr[sx] = A.tensor(S, h, w, 256); Pq[sx] = A.tensor(S, h, w, 128);
      N.conv(u + ".gru.convzr" + sfx + "_inp", hx.slice(128, 128), Pzr[sx]);
      N.conv(u + ".gru.convq" + sfx + "_inp", hx.slice(128, 128), Pq[sx]);
    }
  CorrPyr pyr{};
  for (int l = 0; l < 4; ++l) { pyr.lvl[l] = vol; pyr.h[l] = h; pyr.w[l] = w; }
  pyr.rows_per_sample = Npx; pyr.nl = 1;
  for (int it = 0; it < iters; ++it) {
    const bool last = it == iters - 1;
    if (last) { tap_copy(cx, "ff.coords_last", coords1); tap_copy(cx, "ff.net_last", hcur); }
    // encode_flow_token: 9x9 window of each pixel's own cost map around its current target (decoder.py:233-252)
    corr_lookup(cx, pyr, coords1, cfw);
    f.lin(md + ".flow_token_encoder.0", cfw, ft1, ACT_GELU);
    f.lin(md + ".flow_token_encoder.2", ft1, qr);
    // CrossAttentionLayer (decoder.py:81-117): one query per pixel against its 8 memory tokens
    f.ln(ca + ".norm1", qr, y64, 1e-5f);
    add_pe_coords(cx, y64, coords1, y64);
    f.lin(ca + ".q", y64, q64);
    {
      AttnDims a{};
      a.nb1 = S; a.nb2 = Npx; a.nq = 1; a.nk = 8; a.heads = 8;
      a.q_s1 = Npx * 64; a.q_s2 = 64; a.o_s1 = Npx * 64; a.o_s2 = 64;
      a.k_s1 = a.v_s1 = 8 * Npx * 64; a.k_s2 = a.v_s2 = 64; a.k_sj = a.v_sj = Npx * 64;
      strided_attention(cx, q64.p, k8.p, v8.p, o64.p, a, 8);
    }
    f.lin_res(ca + ".proj", o64, qr, qr, xg);                     // short_cut + proj(cat[x, short_cut])
    f.mlp(ca + ".norm2", 1e-5f, ca + ".ffn.0", ca + ".ffn.3", xg, cgl);
    coords_minus_grid(cx, coords1, flow, hx.slice(382, 2));
    if (it == 0) tap_copy(cx, "ff.dec_corr_0", corr);
    if (last) tap_copy(cx, "ff.corr_last", corr);
    // BasicMotionEncoder (gru.py:75-97)
    N.conv(u + ".encoder.convc1", corr, cor1, ACT_RELU);
    N.conv(u + ".encoder.convc2", cor1, corflo.slice(0, 192), ACT_RELU);
    N.conv7x(u + ".encoder.convf1", flow, flo1, ACT_RELU);
    N.conv(u + ".encoder.convf2", flo1, corflo.slice(192, 64), ACT_RELU);
    N.conv(u + ".encoder.conv", corflo, hx.slice(256, 126), ACT_RELU);
    // Aggregate (gma.py:98-115): mg = mf + gamma * (attn @ to_v(mf))
    f.lin(u + ".aggregator.to_v", mf, vv);
    for (int s = 0; s < S; ++s) {
      float* as = att + (int64_t)s * Npx * Npx;
      if (agg_tc) {
        transpose_2d(cx, vv.batch(s, 1).p, vT, Npx, 128, 128);
        TV vtv = make_tv(vT, 1, 1, 128, (int)Npx);
        if (corr_volume_tc_wants_f16_planes()) split_planes_f16(cx, vtv, vt_planes); else split_planes(cx, vtv, vt_planes);
        TV av = make_tv(as, 1, h, w, (int)Npx);
        if (!cx.dry) corr_volume_tc(cx, av, vt_planes, zeros, agg.batch(s, 1).p, 1.0f / att_mul, true, 128);
      } else {
        gemm_nn(cx, as, vv.batch(s, 1).p, agg.batch(s, 1).p, Npx, Npx, 128, Npx, 128, 128, 1.0f / att_mul);
      }
    }
    axpy_dev(cx, mf, agg, N.V(u + ".aggregator.gamma"), mg);
    if (last) { tap_copy(cx, "ff.motion_last", mf); tap_copy(cx, "ff.mg_last", mg); }   // (126 motion features + the 2 flow channels | mg)
    // SepConvGRU (gru.py:35-73) over [h | inp | mf | mg]
    for (const char* sfx : {"1", "2"}) {
      if (hoist) {
        const int sx = sfx[0] - '1';
        ConvEpi ezr; ezr.res = Pzr[sx]; ezr.act2 = ACT_SIGMOID; ezr.mul = hcur; ezr.out2 = rh; ezr.split_c = 128;
        N.conv_e(u + ".gru.convzr" + sfx + "_hm", hcur, hx.slice(256, 256), zb, ezr);
        ConvEpi eq; eq.res = Pq[sx]; eq.act2 = ACT_TANH; eq.gru_z = zb; eq.gru_h = hcur;
        N.conv_e(u + ".gru.convq" + sfx + "_hm", rh, hx.slice(256, 256), hcur, eq);
        continue;
      }
      if (cx.tc) {
        ConvEpi ezr; ezr.act1 = ACT_SIGMOID; ezr.mul = hcur; ezr.out2 = rh; ezr.split_c = 128;
        N.conv_e(u + ".gru.convzr" + sfx, hx, TV(), zb, ezr);
      } else {
        ConvEpi ez; ez.act1 = ACT_SIGMOID;
        N.conv_e(u + ".gru.convz" + sfx, hx, TV(), zb, ez);
        ConvEpi er; er.act1 = ACT_SIGMOID; er.mul = hcur;
        N.conv_e(u + ".gru.convr" + sfx, hx, TV(), rh, er);
      }
      ConvEpi eq; eq.act1 = ACT_TANH; eq.gru_z = zb; eq.gru_h = hcur;
      N.conv_e(u + ".gru.convq" + sfx, rh, xin, hcur, eq);
    }
    if (it == 0) tap_copy(cx, "ff.dec_net_0", hcur);
    N.conv(u + ".flow_head.conv1", hcur, fh, ACT_RELU);
    { ConvEpi e; e.res = coords1; N.conv_e(u + ".flow_head.conv2", fh, TV(), coords1, e); }
    if (last) {   // only the last prediction is consumed (decoder.py:321, gimmvfi_f.py:122-123)
      N.conv(u + ".mask.0", hcur, fh, ACT_RELU);
      N.conv(u + ".mask.2", fh, mask);
      tap("ff.net_final", hcur); tap("ff.mask", mask);   // (0.25 is folded into mask.2's weights)
      coords_minus_grid(cx, coords1, flow, TV());
      tap("ff.lowres_flow", flow);
      if (flow_low.p) copy_channels(cx, flow, flow_low);
      convex_upsample(cx, flow, mask, flow_up);
    }
  }
  if (!debug_) A.release(mk0);
}

}  // namespace gv
