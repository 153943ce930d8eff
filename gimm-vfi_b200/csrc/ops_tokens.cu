// Token-side kernels of the native FlowFormer estimator (GIMM-VFI-F, SURVEY 8(a) row a24): LayerNorm, the Twins-SVT window / sub-sampled
// attention, the strided multi-head attention of the cost-perceiver and the memory decoder, sinusoidal position codes, depthwise 3x3
// (PEG), space-to-depth for the patch / sub-sampling convolutions, the first 6x6 stride-2 layer over the raw cost maps, row softmax and
// the small GEMM fallbacks.  All tensors are NHWC views (TV): a token sequence (B, H*W, C) of the reference IS an NHWC map, so every
// nn.Linear runs as a 1x1 convolution on the tensor-core convolution kernel (conv_tc.cu) and only the non-GEMM pieces live here.
// Every kernel body is a thread-per-item functor (runs as an OpenMP loop in the test-only host simulation).
// Reference files: flowformer/core/FlowFormer/LatentCostFormer/{twins,encoder,decoder,attention,gma}.py (cited per kernel).
#include "common.h"

namespace gv {

// LinearPositionEmbeddingSine (LatentCostFormer/attention.py:170-182): channel c of a `dim`-wide code of the point (X, Y).
// [sin(3.14 X f / 200) | cos(..X..) | sin(..Y..) | cos(..Y..)], f = 0 .. dim/4 - 1 (3.14, not pi; float op order of the reference).
GV_HD float pe_value(int c, int dim, float X, float Y) {
  const int q = dim >> 2, g = c / q, f = c - g * q;
  const float a = ((3.14f * (g < 2 ? X : Y)) * (float)f) * (1.0f / 200.0f);
  return (g & 1) ? cosf(a) : sinf(a);
}

// ------------------------------------------------------------------ space to depth
// dst[n, y, x, (ky*k + kx)*C + c] = src[n, y*k + ky, x*k + kx, c]: a k x k stride-k convolution (Twins PatchEmbed twins.py:1122-1149,
// the sub-sampling convs of GlobalSubSampleAttn twins.py:890-893 / :452-456) becomes a 1x1 convolution over k*k*C channels.
template <int L, bool Any> struct PatchifyK {   // L channels per item
  TV src, dst; int k;
  GV_HD void operator()(int64_t i) const {
    const int CL = src.c / L, KL = k * k * CL;
    const int ch = (int)(i % KL); int64_t r = i / KL;
    const int x = (int)(r % dst.w); r /= dst.w; const int y = (int)(r % dst.h); const int n = (int)(r / dst.h);
    const int t = ch / CL, c = (ch - t * CL) * L, ky = t / k, kx = t - ky * k;
    const int sy = y * k + ky, sx = x * k + kx;
    float v[L];
    for (int j = 0; j < L; ++j) v[j] = 0.f;
    if (sy < src.h && sx < src.w) ld_lanes<L, Any>(src, src.off(n, sy, sx) + c, v);
    st_lanes<L, Any>(dst, dst.off(n, y, x) + t * src.c + c, v);
  }
};
void patchify(Ctx& cx, const TV& src, const TV& dst, int k) {
  if (dst.c != k * k * src.c || dst.n != src.n) throw std::runtime_error("patchify: shape mismatch");
  lanes_for<PatchifyK>(cx, vec4_ok(src) && vec4_ok(dst), dst.pixels() * dst.c, "patchify", src, dst, k);
}

// ------------------------------------------------------------------ LayerNorm
// y = (x - mean) / sqrt(var + eps) * g + b over the channels of a token (nn.LayerNorm), written into a map that may be LARGER than the
// input (rows / columns beyond it are zero: the padding Twins applies AFTER the norm, twins.py:835-842), optionally followed by
// + position code of (x*pe_scale, y*pe_scale) (twins.py:500-513: keys of the sub-sampled map carry the code of coords * sr).
struct LayerNormK {
  TV x, out; const float* g; const float* b; float eps; float pe_scale; int pe_dim;
  GV_HD void operator()(int64_t i) const {
    const int px = (int)(i % out.w); int64_t r = i / out.w; const int py = (int)(r % out.h); const int n = (int)(r / out.h);
    float* o = out.p + out.off(n, py, px);
    const int C = x.c;
    if (py >= x.h || px >= x.w) { for (int c = 0; c < C; ++c) o[c] = 0.f; return; }
    const float* s = x.p + x.off(n, py, px);
    float sum = 0.f;
    for (int c = 0; c < C; ++c) sum += s[c];
    const float mean = sum / (float)C;
    float var = 0.f;
    for (int c = 0; c < C; ++c) { const float d = s[c] - mean; var = fmaf(d, d, var); }
    const float rstd = 1.0f / sqrtf(var / (float)C + eps);
    if (pe_dim > 0) {
      const float X = (float)px * pe_scale, Y = (float)py * pe_scale;
      for (int c = 0; c < C; ++c) o[c] = ((s[c] - mean) * rstd) * g[c] + b[c] + pe_value(c, pe_dim, X, Y);
    } else {
      for (int c = 0; c < C; ++c) o[c] = ((s[c] - mean) * rstd) * g[c] + b[c];
    }
  }
};
#ifndef GV_HOSTSIM
// one warp per token: a lane owns 4 consecutive channels per 128-channel group (one 16-byte load / store each), shuffle reductions
// (the first version issued 16 predicated scalar loads per lane: 1.2 TB/s, instruction bound per ncu)
__global__ void __launch_bounds__(256) layernorm_warp_kernel(TV x, TV out, const float* __restrict__ g, const float* __restrict__ b, float eps,
                                                             float pe_scale, int pe_dim, int64_t tokens) {
  const int lane = threadIdx.x & 31;
  const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int C = x.c;   // C % 4 == 0, C <= 512
  for (int64_t i = w0; i < tokens; i += nw) {
    const int px = (int)(i % out.w); int64_t r = i / out.w; const int py = (int)(r % out.h); const int n = (int)(r / out.h);
    float* o = out.p + out.off(n, py, px);
    if (py >= x.h || px >= x.w) {
      for (int c = lane * 4; c < C; c += 128) *reinterpret_cast<float4*>(o + c) = make_float4(0.f, 0.f, 0.f, 0.f);
      continue;
    }
    const float* s = x.p + x.off(n, py, px);
    float4 v[4];
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = lane * 4 + 128 * k;
      v[k] = c < C ? *reinterpret_cast<const float4*>(s + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      sum += (v[k].x + v[k].y) + (v[k].z + v[k].w);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
    const float mean = sum / (float)C;
    float var = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (lane * 4 + 128 * k < C) {
        const float d0 = v[k].x - mean, d1 = v[k].y - mean, d2 = v[k].z - mean, d3 = v[k].w - mean;
        var = fmaf(d0, d0, var); var = fmaf(d1, d1, var); var = fmaf(d2, d2, var); var = fmaf(d3, d3, var);
      }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) var += __shfl_xor_sync(0xffffffffu, var, d);
    const float rstd = 1.0f / sqrtf(var / (float)C + eps);
    const float X = (float)px * pe_scale, Y = (float)py * pe_scale;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = lane * 4 + 128 * k;
      if (c < C) {
        const float4 gg = *reinterpret_cast<const float4*>(g + c), bb = *reinterpret_cast<const float4*>(b + c);
        float4 y;
        y.x = ((v[k].x - mean) * rstd) * gg.x + bb.x; y.y = ((v[k].y - mean) * rstd) * gg.y + bb.y;
        y.z = ((v[k].z - mean) * rstd) * gg.z + bb.z; y.w = ((v[k].w - mean) * rstd) * gg.w + bb.w;
        if (pe_dim > 0) { y.x += pe_value(c, pe_dim, X, Y); y.y += pe_value(c + 1, pe_dim, X, Y); y.z += pe_value(c + 2, pe_dim, X, Y); y.w += pe_value(c + 3, pe_dim, X, Y); }
        *reinterpret_cast<float4*>(o + c) = y;
      }
    }
  }
}
#endif
void layernorm(Ctx& cx, const TV& x, const float* g, const float* b, float eps, const TV& out, float pe_scale, int pe_dim) {
  if (out.c != x.c || out.n != x.n || out.h < x.h || out.w < x.w) throw std::runtime_error("layernorm: shape mismatch");
#ifndef GV_HOSTSIM
  if (x.c <= 512 && vec4_ok(x) && vec4_ok(out) && (reinterpret_cast<uintptr_t>(g) & 15) == 0 && (reinterpret_cast<uintptr_t>(b) & 15) == 0) {
    if (cx.dry) return;
    cx.launches++;
    const int64_t tokens = out.pixels();
    if (cx.prof) cx.prof->begin(cx.stream, "layernorm", (double)tokens * x.c);
    int64_t blocks = (tokens + 7) / 8, cap = (int64_t)cx.sm_count * 16;
    if (blocks > cap) blocks = cap;
    layernorm_warp_kernel<<<(unsigned)blocks, 256, 0, cx.stream>>>(x, out, g, b, eps, pe_scale, pe_dim, tokens);
    gv_check_launch("layernorm");
    if (cx.prof) cx.prof->end(cx.stream);
    return;
  }
#endif
  parallel_for(cx, out.pixels(), LayerNormK{x, out, g, b, eps, pe_scale, pe_dim}, "layernorm");
}

// ------------------------------------------------------------------ PEG: x + depthwise 3x3 (PosConv, twins.py:1100-1116)
struct DwConv3ResK {
  TV x, out; const float* w /*[9][C]*/; const float* b;
  GV_HD void operator()(int64_t i) const {
    const int C = x.c;
    const int c = (int)(i % C); int64_t r = i / C;
    const int px = (int)(r % x.w); r /= x.w; const int py = (int)(r % x.h); const int n = (int)(r / x.h);
    float acc = b[c];
    for (int ky = 0; ky < 3; ++ky) {
      const int sy = py + ky - 1;
      if (sy < 0 || sy >= x.h) continue;
      for (int kx = 0; kx < 3; ++kx) {
        const int sx = px + kx - 1;
        if (sx < 0 || sx >= x.w) continue;
        acc = fmaf(x.p[x.off(n, sy, sx) + c], w[(ky * 3 + kx) * C + c], acc);
      }
    }
    out.p[out.off(n, py, px) + c] = acc + x.p[x.off(n, py, px) + c];
  }
};
void dwconv3x3_residual(Ctx& cx, const TV& x, const float* w9c, const float* bias, const TV& out) {
  parallel_for(cx, x.pixels() * x.c, DwConv3ResK{x, out, w9c, bias}, "dwconv3x3_peg");
}

// ------------------------------------------------------------------ window attention (LocallyGroupedAttn, twins.py:814-867 / :331-427)
// q, k, v live on the PADDED map (Hp, Wp multiples of ws); one thread per (window, head, query): online softmax over the ws*ws keys of
// its window (padded tokens take part un-masked, as in the reference); the output goes to the unpadded map.
template <int HD>
struct WindowAttnK {
  TV q, k, v, out; int heads, ws; float scale;
  GV_HD void operator()(int64_t i) const {
    const int W2 = ws * ws;
    const int qi = (int)(i % W2); int64_t r = i / W2;
    const int hd = (int)(r % heads); r /= heads;
    const int wxn = q.w / ws, wyn = q.h / ws;
    const int wx = (int)(r % wxn); r /= wxn; const int wy = (int)(r % wyn); const int n = (int)(r / wyn);
    const int qy = wy * ws + qi / ws, qx = wx * ws + qi % ws;
    if (qy >= out.h || qx >= out.w) return;
    float qv[HD], acc[HD];
    const float* qp = q.p + q.off(n, qy, qx) + hd * HD;
#pragma unroll
    for (int d = 0; d < HD; d += 4) { const F4 t = ld4(qp + d); qv[d] = t.x; qv[d + 1] = t.y; qv[d + 2] = t.z; qv[d + 3] = t.w; acc[d] = acc[d + 1] = acc[d + 2] = acc[d + 3] = 0.f; }
    float m = -3.0e38f, l = 0.f;
    for (int j = 0; j < W2; ++j) {
      const int ky = wy * ws + j / ws, kx = wx * ws + j % ws;
      const float* kp = k.p + k.off(n, ky, kx) + hd * HD;
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < HD; d += 4) { const F4 t = ld4(kp + d); s = fmaf(qv[d], t.x, s); s = fmaf(qv[d + 1], t.y, s); s = fmaf(qv[d + 2], t.z, s); s = fmaf(qv[d + 3], t.w, s); }
      s *= scale;
      const float mn = fmaxf(m, s), corr = expf(m - mn), p = expf(s - mn);
      const float* vp = v.p + v.off(n, ky, kx) + hd * HD;
      l = l * corr + p;
#pragma unroll
      for (int d = 0; d < HD; d += 4) {
        const F4 t = ld4(vp + d);
        acc[d] = fmaf(p, t.x, acc[d] * corr); acc[d + 1] = fmaf(p, t.y, acc[d + 1] * corr);
        acc[d + 2] = fmaf(p, t.z, acc[d + 2] * corr); acc[d + 3] = fmaf(p, t.w, acc[d + 3] * corr);
      }
      m = mn;
    }
    float* o = out.p + out.off(n, qy, qx) + hd * HD;
    const float il = 1.0f / l;
#pragma unroll
    for (int d = 0; d < HD; ++d) o[d] = acc[d] * il;
  }
};
void window_attention(Ctx& cx, const TV& q, const TV& k, const TV& v, const TV& out, int heads, int ws) {
  const int hd = out.c / heads;
  if (q.h % ws || q.w % ws || q.c != out.c || hd * heads != out.c) throw std::runtime_error("window_attention: shape mismatch");
  const int64_t items = (int64_t)q.n * (q.h / ws) * (q.w / ws) * heads * ws * ws;
  const float scale = 1.0f / std::sqrt((float)hd);
  if (hd == 32) parallel_for(cx, items, WindowAttnK<32>{q, k, v, out, heads, ws, scale}, "window_attention_d32");
  else if (hd == 16) parallel_for(cx, items, WindowAttnK<16>{q, k, v, out, heads, ws, scale}, "window_attention_d16");
  else throw std::runtime_error("window_attention: head dim must be 16 or 32");
}

// ------------------------------------------------------------------ strided multi-head attention
// out[b1,b2,i,h,:] = softmax_j(<q[b1,b2,i,h,:], k[b1,b2,j,h,:]> * scale) v[b1,b2,j,h,:]   (attention.py:10-66; twins.py:898-925)
// Two batch levels and explicit strides address every attention of the estimator on its own memory layout: Twins' sub-sampled global
// attention (queries = all tokens of a map, keys = the stride-sr map), the cost-perceiver's latent cross / self attention (8 latent
// tokens per cost map, token-major layout) and the decoder's per-pixel query against the 8 memory tokens.  One thread per
// (batch, head, query), online softmax: neighbouring threads share every key / value address (broadcast loads).
template <int HD>
struct StridedAttnK {
  const float* q; const float* k; const float* v; float* out; AttnDims a; float scale;
  GV_HD void operator()(int64_t i) const {
    const int64_t qi = i % a.nq; int64_t r = i / a.nq;
    const int hd = (int)(r % a.heads); r /= a.heads;
    const int64_t b2 = r % a.nb2, b1 = r / a.nb2;
    const float* qp = q + b1 * a.q_s1 + b2 * a.q_s2 + qi * a.q_si + hd * HD;
    const float* kb = k + b1 * a.k_s1 + b2 * a.k_s2 + hd * HD;
    const float* vb = v + b1 * a.v_s1 + b2 * a.v_s2 + hd * HD;
    float qv[HD], acc[HD];
#pragma unroll
    for (int d = 0; d < HD; d += 4) { const F4 t = ld4(qp + d); qv[d] = t.x; qv[d + 1] = t.y; qv[d + 2] = t.z; qv[d + 3] = t.w; acc[d] = acc[d + 1] = acc[d + 2] = acc[d + 3] = 0.f; }
    float m = -3.0e38f, l = 0.f;
    for (int64_t j = 0; j < a.nk; ++j) {
      const float* kp = kb + j * a.k_sj;
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < HD; d += 4) { const F4 t = ld4(kp + d); s = fmaf(qv[d], t.x, s); s = fmaf(qv[d + 1], t.y, s); s = fmaf(qv[d + 2], t.z, s); s = fmaf(qv[d + 3], t.w, s); }
      s *= scale;
      const float mn = fmaxf(m, s), corr = expf(m - mn), p = expf(s - mn);
      const float* vp = vb + j * a.v_sj;
      l = l * corr + p;
#pragma unroll
      for (int d = 0; d < HD; d += 4) {
        const F4 t = ld4(vp + d);
        acc[d] = fmaf(p, t.x, acc[d] * corr); acc[d + 1] = fmaf(p, t.y, acc[d + 1] * corr);
        acc[d + 2] = fmaf(p, t.z, acc[d + 2] * corr); acc[d + 3] = fmaf(p, t.w, acc[d + 3] * corr);
      }
      m = mn;
    }
    float* o = out + b1 * a.o_s1 + b2 * a.o_s2 + qi * a.o_si + hd * HD;
    const float il = 1.0f / l;
#pragma unroll
    for (int d = 0; d < HD; ++d) o[d] = acc[d] * il;
  }
};
#ifndef GV_HOSTSIM
// Many queries against one key / value set per (batch, head) — Twins' sub-sampled global attention (twins.py:898-925, :466-546): a CTA
// takes 256 queries of one (batch, head), the keys / values stream through shared memory in tiles (every thread reads the same key:
// one broadcast LDS.128 per 4 elements instead of a global load per element), online softmax over groups of 4 keys (5 exp per 4 keys).
template <int HD, int KT>
__global__ void __launch_bounds__(256) attention_shared_kv_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                                                                  float* __restrict__ out, AttnDims a, float scale) {
  extern __shared__ __align__(16) float smem_kv[];
  float* Ks = smem_kv; float* Vs = smem_kv + KT * HD;
  const int head = blockIdx.y; const int64_t b1 = blockIdx.z;
  const int64_t qi = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const bool live = qi < a.nq;
  const float* kb = k + b1 * a.k_s1 + head * HD;
  const float* vb = v + b1 * a.v_s1 + head * HD;
  float qv[HD], acc[HD];
#pragma unroll
  for (int d = 0; d < HD; ++d) { qv[d] = 0.f; acc[d] = 0.f; }
  if (live) {
    const float* qp = q + b1 * a.q_s1 + qi * a.q_si + head * HD;
#pragma unroll
    for (int d = 0; d < HD; d += 4) { const float4 t = *reinterpret_cast<const float4*>(qp + d); qv[d] = t.x * scale; qv[d + 1] = t.y * scale; qv[d + 2] = t.z * scale; qv[d + 3] = t.w * scale; }
  }
  float m = -3.0e38f, l = 0.f;
  for (int64_t j0 = 0; j0 < a.nk; j0 += KT) {
    const int tn = (int)((a.nk - j0) < KT ? (a.nk - j0) : KT);
    const int tn4 = (tn + 3) & ~3;
    __syncthreads();
    for (int e = threadIdx.x; e < tn4 * (HD / 4); e += 256) {
      const int j = e / (HD / 4), c = (e - j * (HD / 4)) * 4;
      float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
      if (j < tn) { kk = *reinterpret_cast<const float4*>(kb + (j0 + j) * a.k_sj + c); vv = *reinterpret_cast<const float4*>(vb + (j0 + j) * a.v_sj + c); }
      *reinterpret_cast<float4*>(Ks + j * HD + c) = kk; *reinterpret_cast<float4*>(Vs + j * HD + c) = vv;
    }
    __syncthreads();
    for (int j = 0; j < tn4; j += 4) {
      float s[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float* kp = Ks + (j + u) * HD;
        float t0 = 0.f, t1 = 0.f;
#pragma unroll
        for (int d = 0; d < HD; d += 8) {
          const float4 x = *reinterpret_cast<const float4*>(kp + d), y = *reinterpret_cast<const float4*>(kp + d + 4);
          t0 = fmaf(qv[d], x.x, t0); t0 = fmaf(qv[d + 1], x.y, t0); t0 = fmaf(qv[d + 2], x.z, t0); t0 = fmaf(qv[d + 3], x.w, t0);
          t1 = fmaf(qv[d + 4], y.x, t1); t1 = fmaf(qv[d + 5], y.y, t1); t1 = fmaf(qv[d + 6], y.z, t1); t1 = fmaf(qv[d + 7], y.w, t1);
        }
        s[u] = (j + u < tn) ? t0 + t1 : -3.0e38f;
      }
      const float mn = fmaxf(fmaxf(m, fmaxf(s[0], s[1])), fmaxf(s[2], s[3]));
      const float corr = expf(m - mn);
      float p[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) p[u] = expf(s[u] - mn);
      l = fmaf(l, corr, (p[0] + p[1]) + (p[2] + p[3]));
      m = mn;
#pragma unroll
      for (int d = 0; d < HD; d += 4) {
        const float4 v0 = *reinterpret_cast<const float4*>(Vs + (j + 0) * HD + d), v1 = *reinterpret_cast<const float4*>(Vs + (j + 1) * HD + d);
        const float4 v2 = *reinterpret_cast<const float4*>(Vs + (j + 2) * HD + d), v3 = *reinterpret_cast<const float4*>(Vs + (j + 3) * HD + d);
        acc[d] = fmaf(p[3], v3.x, fmaf(p[2], v2.x, fmaf(p[1], v1.x, fmaf(p[0], v0.x, acc[d] * corr))));
        acc[d + 1] = fmaf(p[3], v3.y, fmaf(p[2], v2.y, fmaf(p[1], v1.y, fmaf(p[0], v0.y, acc[d + 1] * corr))));
        acc[d + 2] = fmaf(p[3], v3.z, fmaf(p[2], v2.z, fmaf(p[1], v1.z, fmaf(p[0], v0.z, acc[d + 2] * corr))));
        acc[d + 3] = fmaf(p[3], v3.w, fmaf(p[2], v2.w, fmaf(p[1], v1.w, fmaf(p[0], v0.w, acc[d + 3] * corr))));
      }
    }
  }
  if (live) {
    float* o = out + b1 * a.o_s1 + qi * a.o_si + head * HD;
    const float il = 1.0f / l;
#pragma unroll
    for (int d = 0; d < HD; d += 4) *reinterpret_cast<float4*>(o + d) = make_float4(acc[d] * il, acc[d + 1] * il, acc[d + 2] * il, acc[d + 3] * il);
  }
}
template <int HD, int KT>
static void launch_attention_shared_kv(Ctx& cx, const float* q, const float* k, const float* v, float* out, const AttnDims& a, float scale) {
  const int smem = 2 * KT * HD * (int)sizeof(float);
  static volatile unsigned char attr[64];
  gv_set_max_smem(attention_shared_kv_kernel<HD, KT>, smem, attr);
  cx.launches++;
  if (cx.prof) cx.prof->begin(cx.stream, HD == 16 ? "attention_shared_kv_d16" : "attention_shared_kv_d32", 4.0 * (double)a.nb1 * a.heads * a.nq * a.nk * HD);
  dim3 grid((unsigned)((a.nq + 255) / 256), (unsigned)a.heads, (unsigned)a.nb1);
  attention_shared_kv_kernel<HD, KT><<<grid, 256, smem, cx.stream>>>(q, k, v, out, a, scale);
  gv_check_launch("attention_shared_kv");
  if (cx.prof) cx.prof->end(cx.stream);
}
#endif

void strided_attention(Ctx& cx, const float* q, const float* k, const float* v, float* out, const AttnDims& a, int head_dim) {
  const int64_t items = a.nb1 * a.nb2 * a.heads * a.nq;
  const float scale = 1.0f / std::sqrt((float)head_dim);
#ifndef GV_HOSTSIM
  {
    auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    const bool strides4 = !((a.q_s1 | a.q_si | a.k_s1 | a.k_sj | a.v_s1 | a.v_sj | a.o_s1 | a.o_si) & 3);
    if (a.nb2 == 1 && a.nq >= 2048 && a.nk >= 32 && a.nb1 <= 65535 && (head_dim == 16 || head_dim == 32) && al(q) && al(k) && al(v) && al(out) && strides4) {
      if (cx.dry) return;
      if (head_dim == 16) launch_attention_shared_kv<16, 512>(cx, q, k, v, out, a, scale);
      else launch_attention_shared_kv<32, 256>(cx, q, k, v, out, a, scale);
      return;
    }
  }
#endif
  switch (head_dim) {
    case 8: parallel_for(cx, items, StridedAttnK<8>{q, k, v, out, a, scale}, "attention_d8"); break;
    case 16: parallel_for(cx, items, StridedAttnK<16>{q, k, v, out, a, scale}, "attention_d16"); break;
    case 32: parallel_for(cx, items, StridedAttnK<32>{q, k, v, out, a, scale}, "attention_d32"); break;
    default: throw std::runtime_error("strided_attention: head dim must be 8, 16 or 32");
  }
}

// ------------------------------------------------------------------ position codes
// out[n,y,x,:] = [a | b](n,y,x) (zero outside their extent: out may be the padded map) + code(dim = out.c) of the window-local
// (x % ws, y % ws) or absolute (x, y) position: the q / k input of the RPE-context attention blocks (twins.py:359-399, :466-499).
// `b` is the projected context: the reference repeats the context batch along dim 0 (context.repeat(B // ctx_B, 1, 1, 1)), so sample n
// of a group of `grp` consecutive samples reads context sample (n / grp_all) * ctx_per + (n % grp_all) % ctx_per (see flowformer.cu).
struct ConcatPeK {
  TV a, b, out; int ws; int add_pe; int grp_all, ctx_per;
  GV_HD void operator()(int64_t i) const {
    const int C = out.c;
    const int c = (int)(i % C); int64_t r = i / C;
    const int px = (int)(r % out.w); r /= out.w; const int py = (int)(r % out.h); const int n = (int)(r / out.h);
    float v = 0.f;
    if (c < a.c) { if (py < a.h && px < a.w) v = a.p[a.off(n, py, px) + c]; }
    else if (b.p && py < b.h && px < b.w) { const int nb = (n / grp_all) * ctx_per + (n % grp_all) % ctx_per; v = b.p[b.off(nb, py, px) + (c - a.c)]; }
    if (add_pe) v += pe_value(c, C, (float)(ws > 0 ? px % ws : px), (float)(ws > 0 ? py % ws : py));
    out.p[out.off(n, py, px) + c] = v;
  }
};
void concat_pe(Ctx& cx, const TV& a, const TV& b, const TV& out, int ws, bool add_pe, int grp_all, int ctx_per) {
  if (out.c != a.c + (b.p ? b.c : 0)) throw std::runtime_error("concat_pe: channel mismatch");
  parallel_for(cx, out.pixels() * out.c, ConcatPeK{a, b, out, ws, add_pe ? 1 : 0, grp_all, ctx_per}, "concat_pe");
}
// out[n,y,x,c] = code_c(x*scale + shift, y*scale + shift), dim = out.c: the patch-centre code concatenated to the cost-map patch
// embedding (encoder.py:76-89)
struct WritePeK {
  TV out; float scale, shift;
  GV_HD void operator()(int64_t i) const {
    const int C = out.c;
    const int c = (int)(i % C); int64_t r = i / C;
    const int px = (int)(r % out.w); r /= out.w; const int py = (int)(r % out.h); const int n = (int)(r / out.h);
    out.p[out.off(n, py, px) + c] = pe_value(c, C, (float)px * scale + shift, (float)py * scale + shift);
  }
};
void write_pe(Ctx& cx, const TV& out, float scale, float shift) { parallel_for(cx, out.pixels() * out.c, WritePeK{out, scale, shift}, "write_pe"); }
// out = x + code(coords[n,y,x] = (X, Y)), dim = x.c: the decoder's query code (decoder.py:89-108)
struct AddPeCoordsK {
  TV x, coords, out;
  GV_HD void operator()(int64_t i) const {
    const int C = x.c;
    const int c = (int)(i % C); int64_t r = i / C;
    const int px = (int)(r % x.w); r /= x.w; const int py = (int)(r % x.h); const int n = (int)(r / x.h);
    const float* cc = coords.p + coords.off(n, py, px);
    out.p[out.off(n, py, px) + c] = x.p[x.off(n, py, px) + c] + pe_value(c, C, cc[0], cc[1]);
  }
};
void add_pe_coords(Ctx& cx, const TV& x, const TV& coords, const TV& out) { parallel_for(cx, x.pixels() * x.c, AddPeCoordsK{x, coords, out}, "add_pe_coords"); }

// ------------------------------------------------------------------ cost maps: first patch-embedding layer
// Conv2d(1, 16, 6, stride 2, padding 2) + ReLU over every cost map (encoder.py:38-48), the map zero-extended to a multiple of the patch
// size (encoder.py:68-71).  Input: `maps` rows of the all-pairs volume (h x w each, contiguous).  Output: (maps, oh + 4, ow + 4, 16) with a
// zero border of 2 - the pre-padded input of the next 6x6 stride-2 layer (its taps then index the buffer directly).
struct CostConv1K {
  const float* vol; int h, w; TV out; int oh, ow;
  float wt[36 * 16]; float bias[16];   // by value: the functor is the kernel's parameter block, so every weight is a constant-bank operand
  GV_HD void operator()(int64_t i) const {
    const int px = (int)(i % out.w); int64_t r = i / out.w; const int py = (int)(r % out.h); const int64_t m = r / out.h;
    float* o = out.p + (int64_t)m * out.sn + ((int64_t)py * out.w + px) * out.ld;
    const int oy = py - 2, ox = px - 2;
    float acc[16];
    if (oy < 0 || oy >= oh || ox < 0 || ox >= ow) {
#pragma unroll
      for (int c = 0; c < 16; ++c) acc[c] = 0.f;
    } else {
#pragma unroll
      for (int c = 0; c < 16; ++c) acc[c] = bias[c];
      const float* img = vol + m * (int64_t)h * w;
#pragma unroll
      for (int ky = 0; ky < 6; ++ky) {
        const int sy = oy * 2 + ky - 2;
        if (sy < 0 || sy >= h) continue;
#pragma unroll
        for (int kx = 0; kx < 6; ++kx) {
          const int sx = ox * 2 + kx - 2;
          if (sx < 0 || sx >= w) continue;
          const float a = img[(int64_t)sy * w + sx];
#pragma unroll
          for (int c = 0; c < 16; ++c) acc[c] = fmaf(a, wt[(ky * 6 + kx) * 16 + c], acc[c]);
        }
      }
#pragma unroll
      for (int c = 0; c < 16; ++c) acc[c] = acc[c] > 0.f ? acc[c] : 0.f;
    }
#pragma unroll
    for (int c = 0; c < 16; c += 4) { F4 t = {acc[c], acc[c + 1], acc[c + 2], acc[c + 3]}; st4(o + c, t); }
  }
};
void cost_conv1(Ctx& cx, const float* vol, int64_t maps, int h, int w, const float* wt_host, const float* bias_host, const TV& out_padded, int oh, int ow) {
  if (out_padded.n != maps || out_padded.h != oh + 4 || out_padded.w != ow + 4 || out_padded.c != 16 || out_padded.ld % 4 || (reinterpret_cast<uintptr_t>(out_padded.p) & 15))
    throw std::runtime_error("cost_conv1: shape mismatch");
  CostConv1K f;
  f.vol = vol; f.h = h; f.w = w; f.out = out_padded; f.oh = oh; f.ow = ow;
  std::memcpy(f.wt, wt_host, sizeof f.wt); std::memcpy(f.bias, bias_host, sizeof f.bias);
  parallel_for(cx, out_padded.pixels(), f, "cost_conv1_6x6s2");
}

// ------------------------------------------------------------------ GMA attention (gma.py:56-76): softmax over each row, in place,
// times `mul` (a power of two: the attention matrix is stored scaled so that its fp16 hi / lo split in the tensor-core aggregate GEMM
// keeps normal halves; the consumer's output scale undoes it)
struct RowSoftmaxK {
  float* p; int64_t cols; float mul;
  GV_HD void operator()(int64_t r) const {
    float* row = p + r * cols;
    float m = -3.0e38f;
    for (int64_t j = 0; j < cols; ++j) m = fmaxf(m, row[j]);
    float s = 0.f;
    for (int64_t j = 0; j < cols; ++j) { const float e = expf(row[j] - m); row[j] = e; s += e; }
    const float k = mul / s;
    for (int64_t j = 0; j < cols; ++j) row[j] *= k;
  }
};
#ifndef GV_HOSTSIM
__global__ void __launch_bounds__(256) row_softmax_kernel(float* p, int64_t rows, int64_t cols, float mul) {
  __shared__ float red[8];
  for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
    float* row = p + r * cols;
    float m = -3.0e38f;
    for (int64_t j = threadIdx.x; j < cols; j += 256) m = fmaxf(m, row[j]);
    for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = red[0];
    for (int k = 1; k < 8; ++k) m = fmaxf(m, red[k]);
    __syncthreads();
    float s = 0.f;
    for (int64_t j = threadIdx.x; j < cols; j += 256) { const float e = expf(row[j] - m); row[j] = e; s += e; }
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    s = 0.f;
    for (int k = 0; k < 8; ++k) s += red[k];
    __syncthreads();
    const float kk = mul / s;
    for (int64_t j = threadIdx.x; j < cols; j += 256) row[j] *= kk;
  }
}
#endif
void row_softmax(Ctx& cx, float* p, int64_t rows, int64_t cols, float mul) {
#ifndef GV_HOSTSIM
  if (cx.dry) return;
  cx.launches++;
  if (cx.prof) cx.prof->begin(cx.stream, "row_softmax", (double)rows * cols);
  int64_t blocks = rows, cap = (int64_t)cx.sm_count * 8;
  if (blocks > cap) blocks = cap;
  row_softmax_kernel<<<(unsigned)blocks, 256, 0, cx.stream>>>(p, rows, cols, mul);
  gv_check_launch("row_softmax");
  if (cx.prof) cx.prof->end(cx.stream);
#else
  parallel_for(cx, rows, RowSoftmaxK{p, cols, mul}, "row_softmax");
#endif
}

// ------------------------------------------------------------------ small GEMMs on the CUDA cores (fp32 mode / host simulation)
// out[i][d] = scale * sum_k A[i][k] * Bm[k][d]  (A: rows x K, row stride lda; Bm: K x D, row stride ldb): the GMA aggregate attn @ v
// (gma.py:104-105) when the tensor-core GEMM is not used.  Thread per output: A is a broadcast, Bm a coalesced load.
struct GemmNNK {
  const float* A; const float* Bm; float* out; int64_t K; int D; int64_t lda, ldb, ldo; float scale;
  GV_HD void operator()(int64_t i) const {
    const int d = (int)(i % D); const int64_t r = i / D;
    const float* a = A + r * lda;
    float s = 0.f;
    for (int64_t k = 0; k < K; ++k) s = fmaf(a[k], Bm[k * ldb + d], s);
    out[r * ldo + d] = s * scale;
  }
};
void gemm_nn(Ctx& cx, const float* A, const float* Bm, float* out, int64_t rows, int64_t K, int D, int64_t lda, int64_t ldb, int64_t ldo, float scale) {
  parallel_for(cx, rows * D, GemmNNK{A, Bm, out, K, D, lda, ldb, ldo, scale}, "gemm_nn_simt");
}
// dst[c][r] = src[r][c]  (rows x cols -> cols x rows): v^T as the K-major "weights" of the tensor-core aggregate GEMM
struct Transpose2dK {
  const float* src; float* dst; int64_t rows; int cols; int64_t lds;
  GV_HD void operator()(int64_t i) const {
    const int64_t r = i % rows; const int c = (int)(i / rows);
    dst[(int64_t)c * rows + r] = src[r * lds + c];
  }
};
void transpose_2d(Ctx& cx, const float* src, float* dst, int64_t rows, int cols, int64_t lds) {
  parallel_for(cx, rows * cols, Transpose2dK{src, dst, rows, cols, lds}, "transpose_2d");
}

// out = a + alpha * b, alpha read from device memory (GMA's learned gamma, gma.py:113)
struct AxpyDevK {
  TV a, b, out; const float* alpha;
  GV_HD void operator()(int64_t i) const {
    const int C = a.c;
    const int c = (int)(i % C); int64_t r = i / C;
    const int px = (int)(r % a.w); r /= a.w; const int py = (int)(r % a.h); const int n = (int)(r / a.h);
    out.p[out.off(n, py, px) + c] = a.p[a.off(n, py, px) + c] + alpha[0] * b.p[b.off(n, py, px) + c];
  }
};
void axpy_dev(Ctx& cx, const TV& a, const TV& b, const float* alpha, const TV& out) { parallel_for(cx, a.pixels() * a.c, AxpyDevK{a, b, out, alpha}, "axpy_gamma"); }

// broadcast a (1, 1, T, C) parameter block to every sample of `out` viewed as (n, h, w, C) with the token index = n % T ... used for the
// cost-perceiver's latent tokens as the residual of the input layer (encoder.py:466-468): out[n,y,x,:] = src[(n % T)*C + :]
struct BroadcastTokensK {
  const float* src; TV out; int T;
  GV_HD void operator()(int64_t i) const {
    const int C = out.c;
    const int c = (int)(i % C); int64_t r = i / C;
    const int px = (int)(r % out.w); r /= out.w; const int py = (int)(r % out.h); const int n = (int)(r / out.h);
    out.p[out.off(n, py, px) + c] = src[(n % T) * C + c];
  }
};
void broadcast_tokens(Ctx& cx, const float* src, const TV& out, int T) { parallel_for(cx, out.pixels() * out.c, BroadcastTokensK{src, out, T}, "broadcast_tokens"); }

}  // namespace gv
