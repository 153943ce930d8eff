// All-pairs correlation volume, its 2x2 average-pooled pyramid and the 4-level
// 9x9 bilinear lookup (reference: raft/corr.py:127-175, :23-93; sampler
// raft/utils/utils.py:66-80).  fp32 throughout (the RAFT recurrence amplifies
// rounding: see DESIGN.md "precision plan").
#include "common.h"

namespace gv {

// ----------------------------------------------------------------- volume
#ifndef GV_HOSTSIM
// C[n][i][j] = scale * sum_k A[n,i,k] * B[n,j,k];  128x128 tile, BK=16, 8x8 per thread.
__global__ void __launch_bounds__(256) corr_gemm_nt_kernel(TV fa, TV fb, float* __restrict__ vol, float scale) {
  const int M = fa.h * fa.w, K = fa.c;
  const int n = blockIdx.z;
  const int m0 = blockIdx.y * 128, n0 = blockIdx.x * 128;
  __shared__ float As[16][128 + 4];
  __shared__ float Bs[16][128 + 4];
  const int tid = threadIdx.x;
  const int tm = (tid / 16) * 8, tn = (tid % 16) * 8;
  const float* A = fa.p + (int64_t)n * fa.sn;
  const float* B = fb.p + (int64_t)n * fb.sn;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += 16) {
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      int f4 = tid + it * 256;       // 512 float4 per operand tile
      int row = f4 >> 2, q = f4 & 3;
      float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va;
      if (m0 + row < M) va = *reinterpret_cast<const float4*>(A + (int64_t)(m0 + row) * fa.ld + k0 + q * 4);
      if (n0 + row < M) vb = *reinterpret_cast<const float4*>(B + (int64_t)(n0 + row) * fb.ld + k0 + q * 4);
      As[q * 4 + 0][row] = va.x; As[q * 4 + 1][row] = va.y; As[q * 4 + 2][row] = va.z; As[q * 4 + 3][row] = va.w;
      Bs[q * 4 + 0][row] = vb.x; Bs[q * 4 + 1][row] = vb.y; Bs[q * 4 + 2][row] = vb.z; Bs[q * 4 + 3][row] = vb.w;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      float a[8], b[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) { a[i] = As[k][tm + i]; b[i] = Bs[k][tn + i]; }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* C = vol + (int64_t)n * M * M;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int r = m0 + tm + i;
    if (r >= M) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int c = n0 + tn + j;
      if (c < M) C[(int64_t)r * M + c] = acc[i][j] * scale;
    }
  }
}
#endif

void corr_volume(Ctx& cx, const TV& fa, const TV& fb, float* vol, float scale) {
  if (cx.dry) return;
  cx.launches++;
  const int M = fa.h * fa.w;
#ifdef GV_HOSTSIM
  const int K = fa.c;
  for (int n = 0; n < fa.n; ++n) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < M; ++i) {
      const float* a = fa.p + (int64_t)n * fa.sn + (int64_t)i * fa.ld;
      for (int j = 0; j < M; ++j) {
        const float* b = fb.p + (int64_t)n * fb.sn + (int64_t)j * fb.ld;
        float s = 0.f;
        for (int k = 0; k < K; ++k) s += a[k] * b[k];
        vol[((int64_t)n * M + i) * M + j] = s * scale;
      }
    }
  }
#else
  if (fa.c % 16 != 0 || fa.ld % 4 != 0 || fb.ld % 4 != 0) throw std::runtime_error("corr_volume: feature dim must be a multiple of 16");
  dim3 grid((M + 127) / 128, (M + 127) / 128, fa.n);
  if (cx.prof) cx.prof->begin(cx.stream, "corr_gemm_nt", 2.0 * fa.n * (double)M * M * fa.c);
  corr_gemm_nt_kernel<<<grid, 256, 0, cx.stream>>>(fa, fb, vol, scale);
  gv_check_launch("corr_volume");
  if (cx.prof) cx.prof->end(cx.stream);
#endif
}

// [2][pixels][c] planes for the 3xTF32 correlation GEMM: rn_tf32(x) and rn_tf32(x - rn_tf32(x))
struct SplitPlanesK {
  TV src; float* planes; int64_t plane;
  GV_HD float rn(float x) const {  // round-to-nearest-even to TF32
    uint32_t u; memcpy(&u, &x, 4);
    u += 0xfffu + ((u >> 13) & 1u); u &= 0xffffe000u;
    float y; memcpy(&y, &u, 4); return y;
  }
  GV_HD void operator()(int64_t i) const {
    int c = (int)(i % src.c); int64_t px = i / src.c;
    int x = (int)(px % src.w); int64_t r = px / src.w; int y = (int)(r % src.h); int n = (int)(r / src.h);
    float v = src.p[src.off(n, y, x) + c];
    float hi = rn(v);
    planes[i] = hi; planes[plane + i] = rn(v - hi);
  }
};
void split_planes(Ctx& cx, const TV& src, float* planes) {
  int64_t n = src.pixels() * src.c;
  parallel_for(cx, n, SplitPlanesK{src, planes, n}, "split_planes");
}
// half [2][pixels][c] planes for the 3xF16 correlation GEMM: hi = rn_f16(x), lo = rn_f16(x - hi)  (feature maps are O(1): no scaling)
struct SplitPlanesF16K {
  TV src; uint16_t* planes; int64_t plane;
  GV_HD void operator()(int64_t i) const {
    int c = (int)(i % src.c); int64_t px = i / src.c;
    int x = (int)(px % src.w); int64_t r = px / src.w; int y = (int)(r % src.h); int n = (int)(r / src.h);
    const float v = src.p[src.off(n, y, x) + c];
    const uint16_t hi = gv_f2h(v);
    planes[i] = hi; planes[plane + i] = gv_f2h(v - gv_h2f(hi));
  }
};
void split_planes_f16(Ctx& cx, const TV& src, void* planes) {
  int64_t n = src.pixels() * src.c;
  parallel_for(cx, n, SplitPlanesF16K{src, static_cast<uint16_t*>(planes), n}, "split_planes");
}
#ifdef GV_HOSTSIM
// (the host simulation takes the TF32 planes: corr_volume_tc_wants_f16_planes() is false there)
void corr_gemm_3xf16(Ctx&, const void*, int64_t, int, const void*, int64_t, int, int, float, float*) {
  throw std::runtime_error("corr_gemm_3xf16 is a tensor-core kernel; not available in the host simulation");
}
#endif

// 2x2 average of an NHWC feature map (floor semantics): the targets of pyramid level l are the level-(l-1) features pooled
struct PoolFeatK {
  TV src, dst;
  GV_HD void operator()(int64_t i) const {
    const int c = (int)(i % dst.c); int64_t r = i / dst.c;
    const int x = (int)(r % dst.w); r /= dst.w; const int y = (int)(r % dst.h); const int n = (int)(r / dst.h);
    const float* s = src.p + src.off(n, 2 * y, 2 * x) + c;
    const int64_t dx = src.ld, dy = (int64_t)src.w * src.ld;
    dst.p[dst.off(n, y, x) + c] = (s[0] + s[dx] + s[dy] + s[dy + dx]) * 0.25f;
  }
};
void avgpool2_features(Ctx& cx, const TV& src, const TV& dst) {
  parallel_for(cx, dst.pixels() * dst.c, PoolFeatK{src, dst}, "avgpool2_features");
}

// ------------------------------------------------------------------- pool
// F.avg_pool2d(corr, 2, stride=2) over the trailing (h, w) image of every row (raft/corr.py:139-142).
struct CorrPoolK {
  const float* src; float* dst; int h, w, ho, wo;
  GV_HD void operator()(int64_t i) const {
    int x = (int)(i % wo); int64_t r = i / wo; int y = (int)(r % ho); int64_t row = r / ho;
    const float* s = src + row * ((int64_t)h * w) + (int64_t)(2 * y) * w + 2 * x;
    dst[i] = (s[0] + s[1] + s[w] + s[w + 1]) * 0.25f;
  }
};
void corr_pool(Ctx& cx, const float* src, float* dst, int64_t rows, int h, int w) {
  int ho = h / 2, wo = w / 2;
  parallel_for(cx, rows * ho * wo, CorrPoolK{src, dst, h, w, ho, wo}, "corr_pool");
}

#ifndef GV_HOSTSIM
// All three pooled levels of one correlation row in one pass: level 0 is read from HBM once, levels 1 and 2 stay in
// shared memory for their successors (the per-level kernels re-read 1.3x the bytes).  One CTA per row (n, pixel).
__global__ void __launch_bounds__(256) corr_pyramid_kernel(const float* __restrict__ l0, float* __restrict__ l1, float* __restrict__ l2,
                                                            float* __restrict__ l3, int64_t rows, int h, int w) {
  extern __shared__ float sm[];
  const int h1 = h / 2, w1 = w / 2, h2 = h1 / 2, w2 = w1 / 2, h3 = h2 / 2, w3 = w2 / 2;
  float* s1 = sm; float* s2 = sm + h1 * w1;
  for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const float* src = l0 + row * ((int64_t)h * w);
    float* d1 = l1 + row * ((int64_t)h1 * w1);
    if ((w & 3) == 0) {   // two pooled values per thread from one float4 per source row (16-byte aligned: w % 4 == 0)
      const int wp = w1 >> 1;
#pragma unroll 4
      for (int i = threadIdx.x; i < h1 * wp; i += blockDim.x) {
        const int y = i / wp, xp = i - y * wp;
        const float* s = src + (int64_t)(2 * y) * w + 4 * xp;
        const float4 a = __ldcs(reinterpret_cast<const float4*>(s)), b = __ldcs(reinterpret_cast<const float4*>(s + w));
        const float2 v = make_float2((a.x + a.y + b.x + b.y) * 0.25f, (a.z + a.w + b.z + b.w) * 0.25f);
        *reinterpret_cast<float2*>(s1 + y * w1 + 2 * xp) = v;
        *reinterpret_cast<float2*>(d1 + y * w1 + 2 * xp) = v;
      }
    } else
    for (int i = threadIdx.x; i < h1 * w1; i += blockDim.x) {
      const int y = i / w1, x = i - y * w1;
      const float* s = src + (int64_t)(2 * y) * w + 2 * x;
      float2 a, b;
      if ((w & 1) == 0) { a = __ldcs(reinterpret_cast<const float2*>(s)); b = __ldcs(reinterpret_cast<const float2*>(s + w)); }
      else { a = make_float2(s[0], s[1]); b = make_float2(s[w], s[w + 1]); }
      const float v = (a.x + a.y + b.x + b.y) * 0.25f;
      s1[i] = v; d1[i] = v;
    }
    __syncthreads();
    float* d2 = l2 + row * ((int64_t)h2 * w2);
    for (int i = threadIdx.x; i < h2 * w2; i += blockDim.x) {
      const int y = i / w2, x = i - y * w2;
      const float* s = s1 + (2 * y) * w1 + 2 * x;
      const float v = (s[0] + s[1] + s[w1] + s[w1 + 1]) * 0.25f;
      s2[i] = v; d2[i] = v;
    }
    __syncthreads();
    float* d3 = l3 + row * ((int64_t)h3 * w3);
    for (int i = threadIdx.x; i < h3 * w3; i += blockDim.x) {
      const int y = i / w3, x = i - y * w3;
      const float* s = s2 + (2 * y) * w2 + 2 * x;
      d3[i] = (s[0] + s[1] + s[w2] + s[w2 + 1]) * 0.25f;
    }
    __syncthreads();   // s1/s2 are rewritten by the next row
  }
}
#endif

// levels 1..3 of the pyramid from level 0 (raft/corr.py:139-142: three successive avg_pool2d(2, 2))
void corr_pool_pyramid(Ctx& cx, const float* l0, float* l1, float* l2, float* l3, int64_t rows, int h, int w) {
#ifndef GV_HOSTSIM
  const int h1 = h / 2, w1 = w / 2, h2 = h1 / 2, w2 = w1 / 2;
  const size_t smem = ((size_t)h1 * w1 + (size_t)h2 * w2) * sizeof(float);
  if (smem <= 96 * 1024 && h2 / 2 > 0 && w2 / 2 > 0) {
    if (cx.dry) return;
    cx.launches++;
    static volatile unsigned char attr[64];
    gv_set_max_smem(corr_pyramid_kernel, 96 * 1024, attr);
    if (cx.prof) cx.prof->begin(cx.stream, "corr_pool_pyramid", (double)rows * h * w);
    const int64_t grid = rows < (int64_t)cx.sm_count * 8 ? rows : (int64_t)cx.sm_count * 8;
    corr_pyramid_kernel<<<(unsigned)grid, 256, smem, cx.stream>>>(l0, l1, l2, l3, rows, h, w);
    gv_check_launch("corr_pool_pyramid");
    if (cx.prof) cx.prof->end(cx.stream);
    return;
  }
#endif
  corr_pool(cx, l0, l1, rows, h, w);
  corr_pool(cx, l1, l2, rows, h / 2, w / 2);
  corr_pool(cx, l2, l3, rows, h / 4, w / 4);
}

// ----------------------------------------------------------------- lookup
// raft/corr.py:144-165.  out channel = lvl*81 + a*9 + b samples level `lvl` of row
// (n, pixel) at (x/2^lvl + (a-4), y/2^lvl + (b-4)) — the "transposed window" of the
// reference's meshgrid(dy, dx) — bilinear, zero padding, align_corners=True, going
// through the same normalise / un-normalise float round trip as bilinear_sampler +
// grid_sample.
struct CorrLookupK {
  CorrPyr pyr; TV coords, out;
  GV_HD void operator()(int64_t i) const {
    const int nch = pyr.nl * 81;
    int ch = (int)(i % nch); int64_t r = i / nch;
    int x = (int)(r % coords.w); r /= coords.w; int y = (int)(r % coords.h); int n = (int)(r / coords.h);
    int lvl = ch / 81, k = ch % 81, a = k / 9, b = k % 9;
    const float* c = coords.p + coords.off(n, y, x);
    float inv = 1.0f / (float)(1 << lvl);
    int H = pyr.h[lvl], W = pyr.w[lvl];
    float px = c[0] * inv + (float)(a - 4);
    float py = c[1] * inv + (float)(b - 4);
    float xg = 2.f * px / (float)(W - 1) - 1.f;
    float yg = 2.f * py / (float)(H - 1) - 1.f;
    float ix = ((xg + 1.f) / 2.f) * (float)(W - 1);
    float iy = ((yg + 1.f) / 2.f) * (float)(H - 1);
    float x0f = floorf(ix), y0f = floorf(iy);
    int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
    float wx1 = ix - x0f, wx0 = (x0f + 1.f) - ix, wy1 = iy - y0f, wy0 = (y0f + 1.f) - iy;
    int64_t row = (int64_t)n * pyr.rows_per_sample + (int64_t)y * coords.w + x;
    const float* img = pyr.lvl[lvl] + row * ((int64_t)H * W);
    float v = 0.f;
    bool vx0 = x0 >= 0 && x0 < W, vx1 = x1 >= 0 && x1 < W, vy0 = y0 >= 0 && y0 < H, vy1 = y1 >= 0 && y1 < H;
    if (vy0 && vx0) v += img[(int64_t)y0 * W + x0] * (wx0 * wy0);
    if (vy0 && vx1) v += img[(int64_t)y0 * W + x1] * (wx1 * wy0);
    if (vy1 && vx0) v += img[(int64_t)y1 * W + x0] * (wx0 * wy1);
    if (vy1 && vx1) v += img[(int64_t)y1 * W + x1] * (wx1 * wy1);
    out.p[out.off(n, y, x) + ch] = v;
  }
};
#ifndef GV_HOSTSIM
// One warp per (source pixel, level): the 9 x-offsets and 9 y-offsets of the window go through the grid_sample round trip ONCE
// (lanes 0..8 / 9..17: 18 coordinate evaluations instead of 2 x 81), the 81 outputs take their (x0, wx) / (y0, wy) by shuffle and issue
// their four taps back to back; a warp's stores are 32 consecutive channels.  Arithmetic and summation order are those of CorrLookupK
// (bit-identical results); the thread-per-output form spent ~100 instructions per output on the coordinate transform.
__global__ void __launch_bounds__(256) corr_lookup_warp_kernel(CorrPyr pyr, TV coords, TV out, int64_t n_items) {
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t it = warp0; it < n_items; it += nwarps) {
    const int lvl = (int)(it % pyr.nl); int64_t r = it / pyr.nl;
    const int x = (int)(r % coords.w); r /= coords.w; const int y = (int)(r % coords.h); const int n = (int)(r / coords.h);
    const float* c = coords.p + coords.off(n, y, x);
    const float inv = 1.0f / (float)(1 << lvl);
    const int H = pyr.h[lvl], W = pyr.w[lvl];
    // lane l < 9: x offset a = l; lanes 9..17: y offset b = l - 9
    const bool isx = lane < 9;
    const int d = isx ? lane : lane - 9;
    const int S = isx ? W : H;
    const float pc = (isx ? c[0] : c[1]) * inv + (float)(d - 4);
    const float g = 2.f * pc / (float)(S - 1) - 1.f;
    const float ic = ((g + 1.f) / 2.f) * (float)(S - 1);
    const float c0f = floorf(ic);
    const int my0 = (int)c0f;
    const float mw1 = ic - c0f, mw0 = (c0f + 1.f) - ic;
    const int64_t row = (int64_t)n * pyr.rows_per_sample + (int64_t)y * coords.w + x;
    const float* img = pyr.lvl[lvl] + row * ((int64_t)H * W);
    float* o = out.p + out.off(n, y, x) + lvl * 81;
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {
      const int k = pass * 32 + lane, kk = k < 81 ? k : 80;
      const int a = kk / 9, b = kk - a * 9;
      const int x0 = __shfl_sync(0xffffffffu, my0, a), y0 = __shfl_sync(0xffffffffu, my0, 9 + b);
      const float wx0 = __shfl_sync(0xffffffffu, mw0, a), wx1 = __shfl_sync(0xffffffffu, mw1, a);
      const float wy0 = __shfl_sync(0xffffffffu, mw0, 9 + b), wy1 = __shfl_sync(0xffffffffu, mw1, 9 + b);
      if (k < 81) {
        const int x1 = x0 + 1, y1 = y0 + 1;
        const bool vx0 = x0 >= 0 && x0 < W, vx1 = x1 >= 0 && x1 < W, vy0 = y0 >= 0 && y0 < H, vy1 = y1 >= 0 && y1 < H;
        const float t00 = (vy0 && vx0) ? __ldg(img + (int64_t)y0 * W + x0) : 0.f, t01 = (vy0 && vx1) ? __ldg(img + (int64_t)y0 * W + x1) : 0.f;
        const float t10 = (vy1 && vx0) ? __ldg(img + (int64_t)y1 * W + x0) : 0.f, t11 = (vy1 && vx1) ? __ldg(img + (int64_t)y1 * W + x1) : 0.f;
        float v = 0.f;
        if (vy0 && vx0) v += t00 * (wx0 * wy0);
        if (vy0 && vx1) v += t01 * (wx1 * wy0);
        if (vy1 && vx0) v += t10 * (wx0 * wy1);
        if (vy1 && vx1) v += t11 * (wx1 * wy1);
        o[k] = v;
      }
    }
  }
}
#endif
void corr_lookup(Ctx& cx, const CorrPyr& pyr, const TV& coords, const TV& out) {
#ifndef GV_HOSTSIM
  if (!out.f16 && !coords.f16) {
    if (cx.dry) return;
    cx.launches++;
    const int64_t items = coords.pixels() * pyr.nl;
    if (cx.prof) cx.prof->begin(cx.stream, "corr_lookup", (double)coords.pixels() * pyr.nl * 81);
    int64_t blocks = (items + 7) / 8, cap = (int64_t)cx.sm_count * 16;
    if (blocks > cap) blocks = cap;
    corr_lookup_warp_kernel<<<(unsigned)blocks, 256, 0, cx.stream>>>(pyr, coords, out, items);
    gv_check_launch("corr_lookup");
    if (cx.prof) cx.prof->end(cx.stream);
    return;
  }
#endif
  parallel_for(cx, coords.pixels() * pyr.nl * 81, CorrLookupK{pyr, coords, out}, "corr_lookup");
}

// -------------------------------------------------------- volume-free lookup
// BidirCorrBlock (raft/corr.py:23-93) is looked up ONCE per interpolated frame: building the all-pairs volume pyramid for it writes
// N^2 x 4/3 x 2 values (11 GB at 1088x1920) to read back 2 x N x 324.  Bilinear interpolation of the volume is linear in the volume,
// and a level-l volume entry is the dot product with the 2^l x 2^l average-pooled target feature, so the 81 window samples of a level
// only need the dot products with the (at most) 10 x 10 integer neighbours of the window: 100 dots of 256 channels per (pixel, level)
// = 8.6 GFLOP per pair instead of the 1.45 TFLOP GEMM.  Target features are IEEE half (the same 11-bit significand the plain-TF32
// volume GEMM gave them), the source feature and the accumulation are fp32.
struct ToHalfK {
  TV src; uint16_t* dst;
  GV_HD void operator()(int64_t i) const {
    const int c = (int)(i % src.c); int64_t r = i / src.c;
    const int x = (int)(r % src.w); r /= src.w; const int y = (int)(r % src.h); const int n = (int)(r / src.h);
    dst[i] = gv_f2h(src.p[src.off(n, y, x) + c]);
  }
};
void features_to_half(Ctx& cx, const TV& src, void* dst) {
  parallel_for(cx, src.pixels() * src.c, ToHalfK{src, static_cast<uint16_t*>(dst)}, "features_to_half");
}

// grid_sample(align_corners=True) round trip of one window coordinate (raft/utils/utils.py:66-80), as CorrLookupK evaluates it
GV_HD void corr_axis(float c, float inv, int d, int S, int& i0, float& w0, float& w1) {
  const float pc = c * inv + (float)(d - 4);
  const float g = 2.f * pc / (float)(S - 1) - 1.f;
  const float ic = ((g + 1.f) / 2.f) * (float)(S - 1);
  const float c0f = floorf(ic);
  i0 = (int)c0f; w1 = ic - c0f; w0 = (c0f + 1.f) - ic;
}

// thread-per-output form (host build of the engine; the reference for the warp kernel below): four taps, each a C-channel dot
struct CorrLookupDirectK {
  TV src; CorrFeat tgt; TV coords, out;
  GV_HD float dot(const float* a, int n, int lvl, int ty, int tx) const {
    const uint16_t* b = tgt.lvl[lvl] + ((int64_t)n * tgt.h[lvl] * tgt.w[lvl] + (int64_t)ty * tgt.w[lvl] + tx) * tgt.c;
    float acc = 0.f;
    for (int k = 0; k < tgt.c; ++k) acc = fmaf(a[k], gv_h2f(b[k]), acc);
    return acc * tgt.scale;
  }
  GV_HD void operator()(int64_t i) const {
    const int ch = (int)(i % 324); int64_t r = i / 324;
    const int x = (int)(r % coords.w); r /= coords.w; const int y = (int)(r % coords.h); const int n = (int)(r / coords.h);
    const int lvl = ch / 81, k = ch % 81, a = k / 9, b = k % 9;
    const float* c = coords.p + coords.off(n, y, x);
    const float inv = 1.0f / (float)(1 << lvl);
    const int H = tgt.h[lvl], W = tgt.w[lvl];
    int x0, y0; float wx0, wx1, wy0, wy1;
    corr_axis(c[0], inv, a, W, x0, wx0, wx1);
    corr_axis(c[1], inv, b, H, y0, wy0, wy1);
    const int x1 = x0 + 1, y1 = y0 + 1;
    const float* f = src.p + src.off(n, y, x);
    const bool vx0 = x0 >= 0 && x0 < W, vx1 = x1 >= 0 && x1 < W, vy0 = y0 >= 0 && y0 < H, vy1 = y1 >= 0 && y1 < H;
    float v = 0.f;
    if (vy0 && vx0) v += dot(f, n, lvl, y0, x0) * (wx0 * wy0);
    if (vy0 && vx1) v += dot(f, n, lvl, y0, x1) * (wx1 * wy0);
    if (vy1 && vx0) v += dot(f, n, lvl, y1, x0) * (wx0 * wy1);
    if (vy1 && vx1) v += dot(f, n, lvl, y1, x1) * (wx1 * wy1);
    out.p[out.off(n, y, x) + ch] = v;
  }
};

#ifndef GV_HOSTSIM
// One warp per (source pixel, level); the 8 warps of a CTA take 8 x-adjacent pixels of one level, whose windows overlap by ~90 % and
// stay in L1.  A lane owns 8 of the 256 channels: the source feature sits in registers, every neighbour costs one 16-byte load per
// lane (512 contiguous bytes per warp), and 32 neighbours at a time are reduced across the warp with a transposing butterfly
// (31 shuffles for 32 sums).  The 100 dots land in shared memory; the 81 outputs are then the four-tap blends of CorrLookupK.
constexpr int CLD_WARPS = 8;
__global__ void __launch_bounds__(256) corr_lookup_direct_kernel(TV src, CorrFeat tgt, TV coords, TV out, int xblocks, int64_t n_groups) {
  __shared__ float dots_s[CLD_WARPS][128];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* dots = dots_s[warp];
  for (int64_t grp = blockIdx.x; grp < n_groups; grp += gridDim.x) {
    int64_t r = grp;
    const int xb = (int)(r % xblocks); r /= xblocks;
    const int y = (int)(r % coords.h); r /= coords.h;
    const int n = (int)(r % coords.n); const int lvl = (int)(r / coords.n);
    const int x = xb * CLD_WARPS + warp;
    if (x < coords.w) {   // (warp-uniform)
      const float* c = coords.p + coords.off(n, y, x);
      const float inv = 1.0f / (float)(1 << lvl);
      const int H = tgt.h[lvl], W = tgt.w[lvl];
      const bool isx = lane < 9;
      int my0; float mw0, mw1;
      corr_axis(isx ? c[0] : c[1], inv, isx ? lane : (lane < 18 ? lane - 9 : 0), isx ? W : H, my0, mw0, mw1);
      const int bx = __shfl_sync(0xffffffffu, my0, 0), by = __shfl_sync(0xffffffffu, my0, 9);
      float f[8];
      {
        const float4* fp = reinterpret_cast<const float4*>(src.p + src.off(n, y, x) + lane * 8);
        const float4 f0 = __ldg(fp), f1 = __ldg(fp + 1);
        f[0] = f0.x; f[1] = f0.y; f[2] = f0.z; f[3] = f0.w; f[4] = f1.x; f[5] = f1.y; f[6] = f1.z; f[7] = f1.w;
      }
      const uint16_t* tb = tgt.lvl[lvl] + (int64_t)n * H * W * 256 + lane * 8;
#pragma unroll 1
      for (int g = 0; g < 4; ++g) {
        float p[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int nb = g * 32 + j;           // neighbour (gy, gx) of the 10 x 10 grid based at (by, bx)
          const int gy = nb / 10, gx = nb - gy * 10;
          const int ty = by + gy, tx = bx + gx;
          float acc = 0.f;
          if (nb < 100 && ty >= 0 && ty < H && tx >= 0 && tx < W) {
            const uint4 q = __ldg(reinterpret_cast<const uint4*>(tb + ((int64_t)ty * W + tx) * 256));
            const float2 a0 = __half22float2(*reinterpret_cast<const __half2*>(&q.x)), a1 = __half22float2(*reinterpret_cast<const __half2*>(&q.y));
            const float2 a2 = __half22float2(*reinterpret_cast<const __half2*>(&q.z)), a3 = __half22float2(*reinterpret_cast<const __half2*>(&q.w));
            acc = fmaf(f[0], a0.x, acc); acc = fmaf(f[1], a0.y, acc); acc = fmaf(f[2], a1.x, acc); acc = fmaf(f[3], a1.y, acc);
            acc = fmaf(f[4], a2.x, acc); acc = fmaf(f[5], a2.y, acc); acc = fmaf(f[6], a3.x, acc); acc = fmaf(f[7], a3.y, acc);
          }
          p[j] = acc;
        }
        // transposing reduction: after the step with stride s, a lane keeps the half of the neighbour indices whose bit s equals its own
#pragma unroll
        for (int s = 16; s >= 1; s >>= 1) {
          const bool up = (lane & s) != 0;
#pragma unroll
          for (int i = 0; i < s; ++i) {
            const float send = up ? p[i] : p[i + s], keep = up ? p[i + s] : p[i];
            p[i] = keep + __shfl_xor_sync(0xffffffffu, send, s);
          }
        }
        dots[g * 32 + lane] = p[0] * tgt.scale;
      }
      __syncwarp();
      float* o = out.p + out.off(n, y, x) + lvl * 81;
#pragma unroll
      for (int pass = 0; pass < 3; ++pass) {
        const int k = pass * 32 + lane, kk = k < 81 ? k : 80;
        const int a = kk / 9, b = kk - a * 9;
        int x0 = __shfl_sync(0xffffffffu, my0, a), y0 = __shfl_sync(0xffffffffu, my0, 9 + b);
        float wx0 = __shfl_sync(0xffffffffu, mw0, a), wx1 = __shfl_sync(0xffffffffu, mw1, a);
        float wy0 = __shfl_sync(0xffffffffu, mw0, 9 + b), wy1 = __shfl_sync(0xffffffffu, mw1, 9 + b);
        if (k < 81) {
          // window column a normally starts at bx + a; a floor() that lands one off through rounding moves the (then ~zero-weight)
          // far tap outside the 10-wide grid: fold it onto the grid edge
          int ix = x0 - bx, iy = y0 - by;
          if (ix < 0) { ix = 0; x0 = bx; wx0 = wx1; wx1 = 0.f; } else if (ix > 8) { ix = 8; x0 = bx + 8; wx1 = wx0; wx0 = 0.f; }
          if (iy < 0) { iy = 0; y0 = by; wy0 = wy1; wy1 = 0.f; } else if (iy > 8) { iy = 8; y0 = by + 8; wy1 = wy0; wy0 = 0.f; }
          const int x1 = x0 + 1, y1 = y0 + 1;
          const bool vx0 = x0 >= 0 && x0 < W, vx1 = x1 >= 0 && x1 < W, vy0 = y0 >= 0 && y0 < H, vy1 = y1 >= 0 && y1 < H;
          const float* d = dots + iy * 10 + ix;
          float v = 0.f;
          if (vy0 && vx0) v += d[0] * (wx0 * wy0);
          if (vy0 && vx1) v += d[1] * (wx1 * wy0);
          if (vy1 && vx0) v += d[10] * (wx0 * wy1);
          if (vy1 && vx1) v += d[11] * (wx1 * wy1);
          o[k] = v;
        }
      }
      __syncwarp();
    }
  }
}
#endif

bool corr_lookup_direct_supported(const TV& src, const CorrFeat& tgt, const TV& coords, const TV& out) {
  return !src.f16 && !coords.f16 && !out.f16 && src.c == 256 && tgt.c == 256 && src.ld % 4 == 0 && src.sn % 4 == 0 &&
         (reinterpret_cast<uintptr_t>(src.p) & 15) == 0 && src.h == coords.h && src.w == coords.w && src.n == coords.n && out.c >= 324;
}

void corr_lookup_direct(Ctx& cx, const TV& src, const CorrFeat& tgt, const TV& coords, const TV& out) {
  if (!corr_lookup_direct_supported(src, tgt, coords, out)) throw std::runtime_error("corr_lookup_direct: unsupported tensor layout");
#ifndef GV_HOSTSIM
  if (cx.dry) return;
  cx.launches++;
  for (int l = 0; l < 4; ++l)
    if ((reinterpret_cast<uintptr_t>(tgt.lvl[l]) & 15) != 0) throw std::runtime_error("corr_lookup_direct: target features must be 16-byte aligned");
  const int xblocks = (coords.w + CLD_WARPS - 1) / CLD_WARPS;
  const int64_t groups = (int64_t)4 * coords.n * coords.h * xblocks;
  if (cx.prof) cx.prof->begin(cx.stream, "corr_lookup_direct", (double)coords.pixels() * 4 * 100 * 256 * 2);
  int64_t blocks = groups, cap = (int64_t)cx.sm_count * 8;
  if (blocks > cap) blocks = cap;
  corr_lookup_direct_kernel<<<(unsigned)blocks, 256, 0, cx.stream>>>(src, tgt, coords, out, xblocks, groups);
  gv_check_launch("corr_lookup_direct");
  if (cx.prof) cx.prof->end(cx.stream);
#else
  parallel_for(cx, coords.pixels() * 324, CorrLookupDirectK{src, tgt, coords, out}, "corr_lookup_direct");
#endif
}

// ------------------------------------------------ memory-free correlation with gradients (alt_cuda_corr)
// flowformer/alt_cuda_corr/correlation_kernel.cu for training: fp32 features of any C, any radius, N coordinate sets per pixel.
// Output (k = ky + rd * kx) of source pixel p blends the dots D[iy][ix] = <fmap1[p], fmap2[y0 - r + iy][x0 - r + ix]> of its
// (rd + 1)^2 window as D[ky][kx] (1-dy)(1-dx) + D[ky][kx+1] (1-dy) dx + D[ky+1][kx] dy (1-dx) + D[ky+1][kx+1] dy dx (the weights of
// the reference's se / sw / ne / nw terms, :97-114), off-frame dots being 0.
GV_HD AltCell alt_corr_cell(float x, float y, int r, int H2, int W2) {
  AltCell q;
  q.x0 = q.y0 = 0; q.dx = q.dy = 0.f;
  // NaN fails every comparison; outside these bounds all rd + 1 columns (rows) of the window miss fmap2
  q.in = x >= -(float)(r + 2) && x < (float)(W2 + r + 1) && y >= -(float)(r + 2) && y < (float)(H2 + r + 1);
  if (q.in) {
    const float fx = floorf(x), fy = floorf(y);
    q.x0 = (int)fx; q.y0 = (int)fy; q.dx = x - fx; q.dy = y - fy;
  }
  return q;
}
GV_HD float alt_corr_blend(float d00, float d01, float d10, float d11, float dx, float dy) {
  return d00 * ((1.f - dy) * (1.f - dx)) + d01 * ((1.f - dy) * dx) + d10 * (dy * (1.f - dx)) + d11 * (dy * dx);
}
// d(output)/dx and d(output)/dy of that blend (the floor held fixed)
GV_HD void alt_corr_dblend(float d00, float d01, float d10, float d11, float dx, float dy, float& gx, float& gy) {
  gx = (1.f - dy) * (d01 - d00) + dy * (d11 - d10);
  gy = (1.f - dx) * (d10 - d00) + dx * (d11 - d01);
}
// gradient reaching tap (iy, ix) from the (up to) four outputs that read it; g(ky, kx) = incoming gradient of output ky + rd * kx
template <class Gf> GV_HD float alt_corr_tap_grad(const Gf& g, int iy, int ix, int rd, float dx, float dy) {
  float s = 0.f;
  if (iy < rd && ix < rd) s += g(iy, ix) * ((1.f - dy) * (1.f - dx));
  if (iy < rd && ix > 0) s += g(iy, ix - 1) * ((1.f - dy) * dx);
  if (iy > 0 && ix < rd) s += g(iy - 1, ix) * (dy * (1.f - dx));
  if (iy > 0 && ix > 0) s += g(iy - 1, ix - 1) * (dy * dx);
  return s;
}

#ifdef GV_HOSTSIM
// host forms: one item per output element (forward) / per source pixel (backward), every dot a plain loop over C
struct AltCorrDot {
  AltCorrArgs a;
  float operator()(int b, int h, int w, int ty, int tx) const {
    if (ty < 0 || ty >= a.H2 || tx < 0 || tx >= a.W2) return 0.f;
    const float* p = a.f1 + (((int64_t)b * a.H1 + h) * a.W1 + w) * a.C;
    const float* q = a.f2 + (((int64_t)b * a.H2 + ty) * a.W2 + tx) * a.C;
    float s = 0.f;
    for (int c = 0; c < a.C; ++c) s = fmaf(p[c], q[c], s);
    return s;
  }
};
struct AltCorrFwdK {
  AltCorrArgs a; float* out;
  void operator()(int64_t i) const {
    const int rd = 2 * a.r + 1, K = rd * rd;
    int64_t t = i;
    const int w = (int)(t % a.W1); t /= a.W1; const int h = (int)(t % a.H1); t /= a.H1;
    const int k = (int)(t % K); t /= K; const int n = (int)(t % a.N); const int b = (int)(t / a.N);
    const float* cp = a.coords + ((((int64_t)b * a.N + n) * a.H1 + h) * a.W1 + w) * 2;
    const AltCell q = alt_corr_cell(cp[0], cp[1], a.r, a.H2, a.W2);
    float v = 0.f;
    if (q.in) {
      const AltCorrDot D{a};
      const int kx = k / rd, ky = k - kx * rd, ty = q.y0 - a.r + ky, tx = q.x0 - a.r + kx;
      v = alt_corr_blend(D(b, h, w, ty, tx), D(b, h, w, ty, tx + 1), D(b, h, w, ty + 1, tx), D(b, h, w, ty + 1, tx + 1), q.dx, q.dy);
    }
    out[i] = v;
  }
};
struct AltCorrBwdK {
  AltCorrArgs a; const float* cgrad; float* f1g; float* f2g; float* cog;
  void operator()(int64_t i) const {
    const int rd = 2 * a.r + 1, K = rd * rd, wd = rd + 1;
    const int w = (int)(i % a.W1), h = (int)(i / a.W1 % a.H1), b = (int)(i / a.W1 / a.H1);
    const int64_t HW1 = (int64_t)a.H1 * a.W1;
    const float* f1p = a.f1 + i * a.C;
    float* g1 = f1g ? f1g + i * a.C : nullptr;
    if (g1) for (int c = 0; c < a.C; ++c) g1[c] = 0.f;
    const AltCorrDot D{a};
    for (int n = 0; n < a.N; ++n) {
      const int64_t pn = ((int64_t)b * a.N + n) * HW1 + (int64_t)h * a.W1 + w;   // (b, n, h, w)
      const AltCell q = alt_corr_cell(a.coords[pn * 2], a.coords[pn * 2 + 1], a.r, a.H2, a.W2);
      if (!q.in) {
        if (cog) { cog[pn * 2] = 0.f; cog[pn * 2 + 1] = 0.f; }
        continue;
      }
      const float* gp = cgrad + ((int64_t)b * a.N + n) * K * HW1 + (int64_t)h * a.W1 + w;
      auto g = [&](int ky, int kx) { return gp[(int64_t)(ky + rd * kx) * HW1]; };
      for (int iy = 0; iy < wd; ++iy)
        for (int ix = 0; ix < wd; ++ix) {
          const int ty = q.y0 - a.r + iy, tx = q.x0 - a.r + ix;
          if (ty < 0 || ty >= a.H2 || tx < 0 || tx >= a.W2) continue;
          const float G = alt_corr_tap_grad(g, iy, ix, rd, q.dx, q.dy);
          const int64_t o2 = (((int64_t)b * a.H2 + ty) * a.W2 + tx) * a.C;
          for (int c = 0; c < a.C; ++c) {
            if (g1) g1[c] += G * a.f2[o2 + c];
            if (f2g) atomic_add_f(f2g + o2 + c, G * f1p[c]);
          }
        }
      if (cog) {
        float sx = 0.f, sy = 0.f;
        for (int k = 0; k < K; ++k) {
          const int kx = k / rd, ky = k - kx * rd, ty = q.y0 - a.r + ky, tx = q.x0 - a.r + kx;
          float gx, gy;
          alt_corr_dblend(D(b, h, w, ty, tx), D(b, h, w, ty, tx + 1), D(b, h, w, ty + 1, tx), D(b, h, w, ty + 1, tx + 1), q.dx, q.dy, gx, gy);
          const float gk = g(ky, kx);
          sx += gk * gx; sy += gk * gy;
        }
        cog[pn * 2] = sx; cog[pn * 2 + 1] = sy;
      }
    }
  }
};
#else
// CTA = ALT shape (warps, tile_w): a run of tile_w pixels of one row, a warp per pixel at a time.  A lane owns V consecutive channels
// of every 32 V (one 16-byte load per lane and tap when V = 4); 32 window taps at a time are reduced across the warp with the
// transposing butterfly of corr_lookup_direct_kernel, and the dots land in shared memory.  The forward stages its (rd^2, tile_w)
// output block in shared memory and writes it row by row along W; the backward stages the incoming gradient the same way.
template <int V> __device__ __forceinline__ void alt_ld(const float* p, float* v) {
  if constexpr (V == 4) { const float4 q = __ldg(reinterpret_cast<const float4*>(p)); v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w; }
  else v[0] = __ldg(p);
}
template <int V> __device__ __forceinline__ void alt_red(float* p, const float* v) {
  if constexpr (V == 4) asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory");
  else asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v[0]) : "memory");
}
// dots[t] for the taps t = iy * wd + ix of the window anchored at (x0 - r, y0 - r); f1p: the source pixel's C features,
// f2b: sample b of fmap2
template <int V> __device__ __forceinline__ void alt_window_dots(const AltCorrArgs& a, const float* f1p, const float* f2b, int x0, int y0,
                                                                 float* dots, int lane) {
  const int wd = 2 * a.r + 2, taps = wd * wd;
  for (int g0 = 0; g0 < taps; g0 += 32) {
    int mine;   // element offset of tap g0 + lane in f2b, -1 off frame
    {
      const int t = g0 + lane, iy = t / wd, ix = t - iy * wd, ty = y0 - a.r + iy, tx = x0 - a.r + ix;
      mine = (t < taps && ty >= 0 && ty < a.H2 && tx >= 0 && tx < a.W2) ? (ty * a.W2 + tx) * a.C : -1;
    }
    int off[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) off[j] = __shfl_sync(0xffffffffu, mine, j);
    float p[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) p[j] = 0.f;
    for (int c = lane * V; c < a.C; c += 32 * V) {
      float f[V];
      alt_ld<V>(f1p + c, f);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        if (off[j] >= 0) {
          float v[V];
          alt_ld<V>(f2b + off[j] + c, v);
#pragma unroll
          for (int e = 0; e < V; ++e) p[j] = fmaf(f[e], v[e], p[j]);
        }
      }
    }
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
      const bool up = (lane & s) != 0;
#pragma unroll
      for (int i = 0; i < s; ++i) {
        const float send = up ? p[i] : p[i + s], keep = up ? p[i + s] : p[i];
        p[i] = keep + __shfl_xor_sync(0xffffffffu, send, s);
      }
    }
    if (g0 + lane < taps) dots[g0 + lane] = p[0];
  }
}
__device__ __forceinline__ int alt_tpad(int r) { return ((2 * r + 2) * (2 * r + 2) + 31) & ~31; }

template <int V>
__global__ void __launch_bounds__(256) alt_corr_fwd_kernel(AltCorrArgs a, float* __restrict__ out, int tw, int xblocks, int64_t n_tiles) {
  extern __shared__ float alt_sm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int rd = 2 * a.r + 1, wd = rd + 1, K = rd * rd, ld = tw + 1, tpad = alt_tpad(a.r);
  float* dots = alt_sm + warp * tpad;
  float* tile = alt_sm + nw * tpad;   // [K][ld]: output k of pixel p at tile[k * ld + p]
  const int64_t HW1 = (int64_t)a.H1 * a.W1;
  for (int64_t it = blockIdx.x; it < n_tiles; it += gridDim.x) {
    int64_t t = it;
    const int xb = (int)(t % xblocks); t /= xblocks;
    const int h = (int)(t % a.H1); t /= a.H1;
    const int n = (int)(t % a.N); const int b = (int)(t / a.N);
    const int w0 = xb * tw, cols = min(tw, a.W1 - w0);
    const float* f2b = a.f2 + (int64_t)b * a.H2 * a.W2 * a.C;
    for (int p = warp; p < cols; p += nw) {   // (warp-uniform)
      const int w = w0 + p;
      const float* cp = a.coords + ((((int64_t)b * a.N + n) * a.H1 + h) * a.W1 + w) * 2;
      const AltCell q = alt_corr_cell(__ldg(cp), __ldg(cp + 1), a.r, a.H2, a.W2);
      if (q.in) alt_window_dots<V>(a, a.f1 + (((int64_t)b * a.H1 + h) * a.W1 + w) * a.C, f2b, q.x0, q.y0, dots, lane);
      __syncwarp();
      for (int k = lane; k < K; k += 32) {
        float v = 0.f;
        if (q.in) {
          const int kx = k / rd, ky = k - kx * rd;
          const float* d = dots + ky * wd + kx;
          v = alt_corr_blend(d[0], d[1], d[wd], d[wd + 1], q.dx, q.dy);
        }
        tile[k * ld + p] = v;
      }
      __syncwarp();
    }
    __syncthreads();
    float* o = out + ((int64_t)b * a.N + n) * K * HW1 + (int64_t)h * a.W1 + w0;
    for (int i = threadIdx.x; i < K * tw; i += blockDim.x) {
      const int k = i / tw, p = i - k * tw;
      if (p < cols) o[k * HW1 + p] = tile[k * ld + p];
    }
    __syncthreads();
  }
}

template <int V>
__global__ void __launch_bounds__(256) alt_corr_bwd_kernel(AltCorrArgs a, const float* __restrict__ cgrad, float* f1g, float* f2g, float* cog,
                                                           int tw, int xblocks, int64_t n_tiles) {
  extern __shared__ float alt_sm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int rd = 2 * a.r + 1, wd = rd + 1, K = rd * rd, taps = wd * wd, ld = tw + 1, tpad = alt_tpad(a.r);
  float* G = alt_sm + warp * 2 * tpad;   // gradient of each window tap
  float* dots = G + tpad;
  float* tile = alt_sm + nw * 2 * tpad;  // [K][ld]: incoming gradient of output k of pixel p
  const int64_t HW1 = (int64_t)a.H1 * a.W1;
  for (int64_t it = blockIdx.x; it < n_tiles; it += gridDim.x) {
    int64_t t = it;
    const int xb = (int)(t % xblocks); t /= xblocks;
    const int h = (int)(t % a.H1); const int b = (int)(t / a.H1);
    const int w0 = xb * tw, cols = min(tw, a.W1 - w0);
    const float* f2b = a.f2 + (int64_t)b * a.H2 * a.W2 * a.C;
    float* g2b = f2g ? f2g + (int64_t)b * a.H2 * a.W2 * a.C : nullptr;
    for (int n = 0; n < a.N; ++n) {
      const float* gsrc = cgrad + ((int64_t)b * a.N + n) * K * HW1 + (int64_t)h * a.W1 + w0;
      for (int i = threadIdx.x; i < K * tw; i += blockDim.x) {
        const int k = i / tw, p = i - k * tw;
        tile[k * ld + p] = p < cols ? __ldg(gsrc + k * HW1 + p) : 0.f;
      }
      __syncthreads();
      for (int p = warp; p < cols; p += nw) {   // (warp-uniform)
        const int w = w0 + p;
        const int64_t pix = ((int64_t)b * a.H1 + h) * a.W1 + w, pn = ((int64_t)b * a.N + n) * HW1 + (int64_t)h * a.W1 + w;
        const float* f1p = a.f1 + pix * a.C;
        float* g1 = f1g ? f1g + pix * a.C : nullptr;
        const AltCell q = alt_corr_cell(__ldg(a.coords + pn * 2), __ldg(a.coords + pn * 2 + 1), a.r, a.H2, a.W2);
        if (q.in) {
          const float* tp = tile + p;
          auto g = [&](int ky, int kx) { return tp[(ky + rd * kx) * ld]; };
          for (int tt = lane; tt < taps; tt += 32) {
            const int iy = tt / wd, ix = tt - iy * wd;
            G[tt] = alt_corr_tap_grad(g, iy, ix, rd, q.dx, q.dy);
          }
          if (cog) alt_window_dots<V>(a, f1p, f2b, q.x0, q.y0, dots, lane);
          __syncwarp();
          if (cog) {
            float sx = 0.f, sy = 0.f;
            for (int k = lane; k < K; k += 32) {
              const int kx = k / rd, ky = k - kx * rd;
              const float* d = dots + ky * wd + kx;
              float gx, gy;
              alt_corr_dblend(d[0], d[1], d[wd], d[wd + 1], q.dx, q.dy, gx, gy);
              const float gk = g(ky, kx);
              sx = fmaf(gk, gx, sx); sy = fmaf(gk, gy, sy);
            }
#pragma unroll
            for (int s = 16; s >= 1; s >>= 1) { sx += __shfl_xor_sync(0xffffffffu, sx, s); sy += __shfl_xor_sync(0xffffffffu, sy, s); }
            if (lane == 0) { cog[pn * 2] = sx; cog[pn * 2 + 1] = sy; }
          }
        } else if (cog && lane == 0) {
          cog[pn * 2] = 0.f; cog[pn * 2 + 1] = 0.f;
        }
        if (g1 || (g2b && q.in)) {
          for (int c = lane * V; c < a.C; c += 32 * V) {
            float acc[V], f[V];
#pragma unroll
            for (int e = 0; e < V; ++e) acc[e] = n == 0 || !g1 ? 0.f : g1[c + e];   // the same lane wrote it for n - 1
            if (g2b) alt_ld<V>(f1p + c, f);
            if (q.in)
              for (int iy = 0; iy < wd; ++iy) {
                const int ty = q.y0 - a.r + iy;
                if (ty < 0 || ty >= a.H2) continue;
                for (int ix = 0; ix < wd; ++ix) {
                  const int tx = q.x0 - a.r + ix;
                  if (tx < 0 || tx >= a.W2) continue;
                  const float Gt = G[iy * wd + ix];
                  const int off = (ty * a.W2 + tx) * a.C + c;
                  if (g1) {
                    float v[V];
                    alt_ld<V>(f2b + off, v);
#pragma unroll
                    for (int e = 0; e < V; ++e) acc[e] = fmaf(Gt, v[e], acc[e]);
                  }
                  if (g2b) {
                    float u[V];
#pragma unroll
                    for (int e = 0; e < V; ++e) u[e] = Gt * f[e];
                    alt_red<V>(g2b + off, u);
                  }
                }
              }
            if (g1) {
#pragma unroll
              for (int e = 0; e < V; ++e) g1[c + e] = acc[e];
            }
          }
        }
        __syncwarp();   // G / dots are rewritten for the next pixel
      }
      __syncthreads();   // the tile is rewritten for the next n
    }
  }
}
#endif

static size_t alt_corr_smem(int r, int warps, int tile_w) {
  const int64_t wd = 2 * (int64_t)r + 2, rd = wd - 1, tpad = (wd * wd + 31) & ~int64_t(31);
  return (size_t)(2 * warps * tpad + rd * rd * (tile_w + 1)) * sizeof(float);   // the backward's (the forward needs less)
}
bool alt_corr_launch_shape(int r, int* warps, int* tile_w) {
  if (r < 0 || r > 4096) return false;
  int nw = 8, tw = 32;
  while (alt_corr_smem(r, nw, tw) > ALT_CORR_SMEM_MAX) {
    if (tw > nw) tw >>= 1;
    else if (nw > 1) { nw >>= 1; tw = nw; }
    else return false;
  }
  *warps = nw; *tile_w = tw;
  return true;
}

#ifndef GV_HOSTSIM
static bool alt_corr_vec4(const AltCorrArgs& a) {
  return a.C % 4 == 0 && (reinterpret_cast<uintptr_t>(a.f1) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.f2) & 15) == 0;
}
template <class Kern> static void alt_corr_attr(Kern k, volatile unsigned char* flags) { gv_set_max_smem(k, ALT_CORR_SMEM_MAX, flags); }
#endif

void alt_corr_forward(Ctx& cx, const AltCorrArgs& a, float* out) {
  int nw = 0, tw = 0;
  if (!alt_corr_launch_shape(a.r, &nw, &tw)) throw std::runtime_error("alt_corr: radius too large for the shared memory of one window");
  const int K = (2 * a.r + 1) * (2 * a.r + 1);
#ifdef GV_HOSTSIM
  parallel_for(cx, (int64_t)a.B * a.N * K * a.H1 * a.W1, AltCorrFwdK{a, out}, "alt_corr_forward");
#else
  const int64_t items = (int64_t)a.B * a.N * a.H1 * a.W1;
  if (cx.dry || items == 0) return;
  cx.launches++;
  const int xblocks = (a.W1 + tw - 1) / tw;
  const int64_t tiles = (int64_t)a.B * a.N * a.H1 * xblocks;
  const size_t smem = alt_corr_smem(a.r, nw, tw);
  int64_t blocks = tiles, cap = (int64_t)cx.sm_count * 16;
  if (blocks > cap) blocks = cap;
  const int wd = 2 * a.r + 2;
  if (cx.prof) cx.prof->begin(cx.stream, "alt_corr_forward", (double)items * wd * wd * a.C * 2);
  static volatile unsigned char attr[2][64];
  if (alt_corr_vec4(a)) {
    alt_corr_attr(alt_corr_fwd_kernel<4>, attr[0]);
    alt_corr_fwd_kernel<4><<<(unsigned)blocks, nw * 32, smem, cx.stream>>>(a, out, tw, xblocks, tiles);
  } else {
    alt_corr_attr(alt_corr_fwd_kernel<1>, attr[1]);
    alt_corr_fwd_kernel<1><<<(unsigned)blocks, nw * 32, smem, cx.stream>>>(a, out, tw, xblocks, tiles);
  }
  gv_check_launch("alt_corr_forward");
  if (cx.prof) cx.prof->end(cx.stream);
  (void)K;
#endif
}

void alt_corr_backward(Ctx& cx, const AltCorrArgs& a, const float* corr_grad, float* f1g, float* f2g, float* cog) {
  int nw = 0, tw = 0;
  if (!alt_corr_launch_shape(a.r, &nw, &tw)) throw std::runtime_error("alt_corr: radius too large for the shared memory of one window");
  if (!f1g && !f2g && !cog) return;
#ifdef GV_HOSTSIM
  parallel_for(cx, (int64_t)a.B * a.H1 * a.W1, AltCorrBwdK{a, corr_grad, f1g, f2g, cog}, "alt_corr_backward");
#else
  if (cx.dry || (int64_t)a.B * a.H1 * a.W1 == 0) return;
  cx.launches++;
  const int xblocks = (a.W1 + tw - 1) / tw;
  const int64_t tiles = (int64_t)a.B * a.H1 * xblocks;
  const size_t smem = alt_corr_smem(a.r, nw, tw);
  int64_t blocks = tiles, cap = (int64_t)cx.sm_count * 16;
  if (blocks > cap) blocks = cap;
  const int wd = 2 * a.r + 2;
  if (cx.prof) cx.prof->begin(cx.stream, "alt_corr_backward", (double)a.B * a.N * a.H1 * a.W1 * wd * wd * a.C * 4);
  static volatile unsigned char attr[2][64];
  if (alt_corr_vec4(a) && (!f1g || (reinterpret_cast<uintptr_t>(f1g) & 15) == 0) && (!f2g || (reinterpret_cast<uintptr_t>(f2g) & 15) == 0)) {
    alt_corr_attr(alt_corr_bwd_kernel<4>, attr[0]);
    alt_corr_bwd_kernel<4><<<(unsigned)blocks, nw * 32, smem, cx.stream>>>(a, corr_grad, f1g, f2g, cog, tw, xblocks, tiles);
  } else {
    alt_corr_attr(alt_corr_bwd_kernel<1>, attr[1]);
    alt_corr_bwd_kernel<1><<<(unsigned)blocks, nw * 32, smem, cx.stream>>>(a, corr_grad, f1g, f2g, cog, tw, xblocks, tiles);
  }
  gv_check_launch("alt_corr_backward");
  if (cx.prof) cx.prof->end(cx.stream);
#endif
}


}  // namespace gv
