// fp32 implicit-GEMM convolution on NHWC activations with fused epilogues
// (bias, ReLU/LeakyReLU/PReLU/sigmoid/tanh/sin, residual add, gate multiply,
// ConvGRU blend).  This is the exact-precision CUDA-core path used where the
// recurrence amplifies rounding (RAFT) and for small-channel layers; the
// tensor-core path for the wide synthesis layers lives in conv_tc.cu.
//
// GEMM view: M = n*oh*ow output pixels, N = cout, K = kh*kw*cin.  The input may
// be the channel concatenation of two views (in0 | in1) so torch.cat never
// materialises (ResBlock side-channel splice fi_components.py:137-148, GRU
// cat[r*h, x] raft/update.py:57,65).
#include "common.h"

namespace gv {

struct ConvArgs {
  TV in0, in1, out;
  ConvW w;
  ConvGeom g;
  ConvEpi e;
  int c0;      // channels taken from in0 (rest from in1)
  int M;       // total output pixels
  int vec_ok;  // float4 loads allowed on the activation side
};

GV_HD int reflect_idx(int v, int n) { return v < 0 ? -v : (v >= n ? 2 * n - 2 - v : v); }

GV_HD float conv_epilogue(const ConvArgs& a, float v, int n, int oy, int ox, int co) {
  const ConvEpi& e = a.e;
  if (a.w.b) v += a.w.b[co];
  v = apply_act(v, e.act1, e.slope1, co);
  if (e.res.p) v += e.res.p[e.res.off(n, oy, ox) + co];
  v = apply_act(v, e.act2, e.slope2, co);
  if (e.mul.p) v *= e.mul.p[e.mul.off(n, oy, ox) + co];
  if (e.gru_z.p) {
    float z = e.gru_z.p[e.gru_z.off(n, oy, ox) + co];
    float h = e.gru_h.p[e.gru_h.off(n, oy, ox) + co];
    v = (1.f - z) * h + z * v;
  }
  return v;
}

#ifndef GV_HOSTSIM
template <int BN, int TM, int TN>
__global__ void __launch_bounds__(256) conv2d_simt_kernel(ConvArgs a) {
  constexpr int BM = 128, BK = 16;
  constexpr int NT = BN / TN;  // threads along N
  static_assert((BM / TM) * NT == 256, "thread tiling");
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int tn = (tid % NT) * TN, tm = (tid / NT) * TM;
  const int OH = a.out.h, OW = a.out.w, IH = a.in0.h, IW = a.in0.w;
  const int cin = a.w.cin, KW = a.w.kw, taps = a.w.kh * a.w.kw;

  // the two activation rows (pixels) this thread stages per K-step
  int pn[2], py[2], px[2]; bool pv[2];
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    int m = m0 + ((tid + it * 256) >> 2);
    pv[it] = m < a.M;
    int mm = pv[it] ? m : 0;
    px[it] = mm % OW; int r = mm / OW; py[it] = r % OH; pn[it] = r / OH;
  }
  const int q4 = (tid & 3) * 4;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int tap = 0; tap < taps; ++tap) {
    const int ky = tap / KW, kx = tap % KW;
    const float* rowp0[2]; const float* rowp1[2]; bool rv[2];
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      int iy = py[it] * a.g.stride - a.g.ph + ky, ix = px[it] * a.g.stride - a.g.pw + kx;
      if (a.g.reflect) { iy = reflect_idx(iy, IH); ix = reflect_idx(ix, IW); }
      rv[it] = pv[it] && iy >= 0 && iy < IH && ix >= 0 && ix < IW;
      int64_t o = rv[it] ? ((int64_t)iy * IW + ix) : 0;
      rowp0[it] = a.in0.p + (int64_t)pn[it] * a.in0.sn + o * a.in0.ld;
      rowp1[it] = a.in1.p ? a.in1.p + (int64_t)pn[it] * a.in1.sn + o * a.in1.ld : nullptr;
    }
    for (int k0 = 0; k0 < cin; k0 += BK) {
      // ---- stage A: 128 pixels x 16 channels
#pragma unroll
      for (int it = 0; it < 2; ++it) {
        int row = (tid + it * 256) >> 2;
        int ch = k0 + q4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (rv[it]) {
          const float* src; int lim, cc;
          if (ch < a.c0) { src = rowp0[it]; lim = a.c0; cc = ch; } else { src = rowp1[it]; lim = cin - a.c0; cc = ch - a.c0; }
          if (a.vec_ok && cc + 3 < lim) {
            v = *reinterpret_cast<const float4*>(src + cc);
          } else if (ch < cin) {
            float t[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              int c = ch + u; float x = 0.f;
              if (c < cin) x = (c < a.c0) ? rowp0[it][c] : rowp1[it][c - a.c0];
              t[u] = x;
            }
            v = make_float4(t[0], t[1], t[2], t[3]);
          }
        }
        As[q4 + 0][row] = v.x; As[q4 + 1][row] = v.y; As[q4 + 2][row] = v.z; As[q4 + 3][row] = v.w;
      }
      // ---- stage B: 16 x BN weights
      if (tid < BK * BN / 4) {
        int k = tid / (BN / 4), n4 = (tid % (BN / 4)) * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k0 + k < cin && n0 + n4 < a.w.cout_ld)
          v = *reinterpret_cast<const float4*>(a.w.w + ((int64_t)tap * cin + k0 + k) * a.w.cout_ld + n0 + n4);
        *reinterpret_cast<float4*>(&Bs[k][n4]) = v;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < BK; ++k) {
        float av[TM], bv[TN];
#pragma unroll
        for (int i = 0; i < TM; ++i) av[i] = As[k][tm + i];
#pragma unroll
        for (int j = 0; j < TN; ++j) bv[j] = Bs[k][tn + j];
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
  // ---- epilogue
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int m = m0 + tm + i;
    if (m >= a.M) continue;
    int ox = m % OW; int r = m / OW; int oy = r % OH; int n = r / OH;
    float* o = a.out.p + a.out.off(n, oy, ox);
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int co = n0 + tn + j;
      if (co < a.w.cout) o[co] = conv_epilogue(a, acc[i][j], n, oy, ox, co);
    }
  }
}
#endif


#ifndef GV_HOSTSIM
// Convolutions with 1-2 output channels over a wide input (RAFT FlowHead.conv2: 3x3, 256 -> 2, raft/update.py:6-14).
// A GEMM tile would be all padding (N = 16 of which 2 are real) and still pay the whole A-operand pipeline; here one warp
// owns one output pixel: lanes split the input channels (float4 each), the weights sit in shared memory as (co0, co1) pairs,
// two fp32 accumulators per lane, one shuffle reduction.  Exact fp32 arithmetic; reads every input byte ~once from L2
// (the 9-fold tap reuse is served by L1).  y = res + conv + bias (the only epilogue its callers need).
template <int COUT>
__global__ void __launch_bounds__(256) conv_narrow_kernel(ConvArgs a, int warps_total) {
  extern __shared__ float2 wsm[];   // [tap * cin + ci] -> (w[co 0], w[co 1])
  const int cin = a.w.cin, taps = a.w.kh * a.w.kw;
  for (int i = threadIdx.x; i < taps * cin; i += blockDim.x) {
    const float* wp = a.w.w + (size_t)i * a.w.cout_ld;
    wsm[i] = make_float2(wp[0], COUT > 1 ? wp[1] : 0.f);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int OW = a.out.w, OH = a.out.h;
  for (int m = blockIdx.x * wpb + wib; m < warps_total; m += gridDim.x * wpb) {
    const int ox = m % OW; int r = m / OW; const int oy = r % OH; const int n = r / OH;
    float acc0 = 0.f, acc1 = 0.f;
    for (int ky = 0; ky < a.w.kh; ++ky) {
      const int iy = oy + ky - a.g.ph;
      if (iy < 0 || iy >= a.in0.h) continue;
      for (int kx = 0; kx < a.w.kw; ++kx) {
        const int ix = ox + kx - a.g.pw;
        if (ix < 0 || ix >= a.in0.w) continue;
        const float* src = a.in0.p + a.in0.off(n, iy, ix);
        const float2* wt = wsm + (ky * a.w.kw + kx) * cin;
        for (int c = lane * 4; c < cin; c += 128) {
          const float4 v = *reinterpret_cast<const float4*>(src + c);
          const float4 w01 = *reinterpret_cast<const float4*>(wt + c), w23 = *reinterpret_cast<const float4*>(wt + c + 2);
          acc0 = fmaf(v.x, w01.x, acc0); acc1 = fmaf(v.x, w01.y, acc1);
          acc0 = fmaf(v.y, w01.z, acc0); acc1 = fmaf(v.y, w01.w, acc1);
          acc0 = fmaf(v.z, w23.x, acc0); acc1 = fmaf(v.z, w23.y, acc1);
          acc0 = fmaf(v.w, w23.z, acc0); acc1 = fmaf(v.w, w23.w, acc1);
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { acc0 += __shfl_xor_sync(0xffffffffu, acc0, o); acc1 += __shfl_xor_sync(0xffffffffu, acc1, o); }
    if (lane < COUT) {
      float v = (lane == 0 ? acc0 : acc1) + a.w.b[lane];
      if (a.e.res.p) v += a.e.res.p[a.e.res.off(n, oy, ox) + lane];
      a.out.p[a.out.off(n, oy, ox) + lane] = v;
    }
  }
}


// FlowHead.conv2 shape (3x3, 256 -> 2): one warp computes FOUR horizontally adjacent output pixels, so the 3 x 6 input pixels
// and the lane's 18 x 8 weights are fetched once for four outputs (3x fewer load instructions than one pixel per warp).
__global__ void __launch_bounds__(256, 2) conv_narrow3x3_c256_kernel(ConvArgs a, int quads_per_row, int quads_total) {
  extern __shared__ float2 wsm[];   // [tap * 256 + ci] -> (w[co 0], w[co 1])
  for (int i = threadIdx.x; i < 9 * 256; i += blockDim.x) {
    const float* wp = a.w.w + (size_t)i * a.w.cout_ld;
    wsm[i] = make_float2(wp[0], a.w.cout > 1 ? wp[1] : 0.f);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int OW = a.out.w, OH = a.out.h;
  for (int qd = blockIdx.x * wpb + wib; qd < quads_total; qd += gridDim.x * wpb) {
    const int qx = qd % quads_per_row; int r = qd / quads_per_row; const int oy = r % OH; const int n = r / OH;
    const int ox0 = qx * 4;
    float acc[4][2];
#pragma unroll
    for (int p = 0; p < 4; ++p) { acc[p][0] = 0.f; acc[p][1] = 0.f; }
#pragma unroll 1
    for (int hf = 0; hf < 2; ++hf) {          // the lane's channels: hf * 128 + lane * 4 .. + 3
      float4 v[3][6];
#pragma unroll
      for (int dy = 0; dy < 3; ++dy) {
        const int iy = oy + dy - 1;
#pragma unroll
        for (int dx = 0; dx < 6; ++dx) {
          const int ix = ox0 + dx - 1;
          const bool in = iy >= 0 && iy < a.in0.h && ix >= 0 && ix < a.in0.w;
          v[dy][dx] = in ? *reinterpret_cast<const float4*>(a.in0.p + a.in0.off(n, iy, ix) + hf * 128 + lane * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const float2* wt = wsm + t * 256 + hf * 128 + lane * 4;
        const float4 w01 = *reinterpret_cast<const float4*>(wt), w23 = *reinterpret_cast<const float4*>(wt + 2);
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const float4 x = v[t / 3][p + t % 3];
          acc[p][0] = fmaf(x.x, w01.x, acc[p][0]); acc[p][1] = fmaf(x.x, w01.y, acc[p][1]);
          acc[p][0] = fmaf(x.y, w01.z, acc[p][0]); acc[p][1] = fmaf(x.y, w01.w, acc[p][1]);
          acc[p][0] = fmaf(x.z, w23.x, acc[p][0]); acc[p][1] = fmaf(x.z, w23.y, acc[p][1]);
          acc[p][0] = fmaf(x.w, w23.z, acc[p][0]); acc[p][1] = fmaf(x.w, w23.w, acc[p][1]);
        }
      }
    }
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) { acc[p][0] += __shfl_xor_sync(0xffffffffu, acc[p][0], o); acc[p][1] += __shfl_xor_sync(0xffffffffu, acc[p][1], o); }
    if (lane < 4 * a.w.cout) {     // lane = pixel * cout + channel
      const int p = lane / a.w.cout, co = lane % a.w.cout, ox = ox0 + p;
      if (ox < OW) {
        float val = 0.f;
#pragma unroll
        for (int pp = 0; pp < 4; ++pp) if (pp == p) val = co == 0 ? acc[pp][0] : acc[pp][1];
        val += a.w.b[co];
        if (a.e.res.p) val += a.e.res.p[a.e.res.off(n, oy, ox) + co];
        a.out.p[a.out.off(n, oy, ox) + co] = val;
      }
    }
  }
}

static bool conv_narrow_ok(const ConvArgs& a) {
  const auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  return a.w.cout <= 2 && !a.in1.p && a.g.stride == 1 && !a.g.reflect && !a.g.loose_w && a.w.cin % 128 == 0 && a.in0.ld % 4 == 0 && a.in0.sn % 4 == 0 &&
         al16(a.in0.p) && a.e.act1 == ACT_NONE && a.e.act2 == ACT_NONE && !a.e.mul.p && !a.e.gru_z.p && !a.in0.f16 && !a.out.f16 && !a.e.res.f16 &&
         (size_t)a.w.kh * a.w.kw * a.w.cin * sizeof(float2) <= 96 * 1024 &&
         a.w.kh * a.w.kw * a.w.cin >= 1024;   // (a full-resolution 1x1 with few channels is better off as one MMA tile per 128 pixels)
}
#endif


#ifndef GV_HOSTSIM
// Convolutions with very few input channels (GIMM cnn_encoder.0: 3x3, 2 -> 16 at full resolution, gimmvfi_r.py:86-88): the
// layer is pure memory traffic (18 MACs per output value), so one thread owns one output pixel: taps are scalar loads that
// hit L1 (neighbouring threads share them), weights + bias live in shared memory, the COUT results leave as float4 stores.
template <int COUT>
__global__ void __launch_bounds__(256) conv_thin_kernel(ConvArgs a) {
  extern __shared__ float wth[];   // [tap * cin + ci][COUT] then bias[COUT]
  const int cin = a.w.cin, taps = a.w.kh * a.w.kw;
  for (int i = threadIdx.x; i < taps * cin * COUT; i += blockDim.x) wth[i] = a.w.w[(size_t)(i / COUT) * a.w.cout_ld + (i % COUT)];
  for (int i = threadIdx.x; i < COUT; i += blockDim.x) wth[taps * cin * COUT + i] = a.w.b[i];
  __syncthreads();
  const int OW = a.out.w, OH = a.out.h;
  for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < a.M; m += gridDim.x * blockDim.x) {
    const int ox = m % OW; int r = m / OW; const int oy = r % OH; const int n = r / OH;
    float acc[COUT];
#pragma unroll
    for (int j = 0; j < COUT; ++j) acc[j] = 0.f;
    for (int ky = 0; ky < a.w.kh; ++ky) {
      const int iy = oy + ky - a.g.ph;
      if (iy < 0 || iy >= a.in0.h) continue;
      for (int kx = 0; kx < a.w.kw; ++kx) {
        const int ix = ox + kx - a.g.pw;
        if (ix < 0 || ix >= a.in0.w) continue;
        const float* src = a.in0.p + a.in0.off(n, iy, ix);
        const float* wt = wth + (ky * a.w.kw + kx) * cin * COUT;
        for (int c = 0; c < cin; ++c) {
          const float v = src[c];
#pragma unroll
          for (int j = 0; j < COUT; ++j) acc[j] = fmaf(v, wt[c * COUT + j], acc[j]);
        }
      }
    }
    float* o = a.out.p + a.out.off(n, oy, ox);
#pragma unroll
    for (int j = 0; j < COUT; j += 4) {
      F4 v;
      v.x = apply_act(acc[j] + wth[taps * cin * COUT + j], a.e.act1, a.e.slope1, j);
      v.y = apply_act(acc[j + 1] + wth[taps * cin * COUT + j + 1], a.e.act1, a.e.slope1, j + 1);
      v.z = apply_act(acc[j + 2] + wth[taps * cin * COUT + j + 2], a.e.act1, a.e.slope1, j + 2);
      v.w = apply_act(acc[j + 3] + wth[taps * cin * COUT + j + 3], a.e.act1, a.e.slope1, j + 3);
      st4(o + j, v);
    }
  }
}
static bool conv_thin_ok(const ConvArgs& a) {
  return a.w.cout == 16 && a.w.cin <= 4 && !a.in1.p && a.g.stride == 1 && !a.g.reflect && !a.g.loose_w && !a.e.res.p && !a.e.mul.p && !a.e.gru_z.p &&
         a.e.act2 == ACT_NONE && a.e.act1 != ACT_SIGMOID && a.e.act1 != ACT_TANH && a.e.act1 != ACT_SIN && !a.in0.f16 && !a.out.f16 &&
         (reinterpret_cast<uintptr_t>(a.out.p) & 15) == 0 && a.out.ld % 4 == 0 && a.out.sn % 4 == 0;
}
#endif

#ifndef GV_HOSTSIM
// 7x7 convolutions with <= 4 output channels on few input channels at FULL resolution (amt_comb_block.2: 18 -> 3, gimmvfi_r.py:60-64):
// as an MMA tile this layer pays one K step per (tap row, 32 lanes) for N = 3 useful columns (1.2 ms at 1088x1920, bound by the
// per-K-step hand-off of conv_tc.cu).  Here a CTA owns a 128 x 8 output tile; the input halo streams through shared memory 6 channels at
// a time, channel-major ([ci][y][x], plane pitch = 20 mod 32 banks so the staging writes of 6 channels do not collide); a thread owns 4
// x-consecutive pixels: per (channel, tap row) THREE 16-byte loads fetch the 10 inputs its 4 windows share and SEVEN broadcast 16-byte
// loads the weights, for 84-112 FMAs - FMA-bound instead of shared-memory-bound (the first version, one pixel per thread with one scalar
// load per FMA triple, ran at 7.5 TFMA/s).  Exact fp32.
constexpr int C7_TW = 128, C7_TH = 8, C7_CCH = 6, C7_RP = 136, C7_PP = 14 * C7_RP + 4;
template <int CO>
__global__ void __launch_bounds__(256) conv7x7_small_cout_kernel(TV in, const float* __restrict__ w, const float* __restrict__ bias, TV out,
                                                                 int cin, int cout, int act, const float* slope) {
  extern __shared__ __align__(16) float sm_c7[];
  float* wsm = sm_c7;                       // [49][cin][4]
  float* tile = sm_c7 + 49 * cin * 4;       // [C7_CCH][14][C7_RP] (+ plane padding)
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5, n = blockIdx.z;
  const int x0 = blockIdx.x * C7_TW, y0 = blockIdx.y * C7_TH;
  for (int i = threadIdx.x; i < 49 * cin * 4; i += 256) wsm[i] = w[i];
  float acc[4][CO];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int c = 0; c < CO; ++c) acc[p][c] = 0.f;
  for (int c0 = 0; c0 < cin; c0 += C7_CCH) {
    const int cc = (cin - c0) < C7_CCH ? (cin - c0) : C7_CCH;
    __syncthreads();
    for (int i = threadIdx.x; i < cc * 14 * (C7_TW + 6); i += 256) {
      const int ci = i % cc; int r = i / cc; const int px = r % (C7_TW + 6), py = r / (C7_TW + 6);
      const int gy = y0 + py - 3, gx = x0 + px - 3;
      tile[ci * C7_PP + py * C7_RP + px] = (gy >= 0 && gy < in.h && gx >= 0 && gx < in.w) ? in.p[in.off(n, gy, gx) + c0 + ci] : 0.f;
    }
    __syncthreads();
    for (int ci = 0; ci < cc; ++ci) {
      const float* tp = tile + ci * C7_PP + ty * C7_RP + tx * 4;
      const float4* wp = reinterpret_cast<const float4*>(wsm) + (c0 + ci);
#pragma unroll
      for (int ky = 0; ky < 7; ++ky) {
        const float4 a0 = *reinterpret_cast<const float4*>(tp + ky * C7_RP), a1 = *reinterpret_cast<const float4*>(tp + ky * C7_RP + 4),
                     a2 = *reinterpret_cast<const float4*>(tp + ky * C7_RP + 8);
        const float a[12] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w};
#pragma unroll
        for (int kx = 0; kx < 7; ++kx) {
          const float4 ww = wp[(ky * 7 + kx) * cin];
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            acc[p][0] = fmaf(a[p + kx], ww.x, acc[p][0]); acc[p][1] = fmaf(a[p + kx], ww.y, acc[p][1]); acc[p][2] = fmaf(a[p + kx], ww.z, acc[p][2]);
            if (CO == 4) acc[p][CO - 1] = fmaf(a[p + kx], ww.w, acc[p][CO - 1]);
          }
        }
      }
    }
  }
  const int y = y0 + ty;
  if (y < out.h) {
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int x = x0 + tx * 4 + p;
      if (x < out.w) {
        float* o = out.p + out.off(n, y, x);
#pragma unroll
        for (int c = 0; c < CO; ++c)
          if (c < cout) o[c] = apply_act(acc[p][c] + bias[c], act, slope, c);
      }
    }
  }
}
#endif
// returns false when the layer / tensors are not of that class (the caller then takes the generic path)
bool conv7x7_small_cout(Ctx& cx, const TV& in, const ConvW& w, int act, const float* slope, const TV& out) {
#ifdef GV_HOSTSIM
  (void)cx; (void)in; (void)w; (void)act; (void)slope; (void)out;
  return false;
#else
  if (w.kh != 7 || w.kw != 7 || w.cout > 4 || w.cout_ld != 4 || w.cin > 24 || in.c != w.cin || in.f16 || out.f16 || out.c != w.cout || in.n != out.n || in.h != out.h ||
      in.w != out.w || act == ACT_SIGMOID || act == ACT_TANH || act == ACT_SIN || act == ACT_GELU)
    return false;
  if (cx.dry) return true;
  const int smem = (49 * w.cin * 4 + C7_CCH * C7_PP) * (int)sizeof(float);
  static volatile unsigned char attr3[64], attr4[64];
  gv_set_max_smem(conv7x7_small_cout_kernel<3>, smem, attr3);
  gv_set_max_smem(conv7x7_small_cout_kernel<4>, smem, attr4);
  cx.launches++;
  if (cx.prof) {
    char nm[128];
    snprintf(nm, sizeof nm, "conv7x7_small_cout c%d>%d @%dx%dx%d", w.cin, w.cout, out.n, out.h, out.w);
    cx.prof->begin(cx.stream, prof_intern(nm), 2.0 * (double)out.pixels() * w.cout * (double)w.cin * 49);
  }
  dim3 grid((out.w + C7_TW - 1) / C7_TW, (out.h + C7_TH - 1) / C7_TH, out.n);
  if (w.cout == 4) conv7x7_small_cout_kernel<4><<<grid, 256, smem, cx.stream>>>(in, w.w, w.b, out, w.cin, w.cout, act, slope);
  else conv7x7_small_cout_kernel<3><<<grid, 256, smem, cx.stream>>>(in, w.w, w.b, out, w.cin, w.cout, act, slope);
  gv_check_launch("conv7x7_small_cout");
  if (cx.prof) cx.prof->end(cx.stream);
  return true;
#endif
}

// Eligibility of a layer for the tensor-core path (conv_tc.cu; its arithmetic is emulated on the host in tests/hostsim)
bool conv2d_tc_supported(const TV& in0, const TV& in1, const ConvW& w, const ConvGeom& g, const ConvEpi& e, const TV& out, bool split) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (!w.w_tc || (g.stride != 1 && g.stride != 2) || g.reflect) return false;
  if (split && !w.has_lo) return false;
  if (!g.loose_w && (g.ph != w.kh / 2 || g.pw != w.kw / 2)) return false;
  if (g.loose_w && (g.ph != 0 || g.pw != 0)) return false;   // pre-padded input: taps index it directly
  const bool h = in0.f16 != 0;                                 // half activations: f16, 64-channel K blocks
  const int amul = h ? 8 : 4, kblk = h ? 64 : 32;              // 16-byte TMA strides
  if (h && (split || !w.w_tc_h)) return false;
  if (in1.p && (in1.f16 != 0) != h) return false;
  if (e.mul.f16 || e.gru_z.f16 || e.gru_h.f16 || (e.mul.p && e.gru_z.p)) return false;   // only the residual may be half; gate multiply and GRU blend exclude each other
  if (e.split_c && (e.split_c % 32 || !e.out2.p || e.out2.f16 || e.gru_z.p)) return false;   // (a residual is indexed by the merged channel)
  if (!al16(in0.p) || in0.ld % amul || in0.sn % amul) return false;
  if (in1.p && (!al16(in1.p) || in1.ld % amul || in1.sn % amul || in0.c % kblk)) return false;
  if (!g.loose_w && ((in0.h + 2 * g.ph - w.kh) / g.stride + 1 != out.h || (in0.w + 2 * g.pw - w.kw) / g.stride + 1 != out.w)) return false;
  return true;
}

void conv2d(Ctx& cx, const TV& in0, const TV& in1, const ConvW& w, const ConvGeom& g, const ConvEpi& e, const TV& out) {
  if (cx.dry) return;
  ConvArgs a;
  a.in0 = in0; a.in1 = in1; a.out = out; a.w = w; a.g = g; a.e = e;
  a.c0 = in0.c;
  a.M = out.n * out.h * out.w;
  const int cin_total = in0.c + (in1.p ? in1.c : 0);
  if (cin_total != w.cin) throw std::runtime_error("conv2d: cin mismatch (" + std::to_string(cin_total) + " vs " + std::to_string(w.cin) + ")");
  if (e.split_c ? (out.c != e.split_c || e.out2.c != w.cout - e.split_c) : (out.c != w.cout)) throw std::runtime_error("conv2d: cout mismatch");
  {
    int eh = (in0.h + 2 * g.ph - w.kh) / g.stride + 1, ew = (in0.w + 2 * g.pw - w.kw) / g.stride + 1;
    if (((eh != out.h || ew != out.w) && !g.loose_w) || in0.n != out.n) throw std::runtime_error("conv2d: output geometry mismatch");
  }
#ifndef GV_HOSTSIM
  if (conv_narrow_ok(a)) {   // before the tensor-core dispatch: exact fp32 and ~10x faster than a 16-wide MMA tile of padding
    cx.launches++;
    const size_t smem = (size_t)w.kh * w.kw * w.cin * sizeof(float2);
    static volatile unsigned char attr1[64], attr2[64], attr4[64];
    gv_set_max_smem(conv_narrow_kernel<1>, 96 * 1024, attr1);
    gv_set_max_smem(conv_narrow_kernel<2>, 96 * 1024, attr2);
    if (cx.prof) {
      char nm[128];
      snprintf(nm, sizeof nm, "conv_narrow k%dx%d c%d>%d @%dx%dx%d", w.kh, w.kw, w.cin, w.cout, out.n, out.h, out.w);
      cx.prof->begin(cx.stream, prof_intern(nm), 2.0 * (double)a.M * w.cout * (double)w.cin * w.kh * w.kw);
    }
    const int blocks = std::min((a.M + 7) / 8, cx.sm_count * 8);
    if (w.kh == 3 && w.kw == 3 && w.cin == 256 && g.ph == 1 && g.pw == 1) {
      const int qpr = (out.w + 3) / 4, quads = out.n * out.h * qpr;
      gv_set_max_smem(conv_narrow3x3_c256_kernel, 96 * 1024, attr4);
      conv_narrow3x3_c256_kernel<<<std::min((quads + 7) / 8, cx.sm_count * 8), 256, smem, cx.stream>>>(a, qpr, quads);
    } else if (w.cout == 1) conv_narrow_kernel<1><<<blocks, 256, smem, cx.stream>>>(a, a.M);
    else conv_narrow_kernel<2><<<blocks, 256, smem, cx.stream>>>(a, a.M);
    gv_check_launch("conv_narrow");
    if (cx.prof) cx.prof->end(cx.stream);
    return;
  }
  if (conv_thin_ok(a)) {
    cx.launches++;
    const size_t smem = ((size_t)w.kh * w.kw * w.cin + 1) * 16 * sizeof(float);
    if (cx.prof) {
      char nm[128];
      snprintf(nm, sizeof nm, "conv_thin k%dx%d c%d>%d @%dx%dx%d", w.kh, w.kw, w.cin, w.cout, out.n, out.h, out.w);
      cx.prof->begin(cx.stream, prof_intern(nm), 2.0 * (double)a.M * w.cout * (double)w.cin * w.kh * w.kw);
    }
    const int blocks = std::min((a.M + 255) / 256, cx.sm_count * 16);
    conv_thin_kernel<16><<<blocks, 256, smem, cx.stream>>>(a);
    gv_check_launch("conv_thin");
    if (cx.prof) cx.prof->end(cx.stream);
    return;
  }
#endif
  const bool any_f16 = in0.f16 || in1.f16 || out.f16 || e.res.f16;
#ifndef GV_HOSTSIM
  // K-poor 3x3 layers: halo tile loaded once, taps as views of it (same TF32 / half operand arithmetic as conv2d_tc)
  if (cx.tc && !(cx.tc_split && !any_f16) && conv2d_halo_supported(in0, in1, w, g, e, out) && conv2d_tc_supported(in0, in1, w, g, e, out, false)) {
    conv2d_halo(cx, in0, w, g, e, out);
    return;
  }
  // wide half 3x3 layers (the final decoder trunk): each K block's tile + halo loaded once, the nine taps as views of it
  if (cx.tc && conv2d_wide_supported(in0, in1, w, g, e, out)) {
    conv2d_wide(cx, in0, in1, w, g, e, out);
    return;
  }
#endif
  if (cx.tc && conv2d_tc_supported(in0, in1, w, g, e, out, cx.tc_split && !any_f16)) { conv2d_tc(cx, in0, in1, w, g, e, out, cx.tc_split && !any_f16); return; }
  if (any_f16) throw std::runtime_error("conv2d: half-precision tensors are only handled by the tensor-core path (layer not eligible)");
  if (e.split_c) throw std::runtime_error("conv2d: merged two-output convolutions exist on the tensor-core path only");
  cx.launches++;
#ifdef GV_HOSTSIM
  const int OH = out.h, OW = out.w, IH = in0.h, IW = in0.w;
#pragma omp parallel for schedule(static)
  for (int m = 0; m < a.M; ++m) {
    int ox = m % OW; int r = m / OW; int oy = r % OH; int n = r / OH;
    std::vector<float> acc(w.cout, 0.f);
    for (int ky = 0; ky < w.kh; ++ky)
      for (int kx = 0; kx < w.kw; ++kx) {
        int iy = oy * g.stride - g.ph + ky, ix = ox * g.stride - g.pw + kx;
        if (g.reflect) { iy = reflect_idx(iy, IH); ix = reflect_idx(ix, IW); }
        if (iy < 0 || iy >= IH || ix < 0 || ix >= IW) continue;
        const float* p0 = in0.p + in0.off(n, iy, ix);
        const float* p1 = in1.p ? in1.p + in1.off(n, iy, ix) : nullptr;
        const float* wt = w.w + (int64_t)(ky * w.kw + kx) * w.cin * w.cout_ld;
        for (int ci = 0; ci < w.cin; ++ci) {
          float x = ci < a.c0 ? p0[ci] : p1[ci - a.c0];
          const float* wr = wt + (int64_t)ci * w.cout_ld;
          for (int co = 0; co < w.cout; ++co) acc[co] += x * wr[co];
        }
      }
    float* o = out.p + out.off(n, oy, ox);
    for (int co = 0; co < w.cout; ++co) o[co] = conv_epilogue(a, acc[co], n, oy, ox, co);
  }
#else
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  a.vec_ok = in0.ld % 4 == 0 && al16(in0.p) && (in0.sn % 4 == 0) &&
             (!in1.p || (in1.ld % 4 == 0 && al16(in1.p) && in1.sn % 4 == 0 && in0.c % 4 == 0));
  if (in1.p && in0.c % 16 != 0) throw std::runtime_error("conv2d: first concat segment must be a multiple of 16 channels");
  if (w.cout_ld % 4 != 0) throw std::runtime_error("conv2d: cout_ld must be a multiple of 4");
  if (cx.prof) {
    char nm[128];
    snprintf(nm, sizeof nm, "conv2d_simt_n%d k%dx%d s%d c%d>%d @%dx%dx%d", w.cout <= 16 ? 16 : 64, w.kh, w.kw, g.stride, w.cin, w.cout, out.n, out.h, out.w);
    cx.prof->begin(cx.stream, prof_intern(nm), 2.0 * a.M * w.cout * (double)w.cin * w.kh * w.kw);
  }
  if (w.cout <= 16) {
    dim3 grid((a.M + 127) / 128, (w.cout + 15) / 16);
    conv2d_simt_kernel<16, 4, 2><<<grid, 256, 0, cx.stream>>>(a);
  } else {
    dim3 grid((a.M + 127) / 128, (w.cout + 63) / 64);
    conv2d_simt_kernel<64, 8, 4><<<grid, 256, 0, cx.stream>>>(a);
  }
  gv_check_launch("conv2d");
  if (cx.prof) cx.prof->end(cx.stream);
#endif
}

}  // namespace gv
