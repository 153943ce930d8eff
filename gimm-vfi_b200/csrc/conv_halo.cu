// 3x3 (and 1x1) convolution for K-POOR layers (cin <= 32 fp32 / <= 64 half, cout <= 64) on wgmma: the activation tile is loaded ONCE
// with its halo, the weights of all taps stay resident in shared memory, and every tap is an MMA on a view of the loaded tile.
//
// Why: conv_tc.cu walks K as (tap, 32-channel block) and fetches one 16 KB TMA box per K step - 9 boxes = 144 KB per 128-pixel tile of a
// 3x3 layer whose distinct input is 23 KB, plus the weight boxes.  Here a tile costs 54 KB of TMA traffic and no weight traffic.
//
// How: output tile = 8 (x) x 16 (y) pixels, so the 8-row groups of the M = 128 operand are image rows.  Three TMA boxes
// {K, 8 x, 18 y} land the tile's columns shifted by kx = 0, 1, 2 (with the halo rows) 128B-swizzled in shared memory, each 18 KB =
// a whole number of 1024-byte swizzle atoms; tap (ky, kx) is then the operand descriptor of copy kx started ky image rows (= ky atoms)
// further, so every descriptor start is 1024-byte aligned and the canonical K-major SWIZZLE_128B layout holds for every tap.
// Out-of-bounds box elements are zero-filled = the convolution's zero padding.  1x1 layers load the 8 x 16 tile itself (one tap).
//
// Roles: warp 8 TMA producer (weights once, then one stage per tile), warpgroups 0 / 1 the MMAs of image rows 0-7 / 8-15 of the tile
// and their epilogue straight from the accumulator registers: a thread holds two pixels (one column, two rows) x BN / 4 channels as
// channel pairs; the four threads of a quad write 8 consecutive channels = 32 contiguous bytes of the NHWC output.
#include "common.h"

#ifndef GV_HOSTSIM
#include <cuda.h>
#include <cuda_fp16.h>

namespace gv {
namespace tc {
#include "tc_ptx.cuh"
#include "tc_epilogue.cuh"

constexpr int HL_TW = 8, HL_TH = 16;                  // output tile (x, y)
constexpr int HL_BH = HL_TH + 2;                      // halo rows
constexpr int HL_COPY_BYTES = HL_TW * HL_BH * 128;    // one x-shifted copy: 18 KB
constexpr int HL_MAX_STAGES = 4;
constexpr int HL_THREADS = 256 + 32;

struct HaloParams {
  int tiles_x, tiles_y, n_img, H, W, cout, stages, origin, round_out, spin_limit;
  int halo_bytes;   // bytes of one pipeline stage (multiple of 1024)
  int ntaps;        // 9 (3x3) or 1 (1x1)
  const float* bias; int act1; const float* slope1; int act2; const float* slope2;
  TV res, out;
};

// 2 channels (c, c + 1) of an fp32 or half tensor at element offset eoff; channels >= cout read as 0 / are not written
__device__ __forceinline__ void load2_any(const TV& t, int64_t eoff, int c, int cout, float* r) {
  if (t.f16) {
    const __half* q = reinterpret_cast<const __half*>(t.p) + eoff;
    r[0] = __half2float(q[0]); r[1] = c + 1 < cout ? __half2float(q[1]) : 0.f;
  } else {
    r[0] = t.p[eoff]; r[1] = c + 1 < cout ? t.p[eoff + 1] : 0.f;
  }
}
__device__ __forceinline__ void store2(const TV& t, int64_t eoff, const float* o, int c, int cout) {
  const bool two = c + 1 < cout;
  if (t.f16) {
    __half* q = reinterpret_cast<__half*>(t.p) + eoff;
    const float a = fminf(fmaxf(o[0], -65504.f), 65504.f), b = fminf(fmaxf(o[1], -65504.f), 65504.f);
    if (two && (reinterpret_cast<uintptr_t>(q) & 3) == 0) *reinterpret_cast<__half2*>(q) = __floats2half2_rn(a, b);
    else { q[0] = __float2half_rn(a); if (two) q[1] = __float2half_rn(b); }
  } else {
    float* q = t.p + eoff;
    if (two && (reinterpret_cast<uintptr_t>(q) & 7) == 0) *reinterpret_cast<float2*>(q) = make_float2(o[0], o[1]);
    else { q[0] = o[0]; if (two) q[1] = o[1]; }
  }
}

// BN: output channels (32 / 64), F16: half operands, NTAPS: 9 or 1 - all compile-time, so the MMA chain of a tile is straight-line
// code whose accumulators stay in fixed registers (no serialising register moves between the asynchronous MMAs)
template <int BN, bool F16, int NTAPS>
__global__ void __launch_bounds__(HL_THREADS, 1) conv3x3_halo_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                                                                    const __grid_constant__ HaloParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int w_bytes = NTAPS * BN * 128;
  const int w_region = (w_bytes + 1023) & ~1023;
  uint8_t* wsm = smem;
  uint8_t* halo = smem + w_region;
  uint64_t* bars = reinterpret_cast<uint64_t*>(halo + p.stages * p.halo_bytes);
  uint64_t* w_bar = bars;                          // weights landed
  uint64_t* full_bar = bars + 1;                   // [HL_MAX_STAGES]
  uint64_t* empty_bar = bars + 1 + HL_MAX_STAGES;  // [HL_MAX_STAGES]  the 8 consumer warps are done with the stage
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.n_img * p.tiles_y * p.tiles_x;
  const int SPIN = p.spin_limit;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmW)) : "memory");
    mbar_init(w_bar, 1);
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if (elect_one()) {
      mbar_expect_tx(w_bar, (uint32_t)w_bytes);
      tma_load_3d(wsm, &tmW, w_bar, 0, 0, 0);   // {K block, BN rows, taps}
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int r = tile; const int tx = r % p.tiles_x; r /= p.tiles_x; const int ty = r % p.tiles_y; const int n = r / p.tiles_y;
        mbar_wait(&empty_bar[stage], phase ^ 1, SPIN);
        mbar_expect_tx(&full_bar[stage], (uint32_t)p.halo_bytes);
        const int ncopies = NTAPS == 9 ? 3 : 1;
        for (int kx = 0; kx < ncopies; ++kx)
          tma_load_4d(halo + stage * p.halo_bytes + kx * HL_COPY_BYTES, &tmA, &full_bar[stage], 0, tx * HL_TW + p.origin + kx, ty * HL_TH + p.origin, n);
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  const int wg = warp >> 2, wq = warp & 3, gid = lane >> 2, tig = lane & 3;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  mbar_wait(w_bar, 0, SPIN);
  const uint32_t w_s = smem_u32(wsm);
  int stage = 0; uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int r = tile; const int tx = r % p.tiles_x; r /= p.tiles_x; const int ty = r % p.tiles_y; const int n = r / p.tiles_y;
    mbar_wait(&full_bar[stage], phase, SPIN);
    const uint32_t h_s = smem_u32(halo + stage * p.halo_bytes) + (uint32_t)(wg * 64 * 128);   // this warpgroup's 8 image rows
    wgmma_fence();
#pragma unroll
    for (int tap = 0; tap < NTAPS; ++tap) {
      const int ky = tap / 3, kx = tap % 3;
      const uint64_t ad = make_smem_desc(h_s + (uint32_t)(kx * HL_COPY_BYTES + ky * HL_TW * 128));   // copy kx, image row ky
      const uint64_t bd = make_smem_desc(w_s + (uint32_t)(tap * BN * 128));
#pragma unroll
      for (int k = 0; k < 4; ++k)   // 32 bytes of K per MMA (8 tf32 / 16 half); channels beyond cin are TMA zero fill on both operands
        wgmma_ss<BN, F16>(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (tap | k) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<BN / 2>(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);   // the producer refills the stage while this warp runs the epilogue
    if (++stage == p.stages) { stage = 0; phase ^= 1; }
    // ---- epilogue: rows gid / gid + 8 of the warp's 16 = pixel column gid of image rows y0, y0 + 1
    const int x = tx * HL_TW + gid, y0 = ty * HL_TH + wg * 8 + wq * 2;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = 8 * j + 2 * tig;
      if (c >= p.cout) break;
      const float b0 = __ldg(p.bias + c), b1 = __ldg(p.bias + c + 1);   // (bias padded past cout)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int y = y0 + h;
        if (y >= p.H || x >= p.W) continue;
        float o[2] = {acc[4 * j + 2 * h] + b0, acc[4 * j + 2 * h + 1] + b1};
        act_n<2>(o, p.act1, p.slope1, c, p.cout);
        if (p.res.p) { float t[2]; load2_any(p.res, p.res.off(n, y, x) + c, c, p.cout, t); o[0] += t[0]; o[1] += t[1]; }
        if (p.act2 != ACT_NONE) act_n<2>(o, p.act2, p.slope2, c, p.cout);
        if (p.round_out) { o[0] = rn_tf32(o[0]); o[1] = rn_tf32(o[1]); }
        store2(p.out, p.out.off(n, y, x) + c, o, c, p.cout);
      }
    }
  }
}

}  // namespace tc

template <int BN, bool F16, int NTAPS>
static void launch_halo(int grid, int smem, gvStream_t stream, const CUtensorMap& a, const CUtensorMap& w, const tc::HaloParams& p) {
  static volatile unsigned char attr[64];   // per (instantiation, device); set once: the layer-dependent size must always fit
  gv_set_max_smem(tc::conv3x3_halo_kernel<BN, F16, NTAPS>, 227 * 1024, attr);
  tc::conv3x3_halo_kernel<BN, F16, NTAPS><<<grid, tc::HL_THREADS, smem, stream>>>(a, w, p);
}

bool conv2d_halo_supported(const TV& in0, const TV& in1, const ConvW& w, const ConvGeom& g, const ConvEpi& e, const TV& out) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (in1.p || !((w.kh == 3 && w.kw == 3) || (w.kh == 1 && w.kw == 1)) || g.stride != 1 || g.reflect || w.cout > 64) return false;
  if (e.mul.p || e.gru_z.p || e.out2.p || e.split_c) return false;
  const bool h = in0.f16 != 0;
  if (h ? (!w.w_tc_h || w.cin_pad_h != 64 || in0.c > 64) : (!w.w_tc || w.cin_pad != 32 || in0.c > 32)) return false;
  if (!al16(in0.p) || in0.ld % (h ? 8 : 4) || in0.sn % (h ? 8 : 4)) return false;
  const int pad = w.kh / 2;
  if (g.loose_w ? (g.ph != 0 || g.pw != 0 || in0.h < out.h + 2 * pad || in0.w < out.w + 2 * pad || pad == 0) : (g.ph != pad || g.pw != pad || in0.h != out.h || in0.w != out.w)) return false;
  return in0.n == out.n;
}

void conv2d_halo(Ctx& cx, const TV& in0, const ConvW& w, const ConvGeom& g, const ConvEpi& e, const TV& out) {
  using namespace tc;
  const bool f16 = in0.f16 != 0;
  const bool one = w.kh == 1;                          // 1x1: no halo, one tap
  const int ntaps = one ? 1 : 9;
  const int c16 = (w.cout + 15) & ~15;
  const int BN = c16 <= 32 ? 32 : 64;
  if (w.cout_pad < c16) throw std::runtime_error("conv2d_halo: weight padding");
  CUtensorMap mA, mW;
  {
    const cuuint64_t es = f16 ? 2 : 4;
    cuuint64_t dims[4] = {(cuuint64_t)in0.c, (cuuint64_t)in0.w, (cuuint64_t)in0.h, (cuuint64_t)in0.n};
    cuuint64_t str[3] = {(cuuint64_t)in0.ld * es, (cuuint64_t)in0.w * in0.ld * es, (cuuint64_t)in0.sn * es};
    cuuint32_t box[4] = {(cuuint32_t)(f16 ? 64 : 32), (cuuint32_t)HL_TW, (cuuint32_t)(one ? HL_TH : HL_BH), 1};
    encode(&mA, in0.p, 4, dims, str, box, f16);
  }
  {   // weights [tap][cout_pad][K block]: rows beyond cout_pad are zero-filled by TMA
    const int kpad = f16 ? w.cin_pad_h : w.cin_pad;
    const cuuint64_t es = f16 ? 2 : 4;
    cuuint64_t dims[3] = {(cuuint64_t)kpad, (cuuint64_t)w.cout_pad, (cuuint64_t)ntaps};
    cuuint64_t str[2] = {(cuuint64_t)kpad * es, (cuuint64_t)kpad * w.cout_pad * es};
    cuuint32_t box[3] = {(cuuint32_t)(f16 ? 64 : 32), (cuuint32_t)BN, (cuuint32_t)ntaps};
    encode(&mW, f16 ? w.w_tc_h : static_cast<const void*>(w.w_tc), 3, dims, str, box, f16);
  }
  HaloParams p;
  p.tiles_x = (out.w + HL_TW - 1) / HL_TW; p.tiles_y = (out.h + HL_TH - 1) / HL_TH; p.n_img = out.n; p.H = out.h; p.W = out.w; p.cout = w.cout;
  p.origin = (g.loose_w || one) ? 0 : -1; p.round_out = out.f16 ? 0 : 1;
  p.spin_limit = tc_spin_limit();
  p.bias = w.b; p.act1 = e.act1; p.slope1 = e.slope1; p.act2 = e.act2; p.slope2 = e.slope2; p.res = e.res; p.out = out;
  p.ntaps = ntaps;
  p.halo_bytes = one ? HL_TW * HL_TH * 128 : 3 * HL_COPY_BYTES;
  const int w_region = (ntaps * BN * 128 + 1023) & ~1023;
  const int fixed = w_region + 256 + 1024;
  p.stages = (227 * 1024 - fixed) / p.halo_bytes;
  if (p.stages > HL_MAX_STAGES) p.stages = HL_MAX_STAGES;
  if (p.stages < 2) throw std::runtime_error("conv2d_halo: not enough shared memory");
  const int smem = fixed + p.stages * p.halo_bytes;
  const int num_tiles = p.n_img * p.tiles_y * p.tiles_x;
  const int grid = num_tiles < cx.sm_count ? num_tiles : cx.sm_count;
  cx.launches++;
  if (cx.prof) {
    char nm[128];
    snprintf(nm, sizeof nm, "conv2d_halo_%s k%dx%d c%d>%d @%dx%dx%d", f16 ? "f16" : "tf32", w.kh, w.kw, w.cin, w.cout, out.n, out.h, out.w);
    cx.prof->begin(cx.stream, prof_intern(nm), 2.0 * (double)out.n * out.h * out.w * w.cout * (double)w.cin * ntaps);
  }
  const int variant = (BN == 64 ? 4 : 0) | (f16 ? 2 : 0) | (one ? 1 : 0);
  switch (variant) {
    case 0: launch_halo<32, false, 9>(grid, smem, cx.stream, mA, mW, p); break;
    case 1: launch_halo<32, false, 1>(grid, smem, cx.stream, mA, mW, p); break;
    case 2: launch_halo<32, true, 9>(grid, smem, cx.stream, mA, mW, p); break;
    case 3: launch_halo<32, true, 1>(grid, smem, cx.stream, mA, mW, p); break;
    case 4: launch_halo<64, false, 9>(grid, smem, cx.stream, mA, mW, p); break;
    case 5: launch_halo<64, false, 1>(grid, smem, cx.stream, mA, mW, p); break;
    case 6: launch_halo<64, true, 9>(grid, smem, cx.stream, mA, mW, p); break;
    default: launch_halo<64, true, 1>(grid, smem, cx.stream, mA, mW, p); break;
  }
  gv_check_launch("conv2d_halo");
  if (cx.prof) cx.prof->end(cx.stream);
}

}  // namespace gv
#endif  // GV_HOSTSIM
