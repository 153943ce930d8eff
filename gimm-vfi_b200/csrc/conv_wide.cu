// 3x3 stride-1 zero-padded convolution of WIDE half layers (every input segment a multiple of 64 channels, cout a multiple of N) on f16
// wgmma: the final decoder's 256-channel residual trunk.  The activation tile of a 64-channel K block is loaded ONCE with its halo and
// all nine taps are MMAs on views of it, as in conv_halo.cu; the weights stream per (K block, tap).
//
// Why: conv_tc.cu walks K as (tap, K block) and fetches a fresh 16 KB activation box for every tap: 9 x 16 KB per 128-pixel tile and
// 64-channel K block for 23 KB of distinct input.  Here that is 3 x 18 KB, so a (128-pixel, 128-channel) tile moves 216 KB of
// activations + 576 KB of weights from L2 instead of 576 + 576 KB.  Measured (DESIGN §7): that cut leaves the layers without a residual
// as fast as on conv_tc; the gain is the in-place residual layer's, whose conv_tc epilogue is slow.
//
// How: output tile = 8 (x) x 16 (y) pixels, so each 8-row group of the M = 128 operand is one image row = one 1024-byte swizzle atom.
// Per K block the producer issues three TMA boxes {64 ch, 8 x, 18 y} at x offsets -1, 0, +1 (SWIZZLE_128B, out-of-bounds zero fill
// = the padding); tap (ky, kx) is the descriptor of copy kx started ky atoms further.  K blocks come from two tensor maps (two input
// segments, as conv_tc's tmA0 / tmA1).  The {64 k, N} weight box of each (K block, tap) streams through its own ring.
// Roles as conv_tc.cu: warpgroup 2 produces (one elected thread; setmaxnreg hands its registers to the consumers), warpgroups 0 / 1
// run the MMAs of image rows 0-7 / 8-15 with one MMA group in flight across taps, and the epilogue of their rows while the producer
// runs ahead into the next tile.  Epilogue: epi_pieces (tc_epilogue.cuh), 64 channels per pass.
#include "common.h"

#ifndef GV_HOSTSIM
#include <cuda.h>
#include <cuda_fp16.h>

namespace gv {
namespace tc {
#include "tc_ptx.cuh"
#include "tc_epilogue.cuh"

constexpr int WD_TW = 8, WD_TH = 16, WD_BH = WD_TH + 2;   // output tile (x, y), halo rows
constexpr int WD_N = 128;                                  // output channels per tile
constexpr int WD_ROW = WD_TW * 128;                        // one image row of a copy = one swizzle atom
constexpr int WD_COPY = WD_BH * WD_ROW;                    // one x-shifted copy: 18 KB
constexpr int WD_A_BYTES = 3 * WD_COPY;                    // one A stage: 54 KB
constexpr int WD_A_STAGES = 2, WD_B_STAGES = 5;
constexpr int WD_STG_LD = 64 * 4 + 16;                     // staged pixel row: 64 fp32 channels + 16 bytes of bank offset
constexpr int WD_THREADS = 384;
constexpr int WD_PRODUCER_REGS = 40, WD_CONSUMER_REGS = 232;   // 128 x (2 x 232 + 40) = 384 x 168, the launch budget

struct WideParams {
  int tiles_x, tiles_y, n_img, tiles_n, H, W, cout, kblocks, c0_blocks, round_out, spin_limit;
  const float* bias; int act1; const float* slope1; int act2; const float* slope2;
  TV res, out;
};

template <int N>
__global__ void __launch_bounds__(WD_THREADS, 1)
conv3x3_wide_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ WideParams p) {
  constexpr int B_BYTES = N * 128;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_ring = smem;
  uint8_t* b_ring = a_ring + WD_A_STAGES * WD_A_BYTES;
  uint8_t* stg_all = b_ring + WD_B_STAGES * B_BYTES;        // [8 warps][16 pixels][WD_STG_LD]
  uint64_t* bars = reinterpret_cast<uint64_t*>(stg_all + 8 * 16 * WD_STG_LD);
  uint64_t* full_a = bars;
  uint64_t* empty_a = full_a + WD_A_STAGES;
  uint64_t* full_b = empty_a + WD_A_STAGES;
  uint64_t* empty_b = full_b + WD_B_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.n_img * p.tiles_y * p.tiles_x * p.tiles_n;
  const int SPIN = p.spin_limit;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA0)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA1)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB)) : "memory");
    for (int s = 0; s < WD_A_STAGES; ++s) { mbar_init(&full_a[s], 1); mbar_init(&empty_a[s], 8); }
    for (int s = 0; s < WD_B_STAGES; ++s) { mbar_init(&full_b[s], 1); mbar_init(&empty_b[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // tile index -> (pixel tile, N tile): consecutive indices share the pixel tile
  if (warp >= 8) {
    // ===================================================== TMA producer
    setmaxnreg_dec<WD_PRODUCER_REGS>();
    if (warp == 8 && elect_one()) {
      int sa = 0, sb = 0; uint32_t pa = 0, pb = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int nt = tile % p.tiles_n; int r = tile / p.tiles_n;
        const int tx = r % p.tiles_x; r /= p.tiles_x; const int ty = r % p.tiles_y; const int n = r / p.tiles_y;
        for (int kb = 0; kb < p.kblocks; ++kb) {
          mbar_wait(&empty_a[sa], pa ^ 1, SPIN);
          mbar_expect_tx(&full_a[sa], (uint32_t)WD_A_BYTES);
          const CUtensorMap* ta = kb < p.c0_blocks ? &tmA0 : &tmA1;
          const int ch = (kb < p.c0_blocks ? kb : kb - p.c0_blocks) * 64;
          uint8_t* a_dst = a_ring + sa * WD_A_BYTES;
          for (int kx = 0; kx < 3; ++kx) tma_load_4d(a_dst + kx * WD_COPY, ta, &full_a[sa], ch, tx * WD_TW + kx - 1, ty * WD_TH - 1, n);
          if (++sa == WD_A_STAGES) { sa = 0; pa ^= 1; }
          for (int tap = 0; tap < 9; ++tap) {
            mbar_wait(&empty_b[sb], pb ^ 1, SPIN);
            mbar_expect_tx(&full_b[sb], (uint32_t)B_BYTES);
            tma_load_3d(b_ring + sb * B_BYTES, &tmB, &full_b[sb], kb * 64, nt * N, tap);
            if (++sb == WD_B_STAGES) { sb = 0; pb ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ===================================================== consumer warpgroups
  setmaxnreg_inc<WD_CONSUMER_REGS>();
  const int wg = warp >> 2, wq = warp & 3, gid = lane >> 2, tig = lane & 3;
  const uint32_t a_s = smem_u32(a_ring), b_s = smem_u32(b_ring);
  const uint32_t stg_s = smem_u32(stg_all + warp * 16 * WD_STG_LD);
  float acc[N / 2];
  int sa = 0, sb = 0; uint32_t pa = 0, pb = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int nt = tile % p.tiles_n; int r = tile / p.tiles_n;
    const int tx = r % p.tiles_x; r /= p.tiles_x; const int ty = r % p.tiles_y; const int n = r / p.tiles_y;
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    int prev_b = -1, prev_a = -1;   // the stages read by the MMA group in flight (prev_a: only after the last tap of a K block)
    for (int kb = 0; kb < p.kblocks; ++kb) {
      mbar_wait(&full_a[sa], pa, SPIN);
      const uint32_t a_stage = a_s + (uint32_t)(sa * WD_A_BYTES + wg * 8 * WD_ROW);
#pragma unroll 1
      for (int tap = 0; tap < 9; ++tap) {
        const int ky = tap / 3, kx = tap - 3 * ky;
        mbar_wait(&full_b[sb], pb, SPIN);
        const uint64_t ad = make_smem_desc(a_stage + (uint32_t)(kx * WD_COPY + ky * WD_ROW));
        const uint64_t bd = make_smem_desc(b_s + (uint32_t)(sb * B_BYTES));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)   // 32 bytes of every 128-byte row per MMA (16 half) -> +2 in the (addr >> 4) field
          wgmma_ss<N, true>(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (kb | tap | k) ? 1u : 0u);
        wgmma_commit();
        if (prev_b >= 0) {   // the previous group has retired once at most this one is pending
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) { mbar_arrive(&empty_b[prev_b]); if (prev_a >= 0) mbar_arrive(&empty_a[prev_a]); }
        }
        prev_b = sb; prev_a = tap == 8 ? sa : -1;
        if (++sb == WD_B_STAGES) { sb = 0; pb ^= 1; }
      }
      if (++sa == WD_A_STAGES) { sa = 0; pa ^= 1; }
    }
    // ---- epilogue: the warp's 16 pixels (image rows 8 wg + 2 wq, + 1; columns 0-7) x N channels, 64 channels per pass
    const int yw = ty * WD_TH + 8 * wg + 2 * wq;
#pragma unroll
    for (int cp = 0; cp < N / 64; ++cp) {
      const int cb = nt * N + cp * 64;
      auto piece = [&](int q, int& px, int& py, int& c0) {
        const int pix = q >> 3;
        px = tx * WD_TW + (pix & 7); py = yw + (pix >> 3); c0 = cb + (q & 7) * 8;
        return px < p.W && py < p.H && c0 < p.cout;
      };
      uint4 rcur[2];
      if (p.res.p) epi_load_res(p, n, lane, piece, rcur);   // (pass 0: while the last MMAs run)
      if (cp == 0) {
        wgmma_wait<0>();
        reg_fence<N / 2>(acc);
        __syncwarp();
        if (lane == 0) { mbar_arrive(&empty_b[prev_b]); mbar_arrive(&empty_a[prev_a]); }
      }
      // raw accumulators to the staging rows: row = pixel 8 hh + gid, channels 8 j + 2 tig, + 1 of this pass
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          sts64(stg_s + (uint32_t)((8 * hh + gid) * WD_STG_LD + (8 * j + 2 * tig) * 4), acc[4 * (8 * cp + j) + 2 * hh], acc[4 * (8 * cp + j) + 2 * hh + 1]);
      __syncwarp();
      epi_pieces<16 * 8, 8>(p, n, stg_s, WD_STG_LD, lane, piece, rcur);
      __syncwarp();   // the staging rows are rewritten by the next pass
    }
  }
}

}  // namespace tc

bool conv2d_wide_supported(const TV& in0, const TV& in1, const ConvW& w, const ConvGeom& g, const ConvEpi& e, const TV& out) {
  auto seg_ok = [&](const TV& t) {
    return t.f16 && t.c % 64 == 0 && (reinterpret_cast<uintptr_t>(t.p) & 15) == 0 && t.ld % 8 == 0 && t.sn % 8 == 0 && t.n == out.n &&
           t.h == out.h && t.w == out.w;
  };
  if (w.kh != 3 || w.kw != 3 || g.stride != 1 || g.reflect || g.loose_w || g.ph != 1 || g.pw != 1 || !w.w_tc_h) return false;
  if (e.mul.p || e.gru_z.p || e.out2.p || e.split_c) return false;
  if (!seg_ok(in0) || (in1.p && !seg_ok(in1))) return false;
  const int cin = in0.c + (in1.p ? in1.c : 0);
  return cin == w.cin && w.cin_pad_h == cin && w.cout % tc::WD_N == 0 && w.cout_pad >= w.cout;
}

void conv2d_wide(Ctx& cx, const TV& in0, const TV& in1, const ConvW& w, const ConvGeom& g, const ConvEpi& e, const TV& out) {
  using namespace tc;
  (void)g;
  constexpr int N = WD_N;
  auto encode_seg = [](CUtensorMap* m, const TV& t) {
    cuuint64_t dims[4] = {(cuuint64_t)t.c, (cuuint64_t)t.w, (cuuint64_t)t.h, (cuuint64_t)t.n};
    cuuint64_t str[3] = {(cuuint64_t)t.ld * 2, (cuuint64_t)t.w * t.ld * 2, (cuuint64_t)t.sn * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)WD_TW, (cuuint32_t)WD_BH, 1};
    encode(m, t.p, 4, dims, str, box, true);
  };
  CUtensorMap mA0, mA1, mB;
  encode_seg(&mA0, in0);
  if (in1.p) encode_seg(&mA1, in1); else mA1 = mA0;
  {   // packed weights [tap][cout_pad][cin_pad_h] half
    cuuint64_t dims[3] = {(cuuint64_t)w.cin_pad_h, (cuuint64_t)w.cout_pad, 9};
    cuuint64_t str[2] = {(cuuint64_t)w.cin_pad_h * 2, (cuuint64_t)w.cin_pad_h * w.cout_pad * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)N, 1};
    encode(&mB, w.w_tc_h, 3, dims, str, box, true);
  }
  WideParams p;
  p.tiles_x = (out.w + WD_TW - 1) / WD_TW; p.tiles_y = (out.h + WD_TH - 1) / WD_TH; p.n_img = out.n; p.tiles_n = w.cout / N;
  p.H = out.h; p.W = out.w; p.cout = w.cout;
  p.kblocks = w.cin / 64; p.c0_blocks = in0.c / 64;
  p.round_out = out.f16 ? 0 : 1;
  p.spin_limit = tc_spin_limit();
  p.bias = w.b; p.act1 = e.act1; p.slope1 = e.slope1; p.act2 = e.act2; p.slope2 = e.slope2; p.res = e.res; p.out = out;
  const int smem = WD_A_STAGES * WD_A_BYTES + WD_B_STAGES * N * 128 + 8 * 16 * WD_STG_LD + 256 + 1024;
  const int num_tiles = p.n_img * p.tiles_y * p.tiles_x * p.tiles_n;
  const int grid = num_tiles < cx.sm_count ? num_tiles : cx.sm_count;
  cx.launches++;
  if (cx.prof) {
    char nm[128];
    snprintf(nm, sizeof nm, "conv2d_wide_f16 k3x3 c%d>%d @%dx%dx%d", w.cin, w.cout, out.n, out.h, out.w);
    cx.prof->begin(cx.stream, prof_intern(nm), 2.0 * (double)out.n * out.h * out.w * w.cout * (double)w.cin * 9);
  }
  static volatile unsigned char attr[64];
  gv_set_max_smem(conv3x3_wide_kernel<N>, smem, attr);
  conv3x3_wide_kernel<N><<<grid, WD_THREADS, smem, cx.stream>>>(mA0, mA1, mB, p);
  gv_check_launch("conv2d_wide");
  if (cx.prof) cx.prof->end(cx.stream);
}

}  // namespace gv
#endif  // GV_HOSTSIM
