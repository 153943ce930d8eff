// 3x3 (and 1x1) convolution for K-POOR layers (cin <= 32 fp32 / <= 64 half, cout <= 64) on wgmma: the activation tile is loaded ONCE
// with its halo, the weights of all taps stay resident in shared memory, and every tap is an MMA on a view of the loaded tile.
//
// Why: conv_tc.cu walks K as (tap, 32-channel block) and fetches one 16 KB TMA box per K step - 9 boxes = 144 KB per 128-pixel tile of a
// 3x3 layer whose distinct input is 23 KB, plus the weight boxes.  Here a tile costs 54 KB of TMA traffic and no weight traffic.
//
// How: output tile = 8 (x) x 16 (y) pixels, so the 8-row groups of the M = 128 operand are image rows.  Three TMA boxes
// {K, 8 x, 18 y} land the tile's columns shifted by kx = 0, 1, 2 (with the halo rows) swizzled in shared memory, each a whole number
// of swizzle atoms; tap (ky, kx) is then the operand descriptor of copy kx started ky image rows (= ky atoms) further, so every
// descriptor start is atom-aligned and the canonical K-major swizzled layout holds for every tap.  K rows are 128 bytes (SWIZZLE_128B,
// 18 KB per copy), or 64 bytes (SWIZZLE_64B, 9 KB per copy) when the input's channels fit: 32 half / 16 fp32 channels then take half
// the MMAs and half the stage.  Out-of-bounds box elements are zero-filled = the convolution's zero padding.  1x1 layers load the
// 8 x 16 tile itself (one tap).
//
// Roles: warp 8 TMA producer (weights once, then one stage per tile); with 32 output channels warpgroups 0 / 1 alternate whole tiles
// (two m64 accumulators: image rows 0-7 / 8-15), so one warpgroup's epilogue runs under the other's MMAs; with 64 they take image
// rows 0-7 / 8-15 of every tile.  The epilogue stages the raw accumulators per warp in shared
// memory and runs over 8-channel pieces of whole pixels (16- or 32-byte stores of the NHWC output), reading each piece's residual
// one piece ahead, the first while the MMAs run.
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
constexpr int HL_MAX_STAGES = 6;
constexpr int HL_THREADS = 256 + 32;

struct HaloParams {
  int tiles_x, tiles_y, n_img, H, W, cout, stages, origin, round_out, spin_limit;
  int halo_bytes;   // bytes of one pipeline stage (multiple of 1024)
  int stg_ld;       // bytes per pixel of the accumulator staging (BN fp32 channels + 16 bytes of bank offset)
  const float* bias; int act1; const float* slope1; int act2; const float* slope2;
  TV res, out;
};

// K-major operand descriptor of rows of RB bytes: SWIZZLE_128B (RB = 128) or SWIZZLE_64B (RB = 64); 8-row atoms of 8 RB bytes (SBO)
template <int RB>
__device__ __forceinline__ uint64_t halo_desc(uint32_t saddr) {
  if constexpr (RB == 128) return make_smem_desc(saddr);
  else {
    static_assert(RB == 64, "RB");
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(512 >> 4) << 32;
    d |= (uint64_t)2 << 62;   // layout type 2 = SWIZZLE_64B
    return d;
  }
}

// BN: output channels (32 / 64), F16: half operands, NTAPS: 9 or 1, RB: bytes of K per operand row (128, or 64 when the input's
// channels fit in 64 bytes: 32 half / 16 fp32 channels) - all compile-time, so the MMA chain of a tile is straight-line code whose
// accumulators stay in fixed registers (no serialising register moves between the asynchronous MMAs)
template <int BN, bool F16, int NTAPS, int RB>
__global__ void __launch_bounds__(HL_THREADS, 1) conv3x3_halo_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                                                                    const __grid_constant__ HaloParams p) {
  constexpr int KSTEPS = RB / 32;                 // 32 bytes of K per MMA (8 tf32 / 16 half)
  constexpr int COPY = HL_TW * HL_BH * RB;        // one x-shifted copy: a whole number of 1024-byte blocks
  constexpr int ROW = HL_TW * RB;                 // one image row of the tile = 8 operand rows = one swizzle atom
  // BN = 32: each warpgroup owns whole tiles (two m64 accumulators, image rows 0-7 / 8-15), so one warpgroup's epilogue runs under the
  // other's MMAs.  BN = 64: the two warpgroups split each tile (image rows 0-7 / 8-15): owning whole 64-channel tiles measured up to
  // 1.4x slower on these layers, the epilogue of a whole tile on 4 warps outlasting the other warpgroup's MMAs.
  constexpr bool OWN = BN == 32;
  constexpr int NH = OWN ? 2 : 1;                 // m64 halves of a tile per warpgroup
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int w_bytes = NTAPS * BN * RB;
  const int w_region = (w_bytes + 1023) & ~1023;
  uint8_t* wsm = smem;
  uint8_t* halo = smem + w_region;
  uint8_t* stg_all = halo + p.stages * p.halo_bytes;   // [8 warps][NH x 16 pixels][stg_ld bytes]
  uint64_t* bars = reinterpret_cast<uint64_t*>(stg_all + 8 * NH * 16 * p.stg_ld);
  uint64_t* w_bar = bars;                          // weights landed
  uint64_t* full_bar = bars + 1;                   // [HL_MAX_STAGES]
  uint64_t* empty_bar = bars + 1 + HL_MAX_STAGES;  // [HL_MAX_STAGES]  the consuming warps (4, or 8 when the warpgroups split a tile) are done
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.n_img * p.tiles_y * p.tiles_x;
  const int SPIN = p.spin_limit;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmW)) : "memory");
    mbar_init(w_bar, 1);
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], OWN ? 4 : 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // The CTA's i-th tile (tile blockIdx.x + i * gridDim.x) goes through stage i % stages, fill (i / stages); with OWN warpgroup i % 2
  // consumes it (the empty barrier counts that warpgroup's 4 warps), otherwise both do (8 warps).  Both sides derive the phase of fill
  // i from i alone.
  if (warp == 8) {
    if (elect_one()) {
      mbar_expect_tx(w_bar, (uint32_t)w_bytes);
      tma_load_3d(wsm, &tmW, w_bar, 0, 0, 0);   // {K, BN rows, taps}
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int r = tile; const int tx = r % p.tiles_x; r /= p.tiles_x; const int ty = r % p.tiles_y; const int n = r / p.tiles_y;
        mbar_wait(&empty_bar[stage], phase ^ 1, SPIN);
        mbar_expect_tx(&full_bar[stage], (uint32_t)p.halo_bytes);
        const int ncopies = NTAPS == 9 ? 3 : 1;
        for (int kx = 0; kx < ncopies; ++kx)
          tma_load_4d(halo + stage * p.halo_bytes + kx * COPY, &tmA, &full_bar[stage], 0, tx * HL_TW + p.origin + kx, ty * HL_TH + p.origin, n);
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  const int wg = warp >> 2, wq = warp & 3, gid = lane >> 2, tig = lane & 3;
  uint8_t* stg = stg_all + warp * NH * 16 * p.stg_ld;
  float acc[NH][BN / 2];
  mbar_wait(w_bar, 0, SPIN);
  const uint32_t w_s = smem_u32(wsm);
  for (int i = OWN ? wg : 0;; i += OWN ? 2 : 1) {
    const int tile = blockIdx.x + i * gridDim.x;
    if (tile >= num_tiles) break;
    const int stage = i % p.stages;
    const uint32_t phase = (uint32_t)(i / p.stages) & 1u;
    int r = tile; const int tx = r % p.tiles_x; r /= p.tiles_x; const int ty = r % p.tiles_y; const int n = r / p.tiles_y;
    mbar_wait(&full_bar[stage], phase, SPIN);
    const uint32_t h_s = smem_u32(halo + stage * p.halo_bytes);
    wgmma_fence();
#pragma unroll
    for (int tap = 0; tap < NTAPS; ++tap) {
      const int ky = tap / 3, kx = tap % 3;
      const uint64_t bd = halo_desc<RB>(w_s + (uint32_t)(tap * BN * RB));
#pragma unroll
      for (int h = 0; h < NH; ++h) {   // copy kx, image row 8 (h + wg) + ky or 8 h + ky
        const uint64_t ad = halo_desc<RB>(h_s + (uint32_t)(kx * COPY + (8 * (OWN ? h : wg) + ky) * ROW));
#pragma unroll
        for (int k = 0; k < KSTEPS; ++k)   // channels beyond cin are TMA zero fill on both operands
          wgmma_ss<BN, F16>(acc[h], ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (tap | k) ? 1u : 0u);
      }
    }
    wgmma_commit();
    // The epilogue works on 8-channel pieces of whole pixels (epi_pieces): the warp's NH x 16 pixels (image rows 8 h + 2 wq, + 1 with
    // OWN, else 8 wg + 2 wq, + 1; columns 0-7) x BN channels.  The first piece's residual is read while the MMAs run.
    constexpr int CPP = BN / 8;            // pieces per pixel
    constexpr int NPC = NH * 16 * CPP;     // pieces per warp and tile (a multiple of 32)
    const int yw = ty * HL_TH + (OWN ? 0 : 8 * wg) + wq * 2;
    auto piece = [&](int q, int& px, int& py, int& c0) {
      const int pix = q / CPP;
      px = tx * HL_TW + (pix & 7); py = yw + 8 * (pix >> 4) + ((pix >> 3) & 1); c0 = (q % CPP) * 8;
      return px < p.W && py < p.H && c0 < p.cout;
    };
    uint4 rcur[2];
    if (p.res.p) epi_load_res(p, n, lane, piece, rcur);
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < NH; ++h) reg_fence<BN / 2>(acc[h]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);   // the producer refills the stage while this warp runs the epilogue
    // raw accumulators to the staging rows: row = pixel 16 h + 8 hh + gid, channels 8 j + 2 tig, + 1
    const uint32_t stg_s = smem_u32(stg);
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          sts64(stg_s + (uint32_t)((16 * h + 8 * hh + gid) * p.stg_ld + (8 * j + 2 * tig) * 4), acc[h][4 * j + 2 * hh], acc[h][4 * j + 2 * hh + 1]);
    __syncwarp();
    epi_pieces<NPC, CPP>(p, n, stg_s, p.stg_ld, lane, piece, rcur);
    __syncwarp();   // the staging rows are rewritten by the next tile
  }
}

}  // namespace tc

template <int BN, bool F16, int NTAPS, int RB>
static void launch_halo(int grid, int smem, gvStream_t stream, const CUtensorMap& a, const CUtensorMap& w, const tc::HaloParams& p) {
  static volatile unsigned char attr[64];   // per (instantiation, device); set once: the layer-dependent size must always fit
  gv_set_max_smem(tc::conv3x3_halo_kernel<BN, F16, NTAPS, RB>, 227 * 1024, attr);
  tc::conv3x3_halo_kernel<BN, F16, NTAPS, RB><<<grid, tc::HL_THREADS, smem, stream>>>(a, w, p);
}

template <int BN, bool F16, int NTAPS>
static void launch_halo_rb(bool rb64, int grid, int smem, gvStream_t stream, const CUtensorMap& a, const CUtensorMap& w, const tc::HaloParams& p) {
  if (rb64) launch_halo<BN, F16, NTAPS, 64>(grid, smem, stream, a, w, p);
  else launch_halo<BN, F16, NTAPS, 128>(grid, smem, stream, a, w, p);
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
  const int es = f16 ? 2 : 4;
  const int rb = in0.c * es <= 64 ? 64 : 128;          // bytes of K per operand row: 32 half / 16 fp32 input channels fit in 64
  const CUtensorMapSwizzle swz = rb == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
  CUtensorMap mA, mW;
  {
    cuuint64_t dims[4] = {(cuuint64_t)in0.c, (cuuint64_t)in0.w, (cuuint64_t)in0.h, (cuuint64_t)in0.n};
    cuuint64_t str[3] = {(cuuint64_t)in0.ld * es, (cuuint64_t)in0.w * in0.ld * es, (cuuint64_t)in0.sn * es};
    cuuint32_t box[4] = {(cuuint32_t)(rb / es), (cuuint32_t)HL_TW, (cuuint32_t)(one ? HL_TH : HL_BH), 1};
    encode(&mA, in0.p, 4, dims, str, box, f16, 1, swz);
  }
  {   // weights [tap][cout_pad][K block]: rows beyond cout_pad are zero-filled by TMA; a 64-byte box reads the first half of each row
    const int kpad = f16 ? w.cin_pad_h : w.cin_pad;
    cuuint64_t dims[3] = {(cuuint64_t)kpad, (cuuint64_t)w.cout_pad, (cuuint64_t)ntaps};
    cuuint64_t str[2] = {(cuuint64_t)kpad * es, (cuuint64_t)kpad * w.cout_pad * es};
    cuuint32_t box[3] = {(cuuint32_t)(rb / es), (cuuint32_t)BN, (cuuint32_t)ntaps};
    encode(&mW, f16 ? w.w_tc_h : static_cast<const void*>(w.w_tc), 3, dims, str, box, f16, 1, swz);
  }
  HaloParams p;
  p.tiles_x = (out.w + HL_TW - 1) / HL_TW; p.tiles_y = (out.h + HL_TH - 1) / HL_TH; p.n_img = out.n; p.H = out.h; p.W = out.w; p.cout = w.cout;
  p.origin = (g.loose_w || one) ? 0 : -1; p.round_out = out.f16 ? 0 : 1;
  p.spin_limit = tc_spin_limit();
  p.bias = w.b; p.act1 = e.act1; p.slope1 = e.slope1; p.act2 = e.act2; p.slope2 = e.slope2; p.res = e.res; p.out = out;
  p.halo_bytes = (one ? HL_TH : 3 * HL_BH) * HL_TW * rb;
  p.stg_ld = BN * 4 + 16;
  const int w_region = (ntaps * BN * rb + 1023) & ~1023;
  const int fixed = w_region + 8 * (BN == 32 ? 2 : 1) * 16 * p.stg_ld + 256 + 1024;   // (pixels staged per warp: see OWN)
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
  const bool rb64 = rb == 64;
  switch (variant) {
    case 0: launch_halo_rb<32, false, 9>(rb64, grid, smem, cx.stream, mA, mW, p); break;
    case 1: launch_halo_rb<32, false, 1>(rb64, grid, smem, cx.stream, mA, mW, p); break;
    case 2: launch_halo_rb<32, true, 9>(rb64, grid, smem, cx.stream, mA, mW, p); break;
    case 3: launch_halo_rb<32, true, 1>(rb64, grid, smem, cx.stream, mA, mW, p); break;
    case 4: launch_halo_rb<64, false, 9>(rb64, grid, smem, cx.stream, mA, mW, p); break;
    case 5: launch_halo_rb<64, false, 1>(rb64, grid, smem, cx.stream, mA, mW, p); break;
    case 6: launch_halo_rb<64, true, 9>(rb64, grid, smem, cx.stream, mA, mW, p); break;
    default: launch_halo_rb<64, true, 1>(rb64, grid, smem, cx.stream, mA, mW, p); break;
  }
  gv_check_launch("conv2d_halo");
  if (cx.prof) cx.prof->end(cx.stream);
}

}  // namespace gv
#endif  // GV_HOSTSIM
