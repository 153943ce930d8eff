// All-pairs correlation GEMM for sm_90a in the 3xF16 form: vol[i][j] = scale * sum_k A[i][k] * B[j][k], fp32 out, row pitch = the
// number of targets.  Used by RAFT's correlation pyramid, FlowFormer's cost volume and its attention logits.
//
//   operands    both pre-split into half planes [2][rows][K] (split_planes_f16: hi = rn_f16(x), lo = rn_f16(x - hi)), one 3-D
//               tensor map {K, rows, plane} each; ragged M / N edges are TMA zero fill.  A tile is 128 consecutive source rows x 128
//               targets, so a tile's output rows are contiguous.
//   mainloop    SS wgmma (both operands from shared memory): per k16 A_hi*B_lo, A_lo*B_hi, A_hi*B_hi, segments of 2 K steps (of 64)
//               accumulated by the tensor core and summed in fp32 registers, * scale at the end - the arithmetic of the 3xF16 form of
//               conv2d_tc_kernel, on the same MMA inputs.  The MMAs of a K step stay in flight while the next one is issued.
//   epilogue    the result is staged in shared memory and stored with TMA (clipped at the ragged edges); the warpgroup does this
//               while the next tile's first MMAs run, in two halves of 64 columns.  Volumes whose row pitch is not a multiple of
//               16 bytes (RAFT's coarsest level at 1080p: 17 x 30 targets) cannot be a TMA store target; they take plain stores
//               from the same staging tile.
//   roles       warpgroups 0 / 1: MMAs of rows [0, 64) / [64, 128) and their epilogue | warpgroup 2: TMA producer (setmaxnreg)
//
// Shared memory: 3 stages x 64 KB (A hi, A lo, B hi, B lo: 128 rows x 128 bytes each) + 2 x 16 KB staging (one 64 x 64 fp32 half
// tile per warpgroup) = 224 KB.  Registers: two 64-float accumulator sets per consumer thread.  The set holding a finished tile is
// drained while the other one takes the next tile's first segment, so the tile loop alternates their roles.
#include "common.h"

#ifndef GV_HOSTSIM
#include <cuda.h>
#include <cuda_fp16.h>

namespace gv {

namespace tc {

#include "tc_ptx.cuh"

#include "tc_epilogue.cuh"

constexpr int CG_BM = 128, CG_BN = 128, CG_BK = 64, CG_STAGES = 3, CG_SEG = 2;
// M tiles per raster group: 32 x 4 tiles run at one time on 132 SMs.  Level-0 volume at 1080p (H100, 700 W): 3.51 ms with the
// N-fastest order (group 1), 3.18 / 2.93 / 2.88 / 3.07 / 3.21 ms with groups of 4 / 16 / 32 / 64 / 128
constexpr int CG_GROUP = 32;
constexpr int CG_OP_BYTES = 128 * 128;                          // one operand plane of one K step: 128 rows x 64 halves
constexpr int CG_STAGE_BYTES = 4 * CG_OP_BYTES;                 // A hi | A lo | B hi | B lo
constexpr int CG_STG_WG_BYTES = 64 * 64 * 4;                    // per warpgroup: 64 rows x 64 columns, two 32-column TMA boxes
constexpr int CG_THREADS = 384, CG_CONSUMERS = 256;
constexpr int CG_PRODUCER_REGS = 40, CG_CONSUMER_REGS = 232;
constexpr int CG_SMEM = 1024 + CG_STAGES * CG_STAGE_BYTES + 2 * CG_STG_WG_BYTES + 2 * CG_STAGES * 8;

struct CgParams {
  int M, NT, ksteps, tiles_m, tiles_n, num_tiles;
  int tma_store;                   // 0: plain stores (row pitch not a multiple of 16 bytes)
  float scale;
  float* vol;
  int spin_limit;
};

__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src),
               "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ float lds32(uint32_t a) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// Columns [64 HF, 64 HF + 64) of this warpgroup's 64 finished rows (accumulators d) -> staging -> the volume.
// Staging: box b (columns 32 b ..) = 64 rows x 128 bytes, 16-byte chunk c of row r at chunk c ^ (r & 7) (the TMA 128-byte swizzle).
template <int HF>
__device__ __forceinline__ void cg_drain_half(const CgParams& p, const CUtensorMap* tmO, const float* d, int m0, int n0, uint32_t stg, int wg, int wq,
                                              int lane) {
  const int gid = lane >> 2, tig = lane & 3, t = wq * 32 + lane;
  if (t == 0) bulk_wait_read0();   // the previous half's TMA store has read the staging tile
  wg_sync(1 + wg);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int col = 8 * j + 2 * tig, box = col >> 5, cb = col & 31, jj = 8 * HF + j;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = wq * 16 + gid + 8 * h;
      // fmaf(x, scale, 0): the rounding of conv2d_tc_kernel's epilogue (accumulator * out_scale + zero bias)
      sts64(stg + (uint32_t)(box * 8192 + row * 128 + (((cb >> 2) ^ (row & 7)) << 4) + (cb & 3) * 4), fmaf(d[4 * jj + 2 * h], p.scale, 0.f),
            fmaf(d[4 * jj + 2 * h + 1], p.scale, 0.f));
    }
  }
  fence_proxy_async_smem();
  wg_sync(1 + wg);
  const int r0 = m0 + 64 * wg, c0 = n0 + 64 * HF;
  if (p.tma_store) {
    if (t == 0) {
      tma_store_2d(tmO, stg, c0, r0);
      tma_store_2d(tmO, stg + 8192, c0 + 32, r0);
      bulk_commit();
    }
  } else {
    // warp wq: rows 16 wq .. 16 wq + 15, one 128-byte row segment per instruction (the next drain's wg_sync orders the reuse)
    for (int r = 0; r < 16; ++r) {
      const int row = wq * 16 + r, grow = r0 + row;
      if (grow >= p.M) break;
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const int gcol = c0 + 32 * b + lane;
        const float v = lds32(stg + (uint32_t)(b * 8192 + row * 128 + (((lane >> 2) ^ (row & 7)) << 4) + (lane & 3) * 4));
        if (gcol < p.NT) p.vol[(int64_t)grow * p.NT + gcol] = v;
      }
    }
  }
}

// one K step (64 elements): 12 MMAs into d, issued and committed as one group
__device__ __forceinline__ void cg_kstep(float* d, uint32_t sbase, int wg, bool first_of_seg) {
  const uint64_t ahi = make_smem_desc(sbase + wg * (CG_OP_BYTES / 2)), alo = make_smem_desc(sbase + CG_OP_BYTES + wg * (CG_OP_BYTES / 2));
  const uint64_t bhi = make_smem_desc(sbase + 2 * CG_OP_BYTES), blo = make_smem_desc(sbase + 3 * CG_OP_BYTES);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) {   // 16 halves = 32 bytes of every 128-byte row per MMA -> +2 in the (addr >> 4) field; small terms first
    const uint64_t ko = (uint64_t)(2 * k);
    wgmma_ss<CG_BN, true>(d, ahi + ko, blo + ko, (!first_of_seg || k > 0) ? 1u : 0u);   // A_hi * B_lo
    wgmma_ss<CG_BN, true>(d, alo + ko, bhi + ko, 1u);                                     // A_lo * B_hi
    wgmma_ss<CG_BN, true>(d, ahi + ko, bhi + ko, 1u);                                     // A_hi * B_hi
  }
  wgmma_commit();
}

// tile index -> (first source row, first target): groups of CG_GROUP M tiles, M fastest inside a group, so the CTAs running at one time
// share few A and B tiles and the B tiles are re-read from L2 instead of HBM
__device__ __forceinline__ void cg_coords(const CgParams& p, int tile, int& m0, int& n0) {
  const int per = CG_GROUP * p.tiles_n, g = tile / per, r = tile - g * per;
  const int gm = min(CG_GROUP, p.tiles_m - g * CG_GROUP);
  m0 = (g * CG_GROUP + r % gm) * CG_BM; n0 = (r / gm) * CG_BN;
}

struct CgPipe {
  int stage = 0; uint32_t phase = 0;
  int prev = -1;                   // stage read by the most recent commit group, not yet handed back to the producer
};

// wait for the next stage, issue its K step into d, hand the previous step's stage back once its MMAs have retired
__device__ __forceinline__ void cg_step(const CgParams& p, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, CgPipe& s, float* d, int wg, int lane,
                                        bool first_of_seg) {
  mbar_wait(&full_bar[s.stage], s.phase, p.spin_limit);
  cg_kstep(d, smem_u32(smem + s.stage * CG_STAGE_BYTES), wg, first_of_seg);
  if (s.prev >= 0) {   // the previous step's MMAs have retired once at most this step's group is pending
    wgmma_wait<1>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s.prev]);
  }
  s.prev = s.stage;
  if (++s.stage == CG_STAGES) { s.stage = 0; s.phase ^= 1; }
}

// all issued MMAs retired (P and Q hold their final values); the last stage goes back to the producer
__device__ __forceinline__ void cg_retire(uint64_t* empty_bar, CgPipe& s, float* P, float* Q, int lane) {
  wgmma_wait<0>();
  reg_fence<CG_BN / 2>(P); reg_fence<CG_BN / 2>(Q);
  __syncwarp();
  if (lane == 0 && s.prev >= 0) mbar_arrive(&empty_bar[s.prev]);
  s.prev = -1;
}

// One tile: segment 0 (K steps 0, 1) into P, later segments into Q, each folded into P before Q is reused; the result is in P.
// On entry Q holds the previous tile's result (drain_prev): it is drained, one half per K step, while segment 0's MMAs run.
// (Separate loops for segment 0 and the rest: the drain reads Q, which ptxas must see is never the target of an MMA in flight.)
__device__ __forceinline__ void cg_tile(const CgParams& p, const CUtensorMap* tmO, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, CgPipe& s,
                                        float* P, float* Q, bool drain_prev, int pm0, int pn0, uint32_t stg, int wg, int wq, int lane) {
  const int ks_n = p.ksteps;
  cg_step(p, smem, full_bar, empty_bar, s, P, wg, lane, true);
  if (drain_prev) cg_drain_half<0>(p, tmO, Q, pm0, pn0, stg, wg, wq, lane);
  if (ks_n > 1) cg_step(p, smem, full_bar, empty_bar, s, P, wg, lane, false);
  if (drain_prev) cg_drain_half<1>(p, tmO, Q, pm0, pn0, stg, wg, wq, lane);
  for (int ks = CG_SEG; ks < ks_n; ++ks) {
    const bool first = ks % CG_SEG == 0;
    if (first && ks >= 2 * CG_SEG) {   // Q is about to be overwritten: fold the previous segment into P
      cg_retire(empty_bar, s, P, Q, lane);
#pragma unroll
      for (int i = 0; i < CG_BN / 2; ++i) P[i] += Q[i];
    }
    cg_step(p, smem, full_bar, empty_bar, s, Q, wg, lane, first);
  }
  cg_retire(empty_bar, s, P, Q, lane);
  if (ks_n > CG_SEG) {
#pragma unroll
    for (int i = 0; i < CG_BN / 2; ++i) P[i] += Q[i];
  }
}

__global__ void __launch_bounds__(CG_THREADS, 1)
corr_gemm_3xf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO,
                       const __grid_constant__ CgParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stg_base = smem + CG_STAGES * CG_STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stg_base + 2 * CG_STG_WG_BYTES);
  uint64_t* empty_bar = full_bar + CG_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmO)) : "memory");
    for (int s = 0; s < CG_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], CG_CONSUMERS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= CG_CONSUMERS / 32) {
    // ===================================================== TMA producer (one elected thread)
    setmaxnreg_dec<CG_PRODUCER_REGS>();
    if (warp == CG_CONSUMERS / 32 && elect_one()) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        int m0, n0;
        cg_coords(p, tile, m0, n0);
        for (int ks = 0; ks < p.ksteps; ++ks) {
          mbar_wait(&empty_bar[stage], phase ^ 1, p.spin_limit);
          uint8_t* dst = smem + stage * CG_STAGE_BYTES;
          mbar_expect_tx(&full_bar[stage], (uint32_t)CG_STAGE_BYTES);
          tma_load_3d(dst, &tmA, &full_bar[stage], ks * CG_BK, m0, 0);
          tma_load_3d(dst + CG_OP_BYTES, &tmA, &full_bar[stage], ks * CG_BK, m0, 1);
          tma_load_3d(dst + 2 * CG_OP_BYTES, &tmB, &full_bar[stage], ks * CG_BK, n0, 0);
          tma_load_3d(dst + 3 * CG_OP_BYTES, &tmB, &full_bar[stage], ks * CG_BK, n0, 1);
          if (++stage == CG_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================================================== consumer warpgroups
  setmaxnreg_inc<CG_CONSUMER_REGS>();
  const int wg = warp >> 2, wq = warp & 3;
  const uint32_t stg = smem_u32(stg_base + wg * CG_STG_WG_BYTES);
  float b0[CG_BN / 2], b1[CG_BN / 2];
  CgPipe s;
  // tiles alternate between the two accumulator sets: the finished one is drained under the next tile's first MMAs
  int tile = blockIdx.x, m0 = 0, n0 = 0;
  if (tile < p.num_tiles) {
    cg_coords(p, tile, m0, n0);
    cg_tile(p, &tmO, smem, full_bar, empty_bar, s, b0, b1, false, 0, 0, stg, wg, wq, lane);
    for (;;) {
      int pm0 = m0, pn0 = n0;
      tile += gridDim.x;
      if (tile >= p.num_tiles) {
        cg_drain_half<0>(p, &tmO, b0, pm0, pn0, stg, wg, wq, lane); cg_drain_half<1>(p, &tmO, b0, pm0, pn0, stg, wg, wq, lane);
        break;
      }
      cg_coords(p, tile, m0, n0);
      cg_tile(p, &tmO, smem, full_bar, empty_bar, s, b1, b0, true, pm0, pn0, stg, wg, wq, lane);
      pm0 = m0; pn0 = n0;
      tile += gridDim.x;
      if (tile >= p.num_tiles) {
        cg_drain_half<0>(p, &tmO, b1, pm0, pn0, stg, wg, wq, lane); cg_drain_half<1>(p, &tmO, b1, pm0, pn0, stg, wg, wq, lane);
        break;
      }
      cg_coords(p, tile, m0, n0);
      cg_tile(p, &tmO, smem, full_bar, empty_bar, s, b0, b1, true, pm0, pn0, stg, wg, wq, lane);
    }
  }
  if (wq == 0 && lane == 0) bulk_wait0();   // the volume is written before the CTA retires its shared memory
}

}  // namespace tc

void corr_gemm_3xf16(Ctx& cx, const void* a_planes, int64_t a_plane, int M, const void* b_planes, int64_t b_plane, int NT, int K, float scale,
                     float* vol) {
  using namespace tc;
  if (M <= 0 || NT <= 0) return;
  if (K % CG_BK != 0 || K <= 0) throw std::runtime_error("corr_gemm_3xf16: K must be a positive multiple of 64");
  if (!aligned(a_planes, 16) || !aligned(b_planes, 16) || a_plane % 8 || b_plane % 8)
    throw std::runtime_error("corr_gemm_3xf16: half planes must be 16-byte aligned");
  CUtensorMap mA, mB, mO;
  {
    cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)M, 2};
    cuuint64_t str[2] = {(cuuint64_t)K * 2, (cuuint64_t)a_plane * 2};
    cuuint32_t box[3] = {CG_BK, CG_BM, 1};
    encode(&mA, a_planes, 3, dims, str, box, true);
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)NT, 2};
    cuuint64_t str[2] = {(cuuint64_t)K * 2, (cuuint64_t)b_plane * 2};
    cuuint32_t box[3] = {CG_BK, CG_BN, 1};
    encode(&mB, b_planes, 3, dims, str, box, true);
  }
  CgParams p;
  p.M = M; p.NT = NT; p.ksteps = K / CG_BK; p.tiles_m = (M + CG_BM - 1) / CG_BM; p.tiles_n = (NT + CG_BN - 1) / CG_BN; p.num_tiles = p.tiles_m * p.tiles_n;
  p.tma_store = (NT % 4 == 0 && aligned(vol, 16)) ? 1 : 0;
  p.scale = scale; p.vol = vol; p.spin_limit = tc_spin_limit();
  if (p.tma_store) {
    cuuint64_t dims[2] = {(cuuint64_t)NT, (cuuint64_t)M};
    cuuint64_t str[1] = {(cuuint64_t)NT * 4};
    cuuint32_t box[2] = {32, 64};
    encode(&mO, vol, 2, dims, str, box);
  } else {
    mO = mA;   // unused
  }
  const int grid = p.num_tiles < cx.sm_count ? p.num_tiles : cx.sm_count;
  cx.launches++;
  if (cx.prof) cx.prof->begin(cx.stream, "corr_gemm_tc_3xf16", 2.0 * (double)M * NT * K);
  static volatile unsigned char attr[64];
  gv_set_max_smem(tc::corr_gemm_3xf16_kernel, CG_SMEM, attr);
  tc::corr_gemm_3xf16_kernel<<<grid, CG_THREADS, CG_SMEM, cx.stream>>>(mA, mB, mO, p);
  gv_check_launch("corr_gemm_3xf16");
  if (cx.prof) cx.prof->end(cx.stream);
}

}  // namespace gv
#endif  // GV_HOSTSIM
