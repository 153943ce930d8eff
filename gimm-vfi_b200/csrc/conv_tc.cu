// Tensor-core implicit-GEMM convolution for sm_90a: TMA tile loads with halo
// coordinates -> 128B-swizzled shared memory -> wgmma (tf32 / f16 operands, fp32
// accumulators in registers) -> fused, coalesced epilogue.
//
//   GEMM view   M = 128 output pixels (an 8 x 16 spatial tile of one image)
//               N = 32, 64 or 128 output channels per tile (cout tiled if larger)
//               K = taps x cin, walked as (tap, 32-channel block): each K step is ONE
//                   TMA box {32 ch, 16 x, 8 y, 1 n} of the NHWC activation at the
//                   tap-shifted coordinate (out-of-bounds -> zero fill = zero padding,
//                   no im2col, no halo staging code) plus one {32 k, N} weight box.
//   roles       warpgroups 0 / 1: MMAs (M = 64 rows each) and the epilogue of their rows | warpgroup 2: TMA producer
//               (one elected thread issues the loads; the warpgroup gives its registers to the consumers with setmaxnreg)
//   pipelines   smem full/empty ring, persistent over tiles: the producer runs ahead into the next tile while the
//               warpgroups run the epilogue of the current one.
//   stride 2    TMA element strides {1, 2, 2, 1}: the box spans 32 x 16 pixels, every second one is delivered.
//
// Three operand formats:
//   TF32         (SPLIT=false) the tensor core ignores the low 13 mantissa bits of A; weights are rounded RN at
//                pack time; outputs are stored TF32-rounded so the next layer's truncation is exact.  Post-RAFT layers.
//   FP16 storage (SPLIT=false, F16=true) activations and weights in IEEE half, f16 MMAs with K = 64 per
//                128-byte smem row, fp32 accumulation; half outputs / residuals as flagged per tensor (TV::f16).  The final
//                decoder's 256-channel residual trunk in precision mode 3.
//   3xTF32       (SPLIT=true) D += Ahi*Blo + Alo*Bhi + Ahi*Bhi with Ahi = rn_tf32(a), Alo = rn_tf32(a - Ahi).  Each warpgroup
//                reads its fp32 A rows from shared memory into registers, splits them there and feeds the MMAs register
//                A fragments; Bhi / Blo are pre-split at pack time.  The K loop is cut into segments of Params::seg K steps
//                whose accumulators are summed into separate fp32 registers: short tensor-core accumulation chains and a true
//                fp32 sum across segments keep the result at fp32-class accuracy.  Used for the RAFT recurrence, which
//                amplifies operand rounding.  With F16=true ("3xF16") the three MMAs run on f16 hi / lo operand pairs
//                (K step = 64 elements = two 32-channel fp32 A boxes; weights pre-split and pre-scaled at pack time).
#include "common.h"

#ifndef GV_HOSTSIM
#include <cuda.h>
#include <cuda_fp16.h>

namespace gv {

namespace tc {

constexpr int TILE_H = 8, TILE_W = 16, BM = 128, BK = 32, MAX_STAGES = 8;
constexpr int A_BYTES = BM * BK * 4;                // 16 KB
constexpr int STG_PITCH = 32;                       // floats per staged row; the 16-byte chunk c of row r sits at chunk c ^ (r & 7): conflict-free
                                                    // 128-bit row writes (phase 1) and row-segment reads (phase 2) without padding
constexpr int EPI_WG_BYTES = 64 * 64 * 4;           // per warpgroup: a 64-row x 64-column accumulator slice, then the four warps' staging areas
constexpr int BAR_BYTES = 512;
// warpgroups 0 / 1 consume, warpgroup 2 produces.  A whole producer warpgroup (not one warp) so that it can hand its registers to
// the consumers with setmaxnreg.  The launch budget is 168 per thread (65536 / 384, in steps of 8): 128 x (2 x 232 + 40) = 384 x 168.
// 232 holds acc + racc of the split kernel at N = 128 without spills.
constexpr int CONSUMER_THREADS = 256, TC_THREADS = CONSUMER_THREADS + 128;
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;

struct Params {
  int taps, kw, ph, pw;
  int stride;                      // 1 or 2: output pixel (y, x) reads input (y * stride + ky - ph, ...) through TMA element strides
  int kblocks, c0_blocks;          // K blocks in total / from segment 0
  int tiles_x, tiles_y, n_img, tiles_n;
  int H, W;
  int stages;                      // smem ring depth (<= MAX_STAGES), sized on the host
  int cout;
  int round_out;                   // store TF32-rounded (RN) values
  int spin_limit;                  // mbarrier try_wait time limit (x 10 ms) before trapping (0 = wait forever)
  int bk;                          // K elements per 128-byte smem row: 32 (tf32) or 64 (f16)
  int seg;                         // SPLIT: K steps accumulated by the tensor core before the fp32 register sum
  float out_scale;                 // accumulator scale applied before the bias (all-pairs correlation: 1/sqrt(C))
  const float* bias;               // padded past tiles_n * N
  int act1; const float* slope1;
  int act2; const float* slope2;
  TV res, mul, gru_z, gru_h, out;
  TV out2; int split_c;            // channels >= split_c go to out2 (and only they see `mul`): merged z | r gate convolution
};

#include "tc_ptx.cuh"

#include "tc_epilogue.cuh"

// One 32-row x 32-column chunk of the output tile: v[j] = accumulator of (this thread's pixel row, column c0 + j).
// stg_s = shared-window address of this warp's 32 x STG_PITCH staging area; cbase = first output channel of the chunk.
__device__ __forceinline__ void epi_chunk(const Params& p, const uint32_t* v, uint32_t stg_s, int cbase, int quarter, int lane, int tx, int ty,
                                          int n) {
  const int q8 = lane & 7, rsub = lane >> 3;
  // phase 1 (thread = pixel row): bias + act1, stage to smem.  bias is padded to tiles_n*BN (+slack) on the host.
  {
    float o[32];
    const float4* b4p = reinterpret_cast<const float4*>(p.bias + cbase);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 b4 = __ldg(b4p + j);
      o[4 * j] = fmaf(__uint_as_float(v[4 * j]), p.out_scale, b4.x); o[4 * j + 1] = fmaf(__uint_as_float(v[4 * j + 1]), p.out_scale, b4.y);
      o[4 * j + 2] = fmaf(__uint_as_float(v[4 * j + 2]), p.out_scale, b4.z); o[4 * j + 3] = fmaf(__uint_as_float(v[4 * j + 3]), p.out_scale, b4.w);
    }
    act_n<32>(o, p.act1, p.slope1, cbase, p.cout);
    const uint32_t srow = stg_s + (uint32_t)(lane * STG_PITCH * 4);
#pragma unroll
    for (int j = 0; j < 8; ++j) sts128(srow + (uint32_t)((j ^ (lane & 7)) << 4), o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
  }
  __syncwarp();
  // phase 2 (8 lanes = one 128-byte row, 4 rows per instruction): + residual, act2, gate multiply,
  // ConvGRU blend, optional TF32 rounding, coalesced store.  Row `it` of this lane is tile pixel
  // (yy, xx) = (quarter * 2 + it / 4, (it % 4) * 4 + rsub).
  const int c = cbase + q8 * 4;
  if (c < p.cout && n < p.n_img) {
    const bool full4 = c + 3 < p.cout;
    const int y0 = ty * TILE_H + quarter * 2, x0 = tx * TILE_W + rsub;
    const bool interior = y0 + 1 < p.H && tx * TILE_W + TILE_W <= p.W;
    // staged row it * 4 + rsub, logical chunk q8: its swizzle phase (row & 7) is rsub for even `it`, rsub + 4 for odd
    const uint32_t sb_even = stg_s + (uint32_t)(rsub * STG_PITCH * 4 + ((q8 ^ rsub) << 4));
    const uint32_t sb_odd = stg_s + (uint32_t)(rsub * STG_PITCH * 4 + ((q8 ^ (rsub + 4)) << 4));
    const bool second = p.split_c > 0 && cbase >= p.split_c;          // merged z | r convolution: this chunk belongs to out2
    const TV& O = second ? p.out2 : p.out;
    const int c_loc = c - (second ? p.split_c : 0);
    const bool use_mul = p.mul.p && (p.split_c == 0 || second);
    const bool lean = !p.res.p && !use_mul && !p.gru_z.p;
    const int64_t opix0 = (int64_t)y0 * p.W + x0;
    const int64_t obase = (int64_t)n * O.sn + opix0 * O.ld + c_loc;    // element offset of (row 0 of this lane, its first channel)
    const int64_t o_row = (int64_t)p.W * O.ld, o_x = (int64_t)4 * O.ld;
    const uintptr_t oaddr = reinterpret_cast<uintptr_t>(O.p) + (uintptr_t)obase * (O.f16 ? 2 : 4);
    const bool ovec = full4 && ((oaddr & (O.f16 ? 7 : 15)) == 0) && (O.ld % 4 == 0);
    if (lean) {
      float o[32];
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const float4 sv = lds128(((it & 1) ? sb_odd : sb_even) + (uint32_t)(it * 4 * STG_PITCH * 4));
        o[4 * it] = sv.x; o[4 * it + 1] = sv.y; o[4 * it + 2] = sv.z; o[4 * it + 3] = sv.w;
      }
      if (p.act2 != ACT_NONE) act_rows<8>(o, p.act2, p.slope2, c, p.cout);
      if (p.round_out) {
        // store TF32-representable values (round-to-nearest-even): the next TF32 layer then truncates
        // nothing, i.e. its operands are RN- instead of toward-zero-rounded (unbiased)
#pragma unroll
        for (int u = 0; u < 32; ++u) o[u] = rn_tf32(o[u]);
      }
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int yy = it >> 2, xx = (it & 3) * 4;
        if (!interior && (y0 + yy >= p.H || x0 + xx >= p.W)) continue;
        store4(O, obase + yy * o_row + (it & 3) * o_x, o + 4 * it, c, p.cout, ovec);
      }
    } else {
      // side tensors (residual / gate / GRU state): two groups of 4 rows, every global load of a group issued before its
      // first use (one warp's epilogue is latency bound: the 2-row loop this replaces took 2x the main loop at N = 256)
      const int64_t rbase = p.res.p ? p.res.off(n, y0, x0) + c : 0, mbase = use_mul ? p.mul.off(n, y0, x0) + c_loc : 0;
      const int64_t zbase = p.gru_z.p ? p.gru_z.off(n, y0, x0) + c : 0, hbase = p.gru_z.p ? p.gru_h.off(n, y0, x0) + c : 0;
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        float o[16];
        bool ok[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          ok[j] = interior || (y0 + g < p.H && x0 + j * 4 < p.W);
          const float4 sv = lds128(((j & 1) ? sb_odd : sb_even) + (uint32_t)((g * 4 + j) * 4 * STG_PITCH * 4));
          o[4 * j] = sv.x; o[4 * j + 1] = sv.y; o[4 * j + 2] = sv.z; o[4 * j + 3] = sv.w;
        }
        if (p.res.p) {
          float t[16];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (ok[j]) load4_any(p.res, rbase + (int64_t)g * p.res.w * p.res.ld + (int64_t)j * 4 * p.res.ld, c, p.cout, t + 4 * j);
            else { t[4 * j] = t[4 * j + 1] = t[4 * j + 2] = t[4 * j + 3] = 0.f; }
          }
#pragma unroll
          for (int u = 0; u < 16; ++u) o[u] += t[u];
        }
        if (p.act2 != ACT_NONE) act_rows<4>(o, p.act2, p.slope2, c, p.cout);
        if (use_mul) {
          float t[16];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (ok[j]) load4(p.mul.p + mbase + (int64_t)g * p.mul.w * p.mul.ld + (int64_t)j * 4 * p.mul.ld, c, p.cout, t + 4 * j);
            else { t[4 * j] = t[4 * j + 1] = t[4 * j + 2] = t[4 * j + 3] = 0.f; }
          }
#pragma unroll
          for (int u = 0; u < 16; ++u) o[u] *= t[u];
        }
        if (p.gru_z.p) {  // h = (1 - z) * h + z * q   (raft/update.py:58,66)
          float z[16], hh[16];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (ok[j]) {
              load4(p.gru_z.p + zbase + (int64_t)g * p.gru_z.w * p.gru_z.ld + (int64_t)j * 4 * p.gru_z.ld, c, p.cout, z + 4 * j);
              load4(p.gru_h.p + hbase + (int64_t)g * p.gru_h.w * p.gru_h.ld + (int64_t)j * 4 * p.gru_h.ld, c, p.cout, hh + 4 * j);
            } else {
#pragma unroll
              for (int u = 0; u < 4; ++u) { z[4 * j + u] = 0.f; hh[4 * j + u] = 0.f; }
            }
          }
#pragma unroll
          for (int u = 0; u < 16; ++u) o[u] = (1.f - z[u]) * hh[u] + z[u] * o[u];
        }
        if (p.round_out) {
#pragma unroll
          for (int u = 0; u < 16; ++u) o[u] = rn_tf32(o[u]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (ok[j]) store4(O, obase + g * o_row + j * o_x, o + 4 * j, c, p.cout, ovec);
      }
    }
  }
  __syncwarp();
}

// rn split of two fp32 values into f16 hi / lo pairs (a = hi + lo to 22 significand bits)
__device__ __forceinline__ void split_h2(float2 v, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(v.x, v.y);
  const float2 f = __half22float2(h);
  const __half2 l = __floats2half2_rn(v.x - f.x, v.y - f.y);
  hi = *reinterpret_cast<const uint32_t*>(&h); lo = *reinterpret_cast<const uint32_t*>(&l);
}

// N = output channels per tile (32, 64, 128).  Two consumer warpgroups own pixel rows [0, 64) / [64, 128) of the tile: they issue
// the MMAs of their rows (A descriptor offset by 64 rows = 8 KB; the same weight tile) and run the epilogue of their rows from the
// register accumulators.  The 32-row x 32-column chunks the epilogue works on are gathered through shared memory: the warpgroup
// writes a 64 x 64 slice of its accumulators, each warp reads back one 32-row x 32-column chunk as "thread = pixel row".
// F16: f16 MMAs (half storage, or the 3xF16 split) instead of TF32 - a template parameter so that the MMA chain of a K step is
// straight-line code whose accumulators stay in fixed registers (a runtime choice makes the compiler serialise the asynchronous MMAs)
template <bool SPLIT, int N, bool F16>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv2d_tc_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ Params p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: per stage [A 16 KB | (A, channels 32-63: 3xF16) | B N*128 B | (B_lo)], then the two warpgroups' epilogue areas, then barriers
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int b_bytes = N * BK * 4;
  constexpr bool SF16 = SPLIT && F16;
  const int a_all = SF16 ? 2 * A_BYTES : A_BYTES;
  const int stage_bytes = a_all + (SPLIT ? 2 * b_bytes : b_bytes);
  const int STAGES = p.stages;
  uint8_t* epi_base = smem + STAGES * stage_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(epi_base + 2 * EPI_WG_BYTES);
  uint64_t* full_bar = bars;                          // [MAX_STAGES]  TMA bytes landed
  uint64_t* empty_bar = bars + MAX_STAGES;            // [MAX_STAGES]  the 8 consumer warps' MMAs reading the stage retired

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // tile index -> (pixel tile, N tile): consecutive indices share the pixel tile
  const int num_tiles = p.n_img * p.tiles_y * p.tiles_x * p.tiles_n;
  const int ksteps = p.taps * p.kblocks;
  const int SPIN = p.spin_limit;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA0)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA1)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB)) : "memory");
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], CONSUMER_THREADS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= CONSUMER_THREADS / 32) {
    // ===================================================== TMA producer (one elected thread of the producer warpgroup)
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == CONSUMER_THREADS / 32 && elect_one()) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int nt = tile % p.tiles_n; int r = tile / p.tiles_n;
        const int tx = r % p.tiles_x; r /= p.tiles_x; const int ty = r % p.tiles_y; const int n = r / p.tiles_y;
        for (int tap = 0; tap < p.taps; ++tap) {
          const int ky = tap / p.kw, kx = tap % p.kw;
          const int x0 = tx * TILE_W * p.stride + kx - p.pw, y0 = ty * TILE_H * p.stride + ky - p.ph;
          for (int kb = 0; kb < p.kblocks; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1, SPIN);
            uint8_t* a_dst = smem + stage * stage_bytes;
            uint8_t* b_dst = a_dst + a_all;
            mbar_expect_tx(&full_bar[stage], (uint32_t)(a_all + (SPLIT ? 2 * b_bytes : b_bytes)));
            const CUtensorMap* ta = kb < p.c0_blocks ? &tmA0 : &tmA1;
            const int ch = (kb < p.c0_blocks ? kb : kb - p.c0_blocks) * p.bk;
            tma_load_4d(a_dst, ta, &full_bar[stage], ch, x0, y0, n);
            if (SF16) tma_load_4d(a_dst + A_BYTES, ta, &full_bar[stage], ch + 32, x0, y0, n);   // channels [32, 64) of the K block
            tma_load_3d(b_dst, &tmB, &full_bar[stage], kb * p.bk, nt * N, tap);
            if (SPLIT) tma_load_3d(b_dst + b_bytes, &tmB, &full_bar[stage], kb * p.bk, nt * N, tap + p.taps);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ===================================================== consumer warpgroups
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = warp >> 2, wq = warp & 3, gid = lane >> 2, tig = lane & 3;
  const uint32_t ebuf_s = smem_u32(epi_base + wg * EPI_WG_BYTES);
  float acc[N / 2];
  float racc[SPLIT ? N / 2 : 1];
  int stage = 0; uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int nt = tile % p.tiles_n; int r = tile / p.tiles_n;
    const int tx = r % p.tiles_x; r /= p.tiles_x; const int ty = r % p.tiles_y; const int n = r / p.tiles_y;
    // (the first MMA of a tile overwrites acc; defining it here ends the previous tile's values, so that they need no registers
    // through the epilogue)
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    if (SPLIT) {
#pragma unroll
      for (int i = 0; i < (SPLIT ? N / 2 : 1); ++i) racc[i] = 0.f;
    }
    int prev = -1;
    for (int ks = 0; ks < ksteps; ++ks) {
      const bool seg_start = SPLIT ? (ks % p.seg == 0) : (ks == 0);
      const bool seg_end = SPLIT ? (ks % p.seg == p.seg - 1 || ks == ksteps - 1) : (ks == ksteps - 1);
      mbar_wait(&full_bar[stage], phase, SPIN);
      uint8_t* sbase = smem + stage * stage_bytes;
      const uint32_t a_addr = smem_u32(sbase);
      const uint64_t bdesc = make_smem_desc(a_addr + a_all);
      if (!SPLIT) {
        const uint64_t adesc = make_smem_desc(a_addr + wg * (A_BYTES / 2));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {   // 32 bytes of every 128-byte row per MMA (8 tf32 / 16 half) -> +2 in the (addr >> 4) field
          const uint32_t sc = (ks > 0 || k > 0) ? 1u : 0u;
          wgmma_ss<N, F16>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), sc);
        }
        wgmma_commit();
        if (prev >= 0) {   // the previous stage's MMAs have retired once at most this stage's group is pending
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
      } else {
        // this thread's A fragment rows R0 = 64 wg + 16 wq + gid and R0 + 8 (both with swizzle phase gid)
        const uint8_t* r0 = sbase + (wg * 64 + wq * 16 + gid) * 128;
        const uint8_t* r1 = r0 + 8 * 128;
        const uint64_t blo = make_smem_desc(a_addr + a_all + b_bytes);
        uint32_t hi[4][4], lo[4][4];
        if (SF16) {
#pragma unroll
          for (int k = 0; k < 4; ++k) {   // K elements [16 k, 16 k + 16) of the 64-element step: fp32 sub-tile k / 2, channels 16 (k & 1) + ...
            const int sub = (k >> 1) * A_BYTES, c0 = 16 * (k & 1) + 2 * tig, c1 = c0 + 8;
            const int o0 = sub + ((((c0 >> 2) ^ gid)) << 4) + (c0 & 3) * 4, o1 = sub + ((((c1 >> 2) ^ gid)) << 4) + (c1 & 3) * 4;
            split_h2(*reinterpret_cast<const float2*>(r0 + o0), hi[k][0], lo[k][0]);
            split_h2(*reinterpret_cast<const float2*>(r1 + o0), hi[k][1], lo[k][1]);
            split_h2(*reinterpret_cast<const float2*>(r0 + o1), hi[k][2], lo[k][2]);
            split_h2(*reinterpret_cast<const float2*>(r1 + o1), hi[k][3], lo[k][3]);
          }
        } else {
#pragma unroll
          for (int k = 0; k < 4; ++k) {   // K elements 8 k + tig and 8 k + tig + 4 = element tig of 16-byte chunks 2 k, 2 k + 1
            const int o0 = (((2 * k) ^ gid) << 4) + tig * 4, o1 = (((2 * k + 1) ^ gid) << 4) + tig * 4;
            const float v[4] = {*reinterpret_cast<const float*>(r0 + o0), *reinterpret_cast<const float*>(r1 + o0),
                                *reinterpret_cast<const float*>(r0 + o1), *reinterpret_cast<const float*>(r1 + o1)};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const float h = rn_tf32(v[u]);
              hi[k][u] = __float_as_uint(h); lo[k][u] = __float_as_uint(rn_tf32(v[u] - h));
            }
          }
        }
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {   // small terms first
          const uint64_t ko = (uint64_t)(2 * k);
          if (SF16) {
            wgmma_rs<N, true>(acc, hi[k], blo + ko, (!seg_start || k > 0) ? 1u : 0u);   // A_hi * B_lo
            wgmma_rs<N, true>(acc, lo[k], bdesc + ko, 1u);                               // A_lo * B_hi
            wgmma_rs<N, true>(acc, hi[k], bdesc + ko, 1u);                               // A_hi * B_hi
          } else {
            wgmma_rs<N, false>(acc, hi[k], blo + ko, (!seg_start || k > 0) ? 1u : 0u);
            wgmma_rs<N, false>(acc, lo[k], bdesc + ko, 1u);
            wgmma_rs<N, false>(acc, hi[k], bdesc + ko, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence<N / 2>(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (seg_end) {
#pragma unroll
          for (int i = 0; i < (SPLIT ? N / 2 : 1); ++i) racc[i] += acc[i];
        }
      }
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    if (!SPLIT) {
      wgmma_wait<0>();
      reg_fence<N / 2>(acc);
      __syncwarp();
      if (lane == 0 && prev >= 0) mbar_arrive(&empty_bar[prev]);
    }
    // ---- epilogue, 64 columns at a time
    const float* res = SPLIT ? racc : acc;
#pragma unroll
    for (int cp = 0; cp < (N + 63) / 64; ++cp) {
      wg_sync(1 + wg);   // the previous pass's staging reads are done
#pragma unroll
      for (int j = 8 * cp; j < 8 * cp + 8 && j < N / 8; ++j) {
        const int col = 8 * (j - 8 * cp) + 2 * tig;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = wq * 16 + gid + 8 * h;
          // (32-bit shared addresses: 64-bit generic ones stay live across the column passes and cost registers)
          sts64(ebuf_s + (uint32_t)(row * 256 + ((((col >> 2) ^ (row & 7))) << 4) + (col & 3) * 4), res[4 * j + 2 * h], res[4 * j + 2 * h + 1]);
        }
      }
      wg_sync(1 + wg);
      const int chunk = 2 * cp + (wq >> 1), row = (wq & 1) * 32 + lane;
      const int cbase = nt * N + chunk * 32;
      const bool active = chunk * 32 < N && cbase < p.cout;   // warp-uniform
      uint32_t v[32];
      if (active) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 t = lds128(ebuf_s + (uint32_t)(row * 256 + (((8 * (wq >> 1) + i) ^ (row & 7)) << 4)));
          v[4 * i] = __float_as_uint(t.x); v[4 * i + 1] = __float_as_uint(t.y); v[4 * i + 2] = __float_as_uint(t.z); v[4 * i + 3] = __float_as_uint(t.w);
        }
      }
      wg_sync(1 + wg);   // every warp holds its chunk: the slice becomes the four warps' staging areas
      if (active) epi_chunk(p, v, ebuf_s + (uint32_t)(wq * 32 * STG_PITCH * 4), cbase, wg * 2 + (wq & 1), lane, tx, ty, n);
    }
  }
}

// ---------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || !p) throw std::runtime_error("conv_tc: cuTensorMapEncodeTiled is unavailable");
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

void encode(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box,
            bool f16, int pixel_stride, CUtensorMapSwizzle swizzle) {
  cuuint32_t estr[5] = {1, (cuuint32_t)pixel_stride, (cuuint32_t)pixel_stride, 1, 1};   // (activation maps: dims 1, 2 = x, y)
  CUresult r = encode_fn()(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("conv_tc: cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
}

// stride 2: the box spans 2x the tile in x and y and TMA keeps every second element (elementStrides), so shared memory
// receives the same dense 16 x 8 pixel tile as at stride 1
static void encode_act(CUtensorMap* m, const TV& t, int stride = 1) {
  cuuint64_t dims[4] = {(cuuint64_t)t.c, (cuuint64_t)t.w, (cuuint64_t)t.h, (cuuint64_t)t.n};
  const cuuint64_t es = t.f16 ? 2 : 4;
  cuuint64_t str[3] = {(cuuint64_t)t.ld * es, (cuuint64_t)t.w * t.ld * es, (cuuint64_t)t.sn * es};
  cuuint32_t box[4] = {(cuuint32_t)(t.f16 ? 2 * BK : BK), (cuuint32_t)(TILE_W * stride), (cuuint32_t)(TILE_H * stride), 1};   // 128-byte rows either way
  encode(m, t.p, 4, dims, str, box, t.f16 != 0, stride);
}

// N tile of a layer with `cout` output channels: the narrowest of 32 / 64 / 128 that covers an even share of cout
static int pick_n(int cout) {
  const int c32 = (cout + 31) & ~31, tiles = (c32 + 127) / 128, per = (c32 / 32 + tiles - 1) / tiles * 32;
  return per <= 32 ? 32 : (per <= 64 ? 64 : 128);
}

}  // namespace tc

template <bool SPLIT, int N, bool F16>
static void launch_tc_n(int grid, int smem, gvStream_t stream, const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const tc::Params& p) {
  static volatile unsigned char attr_set[64];   // per (instantiation, device)
  gv_set_max_smem(tc::conv2d_tc_kernel<SPLIT, N, F16>, 227 * 1024, attr_set);
  tc::conv2d_tc_kernel<SPLIT, N, F16><<<grid, tc::TC_THREADS, smem, stream>>>(a0, a1, b, p);
}
template <bool SPLIT, bool F16>
static void launch_tc_f(int N, int grid, int smem, gvStream_t stream, const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b,
                        const tc::Params& p) {
  if (N == 32) launch_tc_n<SPLIT, 32, F16>(grid, smem, stream, a0, a1, b, p);
  else if (N == 64) launch_tc_n<SPLIT, 64, F16>(grid, smem, stream, a0, a1, b, p);
  else launch_tc_n<SPLIT, 128, F16>(grid, smem, stream, a0, a1, b, p);
}
// f16: half operands (plain kernel) or the 3xF16 form (split kernel)
static void launch_tc(bool split, bool f16, int N, int grid, int smem, gvStream_t stream, const CUtensorMap& a0, const CUtensorMap& a1,
                      const CUtensorMap& b, const tc::Params& p) {
  if (split) { if (f16) launch_tc_f<true, true>(N, grid, smem, stream, a0, a1, b, p); else launch_tc_f<true, false>(N, grid, smem, stream, a0, a1, b, p); }
  else { if (f16) launch_tc_f<false, true>(N, grid, smem, stream, a0, a1, b, p); else launch_tc_f<false, false>(N, grid, smem, stream, a0, a1, b, p); }
}

// K steps (of p.bk elements) per tensor-core accumulation segment: longer segments break the fp32-class parity bar (DESIGN.md §4)
constexpr int TC_SEG = 2;

int tc_spin_limit() {
  static const int spin = [] { const char* s = getenv("GIMMVFI_TC_SPIN_LIMIT"); return s ? atoi(s) : 400; }();
  return spin;
}
// pipeline depth from the shared-memory budget; returns the dynamic shared-memory size
static int size_stages(tc::Params& p, int stage_bytes) {
  using namespace tc;
  p.stages = (227 * 1024 - 1024 - 2 * EPI_WG_BYTES - BAR_BYTES) / stage_bytes;
  if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
  if (p.stages < 2) throw std::runtime_error("conv_tc: not enough shared memory for 2 pipeline stages");
  return p.stages * stage_bytes + 2 * EPI_WG_BYTES + BAR_BYTES + 1024;
}

void conv2d_tc(Ctx& cx, const TV& in0, const TV& in1, const ConvW& w, const ConvGeom& g, const ConvEpi& e, const TV& out, bool split) {
  using namespace tc;
  CUtensorMap mA0, mA1, mB;
  encode_act(&mA0, in0, g.stride);
  if (in1.p) encode_act(&mA1, in1, g.stride); else mA1 = mA0;
  // any N tiling of the packed weights works: weight rows beyond cout_pad are TMA zero fill, the bias is padded past them
  const int N = pick_n(w.cout), tiles_n = (w.cout + N - 1) / N;
  const int taps = w.kh * w.kw;
  const bool f16 = in0.f16 != 0;
  // 3xF16: the split kernel on f16 hi / lo operand pairs (two 32-channel activation boxes per 64-element K step);
  // needs pre-split weights and a first segment of whole K blocks
  const bool sf16 = split && w.w_tc_s != nullptr && (!in1.p || in0.c % 64 == 0);
  const int bk = (f16 || sf16) ? 2 * BK : BK, cin_pad = f16 ? w.cin_pad_h : (sf16 ? w.cin_pad_s : w.cin_pad);
  if (sf16) {
    cuuint64_t dims[3] = {(cuuint64_t)cin_pad, (cuuint64_t)w.cout_pad, (cuuint64_t)(taps * 2)};
    cuuint64_t str[2] = {(cuuint64_t)cin_pad * 2, (cuuint64_t)cin_pad * w.cout_pad * 2};
    cuuint32_t box[3] = {(cuuint32_t)bk, (cuuint32_t)N, 1};
    encode(&mB, w.w_tc_s, 3, dims, str, box, true);
  } else if (f16) {
    cuuint64_t dims[3] = {(cuuint64_t)cin_pad, (cuuint64_t)w.cout_pad, (cuuint64_t)taps};
    cuuint64_t str[2] = {(cuuint64_t)cin_pad * 2, (cuuint64_t)cin_pad * w.cout_pad * 2};
    cuuint32_t box[3] = {(cuuint32_t)bk, (cuuint32_t)N, 1};
    encode(&mB, w.w_tc_h, 3, dims, str, box, true);
  } else {
    cuuint64_t dims[3] = {(cuuint64_t)w.cin_pad, (cuuint64_t)w.cout_pad, (cuuint64_t)(taps * (w.has_lo ? 2 : 1))};
    cuuint64_t str[2] = {(cuuint64_t)w.cin_pad * 4, (cuuint64_t)w.cin_pad * w.cout_pad * 4};
    cuuint32_t box[3] = {BK, (cuuint32_t)N, 1};
    encode(&mB, w.w_tc, 3, dims, str, box);
  }
  Params p = Params();
  p.taps = taps; p.kw = w.kw; p.ph = g.ph; p.pw = g.pw; p.stride = g.stride;
  p.bk = bk;
  p.c0_blocks = in1.p ? in0.c / bk : (in0.c + bk - 1) / bk;
  p.kblocks = cin_pad / bk;
  p.tiles_x = (out.w + TILE_W - 1) / TILE_W; p.tiles_y = (out.h + TILE_H - 1) / TILE_H; p.n_img = out.n; p.tiles_n = tiles_n;
  p.H = out.h; p.W = out.w; p.cout = w.cout;
  p.round_out = (split || out.f16) ? 0 : 1;   // (a half store already rounds to 10 mantissa bits)
  p.out_scale = sf16 ? 1.f / w.w_scale : 1.f;
  p.seg = TC_SEG;
  p.spin_limit = tc_spin_limit();
  p.bias = w.b; p.act1 = e.act1; p.slope1 = e.slope1; p.act2 = e.act2; p.slope2 = e.slope2;
  p.res = e.res; p.mul = e.mul; p.gru_z = e.gru_z; p.gru_h = e.gru_h; p.out = out; p.out2 = e.out2; p.split_c = e.split_c;
  const int stage_bytes = (sf16 ? 2 : 1) * A_BYTES + (split ? 2 : 1) * N * BK * 4;
  const int smem = size_stages(p, stage_bytes);
  const int num_tiles = out.n * p.tiles_y * p.tiles_x * tiles_n;
  const int grid = num_tiles < cx.sm_count ? num_tiles : cx.sm_count;
  cx.launches++;
  if (cx.prof) {
    char nm[128];
    snprintf(nm, sizeof nm, "conv2d_tc_%s k%dx%d c%d>%d @%dx%dx%d", split ? (sf16 ? "3xf16" : "3xtf32") : (f16 ? "f16" : "tf32"), w.kh, w.kw, w.cin, w.cout, out.n, out.h, out.w);
    cx.prof->begin(cx.stream, prof_intern(nm), 2.0 * (double)out.n * out.h * out.w * w.cout * (double)w.cin * w.kh * w.kw);
  }
  launch_tc(split, split ? sf16 : f16, N, grid, smem, cx.stream, mA0, mA1, mB, p);
  gv_check_launch("conv2d_tc");
  if (cx.prof) cx.prof->end(cx.stream);
}


// All-pairs correlation vol[i][j] = scale * <fa[i,:], fb[j,:]> (raft/corr.py:167-175) as a 3xTF32 GEMM on the
// same kernel: A = fa pixels (M), "weights" = the other frame's features, K-major as they lie in NHWC memory.
// fb_planes = [2][N][C]: plane 0 = rn_tf32(x), plane 1 = rn_tf32(x - plane 0)  (split_planes in corr.cu).
void corr_volume_tc(Ctx& cx, const TV& fa, const float* fb_planes, const float* zero_bias, float* vol, float scale, bool split, int n_targets) {
  using namespace tc;
  if (fa.n != 1) throw std::runtime_error("corr_volume_tc: one sample per launch");
  // M = the source pixels of fa; N = n_targets rows of fb (0: as many as sources).  Pooled pyramid levels are GEMMs against the
  // avg-pooled target features (pooling and the dot product commute), so the level-0 volume is never re-read.
  const int Ms = fa.h * fa.w, NT = n_targets > 0 ? n_targets : Ms, C = fa.c;
  CUtensorMap mA, mB;
  encode_act(&mA, fa);
  // split: fb_planes = [2][N][C] (rn / residual planes).  plain TF32: fb_planes = the raw K-major features [N][C] of the
  // other frame (the tensor core truncates them).
  constexpr int BN = 128;
  const int tiles_n = (NT + BN - 1) / BN;
  const bool sf16 = split && corr_volume_tc_wants_f16_planes() && C % 64 == 0;
  if (sf16) {   // half planes, 64-element K blocks (128-byte rows)
    cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)NT, 2};
    cuuint64_t str[2] = {(cuuint64_t)C * 2, (cuuint64_t)NT * C * 2};
    cuuint32_t box[3] = {2 * BK, (cuuint32_t)BN, 1};
    encode(&mB, fb_planes, 3, dims, str, box, true);
  } else {
    cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)NT, (cuuint64_t)(split ? 2 : 1)};
    cuuint64_t str[2] = {(cuuint64_t)C * 4, (cuuint64_t)NT * C * 4};
    cuuint32_t box[3] = {BK, (cuuint32_t)BN, 1};
    encode(&mB, fb_planes, 3, dims, str, box);
  }
  Params p = Params();
  p.taps = 1; p.kw = 1; p.ph = 0; p.pw = 0; p.stride = 1;
  p.kblocks = sf16 ? C / 64 : C / 32; p.c0_blocks = p.kblocks; p.bk = sf16 ? 2 * BK : BK;
  p.tiles_x = (fa.w + TILE_W - 1) / TILE_W; p.tiles_y = (fa.h + TILE_H - 1) / TILE_H; p.n_img = 1; p.tiles_n = tiles_n;
  p.H = fa.h; p.W = fa.w; p.cout = NT; p.round_out = 0; p.out_scale = scale; p.seg = TC_SEG;
  p.spin_limit = tc_spin_limit();
  p.bias = zero_bias; p.act1 = ACT_NONE; p.slope1 = nullptr; p.act2 = ACT_NONE; p.slope2 = nullptr;
  p.out = make_tv(vol, 1, fa.h, fa.w, NT, NT); p.out2 = TV(); p.split_c = 0;
  const int stage_bytes = (sf16 ? 2 : 1) * A_BYTES + (split ? 2 : 1) * BN * BK * 4;
  const int smem = size_stages(p, stage_bytes);
  const int num_tiles = p.tiles_x * p.tiles_y * tiles_n;
  const int grid = num_tiles < cx.sm_count ? num_tiles : cx.sm_count;
  cx.launches++;
  if (cx.prof) cx.prof->begin(cx.stream, split ? (sf16 ? "corr_gemm_tc_3xf16" : "corr_gemm_tc_3xtf32") : "corr_gemm_tc_tf32", 2.0 * (double)Ms * NT * C);
  launch_tc(split, sf16, BN, grid, smem, cx.stream, mA, mA, mB, p);
  gv_check_launch("corr_volume_tc");
  if (cx.prof) cx.prof->end(cx.stream);
}

bool corr_volume_tc_wants_f16_planes() { return true; }

}  // namespace gv
#endif  // GV_HOSTSIM
