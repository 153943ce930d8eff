// Epilogue building blocks of the tensor-core convolutions (conv_tc.cu, conv_halo.cu, conv_wide.cu): activations, 4-channel loads / stores of
// fp32 or half tensors, shared-memory 128-bit accessors.  Device code only; include inside namespace gv::tc after tc_ptx.cuh.
#pragma once

__device__ __forceinline__ float rn_tf32(float x) {  // round-to-nearest-even to 10 mantissa bits
  uint32_t u = __float_as_uint(x);
  u += 0xfffu + ((u >> 13) & 1u);
  return __uint_as_float(u & 0xffffe000u);
}

// Rare activations (sigmoid / tanh / sin) go through ONE out-of-line copy: inlining the accurate sinf/tanhf/expf
// paths at every element site made the epilogue ~25k SASS instructions (instruction-cache bound, ~10 us per
// 32-column chunk measured).
__device__ __forceinline__ float sin_f32(float x) {
  // Cody-Waite reduction by pi (3 terms) + odd degree-9 minimax polynomial on [-pi/2, pi/2]; |err| < 2e-7 for |x| < 1e3
  // (libm's sinf carries a Payne-Hanek slow path with a local-memory table: ~3x slower as a call)
  const float k = rintf(x * 0.318309886183790672f);
  float r = fmaf(-k, 3.140625f, x);
  r = fmaf(-k, 9.67502593994140625e-4f, r);
  r = fmaf(-k, 1.509957990978376432e-7f, r);
  const float r2 = r * r;
  float p = fmaf(r2, 2.60831598e-6f, -1.98106907e-4f);
  p = fmaf(p, r2, 8.33307858e-3f);
  p = fmaf(p, r2, -1.66666597e-1f);
  p = fmaf(p * r2, r, r);
  return (((int)k) & 1) ? -p : p;
}
static __device__ __noinline__ float act_slow(float v, int act) {
  switch (act) {
    case ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    case ACT_TANH: return tanhf(v);
    case ACT_SIN: return sin_f32(v);
    case ACT_GELU: return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
    default: return v;
  }
}
// 4 channels of an optional side tensor at (pixel, channel c): float4 when in range and 16B aligned
__device__ __forceinline__ void load4(const float* p, int c, int cout, float* r) {
  if (c + 3 < cout && ((reinterpret_cast<uintptr_t>(p) & 15) == 0)) {
    const float4 v = *reinterpret_cast<const float4*>(p);
    r[0] = v.x; r[1] = v.y; r[2] = v.z; r[3] = v.w;
  } else {
#pragma unroll
    for (int u = 0; u < 4; ++u) r[u] = (c + u < cout) ? p[u] : 0.f;
  }
}
// 4 consecutive values -> 4 halves (round-to-nearest-even, saturating at +-65504 so a stray large activation cannot become inf)
__device__ __forceinline__ uint2 pack_h4(const float* o) {
  const float lim = 65504.f;
  const __half2 a = __floats2half2_rn(fminf(fmaxf(o[0], -lim), lim), fminf(fmaxf(o[1], -lim), lim));
  const __half2 b = __floats2half2_rn(fminf(fmaxf(o[2], -lim), lim), fminf(fmaxf(o[3], -lim), lim));
  uint2 r; r.x = *reinterpret_cast<const uint32_t*>(&a); r.y = *reinterpret_cast<const uint32_t*>(&b);
  return r;
}
// store 4 channels (first channel c) of an fp32 or half tensor at element offset eoff
__device__ __forceinline__ void store4(const TV& t, int64_t eoff, const float* o, int c, int cout, bool vec) {
  if (t.f16) {
    __half* q = reinterpret_cast<__half*>(t.p) + eoff;
    if (vec) { *reinterpret_cast<uint2*>(q) = pack_h4(o); }
    else {
#pragma unroll
      for (int u = 0; u < 4; ++u) if (c + u < cout) q[u] = __float2half_rn(fminf(fmaxf(o[u], -65504.f), 65504.f));
    }
  } else {
    float* q = t.p + eoff;
    if (vec) { *reinterpret_cast<float4*>(q) = make_float4(o[0], o[1], o[2], o[3]); }
    else {
#pragma unroll
      for (int u = 0; u < 4; ++u) if (c + u < cout) q[u] = o[u];
    }
  }
}
// 4 channels of an fp32 or half side tensor (residual) at element offset eoff
__device__ __forceinline__ void load4_any(const TV& t, int64_t eoff, int c, int cout, float* r) {
  if (t.f16) {
    const __half* q = reinterpret_cast<const __half*>(t.p) + eoff;
    if (c + 3 < cout && ((reinterpret_cast<uintptr_t>(q) & 7) == 0)) {
      const uint2 v = *reinterpret_cast<const uint2*>(q);
      const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
      r[0] = a.x; r[1] = a.y; r[2] = b.x; r[3] = b.y;
    } else {
#pragma unroll
      for (int u = 0; u < 4; ++u) r[u] = (c + u < cout) ? __half2float(q[u]) : 0.f;
    }
  } else {
    load4(t.p + eoff, c, cout, r);
  }
}

__device__ __forceinline__ float4 lds128(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void sts64(uint32_t a, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ void sts128(uint32_t a, float x, float y, float z, float w) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a), "f"(x), "f"(y), "f"(z), "f"(w) : "memory");
}
// activation over N values whose first channel is c (the dispatch is hoisted out of the element loops: one warp's
// epilogue is a dependent-instruction chain, so every instruction removed from it is ~5 cycles of critical path)
template <int N>
__device__ __forceinline__ void act_n(float* o, int act, const float* slope, int c, int cout) {
  if (act == ACT_NONE) return;
  if (act == ACT_RELU) {
#pragma unroll
    for (int u = 0; u < N; ++u) o[u] = fmaxf(o[u], 0.f);
  } else if (act == ACT_LRELU) {
#pragma unroll
    for (int u = 0; u < N; ++u) o[u] = o[u] > 0.f ? o[u] : 0.1f * o[u];
  } else if (act == ACT_PRELU) {
    if (c + N <= cout && ((reinterpret_cast<uintptr_t>(slope + c) & 15) == 0)) {
#pragma unroll
      for (int u = 0; u < N; u += 4) {
        const float4 sl = __ldg(reinterpret_cast<const float4*>(slope + c + u));
        o[u] = o[u] > 0.f ? o[u] : sl.x * o[u]; o[u + 1] = o[u + 1] > 0.f ? o[u + 1] : sl.y * o[u + 1];
        o[u + 2] = o[u + 2] > 0.f ? o[u + 2] : sl.z * o[u + 2]; o[u + 3] = o[u + 3] > 0.f ? o[u + 3] : sl.w * o[u + 3];
      }
    } else {
#pragma unroll
      for (int u = 0; u < N; ++u) { const float sl = (c + u < cout) ? slope[c + u] : 0.f; o[u] = o[u] > 0.f ? o[u] : sl * o[u]; }
    }
  } else if (act == ACT_SIGMOID) {   // 1 / (1 + 2^(-x log2 e)): MUFU.EX2 + MUFU.RCP, ~2 ulp (inline: the SepConvGRU gates)
#pragma unroll
    for (int u = 0; u < N; ++u) o[u] = __fdividef(1.f, 1.f + exp2f(-1.4426950408889634f * o[u]));
  } else if (act == ACT_TANH) {      // 1 - 2 / (1 + e^(2x)); absolute error ~1e-7 (saturates correctly at +-1)
#pragma unroll
    for (int u = 0; u < N; ++u) o[u] = 1.f - __fdividef(2.f, 1.f + exp2f(2.8853900817779268f * o[u]));
  } else {
#pragma unroll
    for (int u = 0; u < N; ++u) o[u] = act_slow(o[u], act);
  }
}
// the same activation on R rows of 4 channels that all start at channel c (phase 2 of the epilogue): per-channel slopes
// are fetched once, not once per row
template <int R>
__device__ __forceinline__ void act_rows(float* o, int act, const float* slope, int c, int cout) {
  if (act == ACT_PRELU) {
    float sl[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) sl[u] = (c + u < cout) ? __ldg(slope + c + u) : 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int u = 0; u < 4; ++u) o[4 * r + u] = o[4 * r + u] > 0.f ? o[4 * r + u] : sl[u] * o[4 * r + u];
  } else {
    act_n<4 * R>(o, act, slope, c, cout);   // (channel-independent activations)
  }
}

// ---- the per-pixel epilogue of conv_halo.cu and conv_wide.cu: one warp's raw accumulators are staged in shared memory as pixel rows
// of stg_ld bytes (8-channel piece k of staged pixel i at i * stg_ld + 32 k), and a loop over 8-channel pieces of whole pixels applies
// bias -> act1 -> residual -> act2 -> rounding and stores 16 or 32 bytes of the NHWC output.  A runtime loop keeps ONE copy of the
// activation code (unrolled over accumulator pairs it was ~5k instructions, instruction-fetch bound).  P has the fields H, W, cout,
// round_out, bias, act1, slope1, act2, slope2, res, out; piece(q, px, py, c0) maps piece q (staged pixel q / CPP, piece q % CPP) to
// its output pixel and first channel and tells whether it is inside the output.

// the residual of piece q as raw storage bits (8 halves in r[0], or 8 floats in r[0], r[1])
template <class P, class Piece>
__device__ __forceinline__ void epi_load_res(const P& p, int n, int q, const Piece& piece, uint4* rr) {
  int px, py, c0;
  rr[0] = rr[1] = make_uint4(0u, 0u, 0u, 0u);
  if (!piece(q, px, py, c0)) return;
  const int64_t e = p.res.off(n, py, px) + c0;
  if (p.res.f16) {
    const __half* src = reinterpret_cast<const __half*>(p.res.p) + e;
    if (c0 + 8 <= p.cout && (reinterpret_cast<uintptr_t>(src) & 15) == 0) rr[0] = *reinterpret_cast<const uint4*>(src);
    else for (int u = 0; u < 8 && c0 + u < p.cout; ++u) reinterpret_cast<__half*>(rr)[u] = src[u];
  } else {
    const float* src = p.res.p + e;
    if (c0 + 8 <= p.cout && (reinterpret_cast<uintptr_t>(src) & 15) == 0) { rr[0] = *reinterpret_cast<const uint4*>(src); rr[1] = *reinterpret_cast<const uint4*>(src + 4); }
    else for (int u = 0; u < 8 && c0 + u < p.cout; ++u) reinterpret_cast<float*>(rr)[u] = src[u];
  }
}

// pieces lane, lane + 32, ... < NPC; rcur holds the residual of piece `lane` (epi_load_res, issued early by the caller: e.g. while
// the MMAs run); each piece's successor's residual is read before the piece is computed
template <int NPC, int CPP, class P, class Piece>
__device__ __forceinline__ void epi_pieces(const P& p, int n, uint32_t stg_s, int stg_ld, int lane, const Piece& piece, uint4* rcur) {
  uint4 rnext[2];
#pragma unroll 1
  for (int q = lane; q < NPC; q += 32) {
    if (p.res.p && q + 32 < NPC) epi_load_res(p, n, q + 32, piece, rnext);
    int px, py, c0;
    if (piece(q, px, py, c0)) {
      const uint32_t a = stg_s + (uint32_t)((q / CPP) * stg_ld + (q % CPP) * 32);
      const float4 v0 = lds128(a), v1 = lds128(a + 16);
      float o[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
      for (int u = 0; u < 8; ++u) o[u] += c0 + u < p.cout ? __ldg(p.bias + c0 + u) : 0.f;
      act_n<8>(o, p.act1, p.slope1, c0, p.cout);
      if (p.res.p) {
        if (p.res.f16) {
#pragma unroll
          for (int u = 0; u < 8; ++u) o[u] += __half2float(reinterpret_cast<const __half*>(rcur)[u]);
        } else {
#pragma unroll
          for (int u = 0; u < 8; ++u) o[u] += reinterpret_cast<const float*>(rcur)[u];
        }
      }
      if (p.act2 != ACT_NONE) act_n<8>(o, p.act2, p.slope2, c0, p.cout);
      const bool full = c0 + 8 <= p.cout;
      const int64_t e = p.out.off(n, py, px) + c0;
      if (p.out.f16) {
        __half hv[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) hv[u] = __float2half_rn(fminf(fmaxf(o[u], -65504.f), 65504.f));
        __half* dst = reinterpret_cast<__half*>(p.out.p) + e;
        if (full && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(hv);
        else for (int u = 0; u < 8 && c0 + u < p.cout; ++u) dst[u] = hv[u];
      } else {
        if (p.round_out) {
#pragma unroll
          for (int u = 0; u < 8; ++u) o[u] = rn_tf32(o[u]);
        }
        float* dst = p.out.p + e;
        if (full && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
          *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
          *reinterpret_cast<float4*>(dst + 4) = make_float4(o[4], o[5], o[6], o[7]);
        } else for (int u = 0; u < 8 && c0 + u < p.cout; ++u) dst[u] = o[u];
      }
    }
    rcur[0] = rnext[0]; rcur[1] = rnext[1];
  }
}
