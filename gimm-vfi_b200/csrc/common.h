// gimmvfi_b200 — shared declarations for the sm_90a engine.
//
// Two build modes of the SAME sources:
//   * product:  nvcc -gencode arch=compute_90a,code=sm_90a  -> libgimmvfi_b200.so
//   * GV_HOSTSIM (tests/hostsim only): g++ -x c++ -DGV_HOSTSIM -fopenmp.  Every
//     "thread-per-element" kernel body is a __host__ __device__ functor, so the
//     identical code runs as an OpenMP loop on the CPU.  This exists to validate
//     the host orchestration and kernel arithmetic in the GPU-less build
//     container; it is never loaded by the product package.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <string>
#include <vector>
#include <map>
#include <stdexcept>

#ifdef GV_HOSTSIM
#define GV_HD inline
#define GV_DEV inline
typedef void* gvStream_t;
#else
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#define GV_HD __host__ __device__ __forceinline__
#define GV_DEV __device__ __forceinline__
typedef cudaStream_t gvStream_t;
#endif

namespace gv {

// ---------------------------------------------------------------------------
// Tensor view: NHWC, fp32.  element (n,y,x,ch) = p[n*sn + (y*w + x)*ld + ch].
// `c` is the number of channels visible through the view, `ld` the pixel stride
// of the underlying buffer (>= c): a channel slice of a concat buffer is a view.
// ---------------------------------------------------------------------------
struct TV {
  float* p = nullptr;
  int n = 0, h = 0, w = 0, c = 0;
  int ld = 0;
  int64_t sn = 0;
  int f16 = 0;   // 1: elements are IEEE half (p is reinterpreted); only the tensor-core conv reads / writes such tensors
  GV_HD int64_t off(int in, int y, int x) const { return (int64_t)in * sn + ((int64_t)y * w + x) * ld; }
  float* at(int64_t elem) const { return f16 ? reinterpret_cast<float*>(reinterpret_cast<uint16_t*>(p) + elem) : p + elem; }
  TV slice(int c0, int cnt) const { TV t = *this; t.p = at(c0); t.c = cnt; return t; }
  TV batch(int n0, int cnt) const { TV t = *this; t.p = at((int64_t)n0 * sn); t.n = cnt; return t; }
  int64_t pixels() const { return (int64_t)n * h * w; }
};

inline TV make_tv(float* p, int n, int h, int w, int c, int ld = 0) {
  TV t; t.p = p; t.n = n; t.h = h; t.w = w; t.c = c; t.ld = ld ? ld : c; t.sn = (int64_t)h * w * t.ld; return t;
}

// 16-byte vector access for the channel-vectorised pointwise kernels (4 consecutive channels per thread: one thread keeps 16
// bytes per load in flight instead of 4 — the scalar kernels topped out near 1.5 TB/s, a latency x occupancy bound)
struct alignas(16) F4 { float x, y, z, w; };
GV_HD F4 ld4(const float* p) { return *reinterpret_cast<const F4*>(p); }
GV_HD void st4(float* p, const F4& v) { *reinterpret_cast<F4*>(p) = v; }
inline bool aligned(const void* p, int bytes) { return (reinterpret_cast<uintptr_t>(p) & (uintptr_t)(bytes - 1)) == 0; }
// t's base, pixel stride and sample stride allow 4-lane vector access (16 bytes fp32, 8 bytes half) at every 4th channel
inline bool lanes4_ok(const TV& t) { return aligned(t.p, t.f16 ? 8 : 16) && t.ld % 4 == 0 && t.sn % 4 == 0; }
inline bool vec4_ok(const TV& t) { return lanes4_ok(t) && t.c % 4 == 0 && !t.f16; }

// IEEE binary16 with round-to-nearest-even and saturation to +-65504 (host side, bit exact with cvt.rn.satfinite.f16.f32)
inline uint16_t gv_f32_to_f16(float f) {
  uint32_t u; std::memcpy(&u, &f, 4);
  const uint16_t sign = (uint16_t)((u >> 16) & 0x8000u);
  u &= 0x7fffffffu;
  if (u > 0x7f800000u) return (uint16_t)(sign | 0x7e00u);                 // NaN
  if (u >= 0x477ff000u) return (uint16_t)(sign | 0x7bffu);                // >= 65520 (or inf): saturate
  if (u < 0x33000001u) return sign;                                       // < 2^-25: rounds to zero
  if (u < 0x38800000u) {                                                  // subnormal half
    const int shift = 113 - (int)(u >> 23);                               // 1..24
    uint32_t m = (u & 0x7fffffu) | 0x800000u;
    const uint32_t lsb = 1u << (shift + 13), half = lsb >> 1;
    uint32_t q = m >> (shift + 13);
    const uint32_t rem = m & (lsb - 1);
    if (rem > half || (rem == half && (q & 1u))) ++q;
    return (uint16_t)(sign | q);
  }
  uint32_t e = (u >> 23) - 112, m = u & 0x7fffffu;
  uint32_t h = (e << 10) | (m >> 13);
  const uint32_t rem = m & 0x1fffu;
  if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) ++h;
  return (uint16_t)(sign | h);
}

inline float gv_f16_to_f32(uint16_t h) {
  const uint32_t sign = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 0x1fu, m = h & 0x3ffu;
  uint32_t u;
  if (e == 0) {
    if (m == 0) u = sign;
    else { int sh = 0; uint32_t mm = m; while (!(mm & 0x400u)) { mm <<= 1; ++sh; } u = sign | ((uint32_t)(113 - sh) << 23) | ((mm & 0x3ffu) << 13); }
  } else if (e == 31) u = sign | 0x7f800000u | (m << 13);
  else u = sign | ((e + 112) << 23) | (m << 13);
  float f; std::memcpy(&f, &u, 4);
  return f;
}

// half-aware element access for the pointwise kernels that write / read the half-precision tensors of precision mode 4
GV_HD uint16_t gv_f2h(float v) {
#if defined(__CUDA_ARCH__)
  return __half_as_ushort(__float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f)));
#else
  return gv_f32_to_f16(v);
#endif
}
GV_HD float gv_h2f(uint16_t h) {
#if defined(__CUDA_ARCH__)
  return __half2float(__ushort_as_half(h));
#else
  return gv_f16_to_f32(h);
#endif
}
GV_HD float ld1(const TV& t, int64_t eoff) { return t.f16 ? gv_h2f(reinterpret_cast<const uint16_t*>(t.p)[eoff]) : t.p[eoff]; }
GV_HD void st1(const TV& t, int64_t eoff, float v) { if (t.f16) reinterpret_cast<uint16_t*>(t.p)[eoff] = gv_f2h(v); else t.p[eoff] = v; }
struct alignas(8) H4 { uint16_t x, y, z, w; };
GV_HD F4 ld4v(const TV& t, int64_t eoff) {   // 4 consecutive channels: one 16-byte (fp32) or 8-byte (half) access
  if (t.f16) { const H4 h = *reinterpret_cast<const H4*>(reinterpret_cast<const uint16_t*>(t.p) + eoff); F4 r = {gv_h2f(h.x), gv_h2f(h.y), gv_h2f(h.z), gv_h2f(h.w)}; return r; }
  return ld4(t.p + eoff);
}
GV_HD void st4v(const TV& t, int64_t eoff, const F4& v) {
  if (t.f16) { H4 h = {gv_f2h(v.x), gv_f2h(v.y), gv_f2h(v.z), gv_f2h(v.w)}; *reinterpret_cast<H4*>(reinterpret_cast<uint16_t*>(t.p) + eoff) = h; }
  else st4(t.p + eoff, v);
}
// like vec4_ok, half tensors allowed
inline bool vec4_ok_any(const TV& t) { return lanes4_ok(t) && t.c % 4 == 0; }

// L (1 or 4) consecutive channels as floats.  Any = false: fp32 storage, p[i] or one 16-byte access (ld4 / st4);
// Any = true: the half-aware ld1 / st1 / ld4v / st4v, which test t.f16 at run time.
template <int L> GV_HD void ld_lanes(const float* p, float* v) {
  if constexpr (L == 4) { const F4 a = ld4(p); v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; }
  else v[0] = p[0];
}
template <int L, bool Any> GV_HD void ld_lanes(const TV& t, int64_t eoff, float* v) {
  if constexpr (!Any) ld_lanes<L>(t.p + eoff, v);
  else if constexpr (L == 4) { const F4 a = ld4v(t, eoff); v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; }
  else v[0] = ld1(t, eoff);
}
template <int L, bool Any> GV_HD void st_lanes(const TV& t, int64_t eoff, const float* v) {
  if constexpr (L == 4) {
    const F4 a = {v[0], v[1], v[2], v[3]};
    if constexpr (Any) st4v(t, eoff, a); else st4(t.p + eoff, a);
  } else if constexpr (Any) st1(t, eoff, v[0]);
  else t.p[eoff] = v[0];
}
enum Act : int { ACT_NONE = 0, ACT_RELU = 1, ACT_LRELU = 2, ACT_PRELU = 3, ACT_SIGMOID = 4, ACT_TANH = 5, ACT_SIN = 6, ACT_GELU = 7 /* exact (erf) GELU: nn.GELU() of the FlowFormer / Twins MLPs */ };

GV_HD float apply_act(float v, int act, const float* slope, int ch) {
  switch (act) {
    case ACT_RELU: return v > 0.f ? v : 0.f;
    case ACT_LRELU: return v > 0.f ? v : 0.1f * v;
    case ACT_PRELU: return v > 0.f ? v : slope[ch] * v;
    case ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    case ACT_TANH: return tanhf(v);
    case ACT_SIN: return sinf(v);
    case ACT_GELU: return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
    default: return v;
  }
}

// Packed convolution weights (device memory): w[(ky*kw+kx)*cin + ci][cout_ld], bias[cout].
struct ConvW {
  const float* w = nullptr;
  const float* b = nullptr;
  int cin = 0, cout = 0, kh = 1, kw = 1;
  int cout_ld = 0;  // row stride of w (cout rounded up to 4)
  // tensor-core layout (conv_tc.cu): w_tc[2][tap][cout_pad][cin_pad] zero padded; plane 0 = tf32_rn(w),
  // plane 1 = tf32_rn(w - plane0) (the "lo" term of the 3xTF32 split, present when has_lo)
  const float* w_tc = nullptr;
  int cout_pad = 0, cin_pad = 0;
  bool has_lo = false;
  // fp16 copy for layers fed with half-precision activations: w_tc_h[tap][cout_pad][cin_pad_h] (cin padded to 64)
  const void* w_tc_h = nullptr;
  int cin_pad_h = 0;
  // fp16 hi / lo planes of w * w_scale for the 3-term f16 split (conv_tc.cu "3xF16"): w_tc_s[2][tap][cout_pad][cin_pad_s]
  // (cin padded to 64); w_scale = a power of two that lifts max|w| to [2^13, 2^14) so the lo parts stay normal halves
  const void* w_tc_s = nullptr;
  int cin_pad_s = 0;
  float w_scale = 1.f;
};

// N tiling of the tensor-core path: cout padded to 16, split into <= 256-wide tiles of equal width.
inline void tc_tile_n(int cout, int* bn, int* tiles_n) {
  const int c16 = (cout + 15) & ~15;
  const int tn = (c16 + 255) / 256;
  *tiles_n = tn;
  *bn = (((c16 + tn - 1) / tn) + 15) & ~15;
}
inline int tc_cout_pad(int cout) { int bn, tn; tc_tile_n(cout, &bn, &tn); return bn * tn; }

// y = act2( res + act1(conv(x) + b) ) * mul      (res / mul optional)
// gru:  y = (1 - z) * hprev + z * y               (SepConvGRU update, raft/update.py:58,66)
struct ConvEpi {
  int act1 = ACT_NONE; const float* slope1 = nullptr;
  int act2 = ACT_NONE; const float* slope2 = nullptr;
  TV res;   // optional residual (same n,h,w as output; res.p == nullptr -> none)
  TV mul;   // optional elementwise multiplier
  TV gru_z, gru_h;  // optional GRU blend
  // two convolutions over the same input merged along cout (SepConvGRU z | r gates): output channels >= split_c go to out2
  // (as its channels 0..), and `mul` applies to them only.  Tensor-core path only.
  TV out2; int split_c = 0;
};

struct ConvGeom {
  int stride = 1;
  int ph = 0, pw = 0;
  int reflect = 0;  // 0: zero padding, 1: reflect padding (padding_mode="reflect")
  int loose_w = 0;  // x-taps packed into the channel axis of a zero-padded input (Engine::pack_xpacked): the input is
                    // larger than the output and carries its own padding, so the size / padding checks are skipped
};

// ---------------------------------------------------------------------------
// Fused HypoNet (hyponet.cu): byte layout of the packed parameter blob, exactly as it sits in shared memory.  Weight tiles are
// K-major [out row][128-byte K block] in the SWIZZLE_128B pattern of the wgmma descriptors (16-byte chunk c of row r at c ^ (r & 7)).
//   W0  [128][32] fp32 (TF32-rounded)  latent part of layer 0        | W1..W3 [2 K blocks][128][64] half | W4 [2][16][64] half (2 rows used)
//   AFF [4][128] fp32: layer-0 rows of t, y, x and the bias          | B1..B3 [128] fp32 | B4 [16] fp32 (output_bias folded in)
namespace hypo {
constexpr int W0 = 0, W1 = 16384, W4 = 16384 + 3 * 32768, AFF = W4 + 4096, B1 = AFF + 2048, B4 = B1 + 3 * 512, BLOB = B4 + 64;
inline size_t swz(int row, int byte_in_row) { return (size_t)row * 128 + (size_t)((((byte_in_row >> 4) ^ (row & 7)) << 4) | (byte_in_row & 15)); }
}  // namespace hypo
// fp32-class variant (hyponet.cu, hyponet_fused3): layers 1-3 as three f16 MMAs on fp16 hi / lo pairs (weights pre-scaled by
// 2^6 and pre-split; activations split in registers as the next layer's A operand), layers 0 and 4 on the CUDA cores in fp32.
//   W13 [3 layers][hi, lo][2 K blocks][128][64] half, swizzled as above | W0A [36][128] fp32: rows 0..31 latent, 32..34 (t, y, x), 35 bias
//   B13 [3][128] fp32 | W4 [128][2] fp32 | B4 [2] fp32 (output_bias folded in)
namespace hypo3 {
constexpr int W13 = 0, W0A = 3 * 2 * 2 * 16384, B13 = W0A + 36 * 128 * 4, W4 = B13 + 3 * 512, B4 = W4 + 1024, BLOB = B4 + 16;
constexpr float W_SCALE = 64.f;
}  // namespace hypo3

// HypoNet's activation between its layers (modules/utils.py:65-76, layers.py:13-42, hyponet.py:140-141).  HYPO_SIREN1 is the shipped
// sin(x) with w0 = 1, on MUFU sin (__sinf) in the fused kernels; every other form uses the accurate sinf, whose argument reduction keeps
// sin(w0 x) exact to an ulp where the pre-activation grows by w0 (MUFU's absolute error grows with |x| beyond pi).
enum HypoAct : int { HYPO_SIREN1 = 0, HYPO_SIREN = 1, HYPO_RELU = 2, HYPO_SILU = 3, HYPO_DAMP = 4 };
template <int A> GV_HD float hypo_act(float x, float w0) {
  if constexpr (A == HYPO_SIREN1) return sinf(x);
  else if constexpr (A == HYPO_SIREN) return sinf(w0 * x);
  else if constexpr (A == HYPO_RELU) return x > 0.f ? x : 0.f;
  else if constexpr (A == HYPO_SILU) return x / (1.f + expf(-x));
  else {   // Damping: clamp(x, min=1e-30), then sin(w0 x) sqrt(|x|)
    const float c = x > 1e-30f ? x : 1e-30f;
    return sinf(w0 * c) * sqrtf(c);
  }
}
// the forward splat's normalisation mode (modules/softsplat.py:286-352 with the "-zeroeps" suffix the models append)
enum SplatMode : int { SPLAT_LINEAR = 0, SPLAT_SOFTMAX = 1, SPLAT_SUM = 2 };

// ---------------------------------------------------------------------------
// Execution context
// ---------------------------------------------------------------------------
struct Arena {
  char* base = nullptr;
  size_t cap = 0, top = 0, peak = 0;
  bool dry = false;  // planning pass: only track the high-water mark
  float* alloc_f(size_t n_floats) {
    size_t bytes = (n_floats * sizeof(float) + 255) & ~size_t(255);
    size_t o = top;
    top += bytes;
    if (top > peak) peak = top;
    if (dry) return reinterpret_cast<float*>(size_t(4096) + o);  // fake, never dereferenced
    if (top > cap) throw std::runtime_error("gimmvfi: workspace too small (need " + std::to_string(top) + " bytes, have " + std::to_string(cap) + ")");
    return reinterpret_cast<float*>(base + o);
  }
  TV tensor(int n, int h, int w, int c, int ld = 0) { if (!ld) ld = c; return make_tv(alloc_f((size_t)n * h * w * ld), n, h, w, c, ld); }
  TV tensor_h(int n, int h, int w, int c, int ld = 0) {   // half-precision storage (ld % 8 == 0: 16-byte TMA strides)
    if (!ld) ld = (c + 7) & ~7;
    TV t = make_tv(alloc_f(((size_t)n * h * w * ld + 1) / 2), n, h, w, c, ld); t.f16 = 1; return t;
  }
  TV tensor_like(const TV& x, int c) { return x.f16 ? tensor_h(x.n, x.h, x.w, c) : tensor(x.n, x.h, x.w, c); }
  size_t mark() const { return top; }
  void release(size_t m) { top = m; }
};

// Optional per-launch timing (CUDA events on the launching stream), keyed by kernel name.
struct ProfRec { const char* name; double work; void* ev0; void* ev1; };
const char* prof_intern(const std::string& s);  // stable storage for dynamically built kernel labels
struct Profiler {
  std::vector<ProfRec> recs;
  std::vector<void*> pool; size_t used = 0;
  void* get_event();
  void begin(gvStream_t s, const char* name, double work);
  void end(gvStream_t s);
  void reset() { recs.clear(); used = 0; }
  ~Profiler();
};

struct Ctx {
  Profiler* prof = nullptr;
  bool tc = false;        // route eligible convolutions to the tensor-core (wgmma) path
  bool tc_split = false;  // ... with 3xTF32 operand splitting (fp32-class accuracy)
  gvStream_t stream = nullptr;
  Arena arena;
  bool dry = false;       // skip kernel launches (planning)
  int64_t launches = 0;   // kernels launched by the last forward
  int sm_count = 132;
};

void gv_check_launch(const char* what);

#ifndef GV_HOSTSIM
// cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE function attribute: remember it per (call site, device).
// `flags` is a zero-initialised static array of 64 bytes owned by the call site; a benign race sets the attribute twice.
template <class K>
inline void gv_set_max_smem(K kernel, int bytes, volatile unsigned char* flags) {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && flags[dev]) return;
  cudaError_t er = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (er != cudaSuccess) throw std::runtime_error(std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(er));
  if (dev >= 0 && dev < 64) flags[dev] = 1;
}
#endif

// ---------------------------------------------------------------------------
// thread-per-element launcher
// ---------------------------------------------------------------------------
#ifndef GV_HOSTSIM
template <class F>
__global__ void __launch_bounds__(256) gv_elementwise_kernel(F f, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += step) f(i);
}
#endif

template <class F>
inline void parallel_for(Ctx& cx, int64_t n, const F& f, const char* name) {
  if (cx.dry || n <= 0) return;
  cx.launches++;
#ifdef GV_HOSTSIM
  (void)name;
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < n; ++i) f(i);
#else
  if (cx.prof) cx.prof->begin(cx.stream, name, (double)n);
  int64_t blocks = (n + 255) / 256;
  int64_t cap = (int64_t)cx.sm_count * 32;  // grid-stride beyond 32 CTAs/SM
  if (blocks > cap) blocks = cap;
  gv_elementwise_kernel<F><<<(unsigned)blocks, 256, 0, cx.stream>>>(f, n);
  gv_check_launch(name);
  if (cx.prof) cx.prof->end(cx.stream);
#endif
}

// A pointwise op written once over L lanes (functor template K<L, Any>, fields initialised from `a`): K<4, Any> over elems / 4
// items when `four`, else K<1, Any> over elems items, both under the op's kernel name.
template <template <int, bool> class K, bool Any = false, class... A>
inline void lanes_for(Ctx& cx, bool four, int64_t elems, const char* name, const A&... a) {
  if (four) parallel_for(cx, elems / 4, K<4, Any>{a...}, name);
  else parallel_for(cx, elems, K<1, Any>{a...}, name);
}

GV_HD bool gv_isfinite(float v) { return fabsf(v) <= 3.402823466e+38f; }  // false for NaN / +-inf

GV_HD float atomic_add_f(float* addr, float v) {
#if defined(GV_HOSTSIM)
  float old;
#pragma omp atomic capture
  { old = *addr; *addr += v; }
  return old;
#elif defined(__CUDA_ARCH__)
  return atomicAdd(addr, v);
#else
  float old = *addr; *addr += v; return old;
#endif
}

// ---------------------------------------------------------------------------
// op library (ops_*.cu)
// ---------------------------------------------------------------------------
// conv.cu
void conv2d(Ctx& cx, const TV& in0, const TV& in1 /*optional 2nd channel segment*/, const ConvW& w, const ConvGeom& g,
            const ConvEpi& e, const TV& out);
bool conv7x7_small_cout(Ctx& cx, const TV& in, const ConvW& w /*plain packed [tap][cin][4]*/, int act, const float* slope, const TV& out);   // conv.cu
// conv_tc.cu (sm_90a wgmma / TMA path; not part of the host simulation)
bool conv2d_tc_supported(const TV& in0, const TV& in1, const ConvW& w, const ConvGeom& g, const ConvEpi& e, const TV& out, bool split);
void conv2d_tc(Ctx& cx, const TV& in0, const TV& in1, const ConvW& w, const ConvGeom& g, const ConvEpi& e, const TV& out, bool split);
void corr_volume_tc(Ctx& cx, const TV& fa, const float* fb_planes, const float* zero_bias, float* vol, float scale, bool split, int n_targets = 0);
bool corr_volume_tc_wants_f16_planes();   // split mode: true -> fb_planes must come from split_planes_f16 (3xF16 form), else split_planes
// how long the TMA pipelines of conv_tc.cu, conv_halo.cu and corr_gemm.cu wait on an mbarrier before trapping, in units of 10 ms
// (tc_ptx.cuh mbar_wait): GIMMVFI_TC_SPIN_LIMIT, default 400; 0 = wait forever (compute-sanitizer)
int tc_spin_limit();
// corr_gemm.cu (sm_90a): vol[i][j] = scale * <A[i,:], B[j,:]> in the 3xF16 form, row pitch NT; A / B = half planes [2][rows][K] from
// split_planes_f16 (a_plane / b_plane: elements from the hi to the lo plane), K % 64 == 0
void corr_gemm_3xf16(Ctx& cx, const void* a_planes, int64_t a_plane, int M, const void* b_planes, int64_t b_plane, int NT, int K, float scale,
                     float* vol);
// conv_halo.cu (sm_90a): 3x3 / 1x1 stride-1 convolutions of K-poor layers (cin <= 32 fp32 / 64 half, cout <= 64) with the activation
// tile + halo loaded once (three x-shifted copies) and every tap an MMA on a 1024-byte aligned view of it, weights resident
bool conv2d_halo_supported(const TV& in0, const TV& in1, const ConvW& w, const ConvGeom& g, const ConvEpi& e, const TV& out);
void conv2d_halo(Ctx& cx, const TV& in0, const ConvW& w, const ConvGeom& g, const ConvEpi& e, const TV& out);
// conv_wide.cu (sm_90a): 3x3 stride-1 convolutions of wide half layers (input segments of whole 64-channel blocks, cout a multiple of
// 128: the final decoder's 256-channel trunk) with each K block's activation tile + halo loaded once and the weights streamed per tap
bool conv2d_wide_supported(const TV& in0, const TV& in1, const ConvW& w, const ConvGeom& g, const ConvEpi& e, const TV& out);
void conv2d_wide(Ctx& cx, const TV& in0, const TV& in1, const ConvW& w, const ConvGeom& g, const ConvEpi& e, const TV& out);
// hyponet.cu (sm_90a; the host simulation emulates its arithmetic): the whole HypoNet MLP in one kernel
bool hyponet_fused_supported(const TV& lat, const TV& out);
void hyponet_fused(Ctx& cx, const TV& lat /*n,h,w,32*/, const float* coords /*n*h*w x (t,y,x)*/, const void* blob /*hypo:: layout*/, const TV& out /*2 ch*/);
void hyponet_fused3(Ctx& cx, const TV& lat, const float* coords, const void* blob3 /*hypo3:: layout*/, const TV& out);   // fp32-class arithmetic
// hyponet_fused3 on a coordinate grid of another size than the latent: out (n,hc,wc,2), coords n*hc*wc x (t,y,x); layer 0 takes the
// bilinear resize of the latent to (hc, wc) (align_corners = False, = resize_bilinear with scales h / hc, w / wc), interpolated in registers
void hyponet_fused3_resample(Ctx& cx, const TV& lat /*n,h,w,32*/, const float* coords, const void* blob3, const TV& out /*n,hc,wc,2*/);
// The three kernels above with another activation between the layers (HypoAct; HYPO_SIREN1 is the functions above).  The host
// simulation runs them as the per-pixel functors HypoNetEmuK<false / true> (engine.cu).
void hyponet_fused_act(Ctx& cx, const TV& lat, const float* coords, const void* blob, const TV& out, int act, float w0);
void hyponet_fused3_act(Ctx& cx, const TV& lat, const float* coords, const void* blob3, const TV& out, int act, float w0);
void hyponet_fused3_resample_act(Ctx& cx, const TV& lat, const float* coords, const void* blob3, const TV& out, int act, float w0);
// ops_pointwise.cu: x = act(x) in place on every channel of x (HypoNet's activation after a layer that ran as a plain convolution)
void hypo_activation(Ctx& cx, const TV& x, int act, float w0);
// corr.cu
void split_planes(Ctx& cx, const TV& src, float* planes);  // [2][n*h*w][c]: rn_tf32(x) and rn_tf32(x - rn_tf32(x))
void split_planes_f16(Ctx& cx, const TV& src, void* planes);  // half [2][n*h*w][c]: rn_f16(x) and rn_f16(x - rn_f16(x))
void corr_volume(Ctx& cx, const TV& fa, const TV& fb, float* vol, float scale);   // vol[n][i][j] = <fa[n,i], fb[n,j]> * scale
void corr_pool(Ctx& cx, const float* src, float* dst, int64_t rows, int h, int w); // rows x (h*w) -> rows x (h/2*w/2)
void avgpool2_features(Ctx& cx, const TV& src, const TV& dst);   // NHWC 2x2 average, floor semantics (F.avg_pool2d(x, 2, 2))
void corr_pool_pyramid(Ctx& cx, const float* l0, float* l1, float* l2, float* l3, int64_t rows, int h, int w);
struct CorrPyr { const float* lvl[4]; int h[4], w[4]; int64_t rows_per_sample; int nl = 4; /* levels looked up: out has nl * 81 channels (FlowFormer: 1) */ };
void corr_lookup(Ctx& cx, const CorrPyr& pyr, const TV& coords /*n,h,w,2 (x,y)*/, const TV& out /*324 ch*/);
// volume-free lookup: the other frame's features (IEEE half, NHWC, c channels; level l = the 2^l x 2^l average-pooled map, sample-major)
struct CorrFeat { const uint16_t* lvl[4]; int h[4], w[4]; int c; float scale; };
void features_to_half(Ctx& cx, const TV& src, void* dst /*half, dense NHWC*/);
bool corr_lookup_direct_supported(const TV& src, const CorrFeat& tgt, const TV& coords, const TV& out);
void corr_lookup_direct(Ctx& cx, const TV& src /*n,h,w,256 fp32: the source frame's features*/, const CorrFeat& tgt, const TV& coords, const TV& out);
// memory-free correlation with gradients (alt_cuda_corr, gimmvfi_op_alt_corr_*): dense fp32 f1 (B,H1,W1,C), f2 (B,H2,W2,C), coords
// (B,N,H1,W1,2); corr / corr_grad (B,N,(2r+1)^2,H1,W1).  H2 * W2 * C < 2^31 (tap offsets within a sample are 32-bit).
struct AltCorrArgs { const float* f1 = nullptr; const float* f2 = nullptr; const float* coords = nullptr; int B = 0, N = 0, H1 = 0, W1 = 0, H2 = 0, W2 = 0, C = 0, r = 0; };
struct AltCell { int x0, y0; float dx, dy; bool in; };   // window anchor (x0 - r, y0 - r), bilinear fractions; !in: every tap off frame
constexpr size_t ALT_CORR_SMEM_MAX = 227 * 1024;        // dynamic shared memory of one CTA on sm_90a
bool alt_corr_launch_shape(int r, int* warps, int* tile_w);   // false: radius r needs more shared memory than a CTA has
void alt_corr_forward(Ctx& cx, const AltCorrArgs& a, float* corr);   // every element of corr written
// each output optional; f2g must be zero-filled by the caller (scatter with atomics); f1g and cog are fully written (no atomics)
void alt_corr_backward(Ctx& cx, const AltCorrArgs& a, const float* corr_grad, float* f1g, float* f2g, float* cog);
// ops_pointwise.cu
void nchw_to_nhwc(Ctx& cx, const float* src, int64_t src_sn, int64_t src_sc, const TV& dst, float scale, float shift);
void nhwc_to_nchw(Ctx& cx, const TV& src, float* dst, int64_t dst_sn, int64_t dst_sc, float scale, float shift, int clamp01);  // (v + shift) * scale
// index-table stores: sample n of src goes to row rows[n] of dst (rows ride in the kernel parameters, kGatherMax per launch;
// consecutive rows take the plain store)
constexpr int kGatherMax = 64;
void nhwc_to_nchw_rows(Ctx& cx, const TV& src, float* dst, const std::vector<int>& rows, int64_t dst_sn, int64_t dst_sc, float scale, float shift,
                       int clamp01);
// sample_coord_input's grid for n = t.size() samples, each at its own t: coords (n,hc,wc,3) (t, y, x) and tdev (n), on the device
void query_coords(Ctx& cx, const std::vector<float>& t, int hc, int wc, float lo, float span, float* coords, float* tdev);
void copy_channels(Ctx& cx, const TV& src, const TV& dst);
void frames_u8_to_padded_f32(Ctx& cx, const uint8_t* src, int n, int h, int w, float* dst_nchw, int H, int W, int pad_top, int pad_left);
void pred_to_u8(Ctx& cx, const float* src_nchw, int n, int H, int W, uint8_t* dst, int h, int w, int pad_top, int pad_left, int bgr);
// flow_to_image (src/utils/flow_viz.py): a float32 flow read through element strides (n, y, x, channel) -> uint8 (n,h,w,3) colour-wheel
// pictures, one maximum radius per image (scratch: flow_to_image_scratch_floats) unless has_max (then max_div = fl32(max_flow + 1e-5))
struct FlowView { const float* p = nullptr; int64_t sn = 0, sy = 0, sx = 0, sc = 0; int n = 0, h = 0, w = 0; };
int64_t flow_to_image_scratch_floats(int n, int h);
void flow_to_image(Ctx& cx, const FlowView& flow, int has_clip, float clip, int has_max, float max_div, int bgr, float* scratch, uint8_t* dst);
// scene-cut sums of n frame pairs: a, b (n,h,w,3) uint8 RGB, pair i = (a[i], b[i]) -> sums[i] = (sum |dH|, sum |dS|, sum |dV|) of
// their 8-bit HSV (cv2.COLOR_RGB2HSV); every sum written, bit-exact on every run
void scene_sums(Ctx& cx, const uint8_t* a, const uint8_t* b, int n, int h, int w, uint64_t* sums);
// one output frame of a shutter blend: dst (h,w,3) uint8 = trunc(clamp(mean of the n sources, 0, 255)), BGR when bgr.  Source i is a
// float32 (3,H,W) row cropped at (pad_top, pad_left), values x * 255 (is_f32[i]), or an (h,w,3) uint8 RGB frame; one launch
constexpr int kBlendMax = 63;
void blend_u8(Ctx& cx, const void* const* src, const int* is_f32, int n, int H, int W, int pad_top, int pad_left, uint8_t* dst, int h, int w,
              int bgr);
// forward_interpolate (raft/utils/utils.py:33-63) of n dense (2,h,w) flows -> out (n,2,h,w), which must not overlap flow
void forward_interpolate(Ctx& cx, const float* flow, int n, int h, int w, float* out);
void pad_image4(Ctx& cx, const TV& src /*c=3, ld=4*/, const TV& dst /*h+2p, w+2p, ld 4*/, int pad);
void pad_reflect(Ctx& cx, const TV& src, const TV& dst /*h+2p, w+2p*/, int pad);
void pad_zero(Ctx& cx, const TV& src, const TV& dst /*h+2p, w+2p, all dst.ld lanes written*/, int pad);
void fill(Ctx& cx, const TV& dst, float v);
void axpby(Ctx& cx, const TV& a, float alpha, const TV& b, float beta, const TV& out);  // out = alpha*a + beta*b (b optional)
void resize_bilinear(Ctx& cx, const TV& src, const TV& dst, float scale_y, float scale_x, float mult, int accumulate, int act);
void backwarp(Ctx& cx, const TV& src, const TV& flow /*2ch at dst res*/, const TV& dst);
void pixel_shuffle(Ctx& cx, const TV& src, const TV& dst, int times);
void instnorm_stats(Ctx& cx, const TV& x, float* mean_rstd /*n*c*2*/, float* scratch, int64_t scratch_floats);
void instnorm_apply(Ctx& cx, const TV& x, const float* mean_rstd, int act1, const TV& res, int act2, const TV& out);
int64_t instnorm_scratch_floats(const TV& x);
void absmax_per_sample(Ctx& cx, const TV& a, const TV& b, float* out_n, float* scratch);  // out[n] = max(|a|,|b|)
int64_t absmax_scratch_floats(const TV& a);
void convex_upsample(Ctx& cx, const TV& flow, const TV& mask, const TV& out);
void coords_minus_grid(Ctx& cx, const TV& coords1, const TV& flow_out_a, const TV& flow_out_b);
void init_coords(Ctx& cx, const TV& coords);
void splat_weights(Ctx& cx, const TV& f_self, const TV& f_other, const float* g9, const float* alpha_fe, const float* alpha_v, const TV& out);
void normalize_flow_pair(Ctx& cx, const TV& f01, const TV& f10, const float* scaler, const TV& n0, const TV& n1);
void softsplat_accumulate(Ctx& cx, const TV& lat, const TV& flow, const TV& metric, const float* t_per_sample, int t_mode, const TV& acc);
void softsplat_normalize(Ctx& cx, const TV& acc, const TV& out);
// The product splat in the other modes of modules/softsplat.py:286-352 (SplatMode).  SPLAT_SOFTMAX: acc as softsplat_accumulate with
// exp(metric) in place of the metric, normalised by softsplat_normalize.  SPLAT_SUM: acc (16 channels, zero-filled by the caller) +=
// the plain splat of lat, metric ignored; that is the result, nothing is normalised.
void softsplat_accumulate_mode(Ctx& cx, const TV& lat, const TV& flow, const TV& metric, const float* t_per_sample, int t_mode, const TV& acc, int mode);
// the whole splat in one pass (target tiles in shared memory); flow_absmax[n] >= max |flow| of sample n bounds the scan region
bool softsplat_fused(Ctx& cx, const TV& lat, const TV& flow, const TV& metric, const float* t_per_sample, int t_mode, const float* flow_absmax,
                     const TV& out);
// Differentiable splat of modules/softsplat.py:358-663 (softsplat_func) on 4-D strided NCHW tensors of float or double;
// element (n,c,y,x) = p[n*s[0] + c*s[1] + y*s[2] + x*s[3]] (64-bit sizes and strides, in elements).
template <class T> struct SV4 { T* p = nullptr; int64_t sz[4] = {0, 0, 0, 0}, st[4] = {0, 0, 0, 0}; };
// out += the splat of `in` along `flow` (the caller zero-fills out)
template <class T> void softsplat_out_any(Ctx& cx, const SV4<T>& in, const SV4<T>& flow, const SV4<T>& out);
// one pass: ingrad and / or flowgrad (either may have p == nullptr) of the splat for the incoming gradient `outgrad`
template <class T> void softsplat_grad_any(Ctx& cx, const SV4<T>& in, const SV4<T>& flow, const SV4<T>& outgrad, const SV4<T>& ingrad,
                                           const SV4<T>& flowgrad);
void scale_flow_t(Ctx& cx, const TV& flow_t, const float* t_per_sample, const TV& f0, const TV& f1);
void hypo_pack_input(Ctx& cx, const float* coord /*B,Hc,Wc,3*/, const TV& dst /*slice of 3 ch*/);
void unnormalize_flow(Ctx& cx, const TV& ninr, const float* scaler, const TV& out);
void lookup_coords(Ctx& cx, const TV& flow, const float* t_per_sample, int mode, const TV& out);
void flow_mask_split(Ctx& cx, const TV& out133, const TV& f0_in, const TV& f1_in, const TV& f0, const TV& f1, const TV& mask);
void add_inplace_slices(Ctx& cx, const TV& dst, const TV& src);
void final_heads(Ctx& cx, const TV& out24, const TV& flow0, const TV& flow1, const TV& mask, const TV& oflow0, const TV& oflow1,
                 const TV& omask, const TV& ores);
void warp_blend(Ctx& cx, const TV& img0, const TV& img1, const TV& f0, const TV& f1, const TV& mask_logit, const TV& out_nhwc);
void multi_flow_blend(Ctx& cx, const TV& img0, const TV& img1, const TV& f0, const TV& f1, const TV& mask, const TV& res,
                      const TV& warps9, const TV& mean3);
void combine_output(Ctx& cx, const TV& mean3, const TV& conv3, float* dst_nchw);
void combine_output_rows(Ctx& cx, const TV& mean3, const TV& conv3, float* dst_nchw, const std::vector<int>& rows);   // image n -> dst image rows[n]
// LPIPS (src/utils/lpips, AlexNet v0.1): conv1's input as a 4x4 space-to-depth of the padded, prepared images (dst (2n, hs, ws, 48),
// images [in0 ; in1]), MaxPool2d(3, 2), and the head: per-row partial sums of one layer's term, then per image the 5 spatial means
void lpips_prep(Ctx& cx, const float* in0, const float* in1, int n, int h, int w, int quantize, int normalize, const float* shift,
                const float* scale, const TV& dst);
void maxpool3x3s2(Ctx& cx, const TV& src, const TV& dst);
void lpips_head_rows(Ctx& cx, const TV& f /*2n images*/, int n, const float* lin_w, double* partial /*n * f.h*/);
void lpips_head_images(Ctx& cx, const double* const partial[5], const int h[5], const int w[5], int n, float* per_layer /*n x 5, optional*/, float* out /*n*/);

// ops_tokens.cu (FlowFormer / Twins token-side kernels; see the file header)
void patchify(Ctx& cx, const TV& src, const TV& dst, int k);
void layernorm(Ctx& cx, const TV& x, const float* g, const float* b, float eps, const TV& out /*may be larger: zero padded*/, float pe_scale = 0.f, int pe_dim = 0);
void dwconv3x3_residual(Ctx& cx, const TV& x, const float* w9c, const float* bias, const TV& out);
void window_attention(Ctx& cx, const TV& q, const TV& k, const TV& v /*padded maps*/, const TV& out /*unpadded*/, int heads, int ws);
struct AttnDims {
  int64_t nb1, nb2, nq, nk; int heads;
  int64_t q_s1, q_s2, q_si; int64_t k_s1, k_s2, k_sj; int64_t v_s1, v_s2, v_sj; int64_t o_s1, o_s2, o_si;
};
void strided_attention(Ctx& cx, const float* q, const float* k, const float* v, float* out, const AttnDims& a, int head_dim);
void concat_pe(Ctx& cx, const TV& a, const TV& b, const TV& out, int ws, bool add_pe, int grp_all, int ctx_per);
void write_pe(Ctx& cx, const TV& out, float scale, float shift);
void add_pe_coords(Ctx& cx, const TV& x, const TV& coords, const TV& out);
void cost_conv1(Ctx& cx, const float* vol, int64_t maps, int h, int w, const float* wt_host /*[36][16]*/, const float* bias_host /*[16]*/, const TV& out_padded, int oh, int ow);
void row_softmax(Ctx& cx, float* p, int64_t rows, int64_t cols, float mul);
void gemm_nn(Ctx& cx, const float* A, const float* Bm, float* out, int64_t rows, int64_t K, int D, int64_t lda, int64_t ldb, int64_t ldo, float scale);
void transpose_2d(Ctx& cx, const float* src, float* dst, int64_t rows, int cols, int64_t lds);
void axpy_dev(Ctx& cx, const TV& a, const TV& b, const float* alpha, const TV& out);
void broadcast_tokens(Ctx& cx, const float* src, const TV& out, int T);

// device memory helpers (hostsim: plain host memory)
void* dev_alloc(size_t bytes);
void dev_free(void* p);
void dev_upload(void* dst, const void* src, size_t bytes);
void dev_download(void* dst, const void* src, size_t bytes, gvStream_t s);
void dev_memset(void* dst, int v, size_t bytes, gvStream_t s);
void dev_copy(void* dst, const void* src, size_t bytes, gvStream_t s);
void dev_sync(gvStream_t s);

}  // namespace gv
