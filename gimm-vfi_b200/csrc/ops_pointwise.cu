// HBM-bound thread-per-element kernels of the GIMM-VFI-R path (warp / resize /
// splat / normalise / blend ...).  Every kernel body is a functor executed by
// gv::parallel_for (CUDA grid-stride kernel, or an OpenMP loop under GV_HOSTSIM).
// Reference semantics are cited per kernel (paths relative to
// /root/reference/src/models/generalizable_INR/).
#include "common.h"

namespace gv {

// ------------------------------------------------------------------ helpers
// torch.linspace(-1, 1, n)[i]  (symmetric evaluation used by ATen's linspace)
GV_HD float linspace_m1_1(int i, int n) {
  if (n <= 1) return -1.f;
  float step = 2.f / (float)(n - 1);
  return (i < n / 2) ? (-1.f + step * (float)i) : (1.f - step * (float)(n - 1 - i));
}

struct BilinearTap {
  int x0, y0, x1, y1;
  float wx0, wx1, wy0, wy1;  // weights of x0/x1 and y0/y1
  bool vx0, vx1, vy0, vy1;
};

// grid_sample(bilinear, padding_mode="border", align_corners=True) at pixel
// (x + fx, y + fy) expressed the way modules/fi_utils.py:19-49 builds the grid:
// base = linspace(-1,1,W_flow), offset = flow / ((W_src-1)/2).
GV_HD BilinearTap border_tap(int x, int y, float fx, float fy, int wf, int hf, int ws, int hs) {
  float gx = linspace_m1_1(x, wf) + fx / (((float)ws - 1.0f) / 2.0f);
  float gy = linspace_m1_1(y, hf) + fy / (((float)hs - 1.0f) / 2.0f);
  float ix = ((gx + 1.f) / 2.f) * (float)(ws - 1);
  float iy = ((gy + 1.f) / 2.f) * (float)(hs - 1);
  ix = fminf(fmaxf(ix, 0.f), (float)(ws - 1));
  iy = fminf(fmaxf(iy, 0.f), (float)(hs - 1));
  BilinearTap t;
  float fx0 = floorf(ix), fy0 = floorf(iy);
  t.x0 = (int)fx0; t.y0 = (int)fy0; t.x1 = t.x0 + 1; t.y1 = t.y0 + 1;
  t.wx1 = ix - fx0; t.wx0 = (fx0 + 1.f) - ix;
  t.wy1 = iy - fy0; t.wy0 = (fy0 + 1.f) - iy;
  t.vx0 = t.x0 >= 0 && t.x0 < ws; t.vx1 = t.x1 >= 0 && t.x1 < ws;
  t.vy0 = t.y0 >= 0 && t.y0 < hs; t.vy1 = t.y1 >= 0 && t.y1 < hs;
  return t;
}

GV_HD float tap_fetch(const TV& s, int n, const BilinearTap& t, int ch) {
  const float* b = s.p + (int64_t)n * s.sn + ch;
  float v = 0.f;
  if (t.vy0 && t.vx0) v += b[((int64_t)t.y0 * s.w + t.x0) * s.ld] * (t.wx0 * t.wy0);
  if (t.vy0 && t.vx1) v += b[((int64_t)t.y0 * s.w + t.x1) * s.ld] * (t.wx1 * t.wy0);
  if (t.vy1 && t.vx0) v += b[((int64_t)t.y1 * s.w + t.x0) * s.ld] * (t.wx0 * t.wy1);
  if (t.vy1 && t.vx1) v += b[((int64_t)t.y1 * s.w + t.x1) * s.ld] * (t.wx1 * t.wy1);
  return v;
}

// decode a flat index over (n, y, x, c)
struct Idx4 { int n, y, x, c; };
GV_HD Idx4 decode4(int64_t i, int h, int w, int c) {
  Idx4 r;
  r.c = (int)(i % c); i /= c;
  r.x = (int)(i % w); i /= w;
  r.y = (int)(i % h); r.n = (int)(i / h);
  return r;
}

// ------------------------------------------------------------- layout moves
struct NchwToNhwcK {
  const float* src; int64_t sn, sc; TV dst; float scale, shift;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, dst.h, dst.w, dst.c);
    float v = src[(int64_t)q.n * sn + (int64_t)q.c * sc + (int64_t)q.y * dst.w + q.x];
    dst.p[dst.off(q.n, q.y, q.x) + q.c] = v * scale + shift;
  }
};
void nchw_to_nhwc(Ctx& cx, const float* src, int64_t src_sn, int64_t src_sc, const TV& dst, float scale, float shift) {
  parallel_for(cx, dst.pixels() * dst.c, NchwToNhwcK{src, src_sn, src_sc, dst, scale, shift}, "nchw_to_nhwc");
}

struct NhwcToNchwK {
  TV src; float* dst; int64_t sn, sc; float scale, shift; int clamp01;
  GV_HD void operator()(int64_t i) const {
    // iterate in NCHW order so the writes are coalesced
    int x = (int)(i % src.w); int64_t r = i / src.w;
    int y = (int)(r % src.h); r /= src.h;
    int c = (int)(r % src.c); int n = (int)(r / src.c);
    float v = (src.p[src.off(n, y, x) + c] + shift) * scale;
    if (clamp01) v = fminf(fmaxf(v, 0.f), 1.f);
    dst[(int64_t)n * sn + (int64_t)c * sc + (int64_t)y * src.w + x] = v;
  }
};
void nhwc_to_nchw(Ctx& cx, const TV& src, float* dst, int64_t dst_sn, int64_t dst_sc, float scale, float shift, int clamp01) {
  parallel_for(cx, src.pixels() * src.c, NhwcToNchwK{src, dst, dst_sn, dst_sc, scale, shift, clamp01}, "nhwc_to_nchw");
}

// the same with sample n stored at row rows[n] of dst: up to kGatherMax rows per launch, carried in the kernel parameters
struct NhwcToNchwRowsK {
  NhwcToNchwK k; int rows[kGatherMax];
  GV_HD void operator()(int64_t i) const {
    const int64_t per = (int64_t)k.src.c * k.src.h * k.src.w;
    const int n = (int)(i / per);
    NhwcToNchwK s = k;
    s.src.p = k.src.p + (int64_t)n * k.src.sn; s.src.n = 1;
    s.dst = k.dst + (int64_t)rows[n] * k.sn;
    s(i - n * per);
  }
};
static bool consecutive_rows(const TV& src, const std::vector<int>& rows) {   // checks the rows; true: consecutive (the plain store applies)
  if ((int)rows.size() != src.n) throw std::runtime_error("store_rows: one destination row per sample is required");
  for (int r : rows) if (r < 0) throw std::runtime_error("store_rows: negative destination row");
  for (size_t n = 0; n < rows.size(); ++n) if (rows[n] != rows[0] + (int)n) return false;
  return true;
}
void nhwc_to_nchw_rows(Ctx& cx, const TV& src, float* dst, const std::vector<int>& rows, int64_t dst_sn, int64_t dst_sc, float scale, float shift,
                       int clamp01) {
  if (consecutive_rows(src, rows)) return nhwc_to_nchw(cx, src, dst + (int64_t)rows[0] * dst_sn, dst_sn, dst_sc, scale, shift, clamp01);
  for (int n0 = 0; n0 < src.n; n0 += kGatherMax) {
    const int cnt = std::min(src.n - n0, kGatherMax);
    NhwcToNchwRowsK k{};
    k.k = NhwcToNchwK{src.batch(n0, cnt), dst, dst_sn, dst_sc, scale, shift, clamp01};
    for (int i = 0; i < cnt; ++i) k.rows[i] = rows[n0 + i];
    parallel_for(cx, (int64_t)cnt * src.h * src.w * src.c, k, "nhwc_to_nchw_rows");
  }
}

// The pointwise ops below with a 4-channel form are functor templates K<L, Any>: L channels per item, Any = half-aware storage
// (precision mode 4's half tensors).  Each lane's arithmetic is written once; lanes_for picks the width.
template <int L, bool Any> struct CopyK {
  TV src, dst;
  GV_HD void operator()(int64_t i) const {
    const Idx4 q = decode4(i, dst.h, dst.w, dst.c / L);
    float v[L];
    ld_lanes<L, Any>(src, src.off(q.n, q.y, q.x) + q.c * L, v);
    st_lanes<L, Any>(dst, dst.off(q.n, q.y, q.x) + q.c * L, v);
  }
};
void copy_channels(Ctx& cx, const TV& src, const TV& dst) {
  if (src.f16 || dst.f16) { parallel_for(cx, dst.pixels() * dst.c, CopyK<1, true>{src, dst}, "copy_channels"); return; }
  TV s4 = src; s4.c = dst.c;
  lanes_for<CopyK>(cx, vec4_ok(s4) && vec4_ok(dst), dst.pixels() * dst.c, "copy_channels", src, dst);
}

// ---- driver-side pre/post-processing (src/video_Nx.py:40-50,152-153,182-202; src/utils/utils.py:156-185) ----
// uint8 HWC RGB frame -> float32 CHW in [0,1] (x / 255.0) replicate-padded to (H, W): InputPadder.pad
struct FramesU8ToF32K {
  const uint8_t* src; float* dst; int h, w, H, W, pt, pl;
  GV_HD void operator()(int64_t i) const {
    int X = (int)(i % W); int64_t r = i / W; int Y = (int)(r % H); r /= H; int c = (int)(r % 3); int n = (int)(r / 3);
    int y = Y - pt, x = X - pl;
    y = y < 0 ? 0 : (y >= h ? h - 1 : y); x = x < 0 ? 0 : (x >= w ? w - 1 : x);
    dst[i] = (float)src[(((int64_t)n * h + y) * w + x) * 3 + c] / 255.0f;
  }
};
void frames_u8_to_padded_f32(Ctx& cx, const uint8_t* src, int n, int h, int w, float* dst_nchw, int H, int W, int pad_top, int pad_left) {
  parallel_for(cx, (int64_t)n * 3 * H * W, FramesU8ToF32K{src, dst_nchw, h, w, H, W, pad_top, pad_left}, "frames_u8_to_f32");
}
// float32 CHW prediction -> unpadded uint8 HWC, (x * 255.0) truncated like numpy's astype(uint8); optional BGR
struct PredToU8K {
  const float* src; uint8_t* dst; int H, W, h, w, pt, pl, bgr;
  GV_HD void operator()(int64_t i) const {
    int c = (int)(i % 3); int64_t r = i / 3; int x = (int)(r % w); r /= w; int y = (int)(r % h); int n = (int)(r / h);
    int cs = bgr ? 2 - c : c;
    float v = src[(((int64_t)n * 3 + cs) * H + (y + pt)) * W + (x + pl)] * 255.0f;
    v = v < 0.f ? 0.f : (v > 255.f ? 255.f : v);
    dst[i] = (uint8_t)v;
  }
};
void pred_to_u8(Ctx& cx, const float* src_nchw, int n, int H, int W, uint8_t* dst, int h, int w, int pad_top, int pad_left, int bgr) {
  parallel_for(cx, (int64_t)n * h * w * 3, PredToU8K{src_nchw, dst, H, W, h, w, pad_top, pad_left, bgr}, "pred_to_u8");
}

// ---- flow visualisation: the Middlebury colour wheel of src/utils/flow_viz.py (flow_to_image, video_Nx.py:184-189) ----
// numpy mixes precisions there (NEP 50): the normalisation, radius, angle and wheel coordinate are float32, one rounding per
// operation; the interpolation between wheel colours is float64.  Every sum of products below is spelled with explicitly
// rounded operations, so nvcc cannot contract it into an FMA that numpy does not perform.
GV_HD float fv_mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
GV_HD float fv_add(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
GV_HD float fv_div(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
// sample_coord_input (model.sample_coords, CoordSampler3D.shape2coordinate) of n samples at their own t, as (n, hc, wc, 3) (t, y, x),
// and the (n) t vector.  The float32 arithmetic of torch on the device, one rounding per operation: a coordinate is
// lo + span * ((i + 0.5) * (1 / size)) - true division by a host scalar is a product with its float reciprocal there.
struct QueryCoordsK {
  float* coords; float* tout; int hc, wc; float lo, span, ry, rx; float t[kGatherMax];
  GV_HD void operator()(int64_t i) const {
    const int x = (int)(i % wc); int64_t r = i / wc;
    const int y = (int)(r % hc); const int n = (int)(r / hc);
    float* o = coords + i * 3;
    o[0] = t[n];
    o[1] = fv_add(lo, fv_mul(span, fv_mul(fv_add((float)y, 0.5f), ry)));
    o[2] = fv_add(lo, fv_mul(span, fv_mul(fv_add((float)x, 0.5f), rx)));
    if (y == 0 && x == 0) tout[n] = t[n];
  }
};
void query_coords(Ctx& cx, const std::vector<float>& t, int hc, int wc, float lo, float span, float* coords, float* tdev) {
  for (size_t n0 = 0; n0 < t.size(); n0 += kGatherMax) {
    const int cnt = (int)std::min(t.size() - n0, (size_t)kGatherMax);
    QueryCoordsK k{};
    k.coords = coords + (int64_t)n0 * hc * wc * 3; k.tout = tdev + n0; k.hc = hc; k.wc = wc; k.lo = lo; k.span = span;
    k.ry = 1.0f / (float)hc; k.rx = 1.0f / (float)wc;
    for (int i = 0; i < cnt; ++i) k.t[i] = t[n0 + i];
    parallel_for(cx, (int64_t)cnt * hc * wc, k, "query_coords");
  }
}

GV_HD float fv_sqrt(float a) {
#ifdef __CUDA_ARCH__
  return __fsqrt_rn(a);
#else
  return std::sqrt(a);
#endif
}
GV_HD float fv_fma(float a, float b, float c) {   // a * b + c, one rounding on the GPU, two on the host (no contraction there)
#ifdef __CUDA_ARCH__
  return __fmaf_rn(a, b, c);
#else
  return a * b + c;
#endif
}
GV_HD double fv_dmul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
GV_HD double fv_dadd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
// make_colorwheel(): 55 colours in six ramps (RY 15, YG 6, GC 4, CB 11, BM 13, MR 6); floor(255 * j / n) is the integer quotient
GV_HD int fv_wheel(int k, int ch) {
  int r, g, b;
  if (k < 15) { r = 255; g = 255 * k / 15; b = 0; }
  else if (k < 21) { r = 255 - 255 * (k - 15) / 6; g = 255; b = 0; }
  else if (k < 25) { r = 0; g = 255; b = 255 * (k - 21) / 4; }
  else if (k < 36) { r = 0; g = 255 - 255 * (k - 25) / 11; b = 255; }
  else if (k < 49) { r = 255 * (k - 36) / 13; g = 0; b = 255; }
  else { r = 255; g = 0; b = 255 - 255 * (k - 49) / 6; }
  return ch == 0 ? r : (ch == 1 ? g : b);
}
// (u, v) of flow pixel (n, y, x), np.clip(flow, 0, clip) applied when has_clip (negative components become +0, -0.0 stays -0.0)
GV_HD void fv_load(const FlowView& f, int n, int y, int x, int has_clip, float clip, float& u, float& v) {
  const float* p = f.p + (int64_t)n * f.sn + (int64_t)y * f.sy + (int64_t)x * f.sx;
  u = p[0]; v = p[f.sc];
  if (has_clip) {
    u = u < 0.f ? 0.f : (u > clip ? clip : u);
    v = v < 0.f ? 0.f : (v > clip ? clip : v);
  }
}
GV_HD float fv_rad(float u, float v) { return fv_sqrt(fv_add(fv_mul(u, u), fv_mul(v, v))); }

// step 1: max of the radius per row -> rowmax[n * h + y]; step 2: per image -> div[n] = fl32(max + fl32(1e-5))
struct FlowRowMaxK {
  FlowView f; int has_clip; float clip; float* rowmax;
  GV_HD void operator()(int64_t row) const {
    const int n = (int)(row / f.h), y = (int)(row % f.h);
    float m = 0.f, u, v;
    for (int x = 0; x < f.w; ++x) { fv_load(f, n, y, x, has_clip, clip, u, v); m = fmaxf(m, fv_rad(u, v)); }
    rowmax[row] = m;
  }
};
struct FlowImageMaxK {
  const float* rowmax; float* div; int h;
  GV_HD void operator()(int64_t n) const {
    float m = 0.f;
    for (int y = 0; y < h; ++y) m = fmaxf(m, rowmax[n * h + y]);
    div[n] = fv_add(m, 1e-5f);
  }
};
#ifndef GV_HOSTSIM
// GPU form of the two reductions: one CTA per row (resp. image), warp shuffles, no atomics: the result is independent of the order
__device__ __forceinline__ float fv_block_max(float m, float* red) {
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
  if (threadIdx.x < 32)
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __syncthreads();
  return m;
}
__global__ void __launch_bounds__(256) flow_rowmax_kernel(FlowView f, int has_clip, float clip, float* __restrict__ rowmax) {
  __shared__ float red[8];
  const int64_t rows = (int64_t)f.n * f.h;
  for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const int n = (int)(row / f.h), y = (int)(row % f.h);
    float m = 0.f, u, v;
    for (int x = threadIdx.x; x < f.w; x += blockDim.x) { fv_load(f, n, y, x, has_clip, clip, u, v); m = fmaxf(m, fv_rad(u, v)); }
    m = fv_block_max(m, red);
    if (threadIdx.x == 0) rowmax[row] = m;
  }
}
__global__ void __launch_bounds__(256) flow_imagemax_kernel(const float* __restrict__ rowmax, float* __restrict__ div, int h) {
  __shared__ float red[8];
  const int n = blockIdx.x;
  float m = 0.f;
  for (int y = threadIdx.x; y < h; y += blockDim.x) m = fmaxf(m, rowmax[(int64_t)n * h + y]);
  m = fv_block_max(m, red);
  if (threadIdx.x == 0) div[n] = __fadd_rn(m, 1e-5f);
}
#endif

// step 3: flow_uv_to_colors, one thread per pixel -> dst (n,h,w,3) uint8
struct FlowColourK {
  FlowView f; int has_clip; float clip; const float* div; float div_const; int bgr; uint8_t* dst;
  GV_HD void operator()(int64_t i) const {
    const int x = (int)(i % f.w); const int64_t r = i / f.w; const int y = (int)(r % f.h), n = (int)(r / f.h);
    float u, v;
    fv_load(f, n, y, x, has_clip, clip, u, v);
    const float m = div ? div[n] : div_const;
    u = fv_div(u, m); v = fv_div(v, m);
    const float rad = fv_rad(u, v);
    // numpy's float32 arctan2 is not correctly rounded: the double result rounded once is the faithful value.  -v of v = +0.0 is
    // -0.0, so atan2 gives -pi (wheel index 0) there and +pi (index 54) for v = -0.0.
    const float a = fv_div((float)atan2(-(double)v, -(double)u), 3.14159265358979323846f);
    const float fk = fv_mul(fv_div(fv_add(a, 1.f), 2.f), 54.f);
    const int k0 = (int)floorf(fk);
    const int k1 = k0 + 1 == 55 ? 0 : k0 + 1;
    const double fr = (double)fk - (double)k0, omf = fv_dadd(1.0, -fr);
    uint8_t* o = dst + i * 3;
    for (int ch = 0; ch < 3; ++ch) {
      const double c0 = (double)fv_wheel(k0, ch) / 255.0, c1 = (double)fv_wheel(k1, ch) / 255.0;
      double col = fv_dadd(fv_dmul(omf, c0), fv_dmul(fr, c1));
      col = rad <= 1.f ? fv_dadd(1.0, -fv_dmul((double)rad, fv_dadd(1.0, -col))) : fv_dmul(col, 0.75);
      o[bgr ? 2 - ch : ch] = (uint8_t)floor(fv_dmul(255.0, col));
    }
  }
};

int64_t flow_to_image_scratch_floats(int n, int h) { return (int64_t)n * h + n; }
void flow_to_image(Ctx& cx, const FlowView& f, int has_clip, float clip, int has_max, float max_div, int bgr, float* scratch, uint8_t* dst) {
  if (f.n <= 0 || f.h <= 0 || f.w <= 0) return;
  const float* div = nullptr;
  if (!has_max) {
    float* rowmax = scratch;
    float* d = scratch + (int64_t)f.n * f.h;
#ifdef GV_HOSTSIM
    parallel_for(cx, (int64_t)f.n * f.h, FlowRowMaxK{f, has_clip, clip, rowmax}, "flow_rowmax");
    parallel_for(cx, f.n, FlowImageMaxK{rowmax, d, f.h}, "flow_imagemax");
#else
    if (!cx.dry) {
      const int64_t rows = (int64_t)f.n * f.h;
      const int64_t cap = (int64_t)cx.sm_count * 16;
      cx.launches += 2;
      if (cx.prof) cx.prof->begin(cx.stream, "flow_rowmax", (double)rows * f.w * 2.0);
      flow_rowmax_kernel<<<(unsigned)(rows < cap ? rows : cap), 256, 0, cx.stream>>>(f, has_clip, clip, rowmax);
      gv_check_launch("flow_rowmax");
      if (cx.prof) cx.prof->end(cx.stream);
      flow_imagemax_kernel<<<(unsigned)f.n, 256, 0, cx.stream>>>(rowmax, d, f.h);
      gv_check_launch("flow_imagemax");
    }
#endif
    div = d;
  }
  parallel_for(cx, (int64_t)f.n * f.h * f.w, FlowColourK{f, has_clip, clip, div, max_div, bgr, dst}, "flow_colour");
}

// ---- forward_interpolate (raft/utils/utils.py:33-63, flowformer/core/utils/utils.py:35-65): the warm start of the next pair ----
// Source pixel k = (i, j) of a (2,h,w) flow lands at x1 = j + dx, y1 = i + dy, in float64 as numpy promotes int64 + float32; it is valid
// iff 0 < x1 < w and 0 < y1 < h (strict; NaN never is).  Output pixel (qx, qy) takes the (dx, dy) of the nearest valid source, as
// scipy's griddata(method="nearest") does: squared distance rn(rn(ddx^2) + rn(ddy^2)) in float64, x term first, every operation rounded
// on its own (no FMA contraction).  Ties go to the smallest source index; scipy's KD-tree picks among them in its own traversal order,
// the one defined difference.  Without a valid source every output is NaN, as griddata gives.  A brute-force scan in index order: exact
// and deterministic, no workspace.
GV_HD bool fi_source(const float* f, int h, int w, int64_t k, double& x1, double& y1) {
  const int i = (int)(k / w), j = (int)(k % w);
  x1 = fv_dadd((double)j, (double)f[k]);
  y1 = fv_dadd((double)i, (double)f[(int64_t)h * w + k]);
  return x1 > 0.0 && x1 < (double)w && y1 > 0.0 && y1 < (double)h;
}
GV_HD double fi_dist(double x1, double y1, double qx, double qy) {
  const double ddx = fv_dadd(x1, -qx), ddy = fv_dadd(y1, -qy);
  return fv_dadd(fv_dmul(ddx, ddx), fv_dmul(ddy, ddy));
}
// output pixel q of one image: the chosen source's (dx, dy), NaN without one
GV_HD void fi_write(const float* f, float* o, int64_t hw, int64_t q, int64_t best) {
  o[q] = best < 0 ? NAN : f[best];
  o[hw + q] = best < 0 ? NAN : f[hw + best];
}
#ifdef GV_HOSTSIM
struct ForwardInterpK {   // one output pixel per item, every source read from the flow
  const float* flow; float* out; int h, w;
  GV_HD void operator()(int64_t i) const {
    const int64_t hw = (int64_t)h * w, n = i / hw, q = i % hw;
    const float* f = flow + n * 2 * hw;
    const double qx = (double)(q % w), qy = (double)(q / w);
    double best_d = INFINITY; int64_t best = -1;
    for (int64_t k = 0; k < hw; ++k) {
      double x1, y1;
      if (!fi_source(f, h, w, k, x1, y1)) continue;
      const double d = fi_dist(x1, y1, qx, qy);
      if (d < best_d) { best_d = d; best = k; }
    }
    fi_write(f, out + n * 2 * hw, hw, q, best);
  }
};
#else
constexpr int kFiThreads = 128;
// one thread per output pixel, blockIdx.y = image; the sources pass through shared memory one tile of kFiThreads at a time, an invalid
// source stored as x1 = NaN (its distance is NaN, never below the best)
__global__ void __launch_bounds__(kFiThreads) forward_interp_kernel(const float* __restrict__ flow, float* __restrict__ out, int h, int w) {
  __shared__ double sx[kFiThreads], sy[kFiThreads];
  const int64_t hw = (int64_t)h * w, q = (int64_t)blockIdx.x * kFiThreads + threadIdx.x;
  const float* f = flow + (int64_t)blockIdx.y * 2 * hw;
  const double qx = (double)(q % w), qy = (double)(q / w);
  double best_d = INFINITY; int64_t best = -1;
  for (int64_t k0 = 0; k0 < hw; k0 += kFiThreads) {
    const int64_t k = k0 + threadIdx.x;
    double x1 = NAN, y1 = NAN;
    if (k < hw && !fi_source(f, h, w, k, x1, y1)) x1 = NAN;
    sx[threadIdx.x] = x1; sy[threadIdx.x] = y1;
    __syncthreads();
    const int m = hw - k0 < kFiThreads ? (int)(hw - k0) : kFiThreads;
#pragma unroll 4
    for (int t = 0; t < m; ++t) {
      const double d = fi_dist(sx[t], sy[t], qx, qy);
      if (d < best_d) { best_d = d; best = k0 + t; }
    }
    __syncthreads();
  }
  if (q < hw) fi_write(f, out + (int64_t)blockIdx.y * 2 * hw, hw, q, best);
}
#endif

void forward_interpolate(Ctx& cx, const float* flow, int n, int h, int w, float* out) {
  if (n <= 0 || h <= 0 || w <= 0) return;
  const int64_t hw = (int64_t)h * w;
#ifdef GV_HOSTSIM
  parallel_for(cx, n * hw, ForwardInterpK{flow, out, h, w}, "forward_interpolate");
#else
  if (cx.dry) return;
  cx.launches++;
  if (cx.prof) cx.prof->begin(cx.stream, "forward_interpolate", (double)n * hw * hw);
  forward_interp_kernel<<<dim3((unsigned)((hw + kFiThreads - 1) / kFiThreads), (unsigned)n), kFiThreads, 0, cx.stream>>>(flow, out, h, w);
  gv_check_launch("forward_interpolate");
  if (cx.prof) cx.prof->end(cx.stream);
#endif
}

// zero-padded copy of a 3-channel image stored with 4-float pixels (4th lane forced to 0)
struct PadImage4K {
  TV src, dst; int pad;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, dst.h, dst.w, 4);
    int y = q.y - pad, x = q.x - pad;
    float v = 0.f;
    if (q.c < 3 && y >= 0 && y < src.h && x >= 0 && x < src.w) v = src.p[src.off(q.n, y, x) + q.c];
    dst.p[dst.off(q.n, q.y, q.x) + q.c] = v;
  }
};
void pad_image4(Ctx& cx, const TV& src, const TV& dst, int pad) {
  parallel_for(cx, dst.pixels() * 4, PadImage4K{src, dst, pad}, "pad_image4");
}

// reflect-padded copy (padding_mode="reflect"): lets the tensor-core conv, whose TMA can only zero-fill, run the
// reflect-padded layers (gimmvfi_r.py:94-96,106-108) as a "valid" conv on the padded buffer
template <int L, bool Any> struct PadReflectK {
  TV src, dst; int pad;
  GV_HD static int refl(int v, int n) { return v < 0 ? -v : (v >= n ? 2 * n - 2 - v : v); }
  GV_HD void operator()(int64_t i) const {
    const Idx4 q = decode4(i, dst.h, dst.w, dst.c / L);
    const int y = refl(q.y - pad, src.h), x = refl(q.x - pad, src.w);
    float v[L];
    ld_lanes<L, Any>(src, src.off(q.n, y, x) + q.c * L, v);
    st_lanes<L, Any>(dst, dst.off(q.n, q.y, q.x) + q.c * L, v);
  }
};
void pad_reflect(Ctx& cx, const TV& src, const TV& dst, int pad) {
  if (src.f16 != dst.f16) throw std::runtime_error("pad_reflect: source and destination must have the same storage type");
  if (src.f16) {
    // a pure copy: two half channels are one 32-bit element, so an even-strided half tensor is an fp32 tensor of half the width
    auto even = [](const TV& t) { return t.c % 2 == 0 && t.ld % 2 == 0 && t.sn % 2 == 0; };
    auto pairs = [](TV t) { t.f16 = 0; t.c /= 2; t.ld /= 2; t.sn /= 2; return t; };
    const TV s2 = pairs(src), d2 = pairs(dst);
    if (even(src) && even(dst) && vec4_ok(s2) && vec4_ok(d2)) parallel_for(cx, d2.pixels() * (d2.c / 4), PadReflectK<4, false>{s2, d2, pad}, "pad_reflect");
    else parallel_for(cx, dst.pixels() * dst.c, PadReflectK<1, true>{src, dst, pad}, "pad_reflect");
    return;
  }
  lanes_for<PadReflectK>(cx, vec4_ok(src) && vec4_ok(dst), dst.pixels() * dst.c, "pad_reflect", src, dst, pad);
}

// zero-padded copy: dst (n, h+2p, w+2p) gets src's channels in its interior, zeros elsewhere (all dst.ld lanes)
template <int L, bool Any> struct PadZeroK {
  TV src, dst; int pad;
  GV_HD void operator()(int64_t i) const {
    const Idx4 q = decode4(i, dst.h, dst.w, dst.ld / L);
    const int y = q.y - pad, x = q.x - pad, c0 = q.c * L;
    float v[L];
    for (int k = 0; k < L; ++k) v[k] = 0.f;
    if (c0 < src.c && y >= 0 && y < src.h && x >= 0 && x < src.w) {
      ld_lanes<L, Any>(src, src.off(q.n, y, x) + c0, v);   // (c0 + L - 1 < src.ld: the 4-lane form needs ((src.c + 3) & ~3) <= src.ld)
      for (int k = 1; k < L; ++k)
        if (c0 + k >= src.c) v[k] = 0.f;
    }
    st_lanes<L, Any>(dst, dst.off(q.n, q.y, q.x) + c0, v);
  }
};
void pad_zero(Ctx& cx, const TV& src, const TV& dst, int pad) {
  const bool four = lanes4_ok(src) && lanes4_ok(dst) && !src.f16 && !dst.f16 && ((src.c + 3) & ~3) <= src.ld;
  lanes_for<PadZeroK>(cx, four, dst.pixels() * dst.ld, "pad_zero", src, dst, pad);
}

struct FillK {
  TV dst; float v;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, dst.h, dst.w, dst.c);
    dst.p[dst.off(q.n, q.y, q.x) + q.c] = v;
  }
};
void fill(Ctx& cx, const TV& dst, float v) { parallel_for(cx, dst.pixels() * dst.c, FillK{dst, v}, "fill"); }

template <int A> struct HypoActK {
  TV x; float w0;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, x.h, x.w, x.c);
    float* p = x.p + x.off(q.n, q.y, q.x) + q.c;
    *p = hypo_act<A>(*p, w0);
  }
};
void hypo_activation(Ctx& cx, const TV& x, int act, float w0) {
  const int64_t n = x.pixels() * x.c;
  switch (act) {
    case HYPO_SIREN1: parallel_for(cx, n, HypoActK<HYPO_SIREN1>{x, w0}, "hypo_activation"); break;
    case HYPO_SIREN: parallel_for(cx, n, HypoActK<HYPO_SIREN>{x, w0}, "hypo_activation"); break;
    case HYPO_RELU: parallel_for(cx, n, HypoActK<HYPO_RELU>{x, w0}, "hypo_activation"); break;
    case HYPO_SILU: parallel_for(cx, n, HypoActK<HYPO_SILU>{x, w0}, "hypo_activation"); break;
    case HYPO_DAMP: parallel_for(cx, n, HypoActK<HYPO_DAMP>{x, w0}, "hypo_activation"); break;
    default: throw std::runtime_error("hypo_activation: unknown activation");
  }
}

struct AxpbyK {
  TV a, b, out; float alpha, beta;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, out.h, out.w, out.c);
    float v = alpha * a.p[a.off(q.n, q.y, q.x) + q.c];
    if (b.p) v += beta * b.p[b.off(q.n, q.y, q.x) + q.c];
    out.p[out.off(q.n, q.y, q.x) + q.c] = v;
  }
};
void axpby(Ctx& cx, const TV& a, float alpha, const TV& b, float beta, const TV& out) {
  parallel_for(cx, out.pixels() * out.c, AxpbyK{a, b, out, alpha, beta}, "axpby");
}

// ------------------------------------------------------------------ resize
// F.interpolate(mode="bilinear", align_corners=False) — modules/fi_utils.py:67-70.
// src coordinate = rscale * (dst + 0.5) - 0.5 clamped at 0 (ATen area_pixel_compute_source_index).
template <int L, bool Any> struct ResizeK {
  TV src, dst; float rsy, rsx, mult; int accumulate, act;
  GV_HD void operator()(int64_t i) const {
    const Idx4 q = decode4(i, dst.h, dst.w, dst.c / L);
    float sy = rsy * ((float)q.y + 0.5f) - 0.5f; if (sy < 0.f) sy = 0.f;
    float sx = rsx * ((float)q.x + 0.5f) - 0.5f; if (sx < 0.f) sx = 0.f;
    int y0 = (int)sy, x0 = (int)sx;
    if (y0 > src.h - 1) y0 = src.h - 1;
    if (x0 > src.w - 1) x0 = src.w - 1;
    int y1 = y0 + (y0 < src.h - 1 ? 1 : 0), x1 = x0 + (x0 < src.w - 1 ? 1 : 0);
    float ly1 = sy - (float)y0, lx1 = sx - (float)x0;
    float ly0 = 1.f - ly1, lx0 = 1.f - lx1;
    const int64_t b = (int64_t)q.n * src.sn + q.c * L;
    float v00[L], v01[L], v10[L], v11[L];
    ld_lanes<L, Any>(src, b + ((int64_t)y0 * src.w + x0) * src.ld, v00); ld_lanes<L, Any>(src, b + ((int64_t)y0 * src.w + x1) * src.ld, v01);
    ld_lanes<L, Any>(src, b + ((int64_t)y1 * src.w + x0) * src.ld, v10); ld_lanes<L, Any>(src, b + ((int64_t)y1 * src.w + x1) * src.ld, v11);
    const int64_t o = dst.off(q.n, q.y, q.x) + q.c * L;
    float old[L];
    if (accumulate) ld_lanes<L, Any>(dst, o, old);
    float r[L];
    for (int k = 0; k < L; ++k) {
      // ly0 * (lx0 * v00 + lx1 * v01) + ly1 * (lx0 * v10 + lx1 * v11) with the GPU's FMA contraction spelled out (the lx1 and ly0
      // terms fused), as both widths have always computed it: nvcc may fuse either product of a sum, and left alone it chose
      // differently for the two widths
      const float r0 = fv_fma(lx1, v01[k], fv_mul(lx0, v00[k])), r1 = fv_fma(lx1, v11[k], fv_mul(lx0, v10[k]));
      float v = fv_fma(ly0, r0, fv_mul(ly1, r1));
      v = fv_mul(v, mult);
      if (act == ACT_SIGMOID) v = 1.f / (1.f + expf(-v));
      r[k] = accumulate ? (old[k] + v) : v;
    }
    st_lanes<L, Any>(dst, o, r);
  }
};
// The half-aware form (precision mode 4's concat buffers): the same arithmetic, kept as its own functor because the ResizeK<4, true>
// instance of the template above compiled to a different load schedule that measured slower on the full-resolution 4K concat
struct ResizeAnyK4 {
  TV src, dst; float rsy, rsx, mult; int act;
  GV_HD float fin(float v00, float v01, float v10, float v11, float lx0, float lx1, float ly0, float ly1) const {
    float v = ly0 * (lx0 * v00 + lx1 * v01) + ly1 * (lx0 * v10 + lx1 * v11);
    v *= mult;
    if (act == ACT_SIGMOID) v = 1.f / (1.f + expf(-v));
    return v;
  }
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, dst.h, dst.w, dst.c / 4);
    float sy = rsy * ((float)q.y + 0.5f) - 0.5f; if (sy < 0.f) sy = 0.f;
    float sx = rsx * ((float)q.x + 0.5f) - 0.5f; if (sx < 0.f) sx = 0.f;
    int y0 = (int)sy, x0 = (int)sx;
    if (y0 > src.h - 1) y0 = src.h - 1;
    if (x0 > src.w - 1) x0 = src.w - 1;
    int y1 = y0 + (y0 < src.h - 1 ? 1 : 0), x1 = x0 + (x0 < src.w - 1 ? 1 : 0);
    float ly1 = sy - (float)y0, lx1 = sx - (float)x0;
    float ly0 = 1.f - ly1, lx0 = 1.f - lx1;
    const int64_t b = (int64_t)q.n * src.sn + q.c * 4;
    const F4 a00 = ld4v(src, b + ((int64_t)y0 * src.w + x0) * src.ld), a01 = ld4v(src, b + ((int64_t)y0 * src.w + x1) * src.ld);
    const F4 a10 = ld4v(src, b + ((int64_t)y1 * src.w + x0) * src.ld), a11 = ld4v(src, b + ((int64_t)y1 * src.w + x1) * src.ld);
    F4 r;
    r.x = fin(a00.x, a01.x, a10.x, a11.x, lx0, lx1, ly0, ly1); r.y = fin(a00.y, a01.y, a10.y, a11.y, lx0, lx1, ly0, ly1);
    r.z = fin(a00.z, a01.z, a10.z, a11.z, lx0, lx1, ly0, ly1); r.w = fin(a00.w, a01.w, a10.w, a11.w, lx0, lx1, ly0, ly1);
    st4v(dst, dst.off(q.n, q.y, q.x) + q.c * 4, r);
  }
};
void resize_bilinear(Ctx& cx, const TV& src, const TV& dst, float rscale_y, float rscale_x, float mult, int accumulate, int act) {
  TV s4 = src; s4.c = dst.c;
  if (src.f16 || dst.f16) {
    if (accumulate || !vec4_ok_any(s4) || !vec4_ok_any(dst)) throw std::runtime_error("resize_bilinear: half-precision tensors need 4-channel-aligned views and no accumulation");
    parallel_for(cx, dst.pixels() * (dst.c / 4), ResizeAnyK4{src, dst, rscale_y, rscale_x, mult, act}, "resize_bilinear");
    return;
  }
  lanes_for<ResizeK>(cx, vec4_ok(s4) && vec4_ok(dst), dst.pixels() * dst.c, "resize_bilinear", src, dst, rscale_y, rscale_x, mult, accumulate, act);
}

// ---------------------------------------------------------------- backwarp
// modules/fi_utils.py:19-49.  The four corners in tap_fetch's order and products.
template <int L, bool Any> struct BackwarpK {
  TV src, flow, dst;
  GV_HD void corner(float* v, int64_t eoff, float w) const {
    float a[L];
    ld_lanes<L, Any>(src, eoff, a);
    for (int k = 0; k < L; ++k) v[k] += a[k] * w;
  }
  GV_HD void operator()(int64_t i) const {
    const Idx4 q = decode4(i, dst.h, dst.w, dst.c / L);
    const float* f = flow.p + flow.off(q.n, q.y, q.x);
    const BilinearTap t = border_tap(q.x, q.y, f[0], f[1], flow.w, flow.h, src.w, src.h);
    const int64_t b = (int64_t)q.n * src.sn + q.c * L;
    float v[L];
    for (int k = 0; k < L; ++k) v[k] = 0.f;
    if (t.vy0 && t.vx0) corner(v, b + ((int64_t)t.y0 * src.w + t.x0) * src.ld, t.wx0 * t.wy0);
    if (t.vy0 && t.vx1) corner(v, b + ((int64_t)t.y0 * src.w + t.x1) * src.ld, t.wx1 * t.wy0);
    if (t.vy1 && t.vx0) corner(v, b + ((int64_t)t.y1 * src.w + t.x0) * src.ld, t.wx0 * t.wy1);
    if (t.vy1 && t.vx1) corner(v, b + ((int64_t)t.y1 * src.w + t.x1) * src.ld, t.wx1 * t.wy1);
    st_lanes<L, Any>(dst, dst.off(q.n, q.y, q.x) + q.c * L, v);
  }
};
void backwarp(Ctx& cx, const TV& src, const TV& flow, const TV& dst) {
  if (flow.f16) throw std::runtime_error("backwarp: the flow field must be fp32");
  TV s4 = src; s4.c = dst.c;
  if (src.f16 || dst.f16) lanes_for<BackwarpK, true>(cx, vec4_ok_any(s4) && vec4_ok_any(dst), dst.pixels() * dst.c, "backwarp", src, flow, dst);
  else lanes_for<BackwarpK>(cx, vec4_ok(s4) && vec4_ok(dst), dst.pixels() * dst.c, "backwarp", src, flow, dst);
}

// ----------------------------------------------------------- pixel shuffle
// nn.PixelShuffle(2) applied `times` times (fi_components.py:235, :285-286).
struct PixelShuffleK {
  TV src, dst; int times;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, dst.h, dst.w, dst.c);
    int y = q.y, x = q.x, c = q.c;
    for (int k = 0; k < times; ++k) {
      c = c * 4 + (y & 1) * 2 + (x & 1);
      y >>= 1; x >>= 1;
    }
    dst.p[dst.off(q.n, q.y, q.x) + q.c] = src.p[src.off(q.n, y, x) + c];
  }
};
void pixel_shuffle(Ctx& cx, const TV& src, const TV& dst, int times) {
  parallel_for(cx, dst.pixels() * dst.c, PixelShuffleK{src, dst, times}, "pixel_shuffle");
}

// ----------------------------------------------------------- instance norm
// nn.InstanceNorm2d(C): no affine, biased variance, eps 1e-5 (raft/extractor.py:30-34,133-134).
static const int IN_CHUNKS_MAX = 1024;
static int in_chunks(const TV& x) {  // ~64 pixels per thread, enough threads to fill 132 SMs
  int64_t hw = (int64_t)x.h * x.w; int64_t c = hw / 64;
  return (int)(c < 1 ? 1 : (c > IN_CHUNKS_MAX ? IN_CHUNKS_MAX : c));
}
int64_t instnorm_scratch_floats(const TV& x) { return (int64_t)x.n * (IN_CHUNKS_MAX + 32) * x.c * 4; }

struct InPartialK {
  TV x; double* part; int chunks;
  GV_HD void operator()(int64_t i) const {
    int c = (int)(i % x.c); int64_t r = i / x.c;
    int ch = (int)(r % chunks); int n = (int)(r / chunks);
    int64_t hw = (int64_t)x.h * x.w;
    int64_t per = (hw + chunks - 1) / chunks;
    int64_t a = (int64_t)ch * per, b = a + per; if (b > hw) b = hw;
    const float* p = x.p + (int64_t)n * x.sn + c;
    // four independent accumulator pairs: four loads in flight per thread (the single dependent chain was latency bound)
    double s = 0.0, s2 = 0.0, t = 0.0, t2 = 0.0, u = 0.0, u2 = 0.0, w = 0.0, w2 = 0.0;
    int64_t k = a;
    for (; k + 3 < b; k += 4) {
      const double v0 = (double)p[k * x.ld], v1 = (double)p[(k + 1) * x.ld], v2 = (double)p[(k + 2) * x.ld], v3 = (double)p[(k + 3) * x.ld];
      s += v0; s2 += v0 * v0; t += v1; t2 += v1 * v1; u += v2; u2 += v2 * v2; w += v3; w2 += v3 * v3;
    }
    for (; k < b; ++k) { const double v = (double)p[k * x.ld]; s += v; s2 += v * v; }
    part[i * 2] = (s + t) + (u + w); part[i * 2 + 1] = (s2 + t2) + (u2 + w2);
  }
};
// two-level tree over the chunk partials (a single thread per (n,c) looping over 1024 chunks was latency bound)
struct InFoldK {   // part[n][chunks][c] -> fold[n][32][c]
  const double* part; double* fold; int c, chunks;
  GV_HD void operator()(int64_t i) const {
    int ch = (int)(i % c); int64_t r = i / c; int g = (int)(r % 32); int n = (int)(r / 32);
    double s = 0.0, s2 = 0.0;
    for (int k = g; k < chunks; k += 32) { int64_t j = ((int64_t)n * chunks + k) * c + ch; s += part[j * 2]; s2 += part[j * 2 + 1]; }
    fold[i * 2] = s; fold[i * 2 + 1] = s2;
  }
};
struct InFinalK {
  const double* fold; float* mr; int c; double inv_hw;
  GV_HD void operator()(int64_t i) const {
    int ch = (int)(i % c); int n = (int)(i / c);
    double s = 0.0, s2 = 0.0;
    for (int g = 0; g < 32; ++g) { int64_t j = ((int64_t)n * 32 + g) * c + ch; s += fold[j * 2]; s2 += fold[j * 2 + 1]; }
    double m = s * inv_hw; double var = s2 * inv_hw - m * m; if (var < 0.0) var = 0.0;
    mr[i * 2] = (float)m; mr[i * 2 + 1] = (float)(1.0 / sqrt(var + 1e-5));
  }
};
void instnorm_stats(Ctx& cx, const TV& x, float* mean_rstd, float* scratch, int64_t) {
  double* part = reinterpret_cast<double*>(scratch);
  const int chunks = in_chunks(x);
  double* fold = part + (int64_t)x.n * IN_CHUNKS_MAX * x.c * 2;
  parallel_for(cx, (int64_t)x.n * chunks * x.c, InPartialK{x, part, chunks}, "instnorm_partial");
  parallel_for(cx, (int64_t)x.n * 32 * x.c, InFoldK{part, fold, x.c, chunks}, "instnorm_fold");
  parallel_for(cx, (int64_t)x.n * x.c, InFinalK{fold, mean_rstd, x.c, 1.0 / ((double)x.h * x.w)}, "instnorm_final");
}
template <int L, bool Any> struct InApplyK {
  TV x, res, out; const float* mr; int act1, act2;
  GV_HD void operator()(int64_t i) const {
    const Idx4 q = decode4(i, out.h, out.w, out.c / L);
    const int c = q.c * L;
    const float* s = mr + ((int64_t)q.n * x.c + c) * 2;
    float sm[2 * L];   // (mean, rstd) pairs of the L channels
    ld_lanes<L>(s, sm); ld_lanes<L>(s + L, sm + L);
    float a[L], rv[L], o[L];
    ld_lanes<L, Any>(x, x.off(q.n, q.y, q.x) + c, a);
    if (res.p) ld_lanes<L, Any>(res, res.off(q.n, q.y, q.x) + c, rv);
    for (int k = 0; k < L; ++k) {
      float v = (a[k] - sm[2 * k]) * sm[2 * k + 1];
      v = apply_act(v, act1, nullptr, 0);
      if (res.p) v += rv[k];
      o[k] = apply_act(v, act2, nullptr, 0);
    }
    st_lanes<L, Any>(out, out.off(q.n, q.y, q.x) + c, o);
  }
};
void instnorm_apply(Ctx& cx, const TV& x, const float* mean_rstd, int act1, const TV& res, int act2, const TV& out) {
  const bool four = vec4_ok(x) && vec4_ok(out) && (!res.p || vec4_ok(res)) && aligned(mean_rstd, 16) && x.c == out.c;
  lanes_for<InApplyK>(cx, four, out.pixels() * out.c, "instnorm_apply", x, res, out, mean_rstd, act1, act2);
}

// ------------------------------------------------------- flow normalisation
// modules/fi_utils.py:52-60: scaler[n] = max |cat[f01, -f10]|.
static const int AM_CHUNKS = 4096;
int64_t absmax_scratch_floats(const TV& a) { return (int64_t)a.n * AM_CHUNKS; }
struct AbsmaxPartK {
  TV a, b; float* part; int chunks;
  GV_HD void operator()(int64_t i) const {
    int ch = (int)(i % chunks); int n = (int)(i / chunks);
    int64_t hw = (int64_t)a.h * a.w; int64_t per = (hw + chunks - 1) / chunks;
    int64_t s = (int64_t)ch * per, e = s + per; if (e > hw) e = hw;
    float m = 0.f;
    for (int64_t k = s; k < e; ++k) {
      const float* pa = a.p + (int64_t)n * a.sn + k * a.ld;
      const float* pb = b.p + (int64_t)n * b.sn + k * b.ld;
      for (int c = 0; c < a.c; ++c) { m = fmaxf(m, fabsf(pa[c])); m = fmaxf(m, fabsf(pb[c])); }
    }
    part[i] = m;
  }
};
struct AbsmaxFinK {
  const float* part; float* out; int chunks;
  GV_HD void operator()(int64_t n) const {
    float m = 0.f; for (int k = 0; k < chunks; ++k) m = fmaxf(m, part[n * chunks + k]);
    out[n] = m;
  }
};
void absmax_per_sample(Ctx& cx, const TV& a, const TV& b, float* out_n, float* scratch) {
  parallel_for(cx, (int64_t)a.n * AM_CHUNKS, AbsmaxPartK{a, b, scratch, AM_CHUNKS}, "absmax_partial");
  parallel_for(cx, (int64_t)a.n, AbsmaxFinK{scratch, out_n, AM_CHUNKS}, "absmax_final");
}

struct NormFlowK {
  TV f01, f10, n0, n1; const float* s;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, f01.h, f01.w, 2);
    float sc = s[q.n];
    float a = f01.p[f01.off(q.n, q.y, q.x) + q.c];
    float b = -f10.p[f10.off(q.n, q.y, q.x) + q.c];
    n0.p[n0.off(q.n, q.y, q.x) + q.c] = (a / sc + 1.0f) / 2.0f;
    n1.p[n1.off(q.n, q.y, q.x) + q.c] = (b / sc + 1.0f) / 2.0f;
  }
};
void normalize_flow_pair(Ctx& cx, const TV& f01, const TV& f10, const float* scaler, const TV& n0, const TV& n1) {
  parallel_for(cx, f01.pixels() * 2, NormFlowK{f01, f10, n0, n1, scaler}, "normalize_flow");
}

struct UnnormK {
  TV a, out; const float* s;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, out.h, out.w, out.c);
    out.p[out.off(q.n, q.y, q.x) + q.c] = (a.p[a.off(q.n, q.y, q.x) + q.c] * 2.0f - 1.0f) * s[q.n];
  }
};
void unnormalize_flow(Ctx& cx, const TV& ninr, const float* scaler, const TV& out) {
  parallel_for(cx, out.pixels() * out.c, UnnormK{ninr, out, scaler}, "unnormalize_flow");
}

// ------------------------------------------------------ RAFT coordinate ops
struct InitCoordsK {
  TV c;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, c.h, c.w, 2);
    c.p[c.off(q.n, q.y, q.x) + q.c] = q.c == 0 ? (float)q.x : (float)q.y;
  }
};
void init_coords(Ctx& cx, const TV& coords) { parallel_for(cx, coords.pixels() * 2, InitCoordsK{coords}, "init_coords"); }

// flow = coords1 - coords0 (raft/raft.py:148), written to up to two consumers.
struct CoordsMinusGridK {
  TV c, a, b;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, c.h, c.w, 2);
    float v = c.p[c.off(q.n, q.y, q.x) + q.c] - (q.c == 0 ? (float)q.x : (float)q.y);
    if (a.p) a.p[a.off(q.n, q.y, q.x) + q.c] = v;
    if (b.p) b.p[b.off(q.n, q.y, q.x) + q.c] = v;
  }
};
void coords_minus_grid(Ctx& cx, const TV& coords1, const TV& a, const TV& b) {
  parallel_for(cx, coords1.pixels() * 2, CoordsMinusGridK{coords1, a, b}, "coords_minus_grid");
}

// Convex x8 upsampling, raft/raft.py:86-97.  mask (n,h,w,576) already holds 0.25*conv
// (folded into the weights); channel = k*64 + i*8 + j, k = ky*3 + kx.
struct ConvexUpK {
  TV flow, mask, out;
  GV_HD void operator()(int64_t i) const {
    int X = (int)(i % out.w); int64_t r = i / out.w;
    int Y = (int)(r % out.h); int n = (int)(r / out.h);
    int x = X >> 3, j = X & 7, y = Y >> 3, ii = Y & 7;
    const float* m = mask.p + mask.off(n, y, x) + ii * 8 + j;
    float e[9]; float mx = -3.4e38f;
    for (int k = 0; k < 9; ++k) { e[k] = m[k * 64]; mx = fmaxf(mx, e[k]); }
    float sum = 0.f;
    for (int k = 0; k < 9; ++k) { e[k] = expf(e[k] - mx); sum += e[k]; }
    float ox = 0.f, oy = 0.f;
    for (int k = 0; k < 9; ++k) {
      int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
      float fx = 0.f, fy = 0.f;
      if (yy >= 0 && yy < flow.h && xx >= 0 && xx < flow.w) {
        const float* f = flow.p + flow.off(n, yy, xx);
        fx = 8.f * f[0]; fy = 8.f * f[1];
      }
      float wk = e[k] / sum;
      ox += wk * fx; oy += wk * fy;
    }
    float* o = out.p + out.off(n, Y, X);
    o[0] = ox; o[1] = oy;
  }
};
void convex_upsample(Ctx& cx, const TV& flow, const TV& mask, const TV& out) {
  parallel_for(cx, out.pixels(), ConvexUpK{flow, mask, out}, "convex_upsample");
}

// ----------------------------------------------------- GIMM splat weights
// gimmvfi_r.py:444-492 for one direction: var of a 3x3 gaussian (reflect pad) +
// forward/backward consistency  w = 1/(1+err*a_fe) + 1/(1+var*a_v).
struct SplatWeightsK {
  TV fs, fo, out; const float* g9; const float* afe; const float* av;
  GV_HD int refl(int v, int n) const { return v < 0 ? -v : (v >= n ? 2 * n - 2 - v : v); }
  GV_HD void operator()(int64_t i) const {
    int x = (int)(i % fs.w); int64_t r = i / fs.w;
    int y = (int)(r % fs.h); int n = (int)(r / fs.h);
    float var = 0.f;
    for (int c = 0; c < 2; ++c) {
      float sq = 0.f, m = 0.f;
      for (int k = 0; k < 9; ++k) {
        int yy = refl(y + k / 3 - 1, fs.h), xx = refl(x + k % 3 - 1, fs.w);
        float v = fs.p[fs.off(n, yy, xx) + c];
        sq += g9[k] * (v * v); m += g9[k] * v;
      }
      float d = sq - m * m; if (d < 1e-9f) d = 1e-9f;
      var += sqrtf(d);
    }
    var = var / 2.f;
    const float* f = fs.p + fs.off(n, y, x);
    BilinearTap t = border_tap(x, y, f[0], f[1], fs.w, fs.h, fo.w, fo.h);
    float e0 = fabsf(-tap_fetch(fo, n, t, 0) - f[0]);
    float e1 = fabsf(-tap_fetch(fo, n, t, 1) - f[1]);
    float err = (e0 + e1) / 2.f;
    out.p[out.off(n, y, x)] = 1.f / (1.f + err * afe[0]) + 1.f / (1.f + var * av[0]);
  }
};
void splat_weights(Ctx& cx, const TV& f_self, const TV& f_other, const float* g9, const float* alpha_fe, const float* alpha_v, const TV& out) {
  parallel_for(cx, out.pixels(), SplatWeightsK{f_self, f_other, out, g9, alpha_fe, alpha_v}, "splat_weights");
}

// ----------------------------------------------------------- forward splat
// "linear" softmax-splatting, modules/softsplat.py:307-308 + kernel :376-421.
// acc holds 17 channels per target pixel: 16 x sum(in*metric*w) and sum(metric*w).
// One thread per (source pixel, channel): NHWC makes the 17 atomics of a pixel
// land on consecutive addresses (the reference strides them by H*W).
struct SplatAccK {
  TV lat, flow, metric, acc; const float* t; int t_mode;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, lat.h, lat.w, 17);
    float tt = t[q.n]; float sc = t_mode ? (1.f - tt) : tt;
    const float* f = flow.p + flow.off(q.n, q.y, q.x);
    float fx = (float)q.x + f[0] * sc;
    float fy = (float)q.y + f[1] * sc;
    if (!gv_isfinite(fx) || !gv_isfinite(fy)) return;
    float m = metric.p[metric.off(q.n, q.y, q.x)];
    float v = q.c < 16 ? lat.p[lat.off(q.n, q.y, q.x) + q.c] * m : m;
    float x0f = floorf(fx), y0f = floorf(fy);
    int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
    float wnw = ((float)x1 - fx) * ((float)y1 - fy);
    float wne = (fx - (float)x0) * ((float)y1 - fy);
    float wsw = ((float)x1 - fx) * (fy - (float)y0);
    float wse = (fx - (float)x0) * (fy - (float)y0);
    int W = acc.w, H = acc.h;
    float* base = acc.p + (int64_t)q.n * acc.sn + q.c;
    if (x0 >= 0 && x0 < W && y0 >= 0 && y0 < H) atomic_add_f(base + ((int64_t)y0 * W + x0) * acc.ld, v * wnw);
    if (x1 >= 0 && x1 < W && y0 >= 0 && y0 < H) atomic_add_f(base + ((int64_t)y0 * W + x1) * acc.ld, v * wne);
    if (x0 >= 0 && x0 < W && y1 >= 0 && y1 < H) atomic_add_f(base + ((int64_t)y1 * W + x0) * acc.ld, v * wsw);
    if (x1 >= 0 && x1 < W && y1 >= 0 && y1 < H) atomic_add_f(base + ((int64_t)y1 * W + x1) * acc.ld, v * wse);
  }
};
// The same in the other modes (SplatMode): "softmax" splats [in * exp(m) | exp(m)] (softsplat.py:310-311); "sum" splats the 16 latent
// channels alone, metric unused (softsplat.py:289-313: the "sum-zeroeps" string matches no branch, so nothing is appended).
template <int MODE> struct SplatAccModeK {
  TV lat, flow, metric, acc; const float* t; int t_mode;
  static constexpr int CH = MODE == SPLAT_SUM ? 16 : 17;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, lat.h, lat.w, CH);
    float tt = t[q.n]; float sc = t_mode ? (1.f - tt) : tt;
    const float* f = flow.p + flow.off(q.n, q.y, q.x);
    float fx = (float)q.x + f[0] * sc;
    float fy = (float)q.y + f[1] * sc;
    if (!gv_isfinite(fx) || !gv_isfinite(fy)) return;
    const float l = q.c < 16 ? lat.p[lat.off(q.n, q.y, q.x) + q.c] : 0.f;
    float v = l;
    if constexpr (MODE == SPLAT_SOFTMAX) { const float m = expf(metric.p[metric.off(q.n, q.y, q.x)]); v = q.c < 16 ? l * m : m; }
    float x0f = floorf(fx), y0f = floorf(fy);
    int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
    float wnw = ((float)x1 - fx) * ((float)y1 - fy);
    float wne = (fx - (float)x0) * ((float)y1 - fy);
    float wsw = ((float)x1 - fx) * (fy - (float)y0);
    float wse = (fx - (float)x0) * (fy - (float)y0);
    int W = acc.w, H = acc.h;
    float* base = acc.p + (int64_t)q.n * acc.sn + q.c;
    if (x0 >= 0 && x0 < W && y0 >= 0 && y0 < H) atomic_add_f(base + ((int64_t)y0 * W + x0) * acc.ld, v * wnw);
    if (x1 >= 0 && x1 < W && y0 >= 0 && y0 < H) atomic_add_f(base + ((int64_t)y0 * W + x1) * acc.ld, v * wne);
    if (x0 >= 0 && x0 < W && y1 >= 0 && y1 < H) atomic_add_f(base + ((int64_t)y1 * W + x0) * acc.ld, v * wsw);
    if (x1 >= 0 && x1 < W && y1 >= 0 && y1 < H) atomic_add_f(base + ((int64_t)y1 * W + x1) * acc.ld, v * wse);
  }
};
#ifndef GV_HOSTSIM
// The GPU form of the scatter (the functor above is the reference kernel's thread-per-(pixel, channel) decomposition, kept for the
// host simulation and for ragged layouts).  ONE thread per source pixel:
//   * flow, metric, target cell and the four bilinear weights are computed once (the reference does it 17 times per pixel);
//   * the 16 latent channels arrive as four 16-byte loads; with the metric they form five float4 groups = the 80-byte accumulator
//     pixel [16 x sum(in*m*w) | sum(m*w) | 3 pad lanes];
//   * lanes of a warp hold x-consecutive source pixels.  Under a smooth flow lane l's EAST column of target cells is lane l+1's
//     WEST column: the west contributions travel one lane down by warp shuffle and are summed in registers, so an interior
//     lane issues 2 instead of 4 corner updates;
//   * every update is one red.global.add.v4.f32 (16 bytes per atomic): 10-20 vector reductions per pixel instead of 68 scalar ones.
// Summation order differs from the reference's (whose atomics are unordered anyway): fp32 re-association, ~1e-7 relative.
__device__ __forceinline__ void red_add_v4(float* addr, const F4& v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// MODE (SplatMode): SPLAT_SOFTMAX takes exp(m) for the metric, one expf per source pixel; SPLAT_SUM splats the four latent groups alone
// (the accumulator pixel is then the 16 channels of the result, any 16-byte aligned pixel stride)
template <int MODE>
__device__ __forceinline__ void softsplat_acc_v4_body(const TV& lat, const TV& flow, const TV& metric, const TV& acc, const float* __restrict__ t,
                                                      int t_mode, int64_t npix) {
  constexpr int NG = MODE == SPLAT_SUM ? 4 : 5;   // float4 groups per accumulator pixel
  const int lane = threadIdx.x & 31;
  const int W = acc.w, H = acc.h;
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  const int64_t npad = (npix + 31) & ~(int64_t)31;   // whole warps take part in the shuffles
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < npad; i += step) {
    bool act = i < npix;
    int x = 0, y = 0, n = 0, x0 = 0, y0 = 0;
    float wnw = 0.f, wne = 0.f, wsw = 0.f, wse = 0.f, m = 0.f;
    F4 v[5];
#pragma unroll
    for (int g = 0; g < 5; ++g) v[g] = F4{0.f, 0.f, 0.f, 0.f};
    if (act) {
      x = (int)(i % W); const int64_t r = i / W; y = (int)(r % H); n = (int)(r / H);
      const float tt = __ldg(t + n), sc = t_mode ? (1.f - tt) : tt;
      const float2 f = *reinterpret_cast<const float2*>(flow.p + flow.off(n, y, x));
      const float fx = (float)x + f.x * sc, fy = (float)y + f.y * sc;
      act = gv_isfinite(fx) && gv_isfinite(fy);
      if (act) {
        const float x0f = floorf(fx), y0f = floorf(fy);
        x0 = (int)x0f; y0 = (int)y0f;
        const float x1f = (float)(x0 + 1), y1f = (float)(y0 + 1);
        wnw = (x1f - fx) * (y1f - fy); wne = (fx - (float)x0) * (y1f - fy);
        wsw = (x1f - fx) * (fy - (float)y0); wse = (fx - (float)x0) * (fy - (float)y0);
        if constexpr (MODE == SPLAT_SUM) {
          const float* lp = lat.p + lat.off(n, y, x);
#pragma unroll
          for (int g = 0; g < 4; ++g) v[g] = ld4(lp + 4 * g);
        } else {
          m = metric.p[metric.off(n, y, x)];
          if constexpr (MODE == SPLAT_SOFTMAX) m = expf(m);
          const float* lp = lat.p + lat.off(n, y, x);
#pragma unroll
          for (int g = 0; g < 4; ++g) { const F4 a = ld4(lp + 4 * g); v[g] = F4{a.x * m, a.y * m, a.z * m, a.w * m}; }
          v[4] = F4{m, 0.f, 0.f, 0.f};
        }
      }
    }
    // x-neighbour merge: lane l+1 is pixel x+1 of the same row (rows never straddle a merge: x + 1 < W is required)
    const int px0 = __shfl_down_sync(0xffffffffu, x0, 1), py0 = __shfl_down_sync(0xffffffffu, y0, 1);
    const int pact = __shfl_down_sync(0xffffffffu, (int)act, 1);
    const float pwnw = __shfl_down_sync(0xffffffffu, wnw, 1), pwsw = __shfl_down_sync(0xffffffffu, wsw, 1);
    const bool take = lane < 31 && act && pact && x + 1 < W && px0 == x0 + 1 && py0 == y0;   // my east column == its west column
    const bool taken = __shfl_up_sync(0xffffffffu, (int)take, 1) != 0 && lane > 0;          // lane l-1 carries my west column
    const int x1 = x0 + 1, y1 = y0 + 1;
    const bool in_y0 = y0 >= 0 && y0 < H, in_y1 = y1 >= 0 && y1 < H, in_x0 = x0 >= 0 && x0 < W, in_x1 = x1 >= 0 && x1 < W;
    float* base = acc.p + (int64_t)n * acc.sn;
    float* a_nw = base + ((int64_t)y0 * W + x0) * acc.ld;
    float* a_sw = a_nw + (int64_t)W * acc.ld;
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      // the neighbour's west-column VALUES (its own v * its own west weights), fetched by every lane (shuffles are warp collective)
      F4 pv;
      pv.x = __shfl_down_sync(0xffffffffu, v[g].x, 1); pv.y = __shfl_down_sync(0xffffffffu, v[g].y, 1);
      pv.z = __shfl_down_sync(0xffffffffu, v[g].z, 1); pv.w = __shfl_down_sync(0xffffffffu, v[g].w, 1);
      if (!act) continue;
      F4 ne = F4{v[g].x * wne, v[g].y * wne, v[g].z * wne, v[g].w * wne};
      F4 se = F4{v[g].x * wse, v[g].y * wse, v[g].z * wse, v[g].w * wse};
      if (take) {
        ne.x += pv.x * pwnw; ne.y += pv.y * pwnw; ne.z += pv.z * pwnw; ne.w += pv.w * pwnw;
        se.x += pv.x * pwsw; se.y += pv.y * pwsw; se.z += pv.z * pwsw; se.w += pv.w * pwsw;
      }
      if (!taken) {
        if (in_x0 && in_y0) red_add_v4(a_nw + 4 * g, F4{v[g].x * wnw, v[g].y * wnw, v[g].z * wnw, v[g].w * wnw});
        if (in_x0 && in_y1) red_add_v4(a_sw + 4 * g, F4{v[g].x * wsw, v[g].y * wsw, v[g].z * wsw, v[g].w * wsw});
      }
      if (in_x1 && in_y0) red_add_v4(a_nw + acc.ld + 4 * g, ne);
      if (in_x1 && in_y1) red_add_v4(a_sw + acc.ld + 4 * g, se);
    }
  }
}
__global__ void __launch_bounds__(256) softsplat_acc_v4_kernel(TV lat, TV flow, TV metric, TV acc, const float* __restrict__ t, int t_mode,
                                                              int64_t npix) {
  softsplat_acc_v4_body<SPLAT_LINEAR>(lat, flow, metric, acc, t, t_mode, npix);
}
template <int MODE>
__global__ void __launch_bounds__(256) softsplat_acc_v4_mode_kernel(TV lat, TV flow, TV metric, TV acc, const float* __restrict__ t, int t_mode,
                                                                   int64_t npix) {
  softsplat_acc_v4_body<MODE>(lat, flow, metric, acc, t, t_mode, npix);
}
#endif

#ifndef GV_HOSTSIM
// The whole "linear-zeroeps" splat (modules/softsplat.py:286-352) in ONE pass over HBM: a CTA owns a 32 x 32 tile of TARGET pixels whose
// 17-channel accumulators live in shared memory (68 KB), scans the source pixels that can reach it - the tile grown by
// R = ceil(max|flow| * s) + 1, the per-sample flow bound the engine computes anyway for normalize_flow (fi_utils.py:52-60) - adds the
// landing ones with shared-memory atomics, normalises in place and writes the 16 output channels.  DRAM traffic: flows (8 B, re-read
// by neighbouring tiles mostly from L2) + latents and metric of the landing pixels (68 B) + the output (64 B) = the op's algorithmic
// 140 B/px; the three-pass form (memset, global vector reductions, normalise) moves ~430 B/px through a 167 MB accumulator that
// does not fit L2.  Summation order differs from the reference's (unordered atomics there too): fp32 re-association only.
constexpr int SPT = 32;   // tile edge
__global__ void __launch_bounds__(256) softsplat_tile_kernel(TV lat, TV flow, TV metric, TV out, const float* __restrict__ t, int t_mode,
                                                            const float* __restrict__ absmax, int tiles_x, int tiles_y, int n_img) {
  extern __shared__ float sacc[];   // [SPT * SPT][17]
  const int W = out.w, H = out.h, tid = threadIdx.x;
  const int num_tiles = n_img * tiles_x * tiles_y;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int r = tile; const int tx = r % tiles_x; r /= tiles_x; const int ty = r % tiles_y; const int n = r / tiles_y;
    const int X0 = tx * SPT, Y0 = ty * SPT;
    for (int i = tid; i < SPT * SPT * 17; i += 256) sacc[i] = 0.f;
    const float tt = __ldg(t + n), sc = t_mode ? (1.f - tt) : tt;
    const float bound = __ldg(absmax + n) * fabsf(sc);
    const int R = (bound < 1e6f ? (int)ceilf(bound) : 1000000) + 1;   // (a non-finite / absurd bound degrades to scanning the frame)
    const int xa = max(0, X0 - R), xb = min(W, X0 + SPT + R), ya = max(0, Y0 - R), yb = min(H, Y0 + SPT + R);
    const int rw = xb - xa;
    __syncthreads();
    for (int i = tid; i < rw * (yb - ya); i += 256) {
      const int y = ya + i / rw, x = xa + i % rw;
      const float2 f = *reinterpret_cast<const float2*>(flow.p + flow.off(n, y, x));
      const float fx = (float)x + f.x * sc, fy = (float)y + f.y * sc;
      if (!gv_isfinite(fx) || !gv_isfinite(fy)) continue;
      const float x0f = floorf(fx), y0f = floorf(fy);
      const int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
      if (x1 < X0 || x0 >= X0 + SPT || y1 < Y0 || y0 >= Y0 + SPT) continue;   // no corner in this tile
      const float m = metric.p[metric.off(n, y, x)];
      float v[17];
      const float* lp = lat.p + lat.off(n, y, x);
#pragma unroll
      for (int g = 0; g < 4; ++g) { const F4 a = ld4(lp + 4 * g); v[4 * g] = a.x * m; v[4 * g + 1] = a.y * m; v[4 * g + 2] = a.z * m; v[4 * g + 3] = a.w * m; }
      v[16] = m;
      const float x1f = (float)x1, y1f = (float)y1;
      const float wgt[4] = {(x1f - fx) * (y1f - fy), (fx - (float)x0) * (y1f - fy), (x1f - fx) * (fy - (float)y0), (fx - (float)x0) * (fy - (float)y0)};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int cx = (k & 1) ? x1 : x0, cy = (k & 2) ? y1 : y0;
        if (cx < X0 || cx >= X0 + SPT || cy < Y0 || cy >= Y0 + SPT || cx >= W || cy >= H || cx < 0 || cy < 0) continue;
        float* a = sacc + ((cy - Y0) * SPT + (cx - X0)) * 17;
#pragma unroll
        for (int c = 0; c < 17; ++c) atomicAdd(a + c, v[c] * wgt[k]);
      }
    }
    __syncthreads();
    for (int i = tid; i < SPT * SPT * 4; i += 256) {   // "zeroeps" normalisation + store, 4 channels per thread
      const int g = i & 3, p = i >> 2, lx = p % SPT, ly = p / SPT;
      const int x = X0 + lx, y = Y0 + ly;
      if (x >= W || y >= H) continue;
      const float* a = sacc + p * 17;
      float d = a[16]; if (d == 0.f) d = 1.f;
      st4(out.p + out.off(n, y, x) + 4 * g, F4{a[4 * g] / d, a[4 * g + 1] / d, a[4 * g + 2] / d, a[4 * g + 3] / d});
    }
    __syncthreads();
  }
}
#endif
// fused splat: returns false when the layout does not qualify
bool softsplat_fused(Ctx& cx, const TV& lat, const TV& flow, const TV& metric, const float* t_per_sample, int t_mode, const float* flow_absmax,
                     const TV& out) {
#ifndef GV_HOSTSIM
  if (!flow_absmax || lat.c != 16 || out.c != 16 || !vec4_ok(lat) || !vec4_ok(out) || (reinterpret_cast<uintptr_t>(flow.p) & 7) || flow.ld % 2 || flow.sn % 2 ||
      flow.f16 || metric.f16)
    return false;
  if (cx.dry) return true;
  cx.launches++;
  const int tiles_x = (out.w + SPT - 1) / SPT, tiles_y = (out.h + SPT - 1) / SPT;
  const int smem = SPT * SPT * 17 * 4;
  static volatile unsigned char attr[64];
  gv_set_max_smem(softsplat_tile_kernel, smem, attr);
  if (cx.prof) cx.prof->begin(cx.stream, "softsplat_fused", (double)lat.pixels() * 35.0);   // 140 B per pixel (SURVEY 8(d))
  const int tiles = out.n * tiles_x * tiles_y;
  const int grid = tiles < cx.sm_count * 3 ? tiles : cx.sm_count * 3;
  softsplat_tile_kernel<<<grid, 256, smem, cx.stream>>>(lat, flow, metric, out, t_per_sample, t_mode, flow_absmax, tiles_x, tiles_y, out.n);
  gv_check_launch("softsplat_fused");
  if (cx.prof) cx.prof->end(cx.stream);
  return true;
#else
  (void)cx; (void)lat; (void)flow; (void)metric; (void)t_per_sample; (void)t_mode; (void)flow_absmax; (void)out;
  return false;
#endif
}

void softsplat_accumulate(Ctx& cx, const TV& lat, const TV& flow, const TV& metric, const float* t_per_sample, int t_mode, const TV& acc) {
#ifndef GV_HOSTSIM
  // vector form: 16-byte aligned latent / accumulator pixels (acc.ld % 4: the pad lanes receive +0)
  const bool v4 = lat.c == 16 && vec4_ok(lat) && (reinterpret_cast<uintptr_t>(acc.p) & 15) == 0 && acc.ld % 4 == 0 && acc.ld >= 20 && acc.sn % 4 == 0 &&
                  (reinterpret_cast<uintptr_t>(flow.p) & 7) == 0 && flow.ld % 2 == 0 && flow.sn % 2 == 0 && !acc.f16 && !flow.f16 && !metric.f16;
  if (v4) {
    if (cx.dry) return;
    cx.launches++;
    const int64_t npix = lat.pixels();
    if (cx.prof) cx.prof->begin(cx.stream, "softsplat_accumulate", (double)npix * 35.0);   // 140 B per pixel (SURVEY 8(d)): 16+1+2 read, 16 written
    int64_t blocks = (npix + 255) / 256, cap = (int64_t)cx.sm_count * 8;
    if (blocks > cap) blocks = cap;
    softsplat_acc_v4_kernel<<<(unsigned)blocks, 256, 0, cx.stream>>>(lat, flow, metric, acc, t_per_sample, t_mode, npix);
    gv_check_launch("softsplat_accumulate");
    if (cx.prof) cx.prof->end(cx.stream);
    return;
  }
#endif
  parallel_for(cx, lat.pixels() * 17, SplatAccK{lat, flow, metric, acc, t_per_sample, t_mode}, "softsplat_accumulate");
}
void softsplat_accumulate_mode(Ctx& cx, const TV& lat, const TV& flow, const TV& metric, const float* t_per_sample, int t_mode, const TV& acc, int mode) {
  if (mode == SPLAT_LINEAR) return softsplat_accumulate(cx, lat, flow, metric, t_per_sample, t_mode, acc);
  if (mode != SPLAT_SOFTMAX && mode != SPLAT_SUM) throw std::runtime_error("softsplat: unknown splat mode");
  const bool sum = mode == SPLAT_SUM;
#ifndef GV_HOSTSIM
  const bool v4 = lat.c == 16 && vec4_ok(lat) && (reinterpret_cast<uintptr_t>(acc.p) & 15) == 0 && acc.ld % 4 == 0 && acc.ld >= (sum ? 16 : 20) &&
                  acc.sn % 4 == 0 && (reinterpret_cast<uintptr_t>(flow.p) & 7) == 0 && flow.ld % 2 == 0 && flow.sn % 2 == 0 && !acc.f16 && !flow.f16 &&
                  !metric.f16;
  if (v4) {
    if (cx.dry) return;
    cx.launches++;
    const int64_t npix = lat.pixels();
    const char* name = sum ? "softsplat_accumulate_sum" : "softsplat_accumulate_softmax";
    if (cx.prof) cx.prof->begin(cx.stream, name, (double)npix * 35.0);
    int64_t blocks = (npix + 255) / 256, cap = (int64_t)cx.sm_count * 8;
    if (blocks > cap) blocks = cap;
    if (sum) softsplat_acc_v4_mode_kernel<SPLAT_SUM><<<(unsigned)blocks, 256, 0, cx.stream>>>(lat, flow, metric, acc, t_per_sample, t_mode, npix);
    else softsplat_acc_v4_mode_kernel<SPLAT_SOFTMAX><<<(unsigned)blocks, 256, 0, cx.stream>>>(lat, flow, metric, acc, t_per_sample, t_mode, npix);
    gv_check_launch(name);
    if (cx.prof) cx.prof->end(cx.stream);
    return;
  }
#endif
  if (sum) parallel_for(cx, lat.pixels() * 16, SplatAccModeK<SPLAT_SUM>{lat, flow, metric, acc, t_per_sample, t_mode}, "softsplat_accumulate_sum");
  else parallel_for(cx, lat.pixels() * 17, SplatAccModeK<SPLAT_SOFTMAX>{lat, flow, metric, acc, t_per_sample, t_mode}, "softsplat_accumulate_softmax");
}

// "zeroeps" normalisation, modules/softsplat.py:330-344.
template <int L, bool Any> struct SplatNormK {
  TV acc, out;
  GV_HD void operator()(int64_t i) const {
    const Idx4 q = decode4(i, out.h, out.w, 16 / L);
    const float* a = acc.p + acc.off(q.n, q.y, q.x);
    float d = a[16]; if (d == 0.f) d = 1.f;
    float v[L];
    ld_lanes<L>(a + q.c * L, v);
    for (int k = 0; k < L; ++k) v[k] = v[k] / d;
    st_lanes<L, Any>(out, out.off(q.n, q.y, q.x) + q.c * L, v);
  }
};
void softsplat_normalize(Ctx& cx, const TV& acc, const TV& out) {
  const bool four = out.c == 16 && vec4_ok(out) && lanes4_ok(acc) && !acc.f16;
  lanes_for<SplatNormK>(cx, four, out.pixels() * 16, "softsplat_normalize", acc, out);
}

// ------------------------------------------------- differentiable splat (training)
// softsplat_func of modules/softsplat.py:358-663 for any 4-D strided float / double tensors.  The reference runs one thread per
// (pixel, channel) and recomputes the flow, the floor, the corners and the weights C times per pixel (flowgrad 2C times); here one
// thread per SOURCE pixel computes them once and loops over the channels.  The weights and their derivatives are the reference's
// expressions (:401-404, :600-613) evaluated in the same order, with the floor held fixed.  Corners are tested in T arithmetic, so a
// finite coordinate far outside the frame never goes through an integer conversion.
GV_HD bool sv_finite(float v) { return gv_isfinite(v); }
GV_HD bool sv_finite(double v) { return fabs(v) <= 1.7976931348623157e308; }
GV_HD float sv_floor(float v) { return floorf(v); }
GV_HD double sv_floor(double v) { return floor(v); }
GV_HD void sv_red_add(float* a, float v) {
#if defined(GV_HOSTSIM)
#pragma omp atomic
  *a += v;
#elif defined(__CUDA_ARCH__)
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(a), "f"(v) : "memory");
#else
  *a += v;
#endif
}
GV_HD void sv_red_add(double* a, double v) {
#if defined(GV_HOSTSIM)
#pragma omp atomic
  *a += v;
#elif defined(__CUDA_ARCH__)
  atomicAdd(a, v);
#else
  *a += v;
#endif
}
// corner geometry of one source pixel: in-frame flags of the two columns / rows, element offsets within an (n, c) plane
template <class T> struct SplatCell {
  T fx, fy, x0f, y0f, x1f, y1f;
  bool ix0, ix1, iy0, iy1;
  int64_t ox0, ox1, oy0, oy1;
  GV_HD bool any() const { return (ix0 || ix1) && (iy0 || iy1); }
  GV_HD void make(T fx_, T fy_, int64_t H, int64_t W, const int64_t* st) {
    fx = fx_; fy = fy_;
    x0f = sv_floor(fx); y0f = sv_floor(fy); x1f = x0f + (T)1; y1f = y0f + (T)1;
    ix0 = x0f >= (T)0 && x0f < (T)W; ix1 = x1f >= (T)0 && x1f < (T)W;
    iy0 = y0f >= (T)0 && y0f < (T)H; iy1 = y1f >= (T)0 && y1f < (T)H;
    if (!any()) return;   // x0f in [-1, W), y0f in [-1, H) from here on
    const int64_t x0 = (int64_t)x0f, y0 = (int64_t)y0f;
    ox0 = x0 * st[3]; ox1 = ox0 + st[3]; oy0 = y0 * st[2]; oy1 = oy0 + st[2];
  }
};
template <class T> struct SplatOutK {
  SV4<T> in, flow, out;
  GV_HD void operator()(int64_t i) const {
    const int64_t W = in.sz[3], H = in.sz[2];
    const int64_t x = i % W, r = i / W, y = r % H, n = r / H;
    const T* f = flow.p + n * flow.st[0] + y * flow.st[2] + x * flow.st[3];
    const T fx = (T)x + f[0], fy = (T)y + f[flow.st[1]];
    if (!sv_finite(fx) || !sv_finite(fy)) return;
    SplatCell<T> q;
    q.make(fx, fy, H, W, out.st);
    if (!q.any()) return;
    const T wnw = (q.x1f - fx) * (q.y1f - fy), wne = (fx - q.x0f) * (q.y1f - fy);
    const T wsw = (q.x1f - fx) * (fy - q.y0f), wse = (fx - q.x0f) * (fy - q.y0f);
    const T* src = in.p + n * in.st[0] + y * in.st[2] + x * in.st[3];
    T* dst = out.p + n * out.st[0];
    for (int64_t c = 0; c < in.sz[1]; ++c, src += in.st[1], dst += out.st[1]) {
      const T v = *src;
      if (q.ix0 && q.iy0) sv_red_add(dst + q.oy0 + q.ox0, v * wnw);
      if (q.ix1 && q.iy0) sv_red_add(dst + q.oy0 + q.ox1, v * wne);
      if (q.ix0 && q.iy1) sv_red_add(dst + q.oy1 + q.ox0, v * wsw);
      if (q.ix1 && q.iy1) sv_red_add(dst + q.oy1 + q.ox1, v * wse);
    }
  }
};
// The backward is a GATHER: source pixel p reads the incoming gradient at its own four corners and writes only its own ingrad
// elements and its own two flowgrad elements, so no two threads write the same address - no atomics, bit-identical reruns.
template <class T> struct SplatGradK {
  SV4<T> in, flow, og, ig, fg;
  GV_HD void operator()(int64_t i) const {
    const int64_t W = og.sz[3], H = og.sz[2], C = og.sz[1];
    const int64_t x = i % W, r = i / W, y = r % H, n = r / H;
    const T* f = flow.p + n * flow.st[0] + y * flow.st[2] + x * flow.st[3];
    const T fx = (T)x + f[0], fy = (T)y + f[flow.st[1]];
    T* gi = ig.p ? ig.p + n * ig.st[0] + y * ig.st[2] + x * ig.st[3] : nullptr;
    T* gf = fg.p ? fg.p + n * fg.st[0] + y * fg.st[2] + x * fg.st[3] : nullptr;
    SplatCell<T> q;
    const bool fin = sv_finite(fx) && sv_finite(fy);
    if (fin) q.make(fx, fy, H, W, og.st);
    if (!fin || !q.any()) {   // no corner receives anything: both gradients are exactly 0
      if (gi) for (int64_t c = 0; c < C; ++c) gi[c * ig.st[1]] = (T)0;
      if (gf) { gf[0] = (T)0; gf[fg.st[1]] = (T)0; }
      return;
    }
    const T wnw = (q.x1f - fx) * (q.y1f - fy), wne = (fx - q.x0f) * (q.y1f - fy);
    const T wsw = (q.x1f - fx) * (fy - q.y0f), wse = (fx - q.x0f) * (fy - q.y0f);
    // d w / d fx (reference flow channel 0) and d w / d fy (channel 1)
    const T xnw = (T)(-1) * (q.y1f - fy), xne = (T)(+1) * (q.y1f - fy), xsw = (T)(-1) * (fy - q.y0f), xse = (T)(+1) * (fy - q.y0f);
    const T ynw = (q.x1f - fx) * (T)(-1), yne = (fx - q.x0f) * (T)(-1), ysw = (q.x1f - fx) * (T)(+1), yse = (fx - q.x0f) * (T)(+1);
    const T* src = in.p + n * in.st[0] + y * in.st[2] + x * in.st[3];
    const T* g = og.p + n * og.st[0];
    T sx = (T)0, sy = (T)0;
    for (int64_t c = 0; c < C; ++c, g += og.st[1]) {
      const T gnw = q.ix0 && q.iy0 ? g[q.oy0 + q.ox0] : (T)0, gne = q.ix1 && q.iy0 ? g[q.oy0 + q.ox1] : (T)0;
      const T gsw = q.ix0 && q.iy1 ? g[q.oy1 + q.ox0] : (T)0, gse = q.ix1 && q.iy1 ? g[q.oy1 + q.ox1] : (T)0;
      if (gi) {
        T s = (T)0;
        if (q.ix0 && q.iy0) s += gnw * wnw;
        if (q.ix1 && q.iy0) s += gne * wne;
        if (q.ix0 && q.iy1) s += gsw * wsw;
        if (q.ix1 && q.iy1) s += gse * wse;
        gi[c * ig.st[1]] = s;
      }
      if (gf) {
        const T a = src[c * in.st[1]];
        T t;
        if (q.ix0 && q.iy0) { t = gnw * a; sx += t * xnw; sy += t * ynw; }
        if (q.ix1 && q.iy0) { t = gne * a; sx += t * xne; sy += t * yne; }
        if (q.ix0 && q.iy1) { t = gsw * a; sx += t * xsw; sy += t * ysw; }
        if (q.ix1 && q.iy1) { t = gse * a; sx += t * xse; sy += t * yse; }
      }
    }
    if (gf) { gf[0] = sx; gf[fg.st[1]] = sy; }
  }
};
template <class T> void softsplat_out_any(Ctx& cx, const SV4<T>& in, const SV4<T>& flow, const SV4<T>& out) {
  parallel_for(cx, in.sz[0] * in.sz[2] * in.sz[3], SplatOutK<T>{in, flow, out}, "softsplat_out");
}
template <class T> void softsplat_grad_any(Ctx& cx, const SV4<T>& in, const SV4<T>& flow, const SV4<T>& outgrad, const SV4<T>& ingrad,
                                           const SV4<T>& flowgrad) {
  if (!ingrad.p && !flowgrad.p) return;
  parallel_for(cx, outgrad.sz[0] * outgrad.sz[2] * outgrad.sz[3], SplatGradK<T>{in, flow, outgrad, ingrad, flowgrad}, "softsplat_grad");
}
template void softsplat_out_any<float>(Ctx&, const SV4<float>&, const SV4<float>&, const SV4<float>&);
template void softsplat_out_any<double>(Ctx&, const SV4<double>&, const SV4<double>&, const SV4<double>&);
template void softsplat_grad_any<float>(Ctx&, const SV4<float>&, const SV4<float>&, const SV4<float>&, const SV4<float>&, const SV4<float>&);
template void softsplat_grad_any<double>(Ctx&, const SV4<double>&, const SV4<double>&, const SV4<double>&, const SV4<double>&, const SV4<double>&);

// ------------------------------------------------------------ synthesis glue
// gimmvfi_r.py:239-240: flow_t->0 = flow_t * (-t), flow_t->1 = flow_t * (1 - t)
struct ScaleFlowTK {
  TV ft, f0, f1; const float* t;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, ft.h, ft.w, 2);
    float v = ft.p[ft.off(q.n, q.y, q.x) + q.c]; float tt = t[q.n];
    f0.p[f0.off(q.n, q.y, q.x) + q.c] = v * (-tt);
    f1.p[f1.off(q.n, q.y, q.x) + q.c] = v * (1.0f - tt);
  }
};
void scale_flow_t(Ctx& cx, const TV& flow_t, const float* t_per_sample, const TV& f0, const TV& f1) {
  parallel_for(cx, flow_t.pixels() * 2, ScaleFlowTK{flow_t, f0, f1, t_per_sample}, "scale_flow_t");
}

struct HypoPackK {
  const float* coord; TV dst;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, dst.h, dst.w, 3);
    dst.p[dst.off(q.n, q.y, q.x) + q.c] = coord[i];
  }
};
void hypo_pack_input(Ctx& cx, const float* coord, const TV& dst) {
  parallel_for(cx, dst.pixels() * 3, HypoPackK{coord, dst}, "hypo_pack_input");
}

// gimmvfi_r.py:494-504: coord + flow * (1/(1-t))  (mode 0)  |  coord + flow * (1/t)  (mode 1)
struct LookupCoordsK {
  TV flow, out; const float* t; int mode;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, out.h, out.w, 2);
    float tt = t[q.n];
    float sc = mode == 0 ? 1.0f / (1.0f - tt) : 1.0f / tt;
    float g = q.c == 0 ? (float)q.x : (float)q.y;
    out.p[out.off(q.n, q.y, q.x) + q.c] = g + flow.p[flow.off(q.n, q.y, q.x) + q.c] * sc;
  }
};
void lookup_coords(Ctx& cx, const TV& flow, const float* t_per_sample, int mode, const TV& out) {
  parallel_for(cx, out.pixels() * 2, LookupCoordsK{flow, out, t_per_sample, mode}, "lookup_coords");
}

// fi_components.py:272-275 with the init-decoder head re-ordered at pack time to
// [ft(128) | dflow0(2) | dflow1(2) | mask(1)].
struct FlowMaskSplitK {
  TV o, f0i, f1i, f0, f1, mask;
  GV_HD void operator()(int64_t i) const {
    int x = (int)(i % o.w); int64_t r = i / o.w; int y = (int)(r % o.h); int n = (int)(r / o.h);
    const float* s = o.p + o.off(n, y, x) + 128;
    const float* a = f0i.p + f0i.off(n, y, x); const float* b = f1i.p + f1i.off(n, y, x);
    float* A = f0.p + f0.off(n, y, x); float* B = f1.p + f1.off(n, y, x);
    A[0] = a[0] + s[0]; A[1] = a[1] + s[1]; B[0] = b[0] + s[2]; B[1] = b[1] + s[3];
    mask.p[mask.off(n, y, x)] = s[4];
  }
};
void flow_mask_split(Ctx& cx, const TV& out133, const TV& f0_in, const TV& f1_in, const TV& f0, const TV& f1, const TV& mask) {
  parallel_for(cx, out133.pixels(), FlowMaskSplitK{out133, f0_in, f1_in, f0, f1, mask}, "flow_mask_split");
}

struct AddInplaceK {
  TV dst, src;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, dst.h, dst.w, dst.c);
    dst.p[dst.off(q.n, q.y, q.x) + q.c] += src.p[src.off(q.n, q.y, q.x) + q.c];
  }
};
void add_inplace_slices(Ctx& cx, const TV& dst, const TV& src) {
  parallel_for(cx, dst.pixels() * dst.c, AddInplaceK{dst, src}, "add_inplace");
}

// fi_components.py:331-340: split 24 -> 6/6/3/9, add the repeated base flows / mask, sigmoid.
struct FinalHeadsK {
  TV o, fl0, fl1, m, of0, of1, om, ores;
  GV_HD void operator()(int64_t i) const {
    int x = (int)(i % o.w); int64_t r = i / o.w; int y = (int)(r % o.h); int n = (int)(r / o.h);
    const float* s = o.p + o.off(n, y, x);
    const float* a = fl0.p + fl0.off(n, y, x); const float* b = fl1.p + fl1.off(n, y, x);
    float mm = m.p[m.off(n, y, x)];
    float* A = of0.p + of0.off(n, y, x); float* B = of1.p + of1.off(n, y, x);
    float* M = om.p + om.off(n, y, x); float* R = ores.p + ores.off(n, y, x);
    for (int k = 0; k < 6; ++k) { A[k] = s[k] + a[k & 1]; B[k] = s[6 + k] + b[k & 1]; }
    for (int k = 0; k < 3; ++k) M[k] = 1.f / (1.f + expf(-(s[12 + k] + mm)));
    for (int k = 0; k < 9; ++k) R[k] = s[15 + k];
  }
};
void final_heads(Ctx& cx, const TV& out24, const TV& flow0, const TV& flow1, const TV& mask, const TV& oflow0, const TV& oflow1,
                 const TV& omask, const TV& ores) {
  parallel_for(cx, out24.pixels(), FinalHeadsK{out24, flow0, flow1, mask, oflow0, oflow1, omask, ores}, "final_heads");
}

// warp_w_mask, gimmvfi_r.py:213-220 (flows / sigmoid(mask) already at full res).
struct WarpBlendK {
  TV i0, i1, f0, f1, m, out;
  GV_HD void operator()(int64_t i) const {
    Idx4 q = decode4(i, out.h, out.w, 3);
    const float* a = f0.p + f0.off(q.n, q.y, q.x); const float* b = f1.p + f1.off(q.n, q.y, q.x);
    BilinearTap t0 = border_tap(q.x, q.y, a[0], a[1], f0.w, f0.h, i0.w, i0.h);
    BilinearTap t1 = border_tap(q.x, q.y, b[0], b[1], f1.w, f1.h, i1.w, i1.h);
    float mm = m.p[m.off(q.n, q.y, q.x)];
    out.p[out.off(q.n, q.y, q.x) + q.c] = mm * tap_fetch(i0, q.n, t0, q.c) + (1.f - mm) * tap_fetch(i1, q.n, t1, q.c);
  }
};
void warp_blend(Ctx& cx, const TV& img0, const TV& img1, const TV& f0, const TV& f1, const TV& mask, const TV& out) {
  parallel_for(cx, out.pixels() * 3, WarpBlendK{img0, img1, f0, f1, mask, out}, "warp_blend");
}

// multi_flow_combine, fi_components.py:57-88: 3 x (2 warps, blend, + residual) and their mean.  One thread per pixel: the taps are
// computed once per flow pair, the four corners of each frame are fetched as 16-byte pixels (3 colours + padding lane), the nine blended
// values leave as three 16-byte stores.  Per value, tap_fetch's corner order and products.
struct MultiFlowBlendK {
  TV i0, i1, f0, f1, m, res, w9, mean3;
  GV_HD static void fetch3(const TV& s, int n, const BilinearTap& t, float* v) {
    const float* b = s.p + (int64_t)n * s.sn;
    v[0] = v[1] = v[2] = 0.f;
    if (t.vy0 && t.vx0) { const F4 p = ld4(b + ((int64_t)t.y0 * s.w + t.x0) * s.ld); const float w = t.wx0 * t.wy0; v[0] += p.x * w; v[1] += p.y * w; v[2] += p.z * w; }
    if (t.vy0 && t.vx1) { const F4 p = ld4(b + ((int64_t)t.y0 * s.w + t.x1) * s.ld); const float w = t.wx1 * t.wy0; v[0] += p.x * w; v[1] += p.y * w; v[2] += p.z * w; }
    if (t.vy1 && t.vx0) { const F4 p = ld4(b + ((int64_t)t.y1 * s.w + t.x0) * s.ld); const float w = t.wx0 * t.wy1; v[0] += p.x * w; v[1] += p.y * w; v[2] += p.z * w; }
    if (t.vy1 && t.vx1) { const F4 p = ld4(b + ((int64_t)t.y1 * s.w + t.x1) * s.ld); const float w = t.wx1 * t.wy1; v[0] += p.x * w; v[1] += p.y * w; v[2] += p.z * w; }
  }
  GV_HD void operator()(int64_t i) const {
    const int x = (int)(i % w9.w); int64_t r = i / w9.w; const int y = (int)(r % w9.h); const int n = (int)(r / w9.h);
    const float* a = f0.p + f0.off(n, y, x); const float* b = f1.p + f1.off(n, y, x);
    const float* mp = m.p + m.off(n, y, x); const float* rp = res.p + res.off(n, y, x);
    float out[12]; float acc[3] = {0.f, 0.f, 0.f};
    out[9] = out[10] = out[11] = 0.f;
    for (int k = 0; k < 3; ++k) {
      const BilinearTap t0 = border_tap(x, y, a[2 * k], a[2 * k + 1], f0.w, f0.h, i0.w, i0.h);
      const BilinearTap t1 = border_tap(x, y, b[2 * k], b[2 * k + 1], f1.w, f1.h, i1.w, i1.h);
      float v0[3], v1[3];
      fetch3(i0, n, t0, v0); fetch3(i1, n, t1, v1);
      const float mm = mp[k];
      for (int c = 0; c < 3; ++c) {
        float v = mm * v0[c] + (1.f - mm) * v1[c];
        v += rp[3 * k + c];
        out[3 * k + c] = v;
        acc[c] += v;
      }
    }
    float* o = w9.p + w9.off(n, y, x);
    F4 s0 = {out[0], out[1], out[2], out[3]}, s1 = {out[4], out[5], out[6], out[7]}, s2 = {out[8], out[9], out[10], out[11]};
    st4(o, s0); st4(o + 4, s1); st4(o + 8, s2);
    F4 mn = {acc[0] / 3.f, acc[1] / 3.f, acc[2] / 3.f, 0.f};
    st4(mean3.p + mean3.off(n, y, x), mn);
  }
};
void multi_flow_blend(Ctx& cx, const TV& img0, const TV& img1, const TV& f0, const TV& f1, const TV& mask, const TV& res,
                      const TV& warps9, const TV& mean3) {
  auto px4 = [](const TV& t, int lanes) { return lanes4_ok(t) && !t.f16 && t.ld >= lanes; };
  if (!px4(img0, 4) || !px4(img1, 4) || !px4(warps9, 12) || !px4(mean3, 4) || f0.f16 || f1.f16 || mask.f16 || res.f16)
    throw std::runtime_error("multi_flow_blend: frames, warps and mean need 16-byte-aligned fp32 pixels of 4 / 12 / 4 lanes, flows / mask / residual fp32");
  parallel_for(cx, warps9.pixels(), MultiFlowBlendK{img0, img1, f0, f1, mask, res, warps9, mean3}, "multi_flow_blend");
}

// fi_components.py:89-92 + gimmvfi_r.py:308: clamp((mean + comb + 1)/2, 0, 1) -> NCHW
struct CombineOutK {
  TV mean3, conv3; float* dst;
  GV_HD void operator()(int64_t i) const {
    int x = (int)(i % mean3.w); int64_t r = i / mean3.w;
    int y = (int)(r % mean3.h); r /= mean3.h; int c = (int)(r % 3); int n = (int)(r / 3);
    float v = mean3.p[mean3.off(n, y, x) + c] + conv3.p[conv3.off(n, y, x) + c];
    v = (v + 1.0f) / 2.f;
    dst[i] = fminf(fmaxf(v, 0.f), 1.f);
  }
};
void combine_output(Ctx& cx, const TV& mean3, const TV& conv3, float* dst_nchw) {
  parallel_for(cx, mean3.pixels() * 3, CombineOutK{mean3, conv3, dst_nchw}, "combine_output");
}
// the same with sample n stored at image rows[n] of dst
struct CombineOutRowsK {
  CombineOutK k; int rows[kGatherMax];
  GV_HD void operator()(int64_t i) const {
    const int64_t per = (int64_t)3 * k.mean3.h * k.mean3.w;
    const int n = (int)(i / per);
    CombineOutK s = k;
    s.mean3.p = k.mean3.p + (int64_t)n * k.mean3.sn; s.conv3.p = k.conv3.p + (int64_t)n * k.conv3.sn;
    s.dst = k.dst + (int64_t)rows[n] * per;
    s(i - n * per);
  }
};
void combine_output_rows(Ctx& cx, const TV& mean3, const TV& conv3, float* dst_nchw, const std::vector<int>& rows) {
  if (consecutive_rows(mean3, rows)) return combine_output(cx, mean3, conv3, dst_nchw + (int64_t)rows[0] * 3 * mean3.h * mean3.w);
  for (int n0 = 0; n0 < mean3.n; n0 += kGatherMax) {
    const int cnt = std::min(mean3.n - n0, kGatherMax);
    CombineOutRowsK k{};
    k.k = CombineOutK{mean3.batch(n0, cnt), conv3.batch(n0, cnt), dst_nchw};
    for (int i = 0; i < cnt; ++i) k.rows[i] = rows[n0 + i];
    parallel_for(cx, (int64_t)cnt * mean3.h * mean3.w * 3, k, "combine_output_rows");
  }
}

// ---- LPIPS (AlexNet, v0.1; src/utils/lpips) ----
// Input preparation of conv1 (11x11, stride 4, pad 2): NCHW images [in0 batch ; in1 batch] -> the zero-padded image cut into 4x4
// blocks, one 48-channel pixel per block (channel (dy * 4 + dx) * 3 + c), so conv1 becomes a stride-1 3x3 convolution.  Per element,
// in the reference's fp32 operation order: calc_lpips's quantise ((clamp(x, -1, 1) + 1) / 2 * 255, rounded half to even, / 255),
// the module's normalize (2x - 1), ScalingLayer ((x - shift) / scale).  Every operation is explicitly rounded, as in flow_to_image.
struct LpipsPrepK {
  const float* in0; const float* in1; int n, h, w, quantize, normalize; const float* shift; const float* scale; TV dst;
  GV_HD void operator()(int64_t i) const {
    const int ch = (int)(i % 48); int64_t r = i / 48;
    const int xs = (int)(r % dst.w); r /= dst.w;
    const int ys = (int)(r % dst.h); const int n2 = (int)(r / dst.h);
    const int c = ch % 3, k = ch / 3, dx = k % 4, dy = k / 4;
    const int iy = 4 * ys + dy - 2, ix = 4 * xs + dx - 2;
    float v = 0.f;
    if (iy >= 0 && iy < h && ix >= 0 && ix < w) {
      const float* src = n2 < n ? in0 + (int64_t)n2 * 3 * h * w : in1 + (int64_t)(n2 - n) * 3 * h * w;
      v = src[((int64_t)c * h + iy) * w + ix];
      if (quantize) {
        v = fminf(fmaxf(v, -1.f), 1.f);
        v = fv_div(rintf(fv_mul(fv_div(fv_add(v, 1.f), 2.f), 255.f)), 255.f);
      }
      if (normalize) v = fv_add(fv_mul(2.f, v), -1.f);
      v = fv_div(fv_add(v, -shift[c]), scale[c]);
    }
    dst.p[dst.off(n2, ys, xs) + ch] = v;
  }
};
void lpips_prep(Ctx& cx, const float* in0, const float* in1, int n, int h, int w, int quantize, int normalize, const float* shift,
                const float* scale, const TV& dst) {
  if (dst.c != 48 || dst.n != 2 * n || dst.f16) throw std::runtime_error("lpips_prep: dst must be (2n, hs, ws, 48) fp32");
  parallel_for(cx, dst.pixels() * 48, LpipsPrepK{in0, in1, n, h, w, quantize, normalize, shift, scale, dst}, "lpips_prep");
}

// MaxPool2d(3, stride 2), no padding, floor output size (torchvision AlexNet features[2], [5]); NHWC, 4 channels per thread, exact
struct MaxPool3s2K {
  TV src, dst;
  GV_HD void operator()(int64_t i) const {
    const int q = dst.c / 4;
    const int c4 = (int)(i % q); int64_t r = i / q;
    const int x = (int)(r % dst.w); r /= dst.w;
    const int y = (int)(r % dst.h); const int n = (int)(r / dst.h);
    F4 m = ld4(src.p + src.off(n, 2 * y, 2 * x) + 4 * c4);
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx) {
        const F4 v = ld4(src.p + src.off(n, 2 * y + ky, 2 * x + kx) + 4 * c4);
        m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
      }
    st4(dst.p + dst.off(n, y, x) + 4 * c4, m);
  }
};
void maxpool3x3s2(Ctx& cx, const TV& src, const TV& dst) {
  if (src.h < 3 || src.w < 3 || dst.h != (src.h - 3) / 2 + 1 || dst.w != (src.w - 3) / 2 + 1 || dst.n != src.n || dst.c != src.c)
    throw std::runtime_error("maxpool3x3s2: dst must be (n, (h - 3) / 2 + 1, (w - 3) / 2 + 1, c) of src");
  if (!vec4_ok(src) || !vec4_ok(dst)) throw std::runtime_error("maxpool3x3s2: fp32, 16-byte aligned, channels a multiple of 4");
  parallel_for(cx, dst.pixels() * (dst.c / 4), MaxPool3s2K{src, dst}, "maxpool3x3s2");
}

// LPIPS head of one layer: per pixel sum_c w_c (f0_c / (|f0| + 1e-10) - f1_c / (|f1| + 1e-10))^2 (normalize_tensor, the squared
// difference and NetLinLayer's 1x1 convolution), summed along each row in double -> partial[n * h + y].  f holds 2n images: image i
// of in0 at i, of in1 at i + n.  The per-image step adds the rows in a fixed order: no atomics, bit-reproducible.
struct LpipsRowK {
  TV f; int n; const float* lw; double* partial;
  GV_HD void operator()(int64_t row) const {
    const int img = (int)(row / f.h), y = (int)(row % f.h);
    double s = 0.0;
    for (int x = 0; x < f.w; ++x) {
      const float* a = f.p + f.off(img, y, x);
      const float* b = f.p + f.off(img + n, y, x);
      float s0 = 0.f, s1 = 0.f;
      for (int c = 0; c < f.c; ++c) { s0 += a[c] * a[c]; s1 += b[c] * b[c]; }
      const float d0 = sqrtf(s0) + 1e-10f, d1 = sqrtf(s1) + 1e-10f;
      float v = 0.f;
      for (int c = 0; c < f.c; ++c) { const float t = a[c] / d0 - b[c] / d1; v += lw[c] * (t * t); }
      s += (double)v;
    }
    partial[row] = s;
  }
};
struct LpipsImageArgs { const double* partial[5]; int h[5], w[5]; float* per_layer; float* out; };
struct LpipsImageK {
  LpipsImageArgs a;
  GV_HD void operator()(int64_t img) const {
    float tot = 0.f;
    for (int k = 0; k < 5; ++k) {
      double s = 0.0;
      for (int y = 0; y < a.h[k]; ++y) s += a.partial[k][img * a.h[k] + y];
      const float m = (float)(s / ((double)a.h[k] * a.w[k]));
      if (a.per_layer) a.per_layer[img * 5 + k] = m;
      tot += m;
    }
    a.out[img] = tot;
  }
};
#ifndef GV_HOSTSIM
constexpr int LPIPS_MAXV = 12;   // channels per lane: AlexNet's widest ReLU output has 384
// one CTA per row, one warp per pixel (lanes over channels: coalesced), the warp's pixels summed in double by lane 0
__global__ void __launch_bounds__(256) lpips_row_kernel(TV f, int n, const float* __restrict__ lw, double* __restrict__ partial) {
  __shared__ double red[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t rows = (int64_t)n * f.h;
  for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const int img = (int)(row / f.h), y = (int)(row % f.h);
    double acc = 0.0;
    for (int x = warp; x < f.w; x += 8) {
      const float* a = f.p + f.off(img, y, x);
      const float* b = f.p + f.off(img + n, y, x);
      float va[LPIPS_MAXV], vb[LPIPS_MAXV], s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int j = 0; j < LPIPS_MAXV; ++j) {
        const int c = lane + 32 * j;
        va[j] = c < f.c ? a[c] : 0.f; vb[j] = c < f.c ? b[c] : 0.f;
        s0 += va[j] * va[j]; s1 += vb[j] * vb[j];
      }
      for (int o = 16; o; o >>= 1) { s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o); }
      const float d0 = sqrtf(s0) + 1e-10f, d1 = sqrtf(s1) + 1e-10f;
      float v = 0.f;
#pragma unroll
      for (int j = 0; j < LPIPS_MAXV; ++j) {
        const int c = lane + 32 * j;
        if (c < f.c) { const float t = va[j] / d0 - vb[j] / d1; v += lw[c] * (t * t); }
      }
      for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      acc += (double)v;
    }
    if (lane == 0) red[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int k = 0; k < 8; ++k) s += red[k];
      partial[row] = s;
    }
    __syncthreads();
  }
}
// one CTA per image: the rows of each layer in a fixed tree order, in double
__global__ void __launch_bounds__(256) lpips_image_kernel(LpipsImageArgs a) {
  __shared__ double red[256];
  const int img = blockIdx.x;
  float tot = 0.f;
  for (int k = 0; k < 5; ++k) {
    double s = 0.0;
    for (int y = threadIdx.x; y < a.h[k]; y += 256) s += a.partial[k][(int64_t)img * a.h[k] + y];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) {
      if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      const float m = (float)(red[0] / ((double)a.h[k] * a.w[k]));
      if (a.per_layer) a.per_layer[img * 5 + k] = m;
      tot = __fadd_rn(tot, m);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) a.out[img] = tot;
}
#endif
void lpips_head_rows(Ctx& cx, const TV& f, int n, const float* lin_w, double* partial) {
  if (f.n != 2 * n || f.c > 384 || f.f16) throw std::runtime_error("lpips_head_rows: features must be (2n, h, w, <= 384) fp32");
#ifdef GV_HOSTSIM
  parallel_for(cx, (int64_t)n * f.h, LpipsRowK{f, n, lin_w, partial}, "lpips_head_rows");
#else
  if (cx.dry || n <= 0) return;
  const int64_t rows = (int64_t)n * f.h, cap = (int64_t)cx.sm_count * 8;
  cx.launches++;
  if (cx.prof) cx.prof->begin(cx.stream, "lpips_head_rows", (double)rows * f.w * f.c * 2.0);
  lpips_row_kernel<<<(unsigned)(rows < cap ? rows : cap), 256, 0, cx.stream>>>(f, n, lin_w, partial);
  gv_check_launch("lpips_head_rows");
  if (cx.prof) cx.prof->end(cx.stream);
#endif
}
void lpips_head_images(Ctx& cx, const double* const partial[5], const int h[5], const int w[5], int n, float* per_layer, float* out) {
  LpipsImageArgs a;
  for (int k = 0; k < 5; ++k) { a.partial[k] = partial[k]; a.h[k] = h[k]; a.w[k] = w[k]; }
  a.per_layer = per_layer; a.out = out;
#ifdef GV_HOSTSIM
  parallel_for(cx, n, LpipsImageK{a}, "lpips_head_images");
#else
  if (cx.dry || n <= 0) return;
  cx.launches++;
  if (cx.prof) cx.prof->begin(cx.stream, "lpips_head_images", (double)n);
  lpips_image_kernel<<<(unsigned)n, 256, 0, cx.stream>>>(a);
  gv_check_launch("lpips_head_images");
  if (cx.prof) cx.prof->end(cx.stream);
#endif
}

// ---- scene-cut score: PySceneDetect's ContentDetector content value of consecutive uint8 RGB frames ----
// cv2.cvtColor(x, COLOR_RGB2HSV) for 8-bit input in integers (H in [0, 180), S and V in [0, 255]; OpenCV's own fixed-point form):
// sdiv[v] = round(255 * 4096 / v), hdiv[d] = round(180 * 4096 / (6 d)), both 0 at 0.  No quotient falls on a tie, so the integer
// rounding (2a + b) / (2b) is exact.  The tables are built once on the host and ride in the kernel parameters.
GV_HD int scene_sdiv(int v) { return v ? (2 * 255 * 4096 + v) / (2 * v) : 0; }
GV_HD int scene_hdiv(int d) { return d ? (2 * 180 * 4096 + 6 * d) / (12 * d) : 0; }
struct SceneTables { int sdiv[256], hdiv[256]; };
static SceneTables scene_tables() {
  SceneTables t;
  for (int i = 0; i < 256; ++i) { t.sdiv[i] = scene_sdiv(i); t.hdiv[i] = scene_hdiv(i); }
  return t;
}
// one pixel's HSV (v == r wins over v == g, as in OpenCV; the shift of a negative hue is arithmetic)
GV_HD void scene_hsv(int r, int g, int b, const int* sdiv, const int* hdiv, int& H, int& S, int& V) {
  const int v = r > g ? (r > b ? r : b) : (g > b ? g : b);
  const int d = v - (r < g ? (r < b ? r : b) : (g < b ? g : b));
  S = (d * sdiv[v] + 2048) >> 12;
  const int h0 = v == r ? g - b : (v == g ? b - r + 2 * d : r - g + 4 * d);
  const int h = (h0 * hdiv[d] + 2048) >> 12;
  H = h < 0 ? h + 180 : h;
  V = v;
}
// |dH|, |dS|, |dV| of one pixel of a (bytes pa) and b (bytes pb), added to acc
GV_HD void scene_pixel(int ra, int ga, int ba, int rb, int gb, int bb, const int* sdiv, const int* hdiv, uint32_t acc[3]) {
  int h0, s0, v0, h1, s1, v1;
  scene_hsv(ra, ga, ba, sdiv, hdiv, h0, s0, v0);
  scene_hsv(rb, gb, bb, sdiv, hdiv, h1, s1, v1);
  acc[0] += (uint32_t)(h0 > h1 ? h0 - h1 : h1 - h0);
  acc[1] += (uint32_t)(s0 > s1 ? s0 - s1 : s1 - s0);
  acc[2] += (uint32_t)(v0 > v1 ? v0 - v1 : v1 - v0);
}
// the three sums of pixels p0, p0 + step, ... < P of pair (pa, pb); the caller keeps a thread's pixels below 2^32 / 255
GV_HD void scene_pixels(const uint8_t* pa, const uint8_t* pb, int64_t p0, int64_t P, int64_t step, const int* sdiv, const int* hdiv, uint32_t acc[3]) {
  for (int64_t p = p0; p < P; p += step) {
    const uint8_t* x = pa + p * 3; const uint8_t* y = pb + p * 3;
    scene_pixel(x[0], x[1], x[2], y[0], y[1], y[2], sdiv, hdiv, acc);
  }
}
// host simulation: one pair per item, in runs of 2^16 pixels, every sum stored
struct SceneSumsK {
  const uint8_t* a; const uint8_t* b; int64_t P; uint64_t* sums; SceneTables t;
  GV_HD void operator()(int64_t i) const {
    uint64_t s[3] = {0, 0, 0};
    for (int64_t p0 = 0; p0 < P; p0 += 65536) {
      const int64_t cnt = P - p0 < 65536 ? P - p0 : 65536;
      uint32_t acc[3] = {0, 0, 0};
      scene_pixels(a + (i * P + p0) * 3, b + (i * P + p0) * 3, 0, cnt, 1, t.sdiv, t.hdiv, acc);
      for (int c = 0; c < 3; ++c) s[c] += acc[c];
    }
    for (int c = 0; c < 3; ++c) sums[i * 3 + c] = s[c];
  }
};
#ifndef GV_HOSTSIM
constexpr int kSceneThreads = 256;
constexpr int64_t kSceneSmallPixels = 64;   // frames up to this size: one thread per pair
__device__ __forceinline__ void scene_load_tables(const SceneTables& t, int* sdiv, int* hdiv) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) { sdiv[i] = t.sdiv[i]; hdiv[i] = t.hdiv[i]; }
  __syncthreads();
}
// small frames (the 2^24 1x1 pairs of an all-colours check): a thread owns a pair, so it stores its sums; the loads of a warp
// cover 32 consecutive frames
__global__ void __launch_bounds__(kSceneThreads) scene_sums_small_kernel(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, int n,
                                                                       int64_t P, unsigned long long* __restrict__ sums, const __grid_constant__ SceneTables t) {
  __shared__ int sdiv[256], hdiv[256];
  scene_load_tables(t, sdiv, hdiv);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    uint32_t acc[3] = {0, 0, 0};
    scene_pixels(a + i * P * 3, b + i * P * 3, 0, P, 1, sdiv, hdiv, acc);
    for (int c = 0; c < 3; ++c) sums[i * 3 + c] = acc[c];
  }
}
// byte j of 12 little-endian words
__device__ __forceinline__ int scene_byte(const uint32_t* w, int j) { return (int)((w[j >> 2] >> ((j & 3) * 8)) & 0xffu); }
// larger frames: CTA k of a pair's `per_pair` takes every per_pair-th block of 256 units (16 pixels = 3 x 16-byte loads per frame when
// `vec`, else one pixel); the CTA's sums are reduced in registers and shared memory and added with one 64-bit atomic per channel
__global__ void __launch_bounds__(kSceneThreads) scene_sums_kernel(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, int64_t P,
                                                                 int per_pair, int vec, unsigned long long* __restrict__ sums,
                                                                 const __grid_constant__ SceneTables t) {
  __shared__ int sdiv[256], hdiv[256];
  __shared__ unsigned long long red[kSceneThreads / 32][3];
  scene_load_tables(t, sdiv, hdiv);
  const int64_t pair = blockIdx.x / per_pair;
  const int k = blockIdx.x % per_pair;
  const uint8_t* pa = a + pair * P * 3;
  const uint8_t* pb = b + pair * P * 3;
  const int64_t first = (int64_t)k * kSceneThreads + threadIdx.x, step = (int64_t)per_pair * kSceneThreads;
  uint32_t acc[3] = {0, 0, 0};
  if (vec) {
    const uint4* qa = reinterpret_cast<const uint4*>(pa);
    const uint4* qb = reinterpret_cast<const uint4*>(pb);
    for (int64_t g = first; g < P / 16; g += step) {
      uint32_t wa[12], wb[12];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const uint4 x = __ldcs(qa + g * 3 + j), y = __ldcs(qb + g * 3 + j);
        wa[4 * j] = x.x; wa[4 * j + 1] = x.y; wa[4 * j + 2] = x.z; wa[4 * j + 3] = x.w;
        wb[4 * j] = y.x; wb[4 * j + 1] = y.y; wb[4 * j + 2] = y.z; wb[4 * j + 3] = y.w;
      }
#pragma unroll
      for (int p = 0; p < 16; ++p)
        scene_pixel(scene_byte(wa, 3 * p), scene_byte(wa, 3 * p + 1), scene_byte(wa, 3 * p + 2),
                    scene_byte(wb, 3 * p), scene_byte(wb, 3 * p + 1), scene_byte(wb, 3 * p + 2), sdiv, hdiv, acc);
    }
  } else {
    scene_pixels(pa, pb, first, P, step, sdiv, hdiv, acc);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    unsigned long long s = acc[c];
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[warp][c] = s;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    unsigned long long s = 0;
    for (int w = 0; w < kSceneThreads / 32; ++w) s += red[w][threadIdx.x];
    if (s) atomicAdd(sums + pair * 3 + threadIdx.x, s);
  }
}
#endif
void scene_sums(Ctx& cx, const uint8_t* a, const uint8_t* b, int n, int h, int w, uint64_t* sums) {
  if (cx.dry || n <= 0) return;
  const int64_t P = (int64_t)h * w;
  const SceneTables t = scene_tables();
#ifdef GV_HOSTSIM
  parallel_for(cx, n, SceneSumsK{a, b, P, sums, t}, "scene_sums");
#else
  const int64_t cap = (int64_t)cx.sm_count * 8;
  cx.launches++;
  if (cx.prof) cx.prof->begin(cx.stream, "scene_sums", (double)n * P * 6.0);
  unsigned long long* s = reinterpret_cast<unsigned long long*>(sums);
  if (P <= kSceneSmallPixels) {
    const int64_t blocks = std::min(((int64_t)n + kSceneThreads - 1) / kSceneThreads, cap);
    scene_sums_small_kernel<<<(unsigned)blocks, kSceneThreads, 0, cx.stream>>>(a, b, n, P, s, t);
  } else {
    // 16-pixel units when every pair starts on a 16-byte boundary in both stacks (3 P % 16 == 0 <=> P % 16 == 0)
    const int vec = aligned(a, 16) && aligned(b, 16) && P % 16 == 0;
    const int64_t units = vec ? P / 16 : P;
    const int64_t per_pair = std::max<int64_t>(1, std::min((units + kSceneThreads - 1) / kSceneThreads, cap / n));
    const cudaError_t er = cudaMemsetAsync(sums, 0, (size_t)n * 3 * sizeof(uint64_t), cx.stream);
    if (er != cudaSuccess) throw std::runtime_error(std::string("scene_sums: cudaMemsetAsync: ") + cudaGetErrorString(er));
    scene_sums_kernel<<<(unsigned)(n * per_pair), kSceneThreads, 0, cx.stream>>>(a, b, P, (int)per_pair, vec, s, t);
  }
  gv_check_launch("scene_sums");
  if (cx.prof) cx.prof->end(cx.stream);
#endif
}

// ---- shutter blend: one output frame as the mean of its sub-frames (FrameRateConverter's shutter_angle) ----
// The per-pixel arithmetic, shared by the kernel and the host simulation: a channel's float32 sum over the sources in order,
// acc = acc + v with v = x * 255 for a float source and the byte for a uint8 one, then trunc(clamp(acc / n, 0, 255)).  Every operation
// is rounded once (no contraction into an FMA), so n = 1 is pred_to_u8's (x * 255).astype(uint8), and n copies of one byte sum to an
// exact integer that divides back to that byte.
GV_HD float blend_add(float acc, float x, bool f32) { return fv_add(acc, f32 ? fv_mul(x, 255.f) : x); }
GV_HD uint8_t blend_byte(float acc, int n) {
  float v = fv_div(acc, (float)n);
  v = v < 0.f ? 0.f : (v > 255.f ? 255.f : v);
  return (uint8_t)v;
}
struct BlendArgs {
  const void* src[kBlendMax];
  uint64_t f32;   // bit i: source i is a float32 (3,H,W) row, read through the crop; otherwise an (h,w,3) uint8 RGB frame
  uint64_t vec;   // bit i: uint8 source i starts on a 16-byte boundary; bit 63: so does dst
  uint8_t* dst; int n, h, w, H, W, pt, pl, bgr;
};
// host simulation: one item per output byte
struct BlendU8K {
  BlendArgs a;
  GV_HD void operator()(int64_t i) const {
    const int c = (int)(i % 3); const int64_t p = i / 3;
    const int cs = a.bgr ? 2 - c : c;
    const int64_t fo = ((int64_t)cs * a.H + p / a.w + a.pt) * a.W + p % a.w + a.pl;
    float acc = 0.f;
    for (int k = 0; k < a.n; ++k) {
      const bool f = (a.f32 >> k) & 1;
      acc = blend_add(acc, f ? static_cast<const float*>(a.src[k])[fo] : (float)static_cast<const uint8_t*>(a.src[k])[p * 3 + cs], f);
    }
    a.dst[i] = blend_byte(acc, a.n);
  }
};
#ifndef GV_HOSTSIM
constexpr int kBlendThreads = 256, kBlendPerThread = 4;
constexpr int kBlendTile = kBlendThreads * kBlendPerThread;   // pixels per CTA tile: 3072 bytes of a uint8 frame, 192 16-byte words
// `bytes` bytes of a uint8 frame into the tile in shared memory (16-byte words where `vec`, the tail byte by byte), and back out
__device__ __forceinline__ void blend_tile_load(uint8_t* tile, const uint8_t* src, int bytes, bool vec) {
  const int words = vec ? bytes / 16 : 0;
  for (int k = threadIdx.x; k < words; k += kBlendThreads) reinterpret_cast<uint4*>(tile)[k] = __ldcs(reinterpret_cast<const uint4*>(src) + k);
  for (int k = words * 16 + threadIdx.x; k < bytes; k += kBlendThreads) tile[k] = __ldcs(src + k);
}
__device__ __forceinline__ void blend_tile_store(uint8_t* dst, const uint8_t* tile, int bytes, bool vec) {
  const int words = vec ? bytes / 16 : 0;
  for (int k = threadIdx.x; k < words; k += kBlendThreads) reinterpret_cast<uint4*>(dst)[k] = reinterpret_cast<const uint4*>(tile)[k];
  for (int k = words * 16 + threadIdx.x; k < bytes; k += kBlendThreads) dst[k] = tile[k];
}
// A CTA takes tiles of kBlendTile consecutive output pixels; thread x holds pixels x, x + 256, ... of a tile, so a float source is read
// with lanes along x, and a uint8 source goes through shared memory in 16-byte words.  The output is assembled in shared memory and
// stored the same way.  Each source byte is read once (.cs: a sub-frame is not read again).
__global__ void __launch_bounds__(kBlendThreads) blend_u8_kernel(const __grid_constant__ BlendArgs a) {
  __shared__ uint4 words[kBlendTile * 3 / 16];
  uint8_t* tile = reinterpret_cast<uint8_t*>(words);
  const int64_t P = (int64_t)a.h * a.w, plane = (int64_t)a.H * a.W;
  for (int64_t t0 = (int64_t)blockIdx.x * kBlendTile; t0 < P; t0 += (int64_t)gridDim.x * kBlendTile) {
    const int cnt = P - t0 < kBlendTile ? (int)(P - t0) : kBlendTile;
    int64_t fo[kBlendPerThread];
    float acc[kBlendPerThread][3];
#pragma unroll
    for (int q = 0; q < kBlendPerThread; ++q) {
      const int64_t p = t0 + q * kBlendThreads + threadIdx.x;
      fo[q] = (p / a.w + a.pt) * a.W + p % a.w + a.pl;
      acc[q][0] = acc[q][1] = acc[q][2] = 0.f;
    }
    for (int i = 0; i < a.n; ++i) {
      if ((a.f32 >> i) & 1) {
        const float* s = static_cast<const float*>(a.src[i]);
        float v[kBlendPerThread][3];
#pragma unroll
        for (int q = 0; q < kBlendPerThread; ++q)
#pragma unroll
          for (int c = 0; c < 3; ++c) v[q][c] = q * kBlendThreads + (int)threadIdx.x < cnt ? __ldcs(s + c * plane + fo[q]) : 0.f;
#pragma unroll
        for (int q = 0; q < kBlendPerThread; ++q)
#pragma unroll
          for (int c = 0; c < 3; ++c) acc[q][c] = blend_add(acc[q][c], v[q][c], true);
      } else {
        __syncthreads();   // the tile's last contents are consumed
        blend_tile_load(tile, static_cast<const uint8_t*>(a.src[i]) + t0 * 3, cnt * 3, (a.vec >> i) & 1);
        __syncthreads();
#pragma unroll
        for (int q = 0; q < kBlendPerThread; ++q) {
          const int j = q * kBlendThreads + threadIdx.x;
          if (j < cnt)
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[q][c] = blend_add(acc[q][c], (float)tile[j * 3 + c], false);
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kBlendPerThread; ++q) {
      const int j = q * kBlendThreads + threadIdx.x;
      if (j < cnt)
#pragma unroll
        for (int c = 0; c < 3; ++c) tile[j * 3 + c] = blend_byte(a.bgr ? acc[q][2 - c] : acc[q][c], a.n);   // (constant indices: registers)
    }
    __syncthreads();
    blend_tile_store(a.dst + t0 * 3, tile, cnt * 3, (a.vec >> 63) & 1);
  }
}
#endif
void blend_u8(Ctx& cx, const void* const* src, const int* is_f32, int n, int H, int W, int pad_top, int pad_left, uint8_t* dst, int h, int w,
              int bgr) {
  if (cx.dry) return;
  BlendArgs a{};
  int floats = 0;
  for (int i = 0; i < n; ++i) {
    a.src[i] = src[i];
    if (is_f32[i]) { a.f32 |= 1ull << i; ++floats; }
    else if (aligned(src[i], 16)) a.vec |= 1ull << i;
  }
  if (aligned(dst, 16)) a.vec |= 1ull << 63;
  a.dst = dst; a.n = n; a.h = h; a.w = w; a.H = H; a.W = W; a.pt = pad_top; a.pl = pad_left; a.bgr = bgr;
  const int64_t P = (int64_t)h * w;
#ifdef GV_HOSTSIM
  parallel_for(cx, P * 3, BlendU8K{a}, "blend_u8");
#else
  cx.launches++;
  if (cx.prof) cx.prof->begin(cx.stream, "blend_u8", (double)P * (3.0 + 12.0 * floats + 3.0 * (n - floats)));
  const int64_t blocks = std::min((P + kBlendTile - 1) / kBlendTile, (int64_t)cx.sm_count * 8);
  blend_u8_kernel<<<(unsigned)blocks, kBlendThreads, 0, cx.stream>>>(a);
  gv_check_launch("blend_u8");
  if (cx.prof) cx.prof->end(cx.stream);
#endif
}

}  // namespace gv
