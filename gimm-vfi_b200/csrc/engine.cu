// Host orchestration of the GIMM-VFI-R per-pair interpolation path.
// One stream, one pre-planned workspace, zero allocations / host syncs in
// forward().  Reference call stack: gimmvfi_r.py:324-407 (SURVEY.md §3.1).
#include "engine.h"
#include "net.h"
#include "../../include/gimmvfi_b200.h"

#include <algorithm>

namespace gv {

// ---------------------------------------------------------------------------
// device memory helpers
// ---------------------------------------------------------------------------
#ifdef GV_HOSTSIM
void gv_check_launch(const char*) {}
void* dev_alloc(size_t bytes) { return std::malloc(bytes ? bytes : 1); }
void dev_free(void* p) { std::free(p); }
void dev_upload(void* dst, const void* src, size_t bytes) { std::memcpy(dst, src, bytes); }
void dev_download(void* dst, const void* src, size_t bytes, gvStream_t) { std::memcpy(dst, src, bytes); }
void dev_memset(void* dst, int v, size_t bytes, gvStream_t) { std::memset(dst, v, bytes); }
void dev_copy(void* dst, const void* src, size_t bytes, gvStream_t) { std::memcpy(dst, src, bytes); }
void dev_sync(gvStream_t) {}
// hyponet.cu is not part of the host simulation.  hyponet_fused3_resample's layer-0 input is exactly resize_bilinear's output
// (same source index, weights and fp32 expressions), so its emulation resizes into a host buffer and runs the emulated hyponet_fused3.
void hyponet_fused3_resample(Ctx& cx, const TV& lat, const float* coords, const void* blob3, const TV& out) {
  if (lat.c != 32 || lat.f16 || out.c != 2 || out.f16 || out.n != lat.n || lat.pixels() < 1 || out.pixels() < 1) throw std::runtime_error("hyponet_fused3_resample: unsupported tensor layout");
  if (cx.dry) return;
  std::vector<float> buf((size_t)out.n * out.h * out.w * 32);
  const TV r = make_tv(buf.data(), out.n, out.h, out.w, 32);
  const int64_t launches = cx.launches;
  resize_bilinear(cx, lat, r, (float)lat.h / (float)out.h, (float)lat.w / (float)out.w, 1.f, 0, ACT_NONE);
  hyponet_fused3(cx, r, coords, blob3, out);
  cx.launches = launches + 1;   // one kernel on the device
}
// The activation forms of the fused kernels, one pixel per call: the arithmetic of tests/hostsim/tc_hostsim.cu's emulation of
// hyponet_fused / hyponet_fused3 with hypo_act<ACT> in place of sin.  FAST: TF32 latent operands and half activations and weights
// (hypo:: blob); else fp32 layers 0 and 4 and the 22-bit hi + lo pairs of layers 1-3 (hypo3:: blob).
static float tf32_trunc_emu(float x) { uint32_t u; std::memcpy(&u, &x, 4); u &= 0xffffe000u; float y; std::memcpy(&y, &u, 4); return y; }
static float f16_round(float v) { return gv_f16_to_f32(gv_f32_to_f16(v)); }
template <bool FAST, int ACT> struct HypoNetEmuK {
  TV lat, out; const float* coords; const uint8_t* blob; float w0;
  float ldf(size_t off) const { float v; std::memcpy(&v, blob + off, 4); return v; }
  float ldh(size_t off) const { uint16_t h; std::memcpy(&h, blob + off, 2); return gv_f16_to_f32(h); }
  void operator()(int64_t pix) const {
    const int x = (int)(pix % lat.w); int64_t r = pix / lat.w; const int y = (int)(r % lat.h); const int n = (int)(r / lat.h);
    const float* lp = lat.p + lat.off(n, y, x);
    const float* c = coords + pix * 3;
    float a[128], b[128];
    auto pair = [](float v) { const float hi = f16_round(v); return hi + f16_round(v - hi); };
    for (int o = 0; o < 128; ++o) {
      if constexpr (FAST) {
        float acc = 0.f;
        for (int k = 0; k < 32; ++k) acc += tf32_trunc_emu(lp[k]) * ldf(hypo::W0 + hypo::swz(o, k * 4));
        const float* aff = reinterpret_cast<const float*>(blob + hypo::AFF);
        const float z = std::fmaf(c[0], aff[o], std::fmaf(c[1], aff[128 + o], std::fmaf(c[2], aff[256 + o], acc + aff[384 + o])));
        a[o] = f16_round(hypo_act<ACT>(z, w0));
      } else {
        const float* W0 = reinterpret_cast<const float*>(blob + hypo3::W0A);
        float z = W0[35 * 128 + o];
        for (int k = 0; k < 35; ++k) z = std::fmaf(k < 32 ? lp[k] : c[k - 32], W0[k * 128 + o], z);
        a[o] = pair(hypo_act<ACT>(z, w0));
      }
    }
    for (int l = 0; l < 3; ++l) {
      for (int o = 0; o < 128; ++o) {
        float acc = 0.f;
        for (int k = 0; k < 128; ++k) {
          const size_t e = (size_t)(k / 64) * 16384 + hypo::swz(o, (k % 64) * 2);
          acc += a[k] * (FAST ? ldh(hypo::W1 + l * 32768 + e) : ldh(hypo3::W13 + (l * 2 + 0) * 2 * 16384 + e) + ldh(hypo3::W13 + (l * 2 + 1) * 2 * 16384 + e));
        }
        if constexpr (FAST) {
          b[o] = f16_round(hypo_act<ACT>(acc + ldf(hypo::B1 + l * 512 + 4 * o), w0));
        } else {
          const float s = hypo_act<ACT>(acc / hypo3::W_SCALE + ldf(hypo3::B13 + l * 512 + 4 * o), w0);
          b[o] = l < 2 ? pair(s) : s;
        }
      }
      std::memcpy(a, b, sizeof a);
    }
    for (int o = 0; o < 2; ++o) {
      float acc = 0.f;
      if constexpr (FAST) {
        for (int k = 0; k < 128; ++k) acc += a[k] * ldh(hypo::W4 + (k / 64) * 2048 + hypo::swz(o, (k % 64) * 2));
        out.p[out.off(n, y, x) + o] = acc + ldf(hypo::B4 + 4 * o);
      } else {
        for (int k = 0; k < 128; ++k) acc = std::fmaf(a[k], ldf(hypo3::W4 + 4 * (k * 2 + o)), acc);
        out.p[out.off(n, y, x) + o] = acc + ldf(hypo3::B4 + 4 * o);
      }
    }
  }
};
template <bool FAST>
static void hypo_emu(Ctx& cx, const TV& lat, const float* coords, const void* blob, const TV& out, int act, float w0) {
  if (lat.c != 32 || lat.f16 || out.c != 2 || out.f16 || out.n != lat.n || out.h != lat.h || out.w != lat.w) throw std::runtime_error("hyponet: unsupported tensor layout");
  const uint8_t* bl = static_cast<const uint8_t*>(blob);
  const int64_t P = lat.pixels();
  switch (act) {
    case HYPO_SIREN: parallel_for(cx, P, HypoNetEmuK<FAST, HYPO_SIREN>{lat, out, coords, bl, w0}, "hyponet_act"); break;
    case HYPO_RELU: parallel_for(cx, P, HypoNetEmuK<FAST, HYPO_RELU>{lat, out, coords, bl, w0}, "hyponet_act"); break;
    case HYPO_SILU: parallel_for(cx, P, HypoNetEmuK<FAST, HYPO_SILU>{lat, out, coords, bl, w0}, "hyponet_act"); break;
    case HYPO_DAMP: parallel_for(cx, P, HypoNetEmuK<FAST, HYPO_DAMP>{lat, out, coords, bl, w0}, "hyponet_act"); break;
    default: throw std::runtime_error("hyponet: unknown activation");
  }
}
void hyponet_fused_act(Ctx& cx, const TV& lat, const float* coords, const void* blob, const TV& out, int act, float w0) {
  if (act == HYPO_SIREN1) return hyponet_fused(cx, lat, coords, blob, out);
  hypo_emu<true>(cx, lat, coords, blob, out, act, w0);
}
void hyponet_fused3_act(Ctx& cx, const TV& lat, const float* coords, const void* blob3, const TV& out, int act, float w0) {
  if (act == HYPO_SIREN1) return hyponet_fused3(cx, lat, coords, blob3, out);
  hypo_emu<false>(cx, lat, coords, blob3, out, act, w0);
}
void hyponet_fused3_resample_act(Ctx& cx, const TV& lat, const float* coords, const void* blob3, const TV& out, int act, float w0) {
  if (act == HYPO_SIREN1) return hyponet_fused3_resample(cx, lat, coords, blob3, out);
  if (lat.c != 32 || lat.f16 || out.c != 2 || out.f16 || out.n != lat.n || lat.pixels() < 1 || out.pixels() < 1) throw std::runtime_error("hyponet_fused3_resample: unsupported tensor layout");
  if (cx.dry) return;
  std::vector<float> buf((size_t)out.n * out.h * out.w * 32);
  const TV r = make_tv(buf.data(), out.n, out.h, out.w, 32);
  const int64_t launches = cx.launches;
  resize_bilinear(cx, lat, r, (float)lat.h / (float)out.h, (float)lat.w / (float)out.w, 1.f, 0, ACT_NONE);
  hypo_emu<false>(cx, r, coords, blob3, out, act, w0);
  cx.launches = launches + 1;
}
#else
static void cuda_ok(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string("CUDA error in ") + what + ": " + cudaGetErrorString(e));
}
void gv_check_launch(const char* what) { cuda_ok(cudaGetLastError(), what); }
void* dev_alloc(size_t bytes) { void* p = nullptr; cuda_ok(cudaMalloc(&p, bytes ? bytes : 1), "cudaMalloc"); return p; }
void dev_free(void* p) { cudaFree(p); }
void dev_upload(void* dst, const void* src, size_t bytes) { cuda_ok(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice), "cudaMemcpy H2D"); }
void dev_download(void* dst, const void* src, size_t bytes, gvStream_t s) {
  cuda_ok(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s), "cudaMemcpy D2H");
  cuda_ok(cudaStreamSynchronize(s), "sync");
}
void dev_memset(void* dst, int v, size_t bytes, gvStream_t s) { cuda_ok(cudaMemsetAsync(dst, v, bytes, s), "cudaMemsetAsync"); }
void dev_copy(void* dst, const void* src, size_t bytes, gvStream_t s) { cuda_ok(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s), "cudaMemcpy D2D"); }
void dev_sync(gvStream_t s) { cuda_ok(cudaStreamSynchronize(s), "cudaStreamSynchronize"); }
#endif

// RAII: make the engine's device current for the duration of a call and restore the caller's (an engine on cuda:1 must
// not change torch's current device, and its uploads / launches must not land on whatever device happens to be current)
struct DeviceGuard {
#ifndef GV_HOSTSIM
  int prev = -1; bool switched = false;
  explicit DeviceGuard(int dev) {
    cuda_ok(cudaGetDevice(&prev), "cudaGetDevice");
    if (prev != dev) { cuda_ok(cudaSetDevice(dev), "cudaSetDevice"); switched = true; }
  }
  ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
#else
  explicit DeviceGuard(int) {}
#endif
  DeviceGuard(const DeviceGuard&) = delete; DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// ---------------------------------------------------------------------------
// Profiler (CUDA events around every launch; off by default)
// ---------------------------------------------------------------------------
const char* prof_intern(const std::string& s) {
  static std::map<std::string, std::string> pool;
  auto it = pool.find(s);
  if (it == pool.end()) it = pool.emplace(s, s).first;
  return it->second.c_str();
}
#ifdef GV_HOSTSIM
void* Profiler::get_event() { return nullptr; }
void Profiler::begin(gvStream_t, const char*, double) {}
void Profiler::end(gvStream_t) {}
Profiler::~Profiler() {}
#else
void* Profiler::get_event() {
  if (used == pool.size()) { cudaEvent_t e; cuda_ok(cudaEventCreate(&e), "cudaEventCreate"); pool.push_back(e); }
  return pool[used++];
}
void Profiler::begin(gvStream_t s, const char* name, double work) {
  ProfRec r; r.name = name; r.work = work; r.ev0 = get_event(); r.ev1 = get_event();
  cuda_ok(cudaEventRecord((cudaEvent_t)r.ev0, s), "cudaEventRecord");
  recs.push_back(r);
}
void Profiler::end(gvStream_t s) { cuda_ok(cudaEventRecord((cudaEvent_t)recs.back().ev1, s), "cudaEventRecord"); }
Profiler::~Profiler() { for (void* e : pool) cudaEventDestroy((cudaEvent_t)e); }
#endif

std::string Engine::profile_json(gvStream_t stream) {
  std::string out = "{";
  DeviceGuard dg(device_);
#ifndef GV_HOSTSIM
  cuda_ok(cudaStreamSynchronize(stream), "sync");
  struct Acc { double ms = 0, work = 0; int64_t n = 0; };
  std::map<std::string, Acc> acc;
  for (const ProfRec& r : prof_.recs) {
    float ms = 0.f;
    cuda_ok(cudaEventElapsedTime(&ms, (cudaEvent_t)r.ev0, (cudaEvent_t)r.ev1), "cudaEventElapsedTime");
    Acc& a = acc[r.name]; a.ms += ms; a.work += r.work; a.n++;
  }
  bool first = true;
  for (auto& kv : acc) {
    char buf[256];
    snprintf(buf, sizeof buf, "%s\"%s\": {\"ms\": %.6f, \"work\": %.6e, \"launches\": %lld}", first ? "" : ", ", kv.first.c_str(), kv.second.ms,
             kv.second.work, (long long)kv.second.n);
    out += buf; first = false;
  }
#else
  (void)stream;
#endif
  return out + "}";
}

// ---------------------------------------------------------------------------
// Engine: weights
// ---------------------------------------------------------------------------
Engine::Engine(int device) : device_(device) {
  if (const char* kn = getenv("GIMMVFI_RAFT_CORR_DIRECT")) raft_direct_ = atoi(kn);            // 1: always volume-free, 0: never, unset: by size
#ifndef GV_HOSTSIM
  int count = 0;
  cuda_ok(cudaGetDeviceCount(&count), "cudaGetDeviceCount");
  if (device < 0 || device >= count) throw std::runtime_error("gimmvfi: no CUDA device " + std::to_string(device));
  int sms = 132;
  cuda_ok(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device), "cudaDeviceGetAttribute");   // (no cudaSetDevice: the caller's current device stays)
  sm_count_ = sms;
  cudaDeviceProp prop;
  cuda_ok(cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties");
  // the rest of a forward's plan grows with the pixel count as the pyramid's square root does: at a pyramid of 0.4 x the device memory
  // (32 GB on an 80 GB board, a ~3.5 Mpx pair) it is ~35 GB, so the volume path still fits with room for the caller's tensors
  raft_direct_auto_bytes_ = 0.4 * (double)prop.totalGlobalMem;
#endif
  if (const char* kn = getenv("GIMMVFI_RAFT_CORR_DIRECT_GB")) raft_direct_auto_bytes_ = atof(kn) * 1e9;
}

Engine::~Engine() { drop_weights(); }

void Engine::load_weight(const std::string& key, const float* host, const int64_t* shape, int ndim) {
  HostTensor t;
  int64_t n = 1;
  for (int i = 0; i < ndim; ++i) { t.shape.push_back(shape[i]); n *= shape[i]; }
  t.data.assign(host, host + n);
  raw_[key] = std::move(t);
  held_ = Weights::None;
}

// Frees the device weights, with every pointer into them, and the graphs recorded on them.  A frame cache stored under the old
// weights must not be loaded again.
void Engine::drop_weights() {
  DeviceGuard dg(device_);
  for (void* p : dev_allocs_) dev_free(p);
  dev_allocs_.clear(); conv_.clear(); vec_.clear();
  fc_valid_.clear(); ++weights_version_; clear_graphs();
  held_ = Weights::None;
  hypo_blob_ = hypo_blob3_ = nullptr;
  g9_ = alpha_fe_ = alpha_v_ = nullptr;
}

void Engine::need(Entry e) const {
  using W = Weights;
  auto mask = [](std::initializer_list<W> ws) { unsigned m = 0; for (W w : ws) m |= 1u << (int)w; return m; };
  // per Entry: the weights a refusal names as missing, and the weight sets that serve the entry point
  struct EntryRule { const char* needs; unsigned served; };
  static const EntryRule kEntries[] = {
      {"GIMM-VFI-R or GIMM-VFI-F", mask({W::R, W::F})},                 // plan, forward
      {"synthesis", mask({W::R, W::F, W::Synthesis})},                  // plan_from_flow, forward_from_flow
      {"GIMM", mask({W::R, W::F, W::Synthesis, W::Gimm})},              // plan_gimm, forward_gimm, gimmvfi_op_hyponet
      {"RAFT", mask({W::R, W::Raft})},                                  // plan_raft, forward_raft
      {"FlowFormer", mask({W::F, W::FlowFormer})},                      // plan_flowformer, forward_flowformer
      {"LPIPS", mask({W::Lpips})},                                      // plan_lpips, forward_lpips
  };
  // per Weights after None: the set's name, the call that loads it and the entry point it is loaded for
  struct HeldName { const char* name; const char* finalize; const char* use; };
  static const HeldName kHeld[] = {
      {"GIMM-VFI-R", "finalize_weights", "forward"},
      {"GIMM-VFI-F", "finalize_weights_f", "forward"},
      {"synthesis", "finalize_weights_synthesis", "forward_from_flow"},
      {"GIMM", "finalize_weights_gimm", "forward_gimm"},
      {"RAFT", "finalize_weights_raft", "forward_raft"},
      {"FlowFormer", "finalize_weights_flowformer", "forward_flowformer"},
      {"LPIPS", "finalize_weights_lpips", "forward_lpips"},
  };
  const EntryRule& r = kEntries[(int)e];
  if (r.served >> (int)held_ & 1u) return;
  const std::string msg = std::string("gimmvfi: no ") + r.needs + " weights were loaded";
  if (held_ == W::None) throw std::runtime_error(msg + " (finalize_weights* has not been called)");
  const HeldName& h = kHeld[(int)held_ - 1];
  throw std::runtime_error(msg + ": this engine holds " + h.name + " weights only (" + h.finalize + "); use " + h.use);
}

const HostTensor& Engine::raw(const std::string& key) const {
  auto it = raw_.find(key);
  if (it == raw_.end()) throw std::runtime_error("gimmvfi: missing weight '" + key + "'");
  return it->second;
}

const float* Engine::upload(const std::vector<float>& v) {
  void* d = dev_alloc(v.size() * sizeof(float));
  dev_allocs_.push_back(d);
  dev_upload(d, v.data(), v.size() * sizeof(float));
  return static_cast<const float*>(d);
}

const float* Engine::vec(const std::string& key) {
  auto it = vec_.find(key);
  if (it != vec_.end()) return it->second;
  const float* d = upload(raw(key).data);
  vec_[key] = d;
  return d;
}

// Conv2d weight (cout,cin,kh,kw) -> [tap][cin][cout_ld]; optional eval-mode BatchNorm
// folding (bn = name of the BatchNorm2d), output scale and output-channel permutation.
ConvW Engine::pack_conv(const std::string& name, const std::string& bn, float out_scale, const std::vector<int>* perm) {
  const HostTensor& W = raw(name + ".weight");
  if (W.shape.size() != 4 && W.shape.size() != 2) throw std::runtime_error("gimmvfi: '" + name + ".weight' is neither a Conv2d (4-D) nor a Linear (2-D) weight");
  const bool lin = W.shape.size() == 2;   // nn.Linear (cout, cin) = a 1x1 convolution over tokens laid out as an NHWC map
  const int cout = (int)W.shape[0], cin = (int)W.shape[1], kh = lin ? 1 : (int)W.shape[2], kw = lin ? 1 : (int)W.shape[3];
  HostTensor zero_bias;
  if (!raw_.count(name + ".bias")) { zero_bias.shape = {cout}; zero_bias.data.assign(cout, 0.f); }   // bias=False layers
  const HostTensor& Bv = raw_.count(name + ".bias") ? raw(name + ".bias") : zero_bias;
  std::vector<float> s(cout, out_scale), sh(cout, 0.f);
  if (!bn.empty()) {
    const auto& g = raw(bn + ".weight").data; const auto& be = raw(bn + ".bias").data;
    const auto& mu = raw(bn + ".running_mean").data; const auto& var = raw(bn + ".running_var").data;
    for (int co = 0; co < cout; ++co) {
      float k = g[co] / std::sqrt(var[co] + 1e-5f);
      s[co] = k * out_scale; sh[co] = (be[co] - mu[co] * k) * out_scale;
    }
  }
  const int cout_ld = (cout + 3) & ~3;
  std::vector<float> pw((size_t)kh * kw * cin * cout_ld, 0.f), pb(((tc_cout_pad(cout) + 31) & ~31) + 128, 0.f);  // bias padded past any tensor-core N tiling (float4 reads)
  for (int co = 0; co < cout; ++co) {
    const int src = perm ? (*perm)[co] : co;
    for (int ci = 0; ci < cin; ++ci)
      for (int t = 0; t < kh * kw; ++t)
        pw[((size_t)t * cin + ci) * cout_ld + co] = W.data[((size_t)src * cin + ci) * kh * kw + t] * s[src];
    pb[co] = Bv.data[src] * s[src] + sh[src];
  }
  ConvW c;
  c.w = upload(pw); c.b = upload(pb); c.cin = cin; c.cout = cout; c.kh = kh; c.kw = kw; c.cout_ld = cout_ld;
  pack_tc(c, pw);
  // layers of the final decoder's residual trunk read half-precision activations in precision mode 3 (run())
  if (name.rfind("amt_final_decoder.convblock.", 0) == 0 && name.rfind("amt_final_decoder.convblock.0", 0) != 0) pack_tc_f16(c, pw);
  // precision mode 4 (experimental): the 32/64-channel full-resolution chains are stored in half as well -> their consumers
  static const char* const kHalfFed[] = {"cnn_encoder.3.", "cnn_encoder.4.", "cnn_encoder.5.", "cnn_encoder.7", "res_conv.1", "res_conv.3.", "res_conv.5",
                                         "amt_final_decoder.upsample.3.", "amt_final_decoder.upsample.4.", "amt_final_decoder.upsample.5.",
                                         "amt_final_decoder.upsample.6.", "amt_final_decoder.upsample.7", "amt_init_decoder.convblock.1.",
                                         "amt_init_decoder.convblock.2.", "amt_init_decoder.convblock.3.", "amt_init_decoder.convblock.4",
                                         "amt_final_decoder.convblock.0."};
  for (const char* pre : kHalfFed)
    if (name.rfind(pre, 0) == 0) { pack_tc_f16(c, pw); break; }
  conv_[name] = c;
  return c;
}

// round-to-nearest-even to TF32 (10-bit mantissa): the tensor core ignores the low 13 bits
static float tf32_rn(float x) {
  uint32_t u; std::memcpy(&u, &x, 4);
  if ((u & 0x7f800000u) == 0x7f800000u) return x;
  u += 0xfffu + ((u >> 13) & 1u);
  u &= 0xffffe000u;
  float y; std::memcpy(&y, &u, 4);
  return y;
}

// [tap][cin][cout_ld] fp32  ->  [2][tap][cout_pad][cin_pad]: plane 0 = TF32(w) (K-major rows for the wgmma B
// operand), plane 1 = TF32(w - plane0), the low term of the 3xTF32 split
void Engine::pack_tc(ConvW& c, const std::vector<float>& pw) {
  const int cout_pad = tc_cout_pad(c.cout), cin_pad = (c.cin + 31) & ~31, taps = c.kh * c.kw;
  const size_t plane = (size_t)taps * cout_pad * cin_pad;
  std::vector<float> t(2 * plane, 0.f);
  for (int tp = 0; tp < taps; ++tp)
    for (int ci = 0; ci < c.cin; ++ci)
      for (int co = 0; co < c.cout; ++co) {
        const float w = pw[((size_t)tp * c.cin + ci) * c.cout_ld + co];
        const float hi = tf32_rn(w);
        const size_t o = ((size_t)tp * cout_pad + co) * cin_pad + ci;
        t[o] = hi; t[plane + o] = tf32_rn(w - hi);
      }
  c.w_tc = upload(t); c.cout_pad = cout_pad; c.cin_pad = cin_pad; c.has_lo = true;
  // fp16 hi / lo planes of w * 2^e for the 3xF16 split: 64-element K blocks (two 32-channel fp32 activation boxes per K step)
  {
    float mx = 0.f;
    for (float v : pw) mx = std::max(mx, std::fabs(v));
    int e = 0;
    if (mx > 0.f) { int ex; std::frexp(mx, &ex); e = 14 - ex; }   // mx * 2^e in [2^13, 2^14)
    if (e > 24) e = 24;
    if (e < -24) e = -24;
    const float sc = std::ldexp(1.f, e);
    const int cps = (c.cin + 63) & ~63;
    const size_t pl = (size_t)taps * cout_pad * cps;
    std::vector<float> hs((2 * pl + 1) / 2, 0.f);
    uint16_t* h = reinterpret_cast<uint16_t*>(hs.data());
    for (int tp = 0; tp < taps; ++tp)
      for (int ci = 0; ci < c.cin; ++ci)
        for (int co = 0; co < c.cout; ++co) {
          const float w = pw[((size_t)tp * c.cin + ci) * c.cout_ld + co] * sc;
          const uint16_t hi = gv_f32_to_f16(w), lo = gv_f32_to_f16(w - gv_f16_to_f32(hi));
          const size_t o = ((size_t)tp * cout_pad + co) * cps + ci;
          h[o] = hi; h[pl + o] = lo;
        }
    c.w_tc_s = upload(hs); c.cin_pad_s = cps; c.w_scale = sc;
  }
}

// [tap][cin][cout_ld] fp32 -> [tap][cout_pad][cin_pad_h] fp16 (K-major rows of 64-element / 128-byte K blocks): the
// B operand of the f16 tensor-core path for layers whose activations are stored in half precision
void Engine::pack_tc_f16(ConvW& c, const std::vector<float>& pw) {
  const int cout_pad = tc_cout_pad(c.cout), cin_pad = (c.cin + 63) & ~63, taps = c.kh * c.kw;
  std::vector<float> t(((size_t)taps * cout_pad * cin_pad + 1) / 2, 0.f);
  uint16_t* h = reinterpret_cast<uint16_t*>(t.data());
  for (int tp = 0; tp < taps; ++tp)
    for (int ci = 0; ci < c.cin; ++ci)
      for (int co = 0; co < c.cout; ++co)
        h[((size_t)tp * cout_pad + co) * cin_pad + ci] = gv_f32_to_f16(pw[((size_t)tp * c.cin + ci) * c.cout_ld + co]);
  c.w_tc_h = upload(t); c.cin_pad_h = cin_pad;
}

// RAFT stem (7x7, stride 2, cin 3) with the x-taps packed into the channel axis: on a zero-padded image with
// 4-float pixels, the 7 x-taps of one kernel row are 28 contiguous floats, so the conv becomes a (7 x 1) kernel
// over 28 "channels" (K = 7 x 28 instead of 49 taps x 3-of-16 used lanes: 3.5x fewer K chunks).
void Engine::pack_stem(const std::string& name, const std::string& bn) {
  const HostTensor& W = raw(name + ".weight");
  const HostTensor& Bv = raw(name + ".bias");
  const int cout = (int)W.shape[0], cin = (int)W.shape[1], kh = (int)W.shape[2], kw = (int)W.shape[3];
  if (cin != 3 || kh != 7 || kw != 7) throw std::runtime_error("pack_stem: expected a 7x7 conv on 3 channels");
  std::vector<float> s(cout, 1.f), sh(cout, 0.f);
  if (!bn.empty()) {
    const auto& g = raw(bn + ".weight").data; const auto& be = raw(bn + ".bias").data;
    const auto& mu = raw(bn + ".running_mean").data; const auto& var = raw(bn + ".running_var").data;
    for (int co = 0; co < cout; ++co) { float k = g[co] / std::sqrt(var[co] + 1e-5f); s[co] = k; sh[co] = be[co] - mu[co] * k; }
  }
  const int cout_ld = (cout + 3) & ~3, K = 28;
  std::vector<float> pw((size_t)kh * K * cout_ld, 0.f), pb(((tc_cout_pad(cout) + 31) & ~31) + 128, 0.f);
  for (int co = 0; co < cout; ++co) {
    for (int ky = 0; ky < kh; ++ky)
      for (int kx = 0; kx < kw; ++kx)
        for (int c = 0; c < 3; ++c)
          pw[((size_t)ky * K + kx * 4 + c) * cout_ld + co] = W.data[(((size_t)co * cin + c) * kh + ky) * kw + kx] * s[co];
    pb[co] = Bv.data[co] * s[co] + sh[co];
  }
  ConvW c;
  c.w = upload(pw); c.b = upload(pb); c.cin = K; c.cout = cout; c.kh = kh; c.kw = 1; c.cout_ld = cout_ld;
  pack_tc(c, pw);   // stride 2 runs on the tensor-core path too (TMA element strides)
  conv_[name + "#xpacked"] = c;
}

// k x k convolutions (k = 7, 5) on few channels with the x-taps packed into the channel axis (see pack_stem): the input is a
// zero-padded copy with `ldp` floats per pixel, the kernel becomes (k x 1) over K = k*ldp "channels" - k K-step groups instead of k*k.
void Engine::pack_xpacked(const std::string& name, int ldp) {
  const HostTensor& W = raw(name + ".weight");
  const HostTensor& Bv = raw(name + ".bias");
  const int cout = (int)W.shape[0], cin = (int)W.shape[1], kh = (int)W.shape[2], kw = (int)W.shape[3];
  if (kh != kw || cin > ldp) throw std::runtime_error("pack_xpacked: expected a k x k conv with cin <= ldp");
  const int cout_ld = (cout + 3) & ~3, K = kw * ldp;
  std::vector<float> pw((size_t)kh * K * cout_ld, 0.f), pb(((tc_cout_pad(cout) + 31) & ~31) + 128, 0.f);
  for (int co = 0; co < cout; ++co) {
    for (int ky = 0; ky < kh; ++ky)
      for (int kx = 0; kx < kw; ++kx)
        for (int c = 0; c < cin; ++c)
          pw[((size_t)ky * K + kx * ldp + c) * cout_ld + co] = W.data[(((size_t)co * cin + c) * kh + ky) * kw + kx];
    pb[co] = Bv.data[co];
  }
  ConvW c;
  c.w = upload(pw); c.b = upload(pb); c.cin = K; c.cout = cout; c.kh = kh; c.kw = 1; c.cout_ld = cout_ld;
  pack_tc(c, pw);
  conv_[name + "#xp"] = c;
}

void Engine::finalize_weights() {
  DeviceGuard dg(device_);
  drop_weights();
  finalize_raft();
  // --- feature projections (gimmvfi_r.py:51-53)
  pack_conv("amt_last_cproj"); pack_conv("amt_second_last_cproj"); pack_conv("amt_fproj");
  finalize_decoders();
  finalize_gimm_part();
  held_ = Weights::R;
}

// RAFT's parameters (raft/raft.py:62-70) under flow_estimator.: shared by GIMM-VFI-R and the RAFT module alone
void Engine::finalize_raft() {
  // --- RAFT encoders (raft/extractor.py:122-171); cnet's BatchNorm is folded
  for (int e = 0; e < 2; ++e) {
    const std::string p = e == 0 ? "flow_estimator.fnet" : "flow_estimator.cnet";
    const bool bn = e == 1;
    pack_conv(p + ".conv1", bn ? p + ".norm1" : "");
    pack_stem(p + ".conv1", bn ? p + ".norm1" : "");
    for (int li = 1; li <= 3; ++li)
      for (int bi = 0; bi < 2; ++bi) {
        const std::string q = p + ".layer" + std::to_string(li) + "." + std::to_string(bi);
        pack_conv(q + ".conv1", bn ? q + ".norm1" : "");
        pack_conv(q + ".conv2", bn ? q + ".norm2" : "");
        if (bi == 0 && li > 1) pack_conv(q + ".downsample.0", bn ? q + ".downsample.1" : "");
      }
    pack_conv(p + ".conv2");
  }
  // --- RAFT update block (raft/update.py:94-154)
  const std::string u = "flow_estimator.update_block";
  for (const char* n : {".encoder.convc1", ".encoder.convc2", ".encoder.convf1", ".encoder.convf2", ".encoder.conv",
                        ".gru.convz1", ".gru.convr1", ".gru.convq1", ".gru.convz2", ".gru.convr2", ".gru.convq2",
                        ".flow_head.conv1", ".flow_head.conv2", ".mask.0"})
    pack_conv(u + n);
  for (const char* sfx : {"1", "2"}) {   // z | r gates read the same input: one 384 -> 256 convolution (raft/update.py:47-49,55-57)
    const HostTensor& wz = raw(u + ".gru.convz" + sfx + ".weight"); const HostTensor& wr = raw(u + ".gru.convr" + sfx + ".weight");
    const HostTensor& bz = raw(u + ".gru.convz" + sfx + ".bias"); const HostTensor& br = raw(u + ".gru.convr" + sfx + ".bias");
    HostTensor w = wz, b = bz;
    w.shape[0] = wz.shape[0] + wr.shape[0]; w.data.insert(w.data.end(), wr.data.begin(), wr.data.end());
    b.shape[0] = bz.shape[0] + br.shape[0]; b.data.insert(b.data.end(), br.data.begin(), br.data.end());
    raw_[u + ".gru.convzr" + sfx + ".weight"] = w; raw_[u + ".gru.convzr" + sfx + ".bias"] = b;
    pack_conv(u + ".gru.convzr" + sfx);
    // The GRU input is [h | inp | motion features] (raft/update.py:122-124) and `inp` (the context network's output) does not change
    // over the iterations: its share of every gate convolution is computed once per pair ("_inp", carries the bias) and enters the
    // per-iteration convolutions over [h | motion] ("_hm", K = 256 instead of 384) as a pre-activation term.
    for (const char* gate : {"zr", "q"}) {
      const std::string g = u + ".gru.conv" + gate + sfx;
      const HostTensor& wf = raw(g + ".weight"); const HostTensor& bf = raw(g + ".bias");
      const int64_t co = wf.shape[0], ci = wf.shape[1], kk = wf.shape[2] * wf.shape[3];
      if (ci != 384) throw std::runtime_error("gimmvfi: SepConvGRU input width");
      HostTensor w_hm, w_in, b0 = bf;
      w_hm.shape = {co, 256, wf.shape[2], wf.shape[3]}; w_in.shape = {co, 128, wf.shape[2], wf.shape[3]};
      for (int64_t o = 0; o < co; ++o)
        for (int64_t c = 0; c < ci; ++c) {
          std::vector<float>& dst = (c >= 128 && c < 256) ? w_in.data : w_hm.data;
          dst.insert(dst.end(), wf.data.begin() + (o * ci + c) * kk, wf.data.begin() + (o * ci + c + 1) * kk);
        }
      std::fill(b0.data.begin(), b0.data.end(), 0.f);
      raw_[g + "_hm.weight"] = w_hm; raw_[g + "_hm.bias"] = b0;
      raw_[g + "_inp.weight"] = w_in; raw_[g + "_inp.bias"] = bf;
      pack_conv(g + "_hm"); pack_conv(g + "_inp");
    }
  }
  pack_conv(u + ".mask.2", "", 0.25f);  // "scale mask to balance gradients" raft/update.py:153
  pack_xpacked(u + ".encoder.convf1", 4);
}

// A flow estimator loaded on its own: the keys under its children's prefixes are moved under GIMM-VFI's "flow_estimator." prefix
// (replacing what an earlier load left there), so reloading one engine with other weights takes the new ones.
void Engine::prefix_flow_estimator(std::initializer_list<const char*> children) {
  std::vector<std::string> bare;
  for (const auto& kv : raw_)
    for (const char* top : children)
      if (kv.first.compare(0, std::strlen(top), top) == 0) bare.push_back(kv.first);
  for (const std::string& k : bare) { raw_["flow_estimator." + k] = std::move(raw_[k]); raw_.erase(k); }
}

// The RAFT module alone (the reference's initialize_RAFT(), raft/__init__.py:7-24)
void Engine::finalize_weights_raft() {
  DeviceGuard dg(device_);
  drop_weights();
  prefix_flow_estimator({"fnet.", "cnet.", "update_block."});   // the module's three children (raft.py:62-70)
  finalize_raft();
  held_ = Weights::Raft;
}

// AMT decoders / update blocks / combine block (fi_components.py:229-305): shared by GIMM-VFI-R and -F
void Engine::finalize_decoders() {
  // --- decoders (fi_components.py:229-305)
  {
    const std::string p = "amt_init_decoder";
    for (int i = 1; i <= 5; ++i) { pack_conv(p + ".upsample." + std::to_string(i) + ".0"); vec(p + ".upsample." + std::to_string(i) + ".1.weight"); }
    pack_conv(p + ".upsample.6", p + ".upsample.7");
    pack_conv(p + ".convblock.0.0"); vec(p + ".convblock.0.1.weight");
    // head re-ordered to [ft(128) | dflow0(2) | dflow1(2) | mask(1)] so ft_ is an aligned slice
    std::vector<int> perm(133);
    for (int i = 0; i < 128; ++i) perm[i] = 5 + i;
    for (int i = 0; i < 5; ++i) perm[128 + i] = i;
    pack_conv(p + ".convblock.4", "", 1.f, &perm);
  }
  {
    const std::string p = "amt_final_decoder";
    for (int i = 2; i <= 6; ++i) { pack_conv(p + ".upsample." + std::to_string(i) + ".0"); vec(p + ".upsample." + std::to_string(i) + ".1.weight"); }
    pack_conv(p + ".upsample.7", p + ".upsample.8");
    pack_conv(p + ".convblock.0.0"); vec(p + ".convblock.0.1.weight");
    pack_conv(p + ".convblock.4");
  }
  for (const char* d : {"amt_init_decoder", "amt_final_decoder"})
    for (int k = 1; k <= 3; ++k) {
      const std::string q = std::string(d) + ".convblock." + std::to_string(k);
      for (int c = 1; c <= 4; ++c) { pack_conv(q + ".conv" + std::to_string(c) + ".0"); vec(q + ".conv" + std::to_string(c) + ".1.weight"); }
      pack_conv(q + ".conv5"); vec(q + ".prelu.weight");
    }
  for (const char* d : {"amt_update4_low", "amt_update4_high"})
    for (const char* n : {".convc1", ".convc2", ".convf1", ".convf2", ".conv", ".gru.0", ".gru.2", ".feat_head.0", ".feat_head.2", ".flow_head.0", ".flow_head.2"})
      pack_conv(std::string(d) + n);
  pack_conv("amt_comb_block.0"); vec("amt_comb_block.1.weight"); pack_conv("amt_comb_block.2");
  pack_xpacked("amt_comb_block.0", 12); pack_xpacked("amt_comb_block.2", 20);
  pack_xpacked("amt_update4_low.convf1", 4); pack_xpacked("amt_update4_high.convf1", 4);
  pack_xpacked("amt_final_decoder.upsample.2.0", 8);   // 5x5 on 8 channels at full resolution: 5 x 40 lanes instead of 25 taps x 8-of-32 lanes
}

// GIMM-VFI-F's parameter tree minus flow_estimator.* (gimmvfi_f.py:37-111): the synthesis half runs natively on the outputs of an
// external flow estimator (forward_from_flow); there are no feature projections in F (twins features are used as they are)
void Engine::finalize_weights_synthesis() {
  DeviceGuard dg(device_);
  drop_weights();
  finalize_decoders();
  finalize_gimm_part();
  held_ = Weights::Synthesis;
}

// GIMM-VFI-F complete (gimmvfi_f.py:27-111): the synthesis half + the native FlowFormer estimator (flowformer.cu)
void Engine::finalize_weights_f() {
  DeviceGuard dg(device_);
  drop_weights();
  finalize_decoders();
  finalize_gimm_part();
  finalize_flowformer();
  held_ = Weights::F;
}

// The FlowFormer module alone (the reference's initialize_Flowformer(), flowformer/__init__.py): its state_dict keys, with or without
// GIMM-VFI-F's "flow_estimator." prefix.
void Engine::finalize_weights_flowformer() {
  DeviceGuard dg(device_);
  drop_weights();
  prefix_flow_estimator({"memory_encoder.", "memory_decoder.", "context_encoder."});   // the module's three children (transformer.py:29-39)
  finalize_flowformer();
  held_ = Weights::FlowFormer;
}

void Engine::tap_copy(Ctx& cx, const std::string& name, const TV& tv) {
  if (!debug_) return;
  tap_copy_to(cx, name, tv, cx.arena.tensor(tv.n, tv.h, tv.w, tv.c));
}

void Engine::tap_copy_to(Ctx& cx, const std::string& name, const TV& tv, const TV& snap) {
  if (!debug_) return;
  copy_channels(cx, tv, snap);
  taps_[name] = snap;
}

// GIMM's own parameters (gimm.py:36-80 == gimmvfi_r.py:86-111): motion encoder, latent refiner, HypoNet, splat-metric scalars
void Engine::finalize_gimm_part() {
  motion_ = motion_next_;
  const bool nw = motion_.normalize_weight;
  const float ob = motion_.output_bias;
  // --- GIMM encoders (gimmvfi_r.py:86-109)
  for (const char* n : {"cnn_encoder.0", "cnn_encoder.1", "cnn_encoder.3.layers.0", "cnn_encoder.3.layers.2", "cnn_encoder.4.layers.0",
                        "cnn_encoder.4.layers.2", "cnn_encoder.5.layers.0", "cnn_encoder.5.layers.2", "cnn_encoder.7", "res_conv.0",
                        "res_conv.1", "res_conv.3.layers.0", "res_conv.3.layers.2", "res_conv.5"})
    pack_conv(n);
  // --- HypoNet (hyponet.py:99-143): fan-in-normalised columns, bias row, +output_bias on the last layer
  for (int l = 0; l < 5; ++l) {
    const std::string key = "hyponet.params_dict.linear_wb" + std::to_string(l);
    const HostTensor& wb = raw(key);
    const int fin = (int)wb.shape[0] - 1, fout = (int)wb.shape[1];
    const int ld = (fout + 3) & ~3;
    std::vector<float> pw((size_t)fin * ld, 0.f), pb(((tc_cout_pad(fout) + 31) & ~31) + 128, 0.f);
    for (int co = 0; co < fout; ++co) {
      double nrm = 0.0;
      for (int ci = 0; ci < fin; ++ci) { double v = wb.data[(size_t)ci * fout + co]; nrm += v * v; }
      float d = nw ? std::max((float)std::sqrt(nrm), 1e-12f) : 1.f;
      for (int ci = 0; ci < fin; ++ci) pw[(size_t)ci * ld + co] = wb.data[(size_t)ci * fout + co] / d;
      pb[co] = wb.data[(size_t)fin * fout + co] + (l == 4 ? ob : 0.f);
    }
    ConvW c; c.w = upload(pw); c.b = upload(pb); c.cin = fin; c.cout = fout; c.kh = c.kw = 1; c.cout_ld = ld;
    pack_tc(c, pw);
    if (l >= 1) pack_tc_f16(c, pw);   // precision mode 4: the sin() activations between the layers (|x| <= 1) are stored in half
    conv_[key] = c;
  }
  // --- the same five matrices packed for the fused kernel (hyponet.cu): pre-swizzled K-major tiles, fp32 affine rows for (t, y, x)
  {
    std::vector<float> blobf((hypo::BLOB + 3) / 4, 0.f);
    uint8_t* blob = reinterpret_cast<uint8_t*>(blobf.data());
    auto norm_col = [&](const HostTensor& wb, int fin, int fout, int co) {
      if (!nw) return 1.f;
      double nrm = 0.0;
      for (int ci = 0; ci < fin; ++ci) { double v = wb.data[(size_t)ci * fout + co]; nrm += v * v; }
      return std::max((float)std::sqrt(nrm), 1e-12f);
    };
    const HostTensor& w0 = raw("hyponet.params_dict.linear_wb0");
    if (w0.shape[0] != 36 || w0.shape[1] != 128) throw std::runtime_error("hyponet: expected linear_wb0 of shape (36, 128)");
    float* aff = reinterpret_cast<float*>(blob + hypo::AFF);
    for (int n = 0; n < 128; ++n) {
      const float d = norm_col(w0, 35, 128, n);
      for (int k = 0; k < 32; ++k) { const float v = tf32_rn(w0.data[(size_t)k * 128 + n] / d); std::memcpy(blob + hypo::W0 + hypo::swz(n, k * 4), &v, 4); }
      for (int j = 0; j < 3; ++j) aff[j * 128 + n] = w0.data[(size_t)(32 + j) * 128 + n] / d;
      aff[3 * 128 + n] = w0.data[(size_t)35 * 128 + n];
    }
    for (int l = 1; l <= 4; ++l) {
      const HostTensor& wb = raw("hyponet.params_dict.linear_wb" + std::to_string(l));
      const int fout = (int)wb.shape[1];
      if (wb.shape[0] != 129 || fout != (l < 4 ? 128 : 2)) throw std::runtime_error("hyponet: unexpected hidden / output layer shape");
      const int rows = l < 4 ? 128 : 16, base = l < 4 ? hypo::W1 + (l - 1) * 32768 : hypo::W4, kb_bytes = rows * 128;
      float* bias = reinterpret_cast<float*>(blob + (l < 4 ? hypo::B1 + (l - 1) * 512 : hypo::B4));
      for (int n = 0; n < fout; ++n) {
        const float d = norm_col(wb, 128, fout, n);
        for (int k = 0; k < 128; ++k) {
          const uint16_t h = gv_f32_to_f16(wb.data[(size_t)k * fout + n] / d);
          std::memcpy(blob + base + (k / 64) * kb_bytes + hypo::swz(n, (k % 64) * 2), &h, 2);
        }
        bias[n] = wb.data[(size_t)128 * fout + n] + (l == 4 ? ob : 0.f);
      }
    }
    hypo_blob_ = upload(blobf);
    // fp32-class variant (hyponet_fused3): scaled fp16 hi / lo planes of layers 1-3, fp32 rows of layers 0 and 4
    std::vector<float> b3f((hypo3::BLOB + 3) / 4, 0.f);
    uint8_t* b3 = reinterpret_cast<uint8_t*>(b3f.data());
    float* w0a = reinterpret_cast<float*>(b3 + hypo3::W0A);
    for (int n = 0; n < 128; ++n) {
      const float d = norm_col(w0, 35, 128, n);
      for (int k = 0; k < 35; ++k) w0a[k * 128 + n] = w0.data[(size_t)k * 128 + n] / d;
      w0a[35 * 128 + n] = w0.data[(size_t)35 * 128 + n];
    }
    for (int l = 1; l <= 3; ++l) {
      const HostTensor& wb = raw("hyponet.params_dict.linear_wb" + std::to_string(l));
      float* bias = reinterpret_cast<float*>(b3 + hypo3::B13 + (l - 1) * 512);
      for (int n = 0; n < 128; ++n) {
        const float d = norm_col(wb, 128, 128, n);
        for (int k = 0; k < 128; ++k) {
          const float v = wb.data[(size_t)k * 128 + n] / d * hypo3::W_SCALE;
          const uint16_t hi = gv_f32_to_f16(v), lo = gv_f32_to_f16(v - gv_f16_to_f32(hi));
          std::memcpy(b3 + hypo3::W13 + (((l - 1) * 2 + 0) * 2 + k / 64) * 16384 + hypo::swz(n, (k % 64) * 2), &hi, 2);
          std::memcpy(b3 + hypo3::W13 + (((l - 1) * 2 + 1) * 2 + k / 64) * 16384 + hypo::swz(n, (k % 64) * 2), &lo, 2);
        }
        bias[n] = wb.data[(size_t)128 * 128 + n];
      }
    }
    {
      const HostTensor& wb = raw("hyponet.params_dict.linear_wb4");
      float* w4 = reinterpret_cast<float*>(b3 + hypo3::W4);
      float* b4 = reinterpret_cast<float*>(b3 + hypo3::B4);
      for (int n = 0; n < 2; ++n) {
        const float d = norm_col(wb, 128, 2, n);
        for (int k = 0; k < 128; ++k) w4[k * 2 + n] = wb.data[(size_t)k * 2 + n] / d;
        b4[n] = wb.data[(size_t)128 * 2 + n] + ob;
      }
    }
    hypo_blob3_ = upload(b3f);
  }
  g9_ = vec("g_filter"); alpha_fe_ = vec("alpha_fe"); alpha_v_ = vec("alpha_v");
}

// standalone GIMM checkpoint (SURVEY 8(f) row 4): only the keys of gimm.py's module tree are present
void Engine::finalize_weights_gimm() {
  DeviceGuard dg(device_);
  drop_weights();
  finalize_gimm_part();
  held_ = Weights::Gimm;
}


// ---------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------
static ConvW slice_cout(const ConvW& w, int co0, int cnt) {
  ConvW s = w; s.w = w.w + co0; s.b = w.b + co0; s.cout = cnt; s.w_tc = nullptr;  // TC layout is not sliceable this way
  return s;
}

// raft/extractor.py:173-220.  x: (n,H,W,3) -> fmap (n,H/8,W/8,256) [+ layer2/layer3 outputs]
static void raft_encoder(Net& N, const std::string& p, bool instance, const TV& x, const TV& xpad /*zero-padded by 3, 4-float pixels*/,
                         const TV& out256, TV* feat4, TV* feat8,
                         const ConvW* split_tanh_relu_out /*cnet: tanh/relu halves*/, const TV& net_out, const TV& inp_out) {
  Ctx& cx = N.cx; Arena& A = cx.arena;
  const int n = x.n, H2 = x.h / 2, W2 = x.w / 2;
  float* mr = nullptr; float* scratch = nullptr;
  if (instance) {
    mr = A.alloc_f((size_t)n * 128 * 2);
    TV probe = make_tv(nullptr, n, H2, W2, 128);
    scratch = A.alloc_f((size_t)instnorm_scratch_floats(probe));
  }
  auto norm_act = [&](const TV& raw, int act1, const TV& res, int act2, const TV& dst) {
    instnorm_stats(cx, raw, mr, scratch, 0);
    instnorm_apply(cx, raw, mr, act1, res, act2, dst);
  };
  // stem
  TV a = A.tensor(n, H2, W2, 64);
  auto stem = [&](const TV& dst, int act) {   // 7x7 stride-2 stem through the x-packed weights (pack_stem)
    TV in = xpad; in.c = 28;
    ConvGeom g; g.stride = 2; g.ph = 0; g.pw = 0; g.loose_w = 1;
    ConvEpi e; e.act1 = act;
    conv2d(cx, in, TV(), N.W(p + ".conv1#xpacked"), g, e, dst);   // (tensor-core path: TMA element strides take every 2nd pixel)
  };
  if (instance) {
    TV r = A.tensor(n, H2, W2, 64);
    stem(r, ACT_NONE);
    norm_act(r, ACT_RELU, TV(), ACT_NONE, a);
  } else {
    stem(a, ACT_RELU);
  }
  TV cur = a;
  int cin = 64;
  const int dims[3] = {64, 96, 128};
  for (int li = 1; li <= 3; ++li) {
    const int dim = dims[li - 1];
    for (int bi = 0; bi < 2; ++bi) {
      const std::string q = p + ".layer" + std::to_string(li) + "." + std::to_string(bi);
      const int stride = (bi == 0 && li > 1) ? 2 : 1;
      const int oh = cur.h / stride, ow = cur.w / stride;
      TV y1 = A.tensor(n, oh, ow, dim), y2 = A.tensor(n, oh, ow, dim), outb = A.tensor(n, oh, ow, dim);
      TV skip = cur;
      if (instance) {
        TV r = A.tensor(n, oh, ow, dim);
        N.conv(q + ".conv1", cur, r, ACT_NONE, nullptr, stride);
        norm_act(r, ACT_RELU, TV(), ACT_NONE, y1);
        N.conv(q + ".conv2", y1, r, ACT_NONE);
        if (stride != 1) {
          TV d = A.tensor(n, oh, ow, dim);
          N.conv(q + ".downsample.0", cur, d, ACT_NONE, nullptr, stride);
          norm_act(d, ACT_NONE, TV(), ACT_NONE, y2);  // y2 reused as the normalised skip
          skip = y2;
        }
        norm_act(r, ACT_RELU, skip, ACT_RELU, outb);  // relu(x + relu(norm2(conv2)))
      } else {
        N.conv(q + ".conv1", cur, y1, ACT_RELU, nullptr, stride);
        if (stride != 1) { N.conv(q + ".downsample.0", cur, y2, ACT_NONE, nullptr, stride); skip = y2; }
        ConvEpi e; e.act1 = ACT_RELU; e.res = skip; e.act2 = ACT_RELU;
        N.conv_e(q + ".conv2", y1, TV(), outb, e);
      }
      cur = outb; cin = dim;
    }
    if (li == 2 && feat4) *feat4 = cur;
    if (li == 3 && feat8) *feat8 = cur;
  }
  (void)cin;
  if (split_tanh_relu_out) {
    // cnet: net = tanh(first 128), inp = relu(last 128)  (raft/raft.py:133-136)
    const ConvW& w = *split_tanh_relu_out;
    ConvEpi e1; e1.act1 = ACT_TANH;
    conv2d(cx, cur, TV(), slice_cout(w, 0, 128), ConvGeom(), e1, net_out);
    ConvEpi e2; e2.act1 = ACT_RELU;
    conv2d(cx, cur, TV(), slice_cout(w, 128, 128), ConvGeom(), e2, inp_out);
  } else {
    N.conv(p + ".conv2", cur, out256);
  }
}

struct Pyramid {
  float* lvl[4]; int h[4], w[4]; int64_t N;  // rows per sample
  CorrPyr view(int sample0) const {
    CorrPyr c;
    for (int l = 0; l < 4; ++l) { c.lvl[l] = lvl[l] + (int64_t)sample0 * N * h[l] * w[l]; c.h[l] = h[l]; c.w[l] = w[l]; }
    c.rows_per_sample = N;
    return c;
  }
};

// Maximal runs of consecutive pairs whose source and target frames are consecutive as well: {first pair, pairs}.  A run is one batched
// call of the per-sample kernels (GIMM-VFI-R's two directions, (b, B + b) then (B + b, b), are two runs).
static std::vector<std::pair<int, int>> pair_runs(const std::vector<int>& src, const std::vector<int>& tgt) {
  std::vector<std::pair<int, int>> r;
  for (int s = 0; s < (int)src.size(); ++s)
    if (!r.empty() && src[s] == src[s - 1] + 1 && tgt[s] == tgt[s - 1] + 1) ++r.back().second;
    else r.push_back({s, 1});
  return r;
}

// One volume per pair on the batch axis: sample s holds <F[src[s]], F[tgt[s]]> (GIMM-VFI-R's second direction is the transposed
// volume, raft/corr.py:32).  Level l is (P*N) x (h_l*w_l).
// tc: 0 = fp32 CUDA-core GEMM, 1 = wgmma plain TF32, 2 = wgmma 3xF16 (corr_gemm_3xf16) or 3xTF32 (promoted accumulation)
static Pyramid build_pyramid(Ctx& cx, const TV& F /*frames,h,w,256*/, const std::vector<int>& src, const std::vector<int>& tgt, int tensor_cores) {
  Arena& A = cx.arena;
  const int S = (int)src.size();
  Pyramid P; P.N = (int64_t)F.h * F.w;
  int h = F.h, w = F.w;
  for (int l = 0; l < 4; ++l) { P.h[l] = h; P.w[l] = w; P.lvl[l] = A.alloc_f((size_t)S * P.N * h * w); h /= 2; w /= 2; }
  const float scale = 1.0f / std::sqrt((float)F.c);
  if (tensor_cores && F.c % 32 == 0 && F.ld % 4 == 0 && F.ld == F.c) {
    // wgmma GEMMs; the other frame's features act as the K-major "weights".  Level l > 0 is the GEMM against the 2^l x 2^l
    // AVERAGE-POOLED target features: avg_pool2d of the volume over the target axes (raft/corr.py:139-142) commutes with the dot
    // product, so the pooled levels (1/4 + 1/16 + 1/64 of level 0) cost a third more GEMM work and the 8.5 GB level-0 volume
    // (1088x1920) is never re-read (the pooling pass over it took as long as the GEMM that wrote it).
    const bool split = tensor_cores >= 2;
    const size_t mk = A.mark();
    TV Fl[4]; Fl[0] = F;
    for (int l = 1; l < 4; ++l) { Fl[l] = A.tensor(F.n, P.h[l], P.w[l], F.c); avgpool2_features(cx, Fl[l - 1], Fl[l]); }
    if (split && corr_volume_tc_wants_f16_planes() && F.c % 64 == 0) {
      // 3xF16 on pre-split operands: every frame's features are split once per level; a frame's level-0 planes are the sources of
      // its own pairs and the targets of the reverse direction
      uint16_t* pl[4]; int64_t plane[4];
      for (int l = 0; l < 4; ++l) {
        plane[l] = (int64_t)F.n * P.h[l] * P.w[l] * F.c;
        pl[l] = reinterpret_cast<uint16_t*>(A.alloc_f((size_t)plane[l]));   // 2 half planes
        if (P.h[l] * P.w[l] > 0) split_planes_f16(cx, Fl[l], pl[l]);
      }
      for (int s = 0; s < S; ++s)
        for (int l = 0; l < 4; ++l) {
          const int nt = P.h[l] * P.w[l];
          if (nt <= 0 || cx.dry) continue;
          corr_gemm_3xf16(cx, pl[0] + (int64_t)src[s] * P.N * F.c, plane[0], (int)P.N, pl[l] + (int64_t)tgt[s] * nt * F.c, plane[l], nt, F.c, scale,
                          P.lvl[l] + (int64_t)s * P.N * nt);
        }
      A.release(mk);
      return P;
    }
    const int64_t plane = (int64_t)P.N * F.c;
    float* planes = A.alloc_f((size_t)2 * plane);
    const int64_t nz = ((P.N + 255) / 256) * 256 + 512;
    float* zeros = A.alloc_f((size_t)nz);
    if (!cx.dry) dev_memset(zeros, 0, (size_t)nz * sizeof(float), cx.stream);
    for (int s = 0; s < S; ++s) {
      const int other = tgt[s];
      for (int l = 0; l < 4; ++l) {
        const int nt = P.h[l] * P.w[l];
        if (nt <= 0) continue;
        if (split && corr_volume_tc_wants_f16_planes()) split_planes_f16(cx, Fl[l].batch(other, 1), planes);
        else if (split) split_planes(cx, Fl[l].batch(other, 1), planes);
        if (!cx.dry) corr_volume_tc(cx, F.batch(src[s], 1), split ? planes : Fl[l].batch(other, 1).p, zeros, P.lvl[l] + (int64_t)s * P.N * nt, scale, split, nt);
      }
    }
    A.release(mk);
    return P;
  } else
  {
    for (const auto& run : pair_runs(src, tgt))
      corr_volume(cx, F.batch(src[run.first], run.second), F.batch(tgt[run.first], run.second), P.lvl[0] + (int64_t)run.first * P.N * P.N, scale);
  }
  corr_pool_pyramid(cx, P.lvl[0], P.lvl[1], P.lvl[2], P.lvl[3], (int64_t)S * P.N, P.h[0], P.w[0]);
  return P;
}

// AMT update block (fi_components.py:157-222).  `ft` (128 ch view) and `fl4` (4 ch) are updated in place.
static void amt_update(Net& N, const std::string& p, bool low, const TV& ft, const TV& fl4, const TV& flow_in /*4ch at block res*/,
                       const TV& corr648) {
  Ctx& cx = N.cx; Arena& A = cx.arena;
  const size_t mk = A.mark();
  const int n = corr648.n, h = corr648.h, w = corr648.w;
  TV inp = A.tensor(n, h, w, 320);
  if (low) resize_bilinear(cx, ft, inp.slice(192, 128), 2.f, 2.f, 1.f, 0, ACT_NONE);  // resize(net, 1/2)
  else copy_channels(cx, ft, inp.slice(192, 128));
  copy_channels(cx, flow_in, inp.slice(188, 4));
  TV cor = A.tensor(n, h, w, 256), cf = A.tensor(n, h, w, 256), flo = A.tensor(n, h, w, 128);
  N.conv(p + ".convc1", corr648, cor, ACT_LRELU);
  N.conv(p + ".convc2", cor, cf.slice(0, 192), ACT_LRELU);
  N.conv7x(p + ".convf1", flow_in, flo, ACT_LRELU);
  N.conv(p + ".convf2", flo, cf.slice(192, 64), ACT_LRELU);
  N.conv(p + ".conv", cf, inp.slice(0, 188), ACT_LRELU);
  TV g1 = A.tensor(n, h, w, 192), g2 = A.tensor(n, h, w, 192), hd = A.tensor(n, h, w, 192);
  N.conv(p + ".gru.0", inp, g1, ACT_LRELU);
  N.conv(p + ".gru.2", g1, g2);
  TV dnet = A.tensor(n, h, w, 128), dflow = A.tensor(n, h, w, 4);
  N.conv(p + ".feat_head.0", g2, hd, ACT_LRELU);
  N.conv(p + ".feat_head.2", hd, dnet);
  N.conv(p + ".flow_head.0", g2, hd, ACT_LRELU);
  N.conv(p + ".flow_head.2", hd, dflow);
  if (low) {
    resize_bilinear(cx, dnet, ft, 0.5f, 0.5f, 1.f, 1, ACT_NONE);
    resize_bilinear(cx, dflow, fl4, 0.5f, 0.5f, 2.f, 1, ACT_NONE);
  } else {
    add_inplace_slices(cx, ft, dnet);
    add_inplace_slices(cx, fl4, dflow);
  }
  A.release(mk);
}

// ResBlock (fi_components.py:97-154), in place on x.
static void resblock(Net& N, const std::string& q, const TV& x, int C, int S) {
  Ctx& cx = N.cx; Arena& A = cx.arena;
  const size_t mk = A.mark();
  TV a = A.tensor_like(x, C), b = A.tensor_like(x, C), s1 = A.tensor_like(x, S), s2 = A.tensor_like(x, S);
  N.convrelu(q + ".conv1", x, a);
  N.convrelu(q + ".conv2", a.slice(C - S, S), s1);
  { ConvEpi e; e.act1 = ACT_PRELU; e.slope1 = N.V(q + ".conv3.1.weight"); N.conv_e(q + ".conv3.0", a.slice(0, C - S), s1, b, e); }
  N.convrelu(q + ".conv4", b.slice(C - S, S), s2);
  { ConvEpi e; e.res = x; e.act2 = ACT_PRELU; e.slope2 = N.V(q + ".prelu.weight"); N.conv_e(q + ".conv5", b.slice(0, C - S), s2, x, e); }
  A.release(mk);
}

struct RaftPrepK {  // image = 2 * ((255 * x) / 255) - 1   (gimmvfi_r.py:349 + raft/raft.py:111-112)
  TV src, dst;
  GV_HD void operator()(int64_t i) const {
    float v = src.p[i];
    dst.p[i] = 2.f * ((255.f * v) / 255.0f) - 1.0f;
  }
};
struct FlowFormerPrepK {  // NCHW frames in [0,255] -> NHWC 2 * (x / 255.0) - 1.0   (transformer.py:51-52; RAFT: raft.py:111-112)
  const float* src; TV dst;
  GV_HD void operator()(int64_t i) const {
    const int x = (int)(i % dst.w); int64_t r = i / dst.w;
    const int y = (int)(r % dst.h); r /= dst.h;
    const int c = (int)(r % 3); const int n = (int)(r / 3);
    dst.p[dst.off(n, y, x) + c] = 2.f * (src[i] / 255.0f) - 1.0f;
  }
};
struct ScaleShiftK {  // y = a*x + b on a dense tensor
  const float* src; float* dst; float a, b;
  GV_HD void operator()(int64_t i) const { dst[i] = a * src[i] - b; }
};

// dst sample i <- src sample idx[i]: a clip's per-frame products into pair order.  Whole samples (padding lanes included) as 16- or
// 4-byte words; the sample list rides in the kernel parameters, kGatherMax samples per launch.
struct alignas(16) Word16 { uint32_t v[4]; };
template <class Wd> struct GatherSamplesK {
  const Wd* src; Wd* dst; int64_t words; int idx[kGatherMax];
  GV_HD void operator()(int64_t i) const {
    const int64_t n = i / words, k = i - n * words;
    dst[i] = src[(int64_t)idx[n] * words + k];
  }
};
template <class Wd> static void gather_samples_as(Ctx& cx, const TV& src, const std::vector<int>& idx, const TV& dst, int64_t bytes) {
  const int64_t words = bytes / (int64_t)sizeof(Wd);
  for (size_t i0 = 0; i0 < idx.size(); i0 += kGatherMax) {
    GatherSamplesK<Wd> k{};
    const int cnt = (int)std::min(idx.size() - i0, (size_t)kGatherMax);
    for (int i = 0; i < cnt; ++i) k.idx[i] = idx[i0 + i];
    k.src = reinterpret_cast<const Wd*>(src.p);
    k.dst = reinterpret_cast<Wd*>(dst.at((int64_t)i0 * dst.sn));
    k.words = words;
    parallel_for(cx, (int64_t)cnt * words, k, "clip_gather");
  }
}
static void gather_samples(Ctx& cx, const TV& src, const std::vector<int>& idx, const TV& dst) {
  if (src.f16 != dst.f16 || src.sn != dst.sn || src.h != dst.h || src.w != dst.w || src.ld != dst.ld || dst.n != (int)idx.size())
    throw std::runtime_error("clip_gather: source and destination samples differ in shape");
  for (int i : idx) if (i < 0 || i >= src.n) throw std::runtime_error("clip_gather: sample index out of range");
  const int64_t bytes = src.sn * (src.f16 ? 2 : 4);
  if (bytes % 16 == 0 && aligned(src.p, 16) && aligned(dst.p, 16)) gather_samples_as<Word16>(cx, src, idx, dst, bytes);
  else gather_samples_as<uint32_t>(cx, src, idx, dst, bytes);
}

static bool is_identity(const std::vector<int>& idx) {
  for (size_t i = 0; i < idx.size(); ++i) if (idx[i] != (int)i) return false;
  return true;
}

static void check_problem(const Problem& p) {
  if (p.B < 1 || p.T < 1) throw std::runtime_error("gimmvfi: B and T must be >= 1");
  const int H = p.H(), W = p.W();
  if (H % 8 || W % 8 || H < 128 || W < 128)
    throw std::runtime_error("gimmvfi: network resolution must be a multiple of 8 and >= 128 (got " + std::to_string(H) + "x" + std::to_string(W) + ")");
  if (p.Hc != H || p.Wc != W)
    throw std::runtime_error("gimmvfi: coordinate grid must match the network resolution (frame_synthesize consumes flow_t at that size)");
}

// What run() interpolates: the caller frames it reads, the pairs of them, and the output rows of each timestep slot.  The pairs are
// ordered by timestep count, descending, so that slot k runs over the B_k pairs that have more than k timesteps, a prefix: every
// per-pair buffer is batch-major, and slot k works on .batch(0, B_k) views.  One builder per input form validates it and fills this in.
struct Schedule {
  struct Load { int64_t off, sn, sc; int f0, n; };   // io.img_xs + off, sample / channel strides sn / sc -> engine frames [f0, f0 + n)
  std::vector<Load> loads;
  int F = 0;                          // engine frames
  std::vector<int> src, tgt;          // pair p interpolates from engine frame src[p] to tgt[p]
  std::vector<int> pair_rows;         // pair p's row of raft_flow / nflow
  std::vector<std::vector<int>> rows; // slot k: the output row of each of its B_k pairs
  std::vector<float> t;               // the t of every output row; empty: io.t / io.coords at the slot's rows (then consecutive)
  int per_call = 1;                   // FlowFormer: pairs per reference call
  int decide_as = 2;                  // RAFT: choose the lookup path as a run of this many pairs would (0: the pair count)
  bool frame_cache = false;           // the R frame cache (set_frame_cache) may be used
};

// forward_clip(): the F frames of a (F,3,Hf,Wf) input and P = B pairs of them, T timesteps each.  Pair p takes the paths of forward() with
// B = 1 on its frames: one FlowFormer call per direction, and RAFT's lookup chosen for 2 directions (the clip's workspace holds 2P volumes).
static Schedule schedule_clip(const Problem& p, const Clip& c) {
  check_problem(p);
  if ((int)c.src.size() != p.B || (int)c.tgt.size() != p.B) throw std::runtime_error("gimmvfi clip: problem batch must equal the number of pairs");
  for (int i = 0; i < p.B; ++i)
    if (c.src[i] < 0 || c.src[i] >= c.F || c.tgt[i] < 0 || c.tgt[i] >= c.F)
      throw std::runtime_error("gimmvfi clip: pair " + std::to_string(i) + " = (" + std::to_string(c.src[i]) + ", " + std::to_string(c.tgt[i]) +
                               ") indexes outside the " + std::to_string(c.F) + " frames");
  Schedule s;
  s.loads = {{0, 3 * (int64_t)p.Hf * p.Wf, (int64_t)p.Hf * p.Wf, 0, c.F}};
  s.F = c.F; s.src = c.src; s.tgt = c.tgt;
  s.rows.resize(p.T);
  for (int b = 0; b < p.B; ++b) {
    s.pair_rows.push_back(b);
    for (int k = 0; k < p.T; ++k) s.rows[k].push_back(k * p.B + b);
  }
  return s;
}

// forward(): a clip of the frame stack [I0 batch ; I1 batch] of a (B,3,2,Hf,Wf) input and its B pairs (b, B + b), which the estimators
// run batched, and the only form the frame cache serves
static Schedule schedule_batch(const Problem& p) {
  Clip c; c.F = 2 * p.B;
  for (int b = 0; b < p.B; ++b) { c.src.push_back(b); c.tgt.push_back(p.B + b); }
  Schedule s = schedule_clip(p, c);
  const int64_t hw = (int64_t)p.Hf * p.Wf;
  s.loads = {{0, 6 * hw, 2 * hw, 0, p.B}, {hw, 6 * hw, 2 * hw, p.B, p.B}};
  s.per_call = p.B; s.decide_as = 0; s.frame_cache = true;
  return s;
}

// forward_queries(): the queries' distinct pairs, their timesteps in query order and the per-query t.  Only the frames some query uses are
// read and encoded.  The problem's B and T are those of the list.
static Schedule schedule_queries(const Problem& p, const Queries& qs) {
  const int Q = (int)qs.src.size(), F = qs.F;
  if (Q < 1) throw std::runtime_error("gimmvfi queries: at least one query is required");
  if (F < 1) throw std::runtime_error("gimmvfi queries: at least one frame is required");
  if ((int)qs.tgt.size() != Q || (int)qs.t.size() != Q) throw std::runtime_error("gimmvfi queries: src, tgt and t differ in length");
  std::map<std::pair<int, int>, int> pair_of;   // (src, tgt) -> distinct pair, first-appearance order
  std::vector<std::pair<int, int>> pairs;
  std::vector<std::vector<int>> q;
  for (int i = 0; i < Q; ++i) {
    const int a = qs.src[i], b = qs.tgt[i];
    if (a < 0 || a >= F || b < 0 || b >= F)
      throw std::runtime_error("gimmvfi queries: query " + std::to_string(i) + " = (" + std::to_string(a) + ", " + std::to_string(b) +
                               ") indexes outside the " + std::to_string(F) + " frames");
    const float t = qs.t[i];
    if (!std::isfinite(t) || !(t > 0.f && t < 1.f))   // the AMT lookup scales by 1/t and 1/(1-t) (gimmvfi_r.py:494-507)
      throw std::runtime_error("gimmvfi queries: query " + std::to_string(i) + " has t = " + std::to_string(t) + "; t must lie strictly inside (0, 1)");
    auto it = pair_of.find({a, b});
    if (it == pair_of.end()) { it = pair_of.emplace(std::make_pair(a, b), (int)pairs.size()).first; pairs.push_back({a, b}); q.emplace_back(); }
    q[it->second].push_back(i);
  }
  std::vector<int> order(pairs.size());
  for (size_t i = 0; i < order.size(); ++i) order[i] = (int)i;
  std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return q[x].size() > q[y].size(); });
  Problem e = p; e.B = (int)pairs.size(); e.T = (int)q[order[0]].size();
  check_problem(e);
  Schedule s;
  std::vector<int> compact(F, -1);   // the engine frame of each used caller frame, in caller order
  for (const auto& ab : pairs) compact[ab.first] = compact[ab.second] = 0;
  const int64_t hw = (int64_t)p.Hf * p.Wf;
  for (int f = 0; f < F; ++f) {
    if (compact[f] < 0) continue;
    if (f > 0 && compact[f - 1] >= 0) ++s.loads.back().n;   // one load per run of consecutive used frames
    else s.loads.push_back({f * 3 * hw, 3 * hw, hw, s.F, 1});
    compact[f] = s.F++;
  }
  s.rows.resize(e.T);
  for (int d : order) {
    s.src.push_back(compact[pairs[d].first]); s.tgt.push_back(compact[pairs[d].second]);
    s.pair_rows.push_back(d);
    for (size_t k = 0; k < q[d].size(); ++k) s.rows[k].push_back(q[d][k]);
  }
  s.t = qs.t;
  return s;
}

// RAFT.forward (raft/raft.py:100-169) over F prepared frames and a list of (source, target) pairs, batched on the N axis.  fnet runs once
// per frame, cnet (-> net | inp, and the hoisted gate terms) once per distinct source; the context is gathered into pair order unless the
// sources are the frames in order, pair s from frame s (GIMM-VFI-R).  Pair s correlates fmap[src[s]] with fmap[tgt[s]]: the volume
// pyramid, or - when the pair list's pyramid would not fit the memory budget - the volume-free lookup.
// The recurrence amplifies operand rounding: the caller sets fp32-class arithmetic (3xTF32 tensor cores or CUDA cores).
void Engine::run_raft(Ctx& cx, Net& N, const RaftRun& r) {
  Arena& A = cx.arena;
  const std::vector<int>& src = r.src; const std::vector<int>& tgt = r.tgt;
  const int F = r.img.n, S = (int)src.size(), H = r.img.h, W = r.img.w, h = H / 8, w = W / 8;
  if (S < 1 || (int)tgt.size() != S || r.iters < 1) throw std::runtime_error("raft: bad pair list or iteration count");
  for (int s = 0; s < S; ++s)
    if (src[s] < 0 || src[s] >= F || tgt[s] < 0 || tgt[s] >= F) throw std::runtime_error("raft: pair index out of range");
  std::vector<int> srcs, slot(F, -1);   // distinct sources in first-use order
  for (int s = 0; s < S; ++s)
    if (slot[src[s]] < 0) { slot[src[s]] = (int)srcs.size(); srcs.push_back(src[s]); }
  const bool in_order = !r.gather && S == F && is_identity(src);
  if (r.enc0 && !in_order) throw std::runtime_error("raft: skipping encoders needs the sources in frame order");
  const int ns = (int)srcs.size(), e0 = r.enc0, en = F - e0;
  TV hx = A.tensor(S, h, w, 384);                      // [h | inp | motion]
  TV cb = in_order ? hx : A.tensor(ns, h, w, 256);     // net | inp of each distinct source
  {
    TV rin = r.img.batch(e0, en);
    TV raft_pad = A.tensor(en, H + 6, W + 6, 3, 4);
    pad_image4(cx, rin, raft_pad, 3);
    raft_encoder(N, "flow_estimator.fnet", true, rin, raft_pad, r.fmap.batch(e0, en), nullptr, nullptr, nullptr, TV(), TV());
    // the encoder's temporaries stay allocated until the caller releases the arena (bump allocator): c4 / c8 live on
    TV cin = rin, cpad = raft_pad;
    if (!in_order) {
      cin = A.tensor(ns, H, W, 3, 4); cpad = A.tensor(ns, H + 6, W + 6, 3, 4);
      for (int i = 0; i < ns; ++i) copy_channels(cx, r.img.batch(srcs[i], 1), cin.batch(i, 1));
      pad_image4(cx, cin, cpad, 3);
    }
    TV c4, c8;
    const ConvW& wc = N.W("flow_estimator.cnet.conv2");
    TV ctx = in_order ? hx.batch(e0, en) : cb;
    raft_encoder(N, "flow_estimator.cnet", false, cin, cpad, TV(), &c4, &c8, &wc, ctx.slice(0, 128), ctx.slice(128, 128));
    if (!in_order)
      for (int s = 0; s < S; ++s) copy_channels(cx, cb.batch(slot[src[s]], 1), hx.batch(s, 1).slice(0, 256));
    if (r.encoded) r.encoded(c4, c8, hx);
  }
  const TV& fmap = r.fmap;
  tap("raft.fmap", fmap);

  // RAFT's correlation: the all-pairs volume pyramid (fp32-class GEMMs; 8.3 ms of GEMM + 20 lookups at 1080p) - or, when that
  // pyramid would not fit the memory budget (a 4K pair without ds_factor: 2 x 78 GB at level 0 alone), NO volume: every lookup
  // computes the 4 x 100 dot products its window needs from the other frame's (pooled, half-precision) features, like
  // BidirCorrBlock's (SURVEY 8(f) row 3, the GPU successor of alt_cuda_corr).  ~5x the time of the volume path, 0 bytes instead of N^2.
  // (a clip decides as a batch forward of one pair does - decide_as = 2 directions - so that each of its pairs takes the same path)
  const double pyr_bytes = (double)(r.decide_as > 0 ? r.decide_as : S) * (double)h * w * (double)h * w * 4.0 * (4.0 / 3.0);
  const bool raft_direct = (raft_direct_ == 1 || (raft_direct_ < 0 && pyr_bytes > raft_direct_auto_bytes_)) && fmap.c == 256 && h >= 16 && w >= 16;
  Pyramid pyr{}; CorrFeat rfeat{};
  if (raft_direct) {
    TV Fl = fmap;
    rfeat.c = 256; rfeat.scale = 1.0f / std::sqrt((float)fmap.c);
    for (int l = 0; l < 4; ++l) {
      rfeat.h[l] = Fl.h; rfeat.w[l] = Fl.w;
      void* hp = A.alloc_f(((size_t)Fl.pixels() * Fl.c + 1) / 2);
      features_to_half(cx, Fl, hp);
      rfeat.lvl[l] = static_cast<const uint16_t*>(hp);
      if (l < 3) { TV nx = A.tensor(F, Fl.h / 2, Fl.w / 2, Fl.c); avgpool2_features(cx, Fl, nx); Fl = nx; }
    }
  } else {
    pyr = build_pyramid(cx, fmap, src, tgt, tc_mode_ >= 2 ? 2 : 0);   // fp32-class only
  }
  auto rfeat_of = [&](int sample0) {
    CorrFeat f = rfeat;
    for (int l = 0; l < 4; ++l) f.lvl[l] = rfeat.lvl[l] + (int64_t)sample0 * f.h[l] * f.w[l] * f.c;
    return f;
  };
  const std::vector<std::pair<int, int>> runs = pair_runs(src, tgt);
  const std::string u = "flow_estimator.update_block";
  TV coords1 = A.tensor(S, h, w, 2);
  TV flow = A.tensor(S, h, w, 2, 4);   // ld 4: 16-byte pixel stride so the 7x7 2->128 conv can use TMA
  TV corr = A.tensor(S, h, w, 324), cor1 = A.tensor(S, h, w, 256), corflo = A.tensor(S, h, w, 256);
  TV flo1 = A.tensor(S, h, w, 128), zb = A.tensor(S, h, w, 128), rh = A.tensor(S, h, w, 128);
  TV fh = A.tensor(S, h, w, 256), mask = A.tensor(S, h, w, 576);
  TV up_it = r.flow_iters ? A.tensor(S, H, W, 2) : TV();   // the upsampled flow of every iteration but the last
  init_coords(cx, coords1);
  if (r.flow_init) parallel_for(cx, (int64_t)S * 2 * h * w, FlowInitAddK{r.flow_init, coords1}, "raft_flow_init");
  TV hcur = hx.slice(0, 128), xin = hx.slice(128, 256), mot = hx.slice(256, 128);
  // iteration-invariant share of the gate convolutions (tensor-core modes; see finalize_weights), once per distinct source
  const bool hoist = cx.tc;
  TV Pzr[2], Pq[2];
  if (hoist)
    for (int s = 0; s < 2; ++s) {
      const std::string sfx = s == 0 ? "1" : "2";
      Pzr[s] = A.tensor(S, h, w, 256); Pq[s] = A.tensor(S, h, w, 128);
      if (in_order) {
        N.conv(u + ".gru.convzr" + sfx + "_inp", hx.slice(128, 128), Pzr[s]);
        N.conv(u + ".gru.convq" + sfx + "_inp", hx.slice(128, 128), Pq[s]);
        continue;
      }
      const size_t mk = A.mark();
      TV z = A.tensor(ns, h, w, 256), q = A.tensor(ns, h, w, 128);
      N.conv(u + ".gru.convzr" + sfx + "_inp", cb.slice(128, 128), z);
      N.conv(u + ".gru.convq" + sfx + "_inp", cb.slice(128, 128), q);
      for (int p = 0; p < S; ++p) { copy_channels(cx, z.batch(slot[src[p]], 1), Pzr[s].batch(p, 1)); copy_channels(cx, q.batch(slot[src[p]], 1), Pq[s].batch(p, 1)); }
      A.release(mk);
    }
  tap_copy(cx, "raft.cnet", hx.slice(0, 256));   // tanh(net) | relu(inp) in pair order (the GRU overwrites net in place)
  for (int it = 0; it < r.iters; ++it) {
    if (debug_ && it == r.iters - 1) { tap_copy(cx, "raft.coords_last", coords1); tap_copy(cx, "raft.net_last", hcur); }
    if (raft_direct) {   // each run's sources against its targets' features (GIMM-VFI-R: frame 1's for direction 0 and vice versa)
      for (const auto& run : runs)
        corr_lookup_direct(cx, fmap.batch(src[run.first], run.second), rfeat_of(tgt[run.first]), coords1.batch(run.first, run.second),
                           corr.batch(run.first, run.second));
    } else {
      corr_lookup(cx, pyr.view(0), coords1, corr);
    }
    coords_minus_grid(cx, coords1, flow, hx.slice(382, 2));
    // (a copy: every later iteration's lookup overwrites `corr`)
    if (it == 0 && debug_) { TV snap = A.tensor(S, h, w, 324); copy_channels(cx, corr, snap); tap("raft.corr_it0", snap); }
    if (debug_ && it == r.iters - 1) tap_copy(cx, "raft.corr_last", corr);
    // BasicMotionEncoder raft/update.py:94-112
    N.conv(u + ".encoder.convc1", corr, cor1, ACT_RELU);
    N.conv(u + ".encoder.convc2", cor1, corflo.slice(0, 192), ACT_RELU);
    N.conv7x(u + ".encoder.convf1", flow, flo1, ACT_RELU);
    N.conv(u + ".encoder.convf2", flo1, corflo.slice(192, 64), ACT_RELU);
    N.conv(u + ".encoder.conv", corflo, hx.slice(256, 126), ACT_RELU);
    if (debug_ && it == r.iters - 1) tap_copy(cx, "raft.motion_last", mot);   // 126 motion features + the 2 flow channels
    // SepConvGRU raft/update.py:35-73 (horizontal 1x5 then vertical 5x1)
    for (const char* sfx : {"1", "2"}) {
      if (hoist) {
        const int s = sfx[0] - '1';
        ConvEpi ezr; ezr.res = Pzr[s]; ezr.act2 = ACT_SIGMOID; ezr.mul = hcur; ezr.out2 = rh; ezr.split_c = 128;
        N.conv_e(u + ".gru.convzr" + sfx + "_hm", hcur, mot, zb, ezr);
        ConvEpi eq; eq.res = Pq[s]; eq.act2 = ACT_TANH; eq.gru_z = zb; eq.gru_h = hcur;
        N.conv_e(u + ".gru.convq" + sfx + "_hm", rh, mot, hcur, eq);
        continue;
      }
      if (cx.tc) {   // one launch for both gates: 1020 tiles instead of 2 x 510 (fewer, fuller waves)
        ConvEpi ezr; ezr.act1 = ACT_SIGMOID; ezr.mul = hcur; ezr.out2 = rh; ezr.split_c = 128;
        N.conv_e(u + ".gru.convzr" + sfx, hx, TV(), zb, ezr);
      } else {
        ConvEpi ez; ez.act1 = ACT_SIGMOID;
        N.conv_e(u + ".gru.convz" + sfx, hx, TV(), zb, ez);
        ConvEpi er; er.act1 = ACT_SIGMOID; er.mul = hcur;
        N.conv_e(u + ".gru.convr" + sfx, hx, TV(), rh, er);
      }
      ConvEpi eq; eq.act1 = ACT_TANH; eq.gru_z = zb; eq.gru_h = hcur;
      N.conv_e(u + ".gru.convq" + sfx, rh, xin, hcur, eq);
    }
    // FlowHead raft/update.py:6-14; coords1 += delta_flow (raft/raft.py:153)
    N.conv(u + ".flow_head.conv1", hcur, fh, ACT_RELU);
    { ConvEpi e; e.res = coords1; N.conv_e(u + ".flow_head.conv2", fh, TV(), coords1, e); }
    if (it == 0 || it == 4) { /* debug snapshots are cheap copies */
      if (debug_) { TV snap = A.tensor(S, h, w, 2); coords_minus_grid(cx, coords1, snap, TV()); tap("raft.lowres_flow_it" + std::to_string(it), snap); }
    }
    const bool last = it == r.iters - 1;
    if (last || r.flow_iters) {
      // the mask head and the convex upsampling (raft/raft.py:155-163): every iteration for flow_predictions, else the last one only
      N.conv(u + ".mask.0", hcur, fh, ACT_RELU);
      N.conv(u + ".mask.2", fh, mask);
      if (last) tap("raft.mask", mask);   // (0.25 is folded into mask.2's weights)
      coords_minus_grid(cx, coords1, flow, TV());
      const TV& up = last ? r.flow_up : up_it;
      if (last) tap("raft.lowres_flow_final", flow);
      convex_upsample(cx, flow, mask, up);
      if (r.flow_iters) nhwc_to_nchw(cx, up, r.flow_iters + (int64_t)it * S * 2 * H * W, (int64_t)2 * H * W, (int64_t)H * W, 1.f, 0.f, 0);
      if (last && r.flow_low.p) copy_channels(cx, flow, r.flow_low);
    }
  }
  tap("raft.net_final", hcur);
}

// The frame cache (set_frame_cache) of a batch forward, between RAFT's encoders and its GRU (which overwrites net in place): with
// `load` frame 0's products come from the cache, with `store` frame 1's are written to it.  ni: the pairs' net | inp.
void Engine::frame_cache(Ctx& cx, const Problem& P, const TV& fmap, const TV& ni, const TV& feat4, const TV& feat8) {
  const int B = P.B, H = P.H(), W = P.W();
  if (fc_bytes_ < frame_cache_bytes(P)) throw std::runtime_error("gimmvfi: frame cache smaller than frame_cache_bytes()");
  const auto fc_it = fc_valid_.find(fc_);
  if (fc_load_ && (fc_it == fc_valid_.end() || fc_it->second.B != B || fc_it->second.H != H || fc_it->second.W != W || fc_it->second.mode != tc_mode_))
    throw std::runtime_error("gimmvfi: frame cache load requested, but this buffer does not hold a frame stored by a forward of the same "
                             "problem size and precision mode");
  if (fc_store_) fc_valid_[fc_] = FcRec{B, H, W, tc_mode_};
  else if (!fc_load_) fc_valid_.erase(fc_);
  float* q = fc_;
  for (const TV& t : {fmap, ni, feat4, feat8}) {   // the cache: B dense samples of each, in this order
    const TV c = make_tv(q, B, t.h, t.w, t.c); q += (size_t)B * t.h * t.w * t.c;
    if (fc_load_) copy_channels(cx, c, t.batch(0, B));
    if (fc_store_) copy_channels(cx, t.batch(B, B), c);
  }
}

void Engine::run(Ctx& cx, const Problem& P0, const IO& io, const Schedule& sched, const FlowInputs* fin) {
  Problem P = P0;
  P.B = (int)sched.src.size(); P.T = (int)sched.rows.size();   // (a query list's distinct pairs and slots; the problem's own otherwise)
  Net N{*this, cx};
  Arena& A = cx.arena;
  const int B = P.B, Hf = P.Hf, Wf = P.Wf, H = P.H(), W = P.W(), T = P.T;
  const int h = H / 8, w = W / 8, H4 = H / 4, W4 = W / 4;
  const bool ds = P.ds > 0.f;
  const float rds = ds ? (float)(1.0 / (double)P.ds) : 1.f;       // resize(x, ds): src = rds*(dst+.5)-.5
  const double inv_d = ds ? (double)Hf / (double)H : 1.0;          // gimmvfi_r.py:297
  const float inv = (float)inv_d, rinv = (float)(1.0 / inv_d);

  // The estimator's pair list over the frame stack: both directions of every pair, [pairs ; reversed pairs], which is also the sample
  // order of everything downstream.  The per-frame products are gathered into that order unless it is the frames' own (a batch
  // forward's [I0 batch ; I1 batch]); fslot: a frame's sample among the distinct sources, first-use order.
  std::vector<int> esrc(2 * B), etgt(2 * B), pslot(2 * B), fslot(sched.F, -1);   // pslot: each sample's distinct-source slot
  for (int s = 0; s < B; ++s) { esrc[s] = etgt[B + s] = sched.src[s]; etgt[s] = esrc[B + s] = sched.tgt[s]; }
  int nsrc = 0;
  for (int s = 0; s < 2 * B; ++s) { if (fslot[esrc[s]] < 0) fslot[esrc[s]] = nsrc++; pslot[s] = fslot[esrc[s]]; }
  // x's samples in pair order, sample i <- x's sample idx[i]: x itself when idx is the identity, else gathered into `into` (or a new tensor)
  auto pair_order = [&](const TV& x, const std::vector<int>& idx, TV into = TV()) {
    if (is_identity(idx)) return x;
    if (!into.p) into = x.f16 ? A.tensor_h((int)idx.size(), x.h, x.w, x.c, x.ld) : A.tensor((int)idx.size(), x.h, x.w, x.c, x.ld);
    gather_samples(cx, x, idx, into);
    return into;
  };

  // ------------------------------------------------------------ inputs
  TV full01 = A.tensor(sched.F, Hf, Wf, 3, 4);   // frames as NHWC
  for (const Schedule::Load& l : sched.loads) nchw_to_nhwc(cx, io.img_xs + l.off, l.sn, l.sc, full01.batch(l.f0, l.n), 1.f, 0.f);
  TV img01 = full01;
  if (ds) {
    img01 = A.tensor(sched.F, H, W, 3, 4);
    resize_bilinear(cx, full01, img01, rds, rds, 1.f, 0, ACT_NONE);  // gimmvfi_r.py:329-337
  }
  TV raft_in = A.tensor(sched.F, H, W, 3, 4);
  TV syn = A.tensor(sched.F, H, W, 3, 4);  // 2*x - 1  (gimmvfi_r.py:230-231)
  {
    // dense views (ld == 4): run over the padded buffers, padding lane included (harmless)
    int64_t cnt = (int64_t)sched.F * H * W * 4;
    TV s = img01; s.c = 4; TV d = raft_in; d.c = 4;
    parallel_for(cx, cnt, RaftPrepK{s, d}, "raft_prep");
    parallel_for(cx, cnt, ScaleShiftK{img01.p, syn.p, 2.f, 1.0f}, "img_to_pm1");
  }
  TV synf = syn;
  if (ds) {
    synf = A.tensor(sched.F, Hf, Wf, 3, 4);
    parallel_for(cx, (int64_t)sched.F * Hf * Wf * 4, ScaleShiftK{full01.p, synf.p, 2.f, 1.0f}, "img_to_pm1_full");
  }

  // persistent across stages
  TV flow_up = A.tensor(2 * B, H, W, 2);            // [f01 ; f10]
  TV fmap = A.tensor(sched.F, h, w, 256);           // fnet features of every frame
  TV feat4 = A.tensor(nsrc, H4, W4, 128), feat8 = A.tensor(nsrc, h, w, 256);  // projected context features
  float* scaler = A.alloc_f(std::max(B, 64));

  // ------------------------------------------------------------ RAFT (both directions batched)
  // The recurrence amplifies operand rounding -> fp32-class arithmetic only: 3xTF32 tensor cores or CUDA cores.
  cx.tc = tc_mode_ >= 2; cx.tc_split = true;
  TV fproj = A.tensor(sched.F, h, w, 256);          // the maps BidirCorrBlock correlates (R: amt_fproj(fnet map); F: the estimator's own)
  if (fin) {
    // external flow estimator (GIMM-VFI-F): NCHW -> the engine's NHWC buffers, samples [frame-0 batch ; frame-1 batch]
    for (int j = 0; j < 2; ++j) {
      nchw_to_nhwc(cx, fin->flows + (int64_t)j * H * W, (int64_t)4 * H * W, (int64_t)2 * H * W, flow_up.batch(j * B, B), 1.f, 0.f);
      nchw_to_nhwc(cx, fin->feat4[j], (int64_t)128 * H4 * W4, (int64_t)H4 * W4, feat4.batch(j * B, B), 1.f, 0.f);
      nchw_to_nhwc(cx, fin->feat8[j], (int64_t)256 * h * w, (int64_t)h * w, feat8.batch(j * B, B), 1.f, 0.f);
      nchw_to_nhwc(cx, fin->fnet[j], (int64_t)256 * h * w, (int64_t)h * w, fproj.batch(j * B, B), 1.f, 0.f);
    }
  } else if (is_f()) {
    // GIMM-VFI-F: the native FlowFormer estimator fills the same four products (gimmvfi_f.py:114-138); F has no feature projections.
    // The schedule's pairs (b, B + b), then (B + b, b): a batch forward makes one reference call per direction, a clip or a query list
    // one per pair and direction, as a batch forward with B = 1 makes them
    run_flowformer(cx, N, raft_in, esrc, etgt, sched.per_call, ff_iters, false, flow_up, TV(), feat4, feat8, fproj);
  } else {
    const size_t mk = A.mark();
    // frame cache: with `load` the encoders only see the second frames, samples [B, 2B)
    const bool fc_on = sched.frame_cache && fc_ != nullptr && !cx.dry;
    const int e0 = fc_on && fc_load_ ? B : 0, en = nsrc - e0;
    // both directions batched (gimmvfi_r.py:126-132); c4 / c8 below are the distinct sources', first-use order: feat4 / feat8's slots
    RaftRun r;
    r.img = raft_in; r.iters = raft_iters; r.flow_up = flow_up; r.fmap = fmap; r.enc0 = e0;
    r.src = esrc; r.tgt = etgt; r.decide_as = sched.decide_as;
    r.encoded = [&](const TV& c4, const TV& c8, const TV& hx) {
      // context features for the synthesis net (gimmvfi_r.py:134-141)
      N.conv("amt_second_last_cproj", c4, feat4.batch(e0, en));
      N.conv("amt_last_cproj", c8, feat8.batch(e0, en));
      if (fc_on) frame_cache(cx, P, fmap, hx.slice(0, 256), feat4, feat8);
    };
    run_raft(cx, N, r);
    if (!debug_) A.release(mk);
  }
  // (P,2,2,H,W) per-pair outputs from [direction 0 ; direction 1] samples, pair p at row pair_rows[p]
  auto store_pairs = [&](const TV& both, float* dst) {
    for (int j = 0; j < 2; ++j)
      nhwc_to_nchw_rows(cx, both.batch(j * B, B), dst + (int64_t)j * H * W, sched.pair_rows, (int64_t)4 * H * W, (int64_t)2 * H * W, 1.f, 0.f, 0);
  };
  if (io.raft_flow) store_pairs(flow_up, io.raft_flow);

  // Everything downstream of RAFT tolerates TF32 operands (DESIGN.md precision plan).
  cx.tc = tc_mode_ >= 1; cx.tc_split = false;
  // ------------------------------------------------------------ bidirectional volume on projected features
  if (!fin && !is_f()) N.conv("amt_fproj", fmap, fproj);
  fproj = pair_order(fproj, esrc);   // [sources ; targets] of the pairs
  syn = pair_order(syn, esrc);
  synf = ds ? pair_order(synf, esrc) : syn;
  // the bidirectional volume only feeds TF32 layers (AMT update blocks) -> plain TF32 is at their input precision
  // Few interpolated frames per pair (at most corr_direct_max_t timesteps): no volume at all - the lookup computes the dot products its
  // window needs (corr.cu "volume-free lookup").  Otherwise the all-pairs pyramid, looked up at every timestep.  Each pair decides as its
  // own forward would: the pairs are sorted by timestep count, so the pyramid pairs are a prefix [0, Bp) and the direct ones [Bp, B).
  Pyramid bpyr{}; CorrFeat bfeat{};
  constexpr int corr_direct_max_t = 2;
  const bool direct_ok = tc_mode_ >= 1 && fproj.c == 256 && h >= 16 && w >= 16;
  const int Bp = !direct_ok ? B : T > corr_direct_max_t ? (int)sched.rows[corr_direct_max_t].size() : 0;
  const int Bd = B - Bp;
  if (Bd > 0) {
    // half features of the direct pairs' samples, [sources ; targets]: compact sample i < Bd is pair Bp + i's source, Bd + i its target
    std::vector<TV> runs = {fproj};
    if (Bp > 0) runs = {fproj.batch(Bp, Bd), fproj.batch(B + Bp, Bd)};
    bfeat.c = 256; bfeat.scale = 1.0f / std::sqrt((float)fproj.c);
    for (int l = 0; l < 4; ++l) {
      bfeat.h[l] = runs[0].h; bfeat.w[l] = runs[0].w;
      const size_t per = (size_t)runs[0].h * runs[0].w * runs[0].c;
      uint16_t* hp = reinterpret_cast<uint16_t*>(A.alloc_f(((size_t)2 * Bd * per + 1) / 2));
      for (size_t r = 0, n0 = 0; r < runs.size(); n0 += runs[r].n, ++r) features_to_half(cx, runs[r], hp + n0 * per);
      bfeat.lvl[l] = hp;
      if (l < 3) {
        TV nx = A.tensor(2 * Bd, runs[0].h / 2, runs[0].w / 2, runs[0].c);
        for (size_t r = 0, n0 = 0; r < runs.size(); n0 += runs[r].n, ++r) avgpool2_features(cx, runs[r], nx.batch((int)n0, runs[r].n));
        runs = {nx};
      }
    }
  }
  if (Bp > 0) {
    std::vector<int> src(2 * Bp), tgt(2 * Bp);   // [f0 ; f1] against [f1 ; f0] of the pyramid pairs
    for (int s = 0; s < Bp; ++s) { src[s] = tgt[Bp + s] = s; tgt[s] = src[Bp + s] = B + s; }
    bpyr = build_pyramid(cx, fproj, src, tgt, tc_mode_ >= 1 ? 1 : 0);   // gimmvfi_r.py:133, raft/corr.py:23-44
  }
  auto bfeat_of = [&](int sample0) {
    CorrFeat f = bfeat;
    for (int l = 0; l < 4; ++l) f.lvl[l] = bfeat.lvl[l] + (int64_t)sample0 * f.h[l] * f.w[l] * f.c;
    return f;
  };

  // ------------------------------------------------------------ hoisted (t-independent) decoder feature upsampling
  TV fup4 = A.tensor(2 * B, H4, W4, 128);   // NewInitDecoder.upsample   fi_components.py:234-244
  TV fup1 = half_chains(cx) ? A.tensor_h(2 * B, H, W, 64) : A.tensor(2 * B, H, W, 64);      // NewMultiFlowDecoder.upsample fi_components.py:284-295
  // each distinct source is upsampled once: straight into fup4 / fup1 when they are the pairs' samples in order, else into buffers of
  // their own, gathered into pair order below
  const size_t fup_mk = A.mark();
  TV fup4s = fup4, fup1s = fup1;
  if (!is_identity(pslot)) { fup4s = A.tensor(nsrc, H4, W4, 128); fup1s = half_chains(cx) ? A.tensor_h(nsrc, H, W, 64) : A.tensor(nsrc, H, W, 64); }
  {
    const size_t mk = A.mark();
    const std::string p = "amt_init_decoder.upsample.";
    TV a = A.tensor(nsrc, H4, W4, 64), b = A.tensor(nsrc, H4, W4, 64), c = A.tensor(nsrc, H4, W4, 128);
    pixel_shuffle(cx, feat8, a, 1);
    N.convrelu(p + "1", a, b); N.convrelu(p + "2", b, a); N.convrelu(p + "3", a, b); N.convrelu(p + "4", b, a);
    N.convrelu(p + "5", a, c);
    N.conv(p + "6", c, fup4s, ACT_RELU);  // 1x1 + folded BatchNorm + ReLU
    A.release(mk);
  }
  {
    const size_t mk = A.mark();
    const std::string p = "amt_final_decoder.upsample.";
    const bool hs = half_chains(cx);
    TV a = A.tensor(nsrc, H, W, 8);
    TV b = hs ? A.tensor_h(nsrc, H, W, 32) : A.tensor(nsrc, H, W, 32), c = A.tensor_like(b, 32), d = A.tensor_like(b, 64);
    pixel_shuffle(cx, feat4, a, 2);
    if (cx.tc) N.conv7x(p + "2.0", a, b, ACT_PRELU, N.V(p + "2.1.weight"));   // x-packed 5x5 (pack_xpacked)
    else N.convrelu(p + "2", a, b);
    N.convrelu(p + "3", b, c); N.convrelu(p + "4", c, b); N.convrelu(p + "5", b, c);
    N.convrelu(p + "6", c, d);
    N.conv(p + "7", d, fup1s, ACT_RELU);
    A.release(mk);
  }
  pair_order(fup4s, pslot, fup4);
  pair_order(fup1s, pslot, fup1);
  if (!debug_) A.release(fup_mk);
  tap("syn.feat4", feat4); tap("syn.feat8", feat8); tap("syn.fup4", fup4); tap("syn.fproj", fproj);
  tap_copy(cx, "syn.fup1", fup1);   // (half in mode 4)

  // ------------------------------------------------------------ GIMM (t-independent part)  gimmvfi_r.py:158-168
  TV f01 = flow_up.batch(0, B), f10 = flow_up.batch(B, B);
  {
    float* sc = A.alloc_f((size_t)absmax_scratch_floats(f01));
    absmax_per_sample(cx, f01, f10, scaler, sc);
  }
  TV nf = A.tensor(2 * B, H, W, 2);
  normalize_flow_pair(cx, f01, f10, scaler, nf.batch(0, B), nf.batch(B, B));
  if (io.nflow) store_pairs(nf, io.nflow);
  TV wts = A.tensor(2 * B, H, W, 1);
  TV X64 = A.tensor(B, H, W, 64);   // [lat0 | lat1 | splat0 | splat1]
  gimm_encode(N, nf, f01, f10, wts, X64);

  // ------------------------------------------------------------ per-timestep: GIMM decode + frame synthesis
  // Slot ti runs over the first Bk pairs (those with more than ti timesteps): every per-pair buffer below is batch-major, so the slot
  // works on .batch(0, Bk) views of the first direction and .batch(B, Bk) of the second, and stores its outputs at its rows.
  TV grid_flow = A.tensor(B, h, w, 4);   // flow_4_lr = cat(fl0, fl1)
  const size_t t_mark = A.mark();
  for (int ti = 0; ti < T; ++ti) {
    A.release(t_mark);
    // debug taps of the per-timestep tensors are taken at the last timestep: nothing overwrites them after it
    const bool last = ti == T - 1;
    const std::vector<int>& rows = sched.rows[ti];
    const int Bk = (int)rows.size();
    const float *tdev, *coords_t;
    if (sched.t.empty()) {   // the caller's, at the slot's (consecutive) rows
      tdev = io.t + rows[0];
      coords_t = io.coords + (int64_t)rows[0] * P.Hc * P.Wc * 3;
    } else {
      std::vector<float> ts;
      for (int r : rows) ts.push_back(sched.t[r]);
      float* tq = A.alloc_f(std::max(Bk, 64));
      float* cq = A.alloc_f((size_t)Bk * P.Hc * P.Wc * 3);
      if (!cx.dry) query_coords(cx, ts, P.Hc, P.Wc, coord_lo_, coord_span_, cq, tq);
      tdev = tq; coords_t = cq;
      if (last) tap("query.coords", make_tv(cq, Bk, P.Hc, P.Wc, 3));
    }
    TV ninr = A.tensor(Bk, H, W, 2);
    gimm_decode(N, X64.batch(0, Bk), f01.batch(0, Bk), f10.batch(0, Bk), wts.batch(0, Bk), wts.batch(B, Bk), tdev, coords_t, ninr, last);
    if (io.ninrflow) nhwc_to_nchw_rows(cx, ninr, io.ninrflow, rows, (int64_t)2 * H * W, (int64_t)H * W, 1.f, 0.f, 0);
    TV flow_t = A.tensor(Bk, H, W, 2);
    unnormalize_flow(cx, ninr, scaler, flow_t);
    if (io.flowt) nhwc_to_nchw_rows(cx, flow_t, io.flowt, rows, (int64_t)2 * H * W, (int64_t)H * W, 1.f, 0.f, 0);

    // ---- frame_synthesize (gimmvfi_r.py:222-322)
    TV s0 = syn.batch(0, Bk), s1 = syn.batch(B, Bk);
    TV ft0 = A.tensor(Bk, H, W, 2), ft1 = A.tensor(Bk, H, W, 2);
    scale_flow_t(cx, flow_t, tdev, ft0, ft1);
    // NewInitDecoder (fi_components.py:255-276)
    TV fin = A.tensor(Bk, H4, W4, 272);
    TV f0in = fin.slice(256, 2), f1in = fin.slice(258, 2);
    resize_bilinear(cx, ft0, f0in, 4.f, 4.f, 0.25f, 0, ACT_NONE);
    resize_bilinear(cx, ft1, f1in, 4.f, 4.f, 0.25f, 0, ACT_NONE);
    backwarp(cx, fup4.batch(0, Bk), f0in, fin.slice(0, 128));
    backwarp(cx, fup4.batch(B, Bk), f1in, fin.slice(128, 128));
    resize_bilinear(cx, s0, fin.slice(260, 3), 4.f, 4.f, 1.f, 0, ACT_NONE);
    resize_bilinear(cx, s1, fin.slice(263, 3), 4.f, 4.f, 1.f, 0, ACT_NONE);
    backwarp(cx, fin.slice(260, 3), f0in, fin.slice(266, 3));
    backwarp(cx, fin.slice(263, 3), f1in, fin.slice(269, 3));
    TV x4 = half_chains(cx) ? A.tensor_h(Bk, H4, W4, 128) : A.tensor(Bk, H4, W4, 128);   // (mode 4: the H/4 residual trunk in half too)
    N.convrelu("amt_init_decoder.convblock.0", fin, x4);
    for (int k = 1; k <= 3; ++k) resblock(N, "amt_init_decoder.convblock." + std::to_string(k), x4, 128, 64);
    TV o136 = A.tensor(Bk, H4, W4, 133, 136);
    N.conv("amt_init_decoder.convblock.4", x4, o136);
    TV ft_4 = o136.slice(0, 128);
    TV fl4 = A.tensor(Bk, H4, W4, 4), mask4 = A.tensor(Bk, H4, W4, 1);
    flow_mask_split(cx, o136, f0in, f1in, fl4.slice(0, 2), fl4.slice(2, 2), mask4);
    if (last) {   // (ft_4 / fl4 are updated in place by the update blocks: snapshots)
      tap("syn.fin4", fin); tap("syn.mask4_init", mask4);
      tap_copy(cx, "syn.ft4_init", ft_4); tap_copy(cx, "syn.fl4_init", fl4);
    }
    // warp_w_mask(scale=4) -> img_warp_4 (aux output, gimmvfi_r.py:259-261)
    if (io.img_warp_4) {
      const size_t mk = A.mark();
      TV a0 = A.tensor(Bk, H, W, 2), a1 = A.tensor(Bk, H, W, 2), am = A.tensor(Bk, H, W, 1), wb = A.tensor(Bk, H, W, 3, 4);
      resize_bilinear(cx, fl4.slice(0, 2), a0, 0.25f, 0.25f, 4.f, 0, ACT_NONE);
      resize_bilinear(cx, fl4.slice(2, 2), a1, 0.25f, 0.25f, 4.f, 0, ACT_NONE);
      resize_bilinear(cx, mask4, am, 0.25f, 0.25f, 1.f, 0, ACT_SIGMOID);
      warp_blend(cx, s0, s1, a0, a1, am, wb);
      nhwc_to_nchw_rows(cx, wb, io.img_warp_4, rows, (int64_t)3 * H * W, (int64_t)H * W, 0.5f, 1.0f, 1);
      A.release(mk);
    }
    // _amt_corr_scale_lookup(downsample=2)  (gimmvfi_r.py:494-507)
    TV corr648 = A.tensor(Bk, h, w, 648);
    {
      TV gf = grid_flow.batch(0, Bk);
      resize_bilinear(cx, fl4, gf, 2.f, 2.f, 0.5f, 0, ACT_NONE);
      TV cA = A.tensor(Bk, h, w, 2), cB = A.tensor(Bk, h, w, 2);
      lookup_coords(cx, gf.slice(2, 2), tdev, 0, cA);  // coord + flow1 * 1/(1-t) -> volume
      lookup_coords(cx, gf.slice(0, 2), tdev, 1, cB);  // coord + flow0 * 1/t     -> transposed volume
      const int np = std::min(Bp, Bk), nd = Bk - np;
      if (np > 0) {
        corr_lookup(cx, bpyr.view(0), cA.batch(0, np), corr648.batch(0, np).slice(0, 324));
        corr_lookup(cx, bpyr.view(Bp), cB.batch(0, np), corr648.batch(0, np).slice(324, 324));
      }
      if (nd > 0) {   // rows = frame 0's pixels against frame 1's features, and the transposed volume's counterpart
        corr_lookup_direct(cx, fproj.batch(Bp, nd), bfeat_of(Bd), cA.batch(np, nd), corr648.batch(np, nd).slice(0, 324));
        corr_lookup_direct(cx, fproj.batch(B + Bp, nd), bfeat_of(0), cB.batch(np, nd), corr648.batch(np, nd).slice(324, 324));
      }
    }
    amt_update(N, "amt_update4_low", true, ft_4, fl4, grid_flow.batch(0, Bk), corr648);
    if (last) { tap("syn.corr648", corr648); tap_copy(cx, "syn.ft4_low", ft_4); tap_copy(cx, "syn.fl4_low", fl4); }
    {
      TV corr_hi = A.tensor(Bk, H4, W4, 648);
      resize_bilinear(cx, corr648, corr_hi, 0.5f, 0.5f, 1.f, 0, ACT_NONE);  // gimmvfi_r.py:274
      amt_update(N, "amt_update4_high", false, ft_4, fl4, fl4, corr_hi);
      if (last) tap("syn.corr_4_hi", corr_hi);
    }
    if (last) { tap("syn.ft_4", ft_4); tap("syn.fl4", fl4); tap("syn.mask4", mask4); }
    if (io.flowt0_4) nhwc_to_nchw_rows(cx, fl4.slice(0, 2), io.flowt0_4, rows, (int64_t)2 * H4 * W4, (int64_t)H4 * W4, 1.f, 0.f, 0);
    if (io.flowt1_4) nhwc_to_nchw_rows(cx, fl4.slice(2, 2), io.flowt1_4, rows, (int64_t)2 * H4 * W4, (int64_t)H4 * W4, 1.f, 0.f, 0);

    // NewMultiFlowDecoder (fi_components.py:307-340)
    TV F0 = A.tensor(Bk, H, W, 6, 8), F1 = A.tensor(Bk, H, W, 6, 8), Mk = A.tensor(Bk, H, W, 3, 4), Rs = A.tensor(Bk, H, W, 9, 12);
    // debug snapshots of the concat, the fp32 flows / mask and convblock.4's output: allocated here, outside the block that frees them
    const bool snap = debug_ && last;
    TV fin1_snap = snap ? A.tensor(Bk, H, W, 273) : TV(), aux5_snap = snap && half_chains(cx) ? A.tensor(Bk, H, W, 5) : TV();
    TV o24_snap = snap ? A.tensor(Bk, H, W, 24) : TV();
    {
      const size_t mk = A.mark();
      // precision mode 4: the 273-channel concat buffer itself is half precision (written by the half-aware resize / backwarp /
      // copy kernels); the up-sampled flows and mask are additionally kept in fp32 (they drive the warps and the output heads)
      const bool hs = half_chains(cx);
      TV fin1 = hs ? A.tensor_h(Bk, H, W, 273, 280) : A.tensor(Bk, H, W, 273, 276);
      TV aux5 = hs ? A.tensor(Bk, H, W, 5, 8) : TV();
      TV fl0 = hs ? aux5.slice(0, 2) : fin1.slice(256, 2), fl1 = hs ? aux5.slice(2, 2) : fin1.slice(258, 2), mk1 = hs ? aux5.slice(4, 1) : fin1.slice(260, 1);
      resize_bilinear(cx, fl4.slice(0, 2), fl0, 0.25f, 0.25f, 4.f, 0, ACT_NONE);
      resize_bilinear(cx, fl4.slice(2, 2), fl1, 0.25f, 0.25f, 4.f, 0, ACT_NONE);
      resize_bilinear(cx, ft_4, fin1.slice(0, 128), 0.25f, 0.25f, 1.f, 0, ACT_NONE);
      resize_bilinear(cx, mask4, mk1, 0.25f, 0.25f, 1.f, 0, ACT_NONE);
      if (hs) copy_channels(cx, aux5.slice(0, 5), fin1.slice(256, 5));
      backwarp(cx, fup1.batch(0, Bk), fl0, fin1.slice(128, 64));
      backwarp(cx, fup1.batch(B, Bk), fl1, fin1.slice(192, 64));
      copy_channels(cx, s0, fin1.slice(261, 3));
      copy_channels(cx, s1, fin1.slice(264, 3));
      backwarp(cx, s0, fl0, fin1.slice(267, 3));
      backwarp(cx, s1, fl1, fin1.slice(270, 3));
      if (snap) {
        tap_copy_to(cx, "syn.fin1", fin1, fin1_snap);
        if (hs) tap_copy_to(cx, "syn.aux5", aux5, aux5_snap);
      }
      // precision mode 3: the 256-channel residual trunk (9 of the 10 heaviest launches) is stored in fp16 and runs on the
      // f16 tensor-core path (same 10-bit mantissa as TF32, half the bytes per operand, twice the MMA rate)
      TV x1 = (cx.tc && tc_mode_ >= 3) ? A.tensor_h(Bk, H, W, 256) : A.tensor(Bk, H, W, 256);
      N.convrelu("amt_final_decoder.convblock.0", fin1, x1);
      for (int k = 1; k <= 3; ++k) resblock(N, "amt_final_decoder.convblock." + std::to_string(k), x1, 256, 64);
      TV o24 = A.tensor(Bk, H, W, 24);
      N.conv("amt_final_decoder.convblock.4", x1, o24);
      if (snap) tap_copy_to(cx, "syn.o24", o24, o24_snap);
      final_heads(cx, o24, fl0, fl1, mk1, F0, F1, Mk, Rs);
      A.release(mk);
    }
    if (last) { tap("syn.F0", F0); tap("syn.F1", F1); tap("syn.Mk", Mk); tap("syn.Rs", Rs); }
    TV F0f = F0, F1f = F1, Mkf = Mk, Rsf = Rs;
    if (ds) {  // gimmvfi_r.py:294-303
      F0f = A.tensor(Bk, Hf, Wf, 6, 8); F1f = A.tensor(Bk, Hf, Wf, 6, 8); Mkf = A.tensor(Bk, Hf, Wf, 3, 4); Rsf = A.tensor(Bk, Hf, Wf, 9, 12);
      // (views widened to the pixel stride: the padding lanes ride along so that the 16-byte form of the kernel applies - 6 / 3 / 9
      //  channels are not multiples of 4; the scalar form was 12.6 ms of the 4K configuration's 208)
      auto wide = [](TV t) { t.c = t.ld; return t; };
      resize_bilinear(cx, wide(F0), wide(F0f), rinv, rinv, inv, 0, ACT_NONE);
      resize_bilinear(cx, wide(F1), wide(F1f), rinv, rinv, inv, 0, ACT_NONE);
      resize_bilinear(cx, wide(Mk), wide(Mkf), rinv, rinv, 1.f, 0, ACT_NONE);
      resize_bilinear(cx, wide(Rs), wide(Rsf), rinv, rinv, 1.f, 0, ACT_NONE);
      if (last) { tap("syn.F0f", F0f); tap("syn.F1f", F1f); tap("syn.Mkf", Mkf); tap("syn.Rsf", Rsf); }
    }
    if (io.flowt0_1) nhwc_to_nchw_rows(cx, F0f, io.flowt0_1, rows, (int64_t)6 * Hf * Wf, (int64_t)Hf * Wf, 1.f, 0.f, 0);
    if (io.flowt1_1) nhwc_to_nchw_rows(cx, F1f, io.flowt1_1, rows, (int64_t)6 * Hf * Wf, (int64_t)Hf * Wf, 1.f, 0.f, 0);
    // multi_flow_combine + amt_comb_block at FULL resolution (fi_components.py:57-94)
    {
      TV w9 = A.tensor(Bk, Hf, Wf, 9, 12), mean3 = A.tensor(Bk, Hf, Wf, 3, 4), c18 = A.tensor(Bk, Hf, Wf, 18, 20), c3 = A.tensor(Bk, Hf, Wf, 3, 4);
      multi_flow_blend(cx, synf.batch(0, Bk), synf.batch(B, Bk), F0f, F1f, Mkf, Rsf, w9, mean3);
      N.conv7x("amt_comb_block.0", w9, c18, ACT_PRELU, N.V("amt_comb_block.1.weight"));
      N.conv7x("amt_comb_block.2", c18, c3);
      combine_output_rows(cx, mean3, c3, io.imgt_pred, rows);
      if (last) { tap("syn.w9", w9); tap("syn.mean3", mean3); tap("syn.c3", c3); }
    }
  }
}


// ---------------------------------------------------------------------------
// GIMM stages (gimm.py:129-214 == gimmvfi_r.py:158-211), shared by run() and run_gimm()
// ---------------------------------------------------------------------------
// t-independent part: splatting metrics (gimm.py:82-127) and the motion encoder on both normalised flows -> X64[0:32]
void Engine::gimm_encode(Net& N, const TV& nf /*2B: [nf01; nf10]*/, const TV& f01, const TV& f10, const TV& wts /*2B,1*/, const TV& X64) {
  Ctx& cx = N.cx; Arena& A = cx.arena;
  const int B = f01.n, H = f01.h, W = f01.w;
  splat_weights(cx, f01, f10, g9_, alpha_fe_, alpha_v_, wts.batch(0, B));
  splat_weights(cx, f10, f01, g9_, alpha_fe_, alpha_v_, wts.batch(B, B));
  tap("gimm.splat_w", wts);
  {
    const size_t mk = A.mark();
    const bool hs = half_chains(cx);   // precision mode 4: the 32-channel full-resolution chain lives in half precision
    TV a = A.tensor(2 * B, H, W, 16);
    TV x = hs ? A.tensor_h(2 * B, H, W, 32) : A.tensor(2 * B, H, W, 32), y = A.tensor_like(x, 32), m = A.tensor_like(x, 32);
    N.conv("cnn_encoder.0", nf, a);
    N.conv("cnn_encoder.1", a, x, ACT_LRELU);
    for (int i = 3; i <= 5; ++i) {  // LateralBlock fi_components.py:17-29 (+ the LeakyReLU after the last one)
      const std::string q = "cnn_encoder." + std::to_string(i);
      N.conv(q + ".layers.0", x, m, ACT_LRELU);
      ConvEpi e; e.res = x; e.act2 = (i == 5) ? ACT_LRELU : ACT_NONE;
      N.conv_e(q + ".layers.2", m, TV(), y, e);
      std::swap(x, y);
    }
    N.conv("cnn_encoder.7", x.batch(0, B), X64.slice(0, 16), ACT_NONE, nullptr, 1, true);
    N.conv("cnn_encoder.7", x.batch(B, B), X64.slice(16, 16), ACT_NONE, nullptr, 1, true);
    A.release(mk);
  }
  tap("gimm.lat0", X64.slice(0, 16)); tap("gimm.lat1", X64.slice(16, 16));
}

// one timestep: forward splat of both latents to time t, latent refiner, HypoNet -> normalised flow ninr (B,Hc,Wc,2) on the coordinate grid
void Engine::gimm_decode(Net& N, const TV& X64, const TV& f01, const TV& f10, const TV& w01, const TV& w10, const float* tdev,
                         const float* coords_t, const TV& ninr, bool tap_it) {
  Ctx& cx = N.cx; Arena& A = cx.arena;
  const int B = f01.n, H = f01.h, W = f01.w;
  const size_t mk0 = A.mark();
  // ---- forward splat of both latents to time t (gimmvfi_r.py:171-193): memset + vector reductions + normalise (the one-pass
  // softsplat_fused is slower: its shared-memory atomics are compare-and-swap loops, DESIGN.md §3.5)
  const int fwarp = motion_.fwarp;
  if (fwarp == SPLAT_SUM) {   // the plain sum is the result: accumulated straight into the latent buffer
    fill(cx, X64.slice(32, 32), 0.f);
    softsplat_accumulate_mode(cx, X64.slice(0, 16), f01, w01, tdev, 0, X64.slice(32, 16), SPLAT_SUM);
    softsplat_accumulate_mode(cx, X64.slice(16, 16), f10, w10, tdev, 1, X64.slice(48, 16), SPLAT_SUM);
  } else {
    TV acc = A.tensor(2 * B, H, W, 17, 20);
    if (!cx.dry) dev_memset(acc.p, 0, (size_t)2 * B * H * W * 20 * sizeof(float), cx.stream);
    softsplat_accumulate_mode(cx, X64.slice(0, 16), f01, w01, tdev, 0, acc.batch(0, B), fwarp);
    softsplat_accumulate_mode(cx, X64.slice(16, 16), f10, w10, tdev, 1, acc.batch(B, B), fwarp);
    softsplat_normalize(cx, acc.batch(0, B), X64.slice(32, 16));
    softsplat_normalize(cx, acc.batch(B, B), X64.slice(48, 16));
  }
  if (tap_it) { tap("gimm.splat0", X64.slice(32, 16)); tap("gimm.splat1", X64.slice(48, 16)); }
  // HypoNet (hyponet.py:71-146).  Tensor-core modes: ONE fused kernel (hyponet.cu) that takes the refined latent and the caller's
  // coordinate tensor directly; fp32 mode: five 1x1 convolutions on a packed [latent32 | t,y,x] input.
  // The coordinate grid (Hc, Wc) = ninr's size may differ from the flow resolution (GIMM standalone): HypoNet first resizes the
  // latent to the grid (hyponet.py:86-90).  The fused kernel does that in its layer 0 (hyponet_fused3_resample); fp32 mode resizes
  // the refined latent into its grid-sized input.
  const int Hc = ninr.h, Wc = ninr.w;
  const bool same = Hc == H && Wc == W;
  const bool fused = cx.tc && hypo_blob_ != nullptr;
  const bool resample_in_kernel = !same && fused;
  TV hin = resample_in_kernel ? TV() : fused ? A.tensor(B, Hc, Wc, 32) : A.tensor(B, Hc, Wc, 35, 36);
  TV lat = same ? hin.slice(0, 32) : A.tensor(B, H, W, 32);   // the refined latent, at the flow resolution
  {
    const size_t mk = A.mark();
    const bool hs = half_chains(cx);
    TV a = hs ? A.tensor_h(B, H, W, 32) : A.tensor(B, H, W, 32);
    TV x = A.tensor_like(a, 64), m = A.tensor_like(a, 64), y = A.tensor_like(a, 64);
    N.conv("res_conv.0", X64, a);
    N.conv("res_conv.1", a, x, ACT_LRELU);
    N.conv("res_conv.3.layers.0", x, m, ACT_LRELU);
    { ConvEpi e; e.res = x; e.act2 = ACT_LRELU; N.conv_e("res_conv.3.layers.2", m, TV(), y, e); }
    { ConvEpi e; e.res = X64.slice(32, 32); N.conv_e("res_conv.5", y, TV(), lat, e, 1, true); }
    A.release(mk);
  }
  if (tap_it) tap("gimm.latent", lat);
  if (!same && !resample_in_kernel) resize_bilinear(cx, lat, hin.slice(0, 32), (float)H / (float)Hc, (float)W / (float)Wc, 1.f, 0, ACT_NONE);
  const int act = motion_.act;
  const float w0 = motion_.w0;
  if (resample_in_kernel) {
    hyponet_fused3_resample_act(cx, lat, coords_t, hypo_blob3_, ninr, act, w0);
  } else if (fused) {
    // fp32-class: the flow is (2 o - 1) * max|flow|, so operand rounding at 2^-11 becomes ~1e-2 px at 40 px motion and
    // moves real frames by > 1e-3 (tests/test_bench_parity_gpu.py, demo frames)
    hyponet_fused3_act(cx, hin, coords_t, hypo_blob3_, ninr, act, w0);
  } else {
    hypo_pack_input(cx, coords_t, hin.slice(32, 3));
    const size_t mk = A.mark();
    TV a = A.tensor(B, Hc, Wc, 128), b = A.tensor(B, Hc, Wc, 128);
    if (act == HYPO_SIREN1) {
      N.conv("hyponet.params_dict.linear_wb0", hin, a, ACT_SIN);
      N.conv("hyponet.params_dict.linear_wb1", a, b, ACT_SIN);
      N.conv("hyponet.params_dict.linear_wb2", b, a, ACT_SIN);
      N.conv("hyponet.params_dict.linear_wb3", a, b, ACT_SIN);
    } else {   // the other activations as a pass of their own after each layer
      N.conv("hyponet.params_dict.linear_wb0", hin, a); hypo_activation(cx, a, act, w0);
      N.conv("hyponet.params_dict.linear_wb1", a, b); hypo_activation(cx, b, act, w0);
      N.conv("hyponet.params_dict.linear_wb2", b, a); hypo_activation(cx, a, act, w0);
      N.conv("hyponet.params_dict.linear_wb3", a, b); hypo_activation(cx, b, act, w0);
    }
    N.conv("hyponet.params_dict.linear_wb4", b, ninr);
    A.release(mk);
  }
  if (!debug_) A.release(mk0);   // (debug taps keep pointing into this region)
}

// (B,2,2,H,W) flow pair, reference layout [b][c][j][y][x] -> NHWC (2B,H,W,2), sample j*B+b
struct FlowPairLoadK {
  const float* src; TV dst; int B;
  GV_HD void operator()(int64_t i) const {
    const int c = (int)(i & 1); int64_t r = i >> 1;
    const int x = (int)(r % dst.w); r /= dst.w; const int y = (int)(r % dst.h); const int n = (int)(r / dst.h);
    const int j = n / B, b = n - j * B;
    const int64_t hw = (int64_t)dst.h * dst.w;
    dst.p[dst.off(n, y, x) + c] = src[(((int64_t)b * 2 + c) * 2 + j) * hw + (int64_t)y * dst.w + x];
  }
};

// GIMM.forward (gimm.py:129-214): normalised flows xs + raw flows ori_flow + timesteps + coords -> normalised flows at t
void Engine::run_gimm(Ctx& cx, const Problem& P, const GimmIO& io) {
  if (P.B < 1 || P.T < 1) throw std::runtime_error("gimmvfi: B and T must be >= 1");
  const int B = P.B, H = P.Hf, W = P.Wf, T = P.T;
  if (P.ds > 0.f) throw std::runtime_error("gimm: ds_factor does not exist on this path");
  if (H < 8 || W < 8) throw std::runtime_error("gimm: H and W must be >= 8");
  if (P.Hc < 1 || P.Wc < 1) throw std::runtime_error("gimm: the coordinate grid must be at least 1 x 1");
  const int Hc = P.Hc, Wc = P.Wc;   // any size: HypoNet resizes the latent to the grid (hyponet.py:86-90)
  Net N{*this, cx};
  Arena& A = cx.arena;
  cx.tc = tc_mode_ >= 1; cx.tc_split = false;   // downstream-of-RAFT arithmetic (DESIGN.md precision plan)
  TV nf = A.tensor(2 * B, H, W, 2), fl = A.tensor(2 * B, H, W, 2);
  parallel_for(cx, nf.pixels() * 2, FlowPairLoadK{io.xs, nf, B}, "flow_pair_load");
  parallel_for(cx, fl.pixels() * 2, FlowPairLoadK{io.ori_flow, fl, B}, "flow_pair_load");
  TV f01 = fl.batch(0, B), f10 = fl.batch(B, B);
  TV wts = A.tensor(2 * B, H, W, 1);
  TV X64 = A.tensor(B, H, W, 64);
  gimm_encode(N, nf, f01, f10, wts, X64);
  TV ninr = A.tensor(B, Hc, Wc, 2);
  for (int ti = 0; ti < T; ++ti) {
    gimm_decode(N, X64, f01, f10, wts.batch(0, B), wts.batch(B, B), io.t + (int64_t)ti * B, io.coords + (int64_t)ti * B * Hc * Wc * 3, ninr, ti == T - 1);
    nhwc_to_nchw(cx, ninr, io.out + (int64_t)ti * B * 2 * Hc * Wc, (int64_t)2 * Hc * Wc, (int64_t)Hc * Wc, 1.f, 0.f, 0);
  }
}

// A workspace plan: `run` is the forward's run_* on a dry context (nothing launched or touched), under the current debug setting
size_t Engine::dry_run(const std::function<void(Ctx&)>& run) {
  Ctx cx; cx.dry = true; cx.arena.dry = true; cx.sm_count = sm_count_;
  run(cx);
  taps_.clear();
  return cx.arena.peak + 256;
}

// A forward: `run` launches on the caller's stream, with the workspace as its arena
void Engine::launch(void* workspace, size_t workspace_bytes, gvStream_t stream, const std::function<void(Ctx&)>& run) {
  DeviceGuard dg(device_);
  Ctx cx; cx.stream = stream; cx.sm_count = sm_count_;
  prof_.reset();
  cx.prof = profile_ ? &prof_ : nullptr;
  uintptr_t base = (reinterpret_cast<uintptr_t>(workspace) + 255) & ~uintptr_t(255);
  cx.arena.base = reinterpret_cast<char*>(base);
  cx.arena.cap = workspace_bytes - (base - reinterpret_cast<uintptr_t>(workspace));
  taps_.clear();
  run(cx);
  launches_ = cx.launches;
}

// the caller pointers of a dry run: never dereferenced, but optional outputs must be "present"
static float* const kFake = reinterpret_cast<float*>(size_t(64));

size_t Engine::plan_gimm(const Problem& p) {
  need(Entry::Gimm);
  GimmIO io;
  io.xs = io.ori_flow = io.coords = io.t = kFake; io.out = kFake;
  return dry_run([&](Ctx& cx) { run_gimm(cx, p, io); });
}

void Engine::forward_gimm(const Problem& p, const GimmIO& io, void* workspace, size_t workspace_bytes, gvStream_t stream) {
  need(Entry::Gimm);
  if (!io.xs || !io.ori_flow || !io.coords || !io.t || !io.out) throw std::runtime_error("gimm: xs, ori_flow, coords, t and out are required");
  launch(workspace, workspace_bytes, stream, [&](Ctx& cx) { run_gimm(cx, p, io); });
}

size_t Engine::frame_cache_bytes(const Problem& p) {
  const size_t h = (size_t)p.H() / 8, w = (size_t)p.W() / 8, H4 = (size_t)p.H() / 4, W4 = (size_t)p.W() / 4;
  return ((size_t)p.B * h * w * 256 * 3 + (size_t)p.B * H4 * W4 * 128) * sizeof(float);
}

static IO fake_io() {
  IO io;
  io.img_xs = io.coords = io.t = kFake;
  io.imgt_pred = io.img_warp_4 = io.flowt0_1 = io.flowt1_1 = io.flowt0_4 = io.flowt1_4 = io.raft_flow = io.nflow = io.ninrflow = io.flowt = kFake;
  return io;
}

size_t Engine::plan_from_flow(const Problem& p) {
  need(Entry::FromFlow);
  FlowInputs fin; fin.flows = kFake;
  for (int j = 0; j < 2; ++j) fin.feat4[j] = fin.feat8[j] = fin.fnet[j] = kFake;
  return dry_run([&](Ctx& cx) { run(cx, p, fake_io(), schedule_batch(p), &fin); });
}

void Engine::forward_from_flow(const Problem& p, const IO& io, const FlowInputs& fin, void* workspace, size_t workspace_bytes, gvStream_t stream) {
  need(Entry::FromFlow);
  if (!io.img_xs || !io.coords || !io.t || !io.imgt_pred) throw std::runtime_error("gimmvfi: img_xs, coords, t and imgt_pred are required");
  if (!fin.flows || !fin.feat4[0] || !fin.feat4[1] || !fin.feat8[0] || !fin.feat8[1] || !fin.fnet[0] || !fin.fnet[1])
    throw std::runtime_error("gimmvfi: forward_from_flow needs flows, feat4[2], feat8[2] and fnet[2]");
  launch(workspace, workspace_bytes, stream, [&](Ctx& cx) { run(cx, p, io, schedule_batch(p), &fin); });
}

size_t Engine::plan(const Problem& p) {
  need(Entry::Interpolate);
  return dry_run([&](Ctx& cx) { run(cx, p, fake_io(), schedule_batch(p)); });
}

void Engine::clear_graphs() {
#ifndef GV_HOSTSIM
  DeviceGuard dg(device_);
  for (GraphEntry& g : graphs_) if (g.exec) cudaGraphExecDestroy((cudaGraphExec_t)g.exec);
#endif
  graphs_.clear();
}

void Engine::forward(const Problem& p, const IO& io, void* workspace, size_t workspace_bytes, gvStream_t stream) {
  need(Entry::Interpolate);
  if (!io.img_xs || !io.coords || !io.t || !io.imgt_pred) throw std::runtime_error("gimmvfi: img_xs, coords, t and imgt_pred are required");
  const Schedule s = schedule_batch(p);
  launch(workspace, workspace_bytes, stream, [&](Ctx& cx) {
#ifndef GV_HOSTSIM
    // (the legacy default stream - handles 0 / 1 / 2 - cannot be captured: such callers run eagerly)
    if (use_graph_ && !profile_ && !debug_ && fc_ == nullptr && reinterpret_cast<uintptr_t>(stream) > 2) {
      // everything a recorded launch sequence depends on: problem, every caller pointer, the workspace, the arithmetic mode, the weights
      std::vector<uint64_t> key = {(uint64_t)p.B, (uint64_t)p.Hf, (uint64_t)p.Wf, (uint64_t)p.T, (uint64_t)p.Hc, (uint64_t)p.Wc, 0, (uint64_t)tc_mode_,
                                   (uint64_t)(raft_direct_ + 2), (uint64_t)weights_version_, (uint64_t)raft_iters, (uint64_t)workspace, (uint64_t)workspace_bytes, (uint64_t)(uintptr_t)stream};
      std::memcpy(&key[6], &p.ds, sizeof(float));
      const void* ptrs[] = {io.img_xs, io.coords, io.t, io.imgt_pred, io.img_warp_4, io.flowt0_1, io.flowt1_1, io.flowt0_4, io.flowt1_4, io.raft_flow, io.nflow, io.ninrflow, io.flowt};
      for (const void* q : ptrs) key.push_back((uint64_t)(uintptr_t)q);
      GraphEntry* hit = nullptr;
      for (GraphEntry& g : graphs_) if (g.key == key) { hit = &g; break; }
      if (hit && hit->exec) {
        cuda_ok(cudaGraphLaunch((cudaGraphExec_t)hit->exec, stream), "cudaGraphLaunch");
        cx.launches = hit->launches; ++graph_replays_;
        return;
      }
      if (hit && hit->seen >= 1) {   // second sighting: record.  (The first call ran eagerly: lazy one-time host work - function attributes - is done.)
        cudaGraph_t graph = nullptr;
        cuda_ok(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal), "cudaStreamBeginCapture");
        try {
          run(cx, p, io, s);
        } catch (...) {
          cudaStreamEndCapture(stream, &graph);
          if (graph) cudaGraphDestroy(graph);
          throw;
        }
        cuda_ok(cudaStreamEndCapture(stream, &graph), "cudaStreamEndCapture");
        cudaGraphExec_t exec = nullptr;
        cuda_ok(cudaGraphInstantiate(&exec, graph, 0), "cudaGraphInstantiate");
        cudaGraphDestroy(graph);
        hit->exec = exec; hit->launches = cx.launches;
        cuda_ok(cudaGraphLaunch(exec, stream), "cudaGraphLaunch");
        ++graph_replays_;
        return;
      }
      if (!hit) {
        if (graphs_.size() >= 8) { if (graphs_.front().exec) cudaGraphExecDestroy((cudaGraphExec_t)graphs_.front().exec); graphs_.erase(graphs_.begin()); }
        GraphEntry g; g.key = key; g.seen = 1;
        graphs_.push_back(g);
      }
    }
#endif
    run(cx, p, io, s);
  });
}

size_t Engine::plan_clip(const Problem& p, const Clip& c) {
  need(Entry::Interpolate);
  return dry_run([&](Ctx& cx) { run(cx, p, fake_io(), schedule_clip(p, c)); });
}

// (eager: a clip's launch sequence depends on its pair list, which the CUDA-graph key of forward() does not hold)
void Engine::forward_clip(const Problem& p, const Clip& c, const IO& io, void* workspace, size_t workspace_bytes, gvStream_t stream) {
  need(Entry::Interpolate);
  if (!io.img_xs || !io.coords || !io.t || !io.imgt_pred) throw std::runtime_error("gimmvfi: frames, coords, t and imgt_pred are required");
  launch(workspace, workspace_bytes, stream, [&](Ctx& cx) { run(cx, p, io, schedule_clip(p, c)); });
}

size_t Engine::plan_queries(const Problem& p, const Queries& q) {
  need(Entry::Interpolate);
  return dry_run([&](Ctx& cx) { run(cx, p, fake_io(), schedule_queries(p, q)); });
}

// (eager, as forward_clip)
void Engine::forward_queries(const Problem& p, const Queries& q, const IO& io, void* workspace, size_t workspace_bytes, gvStream_t stream) {
  need(Entry::Interpolate);
  if (!io.img_xs || !io.imgt_pred) throw std::runtime_error("gimmvfi: frames and imgt_pred are required");
  if (io.coords || io.t) throw std::runtime_error("gimmvfi: a query list's coordinates and t are made by the engine; io.coords and io.t must be null");
  launch(workspace, workspace_bytes, stream, [&](Ctx& cx) { run(cx, p, io, schedule_queries(p, q)); });
}

// ---------------------------------------------------------------------------
// FlowFormer over a frame set and a pair list (flowformer.cu run_flowformer): FlowFormer.forward(image1, image2) of the reference
// (transformer.py:45-74) for every pair, the encoders shared between the pairs that use the same frame
// ---------------------------------------------------------------------------
void Engine::run_flowformer_pairs(Ctx& cx, const float* frames, int F, int H, int W, const std::vector<int>& src, const std::vector<int>& tgt,
                                  int per_call, int iters, bool gather, const float* flow_init, const FlowFormerOutputs& o) {
  if (F < 1 || H < 32 || W < 32) throw std::runtime_error("flowformer: at least one frame of at least 32 x 32 pixels is required");
  if (H % 32 || W % 32) throw std::runtime_error("gimmvfi: FlowFormer needs a network resolution that is a multiple of 32 (Twins-SVT sub-sampling)");
  if (iters < 1) throw std::runtime_error("flowformer: iters must be >= 1");
  Net N{*this, cx};
  Arena& A = cx.arena;
  cx.tc = tc_mode_ >= 2; cx.tc_split = true;   // the recurrence amplifies operand rounding: fp32-class arithmetic only (as in run())
  const int S = (int)src.size(), h = H / 8, w = W / 8, H4 = H / 4, W4 = W / 4;
  TV img = A.tensor(F, H, W, 3, 4);
  parallel_for(cx, (int64_t)F * 3 * H * W, FlowFormerPrepK{frames, img}, "flowformer_prep");
  TV up = A.tensor(S, H, W, 2), low = o.flow_low ? A.tensor(S, h, w, 2) : TV();
  std::vector<int> slot(F, -1);   // the order in which run_flowformer encodes the distinct sources
  int ns = 0;
  for (int s : src) if (slot[s] < 0) slot[s] = ns++;
  // return_feat=True (transformer.py:57-66): the context Twins' stage outputs and the channel_convertor output of each pair's source,
  // written straight from the encoders' buffers (no workspace of their own)
  auto encoded = [&](const TV& c4, const TV& c8, const TV& fproj) {
    for (int s = 0; s < S; ++s) {
      if (o.cfeat4) nhwc_to_nchw(cx, c4.batch(slot[src[s]], 1), o.cfeat4 + (int64_t)s * 128 * H4 * W4, (int64_t)128 * H4 * W4, (int64_t)H4 * W4, 1.f, 0.f, 0);
      if (o.cfeat8) nhwc_to_nchw(cx, c8.batch(slot[src[s]], 1), o.cfeat8 + (int64_t)s * 256 * h * w, (int64_t)256 * h * w, (int64_t)h * w, 1.f, 0.f, 0);
      if (o.ffeat) nhwc_to_nchw(cx, fproj.batch(src[s], 1), o.ffeat + (int64_t)s * 256 * h * w, (int64_t)256 * h * w, (int64_t)h * w, 1.f, 0.f, 0);
    }
  };
  const bool feats = o.cfeat4 || o.cfeat8 || o.ffeat;
  run_flowformer(cx, N, img, src, tgt, per_call, iters, gather, up, low, TV(), TV(), TV(), flow_init,
                 feats ? std::function<void(const TV&, const TV&, const TV&)>(encoded) : nullptr);
  nhwc_to_nchw(cx, up, o.flow_up, (int64_t)2 * H * W, (int64_t)H * W, 1.f, 0.f, 0);
  if (o.flow_low) nhwc_to_nchw(cx, low, o.flow_low, (int64_t)2 * h * w, (int64_t)h * w, 1.f, 0.f, 0);
}

size_t Engine::plan_flowformer(int n_frames, int h, int w, int n_pairs) {
  need(Entry::FlowFormer);
  if (n_pairs < 1) throw std::runtime_error("flowformer: at least one pair is required");
  if (n_frames < 1) throw std::runtime_error("flowformer: at least one frame is required");
  // the most memory any pair list of this size can take: min(F, P) distinct sources and the context gathered into pair order.  This bound
  // holds because run_flowformer's workspace does not depend on the pair values beyond the number of distinct sources, nor on iters or
  // per_call, flow_init or the feature outputs (written straight from the encoders' buffers), and the gathering path only adds buffers:
  // a change that breaks either must change this plan too.
  std::vector<int> src(n_pairs), tgt(n_pairs);
  for (int s = 0; s < n_pairs; ++s) { src[s] = s % n_frames; tgt[s] = (s + 1) % n_frames; }
  FlowFormerOutputs o; o.flow_up = o.flow_low = kFake;
  // debug: 2 iterations, so that the snapshots of iteration 0 and those of the last iteration are planned in the order a forward takes them
  return dry_run([&](Ctx& cx) { run_flowformer_pairs(cx, kFake, n_frames, h, w, src, tgt, 1, debug_ ? 2 : 1, true, nullptr, o); });
}

void Engine::forward_flowformer(const float* frames, int n_frames, int h, int w, const int32_t* pairs, int n_pairs, int pairs_per_call, int iters,
                                const float* flow_init, const FlowFormerOutputs& out, void* workspace, size_t workspace_bytes, gvStream_t stream) {
  need(Entry::FlowFormer);
  if (!frames || !pairs || !out.flow_up) throw std::runtime_error("flowformer: frames, pairs and flow_up are required");
  if (n_pairs < 1) throw std::runtime_error("flowformer: at least one pair is required");
  if (pairs_per_call < 1 || n_pairs % pairs_per_call) throw std::runtime_error("flowformer: n_pairs must be a multiple of pairs_per_call (>= 1)");
  if (iters < 0) throw std::runtime_error("flowformer: iters must be >= 0 (0: the engine's decoder depth)");
  std::vector<int> src(n_pairs), tgt(n_pairs);
  for (int s = 0; s < n_pairs; ++s) {
    src[s] = pairs[2 * s]; tgt[s] = pairs[2 * s + 1];
    if (src[s] < 0 || src[s] >= n_frames || tgt[s] < 0 || tgt[s] >= n_frames)
      throw std::runtime_error("flowformer: pair " + std::to_string(s) + " = (" + std::to_string(src[s]) + ", " + std::to_string(tgt[s]) +
                               ") indexes outside the " + std::to_string(n_frames) + " frames");
  }
  launch(workspace, workspace_bytes, stream,
         [&](Ctx& cx) { run_flowformer_pairs(cx, frames, n_frames, h, w, src, tgt, pairs_per_call, iters ? iters : ff_iters, false, flow_init, out); });
}

// ---------------------------------------------------------------------------
// RAFT over a frame set and a pair list (run_raft): RAFT.forward(image1, image2, iters, flow_init) of the reference (raft/raft.py:100-169)
// for every pair with batch 1, the encoders shared between the pairs that use the same frame
// ---------------------------------------------------------------------------
void Engine::run_raft_pairs(Ctx& cx, const float* frames, int F, int H, int W, const std::vector<int>& src, const std::vector<int>& tgt, int iters,
                            const float* flow_init, const RaftOutputs& o, bool gather) {
  if (F < 1) throw std::runtime_error("raft: at least one frame is required");
  if (H % 8 || W % 8 || H < 128 || W < 128)   // (the 4-level pyramid halves H/8 three times: raft/corr.py:23-44 divides by zero below 128)
    throw std::runtime_error("raft: frames must be a multiple of 8 and >= 128 in each dimension (got " + std::to_string(H) + "x" + std::to_string(W) + ")");
  if (iters < 1) throw std::runtime_error("raft: iters must be >= 1");
  Net N{*this, cx};
  Arena& A = cx.arena;
  cx.tc = tc_mode_ >= 2; cx.tc_split = true;   // fp32-class arithmetic only (as in run())
  const int S = (int)src.size(), h = H / 8, w = W / 8, H4 = H / 4, W4 = W / 4;
  RaftRun r;
  r.img = A.tensor(F, H, W, 3, 4);
  parallel_for(cx, (int64_t)F * 3 * H * W, FlowFormerPrepK{frames, r.img}, "raft_frame_prep");
  r.src = src; r.tgt = tgt; r.iters = iters; r.gather = gather; r.flow_init = flow_init;
  r.flow_up = A.tensor(S, H, W, 2);
  r.flow_low = o.flow_low ? A.tensor(S, h, w, 2) : TV();
  r.flow_iters = o.flow_iters;
  r.fmap = A.tensor(F, h, w, 256);
  std::vector<int> slot(F, -1);   // the order in which run_raft encodes the distinct sources
  int ns = 0;
  for (int s : src) if (slot[s] < 0) slot[s] = ns++;
  r.encoded = [&](const TV& c4, const TV& c8, const TV&) {   // feats[1:] of cnet(image1, return_feature=True), raft.py:131,169
    for (int s = 0; s < S; ++s) {
      if (o.feat4) nhwc_to_nchw(cx, c4.batch(slot[src[s]], 1), o.feat4 + (int64_t)s * 96 * H4 * W4, (int64_t)96 * H4 * W4, (int64_t)H4 * W4, 1.f, 0.f, 0);
      if (o.feat8) nhwc_to_nchw(cx, c8.batch(slot[src[s]], 1), o.feat8 + (int64_t)s * 128 * h * w, (int64_t)128 * h * w, (int64_t)h * w, 1.f, 0.f, 0);
    }
  };
  run_raft(cx, N, r);
  if (o.flow_up) nhwc_to_nchw(cx, r.flow_up, o.flow_up, (int64_t)2 * H * W, (int64_t)H * W, 1.f, 0.f, 0);
  if (o.flow_low) nhwc_to_nchw(cx, r.flow_low, o.flow_low, (int64_t)2 * h * w, (int64_t)h * w, 1.f, 0.f, 0);
  if (o.fmap)
    for (int s = 0; s < S; ++s) nhwc_to_nchw(cx, r.fmap.batch(src[s], 1), o.fmap + (int64_t)s * 256 * h * w, (int64_t)256 * h * w, (int64_t)h * w, 1.f, 0.f, 0);
}

size_t Engine::plan_raft(int n_frames, int h, int w, int n_pairs, int outputs) {
  need(Entry::Raft);
  if (n_pairs < 1) throw std::runtime_error("raft: at least one pair is required");
  if (n_frames < 1) throw std::runtime_error("raft: at least one frame is required");
  if (outputs & ~GIMMVFI_RAFT_OUT_ITERS) throw std::runtime_error("raft: unknown output flags");
  // the most memory any pair list of this size can take: min(F, P) distinct sources and the context gathered into pair order.  This bound
  // holds because run_raft's workspace does not depend on the pair values beyond the number of distinct sources, nor on iters or
  // flow_init, and the gathering path only adds buffers: a change that breaks either must change this plan too.
  std::vector<int> src(n_pairs), tgt(n_pairs);
  for (int s = 0; s < n_pairs; ++s) { src[s] = s % n_frames; tgt[s] = (s + 1) % n_frames; }
  RaftOutputs o; o.flow_up = o.flow_low = o.feat4 = o.feat8 = o.fmap = kFake;
  if (outputs & GIMMVFI_RAFT_OUT_ITERS) o.flow_iters = kFake;
  // debug: 5 iterations, so that the snapshots of iterations 0 and 4 and those of the last iteration are all planned
  return dry_run([&](Ctx& cx) { run_raft_pairs(cx, kFake, n_frames, h, w, src, tgt, debug_ ? 5 : 1, nullptr, o, true); });
}

void Engine::forward_raft(const float* frames, int n_frames, int h, int w, const int32_t* pairs, int n_pairs, int iters, const float* flow_init,
                          const RaftOutputs& out, void* workspace, size_t workspace_bytes, gvStream_t stream) {
  need(Entry::Raft);
  if (!frames || !pairs) throw std::runtime_error("raft: frames and pairs are required");
  if (n_pairs < 1) throw std::runtime_error("raft: at least one pair is required");
  if (iters < 1) throw std::runtime_error("raft: iters must be >= 1");
  std::vector<int> src(n_pairs), tgt(n_pairs);
  for (int s = 0; s < n_pairs; ++s) {
    src[s] = pairs[2 * s]; tgt[s] = pairs[2 * s + 1];
    if (src[s] < 0 || src[s] >= n_frames || tgt[s] < 0 || tgt[s] >= n_frames)
      throw std::runtime_error("raft: pair " + std::to_string(s) + " = (" + std::to_string(src[s]) + ", " + std::to_string(tgt[s]) +
                               ") indexes outside the " + std::to_string(n_frames) + " frames");
  }
  launch(workspace, workspace_bytes, stream, [&](Ctx& cx) { run_raft_pairs(cx, frames, n_frames, h, w, src, tgt, iters, flow_init, out, false); });
}

// ---------------------------------------------------------------------------
// LPIPS (src/utils/lpips/lpips.py:38-189 with net="alex", version="0.1"): features[0:12] of torchvision's AlexNet
// (pretrained_networks.py:70-110) on [in0 ; in1] in one pass, then the calibrated head of the five ReLU outputs
// ---------------------------------------------------------------------------
static const char* const kLpipsConv[5] = {"net.slice1.0", "net.slice2.3", "net.slice3.6", "net.slice4.8", "net.slice5.10"};
static const int kLpipsShape[5][4] = {{64, 3, 11, 11}, {192, 64, 5, 5}, {384, 192, 3, 3}, {256, 384, 3, 3}, {256, 256, 3, 3}};

void Engine::finalize_weights_lpips() {
  DeviceGuard dg(device_);
  drop_weights();
  auto expect = [&](const std::string& key, std::vector<int64_t> shape) {
    const HostTensor& t = raw(key);
    if (t.shape != shape) throw std::runtime_error("gimmvfi: LPIPS weight '" + key + "' has an unexpected shape");
  };
  expect("scaling_layer.shift", {1, 3, 1, 1}); expect("scaling_layer.scale", {1, 3, 1, 1});
  for (int k = 0; k < 5; ++k) {
    const int* s = kLpipsShape[k];
    expect(std::string(kLpipsConv[k]) + ".weight", {s[0], s[1], s[2], s[3]});
    expect(std::string(kLpipsConv[k]) + ".bias", {s[0]});
    const std::string lin = "lin" + std::to_string(k) + ".model.1.weight", dup = "lins." + std::to_string(k) + ".model.1.weight";
    expect(lin, {1, s[0], 1, 1});
    if (raw_.count(dup) && raw(dup).data != raw(lin).data) throw std::runtime_error("gimmvfi: LPIPS weight '" + dup + "' differs from '" + lin + "'");
  }
  // conv1 (11x11, stride 4, pad 2) on the 4x4 space-to-depth of the padded image: output row y reads padded rows 4y .. 4y+10 = s2d rows
  // y, y+1, y+2, so the kernel zero-extended to 12x12 is a 3x3 kernel over 48 channels (channel (dy * 4 + dx) * 3 + c, as lpips_prep)
  {
    const HostTensor& W = raw("net.slice1.0.weight");
    HostTensor w2; w2.shape = {64, 48, 3, 3}; w2.data.assign((size_t)64 * 48 * 9, 0.f);
    for (int co = 0; co < 64; ++co)
      for (int c = 0; c < 3; ++c)
        for (int ky = 0; ky < 11; ++ky)
          for (int kx = 0; kx < 11; ++kx) {
            const int ch = ((ky % 4) * 4 + kx % 4) * 3 + c;
            w2.data[(((size_t)co * 48 + ch) * 3 + ky / 4) * 3 + kx / 4] = W.data[(((size_t)co * 3 + c) * 11 + ky) * 11 + kx];
          }
    raw_["net.slice1.0#s2d.weight"] = w2; raw_["net.slice1.0#s2d.bias"] = raw("net.slice1.0.bias");
    pack_conv("net.slice1.0#s2d");
  }
  for (int k = 1; k < 5; ++k) pack_conv(kLpipsConv[k]);
  vec("scaling_layer.shift"); vec("scaling_layer.scale");
  for (int k = 0; k < 5; ++k) vec("lin" + std::to_string(k) + ".model.1.weight");
  held_ = Weights::Lpips;
}

void Engine::run_lpips(Ctx& cx, int n, int h, int w, const LpipsIO& io) {
  Net N{*this, cx};
  Arena& A = cx.arena;
  cx.tc = true; cx.tc_split = true;   // every convolution in the fp32-class 3xF16 form
  const int oh = (h + 4 - 11) / 4 + 1, ow = (w + 4 - 11) / 4 + 1;   // AlexNet's conv1 output
  if (n < 1 || h + 4 < 11 || w + 4 < 11 || (oh - 3) / 2 + 1 < 3 || (ow - 3) / 2 + 1 < 3 || oh < 3 || ow < 3)
    throw std::runtime_error("lpips: images of at least 31 x 31 pixels are required (AlexNet's second max-pool needs a 3 x 3 map)");
  const int n2 = 2 * n;
  // the s2d grid covers the taps of every output pixel (one row / column more than the image may need: zeros)
  TV s2d = A.tensor(n2, oh + 2, ow + 2, 48);
  lpips_prep(cx, io.in0, io.in1, n, h, w, io.quantize, io.normalize, N.V("scaling_layer.shift"), N.V("scaling_layer.scale"), s2d);
  TV f[5];
  f[0] = A.tensor(n2, oh, ow, 64);
  {
    ConvGeom g; g.stride = 1; g.ph = 0; g.pw = 0; g.loose_w = 1;
    ConvEpi e; e.act1 = ACT_RELU;
    conv2d(cx, s2d, TV(), N.W("net.slice1.0#s2d"), g, e, f[0]);
  }
  TV p1 = A.tensor(n2, (oh - 3) / 2 + 1, (ow - 3) / 2 + 1, 64);
  maxpool3x3s2(cx, f[0], p1);
  f[1] = A.tensor(n2, p1.h, p1.w, 192);
  N.conv(kLpipsConv[1], p1, f[1], ACT_RELU);
  TV p2 = A.tensor(n2, (p1.h - 3) / 2 + 1, (p1.w - 3) / 2 + 1, 192);
  maxpool3x3s2(cx, f[1], p2);
  f[2] = A.tensor(n2, p2.h, p2.w, 384);
  N.conv(kLpipsConv[2], p2, f[2], ACT_RELU);
  f[3] = A.tensor(n2, p2.h, p2.w, 256);
  N.conv(kLpipsConv[3], f[2], f[3], ACT_RELU);
  f[4] = A.tensor(n2, p2.h, p2.w, 256);
  N.conv(kLpipsConv[4], f[3], f[4], ACT_RELU);
  const double* part[5]; int hs[5], ws[5];
  for (int k = 0; k < 5; ++k) {
    double* pk = reinterpret_cast<double*>(A.alloc_f((size_t)2 * n * f[k].h));
    lpips_head_rows(cx, f[k], n, N.V("lin" + std::to_string(k) + ".model.1.weight"), pk);
    part[k] = pk; hs[k] = f[k].h; ws[k] = f[k].w;
    tap("lpips.relu" + std::to_string(k + 1), f[k]);
  }
  lpips_head_images(cx, part, hs, ws, n, io.per_layer, io.out);
}

size_t Engine::plan_lpips(int n, int h, int w) {
  need(Entry::Lpips);
  LpipsIO io;
  io.in0 = io.in1 = io.out = kFake;
  return dry_run([&](Ctx& cx) { run_lpips(cx, n, h, w, io); });
}

void Engine::forward_lpips(int n, int h, int w, const LpipsIO& io, void* workspace, size_t workspace_bytes, gvStream_t stream) {
  need(Entry::Lpips);
  if (!io.in0 || !io.in1 || !io.out) throw std::runtime_error("lpips: in0, in1 and out are required");
  launch(workspace, workspace_bytes, stream, [&](Ctx& cx) { run_lpips(cx, n, h, w, io); });
}

}  // namespace gv
