// extern "C" boundary (include/gimmvfi_b200.h).  No exceptions cross it.
#include "../../include/gimmvfi_b200.h"
#include "engine.h"

using namespace gv;

struct gimmvfi_engine {
  Engine eng;
  std::string err, prof_json;
  explicit gimmvfi_engine(int dev) : eng(dev) {}
};

static thread_local std::string g_static_err;

#define GV_TRY(e_, body)                                          \
  try { body; return 0; }                                         \
  catch (const std::exception& ex) { if (e_) (e_)->err = ex.what(); else g_static_err = ex.what(); return 1; } \
  catch (...) { if (e_) (e_)->err = "unknown error"; else g_static_err = "unknown error"; return 1; }

static TV to_tv(const gimmvfi_view* v) {
  TV t;
  if (!v) return t;
  t.p = v->data; t.n = v->n; t.h = v->h; t.w = v->w; t.c = v->c; t.ld = v->pixel_stride; t.sn = v->batch_stride;
  return t;
}
static Ctx op_ctx(void* stream) {
  Ctx cx; cx.stream = (gvStream_t)stream;
#ifndef GV_HOSTSIM
  int dev = 0; cudaGetDevice(&dev); int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); cx.sm_count = sms;
#endif
  return cx;
}
static Problem to_problem(const gimmvfi_problem* p) {
  Problem q; q.B = p->batch; q.Hf = p->height; q.Wf = p->width; q.T = p->timesteps; q.ds = p->ds_factor; q.Hc = p->coord_height; q.Wc = p->coord_width;
  return q;
}
static IO to_io(const gimmvfi_io* io) {
  IO q;
  q.img_xs = io->img_xs; q.coords = io->coords; q.t = io->t; q.imgt_pred = io->imgt_pred; q.img_warp_4 = io->img_warp_4;
  q.flowt0_1 = io->flowt0_1; q.flowt1_1 = io->flowt1_1; q.flowt0_4 = io->flowt0_4; q.flowt1_4 = io->flowt1_4;
  q.raft_flow = io->raft_flow; q.nflow = io->nflow; q.ninrflow = io->ninrflow; q.flowt = io->flowt;
  return q;
}

// ---- strided 4-D tensors of the differentiable splat
template <class T> static SV4<T> sv4(const gimmvfi_tensor4* t) {
  SV4<T> s;
  if (!t) return s;
  s.p = static_cast<T*>(t->data);
  for (int d = 0; d < 4; ++d) { s.sz[d] = t->sizes[d]; s.st[d] = t->strides[d]; }
  return s;
}
// every element at a distinct offset and the offsets one contiguous block starting at data (any dimension order)
static bool dense4(const gimmvfi_tensor4& t) {
  int idx[4] = {0, 1, 2, 3};
  for (int a = 0; a < 4; ++a)
    for (int b = a + 1; b < 4; ++b)
      if (t.strides[idx[b]] < t.strides[idx[a]]) std::swap(idx[a], idx[b]);
  int64_t expect = 1;
  for (int k = 0; k < 4; ++k) {
    const int d = idx[k];
    if (t.sizes[d] == 1) continue;
    if (t.strides[d] != expect) return false;
    expect *= t.sizes[d];
  }
  return true;
}
// the host-side checks of gimmvfi_op_softsplat_out / _grad: `c_ref` is out or outgrad (C channels like `in`); ingrad / flowgrad optional
static void splat_check(const gimmvfi_tensor4* in, const gimmvfi_tensor4* flow, const gimmvfi_tensor4* c_ref, const gimmvfi_tensor4* ingrad,
                        const gimmvfi_tensor4* flowgrad, const char* what) {
  const std::string w(what);
  if (!in || !flow || !c_ref) throw std::runtime_error(w + ": in and flow are required");
  const gimmvfi_tensor4* all[5] = {in, flow, c_ref, ingrad, flowgrad};
  for (const gimmvfi_tensor4* t : all) {
    if (!t) continue;
    if (t->dtype != GIMMVFI_FLOAT32 && t->dtype != GIMMVFI_FLOAT64) throw std::runtime_error(w + ": dtype must be float32 or float64");
    if (t->dtype != in->dtype) throw std::runtime_error(w + ": every tensor must have the same dtype");
    for (int d = 0; d < 4; ++d)
      if (t->sizes[d] < 0 || t->sizes[d] > (int64_t(1) << 40) || t->strides[d] < 0) throw std::runtime_error(w + ": negative size or stride");
    if (t->sizes[0] != in->sizes[0] || t->sizes[2] != in->sizes[2] || t->sizes[3] != in->sizes[3])
      throw std::runtime_error(w + ": N, H and W must be equal for every tensor");
  }
  if (flow->sizes[1] != 2) throw std::runtime_error(w + ": flow must have 2 channels");
  if (c_ref->sizes[1] != in->sizes[1] || (ingrad && ingrad->sizes[1] != in->sizes[1]))
    throw std::runtime_error(w + ": in, out / outgrad and ingrad must have the same channels");
  if (flowgrad && flowgrad->sizes[1] != 2) throw std::runtime_error(w + ": flowgrad must have 2 channels");
  // `in` is read by the forward and by flowgrad only
  const bool reads_in = flowgrad || !ingrad;
  if (in->sizes[0] * in->sizes[2] * in->sizes[3] > 0 &&
      (!flow->data || !c_ref->data || (ingrad && !ingrad->data) || (flowgrad && !flowgrad->data) || (reads_in && !in->data)))
    throw std::runtime_error(w + ": NULL data pointer");
}

// ---- dense tensors of the memory-free correlation
static int64_t dense_numel(const gimmvfi_dense& t) {
  int64_t n = 1;
  for (int d = 0; d < t.ndim; ++d) n *= t.sizes[d];
  return n;
}
// t is a float32 tensor of the given sizes (ndim = sizes.size())
static void dense_expect(const gimmvfi_dense* t, const std::vector<int64_t>& sizes, const std::string& w, const char* name) {
  if (!t) throw std::runtime_error(w + ": " + name + " is required");
  if (t->dtype != GIMMVFI_FLOAT32) throw std::runtime_error(w + ": " + name + " must be float32");
  if (t->ndim != (int)sizes.size()) throw std::runtime_error(w + ": " + name + " must have " + std::to_string(sizes.size()) + " dimensions");
  for (int d = 0; d < t->ndim; ++d)
    if (t->sizes[d] != sizes[d]) {
      std::string want = "(";
      for (size_t k = 0; k < sizes.size(); ++k) want += (k ? ", " : "") + std::to_string(sizes[k]);
      throw std::runtime_error(w + ": " + name + " must have the shape " + want + ")");
    }
  if (dense_numel(*t) > 0 && !t->data) throw std::runtime_error(w + ": NULL data pointer in " + name);
}
// the host-side checks shared by the forward and the backward; returns the kernel arguments
static AltCorrArgs alt_corr_args(const gimmvfi_dense* fmap1, const gimmvfi_dense* fmap2, const gimmvfi_dense* coords, int radius, const std::string& w) {
  const gimmvfi_dense* all[3] = {fmap1, fmap2, coords};
  const char* names[3] = {"fmap1", "fmap2", "coords"};
  const int ranks[3] = {4, 4, 5};
  for (int i = 0; i < 3; ++i) {
    const gimmvfi_dense* t = all[i];
    if (!t) throw std::runtime_error(w + ": " + names[i] + " is required");
    if (t->dtype != GIMMVFI_FLOAT32) throw std::runtime_error(w + ": " + names[i] + " must be float32");
    if (t->ndim != ranks[i]) throw std::runtime_error(w + ": " + names[i] + " must have " + std::to_string(ranks[i]) + " dimensions");
    for (int d = 0; d < t->ndim; ++d)
      if (t->sizes[d] < 0 || t->sizes[d] > INT32_MAX) throw std::runtime_error(w + ": " + names[i] + " has a negative or too large size");
  }
  if (fmap2->sizes[0] != fmap1->sizes[0] || coords->sizes[0] != fmap1->sizes[0]) throw std::runtime_error(w + ": B must be equal for every tensor");
  if (coords->sizes[2] != fmap1->sizes[1] || coords->sizes[3] != fmap1->sizes[2]) throw std::runtime_error(w + ": coords and fmap1 must have equal H1 and W1");
  if (coords->sizes[4] != 2) throw std::runtime_error(w + ": the last dimension of coords must be 2 (x, y)");
  if (fmap2->sizes[3] != fmap1->sizes[3]) throw std::runtime_error(w + ": fmap1 and fmap2 must have the same channels");
  if (fmap1->sizes[3] < 1) throw std::runtime_error(w + ": C must be >= 1");
  int nw, tw;
  if (radius < 0) throw std::runtime_error(w + ": radius must be >= 0");
  if (!alt_corr_launch_shape(radius, &nw, &tw)) throw std::runtime_error(w + ": radius too large for the shared memory of one window");
  if (fmap2->sizes[1] * fmap2->sizes[2] * fmap2->sizes[3] > INT32_MAX) throw std::runtime_error(w + ": H2 * W2 * C must be below 2^31");
  for (int i = 0; i < 3; ++i)
    if (dense_numel(*all[i]) > 0 && !all[i]->data) throw std::runtime_error(w + ": NULL data pointer in " + names[i]);
  AltCorrArgs a;
  a.f1 = static_cast<const float*>(fmap1->data); a.f2 = static_cast<const float*>(fmap2->data); a.coords = static_cast<const float*>(coords->data);
  a.B = (int)fmap1->sizes[0]; a.H1 = (int)fmap1->sizes[1]; a.W1 = (int)fmap1->sizes[2]; a.C = (int)fmap1->sizes[3];
  a.H2 = (int)fmap2->sizes[1]; a.W2 = (int)fmap2->sizes[2]; a.N = (int)coords->sizes[1]; a.r = radius;
  return a;
}
static std::vector<int64_t> alt_corr_shape(const AltCorrArgs& a) {
  const int64_t rd = 2 * (int64_t)a.r + 1;
  return {a.B, a.N, rd * rd, a.H1, a.W1};
}

extern "C" {

int gimmvfi_create(int device, gimmvfi_engine** out) {
  gimmvfi_engine* none = nullptr;
  GV_TRY(none, { *out = new gimmvfi_engine(device); })
}
void gimmvfi_destroy(gimmvfi_engine* e) { delete e; }

int gimmvfi_load_weight(gimmvfi_engine* e, const char* key, const float* host_data, const int64_t* shape, int ndim) {
  GV_TRY(e, { e->eng.load_weight(key, host_data, shape, ndim); })
}
int gimmvfi_finalize_weights(gimmvfi_engine* e) { GV_TRY(e, { e->eng.finalize_weights(); }) }

int gimmvfi_plan(gimmvfi_engine* e, const gimmvfi_problem* p, size_t* workspace_bytes) {
  GV_TRY(e, { *workspace_bytes = e->eng.plan(to_problem(p)); })
}

int gimmvfi_forward(gimmvfi_engine* e, const gimmvfi_problem* p, const gimmvfi_io* io, void* workspace, size_t workspace_bytes,
                    void* cuda_stream) {
  GV_TRY(e, { e->eng.forward(to_problem(p), to_io(io), workspace, workspace_bytes, (gvStream_t)cuda_stream); })
}

static Clip to_clip(const gimmvfi_problem* p, const gimmvfi_clip* c) {
  if (!p || !c || !c->pair_list) throw std::runtime_error("gimmvfi clip: problem, clip and pair_list are required");
  if (c->pairs < 1) throw std::runtime_error("gimmvfi clip: at least one pair is required");
  if (c->frames < 1) throw std::runtime_error("gimmvfi clip: at least one frame is required");
  Clip q; q.F = c->frames;
  for (int s = 0; s < c->pairs; ++s) { q.src.push_back(c->pair_list[2 * s]); q.tgt.push_back(c->pair_list[2 * s + 1]); }
  return q;   // (the pair count and indices are checked by the engine's schedule)
}
int gimmvfi_plan_clip(gimmvfi_engine* e, const gimmvfi_problem* p, const gimmvfi_clip* clip, size_t* workspace_bytes) {
  GV_TRY(e, { *workspace_bytes = e->eng.plan_clip(to_problem(p), to_clip(p, clip)); })
}
int gimmvfi_forward_clip(gimmvfi_engine* e, const gimmvfi_problem* p, const gimmvfi_clip* clip, const gimmvfi_io* io, void* workspace,
                         size_t workspace_bytes, void* cuda_stream) {
  GV_TRY(e, {
    if (!io) throw std::runtime_error("gimmvfi_forward_clip: io is required");
    e->eng.forward_clip(to_problem(p), to_clip(p, clip), to_io(io), workspace, workspace_bytes, (gvStream_t)cuda_stream);
  })
}

static Queries to_queries(const gimmvfi_problem* p, const gimmvfi_queries* q) {
  if (!p || !q || !q->pair_list || !q->t) throw std::runtime_error("gimmvfi queries: problem, queries, pair_list and t are required");
  if (q->queries < 1) throw std::runtime_error("gimmvfi queries: at least one query is required");
  if (q->frames < 1) throw std::runtime_error("gimmvfi queries: at least one frame is required");
  Queries r; r.F = q->frames;
  for (int i = 0; i < q->queries; ++i) { r.src.push_back(q->pair_list[2 * i]); r.tgt.push_back(q->pair_list[2 * i + 1]); r.t.push_back(q->t[i]); }
  return r;   // (indices and t are checked by the engine's schedule)
}
int gimmvfi_plan_queries(gimmvfi_engine* e, const gimmvfi_problem* p, const gimmvfi_queries* queries, size_t* workspace_bytes) {
  GV_TRY(e, { *workspace_bytes = e->eng.plan_queries(to_problem(p), to_queries(p, queries)); })
}
int gimmvfi_forward_queries(gimmvfi_engine* e, const gimmvfi_problem* p, const gimmvfi_queries* queries, const gimmvfi_io* io, void* workspace,
                            size_t workspace_bytes, void* cuda_stream) {
  GV_TRY(e, {
    if (!io) throw std::runtime_error("gimmvfi_forward_queries: io is required");
    e->eng.forward_queries(to_problem(p), to_queries(p, queries), to_io(io), workspace, workspace_bytes, (gvStream_t)cuda_stream);
  })
}
int gimmvfi_set_coord_range(gimmvfi_engine* e, double lo, double hi) {
  GV_TRY(e, {
    if (!std::isfinite(lo) || !std::isfinite(hi)) throw std::runtime_error("gimmvfi_set_coord_range: the range must be finite");
    e->eng.set_coord_range(lo, hi);
  })
}

int gimmvfi_finalize_weights_synthesis(gimmvfi_engine* e) { GV_TRY(e, { e->eng.finalize_weights_synthesis(); }) }
int gimmvfi_finalize_weights_f(gimmvfi_engine* e) { GV_TRY(e, { e->eng.finalize_weights_f(); }) }
int gimmvfi_set_flowformer_iters(gimmvfi_engine* e, int iters) { GV_TRY(e, { if (iters < 1) throw std::runtime_error("iters must be >= 1"); e->eng.ff_iters = iters; }) }
int gimmvfi_plan_from_flow(gimmvfi_engine* e, const gimmvfi_problem* p, size_t* workspace_bytes) {
  GV_TRY(e, { *workspace_bytes = e->eng.plan_from_flow(to_problem(p)); })
}
int gimmvfi_forward_from_flow(gimmvfi_engine* e, const gimmvfi_problem* p, const gimmvfi_io* io, const gimmvfi_flow_inputs* fin,
                              void* workspace, size_t workspace_bytes, void* cuda_stream) {
  GV_TRY(e, {
    if (!io || !fin) throw std::runtime_error("gimmvfi_forward_from_flow: io and fin are required");
    FlowInputs f; f.flows = fin->flows;
    for (int j = 0; j < 2; ++j) { f.feat4[j] = fin->feat4[j]; f.feat8[j] = fin->feat8[j]; f.fnet[j] = fin->fnet[j]; }
    e->eng.forward_from_flow(to_problem(p), to_io(io), f, workspace, workspace_bytes, (gvStream_t)cuda_stream);
  })
}
int gimmvfi_finalize_weights_gimm(gimmvfi_engine* e) { GV_TRY(e, { e->eng.finalize_weights_gimm(); }) }
int gimmvfi_gimm_plan(gimmvfi_engine* e, const gimmvfi_problem* p, size_t* workspace_bytes) {
  GV_TRY(e, { *workspace_bytes = e->eng.plan_gimm(to_problem(p)); })
}
int gimmvfi_gimm_forward(gimmvfi_engine* e, const gimmvfi_problem* p, const float* xs, const float* ori_flow, const float* coords, const float* t,
                         float* out, void* workspace, size_t workspace_bytes, void* cuda_stream) {
  GV_TRY(e, {
    GimmIO q; q.xs = xs; q.ori_flow = ori_flow; q.coords = coords; q.t = t; q.out = out;
    e->eng.forward_gimm(to_problem(p), q, workspace, workspace_bytes, (gvStream_t)cuda_stream);
  })
}

int gimmvfi_finalize_weights_lpips(gimmvfi_engine* e) { GV_TRY(e, { e->eng.finalize_weights_lpips(); }) }
int gimmvfi_lpips_plan(gimmvfi_engine* e, int n, int h, int w, size_t* workspace_bytes) {
  GV_TRY(e, { *workspace_bytes = e->eng.plan_lpips(n, h, w); })
}
int gimmvfi_lpips_forward(gimmvfi_engine* e, const float* in0, const float* in1, int n, int h, int w, int flags, float* out, float* per_layer,
                          void* workspace, size_t workspace_bytes, void* cuda_stream) {
  GV_TRY(e, {
    if (flags & ~(GIMMVFI_LPIPS_NORMALIZE | GIMMVFI_LPIPS_QUANTIZE)) throw std::runtime_error("lpips: unknown flags");
    LpipsIO q; q.in0 = in0; q.in1 = in1; q.out = out; q.per_layer = per_layer;
    q.normalize = (flags & GIMMVFI_LPIPS_NORMALIZE) != 0; q.quantize = (flags & GIMMVFI_LPIPS_QUANTIZE) != 0;
    e->eng.forward_lpips(n, h, w, q, workspace, workspace_bytes, (gvStream_t)cuda_stream);
  })
}

int gimmvfi_finalize_weights_flowformer(gimmvfi_engine* e) { GV_TRY(e, { e->eng.finalize_weights_flowformer(); }) }
int gimmvfi_flowformer_plan(gimmvfi_engine* e, int n_frames, int h, int w, int n_pairs, size_t* workspace_bytes) {
  GV_TRY(e, { *workspace_bytes = e->eng.plan_flowformer(n_frames, h, w, n_pairs); })
}
int gimmvfi_flowformer_forward(gimmvfi_engine* e, const float* frames, int n_frames, int h, int w, const int32_t* pairs, int n_pairs, int pairs_per_call,
                               int iters, float* flow_up, float* flow_low, void* workspace, size_t workspace_bytes, void* cuda_stream) {
  GV_TRY(e, {
    FlowFormerOutputs o; o.flow_up = flow_up; o.flow_low = flow_low;
    e->eng.forward_flowformer(frames, n_frames, h, w, pairs, n_pairs, pairs_per_call, iters, nullptr, o, workspace, workspace_bytes,
                              (gvStream_t)cuda_stream);
  })
}
int gimmvfi_flowformer_forward_ex(gimmvfi_engine* e, const float* frames, int n_frames, int h, int w, const int32_t* pairs, int n_pairs,
                                  int pairs_per_call, int iters, const float* flow_init, float* flow_up, float* flow_low, float* cfeat4,
                                  float* cfeat8, float* ffeat, void* workspace, size_t workspace_bytes, void* cuda_stream) {
  GV_TRY(e, {
    FlowFormerOutputs o; o.flow_up = flow_up; o.flow_low = flow_low; o.cfeat4 = cfeat4; o.cfeat8 = cfeat8; o.ffeat = ffeat;
    e->eng.forward_flowformer(frames, n_frames, h, w, pairs, n_pairs, pairs_per_call, iters, flow_init, o, workspace, workspace_bytes,
                              (gvStream_t)cuda_stream);
  })
}

int gimmvfi_finalize_weights_raft(gimmvfi_engine* e) { GV_TRY(e, { e->eng.finalize_weights_raft(); }) }
int gimmvfi_raft_plan(gimmvfi_engine* e, int n_frames, int h, int w, int n_pairs, int outputs, size_t* workspace_bytes) {
  GV_TRY(e, { *workspace_bytes = e->eng.plan_raft(n_frames, h, w, n_pairs, outputs); })
}
int gimmvfi_raft_forward(gimmvfi_engine* e, const float* frames, int n_frames, int h, int w, const int32_t* pairs, int n_pairs, int iters,
                         const float* flow_init, float* flow_up, float* flow_low, float* flow_iters, float* feat4, float* feat8, float* fmap,
                         void* workspace, size_t workspace_bytes, void* cuda_stream) {
  GV_TRY(e, {
    RaftOutputs o;
    o.flow_up = flow_up; o.flow_low = flow_low; o.flow_iters = flow_iters; o.feat4 = feat4; o.feat8 = feat8; o.fmap = fmap;
    e->eng.forward_raft(frames, n_frames, h, w, pairs, n_pairs, iters, flow_init, o, workspace, workspace_bytes, (gvStream_t)cuda_stream);
  })
}

const char* gimmvfi_last_error(gimmvfi_engine* e) { return e ? e->err.c_str() : g_static_err.c_str(); }
int64_t gimmvfi_last_launches(gimmvfi_engine* e) { return e->eng.last_launches(); }
int64_t gimmvfi_weights_version(gimmvfi_engine* e) { return e->eng.weights_version(); }
int gimmvfi_set_raft_iters(gimmvfi_engine* e, int iters) { GV_TRY(e, { if (iters < 1) throw std::runtime_error("iters must be >= 1"); e->eng.raft_iters = iters; }) }
int gimmvfi_set_debug(gimmvfi_engine* e, int on) { GV_TRY(e, { e->eng.set_debug(on != 0); }) }
int gimmvfi_get_tap(gimmvfi_engine* e, const char* name, gimmvfi_view* out) {
  GV_TRY(e, {
    auto it = e->eng.taps().find(name);
    if (it == e->eng.taps().end()) throw std::runtime_error(std::string("no tap named '") + name + "'");
    const TV& t = it->second;
    out->data = t.p; out->n = t.n; out->h = t.h; out->w = t.w; out->c = t.c; out->pixel_stride = t.ld; out->batch_stride = t.sn;
  })
}
size_t gimmvfi_frame_cache_bytes(const gimmvfi_problem* p) { return Engine::frame_cache_bytes(to_problem(p)); }
int gimmvfi_set_frame_cache(gimmvfi_engine* e, void* cache, size_t bytes, int load, int store) {
  GV_TRY(e, { e->eng.set_frame_cache(static_cast<float*>(cache), bytes, load != 0, store != 0); })
}
int gimmvfi_set_tensor_cores(gimmvfi_engine* e, int mode) { GV_TRY(e, { e->eng.set_tensor_cores(mode); }) }
int gimmvfi_set_motion_config(gimmvfi_engine* e, int fwarp_mode, int activation, float w0, float output_bias, int normalize_weight) {
  GV_TRY(e, {
    if (fwarp_mode < GIMMVFI_FWARP_LINEAR || fwarp_mode > GIMMVFI_FWARP_SUM) throw std::runtime_error("set_motion_config: unknown fwarp_mode");
    if (activation < GIMMVFI_ACT_SIREN || activation > GIMMVFI_ACT_DAMP) throw std::runtime_error("set_motion_config: unknown activation");
    if (!std::isfinite(w0) || !std::isfinite(output_bias)) throw std::runtime_error("set_motion_config: w0 and output_bias must be finite");
    MotionConfig m;
    m.fwarp = fwarp_mode == GIMMVFI_FWARP_SOFTMAX ? SPLAT_SOFTMAX : fwarp_mode == GIMMVFI_FWARP_SUM ? SPLAT_SUM : SPLAT_LINEAR;
    const bool siren1 = activation == GIMMVFI_ACT_SIREN && w0 == 1.f;   // the shipped form keeps its own kernels
    m.act = siren1 ? HYPO_SIREN1 : activation == GIMMVFI_ACT_SIREN ? HYPO_SIREN : activation == GIMMVFI_ACT_RELU ? HYPO_RELU
                                 : activation == GIMMVFI_ACT_SILU ? HYPO_SILU : HYPO_DAMP;
    m.w0 = w0; m.output_bias = output_bias; m.normalize_weight = normalize_weight != 0;
    e->eng.set_motion_config(m);
  })
}
int gimmvfi_set_cuda_graph(gimmvfi_engine* e, int on) { GV_TRY(e, { e->eng.set_cuda_graph(on != 0); }) }
int64_t gimmvfi_graph_replays(gimmvfi_engine* e) { return e->eng.graph_replays(); }
int gimmvfi_set_profile(gimmvfi_engine* e, int on) { GV_TRY(e, { e->eng.set_profile(on != 0); }) }
const char* gimmvfi_profile_json(gimmvfi_engine* e, void* stream) {
  try { e->prof_json = e->eng.profile_json((gvStream_t)stream); } catch (const std::exception& ex) { e->err = ex.what(); e->prof_json = "{}"; }
  return e->prof_json.c_str();
}
const char* gimmvfi_build_info(void) {
#ifdef GV_HOSTSIM
  return "gimmvfi_b200 HOSTSIM (test-only CPU emulation of the kernels; not a product build)";
#else
  return "gimmvfi_b200 sm_90a CUDA build";
#endif
}

// ------------------------------------------------------------ per-kernel entry points
int gimmvfi_op_softsplat(const gimmvfi_view* lat, const gimmvfi_view* flow, const gimmvfi_view* metric, const float* t, int t_mode,
                         const gimmvfi_view* scratch, const gimmvfi_view* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    Ctx cx = op_ctx(stream);
    TV acc = to_tv(scratch); acc.c = 17;
    if (acc.ld < 17 || to_tv(lat).c != 16) throw std::runtime_error("softsplat: lat must have 16 channels and scratch pixel_stride >= 17");
    for (int n = 0; n < acc.n; ++n) dev_memset(acc.p + (int64_t)n * acc.sn, 0, (size_t)acc.h * acc.w * acc.ld * sizeof(float), cx.stream);
    softsplat_accumulate(cx, to_tv(lat), to_tv(flow), to_tv(metric), t, t_mode, acc);
    softsplat_normalize(cx, acc, to_tv(out));
  })
}
int gimmvfi_op_softsplat_fused(const gimmvfi_view* lat, const gimmvfi_view* flow, const gimmvfi_view* metric, const float* t, int t_mode,
                               const float* flow_absmax, const gimmvfi_view* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    Ctx cx = op_ctx(stream);
    if (!softsplat_fused(cx, to_tv(lat), to_tv(flow), to_tv(metric), t, t_mode, flow_absmax, to_tv(out)))
      throw std::runtime_error("softsplat_fused: 16-channel 16-byte-aligned latent / output, 8-byte-aligned flow and a flow bound are required");
  })
}
int gimmvfi_op_softsplat_out(const gimmvfi_tensor4* in, const gimmvfi_tensor4* flow, const gimmvfi_tensor4* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    if (!out) throw std::runtime_error("softsplat_out: out is required");
    splat_check(in, flow, out, nullptr, nullptr, "softsplat_out");
    if (!dense4(*out)) throw std::runtime_error("softsplat_out: out must be dense (it is zero-filled by the call)");
    Ctx cx = op_ctx(stream);
    const int64_t numel = out->sizes[0] * out->sizes[1] * out->sizes[2] * out->sizes[3];
    if (numel == 0) return 0;
    const bool f32 = out->dtype == GIMMVFI_FLOAT32;
    dev_memset(out->data, 0, (size_t)numel * (f32 ? sizeof(float) : sizeof(double)), cx.stream);
    if (f32) softsplat_out_any<float>(cx, sv4<float>(in), sv4<float>(flow), sv4<float>(out));
    else softsplat_out_any<double>(cx, sv4<double>(in), sv4<double>(flow), sv4<double>(out));
  })
}
int gimmvfi_op_softsplat_grad(const gimmvfi_tensor4* in, const gimmvfi_tensor4* flow, const gimmvfi_tensor4* outgrad, const gimmvfi_tensor4* ingrad,
                              const gimmvfi_tensor4* flowgrad, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    if (!outgrad) throw std::runtime_error("softsplat_grad: outgrad is required");
    if (!ingrad && !flowgrad) throw std::runtime_error("softsplat_grad: at least one of ingrad / flowgrad is required");
    splat_check(in, flow, outgrad, ingrad, flowgrad, "softsplat_grad");
    Ctx cx = op_ctx(stream);
    if (outgrad->dtype == GIMMVFI_FLOAT32)
      softsplat_grad_any<float>(cx, sv4<float>(in), sv4<float>(flow), sv4<float>(outgrad), sv4<float>(ingrad), sv4<float>(flowgrad));
    else
      softsplat_grad_any<double>(cx, sv4<double>(in), sv4<double>(flow), sv4<double>(outgrad), sv4<double>(ingrad), sv4<double>(flowgrad));
  })
}
int gimmvfi_op_alt_corr_forward(const gimmvfi_dense* fmap1, const gimmvfi_dense* fmap2, const gimmvfi_dense* coords, int radius,
                                const gimmvfi_dense* corr, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    const std::string w = "alt_corr_forward";
    const AltCorrArgs a = alt_corr_args(fmap1, fmap2, coords, radius, w);
    dense_expect(corr, alt_corr_shape(a), w, "corr");
    Ctx cx = op_ctx(stream);
    alt_corr_forward(cx, a, static_cast<float*>(corr->data));
  })
}
int gimmvfi_op_alt_corr_backward(const gimmvfi_dense* fmap1, const gimmvfi_dense* fmap2, const gimmvfi_dense* coords,
                                 const gimmvfi_dense* corr_grad, int radius, const gimmvfi_dense* fmap1_grad, const gimmvfi_dense* fmap2_grad,
                                 const gimmvfi_dense* coords_grad, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    const std::string w = "alt_corr_backward";
    if (!fmap1_grad && !fmap2_grad && !coords_grad) throw std::runtime_error(w + ": at least one of fmap1_grad / fmap2_grad / coords_grad is required");
    const AltCorrArgs a = alt_corr_args(fmap1, fmap2, coords, radius, w);
    dense_expect(corr_grad, alt_corr_shape(a), w, "corr_grad");
    if (fmap1_grad) dense_expect(fmap1_grad, {a.B, a.H1, a.W1, a.C}, w, "fmap1_grad");
    if (fmap2_grad) dense_expect(fmap2_grad, {a.B, a.H2, a.W2, a.C}, w, "fmap2_grad");
    if (coords_grad) dense_expect(coords_grad, {a.B, a.N, a.H1, a.W1, 2}, w, "coords_grad");
    Ctx cx = op_ctx(stream);
    if (fmap2_grad && dense_numel(*fmap2_grad) > 0) dev_memset(fmap2_grad->data, 0, (size_t)dense_numel(*fmap2_grad) * sizeof(float), cx.stream);
    alt_corr_backward(cx, a, static_cast<const float*>(corr_grad->data), fmap1_grad ? static_cast<float*>(fmap1_grad->data) : nullptr,
                      fmap2_grad ? static_cast<float*>(fmap2_grad->data) : nullptr, coords_grad ? static_cast<float*>(coords_grad->data) : nullptr);
  })
}
int gimmvfi_op_backwarp(const gimmvfi_view* src, const gimmvfi_view* flow, const gimmvfi_view* dst, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, { Ctx cx = op_ctx(stream); backwarp(cx, to_tv(src), to_tv(flow), to_tv(dst)); })
}
int gimmvfi_op_resize(const gimmvfi_view* src, const gimmvfi_view* dst, float scale_factor, float mult, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    Ctx cx = op_ctx(stream);
    float r = (float)(1.0 / (double)scale_factor);
    resize_bilinear(cx, to_tv(src), to_tv(dst), r, r, mult, 0, ACT_NONE);
  })
}
int gimmvfi_op_tail_pointwise(int op, const gimmvfi_view* src, const gimmvfi_view* flow, const gimmvfi_view* dst, float scale_factor, float mult,
                              int accumulate, int act, int half_mask, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    Ctx cx = op_ctx(stream);
    TV s = to_tv(src); TV d = to_tv(dst);
    s.f16 = half_mask & 1; d.f16 = (half_mask >> 1) & 1;
    const float r = (float)(1.0 / (double)scale_factor);
    if (op == GIMMVFI_TAIL_RESIZE) resize_bilinear(cx, s, d, r, r, mult, accumulate, act);
    else if (op == GIMMVFI_TAIL_BACKWARP) backwarp(cx, s, to_tv(flow), d);
    else if (op == GIMMVFI_TAIL_COPY) copy_channels(cx, s, d);
    else throw std::runtime_error("tail_pointwise: unknown op");
  })
}
// ---- FlowFormer / Twins token-side kernels (ops_tokens.cu), NHWC views
int gimmvfi_op_layernorm(const gimmvfi_view* x, const float* gamma, const float* beta, float eps, const gimmvfi_view* out, float pe_scale, int pe_dim,
                         void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, { Ctx cx = op_ctx(stream); layernorm(cx, to_tv(x), gamma, beta, eps, to_tv(out), pe_scale, pe_dim); })
}
int gimmvfi_op_window_attention(const gimmvfi_view* q, const gimmvfi_view* k, const gimmvfi_view* v, const gimmvfi_view* out, int heads, int ws,
                                void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, { Ctx cx = op_ctx(stream); window_attention(cx, to_tv(q), to_tv(k), to_tv(v), to_tv(out), heads, ws); })
}
int gimmvfi_op_global_attention(const gimmvfi_view* q, const gimmvfi_view* k, const gimmvfi_view* v, const gimmvfi_view* out, int heads, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    Ctx cx = op_ctx(stream);
    const TV Q = to_tv(q); const TV K = to_tv(k); const TV V = to_tv(v); const TV O = to_tv(out);
    if (Q.c != O.c || K.c != Q.c || V.c != Q.c || Q.c % heads || Q.n != K.n || K.h != V.h || K.w != V.w) throw std::runtime_error("global_attention: shape mismatch");
    AttnDims a{};
    a.nb1 = Q.n; a.nb2 = 1; a.nq = (int64_t)Q.h * Q.w; a.nk = (int64_t)K.h * K.w; a.heads = heads;
    a.q_s1 = Q.sn; a.q_si = Q.ld; a.k_s1 = K.sn; a.k_sj = K.ld; a.v_s1 = V.sn; a.v_sj = V.ld; a.o_s1 = O.sn; a.o_si = O.ld;
    strided_attention(cx, Q.p, K.p, V.p, O.p, a, Q.c / heads);
  })
}
int gimmvfi_op_patchify(const gimmvfi_view* src, const gimmvfi_view* dst, int k, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, { Ctx cx = op_ctx(stream); patchify(cx, to_tv(src), to_tv(dst), k); })
}
int gimmvfi_op_cost_conv1(const float* vol, int64_t maps, int h, int w, const float* w_host, const float* b_host, const gimmvfi_view* out_padded,
                          void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    Ctx cx = op_ctx(stream);
    const TV o = to_tv(out_padded);
    cost_conv1(cx, vol, maps, h, w, w_host, b_host, o, o.h - 4, o.w - 4);
  })
}
int gimmvfi_op_conv7x7_small_cout(const gimmvfi_view* in, const float* w_tap_cin_4, const float* bias, int cout, const gimmvfi_view* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    Ctx cx = op_ctx(stream);
    ConvW w; w.w = w_tap_cin_4; w.b = bias; w.cin = to_tv(in).c; w.cout = cout; w.kh = w.kw = 7; w.cout_ld = 4;
    if (!conv7x7_small_cout(cx, to_tv(in), w, ACT_NONE, nullptr, to_tv(out))) throw std::runtime_error("conv7x7_small_cout: layer / tensors not of that class (or host simulation)");
  })
}
int gimmvfi_op_row_softmax(float* p, int64_t rows, int64_t cols, float mul, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    if (rows < 1 || cols < 1) throw std::runtime_error("row_softmax: rows >= 1 and cols >= 1 required");
    Ctx cx = op_ctx(stream);
    row_softmax(cx, p, rows, cols, mul);
  })
}
int gimmvfi_op_corr_volume(const gimmvfi_view* fa, const gimmvfi_view* fb, float* vol, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, { Ctx cx = op_ctx(stream); TV a = to_tv(fa); corr_volume(cx, a, to_tv(fb), vol, 1.0f / std::sqrt((float)a.c)); })
}
int gimmvfi_op_corr_volume_tc(const gimmvfi_view* fa, const gimmvfi_view* fb, float* scratch, float* vol, int split, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
#ifdef GV_HOSTSIM
    throw std::runtime_error("corr_volume_tc is a tensor-core kernel; not available in the host simulation");
#else
    Ctx cx = op_ctx(stream);
    TV a = to_tv(fa); TV b = to_tv(fb);
    if (a.n != 1 || b.n != 1 || a.c % 32 || a.ld != a.c || b.ld != b.c) throw std::runtime_error("corr_volume_tc: one dense sample with C % 32 == 0");
    const int64_t N = (int64_t)a.h * a.w;
    if ((int64_t)b.h * b.w != N) throw std::runtime_error("corr_volume_tc: fa and fb must have the same number of pixels");
    if (split && corr_volume_tc_wants_f16_planes() && a.c % 64 == 0) {   // half planes of fa, then of fb: 2 N C floats of scratch
      uint16_t* ap = reinterpret_cast<uint16_t*>(scratch); uint16_t* bp = ap + 2 * N * a.c;
      split_planes_f16(cx, a, ap); split_planes_f16(cx, b, bp);
      corr_gemm_3xf16(cx, ap, N * a.c, (int)N, bp, N * a.c, (int)N, a.c, 1.0f / std::sqrt((float)a.c), vol);
      return 0;
    }
    float* planes = scratch; float* zeros = scratch + 2 * N * a.c;
    dev_memset(zeros, 0, (size_t)(((N + 255) / 256) * 256 + 512) * sizeof(float), cx.stream);
    if (split && corr_volume_tc_wants_f16_planes()) split_planes_f16(cx, b, planes);
    else if (split) split_planes(cx, b, planes);
    corr_volume_tc(cx, a, split ? planes : b.p, zeros, vol, 1.0f / std::sqrt((float)a.c), split != 0);
#endif
  })
}
int gimmvfi_op_corr_pool(const float* src, float* dst, int64_t rows, int h, int w, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, { Ctx cx = op_ctx(stream); corr_pool(cx, src, dst, rows, h, w); })
}
int gimmvfi_op_corr_pool_pyramid(const float* l0, float* l1, float* l2, float* l3, int64_t rows, int h, int w, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, { Ctx cx = op_ctx(stream); corr_pool_pyramid(cx, l0, l1, l2, l3, rows, h, w); })
}
int gimmvfi_op_corr_lookup(const float* const lvl[4], const int32_t lvl_h[4], const int32_t lvl_w[4], const gimmvfi_view* coords,
                           const gimmvfi_view* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    Ctx cx = op_ctx(stream);
    TV c = to_tv(coords);
    CorrPyr p;
    for (int l = 0; l < 4; ++l) { p.lvl[l] = lvl[l]; p.h[l] = lvl_h[l]; p.w[l] = lvl_w[l]; }
    p.rows_per_sample = (int64_t)c.h * c.w;
    corr_lookup(cx, p, c, to_tv(out));
  })
}
int gimmvfi_op_corr_lookup_direct(const gimmvfi_view* src, const void* const tgt_half[4], const int32_t lvl_h[4], const int32_t lvl_w[4], float scale,
                                  const gimmvfi_view* coords, const gimmvfi_view* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    Ctx cx = op_ctx(stream);
    TV s = to_tv(src);
    CorrFeat f;
    for (int l = 0; l < 4; ++l) { f.lvl[l] = static_cast<const uint16_t*>(tgt_half[l]); f.h[l] = lvl_h[l]; f.w[l] = lvl_w[l]; }
    f.c = s.c; f.scale = scale;
    corr_lookup_direct(cx, s, f, to_tv(coords), to_tv(out));
  })
}
int gimmvfi_op_conv2d(const gimmvfi_view* in0, const gimmvfi_view* in1, const float* w_packed, const float* bias, int cin, int cout,
                      int cout_ld, int kh, int kw, int stride, int pad_h, int pad_w, int reflect, int act, const float* slope,
                      const gimmvfi_view* residual, const gimmvfi_view* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    Ctx cx = op_ctx(stream);
    ConvW w; w.w = w_packed; w.b = bias; w.cin = cin; w.cout = cout; w.cout_ld = cout_ld; w.kh = kh; w.kw = kw;
    ConvGeom g; g.stride = stride; g.ph = pad_h; g.pw = pad_w; g.reflect = reflect;
    ConvEpi ep; ep.act1 = act; ep.slope1 = slope; ep.res = to_tv(residual);
    conv2d(cx, to_tv(in0), to_tv(in1), w, g, ep, to_tv(out));
  })
}
int gimmvfi_op_conv2d_tc(const gimmvfi_view* in0, const gimmvfi_view* in1, const float* w_tc, const float* bias, int cin, int cout, int kh,
                         int kw, int act1, const float* slope1, const gimmvfi_view* residual, int act2, const float* slope2,
                         const gimmvfi_view* mul, const gimmvfi_view* gru_z, const gimmvfi_view* gru_h, int split,
                         const gimmvfi_view* out, const void* w_tc_s, float w_scale, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
#ifdef GV_HOSTSIM
    throw std::runtime_error("conv2d_tc is a tensor-core kernel; not available in the host simulation");
#else
    Ctx cx = op_ctx(stream);
    ConvW w; w.b = bias; w.cin = cin; w.cout = cout; w.kh = kh; w.kw = kw; w.w_tc = w_tc; w.has_lo = true;
    w.cout_pad = tc_cout_pad(cout); w.cin_pad = (cin + 31) & ~31;
    if (w_tc_s) { w.w_tc_s = w_tc_s; w.cin_pad_s = (cin + 63) & ~63; w.w_scale = w_scale; }   // 3xF16 form of the split kernel
    ConvGeom g; g.stride = 1; g.ph = kh / 2; g.pw = kw / 2;
    ConvEpi ep; ep.act1 = act1; ep.slope1 = slope1; ep.res = to_tv(residual); ep.act2 = act2; ep.slope2 = slope2;
    ep.mul = to_tv(mul); ep.gru_z = to_tv(gru_z); ep.gru_h = to_tv(gru_h);
    if (!conv2d_tc_supported(to_tv(in0), to_tv(in1), w, g, ep, to_tv(out), split != 0)) throw std::runtime_error("conv2d_tc: unsupported configuration");
    conv2d_tc(cx, to_tv(in0), to_tv(in1), w, g, ep, to_tv(out), split != 0);
#endif
  })
}
int gimmvfi_op_conv2d_tc_strided(const gimmvfi_view* in0, const float* w_tc, const float* bias, int cin, int cout, int kh, int kw, int stride,
                                 int act1, int split, const gimmvfi_view* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
#ifdef GV_HOSTSIM
    throw std::runtime_error("conv2d_tc is a tensor-core kernel; not available in the host simulation");
#else
    Ctx cx = op_ctx(stream);
    ConvW w; w.b = bias; w.cin = cin; w.cout = cout; w.kh = kh; w.kw = kw; w.w_tc = w_tc; w.has_lo = true;
    w.cout_pad = tc_cout_pad(cout); w.cin_pad = (cin + 31) & ~31;
    ConvGeom g; g.stride = stride; g.ph = kh / 2; g.pw = kw / 2;
    ConvEpi ep; ep.act1 = act1;
    if (!conv2d_tc_supported(to_tv(in0), TV(), w, g, ep, to_tv(out), split != 0)) throw std::runtime_error("conv2d_tc_strided: unsupported configuration");
    conv2d_tc(cx, to_tv(in0), TV(), w, g, ep, to_tv(out), split != 0);
#endif
  })
}
int gimmvfi_op_conv2d_tc_f16(const gimmvfi_view* in0, const gimmvfi_view* in1, const void* w_tc_h, const float* w_tc, const float* bias, int cin,
                             int cout, int kh, int kw, int act1, const float* slope1, const gimmvfi_view* residual, int act2,
                             const float* slope2, int half_mask, const gimmvfi_view* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
#ifdef GV_HOSTSIM
    throw std::runtime_error("conv2d_tc is a tensor-core kernel; not available in the host simulation");
#else
    Ctx cx = op_ctx(stream);
    ConvW w; w.b = bias; w.cin = cin; w.cout = cout; w.kh = kh; w.kw = kw; w.w_tc = w_tc; w.has_lo = true;
    w.cout_pad = tc_cout_pad(cout); w.cin_pad = (cin + 31) & ~31; w.w_tc_h = w_tc_h; w.cin_pad_h = (cin + 63) & ~63;
    ConvGeom g; g.stride = 1; g.ph = kh / 2; g.pw = kw / 2;
    TV a0 = to_tv(in0); TV a1 = to_tv(in1); TV r = to_tv(residual); TV o = to_tv(out);
    a0.f16 = half_mask & 1; if (a1.p) a1.f16 = half_mask & 1; o.f16 = (half_mask >> 1) & 1; if (r.p) r.f16 = (half_mask >> 2) & 1;
    ConvEpi ep; ep.act1 = act1; ep.slope1 = slope1; ep.res = r; ep.act2 = act2; ep.slope2 = slope2;
    if (!conv2d_tc_supported(a0, a1, w, g, ep, o, false)) throw std::runtime_error("conv2d_tc_f16: unsupported configuration");
    conv2d_tc(cx, a0, a1, w, g, ep, o, false);
#endif
  })
}
int gimmvfi_op_conv2d_wide(const gimmvfi_view* in0, const gimmvfi_view* in1, const void* w_tc_h, const float* bias, int cin, int cout,
                           int act1, const float* slope1, const gimmvfi_view* residual, int act2, const float* slope2, int half_mask,
                           const gimmvfi_view* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
#ifdef GV_HOSTSIM
    throw std::runtime_error("conv2d_wide is a tensor-core kernel; not available in the host simulation");
#else
    Ctx cx = op_ctx(stream);
    ConvW w; w.b = bias; w.cin = cin; w.cout = cout; w.kh = 3; w.kw = 3;
    w.cout_pad = tc_cout_pad(cout); w.w_tc_h = w_tc_h; w.cin_pad_h = (cin + 63) & ~63;
    ConvGeom g; g.stride = 1; g.ph = 1; g.pw = 1;
    TV a0 = to_tv(in0); TV a1 = to_tv(in1); TV r = to_tv(residual); TV o = to_tv(out);
    a0.f16 = half_mask & 1; if (a1.p) a1.f16 = half_mask & 1; o.f16 = (half_mask >> 1) & 1; if (r.p) r.f16 = (half_mask >> 2) & 1;
    ConvEpi ep; ep.act1 = act1; ep.slope1 = slope1; ep.res = r; ep.act2 = act2; ep.slope2 = slope2;
    if (a0.c + (a1.p ? a1.c : 0) != cin || o.c != cout) throw std::runtime_error("conv2d_wide: channel counts do not match the views");
    if (!conv2d_wide_supported(a0, a1, w, g, ep, o)) throw std::runtime_error("conv2d_wide: unsupported configuration");
    conv2d_wide(cx, a0, a1, w, g, ep, o);
#endif
  })
}
int gimmvfi_op_conv2d_halo(const gimmvfi_view* in0, const void* w_tc_h, const float* w_tc, const float* bias, int cin, int cout, int act1,
                           const float* slope1, const gimmvfi_view* residual, int act2, const float* slope2, int half_mask, int prepadded,
                           const gimmvfi_view* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
#ifdef GV_HOSTSIM
    throw std::runtime_error("conv2d_halo is a tensor-core kernel; not available in the host simulation");
#else
    Ctx cx = op_ctx(stream);
    const int k = prepadded == 2 ? 1 : 3;   // prepadded: 0 = 3x3 zero padding 1, 1 = 3x3 on a pre-padded input, 2 = 1x1
    ConvW w; w.b = bias; w.cin = cin; w.cout = cout; w.kh = k; w.kw = k; w.w_tc = w_tc; w.has_lo = true;
    w.cout_pad = tc_cout_pad(cout); w.cin_pad = (cin + 31) & ~31; w.w_tc_h = w_tc_h; w.cin_pad_h = (cin + 63) & ~63;
    ConvGeom g; g.stride = 1; g.ph = prepadded == 1 ? 0 : k / 2; g.pw = g.ph; g.loose_w = prepadded == 1 ? 1 : 0;
    TV a0 = to_tv(in0); TV r = to_tv(residual); TV o = to_tv(out);
    a0.f16 = half_mask & 1; o.f16 = (half_mask >> 1) & 1; if (r.p) r.f16 = (half_mask >> 2) & 1;
    ConvEpi ep; ep.act1 = act1; ep.slope1 = slope1; ep.res = r; ep.act2 = act2; ep.slope2 = slope2;
    if (!conv2d_halo_supported(a0, TV(), w, g, ep, o)) throw std::runtime_error("conv2d_halo: unsupported configuration");
    conv2d_halo(cx, a0, w, g, ep, o);
#endif
  })
}
int gimmvfi_op_hyponet(gimmvfi_engine* e, const gimmvfi_view* latent, const float* coords, const gimmvfi_view* out, int fp32_class, void* stream) {
  GV_TRY(e, {
    e->eng.need(Engine::Entry::Gimm);
    Ctx cx = op_ctx(stream);
    const MotionConfig& m = e->eng.motion();   // the activation the weights were packed for
    if (out->h != latent->h || out->w != latent->w) {   // another grid size: the latent is resized to it inside the fp32-class kernel
      if (!fp32_class) throw std::runtime_error("hyponet: an output grid of another size than the latent needs fp32_class = 1");
      hyponet_fused3_resample_act(cx, to_tv(latent), coords, e->eng.hyponet_blob(true), to_tv(out), m.act, m.w0);
      return 0;
    }
    if (!hyponet_fused_supported(to_tv(latent), to_tv(out))) throw std::runtime_error("hyponet: latent (n,h,w,32) dense fp32, out (n,h,w,2)");
    if (fp32_class) hyponet_fused3_act(cx, to_tv(latent), coords, e->eng.hyponet_blob(true), to_tv(out), m.act, m.w0);
    else hyponet_fused_act(cx, to_tv(latent), coords, e->eng.hyponet_blob(false), to_tv(out), m.act, m.w0);
  })
}
int64_t gimmvfi_instnorm_scratch_floats(int n, int c) {
  TV t; t.n = n; t.c = c;
  return instnorm_scratch_floats(t) + (int64_t)n * c * 2;
}
int gimmvfi_op_instnorm(const gimmvfi_view* x, int relu, float* scratch, const gimmvfi_view* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    Ctx cx = op_ctx(stream);
    TV t = to_tv(x);
    float* mr = scratch + instnorm_scratch_floats(t);
    instnorm_stats(cx, t, mr, scratch, 0);
    instnorm_apply(cx, t, mr, relu ? ACT_RELU : ACT_NONE, TV(), ACT_NONE, to_tv(out));
  })
}
int gimmvfi_op_convex_upsample(const gimmvfi_view* flow, const gimmvfi_view* mask, const gimmvfi_view* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, { Ctx cx = op_ctx(stream); convex_upsample(cx, to_tv(flow), to_tv(mask), to_tv(out)); })
}
int gimmvfi_op_frames_u8_to_padded_f32(const uint8_t* frames, int n, int h, int w, float* dst_nchw, int H, int W, int pad_top, int pad_left,
                                       void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    if (H < h || W < w || pad_top < 0 || pad_left < 0 || pad_top + h > H || pad_left + w > W) throw std::runtime_error("bad padding geometry");
    Ctx cx = op_ctx(stream); frames_u8_to_padded_f32(cx, frames, n, h, w, dst_nchw, H, W, pad_top, pad_left);
  })
}
int gimmvfi_op_pred_to_u8(const float* pred_nchw, int n, int H, int W, uint8_t* dst, int h, int w, int pad_top, int pad_left, int bgr,
                          void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    if (H < h || W < w || pad_top < 0 || pad_left < 0 || pad_top + h > H || pad_left + w > W) throw std::runtime_error("bad padding geometry");
    Ctx cx = op_ctx(stream); pred_to_u8(cx, pred_nchw, n, H, W, dst, h, w, pad_top, pad_left, bgr);
  })
}
int64_t gimmvfi_flow_to_image_scratch_floats(int n, int h) { return flow_to_image_scratch_floats(n, h); }
int gimmvfi_op_flow_to_image(const float* flow, int64_t stride_n, int64_t stride_y, int64_t stride_x, int64_t stride_c, int n, int h, int w,
                             double clip_flow, double max_flow, int bgr, float* scratch, uint8_t* dst, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    if (n < 0 || h < 0 || w < 0) throw std::runtime_error("flow_to_image: negative size");
    if (!flow || !dst) throw std::runtime_error("flow_to_image: flow and dst are required");
    const int has_max = !std::isnan(max_flow);
    if (!has_max && !scratch) throw std::runtime_error("flow_to_image: scratch is required without max_flow");
    FlowView f; f.p = flow; f.sn = stride_n; f.sy = stride_y; f.sx = stride_x; f.sc = stride_c; f.n = n; f.h = h; f.w = w;
    Ctx cx = op_ctx(stream);
    // np.clip casts clip_flow to float32; max_flow + 1e-5 is a Python double, rounded once to float32 by the division
    flow_to_image(cx, f, !std::isnan(clip_flow), (float)clip_flow, has_max, (float)(max_flow + 1e-5), bgr, scratch, dst);
  })
}
int gimmvfi_op_forward_interpolate(const float* flow, int n, int h, int w, float* out, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    if (n < 1 || h < 1 || w < 1) throw std::runtime_error("forward_interpolate: n, h and w must be >= 1");
    if (n > 65535) throw std::runtime_error("forward_interpolate: at most 65535 flows per call");
    if ((int64_t)h * w >= ((int64_t)1 << 31)) throw std::runtime_error("forward_interpolate: h * w must be below 2^31");
    if (!flow || !out) throw std::runtime_error("forward_interpolate: flow and out are required");
    const int64_t bytes = (int64_t)n * 2 * h * w * (int64_t)sizeof(float);
    const char* a = reinterpret_cast<const char*>(flow); const char* b = reinterpret_cast<const char*>(out);
    if (a < b + bytes && b < a + bytes) throw std::runtime_error("forward_interpolate: out must not overlap flow");
    Ctx cx = op_ctx(stream);
    forward_interpolate(cx, flow, n, h, w, out);
  })
}
int gimmvfi_op_scene_sums(const uint8_t* a, const uint8_t* b, int n, int h, int w, uint64_t* sums, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    if (n < 0 || h < 1 || w < 1) throw std::runtime_error("scene_sums: n must be >= 0, h and w >= 1");
    if ((int64_t)h * w >= ((int64_t)1 << 31)) throw std::runtime_error("scene_sums: h * w must be below 2^31");
    if (n > 0 && (!a || !b || !sums)) throw std::runtime_error("scene_sums: a, b and sums are required");
    Ctx cx = op_ctx(stream);
    scene_sums(cx, a, b, n, h, w, sums);
  })
}
int gimmvfi_op_blend_u8(const void* const* src, const int* is_f32, int n, int H, int W, int pad_top, int pad_left, uint8_t* dst, int h, int w,
                        int bgr, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, {
    if (n < 1 || n > kBlendMax) throw std::runtime_error("blend_u8: n must be in [1, 63]");
    if (!src || !is_f32 || !dst) throw std::runtime_error("blend_u8: src, is_f32 and dst are required");
    for (int i = 0; i < n; ++i) if (!src[i]) throw std::runtime_error("blend_u8: a source pointer is null");
    if (h < 1 || w < 1 || pad_top < 0 || pad_left < 0 || pad_top + h > H || pad_left + w > W)
      throw std::runtime_error("blend_u8: the crop (pad_top, pad_left, h, w) must lie inside the H x W rows");
    if ((int64_t)H * W >= ((int64_t)1 << 31)) throw std::runtime_error("blend_u8: H * W must be below 2^31");
    Ctx cx = op_ctx(stream);
    blend_u8(cx, src, is_f32, n, H, W, pad_top, pad_left, dst, h, w, bgr);
  })
}
int gimmvfi_op_pixel_shuffle(const gimmvfi_view* src, const gimmvfi_view* dst, int times, void* stream) {
  gimmvfi_engine* e = nullptr;
  GV_TRY(e, { Ctx cx = op_ctx(stream); pixel_shuffle(cx, to_tv(src), to_tv(dst), times); })
}

}  // extern "C"
