// Engine: weights, workspace planning and the stream-ordered forward pass of
// GIMM-VFI-R (reference hot path: gimmvfi_r.py:324-407).  See DESIGN.md.
#pragma once
#include <functional>

#include "common.h"

namespace gv {

struct HostTensor {
  std::vector<int64_t> shape;
  std::vector<float> data;
};

struct Problem {
  int B = 1;        // pairs in this call
  int Hf = 0, Wf = 0;  // full (caller-padded) resolution
  int T = 1;        // timesteps
  float ds = 0.f;   // ds_factor (0 -> None)
  int Hc = 0, Wc = 0;  // HypoNet coordinate grid (== network resolution at inference)
  int H() const { return ds > 0.f ? (int)std::floor((double)Hf * (double)ds) : Hf; }
  int W() const { return ds > 0.f ? (int)std::floor((double)Wf * (double)ds) : Wf; }
};

// Device pointers, caller-owned.  Layouts are the reference's (NCHW-style), one
// contiguous block per output with the timestep as the outermost dimension.
struct IO {
  const float* img_xs = nullptr;   // (B,3,2,Hf,Wf) in [0,1]
  const float* coords = nullptr;   // (T,B,1,Hc,Wc,3)  last dim (t,y,x)
  const float* t = nullptr;        // (T,B)
  float* imgt_pred = nullptr;      // (T,B,3,Hf,Wf)
  float* img_warp_4 = nullptr;     // (T,B,3,H,W)
  float* flowt0_1 = nullptr;       // (T,B,3,2,Hf,Wf)
  float* flowt1_1 = nullptr;
  float* flowt0_4 = nullptr;       // (T,B,2,H/4,W/4)
  float* flowt1_4 = nullptr;
  float* raft_flow = nullptr;      // (B,2,2,H,W)
  float* nflow = nullptr;          // (B,2,2,H,W)
  float* ninrflow = nullptr;       // (T,B,2,1,Hc,Wc)
  float* flowt = nullptr;          // (T,B,2,Hc,Wc)
};

// A clip (Engine::forward_clip): F frames (IO::img_xs is then (F,3,Hf,Wf)) and Problem::B = P pairs of frame indices, pair p
// interpolating from frame src[p] to frame tgt[p] at the problem's T timesteps.  Any pairs: reversed, repeated or a frame with itself.
struct Clip {
  int F = 0;
  std::vector<int> src, tgt;
};

// A query list (Engine::forward_queries): F frames (IO::img_xs (F,3,Hf,Wf)) and Q queries, query q interpolating from frame src[q] to
// frame tgt[q] at t[q] in (0, 1).  Queries with the same (src, tgt) are the timesteps of one pair, in query order.  Per-timestep outputs
// are (Q, ...) in query order; raft_flow / nflow are (P, ...) over the distinct pairs in first-appearance order.
struct Queries {
  int F = 0;
  std::vector<int> src, tgt;
  std::vector<float> t;
};
struct Schedule;   // engine.cu: the frames, pairs, timesteps and output rows of one interpolation (run())

// Outputs of an EXTERNAL bidirectional flow estimator at the network resolution (GIMM-VFI-F: FlowFormer, gimmvfi_f.py:114-138) in the
// reference's NCHW layouts; with these the engine runs everything downstream of cal_bidirection_flow (forward_from_flow)
struct FlowInputs {
  const float* flows = nullptr;                  // (B,2,2,H,W): [f01 | f10] on dim 2
  const float* feat4[2] = {nullptr, nullptr};    // (B,128,H/4,W/4): features0[0], features1[0]
  const float* feat8[2] = {nullptr, nullptr};    // (B,256,H/8,W/8): features0[1], features1[1]
  const float* fnet[2] = {nullptr, nullptr};     // (B,256,H/8,W/8): the maps BidirCorrBlock correlates
};

struct DebugTap { TV tv; };

// coords1 = coords1 + flow_init, the warm start of RAFT (raft.py:140-141) and of FlowFormer's memory decoder (decoder.py:265-267):
// NCHW (n,2,h,w) onto the NHWC (x, y) coordinates
struct FlowInitAddK {
  const float* init; TV c;
  GV_HD void operator()(int64_t i) const {
    const int x = (int)(i % c.w); int64_t r = i / c.w;
    const int y = (int)(r % c.h); r /= c.h;
    const int ch = (int)(r % 2); const int n = (int)(r / 2);
    c.p[c.off(n, y, x) + ch] += init[i];
  }
};

// FlowFormer.forward (transformer.py:45-74) over a frame set and a pair list: device pointers of the standalone entry point, reference
// NCHW layouts, every one but flow_up optional.  cfeat4 / cfeat8 / ffeat belong to each pair's source frame (return_feat=True).
struct FlowFormerOutputs {
  float* flow_up = nullptr;      // (P,2,H,W)          flow_predictions[-1]                                        decoder.py:321
  float* flow_low = nullptr;     // (P,2,H/8,W/8)      coords1 - coords0 of the last iteration                            :321
  float* cfeat4 = nullptr;       // (P,128,H/4,W/4)    cfeat[0]: the context Twins' first stage output      encoders.py:22-48
  float* cfeat8 = nullptr;       // (P,256,H/8,W/8)    cfeat[1]: its second stage output
  float* ffeat = nullptr;        // (P,256,H/8,W/8)    the channel_convertor output of the source           encoder.py:512-518
};

// RAFT.forward (raft/raft.py:100-169) over a frame set and a pair list: device pointers of the standalone entry point, reference NCHW
// layouts, every one optional.  feat4 / feat8 / fmap belong to each pair's source frame.
struct RaftOutputs {
  float* flow_up = nullptr;      // (P,2,H,W)          flow_up of the last iteration                  raft.py:155-163
  float* flow_low = nullptr;     // (P,2,H/8,W/8)      coords1 - coords0 of the last iteration (test_mode)    :165-166
  float* flow_iters = nullptr;   // (iters,P,2,H,W)    flow_predictions, one upsampled flow per iteration     :163,169
  float* feat4 = nullptr;        // (P,96,H/4,W/4)     feats[1] of cnet (layer2)                   :131, extractor.py:195-200
  float* feat8 = nullptr;        // (P,128,H/8,W/8)    feats[2] of cnet (layer3)                   :131, extractor.py:201-206
  float* fmap = nullptr;         // (P,256,H/8,W/8)    fmap1 of fnet                                           :121
};

// One run of RAFT on prepared frames (Engine::run_raft): inputs, outputs in the engine's NHWC buffers, and the hook GIMM-VFI-R uses
struct RaftRun {
  TV img;                                  // (F,H,W,3 [ld 4]) frames as 2 * (x / 255) - 1 (raft.py:111-112)
  std::vector<int> src, tgt;               // pair s: the flow from frame src[s] to frame tgt[s]
  int iters = 12;
  bool gather = false;                     // always take the gathering path (the planner's upper bound)
  int decide_as = 0;                       // > 0: choose volume or volume-free lookups as a run of this many pairs would (0: the pair count)
  const float* flow_init = nullptr;        // optional (P,2,H/8,W/8) NCHW, added to coords1 (raft.py:140-141)
  TV flow_up;                              // (P,H,W,2)
  TV flow_low;                             // optional (P,H/8,W/8,2)
  float* flow_iters = nullptr;             // optional NCHW (iters,P,2,H,W)
  TV fmap;                                 // (F,H/8,W/8,256): fnet of every frame
  int enc0 = 0;                            // frames [0, enc0) are not encoded: `encoded` fills their fmap and net | inp (sources in frame order only)
  // called after the encoders, before the correlation: c4 / c8 = cnet's layer2 / layer3 outputs of the encoded distinct sources in
  // first-use order (frames [enc0, F) when the sources are the frames in order); hx = the pairs' [net | inp | motion] buffer
  std::function<void(const TV& c4, const TV& c8, const TV& hx)> encoded;
};

// GIMM.forward (gimm.py:129-214) device pointers, reference layouts
struct GimmIO {
  const float* xs = nullptr;        // (B,2,2,H,W) normalised flows [f01 | f10] on dim 2
  const float* ori_flow = nullptr;  // (B,2,2,H,W) raw flows
  const float* coords = nullptr;    // (T,B,1,H,W,3)
  const float* t = nullptr;         // (T,B)
  float* out = nullptr;             // (T,B,2,1,H,W) normalised flow at t (keep_xs_shape=True)
};

// LPIPS (src/utils/lpips/lpips.py:125-189, net="alex", version="0.1") device pointers: two float32 NCHW batches (n,3,h,w)
struct LpipsIO {
  const float* in0 = nullptr;
  const float* in1 = nullptr;
  float* out = nullptr;        // (n)     the distance of each pair
  float* per_layer = nullptr;  // (n,5)   optional: the spatial mean of each layer's term (out = their sum)
  int normalize = 0;           // inputs in [0,1]: 2x - 1 first (the module's normalize=True)
  int quantize = 0;            // calc_lpips: ((clamp(x,-1,1) + 1) / 2 * 255).round() / 255 before everything else
};

// The `arch` settings that change GIMM's motion arithmetic but no parameter shape (gimm.py:144-157, hyponet.py:71-146): the forward
// splat's mode and HypoNet's activation, w0, output_bias and fan-in normalisation.  The defaults are the shipped configs'.
struct MotionConfig {
  int fwarp = SPLAT_LINEAR;     // SplatMode
  int act = HYPO_SIREN1;        // HypoAct (HYPO_SIREN1 stands for siren with w0 = 1)
  float w0 = 1.f;
  float output_bias = 0.5f;
  bool normalize_weight = true;
};

struct Net;

class Engine {
 public:
  // the weight set the last finalize_weights* loaded (None: none yet, weights loaded since, or a finalize that failed part-way)
  enum class Weights { None, R, F, Synthesis, Gimm, Raft, FlowFormer, Lpips };
  // the entry points, grouped by the weight sets that serve them (the table in need())
  enum class Entry { Interpolate, FromFlow, Gimm, Raft, FlowFormer, Lpips };
  explicit Engine(int device);
  ~Engine();
  void load_weight(const std::string& key, const float* host, const int64_t* shape, int ndim);
  void finalize_weights();
  void finalize_weights_gimm();                        // a standalone GIMM checkpoint (gimm.py's module tree only)
  void finalize_weights_synthesis();                   // everything downstream of the flow estimator (GIMM-VFI-F's tree minus flow_estimator.*)
  void finalize_weights_f();                           // the complete GIMM-VFI-F tree: synthesis half + the native FlowFormer estimator (flowformer.cu)
  size_t plan_from_flow(const Problem& p);
  void forward_from_flow(const Problem& p, const IO& io, const FlowInputs& fin, void* workspace, size_t workspace_bytes, gvStream_t stream);
  size_t plan_gimm(const Problem& p);
  void forward_gimm(const Problem& p, const GimmIO& io, void* workspace, size_t workspace_bytes, gvStream_t stream);
  void finalize_weights_flowformer();                  // the FlowFormer module's tree alone (flow_estimator.* of F); only the FlowFormer entry points then
  // FlowFormer.forward over n_frames frames (n,3,h,w) in [0,255] and n_pairs (source, target) frame indices (host, 2 per pair):
  // flow_init (P,2,h/8,w/8) optional; outputs: FlowFormerOutputs.  Consecutive pairs form reference calls of pairs_per_call pairs.
  // iters 0: ff_iters.
  size_t plan_flowformer(int n_frames, int h, int w, int n_pairs);
  void forward_flowformer(const float* frames, int n_frames, int h, int w, const int32_t* pairs, int n_pairs, int pairs_per_call, int iters,
                          const float* flow_init, const FlowFormerOutputs& out, void* workspace, size_t workspace_bytes, gvStream_t stream);
  void finalize_weights_raft();                        // the RAFT module's tree alone (flow_estimator.* of R, prefix stripped); only the RAFT entry points then
  // RAFT.forward over n_frames frames (n,3,h,w) in [0,255] and n_pairs (source, target) frame indices (host, 2 per pair); flow_init
  // (P,2,h/8,w/8) optional.  A RAFT-only or a complete GIMM-VFI-R engine serves it.  plan_raft fits every pair list of that length;
  // outputs & GIMMVFI_RAFT_OUT_ITERS: the forward writes flow_iters (the only output that needs workspace of its own).
  size_t plan_raft(int n_frames, int h, int w, int n_pairs, int outputs);
  void forward_raft(const float* frames, int n_frames, int h, int w, const int32_t* pairs, int n_pairs, int iters, const float* flow_init,
                    const RaftOutputs& out, void* workspace, size_t workspace_bytes, gvStream_t stream);
  void finalize_weights_lpips();                       // the 22-key state_dict of LPIPS(net="alex", version="0.1"); only forward_lpips then
  size_t plan_lpips(int n, int h, int w);
  void forward_lpips(int n, int h, int w, const LpipsIO& io, void* workspace, size_t workspace_bytes, gvStream_t stream);
  size_t plan(const Problem& p);                       // dry run -> workspace bytes
  void forward(const Problem& p, const IO& io, void* workspace, size_t workspace_bytes, gvStream_t stream);
  // GIMM-VFI-R / -F over a clip: the per-frame stages (resize, the estimator's encoders, the context projections and the decoders'
  // feature upsampling) run once per frame, everything after the flow estimate once per pair.  Pair p's outputs are those of forward()
  // with B = 1 on (frames[src[p]], frames[tgt[p]]).  The plan holds for this clip's pair list.
  size_t plan_clip(const Problem& p, const Clip& c);
  void forward_clip(const Problem& p, const Clip& c, const IO& io, void* workspace, size_t workspace_bytes, gvStream_t stream);
  // GIMM-VFI-R / -F over a query list: each pair's estimator, encoders and feature upsampling run once, as in forward_clip, and each
  // pair is interpolated at its own timesteps.  The problem supplies Hf, Wf, ds, Hc and Wc (its B and T are ignored); the engine makes
  // the coordinates and t itself (io.coords and io.t must be null).  The plan depends on the frame count, the distinct pairs and their
  // timestep counts, not on the t values.
  size_t plan_queries(const Problem& p, const Queries& q);
  void forward_queries(const Problem& p, const Queries& q, const IO& io, void* workspace, size_t workspace_bytes, gvStream_t stream);
  // the coordinate range of the query grids (the model's coord_range; sample_coord_input's arithmetic in float32)
  void set_coord_range(double lo, double hi) { coord_lo_ = (float)lo; coord_span_ = (float)(hi - lo); }
  int64_t last_launches() const { return launches_; }
  // CUDA graphs: forward() records the launch sequence of a (problem, buffers, mode) combination the SECOND time it sees it and
  // replays the instantiated graph afterwards - one cudaGraphLaunch instead of ~550 kernel launches and ~1000 host-side tensor-map
  // encodes per forward.  The replay is exactly the recorded stream of kernels with the recorded parameters, so it is only used
  // when every pointer the launches captured is unchanged (key below); profiling, debug taps and the frame cache bypass it.
  void set_cuda_graph(bool on) { use_graph_ = on; if (!on) clear_graphs(); }
  int64_t graph_replays() const { return graph_replays_; }
  // debug taps: name -> NHWC view inside the workspace of the last forward
  void set_debug(bool on) { debug_ = on; }
  // per-kernel CUDA-event timing of the next forward(s): {"name": {"ms", "work", "launches"}}
  void set_profile(bool on) { profile_ = on; }
  // 0: fp32 CUDA cores everywhere; 1: post-RAFT convs on TF32 tensor cores; 2: + RAFT convs on fp32-class (3xF16) tensor cores;
  // 3: + final-decoder residual trunk in fp16; 4: + the 32/64-channel full-resolution chains in fp16 (the default of GIMM-VFI-R / -F,
  // RAFT and FlowFormer)
  void set_tensor_cores(int mode) { tc_mode_ = mode; }
  // the motion settings the next finalize_weights* packs the weights for and the forwards after it run with
  void set_motion_config(const MotionConfig& m) { motion_next_ = m; }
  const MotionConfig& motion() const { return motion_; }
  // precision mode 4 (see DESIGN.md): the 32/64-channel full-resolution chains (motion encoder laterals, latent
  // refiner, final-decoder upsample branch) are stored in half precision like the residual trunk of mode 3
  bool half_chains(const Ctx& cx) const { return cx.tc && tc_mode_ >= 4; }
  std::string profile_json(gvStream_t stream);
  // Video callers (src/video_Nx.py:134-216) walk consecutive pairs (j, j+1), (j+1, j+2), ...: the RAFT encoder products of a
  // call's SECOND frame (fnet map, cnet net/inp, projected context features) can be kept in a caller-owned device buffer and
  // re-used as the next call's FIRST frame (SURVEY 8(f) row 2).  load: frame 0 comes from the cache (the caller guarantees it
  // is the frame the cache was stored from); store: frame 1's products are written to it.  Results are bit-identical.
  static size_t frame_cache_bytes(const Problem& p);
  void set_frame_cache(float* cache, size_t bytes, bool load, bool store) { fc_ = cache; fc_bytes_ = bytes; fc_load_ = load; fc_store_ = store; }
  const std::map<std::string, TV>& taps() const { return taps_; }
  std::string last_error;
  int raft_iters = 20;  // GIMMVFI_R hard-codes iters=20 (gimmvfi_r.py:126-132)
  int ff_iters = 32;    // FlowFormer decoder_depth (flowformer/configs/submission.py:50; gimmvfi_f.py:115 passes iters=None)
  bool is_f() const { return held_ == Weights::F; }
  const float* ff_c1w() const { return ff_c1w_.data(); }   // first cost-map patch-embedding layer, [36 taps][16] and [16] (host copies)
  const float* ff_c1b() const { return ff_c1b_.data(); }
  // debug taps from the estimator's helpers (flowformer.cu)
  bool debug_on() const { return debug_; }
  void tap_pub(const std::string& name, const TV& tv) { tap(name, tv); }
  void tap_copy(Ctx& cx, const std::string& name, const TV& tv);   // a snapshot (the tensor is overwritten later in the forward)
  // the same into `snap`, an fp32 (n, h, w, c) buffer allocated by the caller: before a mark / release block whose tensors it copies,
  // so that the release does not hand the snapshot to the next allocations
  void tap_copy_to(Ctx& cx, const std::string& name, const TV& tv, const TV& snap);
  int device() const { return device_; }
  int64_t weights_version() const { return weights_version_; }
  const void* hyponet_blob(bool fp32_class) const { return fp32_class ? hypo_blob3_ : hypo_blob_; }   // bumped by every finalize_weights*: callers key caches on it
  void need(Entry e) const;   // throws unless the weights held serve e

 private:
  struct Impl;
  void drop_weights();
  void prefix_flow_estimator(std::initializer_list<const char*> children);
  size_t dry_run(const std::function<void(Ctx&)>& run);
  void launch(void* workspace, size_t workspace_bytes, gvStream_t stream, const std::function<void(Ctx&)>& run);
  // fin: the flow estimate of an external estimator, with the schedule of forward()
  void run(Ctx& cx, const Problem& p, const IO& io, const Schedule& sched, const FlowInputs* fin = nullptr);
  void frame_cache(Ctx& cx, const Problem& p, const TV& fmap, const TV& ni, const TV& feat4, const TV& feat8);
  void finalize_decoders();
  void finalize_flowformer();
  void pack_patch_conv(const std::string& name);
  void pack_twins(const std::string& prefix);
  // flow_init: optional (P,2,H/8,W/8) NCHW warm start; encoded: called after the encoders with feat4 / feat8 (distinct sources in
  // first-use order) and fproj (every frame), before anything overwrites them
  void run_flowformer(Ctx& cx, Net& N, const TV& img, const std::vector<int>& src, const std::vector<int>& tgt, int per_call, int iters, bool gather,
                      const TV& flow_up, const TV& flow_low, const TV& feat4, const TV& feat8, const TV& fproj, const float* flow_init = nullptr,
                      const std::function<void(const TV& feat4, const TV& feat8, const TV& fproj)>& encoded = {});
  void run_flowformer_pairs(Ctx& cx, const float* frames, int n_frames, int h, int w, const std::vector<int>& src, const std::vector<int>& tgt,
                            int per_call, int iters, bool gather, const float* flow_init, const FlowFormerOutputs& o);
  void finalize_raft();
  void run_raft(Ctx& cx, Net& N, const RaftRun& r);
  void run_raft_pairs(Ctx& cx, const float* frames, int n_frames, int h, int w, const std::vector<int>& src, const std::vector<int>& tgt, int iters,
                      const float* flow_init, const RaftOutputs& o, bool gather);
  void run_gimm(Ctx& cx, const Problem& p, const GimmIO& io);
  void finalize_gimm_part();
  void run_lpips(Ctx& cx, int n, int h, int w, const LpipsIO& io);
  void gimm_encode(Net& N, const TV& nf, const TV& f01, const TV& f10, const TV& wts, const TV& X64);
  // w01 / w10: the splat weights of the two directions
  void gimm_decode(Net& N, const TV& X64, const TV& f01, const TV& f10, const TV& w01, const TV& w10, const float* tdev, const float* coords_t,
                   const TV& ninr, bool tap_it);
  ConvW pack_conv(const std::string& name, const std::string& bn = "", float out_scale = 1.f, const std::vector<int>* perm = nullptr);
  const float* upload(const std::vector<float>& v);
  const float* vec(const std::string& key);
  const HostTensor& raw(const std::string& key) const;
  void tap(const std::string& name, const TV& tv) { if (debug_) taps_[name] = tv; }

  int device_ = 0;
  Weights held_ = Weights::None;
  bool debug_ = false, profile_ = false;
  int tc_mode_ = 0;
  int64_t weights_version_ = 0;
  bool use_graph_ = false;
  int64_t graph_replays_ = 0;
  struct GraphEntry { std::vector<uint64_t> key; void* exec = nullptr; int64_t launches = 0; int seen = 0; };
  std::vector<GraphEntry> graphs_;
  void clear_graphs();
  std::vector<float> ff_c1w_, ff_c1b_;
  float* fc_ = nullptr; size_t fc_bytes_ = 0; bool fc_load_ = false, fc_store_ = false;
  // what the cache holds (host-side bookkeeping of the last store): a load with a different buffer / problem is refused
  // (one record per cache buffer, so several video streams can share an engine; cleared when the weights change)
  struct FcRec { int B, H, W, mode; };
  std::map<const float*, FcRec> fc_valid_;
  void pack_tc(ConvW& c, const std::vector<float>& packed);
  void pack_tc_f16(ConvW& c, const std::vector<float>& packed);
  void pack_stem(const std::string& name, const std::string& bn);
  void pack_xpacked(const std::string& name, int ldp);
  Profiler prof_;
  int64_t launches_ = 0;
  int sm_count_ = 132;
  std::map<std::string, HostTensor> raw_;
  std::map<std::string, ConvW> conv_;
  std::map<std::string, const float*> vec_;
  std::vector<void*> dev_allocs_;
  std::map<std::string, TV> taps_;
  const void* hypo_blob_ = nullptr;   // packed parameters of the fused HypoNet kernel (common.h hypo::)
  const void* hypo_blob3_ = nullptr;  // ... of its fp32-class variant (common.h hypo3::), the one the forwards run
  int raft_direct_ = -1;              // RAFT's own lookups without a volume: -1 = when the volume pyramid exceeds raft_direct_auto_bytes_ (GIMMVFI_RAFT_CORR_DIRECT)
  double raft_direct_auto_bytes_ = 32e9;   // set to 0.4 x the device memory by the constructor (GIMMVFI_RAFT_CORR_DIRECT_GB overrides)
  const float* g9_ = nullptr; const float* alpha_fe_ = nullptr; const float* alpha_v_ = nullptr;
  MotionConfig motion_next_;   // set_motion_config
  MotionConfig motion_;        // what the packed HypoNet weights were built with (finalize_gimm_part); the forwards read this one
  float coord_lo_ = -1.f, coord_span_ = 2.f;   // set_coord_range: coord_range[0] and coord_range[1] - coord_range[0]

  // op helpers used by run()
  friend struct Net;
};

}  // namespace gv
