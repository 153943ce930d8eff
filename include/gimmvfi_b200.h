/* gimmvfi_b200 — C ABI of the H100-native (sm_90a) GIMM-VFI-R inference path.
 *
 * The reference (GSeanCDAT/GIMM-VFI) is pure Python; it has no FFI for this path.
 * Its only native boundaries are
 *   - the CuPy-JIT'd splat kernel launched with raw data_ptr()s on the current
 *     torch stream (src/models/generalizable_INR/modules/softsplat.py:358-446), and
 *   - the pybind extension alt_cuda_corr.forward / backward(fmap1, fmap2, coords, ..., r)
 *     (.../flowformer/alt_cuda_corr/correlation.cpp:19-53), used by RAFT's
 *     AlternateCorrBlock (raft/corr.py:96-124); its counterpart here is
 *     gimmvfi_op_alt_corr_forward / _backward.
 * This header is what a maintainer binds (ctypes, see INTEGRATION.md) to replace the
 * body of GIMMVFI_R.forward() (src/models/generalizable_INR/gimmvfi_r.py:324-407):
 * raw device pointers + sizes + a cudaStream_t, no torch types, no exceptions across
 * the boundary (every call returns 0 on success; gimmvfi_last_error() explains).
 *
 * Threading / ownership: one engine per GPU and per host thread; all work is
 * enqueued on the caller's stream; the caller owns inputs, outputs and the
 * workspace; forward() performs no allocation and no host synchronisation.
 */
#ifndef GIMMVFI_B200_H_
#define GIMMVFI_B200_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gimmvfi_engine gimmvfi_engine;

/* One call of GIMMVFI_R.forward(img_xs, coord, t, ds_factor=ds). */
typedef struct gimmvfi_problem {
  int32_t batch;       /* B: frame pairs                                            */
  int32_t height;      /* Hf, Wf: caller-padded (x32) input size,                    */
  int32_t width;       /*   src/utils/utils.py:156-185 InputPadder                   */
  int32_t timesteps;   /* T = len(t) = len(coord)                                    */
  float ds_factor;     /* 0 -> None; else gimmvfi_r.py:329-337                       */
  int32_t coord_height; /* Hc, Wc of the coord grids = int(H*ds), coord_sampler.py:35 */
  int32_t coord_width;
} gimmvfi_problem;

/* Device pointers (fp32).  Optional outputs may be NULL.  Layouts are the
 * reference's, with the python list index (timestep) as the outermost dim.
 * H, W = network resolution (= Hf,Wf, or floor(Hf*ds), floor(Wf*ds)). */
typedef struct gimmvfi_io {
  const float* img_xs;   /* (B,3,2,Hf,Wf) in [0,1]                      gimmvfi_r.py:324 */
  const float* coords;   /* (T,B,1,Hc,Wc,3) last dim (t,y,x)     coord_sampler.py:21-43 */
  const float* t;        /* (T,B)                                                        */
  float* imgt_pred;      /* (T,B,3,Hf,Wf)   required                    gimmvfi_r.py:399 */
  float* img_warp_4;     /* (T,B,3,H,W)     other_pred[i][0]                         :400 */
  float* flowt0_1;       /* (T,B,3,2,Hf,Wf) flowt0_pred[i][0]                        :401 */
  float* flowt1_1;       /* (T,B,3,2,Hf,Wf) flowt1_pred[i][0]                        :402 */
  float* flowt0_4;       /* (T,B,2,H/4,W/4) flowt0_pred[i][1]                             */
  float* flowt1_4;       /* (T,B,2,H/4,W/4) flowt1_pred[i][1]                             */
  float* raft_flow;      /* (B,2,2,H,W)                                              :403 */
  float* nflow;          /* (B,2,2,H,W)                                              :405 */
  float* ninrflow;       /* (T,B,2,1,Hc,Wc)                                          :404 */
  float* flowt;          /* (T,B,2,Hc,Wc)                                            :406 */
} gimmvfi_io;

/* NHWC fp32 view used by the per-kernel entry points and debug taps:
 * element (n,y,x,c) = data[n*batch_stride + (y*w + x)*pixel_stride + c]. */
typedef struct gimmvfi_view {
  float* data;
  int32_t n, h, w, c;
  int32_t pixel_stride;
  int64_t batch_stride;
} gimmvfi_view;

/* ---- engine life cycle ---- */
int gimmvfi_create(int device, gimmvfi_engine** out);
void gimmvfi_destroy(gimmvfi_engine* e);
/* state_dict entry (HOST pointer, fp32; int64 buffers are skipped by the caller).
 * Keys are the reference's 414 state_dict keys (gimmvfi_r.py:37-111). */
int gimmvfi_load_weight(gimmvfi_engine* e, const char* key, const float* host_data, const int64_t* shape, int ndim);
/* Packs (layout change, BatchNorm folding, HypoNet column normalisation) and uploads. */
int gimmvfi_finalize_weights(gimmvfi_engine* e);
int gimmvfi_plan(gimmvfi_engine* e, const gimmvfi_problem* p, size_t* workspace_bytes);
int gimmvfi_forward(gimmvfi_engine* e, const gimmvfi_problem* p, const gimmvfi_io* io, void* workspace, size_t workspace_bytes,
                    void* cuda_stream);
/* ---- A clip in one call (GIMM-VFI-R and GIMM-VFI-F with their own estimator) ----
 * `frames` frames and `pairs` (source, target) pairs of frame indices, every pair interpolated at the same T timesteps.  Any pairs are
 * allowed: consecutive or not, reversed, repeated, or a frame with itself.  Per frame: the ds_factor resize, the estimator's encoders
 * (RAFT fnet / cnet, FlowFormer's Twins), the context projections and the decoders' feature upsampling; per pair: correlation, the
 * estimator's iterations, GIMM and the synthesis.  Pair p's outputs are gimmvfi_forward's with batch 1 on (frame src, frame tgt): the
 * same estimator path (RAFT chooses its volume or volume-free lookup as for one pair) and flows, and the splat's float-atomic
 * summation order as the only difference behind it.
 * problem->batch must equal pairs; io->img_xs points at the frames, (F,3,Hf,Wf) in [0,1]; coords (T,P,1,Hc,Wc,3), t (T,P); the
 * outputs are gimmvfi_io's with P in place of B.  The workspace holds P pairs' correlation volumes (RAFT's all-pairs pyramid grows
 * with P): gimmvfi_plan_clip reports it for this pair list, to choose how many pairs one call takes.  A pair list whose volumes do
 * not fit the device needs fewer pairs per call; the clip never changes a pair's lookup path to make them fit.  Not recorded as a
 * CUDA graph; the frame cache does not apply. */
typedef struct gimmvfi_clip {
  int32_t frames;              /* F >= 1                                      */
  int32_t pairs;               /* P >= 1                                      */
  const int32_t* pair_list;    /* HOST (P,2): source, target frame index     */
} gimmvfi_clip;
int gimmvfi_plan_clip(gimmvfi_engine* e, const gimmvfi_problem* p, const gimmvfi_clip* clip, size_t* workspace_bytes);
int gimmvfi_forward_clip(gimmvfi_engine* e, const gimmvfi_problem* p, const gimmvfi_clip* clip, const gimmvfi_io* io, void* workspace,
                         size_t workspace_bytes, void* cuda_stream);
/* ---- A query list in one call: every pair at its own timesteps (GIMM-VFI-R and GIMM-VFI-F with their own estimator) ----
 * `frames` frames and `queries` queries (source, target, t).  The queries that share (source, target) are the timesteps of one pair, in
 * query order; any pairs are allowed, as in the clip call.  Per used frame: the clip's per-frame stages (frames no query references are
 * not read); per distinct pair: correlation, the estimator, GIMM's encoder and the decoders' feature upsampling, once; per query: one
 * timestep of GIMM's decoder and the synthesis.  Query q's outputs are gimmvfi_forward's with batch 1 on (frame src, frame tgt) at that
 * pair's own timestep list, with the splat's float-atomic summation order as the only difference behind it: the same estimator path,
 * and the same choice of GIMM's correlation lookup (volume-free for a pair of at most 2 timesteps, the all-pairs pyramid otherwise).
 * Every index must lie in [0, frames) and every t strictly inside (0, 1) (the lookup divides by t and 1 - t); anything else fails
 * before a launch.
 * problem supplies height, width, ds_factor, coord_height and coord_width; its batch and timesteps are ignored.  The engine makes each
 * query's coordinate grid (sample_coord_input at the network resolution, over the range of gimmvfi_set_coord_range) and t on the
 * device: io->coords and io->t must be NULL.  io->img_xs points at the frames, (F,3,Hf,Wf) in [0,1].  Per-timestep outputs are (Q,...)
 * in query order in place of (T,B,...); raft_flow and nflow are (P,2,2,H,W) over the P distinct pairs in first-appearance order.
 * gimmvfi_plan_queries reports the workspace; it depends on the frame count, the distinct pair list and each pair's timestep count,
 * not on the t values, so a retimer whose pattern of pairs and counts repeats reuses one plan.  Not recorded as a CUDA graph; the
 * frame cache does not apply. */
typedef struct gimmvfi_queries {
  int32_t frames;              /* F >= 1                                      */
  int32_t queries;             /* Q >= 1                                      */
  const int32_t* pair_list;    /* HOST (Q,2): source, target frame index     */
  const float* t;              /* HOST (Q): the timestep of each query        */
} gimmvfi_queries;
int gimmvfi_plan_queries(gimmvfi_engine* e, const gimmvfi_problem* p, const gimmvfi_queries* queries, size_t* workspace_bytes);
int gimmvfi_forward_queries(gimmvfi_engine* e, const gimmvfi_problem* p, const gimmvfi_queries* queries, const gimmvfi_io* io,
                            void* workspace, size_t workspace_bytes, void* cuda_stream);
/* The model's coord_range [lo, hi] for the query grids (default [-1, 1]): coordinate = lo + (hi - lo) * c in float32, (hi - lo) taken
 * in double first, as sample_coord_input computes it. */
int gimmvfi_set_coord_range(gimmvfi_engine* e, double lo, double hi);

/* ---- GIMM-VFI-F (gimmvfi_f.py): everything downstream of the flow estimator ----
 * GIMMVFI_F.forward = FlowFormer (cal_bidirection_flow, gimmvfi_f.py:114-138) + exactly the GIMM / synthesis stages of GIMM-VFI-R
 * without the feature projections.  Those stages run natively on the outputs of an EXTERNAL estimator, given in the reference's
 * NCHW layouts at the network resolution H x W (= Hf x Wf, or floor(Hf*ds) x floor(Wf*ds)):                                      */
typedef struct gimmvfi_flow_inputs {
  const float* flows;      /* (B,2,2,H,W)       [f01 | f10] on dim 2 = `ori_flows` of cal_bidirection_flow        gimmvfi_f.py:127 */
  const float* feat4[2];   /* (B,128,H/4,W/4)   features0[0], features1[0]  (context-encoder stage 1)       encoders.py:22-48 */
  const float* feat8[2];   /* (B,256,H/8,W/8)   features0[1], features1[1]  (context-encoder stage 2)                         */
  const float* fnet[2];    /* (B,256,H/8,W/8)   fnet0, fnet1 -> BidirCorrBlock                               gimmvfi_f.py:121 */
} gimmvfi_flow_inputs;
/* Weights: the GIMM-VFI-F state_dict minus flow_estimator.* (gimmvfi_load_weight each, then this instead of gimmvfi_finalize_weights).
 * A full GIMM-VFI-R engine (gimmvfi_finalize_weights) accepts gimmvfi_forward_from_flow as well (its RAFT is then skipped). */
int gimmvfi_finalize_weights_synthesis(gimmvfi_engine* e);
/* The COMPLETE GIMM-VFI-F state_dict (639 tensors, flow_estimator.* = FlowFormer included; gimmvfi_f.py:27-111): gimmvfi_forward then
 * runs the native FlowFormer estimator (Twins-SVT-L x2, cost-perceiver memory encoder, 32-iteration GMA memory decoder; replaces
 * flowformer/core/FlowFormer/LatentCostFormer/transformer.py:45-74 as called by gimmvfi_f.py:114-138) followed by the synthesis half.
 * The network resolution (H, W after ds_factor) must be a multiple of 32. */
int gimmvfi_finalize_weights_f(gimmvfi_engine* e);
/* decoder_depth of the FlowFormer memory decoder (default 32, flowformer/configs/submission.py:50) */
int gimmvfi_set_flowformer_iters(gimmvfi_engine* e, int iters);
int gimmvfi_plan_from_flow(gimmvfi_engine* e, const gimmvfi_problem* p, size_t* workspace_bytes);
/* io->raft_flow (optional) receives a copy of `flows` (the reference returns them as "raft_flow", gimmvfi_f.py:382). */
int gimmvfi_forward_from_flow(gimmvfi_engine* e, const gimmvfi_problem* p, const gimmvfi_io* io, const gimmvfi_flow_inputs* fin,
                              void* workspace, size_t workspace_bytes, void* cuda_stream);

/* ---- GIMM standalone: GIMM.forward (gimm.py:129-214), the motion-modelling network alone (SURVEY 8(f) row 4) ----
 * Weights: either the full GIMM-VFI-R state_dict (gimmvfi_finalize_weights) or a GIMM checkpoint holding only gimm.py's module
 * tree (cnn_encoder.*, res_conv.*, hyponet.*, g_filter, alpha_v, alpha_fe) followed by gimmvfi_finalize_weights_gimm.
 * problem: batch, height, width = flow resolution (any size >= 8), timesteps = T, ds_factor = 0, coord_height / coord_width =
 * Hc, Wc >= 1 of any size (e.g. sample_coord_input(..., upsample_ratio=r): Hc = int(H r)); HypoNet resizes the latent to the grid
 * (bilinear, align_corners = False, hyponet.py:86-90) before its MLP.
 * xs (B,2,2,H,W): flows normalised as in fi_utils.py:52-60, [f01 | f10] on dim 2; ori_flow (B,2,2,H,W): the raw flows;
 * coords (T,B,1,Hc,Wc,3); t (T,B); out (T,B,2,1,Hc,Wc) = the list of keep_xs_shape=True outputs.
 * (GIMM-VFI-R / -F, gimmvfi_forward*, still need coord_height / coord_width = the network resolution: their frame synthesis takes
 * the flow at that resolution.) */
int gimmvfi_finalize_weights_gimm(gimmvfi_engine* e);
int gimmvfi_gimm_plan(gimmvfi_engine* e, const gimmvfi_problem* p, size_t* workspace_bytes);
int gimmvfi_gimm_forward(gimmvfi_engine* e, const gimmvfi_problem* p, const float* xs, const float* ori_flow, const float* coords,
                         const float* t, float* out, void* workspace, size_t workspace_bytes, void* cuda_stream);

/* ---- LPIPS (src/utils/lpips: LPIPS(net="alex", version="0.1"), the perceptual metric of the evaluation drivers) ----
 * Weights: the module's 22-key state_dict (scaling_layer.{shift,scale}; net.slice1.0, net.slice2.3, net.slice3.6, net.slice4.8,
 * net.slice5.10 .weight / .bias; lin{0..4}.model.1.weight; lins.{0..4}.model.1.weight, which must equal lin*), then
 * gimmvfi_finalize_weights_lpips.  Such an engine serves gimmvfi_lpips_* only, and the other engines refuse gimmvfi_lpips_*.
 * in0, in1: float32 NCHW (n,3,h,w), h, w >= 31; out (n): LPIPS of each pair; per_layer (n,5) optional: the spatial mean of each layer's
 * term (out is their sum).  flags: GIMMVFI_LPIPS_NORMALIZE = the module's normalize=True (2x - 1), GIMMVFI_LPIPS_QUANTIZE = calc_lpips's
 * ((clamp(x,-1,1) + 1) / 2 * 255).round() / 255 applied first.  Convolutions run in the fp32-class 3xF16 form; the head's reductions
 * use no atomics, so two calls on the same inputs give bit-identical results. */
#define GIMMVFI_LPIPS_NORMALIZE 1
#define GIMMVFI_LPIPS_QUANTIZE 2
int gimmvfi_finalize_weights_lpips(gimmvfi_engine* e);
int gimmvfi_lpips_plan(gimmvfi_engine* e, int n, int h, int w, size_t* workspace_bytes);
int gimmvfi_lpips_forward(gimmvfi_engine* e, const float* in0, const float* in1, int n, int h, int w, int flags, float* out, float* per_layer,
                          void* workspace, size_t workspace_bytes, void* cuda_stream);

/* ---- FlowFormer standalone: FlowFormer.forward(image1, image2) (LatentCostFormer/transformer.py:45-74) over a pair list ----
 * Weights: the FlowFormer module's state_dict (the reference's initialize_Flowformer() tree, i.e. GIMM-VFI-F's flow_estimator.* with or
 * without that prefix) followed by gimmvfi_finalize_weights_flowformer.  Such an engine serves gimmvfi_flowformer_* only; a complete
 * GIMM-VFI-F engine (gimmvfi_finalize_weights_f) serves them as well.
 * frames (n_frames,3,h,w) float32 in [0,255] on the device (the engine applies 2 * (x / 255.0) - 1.0); h and w multiples of 32.
 * pairs: HOST int32 [n_pairs][2] = (source, target) frame indices, n_pairs >= 1.  flow_up (n_pairs,2,h,w): the 8x convex-upsampled flow
 * from source to target; flow_low (n_pairs,2,h/8,w/8) optional: coords1 - coords0 of the last iteration.  iters: decoder iterations
 * (0 = the engine's setting, default 32).  Consecutive pairs form reference calls of pairs_per_call pairs each (the batch of one
 * FlowFormer.forward; it matters because the reference's context.repeat lets a pair's cost memory read another pair's context within a
 * call): 1 = every pair on its own, as FlowFormer.forward with batch 1.  The feature Twins runs once per frame and the context Twins once
 * per distinct source frame, so a frame shared by several pairs is encoded once.
 * Memory per pair: the cost volume and the GMA attention matrix are N^2 floats each, N = (h/8)(w/8): 12.8 MB each at 256 x 448,
 * 4.3 GB each at 1088 x 1920.  gimmvfi_flowformer_plan returns a workspace size that fits every pair list of that length. */
int gimmvfi_finalize_weights_flowformer(gimmvfi_engine* e);
int gimmvfi_flowformer_plan(gimmvfi_engine* e, int n_frames, int h, int w, int n_pairs, size_t* workspace_bytes);
int gimmvfi_flowformer_forward(gimmvfi_engine* e, const float* frames, int n_frames, int h, int w, const int32_t* pairs, int n_pairs, int pairs_per_call,
                               int iters, float* flow_up, float* flow_low, void* workspace, size_t workspace_bytes, void* cuda_stream);
/* The whole FlowFormer.forward(image1, image2, flow_init=..., return_feat=True): gimmvfi_flowformer_forward is this call with the last
 * four pointers NULL.  Each is optional:
 *   flow_init (n_pairs,2,h/8,w/8)    added to coords1 before the first iteration (decoder.py:265-267): the warm start of a clip, the
 *                                    previous pair's flow_low pushed forward by gimmvfi_op_forward_interpolate
 *   cfeat4    (n_pairs,128,h/4,w/4)  cfeat[0] of return_feat: the context Twins' first stage output (encoders.py:22-48)
 *   cfeat8    (n_pairs,256,h/8,w/8)  cfeat[1]: its second stage output, the context the decoder reads
 *   ffeat     (n_pairs,256,h/8,w/8)  ffeat: the channel_convertor output the cost volume is built from (encoder.py:512-518)
 * The three features belong to each pair's source frame.  They need no workspace of their own: gimmvfi_flowformer_plan covers them. */
int gimmvfi_flowformer_forward_ex(gimmvfi_engine* e, const float* frames, int n_frames, int h, int w, const int32_t* pairs, int n_pairs,
                                  int pairs_per_call, int iters, const float* flow_init, float* flow_up, float* flow_low, float* cfeat4,
                                  float* cfeat8, float* ffeat, void* workspace, size_t workspace_bytes, void* cuda_stream);

/* ---- RAFT standalone: RAFT.forward(image1, image2, iters, flow_init) (raft/raft.py:100-169) over a pair list ----
 * Weights: the RAFT module's state_dict (the reference's initialize_RAFT() tree, raft/__init__.py:7-24: GIMM-VFI-R's flow_estimator.*
 * with that prefix stripped; fnet.*, cnet.*, update_block.*) followed by gimmvfi_finalize_weights_raft.  Such an engine serves
 * gimmvfi_raft_* only; a complete GIMM-VFI-R engine (gimmvfi_finalize_weights) serves them as well, and every other engine refuses them.
 * frames (n_frames,3,h,w) float32 in [0,255] on the device (the engine applies 2 * (x / 255.0) - 1.0, raft.py:111-112); h and w multiples
 * of 8 and >= 128.  pairs: HOST int32 [n_pairs][2] = (source, target) frame indices, n_pairs >= 1; every pair is RAFT.forward with
 * batch 1 of frames[source], frames[target].  iters >= 1 (the reference's default is 12; GIMM-VFI-R uses 20).
 * flow_init (n_pairs,2,h/8,w/8) optional: added to coords1 before the first iteration (raft.py:140-141).
 * Outputs, each optional (NULL skips it):
 *   flow_up    (n_pairs,2,h,w)          the last iteration's convex-upsampled flow (raft.py:163; test_mode's second, return_feat's first)
 *   flow_low   (n_pairs,2,h/8,w/8)      coords1 - coords0 after the last iteration (raft.py:165-166, test_mode's first)
 *   flow_iters (iters,n_pairs,2,h,w)    flow_predictions: every iteration's upsampled flow (raft.py:163,169)
 *   feat4      (n_pairs,96,h/4,w/4)     feats[1] of cnet(image1, return_feature=True): layer2's output (raft.py:131,168)
 *   feat8      (n_pairs,128,h/8,w/8)    feats[2]: layer3's output
 *   fmap       (n_pairs,256,h/8,w/8)    fmap1 of fnet (raft.py:121,168)
 * feat4, feat8 and fmap belong to each pair's source frame.  fnet runs once per frame and cnet once per distinct source frame.
 * The volume pyramid is N^2 * 4/3 floats per pair (N = (h/8)(w/8)); when the pair list's pyramid exceeds 0.4 x the device memory (or
 * GIMMVFI_RAFT_CORR_DIRECT=1), the lookups compute their dot products from the target's features instead, as in gimmvfi_forward.
 * gimmvfi_raft_plan returns a workspace size that fits every pair list of that length; outputs: GIMMVFI_RAFT_OUT_ITERS when the forward
 * writes flow_iters (the only output with workspace of its own). */
#define GIMMVFI_RAFT_OUT_ITERS 1
int gimmvfi_finalize_weights_raft(gimmvfi_engine* e);
int gimmvfi_raft_plan(gimmvfi_engine* e, int n_frames, int h, int w, int n_pairs, int outputs, size_t* workspace_bytes);
int gimmvfi_raft_forward(gimmvfi_engine* e, const float* frames, int n_frames, int h, int w, const int32_t* pairs, int n_pairs, int iters,
                         const float* flow_init, float* flow_up, float* flow_low, float* flow_iters, float* feat4, float* feat8, float* fmap,
                         void* workspace, size_t workspace_bytes, void* cuda_stream);

const char* gimmvfi_last_error(gimmvfi_engine* e);
int64_t gimmvfi_last_launches(gimmvfi_engine* e);
/* bumped by every gimmvfi_finalize_weights*: callers that keep derived state (the frame cache below) key it on this */
int64_t gimmvfi_weights_version(gimmvfi_engine* e);
int gimmvfi_set_raft_iters(gimmvfi_engine* e, int iters);
/* debug taps: intermediate tensors of the last forward (views into the workspace) */
int gimmvfi_set_debug(gimmvfi_engine* e, int on);
int gimmvfi_get_tap(gimmvfi_engine* e, const char* name, gimmvfi_view* out);
/* Video callers (src/video_Nx.py:134-216) walk consecutive pairs (j, j+1), (j+1, j+2), ...  A caller-owned device buffer of
 * gimmvfi_frame_cache_bytes() keeps the RAFT encoder products of a call's SECOND frame (raft/raft.py:118-136 fnet map and cnet
 * net/inp, gimmvfi_r.py:134-141 projected context features); with load != 0 the next forward takes its FIRST frame's products
 * from it instead of recomputing them (the caller guarantees it is the same frame, same problem), with store != 0 it writes the
 * second frame's products.  cache == NULL switches the mechanism off.  Results are bit-identical to an uncached forward. */
size_t gimmvfi_frame_cache_bytes(const gimmvfi_problem* p);
int gimmvfi_set_frame_cache(gimmvfi_engine* e, void* cache, size_t bytes, int load, int store);
/* 0: fp32 CUDA cores everywhere; 1: post-RAFT convolutions on the wgmma TF32 path (fp32 accumulate);
 * 2: additionally the RAFT convolutions on wgmma with 3xTF32 operand splitting (fp32-class accuracy) */
int gimmvfi_set_tensor_cores(gimmvfi_engine* e, int mode);
/* The arch settings of GIMM's motion path that change no parameter shape (the reference's fwarp_type and hyponet.activation /
 * output_bias / normalize_weight).  They take effect at the next gimmvfi_finalize_weights* (which packs HypoNet's weights for them) and
 * hold for every forward after it.  An engine that never calls this runs the shipped settings: linear splatting, siren with w0 = 1,
 * output_bias 0.5, fan-in normalised weights.
 *   fwarp_mode: GIMMVFI_FWARP_*, the forward splat of the motion latents (softsplat "<mode>-zeroeps")
 *   activation: GIMMVFI_ACT_*, between HypoNet's layers; w0 is siren's and damp's frequency (ignored by relu and silu) */
#define GIMMVFI_FWARP_LINEAR 0
#define GIMMVFI_FWARP_SOFTMAX 1
#define GIMMVFI_FWARP_SUM 2
#define GIMMVFI_ACT_SIREN 0
#define GIMMVFI_ACT_RELU 1
#define GIMMVFI_ACT_SILU 2
#define GIMMVFI_ACT_DAMP 3
int gimmvfi_set_motion_config(gimmvfi_engine* e, int fwarp_mode, int activation, float w0, float output_bias, int normalize_weight);
/* CUDA graphs (off by default): gimmvfi_forward records its launch sequence the second time it is called with the same problem, the
 * same caller pointers (inputs, outputs, workspace), stream and mode, and replays the instantiated graph from then on - one graph
 * launch instead of ~550 kernel launches + ~1000 host-side tensor-map encodes.  Calls with other pointers run eagerly (and start
 * their own record; 8 graphs are kept).  gimmvfi_graph_replays: forwards served by a replay so far. */
int gimmvfi_set_cuda_graph(gimmvfi_engine* e, int on);
int64_t gimmvfi_graph_replays(gimmvfi_engine* e);
/* per-kernel CUDA-event timing of subsequent forwards; profile_json() synchronises the stream and
 * returns {"kernel": {"ms": total, "work": flops-or-elements, "launches": n}, ...} for the LAST forward */
int gimmvfi_set_profile(gimmvfi_engine* e, int on);
const char* gimmvfi_profile_json(gimmvfi_engine* e, void* cuda_stream);
const char* gimmvfi_build_info(void);

/* ---- per-kernel entry points (unit tests; all NHWC fp32 device views) ---- */
/* softsplat "linear-zeroeps": modules/softsplat.py:286-352 (kernel :371-421).
 * lat (n,h,w,16) flow (n,h,w,2) metric (n,h,w,1) t (n) scratch (n,h,w,>=17 ch, pixel_stride>=17) out (n,h,w,16);
 * the splat flow is flow*t (t_mode 0) or flow*(1-t) (t_mode 1). */
int gimmvfi_op_softsplat(const gimmvfi_view* lat, const gimmvfi_view* flow, const gimmvfi_view* metric, const float* t, int t_mode,
                         const gimmvfi_view* scratch, const gimmvfi_view* out, void* stream);
/* ---- differentiable softmax splatting (training): softsplat_func of modules/softsplat.py:358-663 ----
 * A 4-D strided tensor: element (i0,i1,i2,i3) at data[i0*strides[0] + i1*strides[1] + i2*strides[2] + i3*strides[3]] (strides in
 * ELEMENTS, so a channels-last or sliced torch tensor is described in place); dtype GIMMVFI_FLOAT32 or GIMMVFI_FLOAT64. */
#define GIMMVFI_FLOAT32 0
#define GIMMVFI_FLOAT64 1
typedef struct gimmvfi_tensor4 {
  void* data;
  int32_t dtype;
  int64_t sizes[4];
  int64_t strides[4];
} gimmvfi_tensor4;
/* softsplat_out (:371-421): in (N,C,H,W), flow (N,2,H,W) -> out (N,C,H,W) = the bilinear forward splat of in along flow; out is
 * zero-filled by the call and must be dense (its elements one contiguous block, in any dimension order).  Each source pixel adds its
 * four weighted corner contributions with atomics, so fp32 sums are re-associated from run to run; pixels with a non-finite target
 * coordinate add nothing.  Host-side checks: equal N/H/W, 2 flow channels, one dtype everywhere, float32 or float64. */
int gimmvfi_op_softsplat_out(const gimmvfi_tensor4* in, const gimmvfi_tensor4* flow, const gimmvfi_tensor4* out, void* stream);
/* softsplat_ingrad (:478-533) and softsplat_flowgrad (:564-637) in ONE pass: for the incoming gradient outgrad (N,C,H,W) writes
 * ingrad (N,C,H,W) and / or flowgrad (N,2,H,W), either may be NULL (at least one is required).  Every element of a requested
 * output is written (0 for a pixel whose target coordinate is non-finite or whose four corners all leave the frame), so neither needs
 * zeroing.  `in` is read only for flowgrad (its descriptor is still checked).  No atomics: two calls give identical bits. */
int gimmvfi_op_softsplat_grad(const gimmvfi_tensor4* in, const gimmvfi_tensor4* flow, const gimmvfi_tensor4* outgrad, const gimmvfi_tensor4* ingrad,
                              const gimmvfi_tensor4* flowgrad, void* stream);
/* ---- memory-free correlation (training): alt_cuda_corr of flowformer/alt_cuda_corr/correlation_kernel.cu ----
 * A dense row-major tensor of ndim <= 5 dimensions (the last one contiguous, no padding anywhere); dtype GIMMVFI_FLOAT32. */
typedef struct gimmvfi_dense {
  void* data;
  int32_t dtype;
  int32_t ndim;
  int64_t sizes[5];
} gimmvfi_dense;
/* fmap1 (B,H1,W1,C), fmap2 (B,H2,W2,C), coords (B,N,H1,W1,2) holding (x, y) in fmap2 pixels -> corr (B,N,(2r+1)^2,H1,W1).
 * corr[b,n,k,h,w] with k = (oy + r) + (2r+1) * (ox + r), oy, ox in [-r, r] (x offset major, = CorrBlock's meshgrid(dy, dx) order) is
 * the bilinear sample at (x + ox, y + oy) of the dot products <fmap1[b,h,w], fmap2[b,y2,x2]>: with x0 = floor(x), dx = x - x0 (the
 * same for y) it blends the four integer neighbours of the (2r+2)^2 window anchored at (x0 - r, y0 - r) with the weights of the
 * reference kernel (:92-114).  A target outside fmap2 contributes 0; a non-finite coordinate, or one so far outside that no window
 * tap lands in fmap2, makes every tap out of frame (tested in float before any integer conversion).  Every element of corr is
 * written.  C >= 1, N >= 1, r >= 0 (bounded only by the shared memory one CTA needs for a window: r <= 59); every tensor
 * float32 and dense.  Host-side checks: ranks, dtype, equal B / H1 / W1 / C, coords' last dim 2, corr's shape. */
int gimmvfi_op_alt_corr_forward(const gimmvfi_dense* fmap1, const gimmvfi_dense* fmap2, const gimmvfi_dense* coords, int radius,
                                const gimmvfi_dense* corr, void* stream);
/* The gradients of that forward for the incoming corr_grad (B,N,(2r+1)^2,H1,W1); each of fmap1_grad (B,H1,W1,C), fmap2_grad
 * (B,H2,W2,C) and coords_grad (B,N,H1,W1,2) may be NULL (at least one is required) and every element of a requested one is written.
 *   fmap1_grad: a per-source gather, no atomics: two calls give identical bits.
 *   fmap2_grad: zero-filled by the call, then a scatter with red.global.add.f32, so its fp32 sums are re-associated from run to run.
 *   coords_grad: the true derivative of the bilinear weights with the floor held fixed (the convention of grid_sample), 0 where the
 *   coordinate is out of frame.  It needs the window's dot products, which are computed only when it is requested. */
int gimmvfi_op_alt_corr_backward(const gimmvfi_dense* fmap1, const gimmvfi_dense* fmap2, const gimmvfi_dense* coords,
                                 const gimmvfi_dense* corr_grad, int radius, const gimmvfi_dense* fmap1_grad, const gimmvfi_dense* fmap2_grad,
                                 const gimmvfi_dense* coords_grad, void* stream);
/* backward warp: modules/fi_utils.py:19-49 */
/* the same splat in ONE pass (target tiles accumulated in shared memory); flow_absmax[n] (device) >= max |flow| of sample n */
int gimmvfi_op_softsplat_fused(const gimmvfi_view* lat, const gimmvfi_view* flow, const gimmvfi_view* metric, const float* t_per_sample, int t_mode,
                               const float* flow_absmax, const gimmvfi_view* out, void* stream);
int gimmvfi_op_backwarp(const gimmvfi_view* src, const gimmvfi_view* flow, const gimmvfi_view* dst, void* stream);
/* F.interpolate(bilinear, align_corners=False): modules/fi_utils.py:67-70; dst = mult * resize(src) */
int gimmvfi_op_resize(const gimmvfi_view* src, const gimmvfi_view* dst, float scale_factor, float mult, void* stream);
/* test-only: the synthesis tail's pointwise ops in every storage form the engine uses.  half_mask bit 0 / 1: src / dst is IEEE half
   (pixel_stride and batch_stride in elements).  RESIZE: dst (+)= mult * resize(src, scale_factor), then act (ACT_SIGMOID = 4);
   BACKWARP: dst = backwarp(src, flow); COPY: dst = src (channels of dst) */
enum { GIMMVFI_TAIL_RESIZE = 0, GIMMVFI_TAIL_BACKWARP = 1, GIMMVFI_TAIL_COPY = 2 };
int gimmvfi_op_tail_pointwise(int op, const gimmvfi_view* src, const gimmvfi_view* flow, const gimmvfi_view* dst, float scale_factor, float mult,
                              int accumulate, int act, int half_mask, void* stream);
/* all-pairs correlation raft/corr.py:167-175: vol[n][i][j] = <fa[n,i,:], fb[n,j,:]> / sqrt(C) */
/* FlowFormer / Twins-SVT token-side kernels (GIMM-VFI-F's estimator; csrc/ops_tokens.cu).  A token sequence (B, H*W, C) is an NHWC view.
 *   layernorm        nn.LayerNorm over the channels; `out` may be larger than `x` (zero rows / columns: the padding Twins applies after
 *                    the norm, LatentCostFormer/twins.py:835-842); pe_dim > 0 adds LinearPositionEmbeddingSine(x*pe_scale, y*pe_scale)
 *                    (attention.py:170-182)
 *   window_attention LocallyGroupedAttn core (twins.py:846-860): q, k, v on the padded map, ws x ws windows, softmax(q k^T / sqrt(d)) v
 *   global_attention GlobalSubSampleAttn core (twins.py:898-921): every token of q against all tokens of the (sub-sampled) k / v map
 *   patchify         space-to-depth: a k x k stride-k Conv2d (PatchEmbed twins.py:1142, `sr` twins.py:890) = this + a 1x1 convolution
 *   cost_conv1       Conv2d(1, 16, 6, stride 2, padding 2) + ReLU over `maps` cost maps (encoder.py:38-48), zero-extended to a multiple of 8,
 *                    written with a zero border of 2 (out_padded: (maps, oh+4, ow+4, 16)); weights [36][16] / bias [16] are HOST pointers
 *   conv7x7_small_cout  7x7 stride-1 zero-padded Conv2d with <= 4 output channels (amt_comb_block.2, gimmvfi_r.py:60-64), exact fp32;
 *                    weights [49][cin][4] / bias device pointers
 *   row_softmax      in place over a dense rows x cols matrix: p[r][:] = mul * softmax(p[r][:]) (the GMA attention, gma.py:56-76) */
int gimmvfi_op_layernorm(const gimmvfi_view* x, const float* gamma, const float* beta, float eps, const gimmvfi_view* out, float pe_scale, int pe_dim,
                         void* stream);
int gimmvfi_op_window_attention(const gimmvfi_view* q, const gimmvfi_view* k, const gimmvfi_view* v, const gimmvfi_view* out, int heads, int ws,
                                void* stream);
int gimmvfi_op_global_attention(const gimmvfi_view* q, const gimmvfi_view* k, const gimmvfi_view* v, const gimmvfi_view* out, int heads, void* stream);
int gimmvfi_op_patchify(const gimmvfi_view* src, const gimmvfi_view* dst, int k, void* stream);
int gimmvfi_op_cost_conv1(const float* vol, int64_t maps, int h, int w, const float* w_host, const float* b_host, const gimmvfi_view* out_padded,
                          void* stream);
int gimmvfi_op_conv7x7_small_cout(const gimmvfi_view* in, const float* w_tap_cin_4, const float* bias, int cout, const gimmvfi_view* out, void* stream);
int gimmvfi_op_row_softmax(float* p, int64_t rows, int64_t cols, float mul, void* stream);
int gimmvfi_op_corr_volume(const gimmvfi_view* fa, const gimmvfi_view* fb, float* vol, void* stream);
/* the same volume for ONE sample (n == 1, dense views, C % 32 == 0) as a wgmma GEMM: split != 0 -> 3xTF32 (RAFT's volume),
 * else TF32 (the bidirectional volume).  scratch >= 2*h*w*C + h*w + 1024 floats */
int gimmvfi_op_corr_volume_tc(const gimmvfi_view* fa, const gimmvfi_view* fb, float* scratch, float* vol, int split, void* stream);
/* 2x2 average pooling of every row's (h,w) image: raft/corr.py:139-142 */
int gimmvfi_op_corr_pool(const float* src, float* dst, int64_t rows, int h, int w, void* stream);
/* levels 1..3 from level 0 in one pass (three successive corr_pool's, raft/corr.py:139-142) */
int gimmvfi_op_corr_pool_pyramid(const float* l0, float* l1, float* l2, float* l3, int64_t rows, int h, int w, void* stream);
/* 4-level 9x9 lookup raft/corr.py:144-165: lvl[k] = (n*h*w) x (h_k*w_k) pyramids; out (n,h,w,324) */
int gimmvfi_op_corr_lookup(const float* const lvl[4], const int32_t lvl_h[4], const int32_t lvl_w[4], const gimmvfi_view* coords,
                           const gimmvfi_view* out, void* stream);
/* Volume-free form of the same lookup (reference: raft/corr.py:23-93 BidirCorrBlock.__call__, looked up once per interpolated frame):
 * src = the source frame's fp32 features (n,h,w,256); tgt_half[l] = the other frame's features, 2^l x 2^l average-pooled, IEEE half,
 * dense NHWC (n, lvl_h[l], lvl_w[l], 256); out[..., l*81 + a*9 + b] = scale * <src, bilinear sample of level l>, as gimmvfi_op_corr_lookup
 * returns from the volume pyramid. */
int gimmvfi_op_corr_lookup_direct(const gimmvfi_view* src, const void* const tgt_half[4], const int32_t lvl_h[4], const int32_t lvl_w[4], float scale,
                                  const gimmvfi_view* coords, const gimmvfi_view* out, void* stream);
/* conv2d on NHWC: weight packed [kh*kw][cin][cout_ld], act: 0 none,1 relu,2 lrelu(0.1),3 prelu,4 sigmoid,5 tanh,6 sin */
int gimmvfi_op_conv2d(const gimmvfi_view* in0, const gimmvfi_view* in1_or_null, const float* w_packed, const float* bias, int cin,
                      int cout, int cout_ld, int kh, int kw, int stride, int pad_h, int pad_w, int reflect, int act,
                      const float* slope, const gimmvfi_view* residual_or_null, const gimmvfi_view* out, void* stream);
/* wgmma/TMA implicit-GEMM conv (stride 1, "same" zero padding).  w_tc packed [2][kh*kw][cout_pad][cin_pad32]
 * (plane 0 = TF32(w), plane 1 = TF32(w - plane 0); cout_pad = N tiling of cout, see tc_tile_n); bias padded to cout_pad.
 * y = gru( act2(residual + act1(conv + bias)) * mul );  split != 0 -> three-term operand split (fp32-class accuracy, unrounded
 * output): 3xTF32, or — when w_tc_s is given — 3xF16: w_tc_s = half [2][kh*kw][cout_pad][cin_pad64] holding the fp16 hi / lo planes of
 * w * w_scale (w_scale a power of two), activations split on the fly, f16 MMAs at twice the TF32 rate */
int gimmvfi_op_conv2d_tc(const gimmvfi_view* in0, const gimmvfi_view* in1_or_null, const float* w_tc, const float* bias, int cin,
                         int cout, int kh, int kw, int act1, const float* slope1, const gimmvfi_view* residual_or_null, int act2,
                         const float* slope2, const gimmvfi_view* mul_or_null, const gimmvfi_view* gru_z_or_null,
                         const gimmvfi_view* gru_h_or_null, int split, const gimmvfi_view* out, const void* w_tc_s_or_null, float w_scale,
                         void* stream);
/* the same kernel at stride 1 or 2 with "same"-style padding k/2 (RAFT encoder down-sampling convs, raft/extractor.py:42-48,140):
 * out is (n, (h + 2*(kh/2) - kh)/stride + 1, ...); TMA element strides pick every stride-th input pixel */
int gimmvfi_op_conv2d_tc_strided(const gimmvfi_view* in0, const float* w_tc, const float* bias, int cin, int cout, int kh, int kw,
                                 int stride, int act1, int split, const gimmvfi_view* out, void* stream);
/* the same kernel with half-precision storage (precision mode 3: the final decoder's residual trunk, fi_components.py:97-154,
 * 299-305).  half_mask: bit 0 = in0/in1 hold IEEE half (f16 MMAs; weights = w_tc_h [kh*kw][cout_pad][cin_pad64] half),
 * bit 1 = out is half, bit 2 = residual is half; views of half tensors give strides in ELEMENTS.  With bit 0 clear the operands are
 * fp32/TF32 (w_tc as above) and only the store / residual formats change. */
int gimmvfi_op_conv2d_tc_f16(const gimmvfi_view* in0, const gimmvfi_view* in1_or_null, const void* w_tc_h, const float* w_tc,
                             const float* bias, int cin, int cout, int kh, int kw, int act1, const float* slope1,
                             const gimmvfi_view* residual_or_null, int act2, const float* slope2, int half_mask,
                             const gimmvfi_view* out, void* stream);
/* 3x3 stride-1 convolution with zero padding 1 of a wide half layer (csrc/conv_wide.cu: the final decoder's 256-channel trunk): each
 * 64-channel K block's tile + halo is loaded once and the nine taps are MMAs on views of it.  in0 (and in1) hold IEEE half and have
 * channels that are multiples of 64 (16-byte aligned views), cin = their sum, cout a multiple of 128; w_tc_h and the epilogue as
 * gimmvfi_op_conv2d_tc_f16 (half_mask bit 0 must be set; bit 1 = out is half, bit 2 = residual is half).  The residual may be the
 * output itself (in-place ResBlock tail). */
int gimmvfi_op_conv2d_wide(const gimmvfi_view* in0, const gimmvfi_view* in1_or_null, const void* w_tc_h, const float* bias, int cin, int cout,
                           int act1, const float* slope1, const gimmvfi_view* residual_or_null, int act2, const float* slope2, int half_mask,
                           const gimmvfi_view* out, void* stream);
/* nn.InstanceNorm2d + optional relu: raft/extractor.py:133-134; scratch >= gimmvfi_instnorm_scratch_floats */
/* 3x3 (or 1x1) stride-1 convolution of a K-poor layer (cin <= 32 fp32 or <= 64 half, cout <= 64): tile + halo loaded once, the taps as
 * MMAs on views of it, weights resident in shared memory (csrc/conv_halo.cu).  Weight packing as gimmvfi_op_conv2d_tc (plane 0) /
 * gimmvfi_op_conv2d_tc_f16; half_mask bit 0: input half, bit 1: output half, bit 2: residual half; prepadded: 0 = 3x3 with zero padding 1,
 * 1 = 3x3, `in0` is (h+2, w+2) and carries its own padding (valid conv), 2 = 1x1. */
int gimmvfi_op_conv2d_halo(const gimmvfi_view* in0, const void* w_tc_h_or_null, const float* w_tc, const float* bias, int cin, int cout,
                           int act1, const float* slope1, const gimmvfi_view* residual_or_null, int act2, const float* slope2,
                           int half_mask, int prepadded, const gimmvfi_view* out, void* stream);
/* HypoNet.forward (modules/hyponet.py:71-146) as ONE fused wgmma kernel with the engine's loaded weights: latent (n,h,w,32),
 * coords n*h*w x (t,y,x) as the caller's coordinate tensor holds them -> out (n,h,w,2) = normalised flow (output_bias included).
 * fp32_class != 0: the default kernel of the forward pass (fp16 hi/lo operand pairs, fp32-class result); 0: TF32 / half operands.
 * `out` may be (n,hc,wc,2) of another spatial size than `latent`, with coords n*hc*wc x (t,y,x): the latent is then resized to
 * (hc, wc) inside layer 0 (bilinear, align_corners = False); fp32_class != 0 only.  The activation, w0, output_bias and normalisation are
 * those the engine's weights were finalized with (gimmvfi_set_motion_config). */
int gimmvfi_op_hyponet(gimmvfi_engine* e, const gimmvfi_view* latent, const float* coords, const gimmvfi_view* out, int fp32_class,
                       void* cuda_stream);
int64_t gimmvfi_instnorm_scratch_floats(int n, int c);
int gimmvfi_op_instnorm(const gimmvfi_view* x, int relu, float* scratch, const gimmvfi_view* out, void* stream);
/* convex x8 upsampling raft/raft.py:86-97: flow (n,h,w,2), mask (n,h,w,576), out (n,8h,8w,2) */
int gimmvfi_op_convex_upsample(const gimmvfi_view* flow, const gimmvfi_view* mask, const gimmvfi_view* out, void* stream);
/* Driver-side pre/post-processing on the GPU (SURVEY 8(f) row 2; reference src/video_Nx.py:40-50,152-153,182-202):
 * uint8 HWC RGB frames (n,h,w,3) -> float32 (n,3,H,W) = x/255.0, replicate-padded like InputPadder(shape, 32).pad
 * (src/utils/utils.py:156-174: pad_left = pad_w//2, pad_top = pad_h//2) */
int gimmvfi_op_frames_u8_to_padded_f32(const uint8_t* frames, int n, int h, int w, float* dst_nchw, int H, int W, int pad_top,
                                       int pad_left, void* stream);
/* float32 (n,3,H,W) prediction -> unpadded uint8 (n,h,w,3): (x*255.0).astype(uint8) with optional RGB->BGR flip
 * (InputPadder.unpad + video_Nx.py:190-196) */
int gimmvfi_op_pred_to_u8(const float* pred_nchw, int n, int H, int W, uint8_t* dst, int h, int w, int pad_top, int pad_left, int bgr,
                          void* stream);
/* Flow visualisation, flow_to_image of src/utils/flow_viz.py (the Middlebury colour wheel; video_Nx.py:184-189 draws flowt with it):
 * float32 flow, element (i,y,x,ch) at flow[i*stride_n + y*stride_y + x*stride_x + ch*stride_c] for i < n, y < h, x < w, ch < 2, so an
 * NCHW tensor, an (h,w,2) tensor or a crop of either is read in place -> dst (n,h,w,3) uint8, RGB or (bgr != 0) BGR.
 * clip_flow: NaN = none, else both components clipped to [0, clip_flow] first (negative ones become 0, as np.clip(flow, 0, clip)).
 * max_flow: NaN = none: each image is normalised by its own maximum radius (needs scratch >= gimmvfi_flow_to_image_scratch_floats
 * floats); else every image by max_flow (scratch may be NULL).  The arithmetic follows numpy's float32 / float64 mix step by step. */
int64_t gimmvfi_flow_to_image_scratch_floats(int n, int h);
int gimmvfi_op_flow_to_image(const float* flow, int64_t stride_n, int64_t stride_y, int64_t stride_x, int64_t stride_c, int n, int h, int w,
                             double clip_flow, double max_flow, int bgr, float* scratch, uint8_t* dst, void* stream);
/* forward_interpolate of raft/utils/utils.py:33-63 (the same function as flowformer/core/utils/utils.py:35-65), batched: flow (n,2,h,w)
 * float32, contiguous, on the device -> out (n,2,h,w), which must not overlap flow.  Source pixel (i,j) lands at (j + dx, i + dy),
 * computed in float64; it is valid iff 0 < x < w and 0 < y < h.  Each output pixel takes the (dx, dy) of the nearest valid source, as
 * scipy.interpolate.griddata(method="nearest") does, with the squared distance rounded as numpy / scipy round it.  Ties go to the
 * smallest row-major source index (scipy's KD-tree picks among them by its traversal order).  An image without a valid source comes
 * out NaN everywhere, as from the reference.  n*h*w*h*w float64 distances; no workspace; deterministic.
 * Refuses n, h or w < 1, n > 65535, h*w >= 2^31 and overlapping buffers. */
int gimmvfi_op_forward_interpolate(const float* flow, int n, int h, int w, float* out, void* stream);
/* Scene-cut sums of n frame pairs (the content value of PySceneDetect's ContentDetector): a, b (n,h,w,3) uint8 RGB, contiguous, on the
 * device; pair i is (a[i], b[i]).  Both frames go to 8-bit HSV as cv2.cvtColor(x, COLOR_RGB2HSV) does (H in [0,180), S, V in [0,255]),
 * and sums (n,3) uint64 on the device receives (sum |H_a - H_b|, sum |S_a - S_b|, sum |V_a - V_b|) over every pixel, H not wrapped.
 * Every sum is written (the op zeroes what it accumulates into).  Integer sums: bit-exact on every run.  The score is
 * (sums[i][0] + sums[i][1] + sums[i][2]) / (3 h w).  Refuses n < 0, h or w < 1 and h*w >= 2^31. */
int gimmvfi_op_scene_sums(const uint8_t* a, const uint8_t* b, int n, int h, int w, uint64_t* sums, void* stream);
/* One output frame of a shutter blend (motion blur): dst (h,w,3) uint8, contiguous, on the device, is the mean of n sources, 1 <= n <= 63.
 * Source i is src[i], on the device: with is_f32[i] != 0, one (3,H,W) float32 row of an engine output (imgt_pred), read through the crop
 * rows pad_top .. pad_top+h-1 and columns pad_left .. pad_left+w-1, value x * 255; otherwise a contiguous (h,w,3) uint8 RGB frame, value
 * its byte.  Each channel is acc = acc + v over the sources in order in float32, then trunc(clamp(acc / n, 0, 255)), each operation rounded
 * once: n = 1 gives gimmvfi_op_pred_to_u8's bytes, and n copies of one uint8 frame give that frame.  bgr != 0 writes BGR.  One launch, no
 * allocation.  Refuses n outside [1, 63], a null pointer, h or w < 1, a crop outside H x W and H*W >= 2^31. */
int gimmvfi_op_blend_u8(const void* const* src, const int* is_f32, int n, int H, int W, int pad_top, int pad_left, uint8_t* dst, int h, int w,
                        int bgr, void* stream);
/* nn.PixelShuffle(2) applied `times` times */
int gimmvfi_op_pixel_shuffle(const gimmvfi_view* src, const gimmvfi_view* dst, int times, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GIMMVFI_B200_H_ */
