// Net: the layer helpers Engine::run() and the FlowFormer estimator (flowformer.cu) build their forward passes from: a convolution is
// looked up by its state_dict name in the packed-weight table and dispatched by conv2d() (tensor-core / CUDA-core, common.h).
#pragma once
#include "engine.h"

namespace gv {

struct Net {
  Engine& E; Ctx& cx;
  const ConvW& W(const std::string& n) const {
    auto it = E.conv_.find(n);
    if (it == E.conv_.end()) throw std::runtime_error("gimmvfi: conv '" + n + "' not packed");
    return it->second;
  }
  const float* V(const std::string& n) const { return E.vec_.at(n); }
  static ConvGeom geom(const ConvW& w, int stride = 1, bool reflect = false) {
    ConvGeom g; g.stride = stride; g.ph = w.kh / 2; g.pw = w.kw / 2; g.reflect = reflect ? 1 : 0; return g;
  }
  // plain conv + activation
  void conv(const std::string& name, const TV& in, const TV& out, int act = ACT_NONE, const float* slope = nullptr, int stride = 1,
            bool reflect = false) {
    ConvEpi e; e.act1 = act; e.slope1 = slope;
    conv_e(name, in, TV(), out, e, stride, reflect);
  }
  void conv_e(const std::string& name, const TV& in0, const TV& in1, const TV& out, const ConvEpi& e, int stride = 1, bool reflect = false) {
    const ConvW& w = W(name);
    if (reflect && cx.tc && !in1.p && stride == 1 && w.w_tc && in0.ld % (in0.f16 ? 8 : 4) == 0 && (!in0.f16 || w.w_tc_h)) {
      // the TMA path can only zero-fill: materialise the reflect padding once, then a "valid" conv on the padded buffer
      Arena& A = cx.arena;
      const size_t mk = A.mark();
      TV pad = in0.f16 ? A.tensor_h(in0.n, in0.h + 2 * (w.kh / 2), in0.w + 2 * (w.kw / 2), in0.c)
                       : A.tensor(in0.n, in0.h + 2 * (w.kh / 2), in0.w + 2 * (w.kw / 2), in0.c, (in0.c + 3) & ~3);
      pad_reflect(cx, in0, pad, w.kh / 2);
      ConvGeom g; g.stride = 1; g.ph = 0; g.pw = 0; g.loose_w = 1;
      conv2d(cx, pad, TV(), w, g, e, out);
      A.release(mk);
      return;
    }
    conv2d(cx, in0, in1, w, geom(w, stride, reflect), e, out);
  }
  // 7x7 conv on few channels through the x-packed weights: zero-padded copy of `in`, then a (7 x 1) conv over 7*ldp lanes
  void conv7x(const std::string& name, const TV& in, const TV& out, int act = ACT_NONE, const float* slope = nullptr) {
    if (conv7x7_small_cout(cx, in, W(name), act, slope, out)) return;   // <= 4 output channels: exact fp32 shared-memory kernel (conv.cu)
    const ConvW& w = W(name + "#xp");
    const int k = w.kh, ldp = w.cin / k;   // (k x k kernel packed as k x 1 over k * ldp lanes)
    Arena& A = cx.arena;
    const size_t mk = A.mark();
    TV pad = A.tensor(in.n, in.h + 2 * (k / 2), in.w + 2 * (k / 2), ldp, ldp);
    pad_zero(cx, in, pad, k / 2);
    TV v = pad; v.c = w.cin;
    ConvGeom g; g.stride = 1; g.ph = 0; g.pw = 0; g.loose_w = 1;
    ConvEpi e; e.act1 = act; e.slope1 = slope;
    conv2d(cx, v, TV(), w, g, e, out);
    A.release(mk);
  }
  // Sequential(Conv2d, PReLU)  (fi_components.py:32-54)
  void convrelu(const std::string& name, const TV& in, const TV& out) { conv(name + ".0", in, out, ACT_PRELU, V(name + ".1.weight")); }
};

}  // namespace gv
