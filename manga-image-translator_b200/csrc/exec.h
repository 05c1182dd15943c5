// Shared by the three network drivers: an executor that either sizes the workspace (dry run) or launches.
#pragma once
#include "mitb_internal.h"

namespace mitb {

struct Exec {
  Ctx& ctx; cudaStream_t st; bool dry;
  Arena& ws() { return ctx.ws; }

  static ConvOp op_from(const ConvW& w, const View& in, const View& out, int stride = 1, int pad_mode = PAD_ZERO) {
    MITB_CHECK(in.C == w.Cin, "conv: input has %d channels, weight expects %d", in.C, w.Cin);
    MITB_CHECK(out.C == w.Cout, "conv: output has %d channels, weight produces %d", out.C, w.Cout);
    ConvOp op; op.in = in; op.out = out; op.wt = w;
    op.sy = op.sx = stride; op.pad = pad_mode; op.Ho = out.H; op.Wo = out.W;
    op.scale = w.scale; op.shift = w.shift;
    return op;
  }
  // Two K segments accumulated by one launch (FFC: conv1x1(U) + conv3x3_{l->g}(x_l)): segment 1 is `a` over `in`, segment 2 is `b`
  // over a pre-split tensor the caller sets in seg2 (sv, coff, pad), and ab = Loader::cat_k(a, b) holds the tensor-core weights of
  // both.  The epilogue's scale / shift are a's.
  static ConvOp op_from2(const ConvW& a, const ConvW& b, const ConvW& ab, const View& in, const View& out, int stride = 1,
                         int pad_mode = PAD_ZERO) {
    MITB_CHECK(ab.Cout == a.Cout && ab.Cin == a.ntaps * a.Cin + b.ntaps * b.Cin, "conv: merged weight does not hold both K segments");
    ConvOp op = op_from(a, in, out, stride, pad_mode);
    op.wt = ab;                          // K rows a's then b's: segment 1 keeps a's channels and taps
    op.wt.Cin = a.Cin; op.wt.ntaps = a.ntaps;
    for (int t = 0; t < a.ntaps; ++t) { op.wt.tdy[t] = a.tdy[t]; op.wt.tdx[t] = a.tdx[t]; }
    op.seg2.C = b.Cin; op.seg2.ntaps = b.ntaps;
    for (int t = 0; t < b.ntaps; ++t) { op.seg2.tdy[t] = b.tdy[t]; op.seg2.tdx[t] = b.tdx[t]; }
    return op;
  }
  void conv(const ConvOp& op) { if (!dry) launch_conv(op, st); }
  // stride-2 transposed conv given its 4 phase kernels; `tune` edits the epilogue of each phase op
  template <class F>
  void convT2(const ConvW* phases, const View& in, const View& out, F tune) {
    MITB_CHECK(out.H == 2 * in.H && out.W == 2 * in.W, "transposed conv expects a 2x output grid");
    for (int ph = 0; ph < 4; ++ph) {
      ConvOp op = op_from(phases[ph], in, out);
      op.Ho = in.H; op.Wo = in.W; op.oy_mul = 2; op.ox_mul = 2; op.oy_add = ph >> 1; op.ox_add = ph & 1;
      tune(op);
      conv(op);
    }
  }
  void layernorm(const View& in, const View& out, const float* w, const float* b, float eps, const float* pe = nullptr,
                 const View* out2 = nullptr, int T = 1, const SplitView* osv = nullptr) { if (!dry) launch_layernorm(in, out, w, b, eps, pe, out2, T, st, osv); }
  void dwconv7_ln(const View& in, const View& out, const float* wdw, const float* bdw, const float* lnw, const float* lnb,
                  float eps, const SplitView* osv = nullptr) { if (!dry) launch_dwconv7_ln(in, out, wdw, bdw, lnw, lnb, eps, st, osv); }
  // bf16 hi/mid operand tensor living in the bytes of a dense fp32 view of the same shape (2 x 2 bytes per element)
  static SplitView alias_split(const View& v) {
    SplitView s; s.N = v.N; s.H = s.Hp = v.H; s.W = s.Wp = v.W; s.C = v.C;
    s.hi = reinterpret_cast<uint16_t*>(v.p); s.mid = s.hi + s.elems();
    return s;
  }
  void avgpool(const View& in, const View& out, int mode) { if (!dry) launch_avgpool(in, out, mode, st); }
};

// Runs `body` twice: once dry to size the activation workspace, then for real.
template <class F>
void run_with_workspace(Ctx& ctx, cudaStream_t st, F body) {
  Arena& ws = ctx.ws;
  ws.dry = true; ws.off = 0; ws.peak = 0;
  { Exec e{ctx, st, true}; body(e); }
  const size_t need = ws.peak;
  ws.dry = false; ws.off = 0;
  ctx.ensure_ws(need);
  ws.peak = 0;
  g_launch_counter = &ctx.launches; g_prof = &ctx.prof; ++g_launch_epoch;   /* new API call: inputs may have been rewritten by the host */
  { Exec e{ctx, st, false}; body(e); }
  g_launch_counter = nullptr; g_prof = nullptr;
}

}  // namespace mitb
