// Convolution routing: conv_plan() decides which kernel runs a ConvOp (thin 7x7, TMA-fed or register-gather wgmma, fp32 SIMT),
// launch_conv() runs it.
#include "mitb_internal.h"

namespace mitb {

ConvTrace* g_conv_trace = nullptr;
int g_conv_force_bn = 0;

// Split-K factor of the gather kernel for layers whose tile count cannot fill the SMs (deep, spatially tiny layers of the DBNet
// decoder): > 1 exactly when the layer has at most half a wave of 128 x tc_bn tiles and at least 16 K blocks.
static int splitk_splits(const ConvOp& op) {
  if (op.stat_max) return 1;
  const int sms = device_sm_count();
  const long tiles = (((long)op.in.N * op.Ho * op.Wo + 127) / 128) * (op.wt.tc_npad / op.wt.tc_bn);
  const int nkb = op.wt.tc_kpad / 64;
  if (tiles * 2 > sms || nkb < 16) return 1;
  int splits = (int)(sms / tiles);
  if (splits > nkb / 4) splits = nkb / 4;
  return splits < 1 ? 1 : splits;
}

ConvPlan conv_plan(const ConvOp& op) {
  ConvPlan pl;
  if (conv_thin_supported(op)) {
    // with an output-sparsity hint the executed work depends on the mask (device data): no flop figure is claimed for that class
    pl.kernel = CK_THIN;
    pl.sparse = op.tile_mask || op.tile_mask_u8;
    pl.prof = pl.sparse ? "conv7_thin_sparse" : "conv7_thin";
    return pl;
  }
  if (conv_tc_supported(op)) {
    // output-sparse launches (ConvOp::need_px): executed work depends on device data, so they form their own class without a flop claim
    pl.sparse = op.need_px && !op.stat_max;
    pl.prof = op.stat_max ? "conv_tc_rowstat" : pl.sparse ? "conv_tc_sparse" : "conv_tc";
    const bool fused = op.in_sv.valid() || op.out_sv.valid() || op.seg2.sv.valid();   // operand-fused ops exist only on the TMA path
    const int splits = splitk_splits(op);
    if (conv_stem8_supported(op)) pl.kernel = CK_STEM8;
    else if (conv_tma_supported(op) && (fused || splits == 1)) pl.kernel = CK_TMA;
    else { pl.kernel = splits > 1 ? CK_GATHER_SPLITK : CK_GATHER; pl.splits = splits; }
    return pl;
  }
  const bool fewout = !op.stat_max && op.out.C <= 4 && !op.in.planar && op.wt.ldw == 4;
  pl.kernel = fewout ? CK_FEWOUT : CK_SIMT;
  pl.prof = op.stat_max ? "conv_simt_rowstat" : fewout ? "conv_fewout" : "conv_simt";
  return pl;
}

// The drivers fuse operands only for Cout > 4: a fusion policy, not a routing rule.
bool conv_uses_tma(const ConvOp& op) { return op.out.C > 4 && conv_plan(op).kernel == CK_TMA; }
bool conv_tma_capable(const ConvOp& op) { return op.out.C > 4 && conv_tc_supported(op) && conv_tma_supported(op); }

// the layout of the kernel that runs this op's row-stat launch (stat_max set): two column halves per N tile on the tensor cores
int conv_stat_blocks(const ConvOp& op) {
  ConvOp rs = op;
  float probe; rs.stat_max = &probe;                  // planned, never launched
  return conv_plan(rs).kernel == CK_SIMT ? (op.out.C + 127) / 128 : 2 * (op.wt.tc_npad / op.wt.tc_bn);
}

void launch_conv(const ConvOp& op, cudaStream_t st) {
  const ConvW& w = op.wt;
  MITB_CHECK(w.ntaps >= 1 && w.ntaps <= kMaxTaps, "bad tap count %d", w.ntaps);
  MITB_CHECK(op.in.N == op.out.N, "batch mismatch");
  MITB_CHECK(w.ldw % 4 == 0 && w.ldw >= op.out.C, "bad ldw %d for Cout %d", w.ldw, op.out.C);
  if (op.in.planar) {
    MITB_CHECK(w.ntaps == 1 && op.sy == 1 && op.sx == 1 && w.tdy[0] == 0 && w.tdx[0] == 0 &&
               op.Ho == op.in.H && op.Wo == op.in.W, "planar input supports 1x1 convs only");
  } else {
    MITB_CHECK(op.in.C % 4 == 0 && op.in.cs % 4 == 0 && op.in.coff % 4 == 0,
               "NHWC conv input needs channel counts/offsets in multiples of 4 (C=%d cs=%d off=%d)", op.in.C, op.in.cs, op.in.coff);
  }
  if (op.pad == PAD_REFLECT) {
    for (int t = 0; t < w.ntaps; ++t)
      MITB_CHECK(-w.tdy[t] < op.in.H && -w.tdx[t] < op.in.W, "reflect padding wider than the image");
  }
  const int M = op.in.N * op.Ho * op.Wo, Cout = op.out.C;
  if (M == 0) return;
  const ConvPlan plan = conv_plan(op);
  MITB_CHECK(plan.kernel == CK_TMA || plan.kernel == CK_STEM8 || (!op.in_sv.valid() && !op.out_sv.valid() && !op.seg2.sv.valid()),
             "conv: operand-fused ops must run on the TMA path");
  // algorithmic work of this launch: 2*M*K*Cout flops; bytes = input view + weights + output (+ fused residual reads)
  const int K = w.ntaps * op.in.C + (op.seg2.sv.valid() ? op.seg2.ntaps * op.seg2.C : 0);   // + second K segment of an operand-fused launch
  const double flops = 2.0 * M * (double)K * Cout;
  const double bytes = 4.0 * ((double)op.in.pixels() * op.in.C + (op.seg2.sv.valid() ? (double)op.in.pixels() * op.seg2.C : 0.0) + (double)K * Cout +
                              (double)M * Cout * ((op.stat_max ? 0 : 1) + (op.add0.p ? 1 : 0) + (op.add1.p ? 1 : 0)));
  // the per-launch shape list of the profiler (MITB_PROFILE_LAUNCHES) covers the tensor-core and thin kernels
  const bool shape = plan.kernel != CK_SIMT && plan.kernel != CK_FEWOUT;
  ProfScope ps(plan.prof, plan.sparse ? 0.0 : flops, plan.sparse ? 0.0 : bytes, st, shape ? M : 0, shape ? K : 0, shape ? Cout : 0);
  switch (plan.kernel) {
    case CK_THIN: launch_conv_thin(op, st); break;
    case CK_STEM8: case CK_TMA: launch_conv_tma(op, plan.kernel == CK_STEM8, st); break;
    case CK_GATHER: case CK_GATHER_SPLITK: launch_conv_tc(op, plan.splits, st); break;
    default: launch_conv_simt(op, plan.kernel == CK_FEWOUT, st); break;
  }
}

}  // namespace mitb
