// Test hooks of include/mitb.h (not for production use): one fully described convolution through launch_conv(), so that tests
// can reach every option of the fused conv epilogue (ConvOp in mitb_internal.h) on every kernel path and compare it with an
// independent reference, and the OCR's vocabulary head (GEMM + fused log-softmax / argmax) with its row-stat partials.  Host
// code only: the kernels are the ones the networks run.
#include <stddef.h>
#include <string.h>
#include "exec.h"

using namespace mitb;

struct mitb_ctx { Ctx c; };

// the offsets the header states ("@N") for the Python mirror
static_assert(sizeof(mitb_test_view) == 24 && sizeof(mitb_test_split) == 40, "test hook struct layout");
static_assert(offsetof(mitb_test_conv_desc, N) == 8 && offsetof(mitb_test_conv_desc, in_scale) == 40 && offsetof(mitb_test_conv_desc, wt) == 56 &&
              offsetof(mitb_test_conv_desc, cout) == 64 && offsetof(mitb_test_conv_desc, scale) == 96 && offsetof(mitb_test_conv_desc, act) == 120 &&
              offsetof(mitb_test_conv_desc, add0) == 128 && offsetof(mitb_test_conv_desc, add1) == 152 && offsetof(mitb_test_conv_desc, out) == 176 &&
              offsetof(mitb_test_conv_desc, out_H) == 184 && offsetof(mitb_test_conv_desc, out_sv) == 224 &&
              offsetof(mitb_test_conv_desc, os_scale) == 264 && offsetof(mitb_test_conv_desc, os_relu) == 280 &&
              offsetof(mitb_test_conv_desc, in_sv) == 288 && offsetof(mitb_test_conv_desc, seg2) == 328 &&
              offsetof(mitb_test_conv_desc, seg2_wt) == 368 && offsetof(mitb_test_conv_desc, seg2_cin) == 376 &&
              offsetof(mitb_test_conv_desc, need_px) == 400 && offsetof(mitb_test_conv_desc, path) == 408 && sizeof(mitb_test_conv_desc) == 416,
              "test hook descriptor layout");
static_assert(offsetof(mitb_test_conv_info, bn) == 4 && offsetof(mitb_test_conv_info, splits) == 8 && offsetof(mitb_test_conv_info, vec2) == 12 &&
              offsetof(mitb_test_conv_info, tma_act) == 16 && offsetof(mitb_test_conv_info, split_reused) == 20 &&
              offsetof(mitb_test_conv_info, convs) == 24 && offsetof(mitb_test_conv_info, staged) == 28 &&
              offsetof(mitb_test_conv_info, epi_sig) == 32 && sizeof(mitb_test_conv_info) == 36, "test hook info layout");

namespace {

// restores the process-wide kernel switches and the trace / N tile overrides, also when the conv throws
struct HookGuard {
  bool tc = conv_tc_enabled(), tma = conv_tma_enabled();
  ~HookGuard() { conv_tc_set_enabled(tc); conv_tma_set_enabled(tma); g_conv_trace = nullptr; g_conv_force_bn = 0; }
};

// the process-wide kernel switches of a MITB_TEST_PATH_*
void set_path(int path) {
  if (path == MITB_TEST_PATH_SIMT) conv_tc_set_enabled(false);
  if (path == MITB_TEST_PATH_GATHER) conv_tma_set_enabled(false);
  if (path == MITB_TEST_PATH_TMA || path == MITB_TEST_PATH_AUTO) { conv_tc_set_enabled(true); conv_tma_set_enabled(true); }
}

void fill_info(mitb_test_conv_info* info, const ConvTrace& tr) {
  memset(info, 0, sizeof(*info));
  info->kernel = tr.kernel; info->bn = tr.bn; info->splits = tr.splits; info->vec2 = tr.vec2; info->tma_act = tr.tma_act;
  info->split_reused = tr.split_reused; info->convs = tr.convs; info->staged = tr.staged; info->epi_sig = tr.epi_sig;
}

void check_align(const void* p, unsigned a, const char* what) {
  MITB_CHECK(((uintptr_t)p & (a - 1)) == 0, "test_conv: %s must be %u-byte aligned (unaligned slices go through cs / coff)", what, a);
}

View residual(const mitb_test_view& r, int N, int H, int W, int C) {
  View v;
  if (!r.p) return v;
  v.p = (float*)r.p; v.N = N; v.H = H; v.W = W; v.C = C; v.cs = r.cs; v.coff = r.coff; v.planar = r.planar != 0;
  MITB_CHECK(r.cs > 0 && r.coff >= 0 && r.coff + C <= r.cs, "test_conv: residual slice [%d, %d) outside cs %d", r.coff, r.coff + C, r.cs);
  return v;
}

SplitView split(const mitb_test_split& s, int N, int H, int W, int C) {
  SplitView v;
  if (!s.hi) return v;
  MITB_CHECK(s.mid && s.pt >= 0 && s.pl >= 0 && s.Hp >= H + s.pt && s.Wp >= W + s.pl && s.coff >= 0 && s.coff + C <= s.C,
             "test_conv: split tensor does not hold the slice");
  v.hi = s.hi; v.mid = s.mid; v.N = N; v.H = H; v.W = W; v.C = s.C; v.pt = s.pt; v.pl = s.pl; v.Hp = s.Hp; v.Wp = s.Wp;
  return v;
}

}  // namespace

extern "C" {

int mitb_test_struct_sizes(int* desc_bytes, int* info_bytes) {
  if (desc_bytes) *desc_bytes = (int)sizeof(mitb_test_conv_desc);
  if (info_bytes) *info_bytes = (int)sizeof(mitb_test_conv_info);
  return 0;
}

int mitb_test_conv(mitb_ctx* ctx, const mitb_test_conv_desc* d, mitb_test_conv_info* info, void* stream) {
  if (!ctx) return 1;
  HookGuard guard;
  try {
    CUDA_OK(cudaSetDevice(ctx->c.device));
    MITB_CHECK(d && info, "test_conv: null descriptor or info");
    cudaStream_t st = (cudaStream_t)stream;
    const bool fused = d->in_sv.hi || d->out_sv.hi || d->seg2.hi;
    MITB_CHECK(d->path >= MITB_TEST_PATH_AUTO && d->path <= MITB_TEST_PATH_TMA, "test_conv: bad path %d", d->path);
    MITB_CHECK(d->N > 0 && d->H > 0 && d->W > 0 && d->C > 0 && d->cout > 0 && d->kh > 0 && d->kw > 0 && d->stride > 0, "test_conv: bad shape");
    MITB_CHECK(d->wt && d->wt_cin > 0 && d->wt_cin <= d->C, "test_conv: weights need 1..C input channels");
    MITB_CHECK(d->x || d->in_sv.hi, "test_conv: no input");
    MITB_CHECK(d->out || d->out_sv.hi, "test_conv: no output");
    MITB_CHECK(d->act >= ACT_NONE && d->act <= ACT_CLAMP01, "test_conv: bad activation %d", d->act);
    MITB_CHECK(!fused || d->path == MITB_TEST_PATH_AUTO || d->path == MITB_TEST_PATH_TMA, "test_conv: in_sv / out_sv / seg2 exist only on the TMA path");
    const void* al16[] = {d->x, d->in_scale, d->in_shift, d->add0.p, d->add1.p, d->out, d->out_sv.hi, d->out_sv.mid, d->in_sv.hi, d->in_sv.mid,
                          d->seg2.hi, d->seg2.mid};
    const char* al16_name[] = {"x", "in_scale", "in_shift", "add0", "add1", "out", "out_sv.hi", "out_sv.mid", "in_sv.hi", "in_sv.mid", "seg2.hi", "seg2.mid"};
    for (int i = 0; i < 12; ++i) check_align(al16[i], 16, al16_name[i]);
    const void* al4[] = {d->scale, d->shift, d->mul1, d->os_scale, d->os_shift};
    const char* al4_name[] = {"scale", "shift", "mul1", "os_scale", "os_shift"};
    for (int i = 0; i < 5; ++i) check_align(al4[i], 4, al4_name[i]);

    const int Ho = (d->H + 2 * d->pad_y - d->kh) / d->stride + 1, Wo = (d->W + 2 * d->pad_x - d->kw) / d->stride + 1;
    MITB_CHECK(Ho > 0 && Wo > 0, "test_conv: empty output");
    const int oy_mul = d->oy_mul ? d->oy_mul : 1, ox_mul = d->ox_mul ? d->ox_mul : 1;
    const int out_H = d->out_H ? d->out_H : Ho, out_W = d->out_W ? d->out_W : Wo;
    MITB_CHECK(d->oy_add >= 0 && d->ox_add >= 0 && (Ho - 1) * oy_mul + d->oy_add < out_H && (Wo - 1) * ox_mul + d->ox_add < out_W,
               "test_conv: output grid %dx%d too small for the logical grid %dx%d", out_H, out_W, Ho, Wo);

    // weights as mitb_op_conv2d loads them; the tap offsets follow pad_y / pad_x
    DevBlob blob;
    Weights W;
    W.t["w"] = mitb_tensor{"w", d->wt, 4, {d->cout, d->wt_cin, d->kh, d->kw}};
    if (d->seg2.hi) {
      MITB_CHECK(d->seg2_wt && d->seg2_cin > 0 && d->seg2_kh > 0 && d->seg2_kw > 0, "test_conv: seg2 needs weights");
      W.t["w2"] = mitb_tensor{"w2", d->seg2_wt, 4, {d->cout, d->seg2_cin, d->seg2_kh, d->seg2_kw}};
    }
    Loader L{W, blob, st};
    ConvW cw = L.conv_padcin("w", 0, d->C);
    for (int t = 0; t < cw.ntaps; ++t) { cw.tdy[t] = (int8_t)(t / d->kw - d->pad_y); cw.tdx[t] = (int8_t)(t % d->kw - d->pad_x); }
    ConvW w2, cat;                        // FFC's layout (lama.cu): one tensor-core weight whose K rows are segment 1's followed by segment 2's
    if (d->seg2.hi) {
      w2 = L.conv_padcin("w2", 0, d->seg2_cin);
      for (int t = 0; t < w2.ntaps; ++t) { w2.tdy[t] = (int8_t)(t / d->seg2_kw - d->seg2_pad); w2.tdx[t] = (int8_t)(t % d->seg2_kw - d->seg2_pad); }
      cat = L.cat_k(cw, w2);
    }

    View in; in.p = const_cast<float*>(d->x); in.N = d->N; in.H = d->H; in.W = d->W; in.C = d->C;
    in.cs = d->x ? d->cs : d->C; in.coff = d->x ? d->coff : 0; in.planar = d->planar != 0;
    MITB_CHECK(!d->x || (d->cs > 0 && d->coff >= 0 && d->coff + d->C <= d->cs), "test_conv: input slice outside cs");
    View out; out.p = d->out; out.N = d->N; out.H = out_H; out.W = out_W; out.C = d->cout;
    out.cs = d->out ? d->out_cs : d->cout; out.coff = d->out ? d->out_coff : 0; out.planar = d->out_planar != 0;
    MITB_CHECK(!d->out || (d->out_cs > 0 && d->out_coff >= 0 && d->out_coff + d->cout <= d->out_cs), "test_conv: output slice outside cs");

    const int pad_mode = d->pad_mode == 1 ? PAD_REFLECT : PAD_ZERO;
    ConvOp op = d->seg2.hi ? Exec::op_from2(cw, w2, cat, in, out, d->stride, pad_mode) : Exec::op_from(cw, in, out, d->stride, pad_mode);
    op.Ho = Ho; op.Wo = Wo; op.oy_mul = oy_mul; op.oy_add = d->oy_add; op.ox_mul = ox_mul; op.ox_add = d->ox_add;
    op.in_scale = d->in_scale; op.in_shift = d->in_shift; op.in_relu = d->in_relu;
    MITB_CHECK(!op.in_scale == !op.in_shift, "test_conv: in_scale and in_shift go together");
    op.scale = d->scale; op.shift = d->shift; op.mul1 = d->mul1; op.act = d->act;
    op.add0 = residual(d->add0, d->N, out_H, out_W, d->cout);
    op.add1 = residual(d->add1, d->N, out_H, out_W, d->cout);
    op.need_px = d->need_px;
    if (d->out_sv.hi) {
      op.out_sv = split(d->out_sv, d->N, Ho, Wo, d->cout); op.out_sv_coff = d->out_sv.coff;
      op.os_scale = d->os_scale; op.os_shift = d->os_shift; op.os_relu = d->os_relu;
      MITB_CHECK(!op.os_scale == !op.os_shift, "test_conv: os_scale and os_shift go together");
    }
    if (d->in_sv.hi) { op.in_sv = split(d->in_sv, d->N, d->H, d->W, d->C); op.in_sv_coff = d->in_sv.coff; }
    if (d->seg2.hi) {
      op.seg2.sv = split(d->seg2, d->N, Ho, Wo, d->seg2_cin); op.seg2.coff = d->seg2.coff; op.seg2.pad = d->seg2_pad_mode == 1 ? PAD_REFLECT : PAD_ZERO;
    }
    // a fused op on any other kernel would dereference the shape-only views
    MITB_CHECK(!fused || conv_tma_capable(op), "test_conv: this op cannot run on the TMA-fed kernel");

    set_path(d->path);
    ConvTrace tr;
    g_conv_trace = &tr; g_conv_force_bn = d->force_bn;
    CUDA_OK(cudaStreamSynchronize(st));                     // weight copies ready
    ++g_launch_epoch;                                       // a new call: the host may have rewritten the input since the last one
    const int runs = d->runs > 0 ? d->runs : 1;
    for (int r = 0; r < runs; ++r) launch_conv(op, st);
    CUDA_OK(cudaStreamSynchronize(st));
    const bool on_tma = tr.kernel == CK_TMA || tr.kernel == CK_STEM8;
    MITB_CHECK(d->path != MITB_TEST_PATH_TMA || on_tma, "test_conv: the op did not run on the TMA-fed kernel (kernel %d)", tr.kernel);
    MITB_CHECK(!d->force_bn || on_tma, "test_conv: force_bn needs the TMA-fed kernel (kernel %d)", tr.kernel);
    fill_info(info, tr);
    return 0;
  } catch (const std::exception& ex) {
    ctx->c.err = ex.what();
    cudaGetLastError();
    return 2;
  }
}

int mitb_test_vocab_head(mitb_ctx* ctx, const float* x, int n, int t, int c, const float* wt, const float* bias, int v, int path,
                         int32_t* idx, float* logprob, float* pmax, float* psum, int32_t* pidx, long long cap, int32_t* nblk,
                         mitb_test_conv_info* info, void* stream) {
  if (!ctx) return 1;
  HookGuard guard;
  try {
    CUDA_OK(cudaSetDevice(ctx->c.device));
    cudaStream_t st = (cudaStream_t)stream;
    MITB_CHECK(path >= MITB_TEST_PATH_AUTO && path <= MITB_TEST_PATH_TMA, "test_vocab_head: bad path %d", path);
    MITB_CHECK(n > 0 && t > 0 && c > 0 && c % 4 == 0 && v > 0, "test_vocab_head: bad shape");
    MITB_CHECK(x && wt && idx && logprob && nblk && info, "test_vocab_head: null buffer");
    MITB_CHECK(!pmax == !psum && !pmax == !pidx, "test_vocab_head: pmax, psum and pidx go together");
    check_align(x, 16, "x");

    // char_pred as ocr_build loads it
    DevBlob blob;
    Weights W;
    W.t["w"] = mitb_tensor{"w", wt, 2, {v, c}};
    if (bias) W.t["b"] = mitb_tensor{"b", bias, 1, {v}};
    Loader L{W, blob, st};
    ConvW cw = L.conv("w", 0, 0);
    if (bias) cw.shift = L.vec("b");

    // the op as ocr_run makes it, its stat layout read after the path switches are set
    View in; in.p = const_cast<float*>(x); in.N = n; in.H = 1; in.W = t; in.C = c; in.cs = c; in.coff = 0;
    View out = in; out.p = nullptr; out.C = v; out.cs = v;
    ConvOp op = Exec::op_from(cw, in, out);
    set_path(path);
    const int nb = conv_stat_blocks(op);
    const long long need = (long long)n * t * nb;
    if (pmax) MITB_CHECK(cap >= need, "test_vocab_head: partials need %lld elements, cap %lld", need, cap);
    else { pmax = blob.alloc_f(need); psum = blob.alloc_f(need); pidx = (int32_t*)blob.alloc_f(need); }
    op.stat_max = pmax; op.stat_sum = psum; op.stat_idx = pidx; op.stat_ld = nb;

    ConvTrace tr;
    g_conv_trace = &tr;
    CUDA_OK(cudaStreamSynchronize(st));                     // weight copies ready
    ++g_launch_epoch;
    launch_conv(op, st);
    launch_rowstat_final(pmax, psum, pidx, n * t, nb, idx, logprob, st);
    CUDA_OK(cudaStreamSynchronize(st));
    const bool on_tma = tr.kernel == CK_TMA;
    MITB_CHECK(path != MITB_TEST_PATH_TMA || on_tma, "test_vocab_head: the op did not run on the TMA-fed kernel (kernel %d)", tr.kernel);
    fill_info(info, tr);
    *nblk = nb;
    return 0;
  } catch (const std::exception& ex) {
    ctx->c.err = ex.what();
    cudaGetLastError();
    return 2;
  }
}

int mitb_set_epi_specialise(int on) {
  const int prev = epi_specialise() ? 1 : 0;
  g_epi_specialise = on ? 1 : 0;
  return prev;
}

int mitb_test_epi_signature(int act, int sig) { return staged_epi_sig(act, sig); }

int mitb_test_epi_signatures(int* act, int* sig, int cap) { return epi_sig_list(act, sig, cap); }

}  // extern "C"
