// extern "C" boundary of libmitb (see include/mitb.h).  Exceptions never cross it: every entry point converts them
// to a non-zero return code + mitb_last_error().
#include <string.h>
#include "exec.h"

using namespace mitb;

struct mitb_ctx { Ctx c; };

namespace mitb { void launch_bilateral17(const uint8_t* img, int h, int w, uint8_t* out, cudaStream_t st); }

static thread_local std::string g_create_error;

#define API_BEGIN(ctx)                                                     \
  if (!(ctx)) return 1;                                                    \
  try {                                                                    \
    CUDA_OK(cudaSetDevice((ctx)->c.device));
#define API_END(ctx)                                                       \
    return 0;                                                              \
  } catch (const std::exception& ex) {                                     \
    (ctx)->c.err = ex.what(); g_launch_counter = nullptr; g_prof = nullptr;                  \
    (ctx)->c.ws.dry = false;                                               \
    cudaGetLastError();                                                    \
    return 2;                                                              \
  }

static Weights collect(const mitb_tensor* w, int n) {
  Weights W;
  MITB_CHECK(w && n > 0, "empty weight list");
  for (int i = 0; i < n; ++i) {
    MITB_CHECK(w[i].name && w[i].data && w[i].ndim >= 0 && w[i].ndim <= 4, "weight %d is malformed", i);
    W.t[w[i].name] = w[i];
  }
  return W;
}

extern "C" {

const char* mitb_version(void) { return "mitb-b200 0.1 (sm_90a)"; }

int mitb_create(int device, mitb_ctx** out) {
  if (!out) return 1;
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) { g_create_error = "mitb_create: no CUDA device available (there is no CPU fallback)"; cudaGetLastError(); return 3; }
  if (device < 0 || device >= count) { g_create_error = "mitb_create: bad device ordinal"; return 3; }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { g_create_error = "mitb_create: cudaGetDeviceProperties failed"; return 3; }
  // the kernels are built for sm_90a only (wgmma, TMA): anything else cannot load them
  if (prop.major != 9 || prop.minor != 0) { g_create_error = std::string("mitb_create: ") + prop.name + " is not a Hopper (sm_90a) device"; return 3; }
  mitb_ctx* c = new mitb_ctx();
  c->c.device = device;
  *out = c;
  return 0;
}

void mitb_destroy(mitb_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->c.device);
  cudaDeviceSynchronize();
  if (ctx->c.dbnet) dbnet_free(ctx->c.dbnet);
  if (ctx->c.dbnet_r34) dbnet_r34_free(ctx->c.dbnet_r34);
  if (ctx->c.ocr) ocr_free(ctx->c.ocr);
  if (ctx->c.lama) lama_free(ctx->c.lama);
  if (ctx->c.ws.base) cudaFree(ctx->c.ws.base);
  delete ctx;
}

const char* mitb_last_error(const mitb_ctx* ctx) { return ctx ? ctx->c.err.c_str() : g_create_error.c_str(); }
long long mitb_launch_count(const mitb_ctx* ctx) { return ctx ? ctx->c.launches : 0; }
size_t mitb_workspace_bytes(const mitb_ctx* ctx) { return ctx ? ctx->c.ws.cap : 0; }

int mitb_set_tensor_cores(int on) { conv_tc_set_enabled(on != 0); return 0; }
int mitb_set_ffc_mode(int mode) { lama_set_ffc_mode(mode); return 0; }
int mitb_set_sparse_decoder(int on) { lama_set_sparse_decoder(on); return 0; }

int mitb_profile_enable(mitb_ctx* ctx, int on) {
  API_BEGIN(ctx)
  ctx->c.prof.on = on != 0;
  API_END(ctx)
}
const char* mitb_profile_report(mitb_ctx* ctx) {
  if (!ctx) return "{}";
  cudaSetDevice(ctx->c.device);
  ctx->c.prof_json = profiler_report(ctx->c.prof);
  return ctx->c.prof_json.c_str();
}

int mitb_dbnet_load(mitb_ctx* ctx, const mitb_tensor* w, int n) {
  API_BEGIN(ctx)
  if (ctx->c.dbnet) { dbnet_free(ctx->c.dbnet); ctx->c.dbnet = nullptr; }
  Weights W = collect(w, n);
  ctx->c.dbnet = dbnet_build(ctx->c, W);
  API_END(ctx)
}
int mitb_dbnet_unload(mitb_ctx* ctx) {
  API_BEGIN(ctx)
  CUDA_OK(cudaDeviceSynchronize());
  if (ctx->c.dbnet) { dbnet_free(ctx->c.dbnet); ctx->c.dbnet = nullptr; }
  API_END(ctx)
}
int mitb_dbnet_forward(mitb_ctx* ctx, const float* x, int n, int h, int w, float* db, float* mask, void* stream) {
  API_BEGIN(ctx)
  MITB_CHECK(ctx->c.dbnet, "dbnet: forward before load");
  MITB_CHECK(x && db && mask, "dbnet: null buffer");
  dbnet_run(ctx->c, *ctx->c.dbnet, x, nullptr, n, h, w, db, mask, (cudaStream_t)stream);
  API_END(ctx)
}
int mitb_dbnet_forward_u8(mitb_ctx* ctx, const uint8_t* img, int n, int h, int w, float* db, float* mask, void* stream) {
  API_BEGIN(ctx)
  MITB_CHECK(ctx->c.dbnet, "dbnet: forward before load");
  MITB_CHECK(img && db && mask, "dbnet: null buffer");
  dbnet_run(ctx->c, *ctx->c.dbnet, nullptr, img, n, h, w, db, mask, (cudaStream_t)stream);
  API_END(ctx)
}

int mitb_dbnet_r34_load(mitb_ctx* ctx, const mitb_tensor* w, int n) {
  API_BEGIN(ctx)
  if (ctx->c.dbnet_r34) { dbnet_r34_free(ctx->c.dbnet_r34); ctx->c.dbnet_r34 = nullptr; }
  Weights W = collect(w, n);
  ctx->c.dbnet_r34 = dbnet_r34_build(ctx->c, W);
  API_END(ctx)
}
int mitb_dbnet_r34_unload(mitb_ctx* ctx) {
  API_BEGIN(ctx)
  CUDA_OK(cudaDeviceSynchronize());
  if (ctx->c.dbnet_r34) { dbnet_r34_free(ctx->c.dbnet_r34); ctx->c.dbnet_r34 = nullptr; }
  API_END(ctx)
}
int mitb_dbnet_r34_forward(mitb_ctx* ctx, const float* x, int n, int h, int w, float* db, float* mask, void* stream) {
  API_BEGIN(ctx)
  MITB_CHECK(ctx->c.dbnet_r34, "dbnet_r34: forward before load");
  MITB_CHECK(x && db && mask, "dbnet_r34: null buffer");
  dbnet_r34_run(ctx->c, *ctx->c.dbnet_r34, x, nullptr, n, h, w, db, mask, (cudaStream_t)stream);
  API_END(ctx)
}
int mitb_dbnet_r34_forward_u8(mitb_ctx* ctx, const uint8_t* img, int n, int h, int w, float* db, float* mask, void* stream) {
  API_BEGIN(ctx)
  MITB_CHECK(ctx->c.dbnet_r34, "dbnet_r34: forward before load");
  MITB_CHECK(img && db && mask, "dbnet_r34: null buffer");
  dbnet_r34_run(ctx->c, *ctx->c.dbnet_r34, nullptr, img, n, h, w, db, mask, (cudaStream_t)stream);
  API_END(ctx)
}

int mitb_ocr_load(mitb_ctx* ctx, const mitb_tensor* w, int n) {
  API_BEGIN(ctx)
  if (ctx->c.ocr) { ocr_free(ctx->c.ocr); ctx->c.ocr = nullptr; }
  Weights W = collect(w, n);
  ctx->c.ocr = ocr_build(ctx->c, W);
  API_END(ctx)
}
int mitb_ocr_unload(mitb_ctx* ctx) {
  API_BEGIN(ctx)
  CUDA_OK(cudaDeviceSynchronize());
  if (ctx->c.ocr) { ocr_free(ctx->c.ocr); ctx->c.ocr = nullptr; }
  API_END(ctx)
}
int mitb_ocr_timesteps(int wp) { return (wp / 2) / 2 - 1; }
int mitb_ocr_forward(mitb_ctx* ctx, const float* x, int n, int wp, int32_t* argmax, float* logprob, float* colors, void* stream) {
  API_BEGIN(ctx)
  MITB_CHECK(ctx->c.ocr, "ocr: forward before load");
  MITB_CHECK(x && argmax && logprob && colors, "ocr: null buffer");
  ocr_run(ctx->c, *ctx->c.ocr, x, nullptr, n, wp, argmax, logprob, colors, (cudaStream_t)stream);
  API_END(ctx)
}
int mitb_ocr_forward_u8(mitb_ctx* ctx, const uint8_t* img, int n, int wp, int32_t* argmax, float* logprob, float* colors, void* stream) {
  API_BEGIN(ctx)
  MITB_CHECK(ctx->c.ocr, "ocr: forward before load");
  MITB_CHECK(img && argmax && logprob && colors, "ocr: null buffer");
  ocr_run(ctx->c, *ctx->c.ocr, nullptr, img, n, wp, argmax, logprob, colors, (cudaStream_t)stream);
  API_END(ctx)
}

int mitb_lama_load(mitb_ctx* ctx, const mitb_tensor* w, int n) {
  API_BEGIN(ctx)
  if (ctx->c.lama) { lama_free(ctx->c.lama); ctx->c.lama = nullptr; }
  Weights W = collect(w, n);
  ctx->c.lama = lama_build(ctx->c, W);
  API_END(ctx)
}
int mitb_lama_unload(mitb_ctx* ctx) {
  API_BEGIN(ctx)
  CUDA_OK(cudaDeviceSynchronize());
  if (ctx->c.lama) { lama_free(ctx->c.lama); ctx->c.lama = nullptr; }
  API_END(ctx)
}
int mitb_lama_forward(mitb_ctx* ctx, const float* img, const float* mask, const int32_t* rel_pos, const int32_t* direct, int n,
                      int h, int w, float* out, void* stream) {
  API_BEGIN(ctx)
  MITB_CHECK(ctx->c.lama, "lama: forward before load");
  MITB_CHECK(img && mask && out, "lama: null buffer");
  lama_run(ctx->c, *ctx->c.lama, img, mask, rel_pos, direct, h, w, n, h, w, out, (cudaStream_t)stream);
  API_END(ctx)
}
int mitb_lama_forward_mpe256(mitb_ctx* ctx, const float* img, const float* mask, const int32_t* rel_pos256,
                             const int32_t* direct256, int n, int h, int w, float* out, void* stream) {
  API_BEGIN(ctx)
  MITB_CHECK(ctx->c.lama, "lama: forward before load");
  MITB_CHECK(img && mask && out && rel_pos256 && direct256, "lama: null buffer");
  lama_run(ctx->c, *ctx->c.lama, img, mask, rel_pos256, direct256, 256, 256, n, h, w, out, (cudaStream_t)stream);
  API_END(ctx)
}

int mitb_lama_infer_u8(mitb_ctx* ctx, const uint8_t* img, const uint8_t* mask, const int32_t* rel_pos256, const int32_t* direct256,
                       int h, int w, int composite, uint8_t* out, void* stream) {
  API_BEGIN(ctx)
  MITB_CHECK(ctx->c.lama, "lama: forward before load");
  MITB_CHECK(img && mask && out, "lama: null buffer");
  LamaU8Io io; io.img = img; io.mask = mask; io.out = out; io.composite = composite;
  lama_run(ctx->c, *ctx->c.lama, nullptr, nullptr, rel_pos256, direct256, 256, 256, 1, h, w, nullptr, (cudaStream_t)stream, &io);
  API_END(ctx)
}

// ------------------------------------------------------------------ standalone operators
static View nhwc_tmp(Arena& ws, int n, int h, int w, int c) { return ws.view(n, h, w, (c + 3) & ~3).slice(0, c); }

int mitb_op_conv2d(mitb_ctx* ctx, const float* x, int n, int cin, int h, int w, const float* wt, int cout, int kh, int kw,
                   int stride_y, int stride_x, int pad_y, int pad_x, int pad_mode, const float* bias, int act,
                   const float* in_scale, const float* in_shift, int in_relu, float* y, void* stream) {
  API_BEGIN(ctx)
  cudaStream_t st = (cudaStream_t)stream;
  const int ho = (h + 2 * pad_y - kh) / stride_y + 1, wo = (w + 2 * pad_x - kw) / stride_x + 1;
  DevBlob blob;
  mitb_tensor t{"w", wt, 4, {cout, cin, kh, kw}};
  Weights W; W.t["w"] = t;
  Loader L{W, blob, st};
  const int cin4 = (cin + 3) & ~3;
  ConvW cw = L.conv_padcin("w", 0, cin4);
  for (int i = 0; i < cw.ntaps; ++i) { cw.tdy[i] = (int8_t)(i / kw - pad_y); cw.tdx[i] = (int8_t)(i % kw - pad_x); }
  const float *isc = in_scale, *ish = in_shift;
  if (in_scale && cin4 != cin) {   // pad the prologue vectors
    float* a = blob.alloc_f(cin4); float* b = blob.alloc_f(cin4);
    CUDA_OK(cudaMemsetAsync(a, 0, cin4 * 4, st)); CUDA_OK(cudaMemsetAsync(b, 0, cin4 * 4, st));
    CUDA_OK(cudaMemcpyAsync(a, in_scale, cin * 4, cudaMemcpyDeviceToDevice, st));
    CUDA_OK(cudaMemcpyAsync(b, in_shift, cin * 4, cudaMemcpyDeviceToDevice, st));
    isc = a; ish = b;
  }
  run_with_workspace(ctx->c, st, [&](Exec& e) {
    Arena& ws = e.ws();
    View xin = ws.view(n, h, w, cin4);
    View yout = ws.view(n, ho, wo, (cout + 3) & ~3).slice(0, cout);
    if (!e.dry) launch_nchw_to_nhwc(x, n, cin, h, w, xin, st);
    ConvOp op = Exec::op_from(cw, xin, yout, 1, pad_mode);
    op.sy = stride_y; op.sx = stride_x; op.shift = bias; op.act = act;
    op.in_scale = isc; op.in_shift = ish; op.in_relu = in_relu;
    e.conv(op);
    if (!e.dry) launch_nhwc_to_nchw(yout, y, st);
  });
  CUDA_OK(cudaStreamSynchronize(st));
  API_END(ctx)
}

int mitb_op_conv_transpose2d(mitb_ctx* ctx, const float* x, int n, int cin, int h, int w, const float* wt, int cout, int k,
                             int pad, int out_pad, const float* bias, int act, float* y, void* stream) {
  API_BEGIN(ctx)
  cudaStream_t st = (cudaStream_t)stream;
  MITB_CHECK((k == 2 && pad == 0 && out_pad == 0) || (k == 4 && pad == 1 && out_pad == 0) || (k == 3 && pad == 1 && out_pad == 1),
             "conv_transpose2d: unsupported (k,p,op)=(%d,%d,%d)", k, pad, out_pad);
  MITB_CHECK(cin % 4 == 0, "conv_transpose2d: cin must be a multiple of 4");
  DevBlob blob;
  mitb_tensor t{"w", wt, 4, {cin, cout, k, k}};
  Weights W; W.t["w"] = t;
  Loader L{W, blob, st};
  ConvW ph[4];
  for (int p = 0; p < 4; ++p) { ph[p] = L.convT_phase("w", k, pad, p >> 1, p & 1); ph[p].shift = bias; }
  run_with_workspace(ctx->c, st, [&](Exec& e) {
    Arena& ws = e.ws();
    View xin = ws.view(n, h, w, cin);
    View yout = ws.view(n, 2 * h, 2 * w, (cout + 3) & ~3).slice(0, cout);
    if (!e.dry) launch_nchw_to_nhwc(x, n, cin, h, w, xin, st);
    e.convT2(ph, xin, yout, [&](ConvOp& op) { op.act = act; });
    if (!e.dry) launch_nhwc_to_nchw(yout, y, st);
  });
  CUDA_OK(cudaStreamSynchronize(st));
  API_END(ctx)
}

int mitb_op_dwconv7_ln(mitb_ctx* ctx, const float* x, int n, int c, int h, int w, const float* wdw, const float* bdw,
                       const float* lnw, const float* lnb, float eps, float* y, void* stream) {
  API_BEGIN(ctx)
  cudaStream_t st = (cudaStream_t)stream;
  DevBlob blob;
  float* wr = blob.alloc_f((size_t)49 * c);
  std::vector<int> ky(49), kx(49);
  for (int i = 0; i < 49; ++i) { ky[i] = i / 7; kx[i] = i % 7; }
  launch_repack(wr, wdw, c, 1, 49, ky.data(), kx.data(), 49, 49, 7, 1, c, st);
  run_with_workspace(ctx->c, st, [&](Exec& e) {
    Arena& ws = e.ws();
    View xin = ws.view(n, h, w, c), yout = ws.view(n, h, w, c);
    if (!e.dry) launch_nchw_to_nhwc(x, n, c, h, w, xin, st);
    e.dwconv7_ln(xin, yout, wr, bdw, lnw, lnb, eps);
    if (!e.dry) launch_nhwc_to_nchw(yout, y, st);
  });
  CUDA_OK(cudaStreamSynchronize(st));
  API_END(ctx)
}

int mitb_op_maxpool3x3s2(mitb_ctx* ctx, const float* x, int n, int c, int h, int w, float* y, void* stream) {
  API_BEGIN(ctx)
  cudaStream_t st = (cudaStream_t)stream;
  MITB_CHECK(x && y && n >= 1 && c >= 1 && h >= 1 && w >= 1, "maxpool3x3s2: bad arguments");
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1, c4 = (c + 3) & ~3;
  run_with_workspace(ctx->c, st, [&](Exec& e) {
    Arena& ws = e.ws();
    View xin = ws.view(n, h, w, c4), yout = ws.view(n, ho, wo, c4);      // channels c..c4 are zero filled and dropped
    if (!e.dry) {
      launch_nchw_to_nhwc(x, n, c, h, w, xin, st);
      launch_maxpool3x3s2(xin, yout, st);
      launch_nhwc_to_nchw(yout.slice(0, c), y, st);
    }
  });
  CUDA_OK(cudaStreamSynchronize(st));
  API_END(ctx)
}

int mitb_op_layernorm(mitb_ctx* ctx, const float* x, int rows, int c, const float* w, const float* b, float eps, float* y, void* stream) {
  API_BEGIN(ctx)
  View in; in.p = const_cast<float*>(x); in.N = 1; in.H = 1; in.W = rows; in.C = c; in.cs = c;
  View out = in; out.p = y;
  g_launch_counter = &ctx->c.launches; ++g_launch_epoch;
  launch_layernorm(in, out, w, b, eps, nullptr, nullptr, 1, (cudaStream_t)stream);
  g_launch_counter = nullptr;
  API_END(ctx)
}

int mitb_op_rfft2(mitb_ctx* ctx, const float* x, int c, int h, int w, float* spec, void* stream) {
  API_BEGIN(ctx)
  cudaStream_t st = (cudaStream_t)stream;
  const int w2 = w / 2 + 1;
  View in; in.p = const_cast<float*>(x); in.N = 1; in.H = h; in.W = w; in.C = c; in.cs = c; in.planar = true;
  View sp; sp.p = spec; sp.N = 1; sp.H = h; sp.W = w2; sp.C = 2 * c; sp.cs = 2 * c; sp.planar = true;
  run_with_workspace(ctx->c, st, [&](Exec& e) {
    float2* tmp = (float2*)e.ws().alloc((size_t)c * h * w2 * sizeof(float2));
    if (!e.dry) launch_rfft2(in, sp, tmp, st);
  });
  CUDA_OK(cudaStreamSynchronize(st));
  API_END(ctx)
}

int mitb_op_irfft2(mitb_ctx* ctx, const float* spec, int c, int h, int w, float* y, void* stream) {
  API_BEGIN(ctx)
  cudaStream_t st = (cudaStream_t)stream;
  const int w2 = w / 2 + 1;
  View sp; sp.p = const_cast<float*>(spec); sp.N = 1; sp.H = h; sp.W = w2; sp.C = 2 * c; sp.cs = 2 * c; sp.planar = true;
  View out; out.p = y; out.N = 1; out.H = h; out.W = w; out.C = c; out.cs = c; out.planar = true;
  run_with_workspace(ctx->c, st, [&](Exec& e) {
    float2* tmp = (float2*)e.ws().alloc((size_t)c * h * w2 * sizeof(float2));
    if (!e.dry) launch_irfft2(sp, out, nullptr, tmp, st);
  });
  CUDA_OK(cudaStreamSynchronize(st));
  API_END(ctx)
}

int mitb_op_rfft2_nhwc(mitb_ctx* ctx, const float* x, int n, int h, int w, int c, float* spec, void* stream) {
  API_BEGIN(ctx)
  cudaStream_t st = (cudaStream_t)stream;
  const int w2 = w / 2 + 1;
  View in; in.p = const_cast<float*>(x); in.N = n; in.H = h; in.W = w; in.C = c; in.cs = c;
  run_with_workspace(ctx->c, st, [&](Exec& e) {
    float2* tmp = (float2*)e.ws().alloc((size_t)n * c * h * w2 * sizeof(float2));
    if (!e.dry) launch_rfft2_nhwc(in, nullptr, spec, tmp, st);
  });
  CUDA_OK(cudaStreamSynchronize(st));
  API_END(ctx)
}

int mitb_op_irfft2_nhwc(mitb_ctx* ctx, const float* spec, const float* add, int n, int h, int w, int c, float* y, void* stream) {
  API_BEGIN(ctx)
  cudaStream_t st = (cudaStream_t)stream;
  const int w2 = w / 2 + 1;
  View sp; sp.p = const_cast<float*>(spec); sp.N = n; sp.H = h; sp.W = w2; sp.C = 2 * c; sp.cs = 2 * c;
  View out; out.p = y; out.N = n; out.H = h; out.W = w; out.C = c; out.cs = c;
  View res = out; res.p = const_cast<float*>(add);
  run_with_workspace(ctx->c, st, [&](Exec& e) {
    float2* tmp = (float2*)e.ws().alloc((size_t)n * c * h * w2 * sizeof(float2));
    if (!e.dry) launch_irfft2_nhwc(sp, out, nullptr, 0, add ? &res : nullptr, tmp, st);
  });
  CUDA_OK(cudaStreamSynchronize(st));
  API_END(ctx)
}

int mitb_op_attention(mitb_ctx* ctx, const float* qk, const float* v, int n, int t, int heads, int head_dim, float* out, void* stream) {
  API_BEGIN(ctx)
  g_launch_counter = &ctx->c.launches; ++g_launch_epoch;
  launch_attention(qk, v, out, n, t, heads, head_dim, (cudaStream_t)stream);
  g_launch_counter = nullptr;
  API_END(ctx)
}

int mitb_op_mpe_tables(mitb_ctx* ctx, const uint8_t* small, int n, int32_t* rel_pos, int32_t* direct, void* stream) {
  API_BEGIN(ctx)
  g_launch_counter = &ctx->c.launches; ++g_launch_epoch;
  launch_mpe_tables(small, n, rel_pos, direct, (cudaStream_t)stream);
  g_launch_counter = nullptr;
  API_END(ctx)
}

int mitb_op_bilateral17(mitb_ctx* ctx, const uint8_t* img, int h, int w, uint8_t* out, void* stream) {
  API_BEGIN(ctx)
  g_launch_counter = &ctx->c.launches; ++g_launch_epoch;
  launch_bilateral17(img, h, w, out, (cudaStream_t)stream);
  g_launch_counter = nullptr;
  API_END(ctx)
}

int mitb_op_warp_lines_u8(mitb_ctx* ctx, const uint8_t* page, int h, int w, const double* lines, int n, uint8_t* canvas, int canvas_h,
                          int canvas_w, void* stream) {
  API_BEGIN(ctx)
  g_launch_counter = &ctx->c.launches; ++g_launch_epoch;
  launch_warp_lines(page, h, w, lines, n, canvas, canvas_h, canvas_w, (cudaStream_t)stream);
  g_launch_counter = nullptr;
  API_END(ctx)
}

int mitb_op_ctc_collapse(mitb_ctx* ctx, const int32_t* argmax, const float* logprob, const float* colors, int n, int t, int32_t* counts,
                         int32_t* steps, int32_t* chars, float* logprob_out, float* colors_out, void* stream) {
  API_BEGIN(ctx)
  g_launch_counter = &ctx->c.launches; ++g_launch_epoch;
  launch_ctc_collapse(argmax, logprob, colors, n, t, counts, steps, chars, logprob_out, colors_out, (cudaStream_t)stream);
  g_launch_counter = nullptr;
  API_END(ctx)
}

int mitb_op_textline_pairs(mitb_ctx* ctx, const double* quads, int n, double ratio, double discard_connection_gap, double char_gap_tolerance,
                           double char_gap_tolerance2, double font_size_ratio_tol, double aspect_ratio_tol, uint8_t* adj, void* stream) {
  API_BEGIN(ctx)
  g_launch_counter = &ctx->c.launches; ++g_launch_epoch;
  const double pp[6] = {ratio, discard_connection_gap, char_gap_tolerance, char_gap_tolerance2, font_size_ratio_tol, aspect_ratio_tol};
  launch_textline_pairs(quads, n, pp, adj, (cudaStream_t)stream);
  g_launch_counter = nullptr;
  API_END(ctx)
}

#define MITB_OP(body)                                             \
  API_BEGIN(ctx)                                                  \
  g_launch_counter = &ctx->c.launches; ++g_launch_epoch;          \
  body;                                                           \
  g_launch_counter = nullptr;                                     \
  API_END(ctx)

int mitb_op_resize_linear_u8(mitb_ctx* ctx, const uint8_t* src, int sh, int sw, int channels, uint8_t* dst, int dh, int dw, int binarize, void* stream) {
  MITB_OP(launch_resize_linear_u8(src, sh, sw, channels, dst, dh, dw, binarize, (cudaStream_t)stream))
}
int mitb_op_cut_rects(mitb_ctx* ctx, uint8_t* mask, int h, int w, const int32_t* rects, int n, void* stream) {
  MITB_OP(launch_cut_rects(mask, h, w, rects, n, (cudaStream_t)stream))
}
int mitb_op_cc_label(mitb_ctx* ctx, const uint8_t* mask, int h, int w, int32_t* labels, int32_t* stats, int32_t* ncomp, int cap, int32_t* scratch,
                     void* stream) {
  MITB_OP(launch_cc_label(mask, h, w, labels, stats, ncomp, cap, scratch, (cudaStream_t)stream))
}
int mitb_op_owner_map(mitb_ctx* ctx, const int32_t* labels, const int32_t* owner, int n, int32_t* owner_map, void* stream) {
  MITB_OP(launch_owner_map(labels, owner, n, owner_map, (cudaStream_t)stream))
}
int mitb_op_crf_workspace(long long npix, long long nslots2, long long nslots5, unsigned long long* bytes) {
  if (!bytes) return 1;
  *bytes = (unsigned long long)crf_workspace_bytes((long)npix, (long)nslots2, (long)nslots5);
  return 0;
}
int mitb_op_dense_crf(mitb_ctx* ctx, const int32_t* lines2, const int32_t* lines5, int nlines, const uint8_t* img, const int32_t* owner_map, int img_w,
                      int max_pix, int max_cap2, int max_cap5, long long npix, long long nslots2, long long nslots5, int iters, float sxy_g,
                      float w_g, float sxy_b, float srgb, float w_b, float u_on, void* work, uint8_t* refined, int32_t* err, void* stream) {
  MITB_OP(launch_crf(lines2, lines5, nlines, img, owner_map, img_w, max_pix, max_cap2, max_cap5, (long)npix, (long)nslots2, (long)nslots5, iters,
                     sxy_g, w_g, sxy_b, srgb, w_b, u_on, work, refined, err, (cudaStream_t)stream))
}
int mitb_op_dilate_lines(mitb_ctx* ctx, const int32_t* lines, int nlines, int max_pix2, const int32_t* owner_map, const uint8_t* refined,
                         const uint8_t* se, int img_w, uint8_t* final_mask, void* stream) {
  MITB_OP(launch_dilate_lines(lines, nlines, max_pix2, owner_map, refined, se, img_w, final_mask, (cudaStream_t)stream))
}
int mitb_op_dilate_se(mitb_ctx* ctx, const uint8_t* src, int h, int w, const uint8_t* se, int ksize, uint8_t* dst, void* stream) {
  MITB_OP(launch_dilate_se(src, h, w, se, ksize, dst, (cudaStream_t)stream))
}
#undef MITB_OP

}  // extern "C"
