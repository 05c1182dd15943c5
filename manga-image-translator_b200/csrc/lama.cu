// LaMa FFC generator forward, MPE (9 blocks + masked positional encoding) or large (18 blocks).
// Reference: inpainting/inpainting_lama_mpe.py:187-436 (FourierUnit / SpectralTransform / FFC / FFC_BN_ACT / FFCResnetBlock),
// :545-613 (FFCResNetGenerator), :616-632 (MPE), :713-726 (LamaFourier.__call__).
//
// Data layout: the bottleneck tensor is ONE NHWC buffer of 512 channels = [local 128 | global 384]; the three spatial 3x3
// convs of an FFC layer become two implicit GEMMs over channel slices (l2l+g2l share one accumulation over all 512 input
// channels).  The spectral branch runs planar (NCHW): 1x1 conv+BN+ReLU -> rfft2 -> 1x1 spectral conv+BN+ReLU -> irfft2
// (+residual) -> 1x1 conv whose epilogue adds the l2g branch, applies BN_g + ReLU and the block residual.
#include <math.h>
#include "exec.h"

namespace mitb {

static const float kBnEps = 1e-5f;

struct FfcLayer {                      // one FFC_BN_ACT of a res-block
  ConvW to_l;                          // [l2l ; g2l] over 512 input channels -> 128, epilogue bn_l + relu
  ConvW l2g;                           // 128 -> 384 raw
  ConvW sp1;                           // 1x1 384 -> 192, bn + relu (planar out)
  ConvW fu;                            // 1x1 384 -> 384 on the spectrum, bn + relu (planar in/out)
  ConvW sp2;                           // 1x1 192 -> 384, epilogue (+l2g) bn_g relu
  ConvW sp2m;                          // tensor-core weights of [sp2 ; l2g] along K: both accumulate in ONE launch (fused path)
};
struct UpLayer { ConvW ph[4]; };

struct LamaModel {
  DevBlob blob;
  int n_blocks = 0; bool use_mpe = false;
  ConvW stem, d1, d2, d3l, d3g;
  std::vector<FfcLayer> layers;        // 2 per block
  UpLayer up[3];
  ConvW outc;
  const float* mpe_table = nullptr; const float* mpe_dirw = nullptr; float a5 = 0.f, a6 = 0.f;
};

static void fold_bias_bn(Loader& L, const std::string& bias, const std::string& bn, const float** scale, const float** shift, int C) {
  const float *s = nullptr, *b = nullptr;
  L.bn_fold(bn, kBnEps, &s, &b);
  std::vector<float> hs(C), hb(C), bi(C);
  CUDA_OK(cudaMemcpy(hs.data(), s, C * sizeof(float), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(hb.data(), b, C * sizeof(float), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(bi.data(), L.W.get(bias).data, C * sizeof(float), cudaMemcpyDeviceToHost));
  for (int i = 0; i < C; ++i) hb[i] = (float)((double)bi[i] * (double)hs[i] + (double)hb[i]);
  float* d = L.blob.alloc_f(C + 4);
  CUDA_OK(cudaMemcpy(d, hb.data(), C * sizeof(float), cudaMemcpyHostToDevice));
  *scale = s; *shift = d;
}

LamaModel* lama_build(Ctx& ctx, const Weights& W) {
  LamaModel* m = new LamaModel();
  try {
    Loader L{W, m->blob, 0};
    while (W.has("model." + std::to_string(5 + m->n_blocks) + ".conv1.ffc.convl2l.weight")) ++m->n_blocks;
    MITB_CHECK(m->n_blocks > 0, "lama: no FFC res-blocks found in the state_dict");
    m->stem = L.conv("model.1.ffc.convl2l.weight", 3, 3); L.bn_fold("model.1.bn_l.", kBnEps, &m->stem.scale, &m->stem.shift);
    m->d1 = L.conv("model.2.ffc.convl2l.weight", 1, 1); L.bn_fold("model.2.bn_l.", kBnEps, &m->d1.scale, &m->d1.shift);
    m->d2 = L.conv("model.3.ffc.convl2l.weight", 1, 1); L.bn_fold("model.3.bn_l.", kBnEps, &m->d2.scale, &m->d2.shift);
    m->d3l = L.conv("model.4.ffc.convl2l.weight", 1, 1); L.bn_fold("model.4.bn_l.", kBnEps, &m->d3l.scale, &m->d3l.shift);
    m->d3g = L.conv("model.4.ffc.convl2g.weight", 1, 1); L.bn_fold("model.4.bn_g.", kBnEps, &m->d3g.scale, &m->d3g.shift);
    for (int b = 0; b < m->n_blocks; ++b)
      for (int c = 0; c < 2; ++c) {
        const std::string p = "model." + std::to_string(5 + b) + (c == 0 ? ".conv1." : ".conv2.");
        const std::string f = p + "ffc.";
        FfcLayer l;
        l.to_l = L.conv_cat_cin({f + "convl2l.weight", f + "convg2l.weight"}, 1, 1);
        L.bn_fold(p + "bn_l.", kBnEps, &l.to_l.scale, &l.to_l.shift);
        l.l2g = L.conv(f + "convl2g.weight", 1, 1);
        l.sp1 = L.conv(f + "convg2g.conv1.0.weight", 0, 0); L.bn_fold(f + "convg2g.conv1.1.", kBnEps, &l.sp1.scale, &l.sp1.shift);
        l.fu = L.conv(f + "convg2g.fu.conv_layer.weight", 0, 0); L.bn_fold(f + "convg2g.fu.bn.", kBnEps, &l.fu.scale, &l.fu.shift);
        l.sp2 = L.conv(f + "convg2g.conv2.weight", 0, 0); L.bn_fold(p + "bn_g.", kBnEps, &l.sp2.scale, &l.sp2.shift);
        l.sp2m = L.cat_k(l.sp2, l.l2g); l.sp2m.scale = l.sp2.scale; l.sp2m.shift = l.sp2.shift;
        m->layers.push_back(l);
      }
    int k = 5 + m->n_blocks + 1;
    const int ups[3] = {256, 128, 64};
    for (int i = 0; i < 3; ++i) {
      const std::string wn = "model." + std::to_string(k) + ".weight";
      const float *s = nullptr, *sh = nullptr;
      fold_bias_bn(L, "model." + std::to_string(k) + ".bias", "model." + std::to_string(k + 1) + ".", &s, &sh, ups[i]);
      for (int ph = 0; ph < 4; ++ph) { m->up[i].ph[ph] = L.convT_phase(wn, 3, 1, ph >> 1, ph & 1); m->up[i].ph[ph].scale = s; m->up[i].ph[ph].shift = sh; }
      k += 3;
    }
    m->outc = L.conv("model." + std::to_string(k + 1) + ".weight", 3, 3); m->outc.shift = L.vec("model." + std::to_string(k + 1) + ".bias");
    if (W.has("mpe.rel_pos_emb.weight")) {
      m->use_mpe = true;
      m->mpe_table = L.vec("mpe.rel_pos_emb.weight"); m->mpe_dirw = L.vec("mpe.direct_emb.weight");
      m->a5 = L.scalar("mpe.alpha5"); m->a6 = L.scalar("mpe.alpha6");
    }
    CUDA_OK(cudaDeviceSynchronize());
  } catch (...) { delete m; throw; }
  return m;
}

void lama_free(LamaModel* m) { delete m; }

// One FFC_BN_ACT on the 512-channel bottleneck (inpainting_lama_mpe.py:349-369, 394-399).
// X -> Y ; `res` (optional) is the block input added after the activation (FFCResnetBlock, :432).
void run_ffc_layer(Exec& e, const FfcLayer& l, const View& X, const View& Y, const View* res) {
  Arena& ws = e.ws();
  const size_t mk = ws.mark();
  const int n = X.N, h = X.H, w = X.W, w2 = w / 2 + 1;
  View Xl = X.slice(0, 128), Xg = X.slice(128, 384), Yl = Y.slice(0, 128), Yg = Y.slice(128, 384);
  View G = ws.view(n, h, w, 384);
  { ConvOp op = Exec::op_from(l.l2g, Xl, G, 1, PAD_REFLECT); op.scale = nullptr; op.shift = nullptr; e.conv(op); }
  View S = ws.view(n, h, w, 192, true), SP = ws.view(n, h, w2, 384, true), FP = ws.view(n, h, w2, 384, true),
       U = ws.view(n, h, w, 192, true);
  float2* tmp = (float2*)ws.alloc((size_t)n * 192 * h * w2 * sizeof(float2));
  { ConvOp op = Exec::op_from(l.sp1, Xg, S); op.act = ACT_RELU; e.conv(op); }
  if (!e.dry) launch_rfft2(S, SP, tmp, e.st);
  { ConvOp op = Exec::op_from(l.fu, SP, FP); op.act = ACT_RELU; e.conv(op); }
  if (!e.dry) launch_irfft2(FP, U, &S, tmp, e.st);
  {
    ConvOp op = Exec::op_from(l.sp2, U, Yg); op.add0 = G; op.act = ACT_RELU;
    if (res) op.add1 = res->slice(128, 384);
    e.conv(op);
  }
  // local output last: it may overwrite X_l in place (its own residual is read element-wise by the same thread)
  {
    ConvOp op = Exec::op_from(l.to_l, X, Yl, 1, PAD_REFLECT); op.act = ACT_RELU;
    if (res) op.add1 = res->slice(0, 128);
    e.conv(op);
  }
  ws.release(mk);
}

// ---------------------------------------------------------------------------------------------------------------------
// Fused FFC_BN_ACT (the "fused FFC block" of the north star), all tensors NHWC, no operand-split pass and no transposes:
//   X arrives as bf16 hi/mid operands `Xs` [n][h+2][w+2][512] with its reflect halo (written by the previous layer's epilogues)
//   1. sp1   : 1x1 384->192 over Xs[128:512]  -> BN+ReLU -> S fp32 NHWC
//   2. rfft2 : rows then columns on S (channel-vectorised, fft_nhwc.cu); the column pass emits the spectrum directly as the bf16
//              hi/mid operands of the spectral conv                                                   (:228-231)
//   3. fu    : 1x1 384->384 over the spectrum -> BN+ReLU -> F fp32 NHWC                                (:242-243)
//   4. irfft2: columns then rows; the row pass adds the residual S (:305) and emits U as bf16 hi/mid   (:245-252)
//   5. sp2m  : ONE GEMM over two K segments, 1x1 over U (K=192) and the 3x3 reflect l->g conv over Xs[0:128] (K=1152), both
//              accumulating in the same TMEM tile -> BN_g -> ReLU (-> + block residual) -> Ys[128:512] (+ fp32)  (:361-366)
//   6. to_l  : 3x3 reflect over all 512 channels of Xs -> BN_l -> ReLU (-> + residual) -> Ys[0:128] (+ fp32)  (:358-360)
//   7. halo  : reflect border of Ys for the next layer's 3x3 convs
// Yf (optional) receives the fp32 result (needed as the next block's residual and by the decoder).
static View shape_view(int n, int h, int w, int c) { View v; v.N = n; v.H = h; v.W = w; v.C = c; v.cs = c; return v; }

struct FfcFastOps { ConvOp sp1, fu, sp2m, to_l; };

static FfcFastOps ffc_fast_ops(const FfcLayer& l, const SplitView& Xs, const SplitView& Ys, const View* Yf, const View* res, const View& S,
                               const SplitView& SPs, const View& FP, const SplitView& Us) {
  const int n = Xs.N, h = Xs.H, w = Xs.W, w2 = w / 2 + 1;
  FfcFastOps o;
  o.sp1 = Exec::op_from(l.sp1, shape_view(n, h, w, 384), S); o.sp1.in_sv = Xs; o.sp1.in_sv_coff = 128; o.sp1.act = ACT_RELU;
  o.fu = Exec::op_from(l.fu, shape_view(n, h, w2, 384), FP); o.fu.in_sv = SPs; o.fu.act = ACT_RELU;
  {
    View yg = Yf ? Yf->slice(128, 384) : shape_view(n, h, w, 384);
    ConvOp op = Exec::op_from2(l.sp2, l.l2g, l.sp2m, shape_view(n, h, w, 192), yg);
    op.in_sv = Us;
    op.seg2.sv = Xs; op.seg2.coff = 0; op.seg2.pad = PAD_REFLECT;
    op.act = ACT_RELU;
    if (res) op.add1 = res->slice(128, 384);
    op.out_sv = Ys; op.out_sv_coff = 128;
    o.sp2m = op;
  }
  {
    View yl = Yf ? Yf->slice(0, 128) : shape_view(n, h, w, 128);
    ConvOp op = Exec::op_from(l.to_l, shape_view(n, h, w, 512), yl, 1, PAD_REFLECT);
    op.in_sv = Xs; op.act = ACT_RELU;
    if (res) op.add1 = res->slice(0, 128);
    op.out_sv = Ys; op.out_sv_coff = 0;
    o.to_l = op;
  }
  return o;
}

static int g_ffc_mode = 1;             // 0: generic planar path only, 1: fused path when no layer needs split-K, 2: fused whenever capable
void lama_set_ffc_mode(int mode) { g_ffc_mode = mode; }
static int g_sparse_decoder = -1;      // -1: environment default (on unless MITB_DENSE_TAIL=1)
void lama_set_sparse_decoder(int on) { g_sparse_decoder = on ? 1 : 0; }
static bool lama_sparse_decoder() {
  if (g_sparse_decoder < 0) { const char* ev = getenv("MITB_DENSE_TAIL"); g_sparse_decoder = (ev && atoi(ev)) ? 0 : 1; }
  return g_sparse_decoder != 0;
}

static bool ffc_fast_ok(const LamaModel& m, int n, int h, int w) {
  if (g_ffc_mode == 0 || !fft_nhwc_supported(h, w, 192) || h < 4 || w < 4) return false;
  SplitView Xs; Xs.hi = (uint16_t*)0x1000; Xs.mid = Xs.hi; Xs.N = n; Xs.H = h; Xs.W = w; Xs.C = 512; Xs.pt = Xs.pl = 1; Xs.Hp = h + 2; Xs.Wp = w + 2;
  SplitView SPs = Xs; SPs.W = w / 2 + 1; SPs.C = 384; SPs.pt = SPs.pl = 0; SPs.Hp = h; SPs.Wp = SPs.W;
  SplitView Us = SPs; Us.W = Us.Wp = w; Us.C = 192;
  View S = shape_view(n, h, w, 192), FP = shape_view(n, h, w / 2 + 1, 384);
  S.p = FP.p = (float*)0x1000;
  const FfcFastOps o = ffc_fast_ops(m.layers[0], Xs, Xs, nullptr, nullptr, S, SPs, FP, Us);
  if (!(conv_tma_capable(o.sp1) && conv_tma_capable(o.fu) && conv_tma_capable(o.sp2m) && conv_tma_capable(o.to_l))) return false;
  if (g_ffc_mode >= 2) return true;
  return (long)n * h * w >= 128L * 74;            // below this the 3x3 layers want split-K, which only the gather kernel has
}

static void run_ffc_layer_fast(Exec& e, const FfcLayer& l, const SplitView& Xs, const SplitView& Ys, const View* Yf, const View* res) {
  Arena& ws = e.ws();
  const size_t mk = ws.mark();
  const int n = Xs.N, h = Xs.H, w = Xs.W, w2 = w / 2 + 1;
  View S = ws.view(n, h, w, 192), FP = ws.view(n, h, w2, 384);
  SplitView SPs = ws.split_view(n, h, w2, 384), Us = ws.split_view(n, h, w, 192);
  float2* T = (float2*)ws.alloc((size_t)n * h * w2 * 192 * sizeof(float2));
  const FfcFastOps o = ffc_fast_ops(l, Xs, Ys, Yf, res, S, SPs, FP, Us);
  e.conv(o.sp1);
  if (!e.dry) launch_rfft2_nhwc(S, &SPs, nullptr, T, e.st);
  e.conv(o.fu);
  if (!e.dry) launch_irfft2_nhwc(FP, shape_view(n, h, w, 192), &Us, 0, &S, T, e.st);
  e.conv(o.sp2m);
  e.conv(o.to_l);
  if (!e.dry) launch_split_halo(Ys, 0, 512, e.st);
  ws.release(mk);
}

void lama_run(Ctx& ctx, LamaModel& m, const float* img, const float* mask, const int* rel_pos, const int* direct, int th,
              int tw, int n, int h, int w, float* out, cudaStream_t st, const LamaU8Io* u8) {
  MITB_CHECK(n >= 1 && h % 8 == 0 && w % 8 == 0 && h >= 32 && w >= 32, "lama: input %dx%d must be a multiple of 8 (>=32)", h, w);
  MITB_CHECK(!m.use_mpe || (rel_pos && direct), "lama_mpe needs the rel_pos/direct tables");
  run_with_workspace(ctx, st, [&](Exec& e) {
    Arena& ws = e.ws();
    const int h8 = h / 8, w8 = w / 8;
    const bool fast = ffc_fast_ok(m, n, h8, w8);
    View X = ws.view(n, h8, w8, 512), Z = ws.view(n, h8, w8, 512), Y;
    SplitView Xs, Ys, Zs;                 // fused path: bf16 hi/mid operand copies with a 1-pixel reflect halo
    if (fast) { Xs = ws.split_view(n, h8, w8, 512, 1, 1, 1, 1); Ys = ws.split_view(n, h8, w8, 512, 1, 1, 1, 1); Zs = ws.split_view(n, h8, w8, 512, 1, 1, 1, 1); }
    else Y = ws.view(n, h8, w8, 512);
    float* maskf = nullptr;            // planar fp32 {0,1} mask when the input arrives as uint8
    MITB_CHECK(!u8 || n == 1, "lama uint8 entry handles one image per call");
    {
      const size_t mk = ws.mark();
      View x4 = ws.view(n, h, w, 4), s1 = ws.view(n, h, w, 64), s2 = ws.view(n, h / 2, w / 2, 128), s3 = ws.view(n, h / 4, w / 4, 256);
      if (u8) {
        maskf = ws.alloc_f((size_t)h * w);
        if (!e.dry) launch_lama_pack_u8(u8->img, u8->mask, h, w, x4, maskf, st);
      } else if (!e.dry) launch_lama_pack_input(img, mask, n, h, w, x4, st);
      { ConvOp op = Exec::op_from(m.stem, x4, s1, 1, PAD_REFLECT); op.act = ACT_RELU; e.conv(op); }
      if (m.use_mpe && !e.dry) launch_mpe_add(s1, rel_pos, direct, th, tw, u8 ? maskf : mask, m.mpe_table, m.mpe_dirw, m.a5, m.a6, st);
      { ConvOp op = Exec::op_from(m.d1, s1, s2, 2, PAD_REFLECT); op.act = ACT_RELU; e.conv(op); }
      { ConvOp op = Exec::op_from(m.d2, s2, s3, 2, PAD_REFLECT); op.act = ACT_RELU; e.conv(op); }
      { ConvOp op = Exec::op_from(m.d3l, s3, X.slice(0, 128), 2, PAD_REFLECT); op.act = ACT_RELU;
        if (fast && conv_tma_capable(op)) { op.out_sv = Xs; op.out_sv_coff = 0; }
        e.conv(op);
        if (fast && !op.out_sv.valid() && !e.dry) launch_split(X.slice(0, 128), Xs, 0, nullptr, nullptr, 0, st); }
      { ConvOp op = Exec::op_from(m.d3g, s3, X.slice(128, 384), 2, PAD_REFLECT); op.act = ACT_RELU;
        if (fast && conv_tma_capable(op)) { op.out_sv = Xs; op.out_sv_coff = 128; }
        e.conv(op);
        if (fast && !op.out_sv.valid() && !e.dry) launch_split(X.slice(128, 384), Xs, 128, nullptr, nullptr, 0, st); }
      if (fast && !e.dry) launch_split_halo(Xs, 0, 512, st);
      ws.release(mk);
    }
    // FFCResnetBlock x n (inpainting_lama_mpe.py:421-436): X -> Y -> Z (+X), then Z becomes the next X
    for (int b = 0; b < m.n_blocks; ++b) {
      if (fast) {
        run_ffc_layer_fast(e, m.layers[2 * b], Xs, Ys, nullptr, nullptr);
        run_ffc_layer_fast(e, m.layers[2 * b + 1], Ys, Zs, &Z, &X);
        SplitView ts = Xs; Xs = Zs; Zs = ts;
      } else {
        run_ffc_layer(e, m.layers[2 * b], X, Y, nullptr);
        run_ffc_layer(e, m.layers[2 * b + 1], Y, Z, &X);
      }
      View t = X; X = Z; Z = t;
    }
    // upsampling: 3 x [ConvTranspose2d(3,s2,p1,op1) + BN + ReLU], then ReflectionPad(3) + Conv7x7 + sigmoid
    // Output sparsity of the decoder: the result is pred*mask + (1-mask)*img (inpainting_lama_mpe.py:726), so prediction pixels outside
    // the hole are never used.  Walking the receptive fields back from the hole gives, per upsampling stage, the pixels that can reach a
    // hole pixel: the 7x7 conv reads u3 within 3 px of a hole pixel; a stride-2 transposed conv's phases produce the 2x2 block of a
    // grid pixel from its 1-neighbourhood.  Tiles without such a pixel are skipped (left unwritten) - every used output is computed from
    // computed inputs, bit-identically to the dense path (MITB_DENSE_TAIL=1 disables the hints; one image per call only).
    const bool sp = lama_sparse_decoder() && n == 1 && h % 8 == 0 && w % 8 == 0;
    uint8_t *need_u3 = nullptr, *g2 = nullptr, *need_u2 = nullptr, *g1 = nullptr, *need_u1 = nullptr, *g0 = nullptr;
    if (sp) {
      need_u3 = (uint8_t*)ws.alloc((size_t)h * w);
      g2 = (uint8_t*)ws.alloc((size_t)h * w / 4); need_u2 = (uint8_t*)ws.alloc((size_t)h * w / 4);
      g1 = (uint8_t*)ws.alloc((size_t)h * w / 16); need_u1 = (uint8_t*)ws.alloc((size_t)h * w / 16);
      g0 = (uint8_t*)ws.alloc((size_t)h * w / 64);
      if (!e.dry) {
        launch_need_from_mask(u8 ? nullptr : mask, u8 ? u8->mask : nullptr, h, w, 3, need_u3, st);
        launch_need_pool2(need_u3, h, w, g2, need_u2, st);
        launch_need_pool2(need_u2, h / 2, w / 2, g1, need_u1, st);
        launch_need_pool2(need_u1, h / 4, w / 4, g0, nullptr, st);
      }
    }
    View u1 = ws.view(n, h / 4, w / 4, 256), u2 = ws.view(n, h / 2, w / 2, 128), u3 = ws.view(n, h, w, 64);
    e.convT2(m.up[0].ph, X, u1, [&](ConvOp& op) { op.act = ACT_RELU; op.need_px = g0; });
    e.convT2(m.up[1].ph, u1, u2, [&](ConvOp& op) { op.act = ACT_RELU; op.need_px = g1; });
    e.convT2(m.up[2].ph, u2, u3, [&](ConvOp& op) { op.act = ACT_RELU; op.need_px = g2; });
    View pred = ws.view(n, h, w, 3, true);
    { ConvOp op = Exec::op_from(m.outc, u3, pred, 1, PAD_REFLECT); op.act = ACT_SIGMOID;
      if (sp) { if (u8) op.tile_mask_u8 = u8->mask; else op.tile_mask = mask; }      // (maskf's arena slot was released above)
      e.conv(op); }
    if (!e.dry) {
      if (u8) launch_lama_blend_u8(pred, u8->img, u8->mask, u8->out, u8->composite, st);
      else launch_lama_blend(pred, img, mask, out, st);
    }
  });
}

}  // namespace mitb
