// DBNet-ResNet34 text detector forward, the reference's default detector (detection/default.py:15-25, network
// detection/default_utils/DBNet_resnet34.py:76-125).  torchvision ResNet34 backbone (7x7 s2 stem + BN + ReLU, 3x3 s2 max pool,
// post-activation BasicBlocks 3/4/6/3), three AvgPool + 3x(conv3x3+BN+ReLU) down blocks, seven U-Net up blocks (2x(conv3x3+BN+ReLU)
// then ConvTranspose 4x4 s2 + BN + ReLU) whose inputs are channel concatenations [up | skip] realised as slices of shared NHWC
// buffers, the DB head on the 1/4-scale map and the mask head on the 1/2-scale map.  Outputs go straight into the caller's NCHW
// buffers.  backbone.fc.* is not used.
#include "exec.h"

namespace mitb {

struct R34Block { ConvW c1, c2, ds; bool has_ds = false; int stride = 1; };
struct R34DConv { ConvW c[3]; ConvW t[4]; bool up = false; };   // double_conv: c[0..2]; double_conv_up: c[0..1] + ConvT phases t
struct R34Head { ConvW c0; ConvW t1[4]; const float* t2_w = nullptr; const float* t2_b = nullptr; };

struct DbnetR34Model {
  DevBlob blob;
  ConvW stem;
  std::vector<R34Block> layers[4];
  R34DConv down[3], up[7];
  R34Head binarize, thresh;
  ConvW mask[4];
};

static const float kBnEps = 1e-5f;                 // nn.BatchNorm2d default
static const int kLayerC[4] = {64, 128, 256, 512}, kLayerN[4] = {3, 4, 6, 3};

// eval BatchNorm as the epilogue's scale / shift, with the preceding conv's bias (when the state dict has one) folded into the shift
static void bn_affine(Loader& L, const std::string& p, const std::string& bias, const float** scale, const float** shift) {
  L.bn_fold(p, kBnEps, scale, shift);
  if (!L.W.has(bias)) return;
  const int C = (int)L.W.get(p + "weight").shape[0];
  MITB_CHECK(L.W.get(bias).ndim == 1 && (int)L.W.get(bias).shape[0] == C, "%s: bias does not match %s", bias.c_str(), p.c_str());
  std::vector<float> s(C), t(C), b(C);
  CUDA_OK(cudaMemcpy(s.data(), *scale, C * sizeof(float), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(t.data(), *shift, C * sizeof(float), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(b.data(), L.W.get(bias).data, C * sizeof(float), cudaMemcpyDeviceToHost));
  for (int i = 0; i < C; ++i) t[i] = (float)((double)b[i] * (double)s[i] + (double)t[i]);     // (acc + b) * s + t = acc * s + (b * s + t)
  float* d = L.blob.alloc_f(C + 4);
  CUDA_OK(cudaMemcpy(d, t.data(), C * sizeof(float), cudaMemcpyHostToDevice));
  *shift = d;
}

static R34Block load_block(Loader& L, const std::string& p, int cin, int cout, int stride) {
  R34Block b; b.stride = stride;
  b.c1 = L.conv(p + "conv1.weight", 1, 1);
  L.bn_fold(p + "bn1.", kBnEps, &b.c1.scale, &b.c1.shift);
  b.c2 = L.conv_bn(p + "conv2.weight", p + "bn2.", 1, kBnEps);
  MITB_CHECK(b.c1.Cin == cin && b.c1.Cout == cout && b.c2.Cin == cout && b.c2.Cout == cout && b.c1.ntaps == 9 && b.c2.ntaps == 9,
             "%s: expected a %d -> %d BasicBlock", p.c_str(), cin, cout);
  b.has_ds = L.W.has(p + "downsample.0.weight");
  MITB_CHECK(b.has_ds == (stride != 1 || cin != cout), "%s: downsample present iff the block changes shape", p.c_str());
  if (b.has_ds) {
    b.ds = L.conv(p + "downsample.0.weight", 0, 0);
    L.bn_fold(p + "downsample.1.", kBnEps, &b.ds.scale, &b.ds.shift);
    MITB_CHECK(b.ds.Cin == cin && b.ds.Cout == cout && b.ds.ntaps == 1, "%s: downsample shape", p.c_str());
  }
  return b;
}

static R34DConv load_dconv(Loader& L, const std::string& p, bool up, int cin, int mid, int cout) {
  R34DConv d; d.up = up;
  for (int j = 0; j < (up ? 2 : 3); ++j) {
    d.c[j] = L.conv(p + std::to_string(3 * j) + ".weight", 1, 1);
    L.bn_fold(p + std::to_string(3 * j + 1) + ".", kBnEps, &d.c[j].scale, &d.c[j].shift);
  }
  MITB_CHECK(d.c[0].Cin == cin && d.c[0].Cout == mid && d.c[1].Cout == mid && (up || d.c[2].Cout == cout), "%s: unexpected shapes", p.c_str());
  if (up) {
    const float* sc; const float* sh;
    L.bn_fold(p + "7.", kBnEps, &sc, &sh);
    for (int ph = 0; ph < 4; ++ph) { d.t[ph] = L.convT_phase(p + "6.weight", 4, 1, ph >> 1, ph & 1); d.t[ph].scale = sc; d.t[ph].shift = sh; }
    MITB_CHECK(d.t[0].Cin == mid && d.t[0].Cout == cout, "%s6.weight: unexpected shape", p.c_str());
  }
  return d;
}

static R34Head load_head(Loader& L, const std::string& p) {
  R34Head h;
  h.c0 = L.conv(p + "0.weight", 1, 1);
  bn_affine(L, p + "1.", p + "0.bias", &h.c0.scale, &h.c0.shift);
  const float* sc; const float* sh;
  bn_affine(L, p + "4.", p + "3.bias", &sc, &sh);
  for (int ph = 0; ph < 4; ++ph) { h.t1[ph] = L.convT_phase(p + "3.weight", 4, 1, ph >> 1, ph & 1); h.t1[ph].scale = sc; h.t1[ph].shift = sh; }
  const mitb_tensor& t2 = L.W.get(p + "6.weight");
  MITB_CHECK(h.c0.Cin == 64 && h.c0.Cout == 16 && h.t1[0].Cin == 16 && h.t1[0].Cout == 16 && t2.ndim == 4 && t2.shape[0] == 16 && t2.shape[1] == 1 &&
             t2.shape[2] == 4 && t2.shape[3] == 4, "%s: expected DBHead(64)", p.c_str());
  h.t2_w = L.vec(p + "6.weight"); h.t2_b = L.vec(p + "6.bias");     // raw [16,1,4,4] for the fused full-resolution kernel
  return h;
}

DbnetR34Model* dbnet_r34_build(Ctx& ctx, const Weights& W) {
  DbnetR34Model* m = new DbnetR34Model();
  try {
    Loader L{W, m->blob, 0};
    m->stem = L.conv_padcin("backbone.conv1.weight", 3, 4);
    MITB_CHECK(m->stem.Cout == 64 && m->stem.ntaps == 49, "backbone.conv1.weight: expected [64,3,7,7]");
    L.bn_fold("backbone.bn1.", kBnEps, &m->stem.scale, &m->stem.shift);
    int prev = 64;
    for (int li = 0; li < 4; ++li) {
      for (int k = 0; k < kLayerN[li]; ++k) {
        const int stride = (k == 0 && li > 0) ? 2 : 1;
        m->layers[li].push_back(load_block(L, "backbone.layer" + std::to_string(li + 1) + "." + std::to_string(k) + ".", k == 0 ? prev : kLayerC[li],
                                           kLayerC[li], stride));
      }
      prev = kLayerC[li];
    }
    for (int d = 0; d < 3; ++d) m->down[d] = load_dconv(L, "down_conv" + std::to_string(d + 1) + ".conv.", false, 512, 512, 512);
    const int uc[7][3] = {{512, 512, 256}, {768, 512, 256}, {768, 512, 256}, {768, 512, 256}, {512, 256, 128}, {256, 128, 64}, {128, 64, 64}};
    for (int u = 0; u < 7; ++u) m->up[u] = load_dconv(L, "upconv" + std::to_string(u + 1) + ".conv.", true, uc[u][0], uc[u][1], uc[u][2]);
    m->binarize = load_head(L, "conv_db.binarize.");
    m->thresh = load_head(L, "conv_db.thresh.");
    const int mc[4][3] = {{64, 64, 1}, {64, 64, 1}, {64, 32, 1}, {32, 1, 0}};      // cin, cout, pad
    for (int i = 0; i < 4; ++i) {
      const std::string p = "conv_mask." + std::to_string(2 * i) + ".";
      m->mask[i] = L.conv(p + "weight", mc[i][2], mc[i][2]);
      m->mask[i].shift = L.vec(p + "bias");
      MITB_CHECK(m->mask[i].Cin == mc[i][0] && m->mask[i].Cout == mc[i][1], "%sweight: unexpected shape", p.c_str());
    }
    CUDA_OK(cudaDeviceSynchronize());
  } catch (...) { delete m; throw; }
  return m;
}

void dbnet_r34_free(DbnetR34Model* m) { delete m; }

// ResNet34 layers 1-4 after the max pool.  Operand fusion where every conv involved runs on the TMA-fed kernel: the max pool and
// each block's conv2 epilogue also store the NEXT block's input as bf16 hi/mid operands (read by its conv1 and downsample), and
// conv1's epilogue stores only conv2's operands; otherwise the fp32 tensors are written and the convs split them themselves.  The
// residual stream of a stage is updated in place (conv2 reads its identity and writes the same element); the last block of each
// layer writes straight into its skip slice of the decoder's concat buffer.
static void run_backbone(Exec& e, const DbnetR34Model& m, const View& s0, const View* skips) {
  Arena& ws = e.ws();
  const size_t mk = ws.mark();
  const int n = s0.N;
  View pool = ws.view(n, (s0.H - 1) / 2 + 1, (s0.W - 1) / 2 + 1, 64);
  struct Step { ConvOp c1, c2, ds; bool has_ds, c1_tma, c2_tma, ds_tma; SplitView in_sv; };
  std::vector<Step> steps;
  SplitView xs_prev;                                       // operand buffer at the resolution of the current block's input
  { View b = ws.view(pool.N, pool.H, pool.W, 64); xs_prev = Exec::alias_split(b); }
  View x = pool;
  for (int li = 0; li < 4; ++li) {
    const R34Block& b0 = m.layers[li][0];
    const int Ho = x.H / b0.stride, Wo = x.W / b0.stride, C = kLayerC[li];
    View r = ws.view(n, Ho, Wo, C), t = ws.view(n, Ho, Wo, C), xsb = ws.view(n, Ho, Wo, C);
    const SplitView ts = Exec::alias_split(t), xs = Exec::alias_split(xsb);
    for (size_t k = 0; k < m.layers[li].size(); ++k) {
      const R34Block& b = m.layers[li][k];
      const View y = k + 1 == m.layers[li].size() ? skips[li] : r;
      Step s; s.has_ds = b.has_ds; s.in_sv = xs_prev;
      s.c1 = Exec::op_from(b.c1, x, t, b.stride); s.c1.act = ACT_RELU;
      s.c2 = Exec::op_from(b.c2, t, y); s.c2.act = ACT_RELU;
      if (b.has_ds) { View d = ws.view(n, Ho, Wo, C); s.ds = Exec::op_from(b.ds, x, d, b.stride); s.c2.add0 = d; }
      else s.c2.add0 = x;
      s.c1_tma = conv_uses_tma(s.c1); s.c2_tma = conv_uses_tma(s.c2); s.ds_tma = b.has_ds && conv_uses_tma(s.ds);     // decided on the unfused ops
      if (s.c1_tma && s.c2_tma) { s.c1.out_sv = ts; s.c1.out.p = nullptr; s.c2.in_sv = ts; }
      steps.push_back(s);
      x = y; xs_prev = xs;
    }
  }
  // which blocks read their input as operands: conv1 and downsample on the TMA kernel, and a producer able to write them
  std::vector<bool> in_fused(steps.size());
  for (size_t i = 0; i < steps.size(); ++i)
    in_fused[i] = steps[i].c1_tma && (!steps[i].has_ds || steps[i].ds_tma) && (i == 0 || steps[i - 1].c2_tma);
  if (!e.dry) launch_maxpool3x3s2(s0, pool, e.st, in_fused[0] ? &steps[0].in_sv : nullptr);
  for (size_t i = 0; i < steps.size(); ++i) {
    Step& s = steps[i];
    if (in_fused[i]) { s.c1.in_sv = s.in_sv; if (s.has_ds) s.ds.in_sv = s.in_sv; }
    if (i + 1 < steps.size() && in_fused[i + 1]) s.c2.out_sv = steps[i + 1].in_sv;
    if (s.has_ds) e.conv(s.ds);
    e.conv(s.c1);
    e.conv(s.c2);
  }
  ws.release(mk);
}

// double_conv (AvgPool2d(2,2) + three conv3x3+BN+ReLU) or double_conv_up (two conv3x3+BN+ReLU + ConvTranspose 4x4 s2 + BN + ReLU)
static void run_dconv(Exec& e, const R34DConv& d, const View& x, const View& out) {
  Arena& ws = e.ws();
  const size_t mk = ws.mark();
  View in = x;
  if (!d.up) { in = ws.view(x.N, x.H / 2, x.W / 2, x.C); e.avgpool(x, in, 0); }
  const int mid = d.c[0].Cout;
  View a = ws.view(in.N, in.H, in.W, mid), b = ws.view(in.N, in.H, in.W, mid);
  { ConvOp op = Exec::op_from(d.c[0], in, a); op.act = ACT_RELU; e.conv(op); }
  { ConvOp op = Exec::op_from(d.c[1], a, b); op.act = ACT_RELU; e.conv(op); }
  if (d.up) e.convT2(d.t, b, out, [](ConvOp& op) { op.act = ACT_RELU; });
  else { ConvOp op = Exec::op_from(d.c[2], b, out); op.act = ACT_RELU; e.conv(op); }
  ws.release(mk);
}

void dbnet_r34_run(Ctx& ctx, DbnetR34Model& m, const float* x_nchw, const uint8_t* x_u8, int n, int h, int w, float* db, float* mask,
                   cudaStream_t st) {
  // the coarsest map is 1/256; the reference pads to 256 (imgproc.py resize_aspect_ratio) and fails in torch.cat at other sizes
  MITB_CHECK(n >= 1 && h > 0 && w > 0 && h % 256 == 0 && w % 256 == 0, "dbnet_r34: input %dx%d must be a positive multiple of 256", h, w);
  run_with_workspace(ctx, st, [&](Exec& e) {
    Arena& ws = e.ws();
    // persistent buffers: concat inputs of the decoder, cat_k = [ up | skip ]
    View cat1 = ws.view(n, h / 128, w / 128, 768);   // [up256 | h128]
    View cat2 = ws.view(n, h / 64, w / 64, 768);     // [up128 | h64]
    View cat3 = ws.view(n, h / 32, w / 32, 768);     // [up64 | h32]
    View cat4 = ws.view(n, h / 16, w / 16, 512);     // [up32 | h16]
    View cat5 = ws.view(n, h / 8, w / 8, 256);       // [up16 | h8]
    View cat6 = ws.view(n, h / 4, w / 4, 128);       // [up8 | h4]
    View h256 = ws.view(n, h / 256, w / 256, 512);
    View up4 = ws.view(n, h / 2, w / 2, 64);
    {
      const size_t mk = ws.mark();
      View x4 = ws.view(n, h, w, 4);
      if (!e.dry) {
        if (x_u8) launch_u8_to_nhwc(x_u8, n, h, w, 3, x4, 127.5f, 1.0f, 1, st);     // x / 127.5 - 1 (default.py:19)
        else launch_nchw_to_nhwc(x_nchw, n, 3, h, w, x4, st);
      }
      View s0 = ws.view(n, h / 2, w / 2, 64);
      { ConvOp op = Exec::op_from(m.stem, x4, s0, 2); op.act = ACT_RELU; e.conv(op); }
      const View skips[4] = {cat6.slice(64, 64), cat5.slice(128, 128), cat4.slice(256, 256), cat3.slice(256, 512)};
      run_backbone(e, m, s0, skips);
      ws.release(mk);
    }
    run_dconv(e, m.down[0], cat3.slice(256, 512), cat2.slice(256, 512));
    run_dconv(e, m.down[1], cat2.slice(256, 512), cat1.slice(256, 512));
    run_dconv(e, m.down[2], cat1.slice(256, 512), h256);
    run_dconv(e, m.up[0], h256, cat1.slice(0, 256));
    run_dconv(e, m.up[1], cat1, cat2.slice(0, 256));
    run_dconv(e, m.up[2], cat2, cat3.slice(0, 256));
    run_dconv(e, m.up[3], cat3, cat4.slice(0, 256));
    run_dconv(e, m.up[4], cat4, cat5.slice(0, 128));
    run_dconv(e, m.up[5], cat5, cat6.slice(0, 64));
    run_dconv(e, m.up[6], cat6, up4);
    const View up8 = cat6.slice(0, 64);
    // DBHead(64) (DBHead.py:7-34) + the caller's sigmoid on both channels (default.py:23): thresh ends in its own sigmoid
    View dbv; dbv.p = db; dbv.N = n; dbv.H = h; dbv.W = w; dbv.C = 1; dbv.cs = 2; dbv.coff = 0; dbv.planar = true;
    for (int br = 0; br < 2; ++br) {
      const R34Head& hb = br == 0 ? m.binarize : m.thresh;
      const size_t mk = ws.mark();
      View a = ws.view(n, h / 4, w / 4, 16), b = ws.view(n, h / 2, w / 2, 16);
      { ConvOp op = Exec::op_from(hb.c0, up8, a); op.act = ACT_RELU; e.conv(op); }
      e.convT2(hb.t1, a, b, [](ConvOp& op) { op.act = ACT_RELU; });
      View o = dbv; o.coff = br;
      if (!e.dry) launch_convT4_c1(b, hb.t2_w, hb.t2_b, br == 0 ? ACT_SIGMOID : ACT_SIGMOID2, o, st);
      ws.release(mk);
    }
    {  // conv_mask (DBNet_resnet34.py:83-89)
      const size_t mk = ws.mark();
      View a = ws.view(n, h / 2, w / 2, 64), b = ws.view(n, h / 2, w / 2, 64), c = ws.view(n, h / 2, w / 2, 32);
      { ConvOp op = Exec::op_from(m.mask[0], up4, a); op.act = ACT_RELU; e.conv(op); }
      { ConvOp op = Exec::op_from(m.mask[1], a, b); op.act = ACT_RELU; e.conv(op); }
      { ConvOp op = Exec::op_from(m.mask[2], b, c); op.act = ACT_RELU; e.conv(op); }
      View mv; mv.p = mask; mv.N = n; mv.H = h / 2; mv.W = w / 2; mv.C = 1; mv.cs = 1; mv.coff = 0; mv.planar = true;
      { ConvOp op = Exec::op_from(m.mask[3], c, mv); op.act = ACT_SIGMOID; e.conv(op); }
      ws.release(mk);
    }
  });
}

}  // namespace mitb
