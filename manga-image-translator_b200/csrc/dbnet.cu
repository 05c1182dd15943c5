// DBNet-ConvNeXt text detector forward (reference: detection/dbnet_convnext.py:450-509).
// ConvNeXt(depths 3/3/27/3, dims 128/256/512/1024) backbone, two extra stride-2 ConvNeXt stages, six UpconvSkip decoder
// blocks whose inputs are channel-concatenations (realised as slices of shared NHWC buffers, no copies), the DB head on
// the 1/4-scale map and the mask head on the 1/2-scale map.  Outputs are written straight into the caller's NCHW buffers.
#include "exec.h"

namespace mitb {

struct CnBlock {
  int cin = 0, cout = 0; bool dense = false;
  ConvW dense_w;                               // dense 7x7 (UpconvSkip, out<in)
  const float* dw_w = nullptr; const float* dw_b = nullptr;   // depthwise [49][C] + bias (also bias of the dense conv)
  const float* ln_w = nullptr; const float* ln_b = nullptr;
  ConvW fc1, fc2; const float* gamma = nullptr;
  ConvW sc; bool has_sc = false;
};
struct CnStage {
  bool has_ds = false; const float* ds_ln_w = nullptr; const float* ds_ln_b = nullptr; ConvW ds;
  std::vector<CnBlock> blocks;
};
struct Upconv { CnBlock blk; ConvW up[4]; };
struct HeadBranch { ConvW c0; ConvW t1[4]; ConvW t2[4]; const float* t2_w = nullptr; const float* t2_b = nullptr; };

struct DbnetModel {
  DevBlob blob;
  ConvW stem; const float* stem_ln_w; const float* stem_ln_b;
  CnStage stages[4], down1, down2;
  Upconv up[6];
  HeadBranch binarize, thresh;
  ConvW m0, m2, m4;
};

static const float kLnEps = 1e-6f;             // timm LayerNorm / LayerNorm2d default

static CnBlock load_block(Loader& L, const std::string& p, int cin, int cout) {
  CnBlock b; b.cin = cin; b.cout = cout; b.dense = cout < cin;
  if (b.dense) {
    b.dense_w = L.conv(p + "conv_dw.weight", 3, 3);
    b.dense_w.shift = L.vec(p + "conv_dw.bias");
  } else {
    const mitb_tensor& t = L.W.get(p + "conv_dw.weight");
    MITB_CHECK(t.ndim == 4 && t.shape[0] == cout && t.shape[1] == 1 && t.shape[2] == 7 && t.shape[3] == 7, "%s: bad depthwise weight", p.c_str());
    float* d = L.blob.alloc_f((size_t)49 * cout);
    std::vector<int> ky(49), kx(49);
    for (int i = 0; i < 49; ++i) { ky[i] = i / 7; kx[i] = i % 7; }
    launch_repack(d, t.data, cout, 1, 49, ky.data(), kx.data(), 49, 49, 7, 1, cout, L.st);
    b.dw_w = d; b.dw_b = L.vec(p + "conv_dw.bias");
  }
  b.ln_w = L.vec(p + "norm.weight"); b.ln_b = L.vec(p + "norm.bias");
  b.fc1 = L.conv(p + "mlp.fc1.weight", 0, 0); b.fc1.shift = L.vec(p + "mlp.fc1.bias");
  b.fc2 = L.conv(p + "mlp.fc2.weight", 0, 0); b.fc2.shift = L.vec(p + "mlp.fc2.bias");
  b.gamma = L.vec(p + "gamma");
  if (L.W.has(p + "shortcut.conv.weight")) {
    b.has_sc = true; b.sc = L.conv(p + "shortcut.conv.weight", 0, 0); b.sc.shift = L.vec(p + "shortcut.conv.bias");
  }
  return b;
}

static CnStage load_stage(Loader& L, const std::string& p, int cin, int cout, int depth) {
  CnStage s;
  if (L.W.has(p + "downsample.1.weight")) {
    s.has_ds = true;
    s.ds_ln_w = L.vec(p + "downsample.0.weight"); s.ds_ln_b = L.vec(p + "downsample.0.bias");
    s.ds = L.conv(p + "downsample.1.weight", 0, 0); s.ds.shift = L.vec(p + "downsample.1.bias");
    MITB_CHECK(s.ds.Cin == cin && s.ds.Cout == cout, "%s: downsample shape", p.c_str());
  }
  for (int k = 0; k < depth; ++k) s.blocks.push_back(load_block(L, p + "blocks." + std::to_string(k) + ".", cout, cout));
  return s;
}

static void load_convT4(Loader& L, const std::string& wname, int k, int pad, ConvW* out4, const float* bias) {
  for (int ph = 0; ph < 4; ++ph) { out4[ph] = L.convT_phase(wname, k, pad, ph >> 1, ph & 1); out4[ph].shift = bias; }
}

DbnetModel* dbnet_build(Ctx& ctx, const Weights& W) {
  DbnetModel* m = new DbnetModel();
  try {
    Loader L{W, m->blob, 0};
    m->stem = L.conv_padcin("backbone.stem.0.weight", 0, 4);
    m->stem.shift = L.vec("backbone.stem.0.bias");
    m->stem_ln_w = L.vec("backbone.stem.1.weight"); m->stem_ln_b = L.vec("backbone.stem.1.bias");
    const int dims[4] = {128, 256, 512, 1024}, depths[4] = {3, 3, 27, 3};
    int prev = 128;
    for (int i = 0; i < 4; ++i) { m->stages[i] = load_stage(L, "backbone.stages." + std::to_string(i) + ".", prev, dims[i], depths[i]); prev = dims[i]; }
    m->down1 = load_stage(L, "down_conv1.", 1024, 1024, 2);
    m->down2 = load_stage(L, "down_conv2.", 1024, 1024, 2);
    const int uc[6][2] = {{1024, 128}, {1152, 128}, {1152, 128}, {640, 128}, {384, 128}, {256, 64}};
    for (int i = 0; i < 6; ++i) {
      const std::string p = "upconv" + std::to_string(i + 1) + ".";
      m->up[i].blk = load_block(L, p + "conv.", uc[i][0], uc[i][1]);
      load_convT4(L, p + "upconv.weight", 2, 0, m->up[i].up, L.vec(p + "upconv.bias"));
    }
    for (int br = 0; br < 2; ++br) {
      HeadBranch& h = br == 0 ? m->binarize : m->thresh;
      const std::string p = br == 0 ? "conv_db.binarize." : "conv_db.thresh.";
      h.c0 = L.conv(p + "0.weight", 1, 1);
      if (W.has(p + "0.bias")) h.c0.shift = L.vec(p + "0.bias");
      load_convT4(L, p + "2.weight", 4, 1, h.t1, L.vec(p + "2.bias"));
      load_convT4(L, p + "4.weight", 4, 1, h.t2, L.vec(p + "4.bias"));
      h.t2_w = L.vec(p + "4.weight"); h.t2_b = L.vec(p + "4.bias");      // raw [32,1,4,4] for the fused full-resolution kernel
    }
    m->m0 = L.conv("conv_mask.0.weight", 1, 1); m->m0.shift = L.vec("conv_mask.0.bias");
    m->m2 = L.conv("conv_mask.2.weight", 1, 1); m->m2.shift = L.vec("conv_mask.2.bias");
    m->m4 = L.conv("conv_mask.4.weight", 0, 0); m->m4.shift = L.vec("conv_mask.4.bias");
    CUDA_OK(cudaDeviceSynchronize());
  } catch (...) { delete m; throw; }
  return m;
}

void dbnet_free(DbnetModel* m) { delete m; }

// ConvNeXtBlock.forward (dbnet_convnext.py:112-127).  x and out may alias for identity-shortcut blocks.
static void run_block(Exec& e, const CnBlock& b, const View& x, const View& out) {
  Arena& ws = e.ws();
  const size_t mk = ws.mark();
  View t = ws.view(x.N, x.H, x.W, b.cout);
  View hid = ws.view(x.N, x.H, x.W, 4 * b.cout);
  ConvOp op1 = Exec::op_from(b.fc1, t, hid); op1.act = ACT_GELU;
  ConvOp op2 = Exec::op_from(b.fc2, hid, out); op2.mul1 = b.gamma;
  // Operand fusion along LN -> fc1 -> GELU -> fc2 when both GEMMs run on the TMA-fed kernel: the LayerNorm kernel and fc1's
  // epilogue store the NEXT GEMM's bf16 hi/mid operands into the bytes of `t` / `hid` (same size as the fp32 tensors they
  // replace), so neither GEMM needs a split pass and the normalised / hidden activations never exist in fp32.
  const bool fuse = conv_uses_tma(op1) && conv_uses_tma(op2);
  SplitView ts, hs;
  if (fuse) { ts = Exec::alias_split(t); hs = Exec::alias_split(hid); op1.in_sv = ts; op1.out_sv = hs; op1.out.p = nullptr; op2.in_sv = hs; }
  if (b.dense) {
    View d = fuse ? ws.view(x.N, x.H, x.W, b.cout) : t;        // the dense conv's fp32 result (LN input); `t` holds the operands
    ConvOp op = Exec::op_from(b.dense_w, x, d);
    e.conv(op);
    e.layernorm(d, t, b.ln_w, b.ln_b, kLnEps, nullptr, nullptr, 1, fuse ? &ts : nullptr);
  } else {
    e.dwconv7_ln(x, t, b.dw_w, b.dw_b, b.ln_w, b.ln_b, kLnEps, fuse ? &ts : nullptr);
  }
  View sc = x;
  if (b.has_sc) {
    sc = ws.view(x.N, x.H, x.W, b.cout);
    ConvOp op = Exec::op_from(b.sc, x, sc); e.conv(op);
  }
  op2.add1 = sc;
  e.conv(op1);
  e.conv(op2);
  ws.release(mk);
}

// ConvNeXtStage.forward (dbnet_convnext.py:190-193); the last block writes into `out` (a slice of a concat buffer)
static void run_stage(Exec& e, const CnStage& s, const View& x, const View& out) {
  Arena& ws = e.ws();
  const size_t mk = ws.mark();
  View cur = x;
  if (s.has_ds) {
    View t = ws.view(x.N, x.H, x.W, x.C);
    View d = ws.view(x.N, x.H / 2, x.W / 2, s.ds.Cout);
    ConvOp op = Exec::op_from(s.ds, t, d, 2);
    // LayerNorm2d -> 2x2 stride-2 conv: the LN kernel writes the conv's bf16 hi/mid operands directly (no split pass)
    SplitView ts;
    if (conv_uses_tma(op)) { ts = Exec::alias_split(t); op.in_sv = ts; }
    e.layernorm(x, t, s.ds_ln_w, s.ds_ln_b, kLnEps, nullptr, nullptr, 1, ts.valid() ? &ts : nullptr);
    e.conv(op);
    cur = d;
  }
  for (size_t k = 0; k < s.blocks.size(); ++k) run_block(e, s.blocks[k], cur, k + 1 == s.blocks.size() ? out : cur);
  ws.release(mk);
}

// UpconvSkip.forward (dbnet_convnext.py:377-380): dense ConvNeXt block then ConvTranspose2d(k2,s2) into `out`
static void run_upconv(Exec& e, const Upconv& u, const View& x, const View& out) {
  Arena& ws = e.ws();
  const size_t mk = ws.mark();
  View y = ws.view(x.N, x.H, x.W, u.blk.cout);
  run_block(e, u.blk, x, y);
  e.convT2(u.up, y, out, [](ConvOp&) {});
  ws.release(mk);
}

void dbnet_run(Ctx& ctx, DbnetModel& m, const float* x_nchw, const uint8_t* x_u8, int n, int h, int w, float* db, float* mask,
               cudaStream_t st) {
  // every stride of the network divides 128 (coarsest map = 1/128); the reference's own pre-processing pads to 256 (imgproc.py:37-70)
  MITB_CHECK(n >= 1 && h % 128 == 0 && w % 128 == 0 && h > 0 && w > 0, "dbnet: input %dx%d must be a positive multiple of 128", h, w);
  run_with_workspace(ctx, st, [&](Exec& e) {
    Arena& ws = e.ws();
    // persistent buffers: concat inputs of the decoder. cat_k = [ up (128) | skip ]
    View cat6 = ws.view(n, h / 4, w / 4, 256);      // [up8 | h4]
    View cat5 = ws.view(n, h / 8, w / 8, 384);      // [up16 | h8]
    View cat4 = ws.view(n, h / 16, w / 16, 640);    // [up32 | h16]
    View cat3 = ws.view(n, h / 32, w / 32, 1152);   // [up64 | h32]
    View cat2 = ws.view(n, h / 64, w / 64, 1152);   // [up128 | h64]
    View h128 = ws.view(n, h / 128, w / 128, 1024);
    View up4 = ws.view(n, h / 2, w / 2, 64);
    View h4 = cat6.slice(128, 128), h8 = cat5.slice(128, 256), h16 = cat4.slice(128, 512), h32 = cat3.slice(128, 1024),
         h64 = cat2.slice(128, 1024);
    {
      const size_t mk = ws.mark();
      View x4 = ws.view(n, h, w, 4);
      if (!e.dry) {
        if (x_u8) launch_u8_to_nhwc(x_u8, n, h, w, 3, x4, 127.5f, 1.0f, 1, st);
        else launch_nchw_to_nhwc(x_nchw, n, 3, h, w, x4, st);
      }
      View s0 = ws.view(n, h / 4, w / 4, 128);
      { ConvOp op = Exec::op_from(m.stem, x4, s0, 4); e.conv(op); }
      e.layernorm(s0, s0, m.stem_ln_w, m.stem_ln_b, kLnEps);
      run_stage(e, m.stages[0], s0, h4);
      ws.release(mk);
    }
    run_stage(e, m.stages[1], h4, h8);
    run_stage(e, m.stages[2], h8, h16);
    run_stage(e, m.stages[3], h16, h32);
    run_stage(e, m.down1, h32, h64);
    run_stage(e, m.down2, h64, h128);
    run_upconv(e, m.up[0], h128, cat2.slice(0, 128));
    run_upconv(e, m.up[1], cat2, cat3.slice(0, 128));
    run_upconv(e, m.up[2], cat3, cat4.slice(0, 128));
    run_upconv(e, m.up[3], cat4, cat5.slice(0, 128));
    run_upconv(e, m.up[4], cat5, cat6.slice(0, 128));
    run_upconv(e, m.up[5], cat6, up4);
    View up8 = cat6.slice(0, 128);
    // DBHead (dbnet_convnext.py:382-407) + the caller's sigmoid on both channels (:507)
    View dbv; dbv.p = db; dbv.N = n; dbv.H = h; dbv.W = w; dbv.C = 1; dbv.cs = 2; dbv.coff = 0; dbv.planar = true;
    for (int br = 0; br < 2; ++br) {
      const HeadBranch& hb = br == 0 ? m.binarize : m.thresh;
      const size_t mk = ws.mark();
      View a = ws.view(n, h / 4, w / 4, 32), b = ws.view(n, h / 2, w / 2, 32);
      { ConvOp op = Exec::op_from(hb.c0, up8, a); op.act = ACT_SILU; e.conv(op); }
      e.convT2(hb.t1, a, b, [](ConvOp& op) { op.act = ACT_SILU; });
      View o = dbv; o.coff = br;
      if (!e.dry) launch_convT4_c1(b, hb.t2_w, hb.t2_b, br == 0 ? ACT_SIGMOID : ACT_SIGMOID2, o, st);
      ws.release(mk);
    }
    {  // conv_mask (dbnet_convnext.py:455-460)
      const size_t mk = ws.mark();
      View a = ws.view(n, h / 2, w / 2, 64), b = ws.view(n, h / 2, w / 2, 32);
      { ConvOp op = Exec::op_from(m.m0, up4, a); op.act = ACT_SILU; e.conv(op); }
      { ConvOp op = Exec::op_from(m.m2, a, b); op.act = ACT_SILU; e.conv(op); }
      View mv; mv.p = mask; mv.N = n; mv.H = h / 2; mv.W = w / 2; mv.C = 1; mv.cs = 1; mv.coff = 0; mv.planar = true;
      { ConvOp op = Exec::op_from(m.m4, b, mv); op.act = ACT_SIGMOID; e.conv(op); }
      ws.release(mk);
    }
  });
}

}  // namespace mitb
