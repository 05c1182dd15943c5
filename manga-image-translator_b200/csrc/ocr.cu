// 48px ResNet + Transformer CTC line recogniser forward (reference: ocr/model_48px_ctc.py:277-463).
// Pre-activation ResNet [4,6,8,6] (BN+ReLU folded into the consuming conv's loader or the producing conv's epilogue),
// three pre-norm encoder layers (positional encoding on q/k only, no padding mask), colour head, and the vocabulary head
// fused with log-softmax/argmax so the [N,T,V] logits are never written.
#include <math.h>
#include "exec.h"

namespace mitb {

static const float kBnEps = 1e-5f, kLnEps5 = 1e-5f;

struct OcrBlock {
  const float* bn1_s; const float* bn1_b;      // prologue of conv1
  ConvW conv1;                                 // epilogue: bn2 + relu
  ConvW conv2;
  bool has_ds = false; const float* ds_s = nullptr; const float* ds_b = nullptr; ConvW ds;
};
struct OcrTail { const float* s; const float* b; ConvW conv; };   // bnX -> relu -> convX
struct EncLayer {
  const float* n1w; const float* n1b; const float* n2w; const float* n2b;
  ConvW qk, v, out, l1, l2;
};
struct OcrModel {
  DevBlob blob;
  int vocab = 0;
  ConvW conv0_1, conv0_2;
  std::vector<OcrBlock> layer[4];
  OcrTail tail[3];                             // bn1/conv1, bn2/conv2, bn3/conv3
  OcrTail t41, t42;                            // bn4_1/conv4_1 (stride (2,1)), bn4_2/conv4_2 (pad 0) + bn4_3 epilogue
  EncLayer enc[3];
  const float* cpn_w; const float* cpn_b;
  ConvW char_pred, color;
  const float* pe = nullptr; int pe_len = 0;   // [pe_len, 320]
};

int ocr_vocab(const OcrModel& m) { return m.vocab; }

OcrModel* ocr_build(Ctx& ctx, const Weights& W) {
  OcrModel* m = new OcrModel();
  try {
    Loader L{W, m->blob, 0};
    const std::string p = "backbone.ConvNet.";
    m->conv0_1 = L.conv_padcin(p + "conv0_1.weight", 1, 4);
    L.bn_fold(p + "bn0_1.", kBnEps, &m->conv0_1.scale, &m->conv0_1.shift);      // bn0_1 + relu as conv0_1 epilogue
    m->conv0_2 = L.conv(p + "conv0_2.weight", 1, 1);
    const int nblocks[4] = {4, 6, 8, 6};
    for (int l = 0; l < 4; ++l) {
      for (int k = 0; k < nblocks[l]; ++k) {
        const std::string q = p + "layer" + std::to_string(l + 1) + "." + std::to_string(k) + ".";
        OcrBlock b;
        L.bn_fold(q + "bn1.", kBnEps, &b.bn1_s, &b.bn1_b);
        b.conv1 = L.conv(q + "conv1.weight", 1, 1);
        L.bn_fold(q + "bn2.", kBnEps, &b.conv1.scale, &b.conv1.shift);
        b.conv2 = L.conv(q + "conv2.weight", 1, 1);
        if (W.has(q + "downsample.1.weight")) {
          b.has_ds = true;
          L.bn_fold(q + "downsample.0.", kBnEps, &b.ds_s, &b.ds_b);
          b.ds = L.conv(q + "downsample.1.weight", 0, 0);
        }
        m->layer[l].push_back(b);
      }
      if (l < 3) {
        const std::string n = std::to_string(l + 1);
        L.bn_fold(p + "bn" + n + ".", kBnEps, &m->tail[l].s, &m->tail[l].b);
        m->tail[l].conv = L.conv(p + "conv" + n + ".weight", 1, 1);
      }
    }
    L.bn_fold(p + "bn4_1.", kBnEps, &m->t41.s, &m->t41.b);
    m->t41.conv = L.conv(p + "conv4_1.weight", 1, 1);
    L.bn_fold(p + "bn4_2.", kBnEps, &m->t42.s, &m->t42.b);
    m->t42.conv = L.conv(p + "conv4_2.weight", 0, 0);
    L.bn_fold(p + "bn4_3.", kBnEps, &m->t42.conv.scale, &m->t42.conv.shift);      // bn4_3 as conv4_2 epilogue
    for (int i = 0; i < 3; ++i) {
      const std::string q = "encoders.layers." + std::to_string(i) + ".";
      EncLayer& e = m->enc[i];
      e.n1w = L.vec(q + "norm1.weight"); e.n1b = L.vec(q + "norm1.bias");
      e.n2w = L.vec(q + "norm2.weight"); e.n2b = L.vec(q + "norm2.bias");
      e.qk = L.linear_rows(q + "self_attn.in_proj_weight", 0, 640); e.qk.shift = L.vec_slice(q + "self_attn.in_proj_bias", 0, 640);
      e.v = L.linear_rows(q + "self_attn.in_proj_weight", 640, 320); e.v.shift = L.vec_slice(q + "self_attn.in_proj_bias", 640, 320);
      e.out = L.conv(q + "self_attn.out_proj.weight", 0, 0); e.out.shift = L.vec(q + "self_attn.out_proj.bias");
      e.l1 = L.conv(q + "linear1.weight", 0, 0); e.l1.shift = L.vec(q + "linear1.bias");
      e.l2 = L.conv(q + "linear2.weight", 0, 0); e.l2.shift = L.vec(q + "linear2.bias");
    }
    m->cpn_w = L.vec("char_pred_norm.0.weight"); m->cpn_b = L.vec("char_pred_norm.0.bias");
    m->char_pred = L.conv("char_pred.weight", 0, 0); m->char_pred.shift = L.vec("char_pred.bias");
    m->vocab = m->char_pred.Cout;
    m->color = L.conv("color_pred1.0.weight", 0, 0); m->color.shift = L.vec("color_pred1.0.bias");
    // positional encoding table (model_48px_ctc.py:163-178).  The Python host passes the table computed by torch
    // ("pe.table", bit-identical to the reference buffer); otherwise it is recomputed here in fp32 steps.
    if (W.has("pe.table")) {
      const mitb_tensor& t = W.get("pe.table");
      MITB_CHECK(t.ndim == 2 && t.shape[1] == 320, "pe.table must be [len,320]");
      m->pe_len = (int)t.shape[0]; m->pe = L.vec("pe.table");
    } else {
      const int len = 2048, d = 320;
      std::vector<float> pe((size_t)len * d);
      const float c = (float)(-log(10000.0) / d);
      for (int i = 0; i < d / 2; ++i) {
        const float a = (float)(2 * i) * c;
        const float dv = expf(a);
        for (int t = 0; t < len; ++t) { const float arg = (float)t * dv; pe[(size_t)t * d + 2 * i] = sinf(arg); pe[(size_t)t * d + 2 * i + 1] = cosf(arg); }
      }
      float* dp = m->blob.alloc_f(pe.size());
      CUDA_OK(cudaMemcpy(dp, pe.data(), pe.size() * sizeof(float), cudaMemcpyHostToDevice));
      m->pe = dp; m->pe_len = len;
    }
    CUDA_OK(cudaDeviceSynchronize());
  } catch (...) { delete m; throw; }
  return m;
}

void ocr_free(OcrModel* m) { delete m; }

// BN(+ReLU) prologue of whichever conv consumes a tensor next (pre-activation ResNet: applied by the PRODUCER's epilogue when fused)
struct NextBn { const float* s = nullptr; const float* b = nullptr; int relu = 0; };

// BasicBlock.forward (model_48px_ctc.py:389-403); x -> out may alias when there is no downsample path.
// Operand fusion: `xs` (valid or not) is relu(bn1(x)) already split into bf16 hi/mid by x's producer; conv1's epilogue (bn2 + relu)
// writes conv2's operands directly; conv2's epilogue writes the fp32 residual stream AND, into `outs`, the next consumer's
// operands relu(bn_next(out)).  Every fusion is taken only when both ends run on the TMA-fed kernel.
static void run_block(Exec& e, const OcrBlock& b, const View& x, const View& out, const SplitView& xs, const NextBn& nxt, SplitView* outs) {
  Arena& ws = e.ws();
  const size_t mk = ws.mark();
  View y1 = ws.view(x.N, x.H, x.W, b.conv1.Cout);
  ConvOp op1 = Exec::op_from(b.conv1, x, y1); op1.act = ACT_RELU;
  if (xs.valid()) op1.in_sv = xs; else { op1.in_scale = b.bn1_s; op1.in_shift = b.bn1_b; op1.in_relu = 1; }
  View res = x;
  ConvOp op2 = Exec::op_from(b.conv2, y1, out);
  if (conv_uses_tma(op1) && conv_uses_tma(op2)) { SplitView ys = Exec::alias_split(y1); op1.out_sv = ys; op1.out.p = nullptr; op2.in_sv = ys; }
  e.conv(op1);
  if (b.has_ds) {
    res = ws.view(x.N, x.H, x.W, b.ds.Cout);
    ConvOp op = Exec::op_from(b.ds, x, res); op.in_scale = b.ds_s; op.in_shift = b.ds_b; op.in_relu = 0; e.conv(op);
  }
  op2.add1 = res;
  if (outs && outs->valid() && conv_uses_tma(op2)) { op2.out_sv = *outs; op2.os_scale = nxt.s; op2.os_shift = nxt.b; op2.os_relu = nxt.relu; }
  else if (outs) *outs = SplitView();
  e.conv(op2);
  ws.release(mk);
}

void ocr_run(Ctx& ctx, OcrModel& m, const float* x_nchw, const uint8_t* x_u8, int n, int wp, int* idx, float* logprob,
             float* colors, cudaStream_t st) {
  MITB_CHECK(n >= 1 && wp >= 12, "ocr: bad input n=%d wp=%d", n, wp);
  const int w1 = wp / 2, w2 = w1 / 2, w3 = w2 + 1, T = w2 - 1;
  MITB_CHECK(T >= 1 && T <= m.pe_len, "ocr: %d timesteps unsupported", T);
  run_with_workspace(ctx, st, [&](Exec& e) {
    Arena& ws = e.ws();
    View x4 = ws.view(n, 48, wp, 4);
    if (!e.dry) {
      if (x_u8) launch_u8_to_nhwc(x_u8, n, 48, wp, 3, x4, 127.5f, 127.5f, 0, st);
      else launch_nchw_to_nhwc(x_nchw, n, 3, 48, wp, x4, st);
    }
    View a = ws.view(n, 48, wp, 40), b = ws.view(n, 48, wp, 40);
    { ConvOp op = Exec::op_from(m.conv0_1, x4, a); op.act = ACT_RELU; e.conv(op); }
    { ConvOp op = Exec::op_from(m.conv0_2, a, b); e.conv(op); }
    View cur = ws.view(n, 24, w1, 40);
    e.avgpool(b, cur, 0);
    const int chans[4] = {80, 160, 320, 320};
    SplitView cur_s;                              // relu(bn_next(cur)) as bf16 hi/mid operands, when cur's producer wrote them
    for (int l = 0; l < 4; ++l) {
      SplitView layer_s = ws.split_view(cur.N, cur.H, cur.W, chans[l]);       // operands of the residual stream inside this layer
      for (size_t k = 0; k < m.layer[l].size(); ++k) {
        const OcrBlock& blk = m.layer[l][k];
        NextBn nxt;                               // who consumes this block's output: the next block's conv1, else the layer's tail conv
        if (k + 1 < m.layer[l].size()) { nxt.s = m.layer[l][k + 1].bn1_s; nxt.b = m.layer[l][k + 1].bn1_b; nxt.relu = 1; }
        else if (l < 3) { nxt.s = m.tail[l].s; nxt.b = m.tail[l].b; nxt.relu = 1; }
        else { nxt.s = m.t41.s; nxt.b = m.t41.b; nxt.relu = 1; }
        SplitView outs = layer_s;
        if (blk.has_ds || cur.C != chans[l]) {
          View nx = ws.view(cur.N, cur.H, cur.W, chans[l]);
          run_block(e, blk, cur, nx, cur_s, nxt, &outs);
          cur = nx;
        } else {
          run_block(e, blk, cur, cur, cur_s, nxt, &outs);
        }
        cur_s = outs;
      }
      if (l < 3) {
        View t = ws.view(cur.N, cur.H, cur.W, chans[l]);
        ConvOp op = Exec::op_from(m.tail[l].conv, cur, t);
        if (cur_s.valid() && conv_uses_tma(op)) op.in_sv = cur_s; else { op.in_scale = m.tail[l].s; op.in_shift = m.tail[l].b; op.in_relu = 1; }
        cur_s = SplitView();
        if (l == 2) {                             // conv3 feeds layer4.0.conv1 directly (no pool, no downsample path): emit its operands
          SplitView ts = ws.split_view(cur.N, cur.H, cur.W, chans[l]);
          if (conv_uses_tma(op) && !m.layer[3][0].has_ds) { op.out_sv = ts; op.os_scale = m.layer[3][0].bn1_s; op.os_shift = m.layer[3][0].bn1_b; op.os_relu = 1; cur_s = ts; }
        }
        e.conv(op);
        if (l == 0) { View pl = ws.view(n, 12, w2, chans[l]); e.avgpool(t, pl, 0); cur = pl; }
        else if (l == 1) { View pl = ws.view(n, 6, w3, chans[l]); e.avgpool(t, pl, 1); cur = pl; }
        else cur = t;
      }
    }
    View f1 = ws.view(n, 3, w3, 320);
    View x = ws.view(n, 1, T, 320);               // tokens [n*T, 320]
    {
      ConvOp op41 = Exec::op_from(m.t41.conv, cur, f1); op41.sy = 2; op41.sx = 1;
      if (cur_s.valid() && conv_uses_tma(op41)) op41.in_sv = cur_s; else { op41.in_scale = m.t41.s; op41.in_shift = m.t41.b; op41.in_relu = 1; }
      ConvOp op42 = Exec::op_from(m.t42.conv, f1, x);
      if (conv_uses_tma(op41) && conv_uses_tma(op42)) {      // conv4_1's epilogue applies bn4_2 + relu and writes conv4_2's operands
        SplitView fs = Exec::alias_split(f1);
        op41.out_sv = fs; op41.os_scale = m.t42.s; op41.os_shift = m.t42.b; op41.os_relu = 1; op41.out.p = nullptr; op42.in_sv = fs;
      } else { op42.in_scale = m.t42.s; op42.in_shift = m.t42.b; op42.in_relu = 1; }
      e.conv(op41);
      e.conv(op42);
    }
    // ---- transformer encoder (model_48px_ctc.py:253-274)
    View z = ws.view(n, 1, T, 320), zp = ws.view(n, 1, T, 320), qk = ws.view(n, 1, T, 640), vv = ws.view(n, 1, T, 320),
         att = ws.view(n, 1, T, 320), hid = ws.view(n, 1, T, 1280);
    for (int i = 0; i < 3; ++i) {
      const EncLayer& L = m.enc[i];
      e.layernorm(x, z, L.n1w, L.n1b, kLnEps5, m.pe, &zp, T);
      { ConvOp op = Exec::op_from(L.qk, zp, qk); e.conv(op); }
      { ConvOp op = Exec::op_from(L.v, z, vv); e.conv(op); }
      if (!e.dry) launch_attention(qk.p, vv.p, att.p, n, T, 8, 40, st);
      { ConvOp op = Exec::op_from(L.out, att, x); op.add1 = x; e.conv(op); }
      e.layernorm(x, z, L.n2w, L.n2b, kLnEps5);
      {
        ConvOp o1 = Exec::op_from(L.l1, z, hid); o1.act = ACT_GELU;
        ConvOp o2 = Exec::op_from(L.l2, hid, x); o2.add1 = x;
        if (conv_uses_tma(o1) && conv_uses_tma(o2)) { SplitView hs = Exec::alias_split(hid); o1.out_sv = hs; o1.out.p = nullptr; o2.in_sv = hs; }
        e.conv(o1);
        e.conv(o2);
      }
    }
    // ---- heads (model_48px_ctc.py:452-453, 460-463)
    View cv; cv.p = colors; cv.N = n; cv.H = 1; cv.W = T; cv.C = 6; cv.cs = 6; cv.coff = 0;
    { ConvOp op = Exec::op_from(m.color, x, cv); op.act = ACT_CLAMP01; e.conv(op); }
    e.layernorm(x, z, m.cpn_w, m.cpn_b, kLnEps5);
    if (!e.dry) launch_affine_act(z, z, nullptr, nullptr, ACT_GELU, st);
    const int rows = n * T;
    View dummy = z; dummy.C = m.vocab; dummy.cs = m.vocab; dummy.p = nullptr;
    ConvOp vop = Exec::op_from(m.char_pred, z, dummy);
    const int nblk = conv_stat_blocks(vop);
    float* pmax = ws.alloc_f((size_t)rows * nblk); float* psum = ws.alloc_f((size_t)rows * nblk);
    int* pidx = (int*)ws.alloc((size_t)rows * nblk * sizeof(int));
    vop.stat_max = pmax; vop.stat_sum = psum; vop.stat_idx = pidx; vop.stat_ld = nblk;
    e.conv(vop);
    if (!e.dry) launch_rowstat_final(pmax, psum, pidx, rows, nblk, idx, logprob, st);
  });
}

}  // namespace mitb
