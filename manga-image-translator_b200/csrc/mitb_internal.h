// Internal declarations shared by the kernels and the network drivers of libmitb.
// Layout convention: activations are NHWC fp32 "views" (a channel slice of a wider tensor), so channel
// concatenation (DBNet skip connections, LaMa local|global halves) never costs a copy.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <map>
#include <string>
#include <vector>
#include <stdexcept>

#include "../../include/mitb.h"

namespace mitb {

// ------------------------------------------------------------------ errors
struct Error : std::runtime_error { using std::runtime_error::runtime_error; };
#define MITB_CHECK(cond, ...)                                                          \
  do { if (!(cond)) { char _b[512]; snprintf(_b, sizeof _b, __VA_ARGS__);              \
       throw ::mitb::Error(std::string(__FILE__) + ":" + std::to_string(__LINE__) + ": " + _b); } } while (0)
#define CUDA_OK(expr)                                                                  \
  do { cudaError_t _e = (expr); if (_e != cudaSuccess)                                 \
       throw ::mitb::Error(std::string(__FILE__) + ":" + std::to_string(__LINE__) + ": " #expr ": " + \
                           cudaGetErrorString(_e)); } while (0)

// ------------------------------------------------------------------ tensor view
struct View {              // NHWC slice: element (n,y,x,c) at p[((n*H+y)*W+x)*cs + coff + c]
  float* p = nullptr;
  int N = 0, H = 0, W = 0, C = 0;   // C = channels in this view
  int cs = 0, coff = 0;             // channel stride of the backing tensor, offset of this slice
  bool planar = false;              // NCHW instead: element at p[((n*cs + coff + c)*H + y)*W + x]
  View slice(int off, int c) const { View v = *this; v.coff = coff + off; v.C = c; return v; }
  size_t pixels() const { return (size_t)N * H * W; }
};

// bf16 hi/mid operand copies of an activation tensor for the tensor-core kernel (x ~ hi + mid, |x - hi - mid| <= 2^-17 |x|):
// two dense bf16 NHWC tensors [N][Hp][Wp][C]; logical pixel (y, x) lives at (y + pt, x + pl).  A halo (pt/pl > 0, Hp > H + pt)
// holds the reflect padding of the consuming conv (zero padding needs none: TMA out-of-bounds fill).
struct SplitView {
  uint16_t* hi = nullptr; uint16_t* mid = nullptr;
  int N = 0, H = 0, W = 0, C = 0;                 // logical grid, channels per pixel (pitch)
  int pt = 0, pl = 0, Hp = 0, Wp = 0;
  bool valid() const { return hi != nullptr; }
  size_t elems() const { return (size_t)N * Hp * Wp * C; }
};

// ------------------------------------------------------------------ bump arena with mark/release
struct Arena {
  char* base = nullptr; size_t cap = 0, off = 0, peak = 0; bool dry = false;
  float* alloc_f(size_t n) { return (float*)alloc(n * sizeof(float)); }
  void* alloc(size_t bytes) {
    size_t a = (off + 255) & ~size_t(255);
    off = a + bytes; if (off > peak) peak = off;
    if (dry) return (void*)(uintptr_t)(0x1000 + a);      // fake, never dereferenced
    MITB_CHECK(off <= cap, "workspace overflow (%zu > %zu)", off, cap);
    return base + a;
  }
  size_t mark() const { return off; }
  void release(size_t m) { off = m; }
  View view(int N, int H, int W, int C, bool planar = false) {
    View v; v.p = alloc_f((size_t)N * H * W * C); v.N = N; v.H = H; v.W = W; v.C = C; v.cs = C; v.coff = 0;
    v.planar = planar; return v;
  }
  SplitView split_view(int N, int H, int W, int C, int pt = 0, int pb = 0, int pl = 0, int pr = 0) {
    SplitView s; s.N = N; s.H = H; s.W = W; s.C = C; s.pt = pt; s.pl = pl; s.Hp = H + pt + pb; s.Wp = W + pl + pr;
    s.hi = (uint16_t*)alloc(2 * s.elems() * sizeof(uint16_t)); s.mid = s.hi + s.elems();
    return s;
  }
};

// ------------------------------------------------------------------ conv op
enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_GELU = 2, ACT_SILU = 3, ACT_SIGMOID = 4, ACT_SIGMOID2 = 5, ACT_CLAMP01 = 6 };
enum Pad { PAD_ZERO = 0, PAD_REFLECT = 1 };
constexpr int kMaxTaps = 49;

// conv weight handle produced at load time
struct ConvW {
  const float* w = nullptr;           // [ntaps*Cin][ldw] K-major rows, ldw = round4(Cout)
  int ldw = 0, Cin = 0, Cout = 0, ntaps = 1;
  int8_t tdy[kMaxTaps] = {0}, tdx[kMaxTaps] = {0};   // input offset of each tap relative to (oy*sy, ox*sx)
  const float* scale = nullptr; const float* shift = nullptr;   // folded BN / bias (may be null)
  // tensor-core copies of the weights (conv_tc.cu): bf16 hi/mid [tc_npad][tc_kpad], K-major; null -> SIMT path only
  const uint16_t* wh = nullptr; const uint16_t* wm = nullptr; int tc_bn = 0, tc_kpad = 0, tc_npad = 0;
  // per-tap channel-padded copies [tc_npad][ntaps*tc_cp] for the TMA-fed kernel when Cin % 64 != 0 (null otherwise)
  const uint16_t* whp = nullptr; const uint16_t* wmp = nullptr; int tc_cp = 0;
  // Cin = 4 stems on the tensor cores: weights packed [tc_npad][kh*64], k = ky*64 + kx*8 + c (kx < kw <= 8, c < 4, rest zero): one
  // K block per kernel row, fed by an OVERLAPPING-stride tensor map over the 8-channel-padded input (conv_tma.cu)
  const uint16_t* w8h = nullptr; const uint16_t* w8m = nullptr; int w8_kh = 0, w8_kw = 0;
};

// Alignment: the base pointers of in / out / add0 / add1 (and of every split tensor) must be 16-byte aligned, in_scale / in_shift
// too: the SIMT kernel reads and writes float4 whenever cs and coff are multiples of 4 and the split kernels move 16-byte packs.
// scale / shift / mul1 / os_scale / os_shift need 4 bytes (the tensor-core epilogue reads them as float2 only when 8-byte aligned).
struct ConvOp {
  View in, out;                       // out grid may be larger than the logical (Ho,Wo) grid (transposed phases)
  ConvW wt;                           // weights and taps; the epilogue reads scale / shift below, not wt's
  int sy = 1, sx = 1, pad = PAD_ZERO;
  int Ho = 0, Wo = 0;                 // logical output grid of this launch
  int oy_mul = 1, oy_add = 0, ox_mul = 1, ox_add = 0;   // out pixel = (oy*oy_mul+oy_add, ox*ox_mul+ox_add)
  // prologue on the input: relu?(x*in_scale[c]+in_shift[c]) ; padding contributes 0 AFTER the transform
  const float* in_scale = nullptr; const float* in_shift = nullptr; int in_relu = 0;
  // epilogue: v = acc (+add0) ; v = v*scale[c]+shift[c] ; v = act(v) ; v *= mul1[c] ; v += add1
  View add0, add1;                    // same pixel grid as out; p==nullptr when unused
  // Optional output-sparsity hint (conv7_thin only): planar fp32 [N][Ho][Wo]; a CTA tile whose entries are all zero writes zeros
  // instead of computing - for a conv whose only consumer multiplies / selects by this very mask (LaMa's final blend).
  const float* tile_mask = nullptr;
  const uint8_t* tile_mask_u8 = nullptr;   // the same hint from a uint8 mask: "non-zero" means >= 128 (mask / 255 >= 0.5)
  // Output-sparsity hint for the TMA conv kernel: uint8 [N][Ho][Wo] over this launch's LOGICAL output grid; output tiles without a
  // non-zero entry are skipped (left unwritten).  The caller guarantees that nothing it still needs depends on skipped pixels.
  const uint8_t* need_px = nullptr;
  const float* scale = nullptr; const float* shift = nullptr; const float* mul1 = nullptr;   // initialised from wt, callers override
  int act = ACT_NONE;
  // TMA-path operand fusion (only legal when conv_uses_tma() holds for the op):
  //  * in_sv valid  -> the input already exists as bf16 hi/mid (written by its producer); channels [in_sv_coff, +in.C) of it are
  //                    this conv's input, `in` then only carries the shape; the split pass is skipped;
  //  * out_sv valid -> the epilogue ALSO stores the result as bf16 hi/mid at channel offset out_sv_coff of out_sv (interior only;
  //                    launch_split_halo() fills a reflect halo); out.p may then be null (no fp32 store);
  //  * os_scale/os_shift/os_relu: the consumer's BN(+ReLU) prologue applied to the value before it is split (pre-activation ResNet).
  SplitView in_sv; int in_sv_coff = 0;
  SplitView out_sv; int out_sv_coff = 0;
  const float* os_scale = nullptr; const float* os_shift = nullptr; int os_relu = 0;
  // optional second K segment accumulated into the same output (FFC: conv1x1(U) + conv3x3_{l->g}(x_l)): pre-split input only.
  // The weight rows of segment 2 follow those of segment 1 in wt.wh / wt.wm (K-major, both Cin multiples of 64; Exec::op_from2).
  struct Seg2 { SplitView sv; int coff = 0, C = 0, ntaps = 0, pad = PAD_ZERO; int8_t tdy[kMaxTaps] = {0}, tdx[kMaxTaps] = {0}; } seg2;
  // optional fused row statistics (vocabulary head): no tensor output, per (row, column-block) partials
  float* stat_max = nullptr; float* stat_sum = nullptr; int* stat_idx = nullptr; int stat_ld = 0;
};

// conv.cu: which kernel runs an op.  conv_plan() is the only place that decides it; launch_conv() validates the op, runs the
// planned kernel under the plan's profiler class, and the predicates below are derived from the plan.
enum ConvKernel { CK_SIMT = 1, CK_FEWOUT, CK_THIN, CK_GATHER, CK_GATHER_SPLITK, CK_TMA, CK_STEM8 };
struct ConvPlan {
  ConvKernel kernel = CK_SIMT;
  int splits = 1;                     // split-K factor of the gather kernel
  const char* prof = "conv_simt";     // profiler class
  bool sparse = false;                // output-sparse launch: the executed work depends on device data, no flop / byte claim
};
ConvPlan conv_plan(const ConvOp& op);
void launch_conv(const ConvOp& op, cudaStream_t st);
bool conv_uses_tma(const ConvOp& op);      // true when launch_conv() will run this op on the TMA-fed tensor-core kernel
bool conv_tma_capable(const ConvOp& op);   // the op CAN run there (launch_conv() does so whenever in_sv / out_sv / seg2 is set)
int conv_stat_blocks(const ConvOp& op);    // number of column blocks the row-stat epilogue writes per row
// the kernels' entry points: *_supported() says whether the kernel can run the op, launch_conv_*() runs it as planned
bool conv_thin_supported(const ConvOp& op);                         // conv_thin.cu
void launch_conv_thin(const ConvOp& op, cudaStream_t st);
void launch_conv_simt(const ConvOp& op, bool fewout, cudaStream_t st);   // conv_simt.cu
bool conv_tc_supported(const ConvOp& op);                           // conv_tc.cu: register-gather wgmma kernel
void launch_conv_tc(const ConvOp& op, int splits, cudaStream_t st);
bool conv_tma_supported(const ConvOp& op);                          // conv_tma.cu: TMA-fed wgmma kernel
bool conv_stem8_supported(const ConvOp& op);
void launch_conv_tma(const ConvOp& op, bool stem, cudaStream_t st);   // stem: a refused stem map disables stem8, runs launch_conv() again
// weight tensor map (conv_tma.cu): bf16 [rows][kdim] K-major, box {64 k, bn}, 128-byte swizzle; rows beyond `rows` are zero filled
void make_w_tmap(CUtensorMap* m, const uint16_t* base, int kdim, int rows, int bn);
// Host-side record of what launch_conv() ran (test hook mitb_test_conv): null by default, and nothing is recorded then.
// Epilogue signature: which parts of the fused conv epilogue a launch has (tc_common.cuh: epi_sig).  EPI_GENERIC tests every
// part at run time.
enum EpiSig : int {
  EPI_ADD0 = MITB_EPI_ADD0, EPI_SCALE = MITB_EPI_SCALE, EPI_SHIFT = MITB_EPI_SHIFT, EPI_MUL1 = MITB_EPI_MUL1, EPI_ADD1 = MITB_EPI_ADD1,
  EPI_OUT = MITB_EPI_OUT, EPI_OS = MITB_EPI_OS, EPI_OS_AFFINE = MITB_EPI_OS_AFFINE, EPI_OS_RELU = MITB_EPI_OS_RELU, EPI_GENERIC = MITB_EPI_GENERIC
};
// epi_sig: the staged epilogue's signature (EpiSig, tc_common.cuh) that ran, -1 for other epilogues and kernels.
struct ConvTrace { int kernel = 0, bn = 0, splits = 1, vec2 = -1, tma_act = -2, split_reused = 0, convs = 0, staged = -1, epi_sig = -1; };
extern ConvTrace* g_conv_trace;
inline void conv_trace(int kernel, int bn, int splits, int vec2, int tma_act, bool reused, int staged = -1, int epi_sig = -1) {
  if (!g_conv_trace) return;
  ConvTrace& t = *g_conv_trace;
  t.kernel = kernel; t.bn = bn; t.splits = splits; t.vec2 = vec2; t.tma_act = tma_act; t.split_reused += reused ? 1 : 0; ++t.convs;
  t.staged = staged; t.epi_sig = epi_sig;
}
// TMA conv epilogue signatures (conv_tma.cu): g_epi_specialise 1 runs a staged launch on its signature's own kernel where one is
// instantiated, 0 on the generic one; -1 until epi_specialise() reads MITB_EPI_GENERIC (=1: 0).  Test hook mitb_set_epi_specialise.
// staged_epi_sig() is the signature a staged launch runs with.
extern int g_epi_specialise;
bool epi_specialise();
int staged_epi_sig(int act, int sig);
int epi_sig_list(int* act, int* sig, int cap);     // the (activation, signature) pairs with a kernel of their own; returns their count
extern int g_conv_force_bn;                // non-zero: the TMA kernel's N tile (must be one of choose_bn's candidates); test hook only
bool conv_tma_bn_candidate(int Cout, int bn);
bool conv_tc_enabled();
bool conv_tma_enabled();
void conv_tma_set_enabled(bool on);
// fill the reflect halo of channels [coff, coff+C) of a split tensor from its interior (pad <= 3)
void launch_split_halo(const SplitView& sv, int coff, int C, cudaStream_t st);
// fp32 NHWC view -> split tensor (channels [coff, coff+in.C)), optional BN+ReLU prologue, halo by reflection
void launch_split(const View& in, const SplitView& sv, int coff, const float* in_scale, const float* in_shift, int in_relu, cudaStream_t st);
void launch_rowstat_final(const float* pmax, const float* psum, const int* pidx, int rows, int nblk,
                          int* idx, float* logprob, cudaStream_t st);

// weight repack: dst[(t*Cin+c)*ldw + co] = src[co*s_co + c*s_c + ky[t]*s_ky + kx[t]*s_kx] (zero for co>=Cout)
void launch_repack(float* dst, const float* src, int Cout, int Cin, int ntaps, const int* ky, const int* kx,
                   long s_co, long s_c, long s_ky, long s_kx, int ldw, cudaStream_t st);

// ------------------------------------------------------------------ other kernels
// osv (optional): write the result as the consumer conv's bf16 hi/mid operands (dense, halo-free) INSTEAD of fp32 `out`
void launch_layernorm(const View& in, const View& out, const float* w, const float* b, float eps,
                      const float* pe /*[T,C] added into out2*/, const View* out2, int T, cudaStream_t st, const SplitView* osv = nullptr);
void launch_dwconv7_ln(const View& in, const View& out, const float* wdw /*[49][C]*/, const float* bdw,
                       const float* lnw, const float* lnb, float eps, cudaStream_t st, const SplitView* osv = nullptr);
void launch_avgpool(const View& in, const View& out, int mode /*0: 2x2s2, 1: k2 s(2,1) p(0,1)*/, cudaStream_t st);
// MaxPool2d(3, 2, 1); out.p may be null when osv (the consumer conv's dense bf16 hi/mid operands) is given
void launch_maxpool3x3s2(const View& in, const View& out, cudaStream_t st, const SplitView* osv = nullptr);
void launch_convT4_c1(const View& in, const float* w, const float* bias, int act, const View& out, cudaStream_t st);   // Cin 32 or 16
void launch_nchw_to_nhwc(const float* src, int N, int C, int H, int W, const View& dst, cudaStream_t st);
void launch_nhwc_to_nchw(const View& src, float* dst, cudaStream_t st);
void launch_u8_to_nhwc(const uint8_t* src, int N, int H, int W, int C, const View& dst, float mul, float add,
                       int div_first, cudaStream_t st);
void launch_affine_act(const View& in, const View& out, const float* scale, const float* shift, int act,
                       cudaStream_t st);
void launch_attention(const float* qk /*[N*T,2D]*/, const float* v /*[N*T,D]*/, float* out /*[N*T,D]*/,
                      int N, int T, int heads, int hd, cudaStream_t st);
void launch_lama_pack_input(const float* img, const float* mask, int N, int H, int W, const View& dst, cudaStream_t st);
void launch_lama_blend(const View& pred, const float* img, const float* mask, float* out, cudaStream_t st);
void launch_lama_pack_u8(const uint8_t* img, const uint8_t* mask, int H, int W, const View& dst, float* maskf, cudaStream_t st);
void launch_lama_blend_u8(const View& pred, const uint8_t* img, const uint8_t* mask, uint8_t* out, int composite, cudaStream_t st);
// maskrefine.cu: mask refinement (SURVEY 8f N1): cv2-exact uint8 bilinear resize, rectangle cuts, connected components with stats,
// the batched DenseCRF of refine_mask, per-line ellipse dilation
void launch_resize_linear_u8(const uint8_t* src, int sh, int sw, int cn, uint8_t* dst, int dh, int dw, int binarize, cudaStream_t st);
void launch_cut_rects(uint8_t* mask, int h, int w, const int* rects, int n, cudaStream_t st);
void launch_cc_label(const uint8_t* mask, int h, int w, int* labels, int* stats, int* ncomp, int cap, int* scratch, cudaStream_t st);
void launch_owner_map(const int* labels, const int* owner, int n, int* omap, cudaStream_t st);
size_t crf_workspace_bytes(long npix, long nslots2, long nslots5);
void launch_crf(const int* lines2, const int* lines5, int nlines, const uint8_t* img, const int* omap, int img_w, int max_pix, int max_cap2, int max_cap5,
                long npix, long nslots2, long nslots5, int iters, float sxy_g, float w_g, float sxy_b, float srgb, float w_b, float u_on, void* work,
                uint8_t* refined, int* err, cudaStream_t st);
void launch_dilate_lines(const int* lines, int nlines, int max_pix2, const int* omap, const uint8_t* refined, const uint8_t* se, int img_w,
                         uint8_t* final_mask, cudaStream_t st);
void launch_dilate_se(const uint8_t* src, int h, int w, const uint8_t* se, int ksize, uint8_t* dst, cudaStream_t st);
// ops.cu: need maps of LaMa's decoder (which pixels of each upsampling stage can reach a hole pixel of the final blend)
void launch_need_from_mask(const float* mask_f, const uint8_t* mask_u8, int H, int W, int radius, uint8_t* need, cudaStream_t st);
void launch_need_pool2(const uint8_t* src, int H, int W, uint8_t* pooled /*[H/2][W/2]*/, uint8_t* dilated /*[H/2][W/2], radius 1, may be null*/, cudaStream_t st);
// warp.cu: perspective crops of text lines into the OCR chunk canvas (cv2.warpPerspective + rotate, bit-exact) and greedy CTC collapse
void launch_warp_lines(const uint8_t* page, int H, int W, const double* lines /*[n][16]*/, int n, uint8_t* canvas, int canvas_h, int canvas_w,
                       cudaStream_t st);
void launch_textline_pairs(const double* quads /*[n][16]*/, int n, const double* params6 /*host*/, uint8_t* adj /*[n][n]*/, cudaStream_t st);
void launch_ctc_collapse(const int* argmax, const float* logprob, const float* colors, int n, int T, int* counts, int* steps, int* chars,
                         float* lp_out, float* col_out, cudaStream_t st);
void launch_mpe_tables(const uint8_t* small /*[n,256,256] INTER_AREA-reduced mask*/, int n, int* rel_pos, int* direct, cudaStream_t st);
void launch_mpe_add(const View& x, const int* rel_pos, const int* direct, int th, int tw, const float* mask,
                    const float* table, const float* dirw, float a5, float a6, cudaStream_t st);

// real 2-D FFT of planar tensors, norm='ortho' (spectrum planes interleaved c0_re,c0_im,c1_re,...)
struct FftPlan;
FftPlan* fft_plan_get(int n);          // cached per length, lives for the process
void launch_rfft2(const View& in /*planar [C][h][w]*/, const View& spec /*planar [2C][h][w/2+1]*/, float2* tmp,
                  cudaStream_t st);
void launch_irfft2(const View& spec, const View& out, const View* add /*planar, optional residual*/, float2* tmp,
                   cudaStream_t st);

// channel-vectorised NHWC variant (fft_nhwc.cu): h, w must be {2,3,5}-smooth and <= 512, C even
bool fft_nhwc_supported(int h, int w, int C);
void launch_rfft2_nhwc(const View& in, const SplitView* spec_sv, float* spec_f, float2* T, cudaStream_t st);
void launch_irfft2_nhwc(const View& spec, const View& out, const SplitView* out_sv, int sv_coff, const View* add, float2* T, cudaStream_t st);
// Host-side record of what the last FFT launch ran (test hook mitb_test_fft): null by default, and nothing is recorded then.
// tma / box_rows: -1 on the planar path; P / CB: 0 on the NHWC path.
struct FftTrace {
  int h_nst = 0, h_radix[16] = {0}, w_nst = 0, w_radix[16] = {0};
  int rows_tma = -1, rows_box_rows = -1, cols_tma = -1, cols_box_rows = -1, P = 0, CB = 0;
};
extern FftTrace* g_fft_trace;
extern bool g_fft_force_plain;         // NHWC FFT: plain loads wherever the TMA box would run (test hook only)

// ------------------------------------------------------------------ weights
struct Weights {
  std::map<std::string, mitb_tensor> t;
  const mitb_tensor& get(const std::string& name) const {
    auto it = t.find(name); MITB_CHECK(it != t.end(), "missing weight '%s'", name.c_str()); return it->second;
  }
  bool has(const std::string& name) const { return t.count(name) != 0; }
};

struct DevBlob {                       // owning device allocation for repacked weights
  std::vector<void*> ptrs;
  float* alloc_f(size_t n) { void* p = nullptr; CUDA_OK(cudaMalloc(&p, (n ? n : 1) * sizeof(float))); ptrs.push_back(p); return (float*)p; }
  void free_all() { for (void* p : ptrs) cudaFree(p); ptrs.clear(); }
  ~DevBlob() { free_all(); }
};

void conv_tc_prepare(ConvW& cw, DevBlob& blob, cudaStream_t st);   // build the bf16 hi/mid tensor-core weight copies
void conv_tc_set_enabled(bool on);

struct Loader {                        // helpers used by the network builders at load time
  const Weights& W; DevBlob& blob; cudaStream_t st;
  // PyTorch Conv2d weight [Cout,Cin,kh,kw] -> K-major; taps enumerated row-major with offsets (ky-pad_y, kx-pad_x)
  ConvW conv(const std::string& wname, int pad_y, int pad_x);
  // concatenate several Conv2d weights along Cin (same Cout/kh/kw)
  ConvW conv_cat_cin(const std::vector<std::string>& wnames, int pad_y, int pad_x);
  // ConvTranspose2d weight [Cin,Cout,kh,kw], stride 2: phase (py,px) sub-kernel
  ConvW convT_phase(const std::string& wname, int k, int pad, int py, int px);
  // rows [r0, r0+nr) of a Linear weight [out,in] as a 1x1 conv (packed in_proj of nn.MultiheadAttention)
  ConvW linear_rows(const std::string& wname, int r0, int nr);
  const float* vec_slice(const std::string& name, int off, int n);
  ConvW conv_padcin(const std::string& wname, int pad, int cin_pad);   // zero-pad input channels (RGB -> 4)
  // tensor-core-only weight whose K rows are those of `a` followed by those of `b` (same Cout): two K segments of one launch
  ConvW cat_k(const ConvW& a, const ConvW& b);
  const float* vec(const std::string& name);                    // copy a 1-D tensor
  const float* vec_tiled(const std::string& name, int reps);
  void bn_fold(const std::string& prefix, float eps, const float** scale, const float** shift);
  // Conv2d (no bias, zero padding `pad`) followed by an eval BatchNorm: the BN scale is folded into the fp32 K-major weights before
  // the tensor-core copies are made, the BN shift becomes ConvW::shift (scale stays null).  For epilogues that add a residual
  // BEFORE the affine (v = acc + add0; v*scale + shift): post-activation ResNet blocks, relu(bn2(conv2(.)) + identity).
  ConvW conv_bn(const std::string& wname, const std::string& bn_prefix, int pad, float eps);
  float scalar(const std::string& name);
};

// ------------------------------------------------------------------ networks
struct Ctx;
struct DbnetModel; struct OcrModel; struct LamaModel;
DbnetModel* dbnet_build(Ctx&, const Weights&);
void dbnet_free(DbnetModel*);
void dbnet_run(Ctx&, DbnetModel&, const float* x_nchw, const uint8_t* x_u8, int n, int h, int w, float* db,
               float* mask, cudaStream_t st);
struct DbnetR34Model;
DbnetR34Model* dbnet_r34_build(Ctx&, const Weights&);
void dbnet_r34_free(DbnetR34Model*);
void dbnet_r34_run(Ctx&, DbnetR34Model&, const float* x_nchw, const uint8_t* x_u8, int n, int h, int w, float* db, float* mask,
                   cudaStream_t st);
OcrModel* ocr_build(Ctx&, const Weights&);
void ocr_free(OcrModel*);
void ocr_run(Ctx&, OcrModel&, const float* x_nchw, const uint8_t* x_u8, int n, int wp, int* idx, float* logprob,
             float* colors, cudaStream_t st);
int ocr_vocab(const OcrModel&);
LamaModel* lama_build(Ctx&, const Weights&);
void lama_free(LamaModel*);
void lama_set_sparse_decoder(int on);   // output-sparse LaMa decoder (skip tiles the final blend cannot see); default on
void lama_set_ffc_mode(int mode);     // 0 generic planar FFC path, 1 fused NHWC path when no layer needs split-K (default), 2 fused whenever capable
struct LamaU8Io { const uint8_t* img = nullptr; const uint8_t* mask = nullptr; uint8_t* out = nullptr; int composite = 0; };
void lama_run(Ctx&, LamaModel&, const float* img, const float* mask, const int* rel_pos, const int* direct, int th,
              int tw, int n, int h, int w, float* out, cudaStream_t st, const LamaU8Io* u8 = nullptr);

struct Profiler {
  struct Rec { const char* kind; double flops, bytes; cudaEvent_t a, b; int m, k, n; };
  bool on = false; std::vector<Rec> recs; std::vector<cudaEvent_t> pool;
};
extern thread_local Profiler* g_prof;
struct ProfScope {          // records an event pair around the launches issued in its scope (no-op unless profiling)
  ProfScope(const char* kind, double flops, double bytes, cudaStream_t st, int m = 0, int k = 0, int n = 0);
  ~ProfScope();
  Profiler* p_; cudaStream_t st_;
};
std::string profiler_report(Profiler& p);

struct Ctx {
  int device = 0;
  Profiler prof;
  std::string prof_json;
  std::string err;
  Arena ws;
  DbnetModel* dbnet = nullptr; OcrModel* ocr = nullptr; LamaModel* lama = nullptr;
  DbnetR34Model* dbnet_r34 = nullptr;  // the default detector: its own slot, so both detectors can be resident
  long launches = 0;                   // kernels launched by this library (bench.py "gpu_launches")
  void ensure_ws(size_t bytes);
};
extern thread_local long* g_launch_counter;
// Grow-only device scratch, one buffer per (purpose, device).  The library runs one context per device (one process per GPU,
// get_engine() is a per-device singleton) and every kernel that uses a scratch is ordered on that context's stream; growing
// synchronises the device before the old buffer is released.
struct DeviceScratch {
  static constexpr int kMaxDev = 64;
  void* ptr[kMaxDev] = {}; size_t cap[kMaxDev] = {};
  void* get(size_t bytes) {
    int dev = 0; CUDA_OK(cudaGetDevice(&dev));
    MITB_CHECK(dev >= 0 && dev < kMaxDev, "device ordinal %d out of range", dev);
    if (bytes > cap[dev]) {
      if (ptr[dev]) { CUDA_OK(cudaDeviceSynchronize()); CUDA_OK(cudaFree(ptr[dev])); ptr[dev] = nullptr; cap[dev] = 0; }
      const size_t want = bytes + bytes / 8;
      CUDA_OK(cudaMalloc(&ptr[dev], want)); cap[dev] = want;
    }
    return ptr[dev];
  }
};

// One-shot per-DEVICE initialisation (kernel attributes, __constant__ uploads): get_engine() hands out one context per device in
// the same process, so "static bool done" guards would leave every device but the first uninitialised.
struct PerDeviceOnce {
  bool done[DeviceScratch::kMaxDev] = {};
  bool first() {
    int dev = 0; CUDA_OK(cudaGetDevice(&dev));
    MITB_CHECK(dev >= 0 && dev < DeviceScratch::kMaxDev, "device ordinal %d out of range", dev);
    if (done[dev]) return false;
    done[dev] = true; return true;
  }
};
inline int device_sm_count() {
  static int sms[DeviceScratch::kMaxDev] = {};
  int dev = 0; CUDA_OK(cudaGetDevice(&dev));
  MITB_CHECK(dev >= 0 && dev < DeviceScratch::kMaxDev, "device ordinal %d out of range", dev);
  if (!sms[dev]) CUDA_OK(cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev));
  return sms[dev];
}

// fp32 pairs: two independent round-to-nearest operations per call (the fused multiply-add is one rounding, like fmaf)
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

// the conv epilogue's activation (enum Act)
__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case ACT_RELU: return fmaxf(v, 0.f);
    case ACT_GELU: return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
    case ACT_SILU: return v / (1.f + expf(-v));
    case ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    case ACT_SIGMOID2: { float s = 1.f / (1.f + expf(-v)); return 1.f / (1.f + expf(-s)); }
    case ACT_CLAMP01: return fminf(fmaxf(v, 0.f), 1.f);
    default: return v;
  }
}
// reflect padding (PyTorch 'reflect', no edge repeat) of index i into [0, n), for |i| reaching at most n - 1 past an edge
__device__ __forceinline__ int reflect_idx(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * n - 2 - i;
  return i;
}

extern unsigned long g_launch_epoch;     // bumped by EVERY kernel launch of the library (conv_tma.cu's split reuse keys on it)
inline void count_launch() { ++g_launch_epoch; if (g_launch_counter) ++*g_launch_counter; }

}  // namespace mitb
