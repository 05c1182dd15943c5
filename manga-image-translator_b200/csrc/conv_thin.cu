// Full-resolution 7x7 convolution with a thin output (Cout <= 4): LaMa's final ReflectionPad2d(3) + Conv2d(64->3, k7) +
// Sigmoid (inpainting_lama_mpe.py:596-601).  59 GFLOP of fp32 per 2048x1536 page, but as an implicit GEMM every input
// value would be re-fetched 49 times from L2 (39 GB of gather traffic).  Here a CTA stages the input tile with its 3-pixel
// halo in shared memory ONCE per 8-channel slab (planar [c][y][x] layout, reflect/zero padding resolved while staging)
// and each thread produces 4 horizontally adjacent pixels x Cout channels from registers:
//   per (channel, tap row): 3 LDS.128 of inputs + 7 broadcast LDS.128 of weights feed 56 fp32 pair FMAs (two output channels
//   per pair, the input value broadcast to both)  ->  FMA-pipe bound.
#include "mitb_internal.h"

namespace mitb {

namespace {
constexpr int TW = 64, TH = 16, HALO = 3, KS = 7;
constexpr int SW = TW + 2 * HALO + 2;            // 72: row pitch (x from -4 .. 67 so that float4 loads stay aligned)
constexpr int SH = TH + 2 * HALO;                // 22
constexpr int CCH = 8;                           // channels per slab

struct ThinParams {
  const float* in; int N, H, W, in_cs, in_coff, Cin;
  const float* w;                                // [tap][Cin][4] (K-major fp32, ldw = 4)
  float* out; int out_cs, out_coff, Cout, out_planar;
  const float* shift; int act, pad;
  const float* tile_mask;                        // see ConvOp::tile_mask
  const uint8_t* tile_mask_u8;
};

__device__ __forceinline__ float act_thin(float v, int act) {
  switch (act) {
    case ACT_RELU: return fmaxf(v, 0.f);
    case ACT_SILU: return v / (1.f + expf(-v));
    case ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    default: return v;
  }
}

__global__ void __launch_bounds__(256, 2) conv7_thin_kernel(const ThinParams p) {
  extern __shared__ __align__(16) float thin_smem[];
  float (*tile)[SH][SW] = reinterpret_cast<float (*)[SH][SW]>(thin_smem);                       // [CCH][22][72] = 50688 B
  float (*wsm)[KS * KS][4] = reinterpret_cast<float (*)[KS * KS][4]>(thin_smem + CCH * SH * SW);  // [CCH][49][4] = 6272 B
  const int tx0 = blockIdx.x * TW, ty0 = blockIdx.y * TH, n = blockIdx.z;
  const int tid = threadIdx.x;
  const int lx = (tid & 15) * 4, ly = tid >> 4;          // this thread's 4 output pixels: (ty0+ly, tx0+lx .. +3)
  bool warp_active = true;
  if (p.tile_mask || p.tile_mask_u8) {
    // Output sparsity: LaMa's result is pred*mask + (1-mask)*img (inpainting_lama_mpe.py:726), so prediction pixels where the mask is 0
    // are never used.  A tile without a single hole pixel stores zeros (finite, so that pred*0 stays 0) and skips its 12.8 MFLOP.
    int any = 0;
    const int oy_ = ty0 + ly;
    if (oy_ < p.H) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int ox_ = tx0 + lx + i;
        if (ox_ >= p.W) continue;
        const size_t mi = ((size_t)n * p.H + oy_) * p.W + ox_;
        if (p.tile_mask ? p.tile_mask[mi] != 0.f : p.tile_mask_u8[mi] >= 128) any = 1;
      }
    }
    warp_active = __any_sync(0xffffffffu, any) != 0;    // a warp = 2 rows x 64 pixels of the tile: skip its FMAs (not its staging) when hole free
    if (!__syncthreads_or(any)) {
      if (oy_ < p.H) {
        const size_t plane_ = (size_t)p.H * p.W;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int ox_ = tx0 + lx + i;
          if (ox_ >= p.W) continue;
          const size_t pix_ = (size_t)oy_ * p.W + ox_;
          for (int j = 0; j < p.Cout; ++j) {
            if (p.out_planar) p.out[((size_t)n * p.out_cs + p.out_coff + j) * plane_ + pix_] = 0.f;
            else p.out[((size_t)n * plane_ + pix_) * p.out_cs + p.out_coff + j] = 0.f;
          }
        }
      }
      return;
    }
  }
  float2 acc[4][2];                                      // [pixel][output-channel pair]
#pragma unroll
  for (int i = 0; i < 4; ++i) { acc[i][0] = make_float2(0.f, 0.f); acc[i][1] = make_float2(0.f, 0.f); }

  for (int c0 = 0; c0 < p.Cin; c0 += CCH) {
    __syncthreads();
    // ---- stage the slab: pixels (y in [ty0-3, ty0+TH+3), x in [tx0-4, tx0+TW+4)), 8 channels, padding resolved here
    for (int i = tid; i < SH * SW; i += 256) {
      const int sy = i / SW, sx = i - sy * SW;
      int gy = ty0 + sy - HALO, gx = tx0 + sx - 4;
      bool ok = true;
      if (p.pad == PAD_REFLECT) {
        if (gy < 0) gy = -gy; if (gy >= p.H) gy = 2 * p.H - 2 - gy;
        if (gx < 0) gx = -gx; if (gx >= p.W) gx = 2 * p.W - 2 - gx;
        ok = gy >= 0 && gy < p.H && gx >= 0 && gx < p.W;      // far outside the image (tile overhang): unused values
      } else ok = gy >= 0 && gy < p.H && gx >= 0 && gx < p.W;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
      if (ok) {
        const float* src = p.in + ((size_t)(n * p.H + gy) * p.W + gx) * p.in_cs + p.in_coff + c0;
        a = __ldg(reinterpret_cast<const float4*>(src)); b = __ldg(reinterpret_cast<const float4*>(src) + 1);
      }
      tile[0][sy][sx] = a.x; tile[1][sy][sx] = a.y; tile[2][sy][sx] = a.z; tile[3][sy][sx] = a.w;
      tile[4][sy][sx] = b.x; tile[5][sy][sx] = b.y; tile[6][sy][sx] = b.z; tile[7][sy][sx] = b.w;
    }
    for (int i = tid; i < CCH * KS * KS; i += 256) {
      const int c = i / (KS * KS), t = i - c * (KS * KS);
      *reinterpret_cast<float4*>(&wsm[c][t][0]) = __ldg(reinterpret_cast<const float4*>(p.w + ((size_t)t * p.Cin + c0 + c) * 4));
    }
    __syncthreads();
    // ---- accumulate
    if (warp_active)
#pragma unroll 1
    for (int c = 0; c < CCH; ++c) {
#pragma unroll
      for (int dy = 0; dy < KS; ++dy) {
        // inputs x = lx-3 .. lx+6 live at smem columns (lx+1) .. (lx+10); load the aligned span [lx, lx+12)
        const float4 v0 = *reinterpret_cast<const float4*>(&tile[c][ly + dy][lx]);
        const float4 v1 = *reinterpret_cast<const float4*>(&tile[c][ly + dy][lx + 4]);
        const float4 v2 = *reinterpret_cast<const float4*>(&tile[c][ly + dy][lx + 8]);
        const float in[12] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w, v2.x, v2.y, v2.z, v2.w};
#pragma unroll
        for (int dx = 0; dx < KS; ++dx) {
          const float4 wv = *reinterpret_cast<const float4*>(&wsm[c][dy * KS + dx][0]);
          const float2 w01 = make_float2(wv.x, wv.y), w23 = make_float2(wv.z, wv.w);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float x = in[1 + i + dx];                 // scalar operand broadcast to both channels
            acc[i][0] = ffma2(make_float2(x, x), w01, acc[i][0]);
            acc[i][1] = ffma2(make_float2(x, x), w23, acc[i][1]);
          }
        }
      }
    }
  }
  const int oy = ty0 + ly;
  if (oy >= p.H) return;
  const size_t plane = (size_t)p.H * p.W;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int ox = tx0 + lx + i;
    if (ox >= p.W) continue;
    const size_t pix = (size_t)oy * p.W + ox;
    for (int j = 0; j < p.Cout; ++j) {
      const float a = j == 0 ? acc[i][0].x : j == 1 ? acc[i][0].y : j == 2 ? acc[i][1].x : acc[i][1].y;
      float v = a + (p.shift ? p.shift[j] : 0.f);
      v = act_thin(v, p.act);
      if (p.tile_mask || p.tile_mask_u8) {               // pixels the blend does not use: a finite constant
        const size_t mi = ((size_t)n * p.H + oy) * p.W + ox;
        if (!(p.tile_mask ? p.tile_mask[mi] != 0.f : p.tile_mask_u8[mi] >= 128)) v = 0.f;
      }
      if (p.out_planar) p.out[((size_t)n * p.out_cs + p.out_coff + j) * plane + pix] = v;
      else p.out[((size_t)n * plane + pix) * p.out_cs + p.out_coff + j] = v;
    }
  }
}
}  // namespace

bool conv_thin_supported(const ConvOp& op) {
  if (op.in.planar || op.stat_max || op.wt.ntaps != KS * KS || op.out.C > 4 || op.wt.ldw != 4) return false;
  if (op.sy != 1 || op.sx != 1 || op.in.C % CCH != 0 || op.in.cs % 4 != 0 || op.in.coff % 4 != 0) return false;
  if (op.Ho != op.in.H || op.Wo != op.in.W || op.oy_mul != 1 || op.ox_mul != 1 || op.oy_add || op.ox_add) return false;
  if (op.in_scale || op.add0.p || op.add1.p || op.scale || op.mul1) return false;
  if (op.act != ACT_NONE && op.act != ACT_RELU && op.act != ACT_SILU && op.act != ACT_SIGMOID) return false;
  for (int t = 0; t < op.wt.ntaps; ++t)
    if (op.wt.tdy[t] != t / KS - HALO || op.wt.tdx[t] != t % KS - HALO) return false;
  return op.in.H >= 4 && op.in.W >= 4;
}

void launch_conv_thin(const ConvOp& op, cudaStream_t st) {
  ThinParams p;
  p.in = op.in.p; p.N = op.in.N; p.H = op.in.H; p.W = op.in.W; p.in_cs = op.in.cs; p.in_coff = op.in.coff; p.Cin = op.in.C;
  p.w = op.wt.w; p.out = op.out.p; p.out_cs = op.out.cs; p.out_coff = op.out.coff; p.Cout = op.out.C; p.out_planar = op.out.planar;
  p.shift = op.shift; p.act = op.act; p.pad = op.pad; p.tile_mask = op.tile_mask; p.tile_mask_u8 = op.tile_mask_u8;
  const size_t smem = (size_t)(CCH * SH * SW + CCH * KS * KS * 4) * sizeof(float);
  static PerDeviceOnce attr;
  if (attr.first()) CUDA_OK(cudaFuncSetAttribute(conv7_thin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((p.W + TW - 1) / TW, (p.H + TH - 1) / TH, p.N);
  conv_trace(CK_THIN, 0, 1, -1, -2, false);
  conv7_thin_kernel<<<grid, 256, smem, st>>>(p);
  count_launch();
  CUDA_OK(cudaGetLastError());
}

}  // namespace mitb

// ---------------------------------------------------------------------------------------------------------------------
// ConvTranspose2d(Cin -> 1, k4, s2, p1) + activation, the last layer of both DBHead branches (dbnet_convnext.py:393,445)
// at full page resolution.  As four sub-pixel implicit GEMMs the 32-channel input is gathered 4 x 4 times; here a CTA
// stages a 16x16 block of input positions with a 1-pixel halo in shared memory once and every thread emits the 2x2
// output block of its position: y = 2i - 1 + ky  ->  output (2i+py) takes ky in {1,3} (py=0: rows i, i-1) or {0,2}
// (py=1: rows i+1, i).
namespace mitb {
namespace {
constexpr int CT_T = 16;                          // tile edge (input positions)

// CIN = 32 (DBNet-ConvNeXt head) or 16 (DBNet-ResNet34 head); channel pitch CIN + 4 floats
template <int CIN>
__global__ void __launch_bounds__(256) convT4_c1_kernel(const float* in, int H, int W, int in_cs, int in_coff, const float* w,
                                                        const float* bias, int act, float* out, int out_cs, int out_coff) {
  static_assert(CIN == 32 || CIN == 16, "convT4_c1: Cin 32 or 16");
  constexpr int CT_PITCH = CIN + 4, C4 = CIN / 4, LOG_CIN = CIN == 32 ? 5 : 4, LOG_C4 = LOG_CIN - 2;
  __shared__ __align__(16) float tile[(CT_T + 2) * (CT_T + 2) * CT_PITCH];     // CIN = 32: 18*18*36*4 = 46656 B
  __shared__ __align__(16) float wsm[16 * CIN];                                 // [ky*4+kx][cin]
  const int n = blockIdx.z, i0 = blockIdx.y * CT_T, j0 = blockIdx.x * CT_T;
  const int tid = threadIdx.x;
  for (int t = tid; t < 16 * CIN; t += 256) { const int c = t & (CIN - 1), k = t >> LOG_CIN; wsm[k * CIN + c] = w[c * 16 + k]; }
  for (int t = tid; t < (CT_T + 2) * (CT_T + 2) * C4; t += 256) {
    const int c4 = t & (C4 - 1), pp = t >> LOG_C4;
    const int ty = pp / (CT_T + 2), tx = pp - ty * (CT_T + 2);
    const int gy = i0 + ty - 1, gx = j0 + tx - 1;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gy >= 0 && gy < H && gx >= 0 && gx < W)
      v = __ldg(reinterpret_cast<const float4*>(in + ((size_t)(n * H + gy) * W + gx) * in_cs + in_coff + c4 * 4));
    *reinterpret_cast<float4*>(&tile[pp * CT_PITCH + c4 * 4]) = v;
  }
  __syncthreads();
  const int ly = tid >> 4, lx = tid & 15;
  const int i = i0 + ly, j = j0 + lx;
  if (i >= H || j >= W) return;
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
  for (int py = 0; py < 2; ++py)
#pragma unroll
    for (int px = 0; px < 2; ++px)
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const int ky = py == 0 ? 1 + 2 * a : 2 * a, dy = (py + 1 - ky) / 2;      // exact: (py+1-ky) is even
          const int kx = px == 0 ? 1 + 2 * b : 2 * b, dx = (px + 1 - kx) / 2;
          const float* src = &tile[((ly + 1 + dy) * (CT_T + 2) + (lx + 1 + dx)) * CT_PITCH];
          const float* wk = &wsm[(ky * 4 + kx) * CIN];
          float s = 0.f;
#pragma unroll
          for (int c = 0; c < CIN; c += 4) {
            const float4 x = *reinterpret_cast<const float4*>(src + c), ww = *reinterpret_cast<const float4*>(wk + c);
            s = fmaf(x.x, ww.x, s); s = fmaf(x.y, ww.y, s); s = fmaf(x.z, ww.z, s); s = fmaf(x.w, ww.w, s);
          }
          acc[py][px] += s;
        }
  const float bv = bias ? bias[0] : 0.f;
  const size_t plane = (size_t)(2 * H) * (2 * W);
  float* o = out + ((size_t)n * out_cs + out_coff) * plane;
#pragma unroll
  for (int py = 0; py < 2; ++py) {
    float v0 = acc[py][0] + bv, v1 = acc[py][1] + bv;
    if (act == ACT_SIGMOID || act == ACT_SIGMOID2) { v0 = 1.f / (1.f + expf(-v0)); v1 = 1.f / (1.f + expf(-v1)); }
    if (act == ACT_SIGMOID2) { v0 = 1.f / (1.f + expf(-v0)); v1 = 1.f / (1.f + expf(-v1)); }
    *reinterpret_cast<float2*>(o + (size_t)(2 * i + py) * (2 * W) + 2 * j) = make_float2(v0, v1);
  }
}
}  // namespace

// in: NHWC view with 32 or 16 channels; w: ConvTranspose2d weight [Cin,1,4,4] (PyTorch layout, fp32 device); out: planar view, C == 1
void launch_convT4_c1(const View& in, const float* w, const float* bias, int act, const View& out, cudaStream_t st) {
  MITB_CHECK(!in.planar && (in.C == 32 || in.C == 16) && in.cs % 4 == 0 && in.coff % 4 == 0, "convT4_c1 expects a 32- or 16-channel NHWC input");
  MITB_CHECK(out.planar && out.C == 1 && out.H == 2 * in.H && out.W == 2 * in.W && out.N == in.N, "convT4_c1 output shape");
  dim3 grid((in.W + CT_T - 1) / CT_T, (in.H + CT_T - 1) / CT_T, in.N);
  ProfScope ps("convT4_c1", 2.0 * in.pixels() * 4 * 4 * in.C, 4.0 * (in.pixels() * in.C + in.pixels() * 4), st);
  if (in.C == 32) convT4_c1_kernel<32><<<grid, 256, 0, st>>>(in.p, in.H, in.W, in.cs, in.coff, w, bias, act, out.p, out.cs, out.coff);
  else convT4_c1_kernel<16><<<grid, 256, 0, st>>>(in.p, in.H, in.W, in.cs, in.coff, w, bias, act, out.p, out.cs, out.coff);
  count_launch();
  CUDA_OK(cudaGetLastError());
}
}  // namespace mitb
