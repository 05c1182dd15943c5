// Implicit-GEMM convolution, fp32 SIMT tiles (128 x {128,64} x 16, 256 threads, 8x8 / 8x4 register tiles).
//
// C[M = N*Ho*Wo pixels, Cout] = A[M, K = ntaps*Cin] (gathered on the fly from the NHWC view) x Wt[K, Cout].
// One kernel covers every dense contraction of the three networks: 1x1 / 3x3 / 7x7, stride 1/2, zero or
// reflect padding, the sub-pixel phases of the transposed convolutions (tap list + strided output mapping),
// the BN+ReLU *prologue* of the pre-activation OCR ResNet, and a fused epilogue
//      v = acc (+add0) ; v = v*scale[c] + shift[c] ; v = act(v) ; v *= mul1[c] ; v += add1
// which folds bias / BatchNorm / activation / ConvNeXt layer-scale / residuals / the FFC branch sum.
// The vocabulary head uses the ROWSTAT epilogue: online (max, argmax, sum-exp) per row, so the [N,T,V]
// logits never reach HBM (model_48px_ctc.py:460-461 computes log_softmax + max over them).
//
// This is the exact-fp32 path.  Layers that are large dense contractions are routed to the wgmma kernels (conv_tma.cu,
// conv_tc.cu) by conv_plan() (conv.cu); this kernel remains the path for thin layers and the parity anchor of those.
#include <float.h>
#include <limits.h>
#include "mitb_internal.h"

namespace mitb {

thread_local long* g_launch_counter = nullptr;
unsigned long g_launch_epoch = 0;

struct ConvKParams {
  const float* in; int N, H, W, in_cs, in_coff, Cin, in_planar;
  const float* w; int ldw, ntaps; int8_t tdy[kMaxTaps], tdx[kMaxTaps];
  int sy, sx, pad, Ho, Wo;
  float* out; int oH, oW, out_cs, out_coff, Cout, out_planar, oy_mul, oy_add, ox_mul, ox_add;
  const float* in_scale; const float* in_shift; int in_relu;
  const float* add0; int add0_cs, add0_coff, add0_planar;
  const float* add1; int add1_cs, add1_coff, add1_planar;
  const float* scale; const float* shift; const float* mul1; int act;
  float* stat_max; float* stat_sum; int* stat_idx; int stat_ld;
  int M, K;
};

constexpr int BM = 128, BK = 16, NT = 256, APAD = 4;

template <int BN, bool PLANAR_IN, bool ROWSTAT>
__global__ void __launch_bounds__(NT) conv_igemm_kernel(const ConvKParams p) {
  __shared__ __align__(16) float As[2][BK][BM + APAD];
  __shared__ __align__(16) float Bs[2][BK][BN];
  constexpr int TN = BN / 16;                 // columns per thread (8 or 4)
  constexpr int BLOADS = BK * BN / 4 / NT;    // float4 weight loads per thread (2 or 1)
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int HoWo = p.Ho * p.Wo;
  const int HW = p.H * p.W;

  // ---------------- A loader state
  int a_img[2], a_iy0[2], a_ix0[2];           // NHWC mode: two pixel slots per thread
  bool a_ok[2];
  const int kq = tid & 3;                      // quad (4 consecutive k) handled by this thread
  int cur_tap = 0, cur_c = kq * 4;             // decoded position of k = kt*16 + kq*4
  if (!PLANAR_IN) {
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      int m = m0 + (tid >> 2) + 64 * s;
      a_ok[s] = m < p.M;
      int mm = a_ok[s] ? m : 0;
      int nimg = mm / HoWo, r = mm - nimg * HoWo;
      int oy = r / p.Wo, ox = r - oy * p.Wo;
      a_img[s] = nimg; a_iy0[s] = oy * p.sy; a_ix0[s] = ox * p.sx;
    }
    while (cur_c >= p.Cin) { cur_c -= p.Cin; ++cur_tap; }
  }
  float4 a_reg[2];
  float4 b_reg[BLOADS];

  auto load_tile = [&](int kt) {
    if (!PLANAR_IN) {
      const int k = kt * BK + kq * 4;
      const bool kval = k < p.K;
      float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
      if (p.in_scale && kval) {
        sc = *reinterpret_cast<const float4*>(p.in_scale + cur_c);
        sh = *reinterpret_cast<const float4*>(p.in_shift + cur_c);
      }
      const int dy = kval ? p.tdy[cur_tap] : 0, dx = kval ? p.tdx[cur_tap] : 0;
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (kval && a_ok[s]) {
          int iy = a_iy0[s] + dy, ix = a_ix0[s] + dx;
          bool inb = true;
          if (p.pad == PAD_REFLECT) { iy = reflect_idx(iy, p.H); ix = reflect_idx(ix, p.W); }
          else inb = (iy >= 0) & (iy < p.H) & (ix >= 0) & (ix < p.W);
          if (inb) {
            const float* src = p.in + ((size_t)(a_img[s] * p.H + iy) * p.W + ix) * p.in_cs + p.in_coff + cur_c;
            v = __ldg(reinterpret_cast<const float4*>(src));
            if (p.in_scale) {
              v.x = v.x * sc.x + sh.x; v.y = v.y * sc.y + sh.y; v.z = v.z * sc.z + sh.z; v.w = v.w * sc.w + sh.w;
              if (p.in_relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
            }
          }
        }
        a_reg[s] = v;
      }
      // advance the (tap, channel) cursor by one K tile
      cur_c += BK;
      while (cur_c >= p.Cin) { cur_c -= p.Cin; ++cur_tap; }
    } else {
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const int idx = tid + NT * s;
        const int kl = idx >> 5, m4 = idx & 31;
        const int k = kt * BK + kl, m = m0 + m4 * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < p.K && m < p.M) {
          float sc = 1.f, sh = 0.f;
          if (p.in_scale) { sc = p.in_scale[k]; sh = p.in_shift[k]; }
          if ((HW & 3) == 0 && m + 3 < p.M) {
            int nimg = m / HW, pix = m - nimg * HW;
            v = __ldg(reinterpret_cast<const float4*>(p.in + ((size_t)nimg * p.in_cs + p.in_coff + k) * HW + pix));
          } else {
            float t[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              int me = m + e; t[e] = 0.f;
              if (me < p.M) { int nimg = me / HW, pix = me - nimg * HW; t[e] = __ldg(p.in + ((size_t)nimg * p.in_cs + p.in_coff + k) * HW + pix); }
            }
            v = make_float4(t[0], t[1], t[2], t[3]);
          }
          if (p.in_scale) {
            v.x = v.x * sc + sh; v.y = v.y * sc + sh; v.z = v.z * sc + sh; v.w = v.w * sc + sh;
            if (p.in_relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
          }
          // rows beyond M inside a partially valid quad were loaded as 0 by the scalar path
        }
        a_reg[s] = v;
      }
    }
#pragma unroll
    for (int s = 0; s < BLOADS; ++s) {
      const int idx = tid + NT * s;
      const int row = idx / (BN / 4), c4 = idx % (BN / 4);
      const int k = kt * BK + row, n = n0 + c4 * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k < p.K && n < p.ldw) v = __ldg(reinterpret_cast<const float4*>(p.w + (size_t)k * p.ldw + n));
      b_reg[s] = v;
    }
  };

  auto store_tile = [&](int buf) {
    if (!PLANAR_IN) {
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const int m = (tid >> 2) + 64 * s;
        As[buf][kq * 4 + 0][m] = a_reg[s].x; As[buf][kq * 4 + 1][m] = a_reg[s].y;
        As[buf][kq * 4 + 2][m] = a_reg[s].z; As[buf][kq * 4 + 3][m] = a_reg[s].w;
      }
    } else {
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const int idx = tid + NT * s;
        *reinterpret_cast<float4*>(&As[buf][idx >> 5][(idx & 31) * 4]) = a_reg[s];
      }
    }
#pragma unroll
    for (int s = 0; s < BLOADS; ++s) {
      const int idx = tid + NT * s;
      *reinterpret_cast<float4*>(&Bs[buf][idx / (BN / 4)][(idx % (BN / 4)) * 4]) = b_reg[s];
    }
  };

  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nkt = (p.K + BK - 1) / BK;
  load_tile(0);
  store_tile(0);
  __syncthreads();
  int buf = 0;
  for (int kt = 0; kt < nkt; ++kt) {
    if (kt + 1 < nkt) load_tile(kt + 1);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[8], b[TN];
      *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      *reinterpret_cast<float4*>(&a[4]) = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      *reinterpret_cast<float4*>(&b[0]) = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      if (TN == 8) *reinterpret_cast<float4*>(&b[4]) = *reinterpret_cast<const float4*>(&Bs[buf][kk][BN / 2 + tx * 4]);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nkt) store_tile(buf ^ 1);
    __syncthreads();
    buf ^= 1;
  }

  // ---------------- epilogue
  if (ROWSTAT) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
      float bm = -INFINITY, bs = 0.f; int bi = INT_MAX;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int c = n0 + (j < 4 ? tx * 4 + j : BN / 2 + tx * 4 + (j - 4));
        if (c < p.Cout) {
          float v = acc[i][j] + (p.shift ? p.shift[c] : 0.f);
          if (v > bm) { bs = bs * expf(bm - v) + 1.f; bm = v; bi = c; }   // first occurrence wins ties (c ascending within j<4 / j>=4 halves)
          else bs += expf(v - bm);
        }
      }
      // the two column halves of a thread are not monotone in c across threads; ties are resolved by index below
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) {
        float om = __shfl_xor_sync(0xffffffffu, bm, o);
        float os = __shfl_xor_sync(0xffffffffu, bs, o);
        int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (om > bm || (om == bm && oi < bi)) { float t = bm; bm = om; om = t; t = bs; bs = os; os = t; bi = oi; }
        if (om != -INFINITY) bs += os * expf(om - bm);
      }
      if (tx == 0 && m < p.M) {
        size_t o = (size_t)m * p.stat_ld + blockIdx.y;
        p.stat_max[o] = bm; p.stat_sum[o] = bs; p.stat_idx[o] = bi;
      }
    }
    return;
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= p.M) continue;
    const int nimg = m / HoWo, r = m - nimg * HoWo;
    const int oy = r / p.Wo, ox = r - oy * p.Wo;
    const int py = oy * p.oy_mul + p.oy_add, px = ox * p.ox_mul + p.ox_add;
    const size_t opix = ((size_t)nimg * p.oH + py) * p.oW + px;          // NHWC pixel index
    const size_t oplane = (size_t)p.oH * p.oW;
    const size_t opl_pix = (size_t)py * p.oW + px;
#pragma unroll
    for (int jg = 0; jg < TN / 4; ++jg) {
      const int c0 = n0 + (jg == 0 ? tx * 4 : BN / 2 + tx * 4);
      if (c0 >= p.Cout) continue;
      float v[4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) v[jj] = acc[i][jg * 4 + jj];
      const bool full = c0 + 3 < p.Cout;
      auto fetch = [&](const float* base, int cs, int coff, int planar, float* dst) {
        if (!planar && full && ((cs | coff) & 3) == 0) {
          float4 t = *reinterpret_cast<const float4*>(base + opix * cs + coff + c0);
          dst[0] = t.x; dst[1] = t.y; dst[2] = t.z; dst[3] = t.w;
        } else {
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            dst[jj] = 0.f;
            if (c0 + jj < p.Cout)
              dst[jj] = planar ? base[((size_t)nimg * cs + coff + c0 + jj) * oplane + opl_pix]
                               : base[opix * cs + coff + c0 + jj];
          }
        }
      };
      if (p.add0) { float t[4]; fetch(p.add0, p.add0_cs, p.add0_coff, p.add0_planar, t);
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) v[jj] += t[jj]; }
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int c = c0 + jj;
        if (c < p.Cout) {
          float x = v[jj];
          if (p.scale) x *= p.scale[c];
          if (p.shift) x += p.shift[c];
          x = apply_act(x, p.act);
          if (p.mul1) x *= p.mul1[c];
          v[jj] = x;
        }
      }
      if (p.add1) { float t[4]; fetch(p.add1, p.add1_cs, p.add1_coff, p.add1_planar, t);
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) v[jj] += t[jj]; }
      if (!p.out_planar && full && ((p.out_cs | p.out_coff) & 3) == 0) {
        *reinterpret_cast<float4*>(p.out + opix * p.out_cs + p.out_coff + c0) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj)
          if (c0 + jj < p.Cout) {
            if (p.out_planar) p.out[((size_t)nimg * p.out_cs + p.out_coff + c0 + jj) * oplane + opl_pix] = v[jj];
            else p.out[opix * p.out_cs + p.out_coff + c0 + jj] = v[jj];
          }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// Thin-output convolution (Cout <= 4): one thread per output pixel, float4 loads over Cin, weights broadcast
// through L1.  Used for the 1-channel DBNet heads and LaMa's 64->3 output conv.
template <int CO>
__global__ void __launch_bounds__(128) conv_fewout_kernel(const ConvKParams p) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= p.M) return;
  const int HoWo = p.Ho * p.Wo;
  const int nimg = m / HoWo, r = m - nimg * HoWo;
  const int oy = r / p.Wo, ox = r - oy * p.Wo;
  float acc[CO];
#pragma unroll
  for (int j = 0; j < CO; ++j) acc[j] = 0.f;
  for (int t = 0; t < p.ntaps; ++t) {
    int iy = oy * p.sy + p.tdy[t], ix = ox * p.sx + p.tdx[t];
    if (p.pad == PAD_REFLECT) { iy = reflect_idx(iy, p.H); ix = reflect_idx(ix, p.W); }
    else if (iy < 0 || iy >= p.H || ix < 0 || ix >= p.W) continue;
    const float* src = p.in + ((size_t)(nimg * p.H + iy) * p.W + ix) * p.in_cs + p.in_coff;
    const float* wr = p.w + (size_t)t * p.Cin * p.ldw;
    for (int c = 0; c < p.Cin; c += 4) {
      float4 v = __ldg(reinterpret_cast<const float4*>(src + c));
      if (p.in_scale) {
        float4 sc = *reinterpret_cast<const float4*>(p.in_scale + c), sh = *reinterpret_cast<const float4*>(p.in_shift + c);
        v.x = v.x * sc.x + sh.x; v.y = v.y * sc.y + sh.y; v.z = v.z * sc.z + sh.z; v.w = v.w * sc.w + sh.w;
        if (p.in_relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
      }
      const float xs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float4 wv = __ldg(reinterpret_cast<const float4*>(wr + (size_t)(c + e) * p.ldw));   // ldw == 4
        const float ws[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
        for (int j = 0; j < CO; ++j) acc[j] = fmaf(xs[e], ws[j], acc[j]);
      }
    }
  }
  const int py = oy * p.oy_mul + p.oy_add, px = ox * p.ox_mul + p.ox_add;
  const size_t opix = ((size_t)nimg * p.oH + py) * p.oW + px;
  const size_t oplane = (size_t)p.oH * p.oW, opl_pix = (size_t)py * p.oW + px;
#pragma unroll
  for (int j = 0; j < CO; ++j) {
    float x = acc[j];
    if (p.add0) x += p.add0_planar ? p.add0[((size_t)nimg * p.add0_cs + p.add0_coff + j) * oplane + opl_pix]
                                   : p.add0[opix * p.add0_cs + p.add0_coff + j];
    if (p.scale) x *= p.scale[j];
    if (p.shift) x += p.shift[j];
    x = apply_act(x, p.act);
    if (p.mul1) x *= p.mul1[j];
    if (p.add1) x += p.add1_planar ? p.add1[((size_t)nimg * p.add1_cs + p.add1_coff + j) * oplane + opl_pix]
                                   : p.add1[opix * p.add1_cs + p.add1_coff + j];
    if (p.out_planar) p.out[((size_t)nimg * p.out_cs + p.out_coff + j) * oplane + opl_pix] = x;
    else p.out[opix * p.out_cs + p.out_coff + j] = x;
  }
}

// ---------------------------------------------------------------------------------------------------
__global__ void rowstat_final_kernel(const float* pmax, const float* psum, const int* pidx, int rows, int nblk,
                                     int* idx, float* logprob) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float bm = -INFINITY, bs = 0.f; int bi = INT_MAX;
  for (int b = lane; b < nblk; b += 32) {
    float om = pmax[(size_t)row * nblk + b], os = psum[(size_t)row * nblk + b]; int oi = pidx[(size_t)row * nblk + b];
    if (om > bm || (om == bm && oi < bi)) { float t = bm; bm = om; om = t; t = bs; bs = os; os = t; bi = oi; }
    if (om != -INFINITY) bs += os * expf(om - bm);
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float om = __shfl_xor_sync(0xffffffffu, bm, o);
    float os = __shfl_xor_sync(0xffffffffu, bs, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (om > bm || (om == bm && oi < bi)) { float t = bm; bm = om; om = t; t = bs; bs = os; os = t; bi = oi; }
    if (om != -INFINITY) bs += os * expf(om - bm);
  }
  if (lane == 0) { idx[row] = bi; logprob[row] = -logf(bs); }    // logit[argmax] - logsumexp = -log(sum exp(v - max))
}

void launch_rowstat_final(const float* pmax, const float* psum, const int* pidx, int rows, int nblk, int* idx,
                          float* logprob, cudaStream_t st) {
  rowstat_final_kernel<<<(rows + 3) / 4, 128, 0, st>>>(pmax, psum, pidx, rows, nblk, idx, logprob);
  count_launch();
  CUDA_OK(cudaGetLastError());
}

__global__ void repack_kernel(float* dst, const float* src, int Cout, int Cin, int ntaps, const int* ky, const int* kx,
                              long s_co, long s_c, long s_ky, long s_kx, int ldw) {
  const long total = (long)ntaps * Cin * ldw;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int co = (int)(i % ldw); const long k = i / ldw; const int c = (int)(k % Cin); const int t = (int)(k / Cin);
    dst[i] = co < Cout ? src[co * s_co + c * s_c + ky[t] * s_ky + kx[t] * s_kx] : 0.f;
  }
}

void launch_repack(float* dst, const float* src, int Cout, int Cin, int ntaps, const int* ky, const int* kx,
                   long s_co, long s_c, long s_ky, long s_kx, int ldw, cudaStream_t st) {
  int* d = nullptr;
  CUDA_OK(cudaMalloc(&d, sizeof(int) * 2 * ntaps));
  CUDA_OK(cudaMemcpyAsync(d, ky, sizeof(int) * ntaps, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(d + ntaps, kx, sizeof(int) * ntaps, cudaMemcpyHostToDevice, st));
  const long total = (long)ntaps * Cin * ldw;
  int blocks = (int)((total + 255) / 256); if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
  repack_kernel<<<blocks, 256, 0, st>>>(dst, src, Cout, Cin, ntaps, d, d + ntaps, s_co, s_c, s_ky, s_kx, ldw);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaStreamSynchronize(st));
  CUDA_OK(cudaFree(d));
}


static void fill_params(const ConvOp& op, ConvKParams& p) {
  p.in = op.in.p; p.N = op.in.N; p.H = op.in.H; p.W = op.in.W; p.in_cs = op.in.cs; p.in_coff = op.in.coff;
  p.Cin = op.in.C; p.in_planar = op.in.planar;
  p.w = op.wt.w; p.ldw = op.wt.ldw; p.ntaps = op.wt.ntaps;
  for (int t = 0; t < op.wt.ntaps; ++t) { p.tdy[t] = op.wt.tdy[t]; p.tdx[t] = op.wt.tdx[t]; }
  p.sy = op.sy; p.sx = op.sx; p.pad = op.pad; p.Ho = op.Ho; p.Wo = op.Wo;
  p.out = op.out.p; p.oH = op.out.H; p.oW = op.out.W; p.out_cs = op.out.cs; p.out_coff = op.out.coff;
  p.Cout = op.out.C; p.out_planar = op.out.planar;
  p.oy_mul = op.oy_mul; p.oy_add = op.oy_add; p.ox_mul = op.ox_mul; p.ox_add = op.ox_add;
  p.in_scale = op.in_scale; p.in_shift = op.in_shift; p.in_relu = op.in_relu;
  p.add0 = op.add0.p; p.add0_cs = op.add0.cs; p.add0_coff = op.add0.coff; p.add0_planar = op.add0.planar;
  p.add1 = op.add1.p; p.add1_cs = op.add1.cs; p.add1_coff = op.add1.coff; p.add1_planar = op.add1.planar;
  p.scale = op.scale; p.shift = op.shift; p.mul1 = op.mul1; p.act = op.act;
  p.stat_max = op.stat_max; p.stat_sum = op.stat_sum; p.stat_idx = op.stat_idx; p.stat_ld = op.stat_ld;
  p.M = op.in.N * op.Ho * op.Wo; p.K = op.wt.ntaps * op.in.C;
}

// the fp32 kernels: the row-stat epilogue when op.stat_max is set, the thin-output kernel when conv_plan() picked CK_FEWOUT, else the
// 128 x {64, 128} tile kernel
void launch_conv_simt(const ConvOp& op, bool fewout, cudaStream_t st) {
  ConvKParams p; fill_params(op, p);
  const int Cout = op.out.C;
  if (op.stat_max) {
    MITB_CHECK(!op.in.planar, "row-stat epilogue expects NHWC input");
    dim3 grid((p.M + BM - 1) / BM, (Cout + 127) / 128);
    MITB_CHECK(op.stat_ld == (int)grid.y, "stat_ld must equal conv_stat_blocks(Cout)");
    conv_trace(CK_SIMT, 128, 1, -1, -2, false);
    conv_igemm_kernel<128, false, true><<<grid, NT, 0, st>>>(p);
  } else if (fewout) {
    dim3 grid((p.M + 127) / 128);
    conv_trace(CK_FEWOUT, Cout, 1, -1, -2, false);
    switch (Cout) {
      case 1: conv_fewout_kernel<1><<<grid, 128, 0, st>>>(p); break;
      case 2: conv_fewout_kernel<2><<<grid, 128, 0, st>>>(p); break;
      case 3: conv_fewout_kernel<3><<<grid, 128, 0, st>>>(p); break;
      default: conv_fewout_kernel<4><<<grid, 128, 0, st>>>(p); break;
    }
  } else {
    const int t128 = (Cout + 127) / 128 * 128, t64 = (Cout + 63) / 64 * 64;
    const bool use64 = t64 * 10 < t128 * 9;
    conv_trace(CK_SIMT, use64 ? 64 : 128, 1, -1, -2, false);
    if (use64) {
      dim3 grid((p.M + BM - 1) / BM, (Cout + 63) / 64);
      if (op.in.planar) conv_igemm_kernel<64, true, false><<<grid, NT, 0, st>>>(p);
      else conv_igemm_kernel<64, false, false><<<grid, NT, 0, st>>>(p);
    } else {
      dim3 grid((p.M + BM - 1) / BM, (Cout + 127) / 128);
      if (op.in.planar) conv_igemm_kernel<128, true, false><<<grid, NT, 0, st>>>(p);
      else conv_igemm_kernel<128, false, false><<<grid, NT, 0, st>>>(p);
    }
  }
  count_launch();
  CUDA_OK(cudaGetLastError());
}

}  // namespace mitb
