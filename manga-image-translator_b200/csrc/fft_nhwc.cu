// Channel-vectorised real 2-D FFT on NHWC tensors for LaMa's FourierUnit (inpainting_lama_mpe.py:214-257):
// torch.fft.rfftn / irfftn over (h, w), norm='ortho', with the channel axis INNERMOST end to end, so that
//   * the 1x1 convs around the transform read and write plain NHWC matrices (no planar transposes), and the spectrum
//     [h][w/2+1][c][re,im] IS the reference's interleaved channel order c0_re, c0_im, c1_re, ... (:229-231) as an NHWC tensor
//     with 2C channels - the spectral 1x1 conv is a plain GEMM over it;
//   * every global access of a warp is 32 consecutive complex channels (256 contiguous bytes), staged into shared memory by
//     one TMA box per CTA (cp.async.bulk.tensor, mbarrier completion) where the tile shape allows;
//   * one warp performs 32 independent FFTs in lock step, lane = channel: all butterfly indices and twiddles are
//     warp-uniform (no divergence, no bank conflicts, twiddle reads broadcast), the transform runs IN PLACE in shared
//     memory (decimation in frequency, mixed radix {16,12,4,2,3,5}; 16 = 4x4 and 12 = 4x3 fused in registers); the digit-reversed result order is undone for free when the
//     rows are written back (each frequency is its own 256-byte segment).
// Real-input trick: two CHANNELS are packed into one complex sequence (z = x_c0 + i x_c1 is just a float2 load of an NHWC
// pixel), separated after the row transform; the inverse packs two Hermitian spectra the same way.
//   forward : rows   rfft_rows   S fp32 [N][h][w][C]        -> T complex [N][h][w2][C]
//             cols   fft_cols    T                          -> spectrum [N][h][w2][2C] * 1/sqrt(hw), as bf16 hi/mid split
//                                                              operands of the spectral conv and/or fp32
//   inverse : cols   ifft_cols   F fp32 [N][h][w2][2C]      -> T complex
//             rows   irfft_rows  T (+ residual S)           -> U [N][h][w][C] * 1/sqrt(hw) + S, as bf16 hi/mid split and/or fp32
// The complex intermediate T is written once and read once (L2 resident for LaMa sizes).
#include <cuda.h>
#include <math.h>
#include <string.h>
#include <stdlib.h>
#include <mutex>
#include <cuda_bf16.h>
#include "mitb_internal.h"

namespace mitb {

namespace {

constexpr int FV = 32;                 // complex channels per CTA (= lanes of a warp)
constexpr int FT = 256, FW = FT / 32;  // threads / warps per CTA
constexpr int kMaxSt = 10;

struct FftNDev { int n, nst, nbt; int radix[kMaxSt]; const float2* tw; const uint16_t* rev; };   // nbt: butterflies over all stages

#include "tc_common.cuh"

// complex arithmetic on fp32 pairs (ffma2 / fmul2 / fadd2 of mitb_internal.h): one fused multiply-add per component
__device__ __forceinline__ float2 cmulf(float2 a, float2 b) {
  return ffma2(make_float2(a.x, a.x), b, fmul2(make_float2(a.y, a.y), make_float2(-b.y, b.x)));
}
__device__ __forceinline__ float2 caddf(float2 a, float2 b) { return fadd2(a, b); }
__device__ __forceinline__ float2 csubf(float2 a, float2 b) { return ffma2(b, make_float2(-1.f, -1.f), a); }
// multiply by -i (forward) or +i (inverse)
__device__ __forceinline__ float2 rot90(float2 a, bool inv) { return inv ? make_float2(-a.y, a.x) : make_float2(a.y, -a.x); }

// In-place decimation-in-frequency FFT of FV interleaved sequences X[i * FV + lane], i < n: natural-order input, the
// output element k ends at position rev[k].  All threads of the CTA call it; `tw` is the shared-memory twiddle table
// exp(-2 pi i j / n), j < n; `bt` the shared-memory butterfly table (one entry per butterfly of every stage: first element
// index | twiddle step << 16), so the hot loop has no integer division.  INV conjugates twiddles (unscaled inverse).
template <bool INV>
__device__ __forceinline__ float2 twc(const float2* tw, int i) { float2 w = tw[i]; if (INV) w.y = -w.y; return w; }

// 4- and 3-point DFTs in registers, natural order in and out (forward: exp(-2 pi i jq / r); INV: conjugate)
template <bool INV>
__device__ __forceinline__ void dft4(float2& a0, float2& a1, float2& a2, float2& a3) {
  const float2 t0 = caddf(a0, a2), t1 = csubf(a0, a2), t2 = caddf(a1, a3), t3 = rot90(csubf(a1, a3), INV);
  a0 = caddf(t0, t2); a1 = caddf(t1, t3); a2 = csubf(t0, t2); a3 = csubf(t1, t3);
}
template <bool INV>
__device__ __forceinline__ void dft3(float2& a0, float2& a1, float2& a2) {
  const float2 t1 = caddf(a1, a2);
  const float2 t2 = ffma2(t1, make_float2(-0.5f, -0.5f), a0);
  const float2 t3 = fmul2(csubf(a1, a2), make_float2(0.86602540378443864676f, 0.86602540378443864676f));
  // forward: y1 = t2 - i t3, y2 = t2 + i t3 ; inverse: swapped
  const float2 y1 = make_float2(t2.x + t3.y, t2.y - t3.x), y2 = make_float2(t2.x - t3.y, t2.y + t3.x);
  a0 = caddf(a0, t1);
  a1 = INV ? y2 : y1; a2 = INV ? y1 : y2;
}
// multiply by the constant twiddle exp(-2 pi i e / N) = (c, -s) (INV: conjugate)
template <bool INV>
__device__ __forceinline__ float2 cmulk(float2 a, float c, float s) { return cmulf(a, make_float2(c, INV ? s : -s)); }

template <bool INV>
__device__ __forceinline__ void fft_dif(float2* X, const float2* tw, const uint32_t* bt, const FftNDev& pl, int lane, int warp) {
  int L = pl.n;
  for (int st = 0; st < pl.nst; ++st) {
    const int r = pl.radix[st];
    const int m = L / r;                 // length of the sub-sequences this stage produces
    const int nb = pl.n / r;
    const uint32_t sm = (uint32_t)m * FV;
    if (r == 16) {
      // two radix-4 steps fused in registers: j = j1 + 4 j2, q = 4 q1 + q2, w16^(jq) = w4^(j1 q1) w16^(j1 q2) w4^(j2 q2).
      // Halves the shared-memory round trips, table lookups and barriers of two radix-4 stages (the kernels are issue bound).
      const float C1 = 0.92387953251128675613f, S1 = 0.38268343236508977173f, H = 0.70710678118654752440f;
      for (int b = warp; b < nb; b += FW) {
        const uint32_t e = bt[b];
        float2* x = X + (e & 0xffffu) * FV + lane;
        const int kt = (int)(e >> 16);
        float2 a[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) a[j] = x[j * sm];
#pragma unroll
        for (int j1 = 0; j1 < 4; ++j1) dft4<INV>(a[j1], a[j1 + 4], a[j1 + 8], a[j1 + 12]);        // b[j1][q2] -> a[j1 + 4 q2]
        a[5] = cmulk<INV>(a[5], C1, S1);  a[6] = cmulk<INV>(a[6], H, H);     a[7] = cmulk<INV>(a[7], S1, C1);      // w16^1, ^2, ^3
        a[9] = cmulk<INV>(a[9], H, H);    a[10] = rot90(a[10], INV);         a[11] = cmulk<INV>(a[11], -H, H);     // w16^2, ^4, ^6
        a[13] = cmulk<INV>(a[13], S1, C1); a[14] = cmulk<INV>(a[14], -H, H); a[15] = cmulk<INV>(a[15], -C1, -S1);  // w16^3, ^6, ^9
#pragma unroll
        for (int q2 = 0; q2 < 4; ++q2) dft4<INV>(a[4 * q2], a[4 * q2 + 1], a[4 * q2 + 2], a[4 * q2 + 3]);     // y[4 q1 + q2] -> a[4 q2 + q1]
        if (kt) {
#pragma unroll
          for (int q = 1; q < 16; ++q) a[4 * (q & 3) + (q >> 2)] = cmulf(a[4 * (q & 3) + (q >> 2)], twc<INV>(tw, q * kt));
        }
#pragma unroll
        for (int q = 0; q < 16; ++q) x[q * sm] = a[4 * (q & 3) + (q >> 2)];
      }
    } else if (r == 12) {
      // radix 4 x radix 3 fused in registers: j = j1 + 3 j2, q = 4 q1 + q2, w12^(jq) = w3^(j1 q1) w12^(j1 q2) w4^(j2 q2)
      const float C1 = 0.86602540378443864676f;
      for (int b = warp; b < nb; b += FW) {
        const uint32_t e = bt[b];
        float2* x = X + (e & 0xffffu) * FV + lane;
        const int kt = (int)(e >> 16);
        float2 a[12];
#pragma unroll
        for (int j = 0; j < 12; ++j) a[j] = x[j * sm];
#pragma unroll
        for (int j1 = 0; j1 < 3; ++j1) dft4<INV>(a[j1], a[j1 + 3], a[j1 + 6], a[j1 + 9]);           // b[j1][q2] -> a[j1 + 3 q2]
        a[4] = cmulk<INV>(a[4], C1, 0.5f);   a[5] = cmulk<INV>(a[5], 0.5f, C1);                         // q2 = 1: w12^1, w12^2
        a[7] = cmulk<INV>(a[7], 0.5f, C1);   a[8] = cmulk<INV>(a[8], -0.5f, C1);                        // q2 = 2: w12^2, w12^4
        a[10] = rot90(a[10], INV);           a[11] = make_float2(-a[11].x, -a[11].y);                   // q2 = 3: w12^3 = -i, w12^6 = -1
#pragma unroll
        for (int q2 = 0; q2 < 4; ++q2) dft3<INV>(a[3 * q2], a[3 * q2 + 1], a[3 * q2 + 2]);           // y[4 q1 + q2] -> a[3 q2 + q1]
        if (kt) {
#pragma unroll
          for (int q = 1; q < 12; ++q) a[3 * (q & 3) + (q >> 2)] = cmulf(a[3 * (q & 3) + (q >> 2)], twc<INV>(tw, q * kt));
        }
#pragma unroll
        for (int q = 0; q < 12; ++q) x[q * sm] = a[3 * (q & 3) + (q >> 2)];
      }
    } else if (r == 4) {
      for (int b = warp; b < nb; b += FW) {
        const uint32_t e = bt[b];
        float2* x = X + (e & 0xffffu) * FV + lane;
        const int kt = (int)(e >> 16);
        const float2 a0 = x[0], a1 = x[sm], a2 = x[2 * sm], a3 = x[3 * sm];
        const float2 t0 = caddf(a0, a2), t1 = csubf(a0, a2), t2 = caddf(a1, a3), t3 = rot90(csubf(a1, a3), INV);
        float2 y1 = caddf(t1, t3), y2 = csubf(t0, t2), y3 = csubf(t1, t3);
        if (kt) { y1 = cmulf(y1, twc<INV>(tw, kt)); y2 = cmulf(y2, twc<INV>(tw, 2 * kt)); y3 = cmulf(y3, twc<INV>(tw, 3 * kt)); }
        x[0] = caddf(t0, t2); x[sm] = y1; x[2 * sm] = y2; x[3 * sm] = y3;
      }
    } else if (r == 2) {
      for (int b = warp; b < nb; b += FW) {
        const uint32_t e = bt[b];
        float2* x = X + (e & 0xffffu) * FV + lane;
        const int kt = (int)(e >> 16);
        const float2 a0 = x[0], a1 = x[sm];
        float2 y1 = csubf(a0, a1);
        if (kt) y1 = cmulf(y1, twc<INV>(tw, kt));
        x[0] = caddf(a0, a1); x[sm] = y1;
      }
    } else if (r == 3) {
      for (int b = warp; b < nb; b += FW) {
        const uint32_t e = bt[b];
        float2* x = X + (e & 0xffffu) * FV + lane;
        const int kt = (int)(e >> 16);
        const float2 a0 = x[0], a1 = x[sm], a2 = x[2 * sm];
        const float2 t1 = caddf(a1, a2);
        const float2 t2 = make_float2(a0.x - 0.5f * t1.x, a0.y - 0.5f * t1.y);
        const float2 d = csubf(a1, a2);
        const float2 t3 = make_float2(0.86602540378443864676f * d.x, 0.86602540378443864676f * d.y);
        // forward: y1 = t2 - i t3, y2 = t2 + i t3 ; inverse: swapped
        float2 y1 = make_float2(t2.x + t3.y, t2.y - t3.x), y2 = make_float2(t2.x - t3.y, t2.y + t3.x);
        if (INV) { const float2 t = y1; y1 = y2; y2 = t; }
        if (kt) { y1 = cmulf(y1, twc<INV>(tw, kt)); y2 = cmulf(y2, twc<INV>(tw, 2 * kt)); }
        x[0] = caddf(a0, t1); x[sm] = y1; x[2 * sm] = y2;
      }
    } else {   // r == 5
      const float c1 = 0.30901699437494742410f, c2 = -0.80901699437494742410f;
      const float s1 = 0.95105651629515357212f, s2 = 0.58778525229247312917f;
      for (int b = warp; b < nb; b += FW) {
        const uint32_t e = bt[b];
        float2* x = X + (e & 0xffffu) * FV + lane;
        const int kt = (int)(e >> 16);
        const float2 a0 = x[0], a1 = x[sm], a2 = x[2 * sm], a3 = x[3 * sm], a4 = x[4 * sm];
        const float2 b1 = caddf(a1, a4), b2 = caddf(a2, a3), d1 = csubf(a1, a4), d2 = csubf(a2, a3);
        const float2 p1 = make_float2(a0.x + c1 * b1.x + c2 * b2.x, a0.y + c1 * b1.y + c2 * b2.y);
        const float2 p2 = make_float2(a0.x + c2 * b1.x + c1 * b2.x, a0.y + c2 * b1.y + c1 * b2.y);
        const float2 q1 = make_float2(s1 * d1.x + s2 * d2.x, s1 * d1.y + s2 * d2.y);
        const float2 q2 = make_float2(s2 * d1.x - s1 * d2.x, s2 * d1.y - s1 * d2.y);
        // forward: y1 = p1 - i q1, y4 = p1 + i q1, y2 = p2 - i q2, y3 = p2 + i q2 ; inverse: signs flipped
        float2 y1 = make_float2(p1.x + q1.y, p1.y - q1.x), y4 = make_float2(p1.x - q1.y, p1.y + q1.x);
        float2 y2 = make_float2(p2.x + q2.y, p2.y - q2.x), y3 = make_float2(p2.x - q2.y, p2.y + q2.x);
        if (INV) { float2 t = y1; y1 = y4; y4 = t; t = y2; y2 = y3; y3 = t; }
        if (kt) { y1 = cmulf(y1, twc<INV>(tw, kt)); y2 = cmulf(y2, twc<INV>(tw, 2 * kt)); y3 = cmulf(y3, twc<INV>(tw, 3 * kt)); y4 = cmulf(y4, twc<INV>(tw, 4 * kt)); }
        x[0] = caddf(a0, caddf(b1, b2)); x[sm] = y1; x[2 * sm] = y2; x[3 * sm] = y3; x[4 * sm] = y4;
      }
    }
    __syncthreads();
    bt += nb;
    L = m;
  }
}

// butterfly table of every stage (see fft_dif): entry = (g * L + k) | (k * (n / L)) << 16 for butterfly b = g * m + k
__device__ __forceinline__ void build_btab(const FftNDev& pl, uint32_t* bt) {
  int L = pl.n, off = 0;
  for (int st = 0; st < pl.nst; ++st) {
    const int r = pl.radix[st], m = L / r, nb = pl.n / r, ts = pl.n / L;
    for (int b = threadIdx.x; b < nb; b += FT) {
      const int g = b / m, k = b - g * m;
      bt[off + b] = (uint32_t)(g * L + k) | ((uint32_t)(k * ts) << 16);
    }
    off += nb; L = m;
  }
}

struct FftKParams {
  FftNDev pl;
  CUtensorMap tmap;                 // 2-D fp32 map of the input tile rows (box {64 floats, box_rows}); used when use_tma
  int use_tma, box_rows;
  const float* in; float* out_f;    // fp32 input / optional fp32 output
  uint16_t* out_hi; uint16_t* out_mid; int o_pitch, o_coff;   // optional bf16 hi/mid split output (dense pixel order of the output grid)
  const float* add; int add_cs, add_coff;                      // irfft_rows: residual view (same pixel grid as the output)
  int N, h, w, w2, C;               // C = real channels of the spatial tensor (= complex channels of T)
  int in_cs, in_coff, out_cs, out_coff;
  float scale;
};

__device__ __forceinline__ void load_tables(const FftNDev& pl, float2* tw, uint16_t* rev, uint32_t* bt) {
  for (int i = threadIdx.x; i < pl.n; i += FT) { tw[i] = __ldg(pl.tw + i); rev[i] = __ldg(pl.rev + i); }
  build_btab(pl, bt);
}

// tile rows -> X[row * FV + lane] (float2): one TMA box {64 floats, box_rows} per `box_rows` rows, or plain coalesced loads
__device__ __forceinline__ void stage_tile(const FftKParams& p, float2* X, uint64_t* bar, int nrows, int col_f, long row0,
                                           const float* base, long row_stride_f, bool lanes_ok, int lane, int warp) {
  if (p.use_tma) {
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(smem_u32(bar), (uint32_t)nrows * FV * 8u);
      for (int r0 = 0; r0 < nrows; r0 += p.box_rows)
        tma_load_2d(smem_u32(X + (size_t)r0 * FV), &p.tmap, smem_u32(bar), col_f, (int)(row0 + r0));
    }
    mbar_wait(smem_u32(bar), 0);
  } else {
    for (int r = warp; r < nrows; r += FW)
      X[(size_t)r * FV + lane] = lanes_ok ? __ldg(reinterpret_cast<const float2*>(base + (size_t)r * row_stride_f) + lane) : make_float2(0.f, 0.f);
  }
}

__device__ __forceinline__ void store_pair(const FftKParams& p, size_t pix, int ch /*first of the two real channels*/, float2 v) {
  if (p.out_f) *reinterpret_cast<float2*>(p.out_f + pix * p.out_cs + p.out_coff + ch) = v;
  if (p.out_hi) {
    const __nv_bfloat162 hb = __floats2bfloat162_rn(v.x, v.y);
    const uint32_t hbits = *reinterpret_cast<const uint32_t*>(&hb);
    const __nv_bfloat162 mb = __floats2bfloat162_rn(v.x - __uint_as_float(hbits << 16), v.y - __uint_as_float(hbits & 0xffff0000u));
    const size_t o = pix * p.o_pitch + p.o_coff + ch;
    *reinterpret_cast<uint32_t*>(p.out_hi + o) = hbits;
    *reinterpret_cast<uint32_t*>(p.out_mid + o) = *reinterpret_cast<const uint32_t*>(&mb);
  }
}

// smem: X[n][FV] float2 | tw[n] float2 | bt[nbt] u32 | rev[n] u16 | mbarrier
#define FFT_SMEM_CARVE(n)                                                                   \
  extern __shared__ __align__(128) uint8_t fsm_raw[];                                       \
  float2* X = reinterpret_cast<float2*>(fsm_raw);                                           \
  float2* tw = X + (size_t)(n) * FV;                                                        \
  uint32_t* bt = reinterpret_cast<uint32_t*>(tw + (n));                                     \
  uint16_t* rev = reinterpret_cast<uint16_t*>(bt + p.pl.nbt);                               \
  uint64_t* bar = reinterpret_cast<uint64_t*>(fsm_raw + (((size_t)(n) * FV * 8 + (size_t)(n) * 10 + (size_t)p.pl.nbt * 4 + 15) & ~(size_t)15)); \
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;                               \
  if (threadIdx.x == 0) { mbar_init(smem_u32(bar), 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// ---- forward rows: S [N*h rows][w][C] real -> T [N*h][w2][C] complex.  CTA = (row, chunk of 32 channel PAIRS)
__global__ void __launch_bounds__(FT, 3) rfft_rows_nhwc_kernel(const __grid_constant__ FftKParams p) {
  FFT_SMEM_CARVE(p.pl.n)
  const int row = blockIdx.x, chunk = blockIdx.y;
  const int pair = chunk * FV + lane;
  const bool ok = 2 * pair < p.C;
  load_tables(p.pl, tw, rev, bt);
  __syncthreads();
  stage_tile(p, X, bar, p.w, p.in_coff + chunk * 2 * FV, (long)row * p.w, p.in + ((size_t)row * p.w) * p.in_cs + p.in_coff + chunk * 2 * FV,
             p.in_cs, ok, lane, warp);
  __syncthreads();
  fft_dif<false>(X, tw, bt, p.pl, lane, warp);
  float2* dst = reinterpret_cast<float2*>(p.out_f) + (size_t)row * p.w2 * p.C;
#pragma unroll 4
  for (int k = warp; k < p.w2; k += FW) {
    const int kc = k ? p.w - k : 0;
    const float2 z = X[(size_t)rev[k] * FV + lane], zc = X[(size_t)rev[kc] * FV + lane];
    if (ok) {
      const float4 o = make_float4(0.5f * (z.x + zc.x), 0.5f * (z.y - zc.y), 0.5f * (z.y + zc.y), -0.5f * (z.x - zc.x));
      *reinterpret_cast<float4*>(dst + (size_t)k * p.C + 2 * pair) = o;       // channels 2*pair (re,im), 2*pair+1 (re,im)
    }
  }
}

// ---- columns: complex FFT over h.  forward: T -> spectrum * scale (split and/or fp32 [..][2C]); inverse: F fp32 [..][2C] -> T
// CTA = (n * w2 + kx, chunk of 32 complex channels)
template <bool INV>
__global__ void __launch_bounds__(FT, 3) fft_cols_nhwc_kernel(const __grid_constant__ FftKParams p) {
  FFT_SMEM_CARVE(p.pl.n)
  const int n = blockIdx.x / p.w2, kx = blockIdx.x - n * p.w2, chunk = blockIdx.y;
  const int ch = chunk * FV + lane;                     // complex channel
  const bool ok = ch < p.C;
  load_tables(p.pl, tw, rev, bt);
  __syncthreads();
  // input element (ky, kx, ch) as float2 at in + (((n*h + ky)*w2 + kx) * in_cs + in_coff + 2*ch) floats
  const size_t pix0 = (size_t)n * p.h * p.w2 + kx;
  stage_tile(p, X, bar, p.h, kx * p.in_cs + p.in_coff + chunk * 2 * FV, (long)n * p.h,
             p.in + pix0 * p.in_cs + p.in_coff + chunk * 2 * FV, (long)p.w2 * p.in_cs, ok, lane, warp);
  __syncthreads();
  fft_dif<INV>(X, tw, bt, p.pl, lane, warp);
#pragma unroll 4
  for (int ky = warp; ky < p.h; ky += FW) {
    float2 z = X[(size_t)rev[ky] * FV + lane];
    if (!ok) continue;
    const size_t pix = pix0 + (size_t)ky * p.w2;
    if (!INV) { z.x *= p.scale; z.y *= p.scale; }
    store_pair(p, pix, 2 * ch, z);
  }
}

// ---- inverse rows: T [N*h][w2][C] complex (+ residual) -> U [N*h][w][C] real.  CTA = (row, chunk of 32 channel pairs)
__global__ void __launch_bounds__(FT, 3) irfft_rows_nhwc_kernel(const __grid_constant__ FftKParams p) {
  FFT_SMEM_CARVE(p.pl.n)
  const int row = blockIdx.x, chunk = blockIdx.y;
  const int pair = chunk * FV + lane;
  const bool ok = 2 * pair < p.C;
  load_tables(p.pl, tw, rev, bt);
  const float2* src = reinterpret_cast<const float2*>(p.in) + (size_t)row * p.w2 * p.C;
#pragma unroll 4                                       // several rows' loads in flight per warp
  for (int k = warp; k < p.w2; k += FW) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ok) v = __ldg(reinterpret_cast<const float4*>(src + (size_t)k * p.C + 2 * pair));
    float2 A = make_float2(v.x, v.y), B = make_float2(v.z, v.w);
    const bool self = (k == 0) || (2 * k == p.w);
    if (self) { A.y = 0.f; B.y = 0.f; }                              // C2R ignores Im of the DC / Nyquist bins
    X[(size_t)k * FV + lane] = make_float2(A.x - B.y, A.y + B.x);   // A + iB
    if (!self) X[(size_t)(p.w - k) * FV + lane] = make_float2(A.x + B.y, -A.y + B.x);   // conj(A) + i conj(B)
  }
  __syncthreads();
  fft_dif<true>(X, tw, bt, p.pl, lane, warp);
#pragma unroll 4
  for (int x = warp; x < p.w; x += FW) {
    float2 z = X[(size_t)rev[x] * FV + lane];
    if (!ok) continue;
    const size_t pix = (size_t)row * p.w + x;
    z.x *= p.scale; z.y *= p.scale;
    if (p.add) { const float2 a = __ldg(reinterpret_cast<const float2*>(p.add + pix * p.add_cs + p.add_coff + 2 * pair)); z.x += a.x; z.y += a.y; }
    store_pair(p, pix, 2 * pair, z);
  }
}

// ---------------------------------------------------------------------------------------------------------------- host
struct PlanN { FftNDev dev; };
std::mutex g_mu;
std::map<std::pair<int, int>, PlanN*> g_plans;

bool factor(int n, int* radix, int* nst) {
  int r = n, k = 0;
  auto push = [&](int f) { if (k < kMaxSt) radix[k] = f; ++k; };
  while (r % 16 == 0) { push(16); r /= 16; }              // fused stages first: (4 x 4) and (4 x 3) in registers
  if (r % 12 == 0) { push(12); r /= 12; }
  while (r % 4 == 0) { push(4); r /= 4; }
  while (r % 2 == 0) { push(2); r /= 2; }
  while (r % 3 == 0) { push(3); r /= 3; }
  while (r % 5 == 0) { push(5); r /= 5; }
  *nst = k;
  return r == 1 && k <= kMaxSt && n >= 2;
}

PlanN* plan_get(int n) {
  int dev = 0; CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(g_mu);
  auto key = std::make_pair(dev, n);
  auto it = g_plans.find(key);
  if (it != g_plans.end()) return it->second;
  PlanN* p = new PlanN();
  p->dev.n = n;
  MITB_CHECK(factor(n, p->dev.radix, &p->dev.nst), "fft_nhwc: length %d is not {2,3,5}-smooth", n);
  p->dev.nbt = 0;
  for (int s = 0; s < p->dev.nst; ++s) p->dev.nbt += n / p->dev.radix[s];
  std::vector<float2> tw(n);
  for (int i = 0; i < n; ++i) { const double a = -2.0 * M_PI * (double)i / (double)n; tw[i] = make_float2((float)cos(a), (float)sin(a)); }
  // position of output k after the in-place DIF stages: pos(k; L; r1..) = (k % r1) * (L / r1) + pos(k / r1; L / r1; r2..)
  std::vector<uint16_t> rev(n);
  for (int k = 0; k < n; ++k) {
    int kk = k, L = n, pos = 0;
    for (int s = 0; s < p->dev.nst; ++s) { const int r = p->dev.radix[s]; L /= r; pos += (kk % r) * L; kk /= r; }
    rev[k] = (uint16_t)pos;
  }
  float2* dtw = nullptr; uint16_t* drev = nullptr;
  CUDA_OK(cudaMalloc(&dtw, sizeof(float2) * n)); CUDA_OK(cudaMalloc(&drev, sizeof(uint16_t) * n));
  CUDA_OK(cudaMemcpy(dtw, tw.data(), sizeof(float2) * n, cudaMemcpyHostToDevice));
  CUDA_OK(cudaMemcpy(drev, rev.data(), sizeof(uint16_t) * n, cudaMemcpyHostToDevice));
  p->dev.tw = dtw; p->dev.rev = drev;
  g_plans[key] = p;
  return p;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn enc() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr; cudaDriverEntryPointQueryResult q;
    CUDA_OK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    MITB_CHECK(p && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available in this driver");
    fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 2-D fp32 map [rows][cols_f] (row pitch in floats), box {64 floats, box_rows}; false if the shape cannot be encoded
bool make_tile_map(CUtensorMap* m, const float* base, long rows, long cols_f, long pitch_f, int box_rows) {
  if (pitch_f % 4 != 0 || ((uintptr_t)base & 15) != 0 || cols_f < 2 * FV || rows < box_rows) return false;
  const cuuint64_t gdim[2] = {(cuuint64_t)cols_f, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)pitch_f * 4};
  const cuuint32_t box[2] = {(cuuint32_t)(2 * FV), (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return enc()(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
int box_rows_for(int n) { int b = n; while (b > 256) { int d = 2; while (b % d) ++d; b /= d; } return b; }   // largest "nice" divisor <= 256

int nbt_for(int n) { int radix[kMaxSt], nst = 0, t = 0; if (!factor(n, radix, &nst)) return 0; for (int s = 0; s < nst; ++s) t += n / radix[s]; return t; }
size_t smem_for(int n) { return (((size_t)n * FV * 8 + (size_t)n * 10 + (size_t)nbt_for(n) * 4 + 15) & ~(size_t)15) + 16; }

bool use_tma_env() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("MITB_FFT_NO_TMA"); v = (e && atoi(e)) ? 0 : 1; }
  return v != 0;
}

template <class K>
void set_attr(K kernel, PerDeviceOnce& once) {
  if (once.first()) CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
}

}  // namespace

bool fft_nhwc_supported(int h, int w, int C) {
  int radix[kMaxSt], nst;
  if (!factor(h, radix, &nst) || !factor(w, radix, &nst)) return false;
  if (h > 512 || w > 512 || smem_for(h > w ? h : w) > 200 * 1024) return false;
  return C % 2 == 0 && C >= 2;
}

// S fp32 NHWC view [N][h][w][C] -> spectrum [N][h][w2][2C]: bf16 hi/mid into `spec_sv` (channels [0, 2C), no halo) when valid,
// fp32 into spec_f when non-null.  T = complex scratch of N*h*w2*C float2.
void launch_rfft2_nhwc(const View& in, const SplitView* spec_sv, float* spec_f, float2* T, cudaStream_t st) {
  const int N = in.N, h = in.H, w = in.W, C = in.C, w2 = w / 2 + 1;
  MITB_CHECK(!in.planar && fft_nhwc_supported(h, w, C) && in.cs % 2 == 0 && in.coff % 2 == 0, "rfft2_nhwc: unsupported view %dx%dx%d", h, w, C);
  MITB_CHECK(!spec_sv || !spec_sv->valid() || (spec_sv->N == N && spec_sv->H == h && spec_sv->W == w2 && spec_sv->C == 2 * C &&
                                                 spec_sv->Hp == h && spec_sv->Wp == w2), "rfft2_nhwc: spectrum split view mismatch");
  static PerDeviceOnce a1, a2;
  set_attr(rfft_rows_nhwc_kernel, a1); set_attr(fft_cols_nhwc_kernel<false>, a2);
  ProfScope ps("fft_rfft2", 2.5 * N * C * (double)h * w * log2((double)h * w), 4.0 * N * C * ((double)h * w + 2.0 * h * w2), st);
  FftKParams p; memset(&p, 0, sizeof(p));
  p.N = N; p.h = h; p.w = w; p.w2 = w2; p.C = C;
  // rows
  p.pl = plan_get(w)->dev; p.in = in.p; p.in_cs = in.cs; p.in_coff = in.coff; p.out_f = reinterpret_cast<float*>(T);
  p.box_rows = box_rows_for(w);
  p.use_tma = use_tma_env() && C % (2 * FV) == 0 && make_tile_map(&p.tmap, in.p, (long)N * h * w, in.cs, in.cs, p.box_rows);
  rfft_rows_nhwc_kernel<<<dim3(N * h, (C / 2 + FV - 1) / FV), FT, smem_for(w), st>>>(p);
  count_launch();
  // cols
  p.pl = plan_get(h)->dev; p.in = reinterpret_cast<const float*>(T); p.in_cs = 2 * C; p.in_coff = 0;
  p.out_f = spec_f; p.out_cs = 2 * C; p.out_coff = 0;
  if (spec_sv && spec_sv->valid()) { p.out_hi = spec_sv->hi; p.out_mid = spec_sv->mid; p.o_pitch = spec_sv->C; p.o_coff = 0; }
  MITB_CHECK(p.out_f || p.out_hi, "rfft2_nhwc: no output");
  p.scale = (float)(1.0 / sqrt((double)h * (double)w));
  p.box_rows = box_rows_for(h);
  p.use_tma = use_tma_env() && C % FV == 0 && make_tile_map(&p.tmap, p.in, (long)N * h, (long)w2 * 2 * C, (long)w2 * 2 * C, p.box_rows);
  fft_cols_nhwc_kernel<false><<<dim3(N * w2, (C + FV - 1) / FV), FT, smem_for(h), st>>>(p);
  count_launch();
  CUDA_OK(cudaGetLastError());
}

// F fp32 [N][h][w2][2C] (NHWC view) -> out [N][h][w][C] = irfft2(F) (+ add): bf16 hi/mid into out_sv channels [sv_coff, +C) (no
// halo) when valid, fp32 into `out` when out.p non-null.
void launch_irfft2_nhwc(const View& spec, const View& out, const SplitView* out_sv, int sv_coff, const View* add, float2* T, cudaStream_t st) {
  const int N = spec.N, h = spec.H, w2 = spec.W, C = spec.C / 2, w = out.W;
  MITB_CHECK(!spec.planar && spec.cs % 2 == 0 && spec.coff % 2 == 0 && out.H == h && w / 2 + 1 == w2 && out.C == C && out.N == N &&
             fft_nhwc_supported(h, w, C), "irfft2_nhwc: shape mismatch");
  MITB_CHECK(!add || (!add->planar && add->N == N && add->H == h && add->W == w && add->C == C && add->cs % 2 == 0 && add->coff % 2 == 0),
             "irfft2_nhwc: residual shape mismatch");
  static PerDeviceOnce a1, a2;
  set_attr(irfft_rows_nhwc_kernel, a1); set_attr(fft_cols_nhwc_kernel<true>, a2);
  ProfScope ps("fft_irfft2", 2.5 * N * C * (double)h * w * log2((double)h * w), 4.0 * N * C * ((double)h * w * (add ? 2 : 1) + 2.0 * h * w2), st);
  FftKParams p; memset(&p, 0, sizeof(p));
  p.N = N; p.h = h; p.w = w; p.w2 = w2; p.C = C;
  // cols (inverse): F -> T
  p.pl = plan_get(h)->dev; p.in = spec.p; p.in_cs = spec.cs; p.in_coff = spec.coff;
  p.out_f = reinterpret_cast<float*>(T); p.out_cs = 2 * C; p.out_coff = 0;
  p.box_rows = box_rows_for(h);
  p.use_tma = use_tma_env() && C % FV == 0 && make_tile_map(&p.tmap, spec.p, (long)N * h, (long)w2 * spec.cs, (long)w2 * spec.cs, p.box_rows);
  fft_cols_nhwc_kernel<true><<<dim3(N * w2, (C + FV - 1) / FV), FT, smem_for(h), st>>>(p);
  count_launch();
  // rows (inverse): T -> out
  p.pl = plan_get(w)->dev; p.in = reinterpret_cast<const float*>(T); p.in_cs = 2 * C; p.in_coff = 0;
  p.out_f = out.p; p.out_cs = out.cs; p.out_coff = out.coff; p.out_hi = nullptr; p.out_mid = nullptr;
  MITB_CHECK(!out.p || (!out.planar && out.cs % 2 == 0 && out.coff % 2 == 0), "irfft2_nhwc: unaligned output view");
  if (out_sv && out_sv->valid()) {
    MITB_CHECK(out_sv->N == N && out_sv->H == h && out_sv->W == w && out_sv->Hp == h && out_sv->Wp == w && sv_coff % 2 == 0 && sv_coff + C <= out_sv->C &&
               out_sv->C % 2 == 0, "irfft2_nhwc: output split view mismatch");
    p.out_hi = out_sv->hi; p.out_mid = out_sv->mid; p.o_pitch = out_sv->C; p.o_coff = sv_coff;
  }
  MITB_CHECK(p.out_f || p.out_hi, "irfft2_nhwc: no output");
  p.add = add ? add->p : nullptr; p.add_cs = add ? add->cs : 0; p.add_coff = add ? add->coff : 0;
  p.scale = (float)(1.0 / sqrt((double)h * (double)w));
  p.use_tma = 0;
  irfft_rows_nhwc_kernel<<<dim3(N * h, (C / 2 + FV - 1) / FV), FT, smem_for(w), st>>>(p);
  count_launch();
  CUDA_OK(cudaGetLastError());
}

}  // namespace mitb
