// wgmma (Hopper warpgroup MMA) implicit-GEMM convolution for sm_90a, register-gather variant.
//
// Same contract as the SIMT kernel in conv_simt.cu (tap list, zero/reflect padding, strided output mapping for the
// transposed-conv phases, BN+ReLU prologue, fused epilogue), contraction on the tensor cores.  The main path is conv_tma.cu
// (activations split once, every operand by TMA); this kernel keeps the layers that one does not take: inputs whose channel
// count is not a multiple of 8 and tiny-M / huge-K decoder layers that need split-K.
//
//   * 128-pixel x BN-channel output tile per CTA, two warpgroups of 64 rows each, fp32 accumulators in registers.
//   * fp32 accuracy from bf16 tensor cores by operand splitting ("bf16x3"): x = hi + mid with hi = bf16(x),
//     mid = bf16(x - hi); D += A_hi*B_hi + A_hi*B_mid + A_mid*B_hi.  The dropped terms are <= ~3*2^-18 relative
//     (about 1e-5), far inside the 1e-3 parity budget, at 1/3 of the bf16 tensor rate.
//   * K is consumed in blocks of 64 (one 128-byte swizzle row of bf16), two shared-memory stages.  All 256 threads gather the
//     activation block of the next stage from the NHWC view (thread = one float4 column of 8 rows; a warp load covers two
//     complete 256-byte row segments) or the planar view (two threads per row, coalesced along pixels), apply the optional
//     BN+ReLU prologue, split hi/mid and store both tiles in the K-major SWIZZLE_128B layout, while the wgmma of the previous
//     block runs; thread 0 streams the pre-split K-major bf16 weight tiles (hi/mid) with TMA onto the stage's mbarrier.
//   * Persistent: one CTA per SM loops over output tiles; split-K (splitk_reduce_kernel) when tiles cannot fill the SMs.
#include <cuda.h>
#include <string.h>
#include <cuda_bf16.h>
#include "mitb_internal.h"

namespace mitb {

namespace {

constexpr int TC_BM = 128, TC_BK = 64;
constexpr int TC_THREADS = 256;              // two warpgroups: gather + wgmma + epilogue

#include "tc_common.cuh"

struct TcParams {
  const float* in; int N, H, W, in_cs, in_coff, Cin, in_planar;
  CUtensorMap tmh, tmm;                                       // TMA descriptors of the hi / mid weight matrices
  int kpad, npad;                                             // weights [npad][kpad] bf16, K-major, zero padded
  int ntaps; int8_t tdy[kMaxTaps], tdx[kMaxTaps];
  int sy, sx, pad, Ho, Wo;
  const float* in_scale; const float* in_shift; int in_relu;
  int M, K, splits;
  int tmin_dy, tmax_dy, tmin_dx, tmax_dx;                     // extent of the tap offsets (fast interior addressing)
  EpiParams e;
};

template <int BN>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const __grid_constant__ TcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [stage 0, 1][A_hi 16K | A_mid 16K | B_hi BN*128 | B_mid BN*128], then the two "full" barriers
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  constexpr uint32_t a_bytes = TC_BM * 128, b_bytes = (uint32_t)BN * 128;
  constexpr uint32_t stage_bytes = 2 * a_bytes + 2 * b_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 2 * stage_bytes);
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar_base = smem_u32(bars);
  auto full_bar = [&](int s) { return bar_base + 8u * s; };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int nkb = p.kpad / TC_BK;
  const int mt = (p.M + TC_BM - 1) / TC_BM, nt = p.npad / BN;
  const int total_tiles = mt * nt * p.splits;
  const int HoWo = p.Ho * p.Wo;

  if (tid == 0) {
    for (int s = 0; s < 2; ++s) mbar_init(full_bar(s), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // NHWC gather: thread owns float4 column f4 of the 8 rows rb + 16 i (same swizzle phase, 2048 B apart)
  const int f4 = tid & 15, rb = tid >> 4;
  const uint32_t soff0 = (uint32_t)rb * 128u + ((((uint32_t)f4 >> 1) ^ ((uint32_t)rb & 7u)) << 4) + ((uint32_t)f4 & 1u) * 8u;
  // planar gather: two threads per GEMM row, 32 k each
  const int pr = tid & 127, phalf = tid >> 7;
  const uint32_t prow_off = (uint32_t)pr * 128u, psw = (uint32_t)(pr & 7);

  int it = 0;                                      // global K-block counter of this CTA (stage = it & 1)
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    // tile t -> (split z, M tile, N tile); N fastest so CTAs running together share the activation rows in L2
    const int z = t / (mt * nt), rr0 = t - z * (mt * nt);
    const int m0 = (rr0 / nt) * TC_BM, n0 = (rr0 % nt) * BN;
    const int kb_begin = (int)(((long)z * nkb) / p.splits), kb_end = (int)(((long)(z + 1) * nkb) / p.splits);

    // ---- NHWC row setup: pointer to the pixel under tap (0,0) and its (iy0, ix0); rows whose whole tap window lies inside the
    // image take the fast address path (pointer + per-K-block tap offset), border rows redo the padded index arithmetic
    uint32_t roff[8]; int ryx[8]; uint32_t okmask = 0, imask = 0;     // element offsets fit 32 bits (checked on the host)
    int tap = 0, ci = 0;
    // ---- planar row setup
    int pnimg = 0, ppix = 0; bool prow_ok = false;
    if (!p.in_planar) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int m = m0 + rb + 16 * i;
        ryx[i] = 0; roff[i] = 0;
        if (m < p.M) {
          const int nimg = m / HoWo, rr = m - nimg * HoWo;
          const int oy = rr / p.Wo, ox = rr - oy * p.Wo;
          const int iy0 = oy * p.sy, ix0 = ox * p.sx;
          ryx[i] = (iy0 << 16) | ix0;
          roff[i] = (uint32_t)(((size_t)(nimg * p.H + iy0) * p.W + ix0) * p.in_cs + p.in_coff);
          okmask |= 1u << i;
          if (iy0 + p.tmin_dy >= 0 && iy0 + p.tmax_dy < p.H && ix0 + p.tmin_dx >= 0 && ix0 + p.tmax_dx < p.W) imask |= 1u << i;
        }
      }
      const int k0 = kb_begin * TC_BK + f4 * 4; tap = k0 / p.Cin; ci = k0 - tap * p.Cin;
    } else {
      const int m = m0 + pr;
      prow_ok = m < p.M;
      if (prow_ok) { pnimg = m / HoWo; ppix = m - pnimg * HoWo; }
    }

    float4 v[8]; uint32_t valid = 0; int cur_ci = 0;   // NHWC block in flight
    float pv[4][8]; int pk = 0;                        // planar block in flight
    auto load_block = [&](int kbl) {
      if (!p.in_planar) {
        const int k = kbl * TC_BK + f4 * 4;
        cur_ci = ci; valid = 0;
        const bool kval = k < p.K;
        const int dy = kval ? p.tdy[tap] : 0, dx = kval ? p.tdx[tap] : 0;
        const int toff = (dy * p.W + dx) * p.in_cs + ci;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (kval && ((imask >> i) & 1u)) {
            v[i] = __ldg(reinterpret_cast<const float4*>(p.in + (roff[i] + (uint32_t)toff)));
            valid |= 1u << i;
          } else if (kval && ((okmask >> i) & 1u)) {
            const int iy0 = ryx[i] >> 16, ix0 = ryx[i] & 0xffff;
            int iy = iy0 + dy, ix = ix0 + dx;
            bool inb = true;
            if (p.pad == PAD_REFLECT) { iy = reflect_idx(iy, p.H); ix = reflect_idx(ix, p.W); }
            else inb = (iy >= 0) & (iy < p.H) & (ix >= 0) & (ix < p.W);
            if (inb) {
              v[i] = __ldg(reinterpret_cast<const float4*>(p.in + (roff[i] + (uint32_t)(((iy - iy0) * p.W + (ix - ix0)) * p.in_cs + ci))));
              valid |= 1u << i;
            }
          }
        }
        ci += TC_BK; while (ci >= p.Cin) { ci -= p.Cin; ++tap; }
      } else {
        pk = kbl * TC_BK + phalf * 32;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int k = pk + j * 8;
#pragma unroll
          for (int e = 0; e < 8; ++e)
            pv[j][e] = (prow_ok && k + e < p.K) ? __ldg(p.in + ((size_t)pnimg * p.in_cs + p.in_coff + k + e) * ((size_t)p.H * p.W) + ppix) : 0.f;
        }
      }
    };
    // BN+ReLU prologue (padding stays 0 after the transform) + hi/mid split + swizzled stores into stage s
    auto store_block = [&](int s) {
      uint8_t* a_hi = smem + (size_t)s * stage_bytes;
      uint8_t* a_mid = a_hi + a_bytes;
      if (!p.in_planar) {
        float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p.in_scale && valid) {
          sc = __ldg(reinterpret_cast<const float4*>(p.in_scale + cur_ci)); sh = __ldg(reinterpret_cast<const float4*>(p.in_shift + cur_ci));
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float4 x = v[i];
          if (p.in_scale && ((valid >> i) & 1u)) {
            x.x = x.x * sc.x + sh.x; x.y = x.y * sc.y + sh.y; x.z = x.z * sc.z + sh.z; x.w = x.w * sc.w + sh.w;
            if (p.in_relu) { x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f); }
          }
          uint2 hi, mid;
          split4(x, hi, mid);
          const uint32_t off = soff0 + (uint32_t)i * 2048u;
          *reinterpret_cast<uint2*>(a_hi + off) = hi;
          *reinterpret_cast<uint2*>(a_mid + off) = mid;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int k = pk + j * 8;
          if (p.in_scale && prow_ok) {
#pragma unroll
            for (int e = 0; e < 8; ++e)
              if (k + e < p.K) {
                const float tt = pv[j][e] * __ldg(p.in_scale + k + e) + __ldg(p.in_shift + k + e);
                pv[j][e] = p.in_relu ? fmaxf(tt, 0.f) : tt;
              }
          }
          uint4 hi, mid;
          split8(pv[j], hi, mid);
          const uint32_t off = prow_off + ((((uint32_t)(phalf * 4 + j)) ^ psw) << 4);
          *reinterpret_cast<uint4*>(a_hi + off) = hi;
          *reinterpret_cast<uint4*>(a_mid + off) = mid;
        }
      }
    };

    float acc[BN / 2];
    load_block(kb_begin);
    for (int kb = kb_begin; kb < kb_end; ++kb, ++it) {
      const int s = it & 1;
      wgmma_wait<1>();                                 // this warp's MMAs of block it-2 (the last reader of stage s) are done
      __syncthreads();                                 // ... and every other warp's
      if (tid == 0) {
        mbar_arrive_expect_tx(full_bar(s), 2 * b_bytes);
        const uint32_t b_hi = smem_base + (uint32_t)s * stage_bytes + 2 * a_bytes;
        tma_load_2d(b_hi, &p.tmh, full_bar(s), kb * TC_BK, n0);
        tma_load_2d(b_hi + b_bytes, &p.tmm, full_bar(s), kb * TC_BK, n0);
      }
      store_block(s);
      fence_async_smem();                              // generic-proxy stores -> async-proxy (wgmma) reads
      if (kb + 1 < kb_end) load_block(kb + 1);         // in flight while this block is multiplied
      __syncthreads();
      mbar_wait(full_bar(s), (it >> 1) & 1);
      const uint32_t a_hi = smem_base + (uint32_t)s * stage_bytes + (uint32_t)wg * (64u * 128u), a_mid = a_hi + a_bytes;
      const uint32_t b_hi = smem_base + (uint32_t)s * stage_bytes + 2 * a_bytes, b_mid = b_hi + b_bytes;
      fence_acc(acc);
      wgmma_fence();
      wgmma_kblock_x3<BN>(acc, make_desc_sw128(a_hi), make_desc_sw128(a_mid), make_desc_sw128(b_hi), make_desc_sw128(b_mid), kb == kb_begin);
      wgmma_commit();
      fence_acc(acc);
    }
    wgmma_wait<0>();
    fence_acc(acc);
    epilogue_tile<-1, BN>(p.e, acc, wg * 64 + (warp & 3) * 16 + (lane >> 2), n0, z, [&](int r, int& nimg, int& oy, int& ox) -> bool {
      const int m = m0 + r;
      if (m >= p.M) return false;
      nimg = m / HoWo; const int pp = m - nimg * HoWo;
      oy = pp / p.Wo; ox = pp - oy * p.Wo;
      return true;
    });
  }
}

// split-K second pass: sum the partials and run the regular epilogue (one thread per 4 output channels of a pixel)
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const __grid_constant__ EpiParams p, int splits) {
  const int nq = (p.Cout + 3) / 4;
  const long total = (long)p.M * nq;
  const int HoWo = p.Ho * p.Wo;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int m = (int)(i / nq), cq = (int)(i - (long)m * nq) * 4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int z = 0; z < splits; ++z) {
      const float4 t = *reinterpret_cast<const float4*>(p.partial + ((size_t)z * p.M + m) * p.npad + cq);
      acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
    }
    const int nimg = m / HoWo, rr = m - nimg * HoWo;
    const int py = (rr / p.Wo) * p.oy_mul + p.oy_add, px = (rr % p.Wo) * p.ox_mul + p.ox_add;
    const size_t opix = ((size_t)nimg * p.oH + py) * p.oW + px;
    const size_t oplane = (size_t)p.oH * p.oW, opl_pix = (size_t)py * p.oW + px;
    float v4[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = cq + e;
      if (c >= p.Cout) break;
      float x = v4[e];
      if (p.add0) x += p.add0_planar ? p.add0[((size_t)nimg * p.add0_cs + p.add0_coff + c) * oplane + opl_pix] : p.add0[opix * p.add0_cs + p.add0_coff + c];
      if (p.scale) x *= __ldg(p.scale + c);
      if (p.shift) x += __ldg(p.shift + c);
      x = apply_act(x, p.act);
      if (p.mul1) x *= __ldg(p.mul1 + c);
      if (p.add1) x += p.add1_planar ? p.add1[((size_t)nimg * p.add1_cs + p.add1_coff + c) * oplane + opl_pix] : p.add1[opix * p.add1_cs + p.add1_coff + c];
      if (p.out_planar) p.out[((size_t)nimg * p.out_cs + p.out_coff + c) * oplane + opl_pix] = x;
      else p.out[opix * p.out_cs + p.out_coff + c] = x;
    }
  }
}

// fp32 K-major [K][ldw] (the SIMT layout) -> bf16 hi/mid [npad][kpad] K-major, zero padded
__global__ void split_weights_kernel(const float* w, int K, int Cout, int ldw, uint16_t* wh, uint16_t* wm, int kpad, int npad) {
  const long total = (long)npad * kpad;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int k = (int)(i % kpad), n = (int)(i / kpad);
    float x = (k < K && n < Cout) ? w[(size_t)k * ldw + n] : 0.f;
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    const __nv_bfloat16 m = __float2bfloat16_rn(x - __bfloat162float(h));
    wh[i] = __bfloat16_as_ushort(h); wm[i] = __bfloat16_as_ushort(m);
  }
}

// same, with every tap's channel range padded to cp (multiple of 64): k' = tap*cp + c
__global__ void split_weights_padded_kernel(const float* w, int ntaps, int Cin, int cp, int Cout, int ldw, uint16_t* wh, uint16_t* wm, int npad) {
  const int kp = ntaps * cp;
  const long total = (long)npad * kp;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int k = (int)(i % kp), n = (int)(i / kp);
    const int tap = k / cp, c = k - tap * cp;
    float x = (c < Cin && n < Cout) ? w[(size_t)(tap * Cin + c) * ldw + n] : 0.f;
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    const __nv_bfloat16 m = __float2bfloat16_rn(x - __bfloat162float(h));
    wh[i] = __bfloat16_as_ushort(h); wm[i] = __bfloat16_as_ushort(m);
  }
}

// N tile of the weight copies (and of the row-stat layout): at most 128 columns (64 fp32 accumulator registers per thread of a
// warpgroup), a multiple of 32 (the wgmma widths instantiated)
int pick_bn(int Cout) {
  const int tiles = (Cout + 127) / 128;
  int bn = (Cout + tiles - 1) / tiles;
  bn = (bn + 31) & ~31;
  if (bn < 32) bn = 32;
  return bn;
}

}  // namespace

static bool g_tc_enabled = true;
void conv_tc_set_enabled(bool on) { g_tc_enabled = on; }
bool conv_tc_enabled() { return g_tc_enabled; }

// fp32 K-major [(ky*kw+kx)*4 + c][ldw] -> bf16 hi/mid [npad][kh*64] with k = ky*64 + kx*8 + c (zero elsewhere): Cin = 4 stems
__global__ void split_weights_stem8_kernel(const float* w, int kh, int kw, int Cout, int ldw, uint16_t* wh, uint16_t* wm, int npad) {
  const int kp = kh * 64;
  const long total = (long)npad * kp;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int k = (int)(i % kp), n = (int)(i / kp);
    const int ky = k >> 6, kx = (k & 63) >> 3, c = k & 7;
    float x = (kx < kw && c < 4 && n < Cout) ? w[(size_t)((ky * kw + kx) * 4 + c) * ldw + n] : 0.f;
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    const __nv_bfloat16 m = __float2bfloat16_rn(x - __bfloat162float(h));
    wh[i] = __bfloat16_as_ushort(h); wm[i] = __bfloat16_as_ushort(m);
  }
}

// Build the tensor-core weight copies for a conv (called at load time by the Loader)
void conv_tc_prepare(ConvW& cw, DevBlob& blob, cudaStream_t st) {
  const int K = cw.ntaps * cw.Cin;
  const int bn = pick_bn(cw.Cout);
  const int ntiles = (cw.Cout + bn - 1) / bn;
  cw.tc_bn = bn; cw.tc_kpad = (K + TC_BK - 1) / TC_BK * TC_BK; cw.tc_npad = ntiles * bn;
  const size_t n = (size_t)cw.tc_npad * cw.tc_kpad;
  uint16_t* wh = (uint16_t*)blob.alloc_f((n + 1) / 2 + 4);
  uint16_t* wm = (uint16_t*)blob.alloc_f((n + 1) / 2 + 4);
  int blocks = (int)((n + 255) / 256); if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
  split_weights_kernel<<<blocks, 256, 0, st>>>(cw.w, K, cw.Cout, cw.ldw, wh, wm, cw.tc_kpad, cw.tc_npad);
  CUDA_OK(cudaGetLastError());
  cw.wh = wh; cw.wm = wm;
  if (cw.Cin % 64 != 0 && cw.Cin % 8 == 0 && cw.Cin >= 16) {
    // the TMA-fed kernel consumes K blocks of 64 channels of one tap: give it a copy with each tap padded to a multiple of 64
    const int cp = (cw.Cin + 63) / 64 * 64;
    const size_t np = (size_t)cw.tc_npad * cw.ntaps * cp;
    uint16_t* whp = (uint16_t*)blob.alloc_f((np + 1) / 2 + 4);
    uint16_t* wmp = (uint16_t*)blob.alloc_f((np + 1) / 2 + 4);
    int b2 = (int)((np + 255) / 256); if (b2 > device_sm_count() * 16) b2 = device_sm_count() * 16;
    split_weights_padded_kernel<<<b2, 256, 0, st>>>(cw.w, cw.ntaps, cw.Cin, cp, cw.Cout, cw.ldw, whp, wmp, cw.tc_npad);
    CUDA_OK(cudaGetLastError());
    cw.whp = whp; cw.wmp = wmp; cw.tc_cp = cp;
  }
  if (cw.Cin == 4 && cw.ntaps > 1) {
    // full kh x kw tap grid in row-major order (what Loader::conv / conv_padcin produce)? then pack the stem layout
    int kw = 1; while (kw < cw.ntaps && cw.tdy[kw] == cw.tdy[0]) ++kw;
    const int kh = cw.ntaps / kw;
    bool grid = kh * kw == cw.ntaps && kw <= 8;
    for (int t = 0; t < cw.ntaps && grid; ++t) grid = cw.tdy[t] == cw.tdy[0] + t / kw && cw.tdx[t] == cw.tdx[0] + t % kw;
    if (grid) {
      const size_t n8 = (size_t)cw.tc_npad * kh * 64;
      uint16_t* w8h = (uint16_t*)blob.alloc_f((n8 + 1) / 2 + 4);
      uint16_t* w8m = (uint16_t*)blob.alloc_f((n8 + 1) / 2 + 4);
      int b3 = (int)((n8 + 255) / 256); if (b3 > device_sm_count() * 16) b3 = device_sm_count() * 16;
      split_weights_stem8_kernel<<<b3, 256, 0, st>>>(cw.w, kh, kw, cw.Cout, cw.ldw, w8h, w8m, cw.tc_npad);
      CUDA_OK(cudaGetLastError());
      cw.w8h = w8h; cw.w8m = w8m; cw.w8_kh = kh; cw.w8_kw = kw;
    }
  }
}

bool conv_tc_supported(const ConvOp& op) {
  if (!g_tc_enabled || !op.wt.wh || !op.wt.wm) return false;
  const int K = op.wt.ntaps * op.in.C;
  if (K < 32) return false;
  if (op.in.planar) return op.wt.ntaps == 1;
  return op.in.C % 4 == 0 && op.in.cs % 4 == 0 && op.in.coff % 4 == 0;
}

// the register-gather kernel, split-K over `splits` (conv_plan()) with a second reduce launch
void launch_conv_tc(const ConvOp& op, int splits, cudaStream_t st) {
  const ConvW& w = op.wt;
  TcParams p;
  p.in = op.in.p; p.N = op.in.N; p.H = op.in.H; p.W = op.in.W; p.in_cs = op.in.cs; p.in_coff = op.in.coff; p.Cin = op.in.C;
  p.in_planar = op.in.planar;
  make_w_tmap(&p.tmh, w.wh, w.tc_kpad, w.tc_npad, w.tc_bn);
  make_w_tmap(&p.tmm, w.wm, w.tc_kpad, w.tc_npad, w.tc_bn);
  p.kpad = w.tc_kpad; p.npad = w.tc_npad;
  p.ntaps = w.ntaps;
  p.tmin_dy = p.tmin_dx = 127; p.tmax_dy = p.tmax_dx = -127;
  for (int t = 0; t < w.ntaps; ++t) {
    p.tdy[t] = w.tdy[t]; p.tdx[t] = w.tdx[t];
    if (w.tdy[t] < p.tmin_dy) p.tmin_dy = w.tdy[t];
    if (w.tdy[t] > p.tmax_dy) p.tmax_dy = w.tdy[t];
    if (w.tdx[t] < p.tmin_dx) p.tmin_dx = w.tdx[t];
    if (w.tdx[t] > p.tmax_dx) p.tmax_dx = w.tdx[t];
  }
  p.sy = op.sy; p.sx = op.sx; p.pad = op.pad; p.Ho = op.Ho; p.Wo = op.Wo;
  p.in_scale = op.in_scale; p.in_shift = op.in_shift; p.in_relu = op.in_relu;
  fill_epi(p.e, op);
  MITB_CHECK(!op.stat_max || op.stat_ld == 2 * (w.tc_npad / w.tc_bn), "tc conv: stat_ld must equal conv_stat_blocks(op)");
  p.M = op.in.N * op.Ho * op.Wo; p.K = w.ntaps * op.in.C;
  const int BN = w.tc_bn;
  MITB_CHECK(BN >= 32 && BN <= 128 && BN % 32 == 0, "tc conv: bad BN %d", BN);
  MITB_CHECK(p.in_planar || p.Cin % 4 == 0, "tc conv: Cin must be a multiple of 4");
  MITB_CHECK((size_t)op.in.pixels() * op.in.cs < (size_t)1 << 31, "tc conv: input tensor too large for 32-bit element offsets");
  const size_t stage_bytes = 2 * (size_t)TC_BM * 128 + 2 * (size_t)BN * 128;
  const size_t smem = 2 * stage_bytes + 2 * 8 + 1024;
  const int num_sms = device_sm_count();
  static PerDeviceOnce tc_attr;
  if (tc_attr.first()) {
    CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<96>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  }
  const int tiles = ((p.M + TC_BM - 1) / TC_BM) * (p.npad / BN);
  p.splits = splits;
  if (splits > 1) {
    const size_t need = (size_t)splits * p.M * p.npad * sizeof(float);
    static DeviceScratch g_partial;                                           // split-K partial sums
    p.e.partial = static_cast<float*>(g_partial.get(need)); p.e.npad = p.npad;
  }
  const int total_tiles = tiles * splits;
  const int grid = total_tiles < num_sms ? total_tiles : num_sms;      // persistent: one CTA per SM
  conv_trace(splits > 1 ? CK_GATHER_SPLITK : CK_GATHER, BN, splits, p.e.vec2, -2, false);
  switch (BN) {
    case 32: conv_tc_kernel<32><<<grid, TC_THREADS, smem, st>>>(p); break;
    case 64: conv_tc_kernel<64><<<grid, TC_THREADS, smem, st>>>(p); break;
    case 96: conv_tc_kernel<96><<<grid, TC_THREADS, smem, st>>>(p); break;
    default: conv_tc_kernel<128><<<grid, TC_THREADS, smem, st>>>(p); break;
  }
  count_launch();
  if (splits > 1) {
    const long total = (long)p.M * ((op.out.C + 3) / 4);
    int blocks = (int)((total + 255) / 256); if (blocks > num_sms * 8) blocks = num_sms * 8;
    splitk_reduce_kernel<<<blocks, 256, 0, st>>>(p.e, splits);
    count_launch();
  }
  CUDA_OK(cudaGetLastError());
}

}  // namespace mitb
