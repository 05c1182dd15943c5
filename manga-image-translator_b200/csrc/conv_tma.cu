// TMA-fed wgmma implicit-GEMM convolution for sm_90a (stride 1 or 2, Cin a multiple of 8; the main conv path).
//
// conv_tc.cu gathers the fp32 activation tile with the MMA warps and splits it into bf16 hi/mid inside the main loop, and a
// 3x3 conv repeats the conversion of every input element 9 times (once per tap) per N tile.  Here the conversion happens ONCE
// per input element in a separate memory-bound pass (split_pad_kernel: fp32 view -> dense bf16 hi / mid NHWC tensors, optional
// BN+ReLU prologue, reflect halo materialised, planar inputs transposed), and the GEMM main loop only moves operands by TMA:
//   warp 8      producer: per K block (= 64 channels of one tap) four TMA loads - the activation box {64 ch, bw, bh} of the
//               hi and mid tensors at the tap-shifted pixel coordinates (zero padding = TMA out-of-bounds fill) and the
//               weight boxes {64 k, BN} - all landing in the K-major SWIZZLE_128B layout, completing on the stage's "full"
//               mbarrier (expect_tx); a ring of 3..6 stages; warps 9-11 of its warpgroup exit once they gave up their registers;
//   warps 0-7   two consumer warpgroups in ping-pong: each owns whole 128-row tiles, alternately, and issues 24 wgmma per K
//               block (two 64-row halves, bf16x3: Ah*Bh + Ah*Bm + Am*Bh, fp32 accumulators in registers); the stage is released
//               on its "empty" mbarrier once the wgmma that read it retired (one K block of wgmma stays in flight); then the
//               epilogue ((+add0)*scale+shift -> act -> *mul1 -> +add1 -> fp32 stores and / or split operands), staged through
//               shared memory (epilogue_staged) or, for planar / unaligned outputs and the vocabulary head, straight from the
//               accumulator registers (tc_common.cuh), while the other warpgroup's main loop runs on the tensor core.
// Operand fusion (ConvOp::in_sv / out_sv / seg2): a producer's epilogue can store its result directly as the consumer's bf16
// hi/mid operand tensor (SplitView, optionally with a reflect halo and the consumer's BN+ReLU prologue applied), so the split
// pass disappears; and a second K segment with its own tensor maps lets two convolutions of different inputs accumulate into one
// accumulator (FFC: conv1x1(U) + conv3x3_{l->g}(x_l) -> BN_g -> ReLU -> +residual in ONE launch).
// An output tile is a bh x bw pixel patch of one image (bw*bh = 128, bw a power of two) so that a tap is a rectangular TMA
// box; 1x1 convs use the flattened [pixels][C] matrix (bw = 128, bh = 1).  Persistent CTAs, one per SM.
#include <cuda.h>
#include <string.h>
#include <stdio.h>
#include <stdlib.h>
#include <cuda_bf16.h>
#include "mitb_internal.h"

namespace mitb {

namespace {

constexpr int TC_BM = 128, TC_BK = 64;
constexpr int TM_WG_WARPS = 4;
constexpr int TM_THREADS = 3 * TM_WG_WARPS * 32;     // two consumer warpgroups + the producer warpgroup
// Register split: 2 x 128 x 232 + 128 x 40 <= 64 K.  Any 3 warps of one SM sub-partition are capped at 168 registers each
// otherwise, too few for a warpgroup's 128 x 128 accumulator (128 registers) next to its epilogue.
constexpr int TM_CONSUMER_REGS = 232, TM_PRODUCER_REGS = 40;

#include "tc_common.cuh"

struct SegParams {                                             // one K segment = one input tensor
  CUtensorMap ta_hi, ta_mid;                                  // activations: 4-D (C, Wp, Hp, N) bf16, box {64, bw, bh, 1}
  int ntaps, cblks, c0; int8_t tdy[kMaxTaps], tdx[kMaxTaps];  // channel offset of the slice; tap offsets in (padded) input coordinates
};
struct TmaParams {
  SegParams seg[2]; int nseg, nkb;
  CUtensorMap tb_hi, tb_mid;                                  // weights: 2-D (K, Npad) bf16, box {64, BN}
  int N, Ho, Wo, M, lin;                                      // lin: tile = 128 consecutive rows of the flattened [M][C] matrix
  int sy, sx;                                                 // conv stride (TMA element strides of the activation box)
  int bw_log2, tiles_x, tiles_y;
  int npad, stages;
  int staged;                                                 // fused chain through epilogue_staged (stage_epilogue), else epilogue_tile
  int bar_off;                                                // shared-memory offset of the barriers: after the stages and, if
                                                              // the epilogue is staged, its chunks and row tables
  const uint8_t* tile_need;                                   // per 128-row M tile: 0 = skip (ConvOp::need_px reduced over the tile), null: all
  EpiParams e;
};

// Phase timing (build with EXTRA=-DMITB_CONV_PHASES, read by tools/conv_phases.py): clock64 sums over all consumer warpgroups
// of a launch for [0] the wait on a tile's first full barrier, [1] the main loop, [2] wgmma_wait<0>, [3] the epilogue; [4] counts
// processed tiles; [5..7] split a staged epilogue into chunk writes + barriers, column vector loads and the row walk (sums over
// all consumer threads).  The default build contains none of it.
constexpr int N_PHASES = 8;
#ifdef MITB_CONV_PHASES
__device__ unsigned long long g_conv_phases[N_PHASES];
#define PHASE_CLOCK(v) v = clock64()
#else
#define PHASE_CLOCK(v)
#endif

template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// ---- Staged epilogue of the fused chain (EpiParams::vec2 outputs).  In the accumulator layout a thread holds 2 columns of each
// 8-column group in 4 rows, so a chain applied straight from the registers moves 8 bytes per row and address, and each thread has
// few independent values to hide the latency of its loads with.  Instead each consumer warpgroup passes its tile through shared memory
// 32 columns at a time: the fragments are written to a 128 x 32 fp32 chunk and read back row-major, each thread owning W (4, or 2
// where the operands' alignment allows only 8 bytes) fixed channels and walking the rows.  A warp then moves whole 128-byte row
// segments of out / add0 / add1 (64 bytes of os_hi / os_mid) per instruction, the column vectors are loaded once per chunk, and the
// latency is hidden by rows in flight.  The element chain is epi_chain2 / epi_split2, as in epilogue_tile.
constexpr int EPI_CW = 32;                                                   // columns per chunk
constexpr uint32_t EPI_CHUNK_BYTES = TC_BM * EPI_CW * 4;                     // 16 KB per consumer warpgroup
constexpr uint32_t EPI_SMEM_BYTES = 2 * (EPI_CHUNK_BYTES + TC_BM * 4);       // + per warpgroup a 128-entry row table

// float offset of (row r, column col) in a chunk: the 16-byte units of a row are XOR-swizzled by r & 3, so that the fragment stores
// (a half warp writes 32 bytes of each of 4 consecutive rows) and the row reads (8 or 16 lanes read 128 bytes of one row) are both
// free of bank conflicts
__device__ __forceinline__ int chunk_off(int r, int col) { return r * EPI_CW + (((col >> 2) ^ ((r & 3) << 1)) << 2) + (col & 3); }

template <int W> __device__ __forceinline__ void ld_w(float (&v)[W], const float* q);
template <> __device__ __forceinline__ void ld_w<4>(float (&v)[4], const float* q) {
  const float4 t = *reinterpret_cast<const float4*>(q); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <> __device__ __forceinline__ void ld_w<2>(float (&v)[2], const float* q) {
  const float2 t = *reinterpret_cast<const float2*>(q); v[0] = t.x; v[1] = t.y;
}
template <int W> __device__ __forceinline__ void ldg_w(float (&v)[W], const float* q);
template <> __device__ __forceinline__ void ldg_w<4>(float (&v)[4], const float* q) {
  const float4 t = __ldg(reinterpret_cast<const float4*>(q)); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <> __device__ __forceinline__ void ldg_w<2>(float (&v)[2], const float* q) {
  const float2 t = __ldg(reinterpret_cast<const float2*>(q)); v[0] = t.x; v[1] = t.y;
}
template <int W> __device__ __forceinline__ void st_w(float* q, const float (&v)[W]);
template <> __device__ __forceinline__ void st_w<4>(float* q, const float (&v)[4]) { *reinterpret_cast<float4*>(q) = make_float4(v[0], v[1], v[2], v[3]); }
template <> __device__ __forceinline__ void st_w<2>(float* q, const float (&v)[2]) { *reinterpret_cast<float2*>(q) = make_float2(v[0], v[1]); }
template <int W> __device__ __forceinline__ void st_bf16_w(uint16_t* q, const uint32_t (&v)[W / 2]);
template <> __device__ __forceinline__ void st_bf16_w<4>(uint16_t* q, const uint32_t (&v)[2]) { *reinterpret_cast<uint2*>(q) = make_uint2(v[0], v[1]); }
template <> __device__ __forceinline__ void st_bf16_w<2>(uint16_t* q, const uint32_t (&v)[1]) { *reinterpret_cast<uint32_t*>(q) = v[0]; }

// Rows in flight per thread in epilogue_staged: as many as the registers left next to the accumulators hold without spills
// (ptxas -v over every instantiation).  Each row in flight holds W chunk values, W per residual operand and two pixel indices.  The
// generic signature keeps registers for every operand: at BN = 128 the 96 accumulator registers still live during the first chunk
// leave room for one 16-byte row only.
template <int SIG, int BN, int W> __host__ __device__ constexpr int epi_rows() {
  if (SIG == EPI_GENERIC) return (BN == 128 ? 4 : 8) / W;
  const int res = ((SIG & EPI_ADD0) ? 1 : 0) + ((SIG & EPI_ADD1) ? 1 : 0);
  return res == 0 ? 32 / W : res == 1 ? 16 / W : (BN == 128 ? 4 : 8) / W;
}

#ifdef MITB_CONV_PHASES
#define EPI_CLOCK(i) do { const long long now_ = clock64(); ep[i] += now_ - ep_t; ep_t = now_; } while (0)
#else
#define EPI_CLOCK(i)
#endif

// The fused chain of one 128 x BN tile: acc0 holds rows 0-63, acc1 rows 64-127 (fragment layout of epilogue_tile; `row` is this
// thread's first row); both are consumed.  rowpix(r, ...) as in epilogue_tile; rowm(r) is the tile row's index in the logical output
// grid, which is the pixel index of out / add0 / add1 whenever there is a split output (launch_conv_tma admits out_sv only on the conv's
// own grid), so the row table needs one entry per row.  `bar` is this warpgroup's named barrier.  SIG (EpiSig) is the launch's
// epilogue signature: only its operands are declared, loaded and applied.  ep: phase-timer sums (chunk writes + barriers, column
// vector loads, row walk), MITB_CONV_PHASES builds only.
template <int ACT, int BN, int W, int SIG, class RowPix, class RowM>
__device__ __forceinline__ void epilogue_staged(const EpiParams& e, float (&acc0)[BN / 2], float (&acc1)[BN / 2], int row, int n0, float* chunk,
                                                int* rtab, int bar, RowPix rowpix, RowM rowm, long long* ep) {
  constexpr int TPR = EPI_CW / W, RPP = TC_BM / TPR, NR = epi_rows<SIG, BN, W>();   // threads per row, rows per pass, rows in flight
  static_assert((TC_BM / RPP) % NR == 0, "rows in flight must divide a thread's rows");
  const bool add0 = epi_has<SIG, EPI_ADD0>(e.add0), add1 = epi_has<SIG, EPI_ADD1>(e.add1), out = epi_has<SIG, EPI_OUT>(e.out);
  const bool os = epi_has<SIG, EPI_OS>(e.os_hi), os_aff = epi_has<SIG, EPI_OS_AFFINE>(e.os_scale);
  constexpr bool kA0 = SIG == EPI_GENERIC || (SIG & EPI_ADD0), kA1 = SIG == EPI_GENERIC || (SIG & EPI_ADD1);   // arrays to declare
#ifdef MITB_CONV_PHASES
  long long ep_t = clock64();
#endif
  const int t = threadIdx.x & 127, cl = 2 * (t & 3);
  const int q = t % TPR, r0 = t / TPR;
  named_bar_sync(bar, 128);                           // the previous tile's reads of the chunk and the row table are done
  {
    // row table: pixel index of the split output if there is one, else of out; -1 outside the output
    int nimg = 0, oy = 0, ox = 0;
    const bool ok = rowpix(t, nimg, oy, ox);
    rtab[t] = !ok ? -1 : os ? (nimg * e.os_Hp + oy + e.os_pt) * e.os_Wp + ox + e.os_pl
                            : (nimg * e.oH + oy * e.oy_mul + e.oy_add) * e.oW + ox * e.ox_mul + e.ox_add;
  }
#pragma unroll 1
  for (int c0 = n0; c0 < n0 + BN && c0 < e.Cout; c0 += EPI_CW) {
    if (c0 != n0) named_bar_sync(bar, 128);           // the previous chunk's reads are done
    // this chunk's fragments, acc[0..15] (the registers rotate down by one chunk per iteration): columns 8 jj + cl, rows row + 8 h.
    // The 16 store addresses are recomputed per chunk (rr is opaque to the compiler): hoisted out of the loop they would hold 16
    // registers through it and make the BN = 128 instantiations spill.
    int rr = row;
    asm volatile("" : "+r"(rr));
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        *reinterpret_cast<float2*>(chunk + chunk_off(rr + 8 * h, 8 * jj + cl)) = make_float2(acc0[4 * jj + 2 * h], acc0[4 * jj + 2 * h + 1]);
        *reinterpret_cast<float2*>(chunk + chunk_off(64 + rr + 8 * h, 8 * jj + cl)) = make_float2(acc1[4 * jj + 2 * h], acc1[4 * jj + 2 * h + 1]);
      }
    }
    named_bar_sync(bar, 128);
    EPI_CLOCK(0);
    const int c = c0 + W * q;                           // Cout is a multiple of W: a thread's channels are all inside or all past it
    if (c < e.Cout) {
      float sc[W], sh[W], m1[W], os_s[W], os_t[W];
#pragma unroll
      for (int k = 0; k < W; ++k) sc[k] = sh[k] = m1[k] = os_s[k] = os_t[k] = 0.f;
      if (epi_has<SIG, EPI_SCALE>(e.scale)) ldg_w<W>(sc, e.scale + c);
      if (epi_has<SIG, EPI_SHIFT>(e.shift)) ldg_w<W>(sh, e.shift + c);
      if (epi_has<SIG, EPI_MUL1>(e.mul1)) ldg_w<W>(m1, e.mul1 + c);
      if (os_aff) { ldg_w<W>(os_s, e.os_scale + c); ldg_w<W>(os_t, e.os_shift + c); }
      EPI_CLOCK(1);
#pragma unroll 1
      for (int i0 = 0; i0 < TC_BM / RPP; i0 += NR) {
        // the chunk reads and residual loads of all rows in flight ahead of the first chain and store: add0 / add1 may alias out
        int px[NR], opx[NR];
        float v[NR][W], a0[kA0 ? NR : 1][W], a1[kA1 ? NR : 1][W];
#pragma unroll
        for (int i = 0; i < NR; ++i) {
          const int r = r0 + (i0 + i) * RPP;
          px[i] = rtab[r];
          opx[i] = os ? rowm(r) : px[i];
          ld_w<W>(v[i], chunk + chunk_off(r, W * q));
          if constexpr (kA0) {
#pragma unroll
            for (int k = 0; k < W; ++k) a0[i][k] = 0.f;
            if (add0 && px[i] >= 0) ld_w<W>(a0[i], e.add0 + (size_t)opx[i] * e.add0_cs + e.add0_coff + c);
          }
          if constexpr (kA1) {
#pragma unroll
            for (int k = 0; k < W; ++k) a1[i][k] = 0.f;
            if (add1 && px[i] >= 0) ld_w<W>(a1[i], e.add1 + (size_t)opx[i] * e.add1_cs + e.add1_coff + c);
          }
        }
#pragma unroll
        for (int i = 0; i < NR; ++i) {
          if (px[i] < 0) continue;
          const int ia0 = kA0 ? i : 0, ia1 = kA1 ? i : 0;
#pragma unroll
          for (int k = 0; k < W; k += 2)
            epi_chain2<ACT, SIG>(e, v[i][k], v[i][k + 1], kA0 ? make_float2(a0[ia0][k], a0[ia0][k + 1]) : make_float2(0.f, 0.f),
                                 make_float2(sc[k], sc[k + 1]), make_float2(sh[k], sh[k + 1]), make_float2(m1[k], m1[k + 1]),
                                 kA1 ? make_float2(a1[ia1][k], a1[ia1][k + 1]) : make_float2(0.f, 0.f));
          if (out) st_w<W>(e.out + (size_t)opx[i] * e.out_cs + e.out_coff + c, v[i]);
          if (os) {
            uint32_t hh[W / 2], mm[W / 2];
#pragma unroll
            for (int k = 0; k < W; k += 2)
              epi_split2<SIG>(e, v[i][k], v[i][k + 1], make_float2(os_s[k], os_s[k + 1]), make_float2(os_t[k], os_t[k + 1]), hh[k / 2], mm[k / 2]);
            const size_t so = (size_t)px[i] * e.os_pitch + e.os_coff + c;
            st_bf16_w<W>(e.os_hi + so, hh);
            st_bf16_w<W>(e.os_mid + so, mm);
          }
        }
      }
    }
    EPI_CLOCK(2);
#pragma unroll
    for (int i = 0; i + 16 < BN / 2; ++i) { acc0[i] = acc0[i + 16]; acc1[i] = acc1[i + 16]; }
  }
}
#undef EPI_CLOCK

// expect_tx + the four operand boxes of one K block, issued by one elected lane of a converged warp
__device__ __forceinline__ void tma_kblock(uint32_t bar, uint32_t bytes, uint32_t a_hi, uint32_t a_mid, uint32_t b_hi, uint32_t b_mid,
                                           const CUtensorMap* ta_hi, const CUtensorMap* ta_mid, const CUtensorMap* tb_hi,
                                           const CUtensorMap* tb_mid, int c, int x, int y, int n, int k, int n0) {
  asm volatile(
      "{\n"
      ".reg .pred pe;\n"
      "elect.sync _|pe, 0xffffffff;\n"
      "@pe mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n"
      "@pe cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%2], [%6, {%10, %11, %12, %13}], [%0];\n"
      "@pe cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%3], [%7, {%10, %11, %12, %13}], [%0];\n"
      "@pe cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%4], [%8, {%14, %15}], [%0];\n"
      "@pe cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%5], [%9, {%14, %15}], [%0];\n"
      "}\n" ::"r"(bar), "r"(bytes), "r"(a_hi), "r"(a_mid), "r"(b_hi), "r"(b_mid), "l"(ta_hi), "l"(ta_mid), "l"(tb_hi), "l"(tb_mid),
      "r"(c), "r"(x), "r"(y), "r"(n), "r"(k), "r"(n0) : "memory");
}

// SIG: EPI_GENERIC runs the epilogue p.staged selects with run-time tests of the chain's parts; any other signature is a staged
// launch with exactly those parts (epilogue_staged).
template <int ACT, int BN, int SIG>
__global__ void __launch_bounds__(TM_THREADS, 1) conv_tma_kernel(const __grid_constant__ TmaParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int S = p.stages;
  constexpr uint32_t a_bytes = TC_BM * 128, b_bytes = (uint32_t)BN * 128;
  constexpr uint32_t stage_bytes = 2 * a_bytes + 2 * b_bytes;
  uint8_t* epi_smem = smem + (size_t)S * stage_bytes;                             // staged epilogue: chunks, row tables
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.bar_off);                  // full[S], empty[S]
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar_base = smem_u32(bars);
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (S + s); };

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);      // warp-uniform to the compiler: wgmma stays unserialized
  const int nkb = p.nkb;
  const int bw = 1 << p.bw_log2, bh = TC_BM >> p.bw_log2;
  const int mt = p.N * p.tiles_y * p.tiles_x, nt = p.npad / BN;
  const int total_tiles = mt * nt;

  if (tid == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), TM_WG_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // tile t -> (image, patch origin, N tile); N fastest so CTAs running together share the activation boxes in L2
  auto decode = [&](int t, int& nimg, int& oy0, int& ox0, int& n0) {
    const int mtile = t / nt; n0 = (t - mtile * nt) * BN;
    const int per_img = p.tiles_y * p.tiles_x;
    nimg = mtile / per_img; const int r = mtile - nimg * per_img;
    const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
    oy0 = ty * bh; ox0 = tx * bw;
  };
  // output sparsity: every role walks the same tile sequence and skips the same tiles
  auto needed = [&](int t) -> bool { return !p.tile_need || p.tile_need[t / nt] != 0; };

  if (warp < 2 * TM_WG_WARPS) {
    // =========================== consumers: ping-pong over whole tiles ===========================
    // Warpgroup wg takes the processed tiles j with j % 2 == wg and runs main loop and epilogue of the full 128 x BN tile.  Two
    // named barriers hand the tensor core from one warpgroup to the other once a main loop has issued its last K block, so the
    // epilogue of one tile runs while the other warpgroup's main loop keeps the tensor core busy.
    setmaxnreg_inc<TM_CONSUMER_REGS>();
    const int wg = warp >> 2;
    const int HoWo = p.Ho * p.Wo;
    const int row = (warp & 3) * 16 + (lane >> 2);
    int s = 0; uint32_t ph = 0;
    int j = 0;                                           // tiles processed by this CTA so far, both warpgroups
    if (wg == 1) named_bar_arrive(1, 2 * TM_WG_WARPS * 32);   // warpgroup 0 takes the first turn
#ifdef MITB_CONV_PHASES
    long long c0 = 0, c1 = 0, c2 = 0, c3 = 0, c4 = 0, sum[4] = {0, 0, 0, 0}, ntl = 0, ep[3] = {0, 0, 0};
#else
    long long* ep = nullptr;
#endif
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      if (!needed(t)) continue;
      if ((j++ & 1) != wg) {                             // the other warpgroup's tile: skip its stages of the ring
        const int q = s + nkb;
        ph ^= (uint32_t)((q / S) & 1);
        s = q % S;
        continue;
      }
      int nimg_t, oy0, ox0, n0;
      decode(t, nimg_t, oy0, ox0, n0);
      float acc0[BN / 2], acc1[BN / 2];                  // rows 0-63 and 64-127 of the tile
      int prev = -1;
      named_bar_sync(1 + wg, 2 * TM_WG_WARPS * 32);       // this warpgroup's turn on the tensor core
      PHASE_CLOCK(c0);
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(full_bar(s), ph);
#ifdef MITB_CONV_PHASES
        if (kb == 0) c1 = clock64();
#endif
        const uint32_t a_hi = smem_base + (uint32_t)s * stage_bytes, a_mid = a_hi + a_bytes;
        const uint32_t b_hi = a_mid + a_bytes, b_mid = b_hi + b_bytes;
        const uint64_t dbh = make_desc_sw128(b_hi), dbm = make_desc_sw128(b_mid);
        fence_acc(acc0);
        fence_acc(acc1);
        wgmma_fence();
        wgmma_kblock_x3<BN>(acc0, make_desc_sw128(a_hi), make_desc_sw128(a_mid), dbh, dbm, kb == 0);
        wgmma_kblock_x3<BN>(acc1, make_desc_sw128(a_hi + 64u * 128u), make_desc_sw128(a_mid + 64u * 128u), dbh, dbm, kb == 0);
        wgmma_commit();
        wgmma_wait<1>();                                 // the previous K block's wgmma retired -> its stage is free
        fence_acc(acc0);
        fence_acc(acc1);
        if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
        prev = s;
        if (++s == S) { s = 0; ph ^= 1u; }
      }
      named_bar_arrive(1 + (wg ^ 1), 2 * TM_WG_WARPS * 32);   // the other warpgroup's turn
      PHASE_CLOCK(c2);
      wgmma_wait<0>();
      fence_acc(acc0);
      fence_acc(acc1);
      PHASE_CLOCK(c3);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(prev));
      auto rowpix = [&](int r, int& nimg, int& oy, int& ox) -> bool {
        if (p.lin) {
          const int m = ox0 + r;
          if (m >= p.M || nimg_t >= p.N) return false;
          nimg = m / HoWo; const int pp = m - nimg * HoWo;
          oy = pp / p.Wo; ox = pp - oy * p.Wo;
          return true;
        }
        nimg = nimg_t; oy = oy0 + (r >> p.bw_log2); ox = ox0 + (r & (bw - 1));
        return oy < p.Ho && ox < p.Wo && nimg < p.N;
      };
      if (SIG != EPI_GENERIC || p.staged) {
        auto rowm = [&](int r) -> int {
          return p.lin ? ox0 + r : (nimg_t * p.Ho + oy0 + (r >> p.bw_log2)) * p.Wo + ox0 + (r & (bw - 1));
        };
        float* chunk = reinterpret_cast<float*>(epi_smem + wg * EPI_CHUNK_BYTES);
        int* rtab = reinterpret_cast<int*>(epi_smem + 2 * EPI_CHUNK_BYTES) + wg * TC_BM;
        if (p.e.vec4) epilogue_staged<ACT, BN, 4, SIG>(p.e, acc0, acc1, row, n0, chunk, rtab, 3 + wg, rowpix, rowm, ep);
        else epilogue_staged<ACT, BN, 2, SIG>(p.e, acc0, acc1, row, n0, chunk, rtab, 3 + wg, rowpix, rowm, ep);
      } else if constexpr (SIG == EPI_GENERIC) {
        epilogue_tile<ACT, BN>(p.e, acc0, row, n0, 0, rowpix);
        epilogue_tile<ACT, BN>(p.e, acc1, 64 + row, n0, 0, rowpix);
      }
#ifdef MITB_CONV_PHASES
      c4 = clock64();
      sum[0] += c1 - c0; sum[1] += c2 - c1; sum[2] += c3 - c2; sum[3] += c4 - c3; ++ntl;
#endif
    }
    // the turn opened after the last tile is taken by the warpgroup it was opened for, so both barriers end balanced
    if ((j & 1) == wg) named_bar_sync(1 + wg, 2 * TM_WG_WARPS * 32);
#ifdef MITB_CONV_PHASES
    if ((tid & 127) == 0) {
      for (int i = 0; i < 4; ++i) atomicAdd(&g_conv_phases[i], (unsigned long long)sum[i]);
      atomicAdd(&g_conv_phases[4], (unsigned long long)ntl);
    }
    for (int i = 0; i < 3; ++i) atomicAdd(&g_conv_phases[5 + i], (unsigned long long)ep[i]);
#endif
  } else {
    // =========================== producer warpgroup: its first warp issues four TMA boxes per K block =============
    setmaxnreg_dec<TM_PRODUCER_REGS>();
    if (warp != 2 * TM_WG_WARPS) return;
    int s = 0; uint32_t ph = 1;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      if (!needed(t)) continue;
      int nimg, oy0, ox0, n0;
      decode(t, nimg, oy0, ox0, n0);
      int kb = 0;
      for (int sg = 0; sg < p.nseg; ++sg) {
        const SegParams& sp = p.seg[sg];
        int tap = 0, cb = 0;
        const int nk = sp.ntaps * sp.cblks;
        for (int i = 0; i < nk; ++i, ++kb) {
          mbar_wait(empty_bar(s), ph);
          const uint32_t a_hi = smem_base + (uint32_t)s * stage_bytes, a_mid = a_hi + a_bytes;
          const uint32_t b_hi = a_mid + a_bytes, b_mid = b_hi + b_bytes;
          const int x = ox0 * p.sx + sp.tdx[tap], y = oy0 * p.sy + sp.tdy[tap];
          tma_kblock(full_bar(s), stage_bytes, a_hi, a_mid, b_hi, b_mid, &sp.ta_hi, &sp.ta_mid, &p.tb_hi, &p.tb_mid,
                     sp.c0 + cb * TC_BK, x, y, nimg, kb * TC_BK, n0);
          if (++cb == sp.cblks) { cb = 0; ++tap; }
          if (++s == S) { s = 0; ph ^= 1u; }
        }
      }
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// fp32 view -> bf16 hi / mid split tensor (one thread = 8 channels of one padded pixel), channels [coff, coff + C) of `sv`.
// Halo rows/cols (pt/pl) are filled by reflection (PAD_REFLECT); zero padding needs no halo (TMA out-of-bounds fill).
// The BN+ReLU prologue of the pre-activation ResNet is applied here, once per element.
struct SplitParams {
  const float* in; int N, H, W, C, cs, coff, planar;
  int Hp, Wp, pt, pl;
  const float* in_scale; const float* in_shift; int in_relu;
  uint16_t* hi; uint16_t* mid; int o_pitch, o_coff;
};

__global__ void __launch_bounds__(256) split_pad_kernel(const SplitParams q) {
  const int c8n = q.C >> 3;
  const long npix = (long)q.N * q.Hp * q.Wp;
  const long total = npix * c8n;
  const size_t HW = (size_t)q.H * q.W;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    long pix; int c8;
    if (q.planar) { c8 = (int)(i / npix); pix = i - (long)c8 * npix; }      // pixel fastest: plane reads coalesced
    else { pix = i / c8n; c8 = (int)(i - pix * c8n); }                        // channel fastest: NHWC reads coalesced
    const int x = (int)(pix % q.Wp); const long r = pix / q.Wp;
    const int y = (int)(r % q.Hp), n = (int)(r / q.Hp);
    const int sy = reflect_idx(y - q.pt, q.H), sx = reflect_idx(x - q.pl, q.W);
    const int c0 = c8 * 8;
    float v[8];
    if (q.planar) {
      const float* src = q.in + ((size_t)n * q.cs + q.coff + c0) * HW + (size_t)sy * q.W + sx;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = __ldg(src + (size_t)e * HW);
    } else {
      const float* src = q.in + ((size_t)(n * q.H + sy) * q.W + sx) * q.cs + q.coff + c0;
      const float4 a = __ldg(reinterpret_cast<const float4*>(src)), b = __ldg(reinterpret_cast<const float4*>(src) + 1);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    }
    if (q.in_scale) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float t = v[e] * __ldg(q.in_scale + c0 + e) + __ldg(q.in_shift + c0 + e);
        v[e] = q.in_relu ? fmaxf(t, 0.f) : t;
      }
    }
    uint4 hi, mid;
    split8(v, hi, mid);
    const size_t o = (size_t)pix * q.o_pitch + q.o_coff + c0;
    *reinterpret_cast<uint4*>(q.hi + o) = hi;
    *reinterpret_cast<uint4*>(q.mid + o) = mid;
  }
}

// Reflect halo of channels [coff, coff + C) of a split tensor, copied from its interior (one thread = 8 channels of one halo pixel).
__global__ void __launch_bounds__(256) split_halo_kernel(uint16_t* hi, uint16_t* mid, int N, int H, int W, int Hp, int Wp, int pt, int pl,
                                                         int pitch, int coff, int C) {
  const int c8n = C >> 3;
  const long rows_h = (long)(Hp - H) * Wp;                 // full-width halo rows (top + bottom)
  const long per_img = rows_h + (long)H * (Wp - W);        // + left/right columns of the interior rows
  const long total = (long)N * per_img * c8n;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % c8n); const long hp = i / c8n;
    const int n = (int)(hp / per_img); const long j = hp - (long)n * per_img;
    int y, x;
    if (j < rows_h) { const int r = (int)(j / Wp); x = (int)(j - (long)r * Wp); y = r < pt ? r : r + H; }
    else { const long k = j - rows_h; const int r = (int)(k / (Wp - W)); const int xx = (int)(k - (long)r * (Wp - W)); y = pt + r; x = xx < pl ? xx : xx + W; }
    const int sy = reflect_idx(y - pt, H) + pt, sx = reflect_idx(x - pl, W) + pl;
    const size_t so = ((size_t)(n * Hp + sy) * Wp + sx) * pitch + coff + c8 * 8;
    const size_t dst_o = ((size_t)(n * Hp + y) * Wp + x) * pitch + coff + c8 * 8;
    *reinterpret_cast<uint4*>(hi + dst_o) = *reinterpret_cast<const uint4*>(hi + so);
    *reinterpret_cast<uint4*>(mid + dst_o) = *reinterpret_cast<const uint4*>(mid + so);
  }
}

// Cin = 4 stem: fp32 NHWC (4 channels) -> bf16 hi / mid [N][Hp][Wp][8] (channels 4..7 zero), halo materialised for BOTH padding modes
// (reflect, or zeros): the stem's tensor map reads 8-pixel windows that straddle the image border, so out-of-bounds fill cannot help.
__global__ void __launch_bounds__(256) split_stem8_kernel(const float* in, int N, int H, int W, int cs, int coff, int Hp, int Wp, int pt, int pl,
                                                          int reflect, uint16_t* hi, uint16_t* mid) {
  const long npix = (long)N * Hp * Wp;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < npix; i += (long)gridDim.x * blockDim.x) {
    const int x = (int)(i % Wp); const long r = i / Wp;
    const int y = (int)(r % Hp), n = (int)(r / Hp);
    int sy = y - pt, sx = x - pl;
    bool ok = true;
    if (reflect) { sy = reflect_idx(sy, H); sx = reflect_idx(sx, W); ok = sx >= 0 && sx < W && sy >= 0 && sy < H; }
    else ok = sy >= 0 && sy < H && sx >= 0 && sx < W;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ok) v = __ldg(reinterpret_cast<const float4*>(in + ((size_t)(n * H + sy) * W + sx) * cs + coff));
    uint2 h, m;
    split4(v, h, m);
    *reinterpret_cast<uint4*>(hi + (size_t)i * 8) = make_uint4(h.x, h.y, 0u, 0u);
    *reinterpret_cast<uint4*>(mid + (size_t)i * 8) = make_uint4(m.x, m.y, 0u, 0u);
  }
}

// ConvOp::need_px (uint8 over the logical output grid) -> one flag per 128-row M tile, same tile geometry as the conv kernel
__global__ void __launch_bounds__(128) tile_need_kernel(const uint8_t* need_px, int N, int Ho, int Wo, int M, int lin, int bw_log2, int tiles_x,
                                                        int tiles_y, uint8_t* tile_need) {
  const int mtile = blockIdx.x, r = threadIdx.x;
  int v = 0;
  if (lin) {
    const int m = mtile * 128 + r;
    if (m < M) v = need_px[m];
  } else {
    const int per_img = tiles_y * tiles_x;
    const int nimg = mtile / per_img, rr = mtile - nimg * per_img;
    const int ty = rr / tiles_x, tx = rr - ty * tiles_x;
    const int bw = 1 << bw_log2, bh = 128 >> bw_log2;
    const int oy = ty * bh + (r >> bw_log2), ox = tx * bw + (r & (bw - 1));
    if (nimg < N && oy < Ho && ox < Wo) v = need_px[((size_t)nimg * Ho + oy) * Wo + ox];
  }
  const int any = __syncthreads_or(v);
  if (r == 0) tile_need[mtile] = (uint8_t)(any != 0);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr; cudaDriverEntryPointQueryResult q;
    CUDA_OK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    MITB_CHECK(p && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available in this driver");
    fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 4-D activation map over a dense bf16 tensor [N][Hp][Wp][C]: box = {64 ch, bw, bh, 1} pixels taken every (sx, sy)-th element,
// 128-byte swizzle, zero out-of-bounds fill (= zero padding of the convolution, and zero for channels >= C)
void make_act_tmap(CUtensorMap* m, const uint16_t* base, int N, int Hp, int Wp, int C, int bw, int bh, int sx, int sy) {
  const cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)Wp, (cuuint64_t)Hp, (cuuint64_t)N};
  const cuuint64_t gstride[3] = {(cuuint64_t)C * 2, (cuuint64_t)Wp * C * 2, (cuuint64_t)Hp * Wp * C * 2};
  const cuuint32_t box[4] = {(cuuint32_t)TC_BK, (cuuint32_t)(bw * sx), (cuuint32_t)(bh * sy), 1};
  const cuuint32_t estr[4] = {1, (cuuint32_t)sx, (cuuint32_t)sy, 1};
  const CUresult r = encode_fn()(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)base, gdim, gstride, box, estr,
                                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  MITB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d) for activations [%d,%d,%d,%d] box %dx%d stride %dx%d", (int)r, N, Hp, Wp, C,
             bw, bh, sx, sy);
}

// Stem map over the 8-channel-padded tensor [N][Hp][Wp][8]: dimension 0 = 64 consecutive elements = an 8-pixel x 8-channel window,
// dimension 1 = the window's first pixel with a stride of ONE pixel (16 bytes) - consecutive windows overlap by 7 pixels, which a
// tensor map is free to describe (addresses are just sum(coord * stride)).  One box row = one output pixel's kernel row.
// Stride-2 stems take every second window and row through element strides of 2 on dimensions 1 and 2 (box 2bw x 2bh, as
// make_act_tmap does for strided convs); the smem tile is the same bw x bh windows.
bool make_stem_tmap(CUtensorMap* m, const uint16_t* base, int N, int Hp, int Wp, int bw, int bh, int s) {
  const cuuint64_t gdim[4] = {64, (cuuint64_t)(Wp - 7), (cuuint64_t)Hp, (cuuint64_t)N};
  const cuuint64_t gstride[3] = {16, (cuuint64_t)Wp * 16, (cuuint64_t)Hp * Wp * 16};
  const cuuint32_t box[4] = {64, (cuuint32_t)(bw * s), (cuuint32_t)(bh * s), 1};
  const cuuint32_t estr[4] = {1, (cuuint32_t)s, (cuuint32_t)s, 1};
  return encode_fn()(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)base, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// N tile width: minimise waves x tile time.  Main loop = K blocks x max(tensor floor, operand bytes over the SM's share of L2
// bandwidth); candidates split Cout into j equal tiles rounded up to 32 (the wgmma widths instantiated, at most 128).  Tensor
// floor: 3 x 128 x bn x 64 bf16 MACs per K block at the H100 SXM data-sheet dense bf16 rate (~2048 MAC per clock per SM) =
// 12 bn cycles (measured with tools/conv_phases.py: 1490-1660 clk per K block at bn = 128 on L2-resident layers).  The two
// consumer warpgroups alternate whole tiles and one warpgroup's epilogue overlaps the other's main loop, so a CTA finishes two
// tiles per max(2 main, main + epilogue): tile time = max(main, (main + epilogue) / 2) + a fixed cost (mode 1; mode 0 is the
// sum, for a schedule without overlap).  The epilogue cycles per column are measured (tools/conv_phases.py): epi_reg for the
// register epilogue, epi / epi_gelu for the staged one; the L2 share (42 B/clk) is an estimate.  MITB_CM="mode,epi_gelu,epi,fix,
// epi_reg" overrides the constants (tools/cost_model_sweep.py).
struct CostModel { int mode; double epi_gelu, epi, fix, epi_reg; };
const CostModel& cost_model() {
  static CostModel cm = {1, 225.0, 350.0, 600.0, 450.0};
  static bool init = false;
  if (!init) {
    init = true;
    if (const char* e = getenv("MITB_CM")) {
      int mode = 0; double a = 0, b = 0, c = 0, d = 0;
      if (sscanf(e, "%d,%lf,%lf,%lf,%lf", &mode, &a, &b, &c, &d) == 5) cm = {mode, a, b, c, d};
    }
  }
  return cm;
}

double tile_main_loop(int nkb, int bn) {
  const double mma = 12.0 * bn, l2 = (32768.0 + 256.0 * bn) / 42.0;
  return nkb * (mma > l2 ? mma : l2);
}
// Staged epilogue (epilogue_staged) only where the register epilogue would not hide behind the other warpgroup's main loop: its
// chunks take 33 KB of shared memory, a pipeline stage at BN = 32 and 96, which a long main loop feels and a hidden epilogue does
// not repay.  The 10 % margin: at the crossover the staged epilogue measured slower (49152 x 2304 x 384, BN 128: main loop 56 k,
// register epilogue 58 k clocks by the model; 5-9 % slower staged).
bool stage_epilogue(bool vec2, int nkb, int bn) { return vec2 && tile_main_loop(nkb, bn) < 0.9 * cost_model().epi_reg * bn; }

int choose_bn(int Cout, long mtiles, int nkb, int sms, bool gelu, bool vec2) {
  const CostModel& cm = cost_model();
  double best = 1e30; int best_bn = 32;
  for (int j = 1; j <= 16; ++j) {
    int bn = ((Cout + j - 1) / j + 31) & ~31;
    if (bn > 128) continue;
    const long nt = (Cout + bn - 1) / bn;
    const long waves = (mtiles * nt + sms - 1) / sms;
    const double main_loop = tile_main_loop(nkb, bn);
    const double epi = (stage_epilogue(vec2, nkb, bn) ? (gelu ? cm.epi_gelu : cm.epi) : cm.epi_reg) * bn;
    const double overlap = (main_loop + epi) / 2;
    const double tile = (cm.mode == 1 ? (main_loop > overlap ? main_loop : overlap) : main_loop + epi) + cm.fix;
    const double cost = waves * tile;
    if (cost < best * 0.999) { best = cost; best_bn = bn; }
  }
  return best_bn;
}

bool g_tma_enabled = true;

// The (activation, epilogue signature) pairs with a conv_tma_kernel of their own: every pair the staged launches of one bench page
// have (tools/conv_phases.py lists them) - ConvNeXt fc1 (shift, GELU, split) and fc2 (shift, mul1, add1, out), the FFC's spectral
// and global convs (scale, shift, ReLU, split / + residual and out), the OCR's residual layers (add1, out, split with the next
// layer's BN + ReLU) and the plain detector / inpainter / OCR convs.  Any other staged launch runs the generic signature.
#define MITB_EPI_SIGS(X)                                                                \
  X(ACT_GELU, EPI_SHIFT | EPI_OS)                                                      \
  X(ACT_GELU, EPI_SHIFT | EPI_OUT)                                                     \
  X(ACT_NONE, EPI_SHIFT | EPI_MUL1 | EPI_ADD1 | EPI_OUT)                               \
  X(ACT_NONE, EPI_ADD1 | EPI_OUT | EPI_OS | EPI_OS_AFFINE | EPI_OS_RELU)               \
  X(ACT_NONE, EPI_SHIFT | EPI_ADD1 | EPI_OUT)                                          \
  X(ACT_NONE, EPI_SHIFT | EPI_OUT)                                                     \
  X(ACT_NONE, EPI_OUT)                                                                 \
  X(ACT_RELU, EPI_SCALE | EPI_SHIFT | EPI_OUT)                                         \
  X(ACT_RELU, EPI_SCALE | EPI_SHIFT | EPI_OS)                                          \
  X(ACT_RELU, EPI_SCALE | EPI_SHIFT | EPI_ADD1 | EPI_OUT | EPI_OS)                     \
  X(ACT_SILU, EPI_SHIFT | EPI_OUT)

template <int A, int SIG> void tma_kernel_attrs() {
  CUDA_OK(cudaFuncSetAttribute(conv_tma_kernel<A, 32, SIG>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  CUDA_OK(cudaFuncSetAttribute(conv_tma_kernel<A, 64, SIG>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  CUDA_OK(cudaFuncSetAttribute(conv_tma_kernel<A, 96, SIG>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  CUDA_OK(cudaFuncSetAttribute(conv_tma_kernel<A, 128, SIG>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
}
template <int A, int SIG> void tma_kernel_launch(int BN, int grid, size_t smem, cudaStream_t st, const TmaParams& p) {
  switch (BN) {
    case 32: conv_tma_kernel<A, 32, SIG><<<grid, TM_THREADS, smem, st>>>(p); break;
    case 64: conv_tma_kernel<A, 64, SIG><<<grid, TM_THREADS, smem, st>>>(p); break;
    case 96: conv_tma_kernel<A, 96, SIG><<<grid, TM_THREADS, smem, st>>>(p); break;
    default: conv_tma_kernel<A, 128, SIG><<<grid, TM_THREADS, smem, st>>>(p); break;
  }
}

// halo a conv needs around its input for reflect padding (zero padding: none)
void conv_halo(const int8_t* tdy, const int8_t* tdx, int ntaps, int pad, int H, int W, int Ho, int Wo, int sy, int sx, int& pt, int& pb,
               int& pl, int& pr) {
  pt = pb = pl = pr = 0;
  if (pad != PAD_REFLECT) return;
  int tmin_dy = 127, tmax_dy = -127, tmin_dx = 127, tmax_dx = -127;
  for (int t = 0; t < ntaps; ++t) {
    tmin_dy = tdy[t] < tmin_dy ? tdy[t] : tmin_dy; tmax_dy = tdy[t] > tmax_dy ? tdy[t] : tmax_dy;
    tmin_dx = tdx[t] < tmin_dx ? tdx[t] : tmin_dx; tmax_dx = tdx[t] > tmax_dx ? tdx[t] : tmax_dx;
  }
  pt = tmin_dy < 0 ? -tmin_dy : 0; pl = tmin_dx < 0 ? -tmin_dx : 0;
  pb = (Ho - 1) * sy + tmax_dy - (H - 1); if (pb < 0) pb = 0;
  pr = (Wo - 1) * sx + tmax_dx - (W - 1); if (pr < 0) pr = 0;
}

}  // namespace

int g_epi_specialise = -1;                 // -1: unset, MITB_EPI_GENERIC=1 forces the generic signature

// signature a staged launch with activation instantiation `act` and the chain's parts `sig` runs with
bool epi_specialise() {
  if (g_epi_specialise < 0) { const char* ev = getenv("MITB_EPI_GENERIC"); g_epi_specialise = (ev && atoi(ev)) ? 0 : 1; }
  return g_epi_specialise != 0;
}

int staged_epi_sig(int act, int sig) {
  if (!epi_specialise()) return EPI_GENERIC;
#define MITB_EPI_MATCH(A, S) if (act == (A) && sig == (S)) return S;
  MITB_EPI_SIGS(MITB_EPI_MATCH)
#undef MITB_EPI_MATCH
  return EPI_GENERIC;
}

int epi_sig_list(int* act, int* sig, int cap) {
  int n = 0;
#define MITB_EPI_LIST(A, S) { if (n < cap) { act[n] = A; sig[n] = S; } ++n; }
  MITB_EPI_SIGS(MITB_EPI_LIST)
#undef MITB_EPI_LIST
  return n;
}

void make_w_tmap(CUtensorMap* m, const uint16_t* base, int kdim, int rows, int bn) {
  const cuuint64_t gdim[2] = {(cuuint64_t)kdim, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)kdim * 2};
  const cuuint32_t box[2] = {(cuuint32_t)TC_BK, (cuuint32_t)bn};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = encode_fn()(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)base, gdim, gstride, box, estr,
                                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  MITB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d) for weights [%d x %d] box %d", (int)r, rows, kdim, bn);
}

void conv_tma_set_enabled(bool on) { g_tma_enabled = on; }
bool conv_tma_enabled() { return g_tma_enabled; }
bool conv_tma_bn_candidate(int Cout, int bn) {
  for (int j = 1; j <= 16; ++j)
    if ((((Cout + j - 1) / j + 31) & ~31) == bn && bn <= 128) return true;
  return false;
}

void launch_split(const View& in, const SplitView& sv, int coff, const float* in_scale, const float* in_shift, int in_relu, cudaStream_t st) {
  MITB_CHECK(sv.valid() && sv.N == in.N && sv.H == in.H && sv.W == in.W && coff + in.C <= sv.C, "split: shape mismatch");
  MITB_CHECK(in.C % 8 == 0 && sv.C % 8 == 0 && coff % 8 == 0, "split: channel counts/offsets must be multiples of 8");
  MITB_CHECK(in.planar || (in.cs % 4 == 0 && in.coff % 4 == 0), "split: unaligned NHWC view");
  SplitParams q;
  q.in = in.p; q.N = in.N; q.H = in.H; q.W = in.W; q.C = in.C; q.cs = in.cs; q.coff = in.coff; q.planar = in.planar;
  q.Hp = sv.Hp; q.Wp = sv.Wp; q.pt = sv.pt; q.pl = sv.pl;
  q.in_scale = in_scale; q.in_shift = in_shift; q.in_relu = in_relu;
  q.hi = sv.hi; q.mid = sv.mid; q.o_pitch = sv.C; q.o_coff = coff;
  const long total = (long)sv.N * sv.Hp * sv.Wp * (in.C / 8);
  long blocks = (total + 255) / 256; if (blocks > device_sm_count() * 32L) blocks = device_sm_count() * 32L;
  if (blocks < 1) return;
  split_pad_kernel<<<(int)blocks, 256, 0, st>>>(q);
  count_launch();
  CUDA_OK(cudaGetLastError());
}

void launch_split_halo(const SplitView& sv, int coff, int C, cudaStream_t st) {
  if (sv.Hp == sv.H && sv.Wp == sv.W) return;
  MITB_CHECK(sv.valid() && C % 8 == 0 && coff % 8 == 0 && sv.C % 8 == 0 && coff + C <= sv.C, "split halo: bad channel slice");
  MITB_CHECK(sv.pt < sv.H && sv.pl < sv.W && sv.Hp - sv.H - sv.pt < sv.H && sv.Wp - sv.W - sv.pl < sv.W, "split halo wider than the image");
  const long total = (long)sv.N * ((long)(sv.Hp - sv.H) * sv.Wp + (long)sv.H * (sv.Wp - sv.W)) * (C / 8);
  long blocks = (total + 255) / 256; if (blocks > device_sm_count() * 8L) blocks = device_sm_count() * 8L;
  ProfScope ps("split_halo", 0.0, 4.0 * total * 8, st);
  split_halo_kernel<<<(int)blocks, 256, 0, st>>>(sv.hi, sv.mid, sv.N, sv.H, sv.W, sv.Hp, sv.Wp, sv.pt, sv.pl, sv.C, coff, C);
  count_launch();
  CUDA_OK(cudaGetLastError());
}

bool conv_tma_supported(const ConvOp& op) {
  static int env = -1;
  if (env < 0) { const char* e = getenv("MITB_NO_TMA_CONV"); env = (e && atoi(e)) ? 0 : 1; }
  if (!g_tma_enabled || !env || !op.wt.wh || !op.wt.wm) return false;
  if (op.sy < 1 || op.sy > 2 || op.sx < 1 || op.sx > 2) return false;
  const int C = op.in.C;
  if (C % 64 == 0) { if (!op.seg2.sv.valid() && op.wt.tc_kpad != op.wt.ntaps * C) return false; }   // main copy is already in (tap, 64-channel block) order
  else if (!(op.wt.whp && op.wt.wmp && op.wt.tc_cp >= C)) return false;             // needs the per-tap padded copy (Cin % 8 == 0, >= 16)
  if (!op.in_sv.valid()) {
    if (!op.in.planar && (op.in.cs % 4 != 0 || op.in.coff % 4 != 0)) return false;
    if (op.in.planar && op.wt.ntaps != 1) return false;
  }
  const long M = (long)op.in.N * op.Ho * op.Wo;
  if (M < 128) return false;
  return true;
}

static bool g_stem_map_failed = false;       // the driver refused the overlapping-stride map once: keep the gather kernel for stems

bool conv_stem8_supported(const ConvOp& op) {
  static int env = -1;
  if (env < 0) { const char* e = getenv("MITB_NO_STEM8"); env = (e && atoi(e)) ? 0 : 1; }
  if (!g_tma_enabled || !env || g_stem_map_failed || !op.wt.w8h || !op.wt.w8m) return false;
  // strides 1 and 2 only (the ConvNeXt 4x4 s4 stem keeps the gather kernel)
  if (op.in.C != 4 || op.in.planar || op.sx != op.sy || (op.sx != 1 && op.sx != 2) || op.wt.ntaps != op.wt.w8_kh * op.wt.w8_kw) return false;
  if ((op.in.cs | op.in.coff) & 3) return false;
  if (op.in_sv.valid() || op.seg2.sv.valid() || op.stat_max || op.out.C <= 4) return false;
  if (op.pad == PAD_REFLECT && (-op.wt.tdy[0] >= op.in.H || -op.wt.tdx[0] >= op.in.W)) return false;
  return (long)op.in.N * op.Ho * op.Wo >= 128;
}

void launch_conv_tma(const ConvOp& op, bool stem, cudaStream_t st) {
  const int C = op.in.C, N = op.in.N, H = op.in.H, W = op.in.W;
  const bool padded_w = !stem && C % 64 != 0;
  const int cblks = stem ? 1 : (C + TC_BK - 1) / TC_BK;              // K blocks per tap; channels >= C arrive as zeros (TMA bounds)
  int pt, pb, pl, pr;
  conv_halo(op.wt.tdy, op.wt.tdx, op.wt.ntaps, stem ? PAD_REFLECT : op.pad, H, W, op.Ho, op.Wo, op.sy, op.sx, pt, pb, pl, pr);
  if (stem) pr += 8 - op.wt.w8_kw;                                       // every window is 8 pixels wide (the extra taps have zero weights)
  SplitView sv; int sv_coff = 0;
  int dev = 0; CUDA_OK(cudaGetDevice(&dev));
  // the split cache below: remembers which tensor the per-device scratch currently holds
  struct SplitKey {
    const float* in; int N, H, W, C, cs, coff, planar, Hp, Wp, pt, pl, relu; const float* sc; const float* sh; cudaStream_t st; int dev;
    bool same(const SplitKey& o) const {
      return in == o.in && N == o.N && H == o.H && W == o.W && C == o.C && cs == o.cs && coff == o.coff && planar == o.planar &&
             Hp == o.Hp && Wp == o.Wp && pt == o.pt && pl == o.pl && relu == o.relu && sc == o.sc && sh == o.sh && st == o.st && dev == o.dev;
    }
  };
  static SplitKey g_key; static bool g_key_valid = false; static unsigned long g_key_epoch = 0; static const uint16_t* g_key_hi = nullptr;
  bool remember = false, reused = false;
  if (op.in_sv.valid()) {
    // ---- the producer already wrote this conv's bf16 hi / mid operands (ConvOp::out_sv of an earlier op, or launch_split)
    sv = op.in_sv; sv_coff = op.in_sv_coff;
    MITB_CHECK(sv.N == N && sv.H == H && sv.W == W && sv_coff + C <= sv.C && sv.C % 8 == 0 && sv_coff % 8 == 0, "tma conv: in_sv shape mismatch");
    MITB_CHECK(sv.pt >= pt && sv.pl >= pl && sv.Hp - sv.H - sv.pt >= pb && sv.Wp - sv.W - sv.pl >= pr, "tma conv: in_sv halo too small");
    if (op.pad != PAD_REFLECT && (sv.Hp != sv.H || sv.Wp != sv.W)) {      // zero padding over a halo'd tensor: only if no tap leaves the image
      int zt, zb, zl, zr;
      conv_halo(op.wt.tdy, op.wt.tdx, op.wt.ntaps, PAD_REFLECT, H, W, op.Ho, op.Wo, op.sy, op.sx, zt, zb, zl, zr);
      MITB_CHECK(zt == 0 && zb == 0 && zl == 0 && zr == 0, "tma conv: zero padding needs a halo-free in_sv");
    }
    MITB_CHECK(!op.in_scale, "tma conv: in_sv carries its prologue already");
    MITB_CHECK(!padded_w || sv_coff + C == sv.C, "tma conv: Cin %% 64 != 0 needs the slice to end at the tensor's last channel");
  } else if (stem) {
    sv.N = N; sv.H = H; sv.W = W; sv.C = 8; sv.pt = pt; sv.pl = pl; sv.Hp = H + pt + pb; sv.Wp = W + pl + pr;
    static DeviceScratch g_stem;
    sv.hi = static_cast<uint16_t*>(g_stem.get(2 * sv.elems() * sizeof(uint16_t))); sv.mid = sv.hi + sv.elems();
    const long npix = (long)N * sv.Hp * sv.Wp;
    long blocks = (npix + 255) / 256; if (blocks > device_sm_count() * 32L) blocks = device_sm_count() * 32L;
    split_stem8_kernel<<<(int)blocks, 256, 0, st>>>(op.in.p, N, H, W, op.in.cs, op.in.coff, sv.Hp, sv.Wp, pt, pl, op.pad == PAD_REFLECT ? 1 : 0,
                                                    sv.hi, sv.mid);
    count_launch();
    MITB_CHECK(!op.in_scale, "stem conv: no input prologue");
  } else {
    // ---- split pass into the per-device scratch, skipped when the previous kernel launched by this library was a TMA conv
    // over exactly the same input (the four sub-pixel phases of a transposed conv, sibling convs of one tensor).
    // Safe by construction: ANY other launch in between bumps g_launch_epoch, and a conv whose output overlaps the cached
    // input invalidates the entry.
    MITB_CHECK(C % 8 == 0, "tma conv: Cin must be a multiple of 8");
    sv.N = N; sv.H = H; sv.W = W; sv.C = C; sv.pt = pt; sv.pl = pl; sv.Hp = H + pt + pb; sv.Wp = W + pl + pr;
    static DeviceScratch g_split;                                             // bf16 hi | mid of the current conv's input
    sv.hi = static_cast<uint16_t*>(g_split.get(2 * sv.elems() * sizeof(uint16_t))); sv.mid = sv.hi + sv.elems();
    const SplitKey key{op.in.p, N, H, W, C, op.in.cs, op.in.coff, op.in.planar, sv.Hp, sv.Wp, pt, pl, op.in_relu, op.in_scale, op.in_shift, st, dev};
    const bool reuse = g_key_valid && g_key_epoch == g_launch_epoch && g_key_hi == sv.hi && key.same(g_key);
    if (!reuse) launch_split(op.in, sv, 0, op.in_scale, op.in_shift, op.in_relu, st);
    reused = reuse;
    // remember this split unless the conv writes into the tensor it was made from
    const float* ib = op.in.p; const float* ie = ib + (size_t)op.in.N * op.in.H * op.in.W * op.in.cs;
    const float* ob = op.out.p; const float* oe = ob ? ob + (size_t)op.out.N * op.out.H * op.out.W * op.out.cs : ob;
    const bool overlap = ob && ob < ie && ib < oe;
    g_key = key; g_key_hi = sv.hi; remember = !overlap;
  }
  g_key_valid = remember;                                                    // g_key_epoch is stamped after this conv's own launch, below

  const int num_sms = device_sm_count();
  static PerDeviceOnce tma_attr;
  if (tma_attr.first()) {
    tma_kernel_attrs<ACT_NONE, EPI_GENERIC>(); tma_kernel_attrs<ACT_RELU, EPI_GENERIC>(); tma_kernel_attrs<ACT_GELU, EPI_GENERIC>();
    tma_kernel_attrs<ACT_SILU, EPI_GENERIC>(); tma_kernel_attrs<-1, EPI_GENERIC>();
#define MITB_EPI_ATTR(A, S) tma_kernel_attrs<A, S>();
    MITB_EPI_SIGS(MITB_EPI_ATTR)
#undef MITB_EPI_ATTR
  }

  TmaParams p;
  memset(&p, 0, sizeof(p));
  const bool two = op.seg2.sv.valid();
  p.nseg = two ? 2 : 1;
  p.seg[0].ntaps = stem ? op.wt.w8_kh : op.wt.ntaps; p.seg[0].cblks = cblks; p.seg[0].c0 = sv_coff;
  if (stem) for (int t = 0; t < op.wt.w8_kh; ++t) { p.seg[0].tdy[t] = (int8_t)(op.wt.tdy[t * op.wt.w8_kw] + sv.pt); p.seg[0].tdx[t] = (int8_t)(op.wt.tdx[0] + sv.pl); }
  else for (int t = 0; t < op.wt.ntaps; ++t) { p.seg[0].tdy[t] = (int8_t)(op.wt.tdy[t] + sv.pt); p.seg[0].tdx[t] = (int8_t)(op.wt.tdx[t] + sv.pl); }
  p.N = N; p.Ho = op.Ho; p.Wo = op.Wo; p.M = N * op.Ho * op.Wo; p.sy = op.sy; p.sx = op.sx;
  const bool lin = !stem && !two && op.wt.ntaps == 1 && op.Ho == H && op.Wo == W && op.sy == 1 && op.sx == 1 && op.wt.tdy[0] == 0 && op.wt.tdx[0] == 0 &&
                   sv.Hp == H && sv.Wp == W;
  p.lin = lin ? 1 : 0;                                              // 1x1: flattened [pixels][C] matrix
  int bw, bh;
  if (lin) { bw = 128; bh = 1; p.tiles_x = (p.M + 127) / 128; p.tiles_y = 1; p.N = 1; }
  else {
    long best = -1; bw = 128;
    for (int cand = 128; cand >= 8; cand >>= 1) {
      const int ch = 128 / cand;
      const long cost = (long)((op.Wo + cand - 1) / cand) * cand * (long)((op.Ho + ch - 1) / ch) * ch;
      // output-sparse launches: among equally tight tilings prefer the compact 16 x 8 patch - a 128 x 1 strip crosses several text
      // boxes per row and is almost never skippable (measured: no gain with strips)
      if (best < 0 || cost < best || (op.need_px && cost == best && cand >= 16)) { best = cost; bw = cand; }
    }
    bh = 128 / bw;
    p.tiles_x = (op.Wo + bw - 1) / bw; p.tiles_y = (op.Ho + bh - 1) / bh;
  }
  p.bw_log2 = 0; while ((1 << p.bw_log2) < bw) ++p.bw_log2;
  if (stem) {
    if (!make_stem_tmap(&p.seg[0].ta_hi, sv.hi, N, sv.Hp, sv.Wp, bw, bh, op.sx) || !make_stem_tmap(&p.seg[0].ta_mid, sv.mid, N, sv.Hp, sv.Wp, bw, bh, op.sx)) {
      g_stem_map_failed = true;                                        // fall back for good: conv_stem8_supported() is false from now on
      launch_conv(op, st);
      return;
    }
  } else if (lin) { make_act_tmap(&p.seg[0].ta_hi, sv.hi, 1, 1, N * sv.Hp * sv.Wp, sv.C, bw, bh, 1, 1); make_act_tmap(&p.seg[0].ta_mid, sv.mid, 1, 1, N * sv.Hp * sv.Wp, sv.C, bw, bh, 1, 1); }
  else { make_act_tmap(&p.seg[0].ta_hi, sv.hi, N, sv.Hp, sv.Wp, sv.C, bw, bh, op.sx, op.sy); make_act_tmap(&p.seg[0].ta_mid, sv.mid, N, sv.Hp, sv.Wp, sv.C, bw, bh, op.sx, op.sy); }
  int kdim = (stem ? op.wt.w8_kh : op.wt.ntaps) * cblks * TC_BK;
  if (two) {
    const ConvOp::Seg2& s2 = op.seg2;
    MITB_CHECK(!padded_w && s2.C % 64 == 0 && s2.ntaps >= 1 && s2.sv.N == N && s2.sv.H == op.Ho && s2.sv.W == op.Wo && op.sy == 1 && op.sx == 1 &&
               s2.coff + s2.C <= s2.sv.C && s2.sv.C % 8 == 0, "tma conv: bad second K segment");
    int qt, qb, ql, qr;
    conv_halo(s2.tdy, s2.tdx, s2.ntaps, s2.pad, s2.sv.H, s2.sv.W, op.Ho, op.Wo, 1, 1, qt, qb, ql, qr);
    MITB_CHECK(s2.sv.pt >= qt && s2.sv.pl >= ql && s2.sv.Hp - s2.sv.H - s2.sv.pt >= qb && s2.sv.Wp - s2.sv.W - s2.sv.pl >= qr, "tma conv: seg2 halo too small");
    if (s2.pad != PAD_REFLECT && (s2.sv.Hp != s2.sv.H || s2.sv.Wp != s2.sv.W)) {
      conv_halo(s2.tdy, s2.tdx, s2.ntaps, PAD_REFLECT, s2.sv.H, s2.sv.W, op.Ho, op.Wo, 1, 1, qt, qb, ql, qr);
      MITB_CHECK(qt == 0 && qb == 0 && ql == 0 && qr == 0, "tma conv: zero padding needs a halo-free seg2");
    }
    p.seg[1].ntaps = s2.ntaps; p.seg[1].cblks = s2.C / TC_BK; p.seg[1].c0 = s2.coff;
    for (int t = 0; t < s2.ntaps; ++t) { p.seg[1].tdy[t] = (int8_t)(s2.tdy[t] + s2.sv.pt); p.seg[1].tdx[t] = (int8_t)(s2.tdx[t] + s2.sv.pl); }
    make_act_tmap(&p.seg[1].ta_hi, s2.sv.hi, N, s2.sv.Hp, s2.sv.Wp, s2.sv.C, bw, bh, 1, 1);
    make_act_tmap(&p.seg[1].ta_mid, s2.sv.mid, N, s2.sv.Hp, s2.sv.Wp, s2.sv.C, bw, bh, 1, 1);
    kdim += s2.ntaps * s2.C;
    MITB_CHECK(op.wt.tc_kpad == kdim, "tma conv: merged weight has K %d, segments need %d", op.wt.tc_kpad, kdim);
  }
  p.nkb = kdim / TC_BK;
  // ---- N tile: fixed by the row-stat layout for the vocabulary head, otherwise chosen per launch against wave quantisation
  const long mtiles = (long)p.N * p.tiles_y * p.tiles_x;
  fill_epi(p.e, op);
  int BN = op.stat_max ? op.wt.tc_bn : choose_bn(op.out.C, mtiles, p.nkb, num_sms, op.act == ACT_GELU, p.e.vec2 != 0);
  if (g_conv_force_bn && !op.stat_max) {
    MITB_CHECK(conv_tma_bn_candidate(op.out.C, g_conv_force_bn), "tma conv: BN %d is not a candidate N tile for Cout %d", g_conv_force_bn, op.out.C);
    BN = g_conv_force_bn;
  }
  MITB_CHECK(BN >= 32 && BN <= 128 && BN % 32 == 0, "tma conv: bad BN %d", BN);
  p.npad = (op.out.C + BN - 1) / BN * BN;
  make_w_tmap(&p.tb_hi, stem ? op.wt.w8h : padded_w ? op.wt.whp : op.wt.wh, kdim, op.wt.tc_npad, BN);
  make_w_tmap(&p.tb_mid, stem ? op.wt.w8m : padded_w ? op.wt.wmp : op.wt.wm, kdim, op.wt.tc_npad, BN);
  if (op.out_sv.valid()) {
    const SplitView& o = op.out_sv;
    MITB_CHECK(!op.out.planar && op.out.C % 4 == 0 && !op.stat_max && op.oy_mul == 1 && op.ox_mul == 1 && op.oy_add == 0 && op.ox_add == 0 &&
               o.N == N && o.H == op.Ho && o.W == op.Wo && o.C % 4 == 0 && op.out_sv_coff % 4 == 0 && op.out_sv_coff + op.out.C <= o.C &&
               (!op.out.p || (op.out.H == op.Ho && op.out.W == op.Wo && ((op.out.cs | op.out.coff) & 3) == 0)) &&
               (!op.add0.p || (!op.add0.planar && ((op.add0.cs | op.add0.coff) & 3) == 0)) &&
               (!op.add1.p || (!op.add1.planar && ((op.add1.cs | op.add1.coff) & 3) == 0)),
               "tma conv: out_sv needs an NHWC output on the conv's own pixel grid");
    if (!op.out.p) { p.e.oH = op.Ho; p.e.oW = op.Wo; }
  } else MITB_CHECK(op.out.p || op.stat_max, "tma conv: no output");
  MITB_CHECK(!op.stat_max || op.stat_ld == 2 * (op.wt.tc_npad / op.wt.tc_bn), "tma conv: stat_ld must equal conv_stat_blocks(op)");
  if (op.need_px && !op.stat_max) {
    // reduce the pixel-level hint to this launch's tile grid (one tiny launch; the scratch is per device and stream ordered)
    static DeviceScratch g_need;
    uint8_t* tn = static_cast<uint8_t*>(g_need.get((size_t)mtiles + 16));
    tile_need_kernel<<<(unsigned)mtiles, 128, 0, st>>>(op.need_px, N, op.Ho, op.Wo, N * op.Ho * op.Wo, p.lin, p.bw_log2, p.tiles_x, p.tiles_y, tn);
    count_launch();
    p.tile_need = tn;
  }
  const size_t stage_bytes = 2 * (size_t)TC_BM * 128 + 2 * (size_t)BN * 128;
  // the staged epilogue's chunks and row tables leave 4, 4, 3, 3 stages at BN 32, 64, 96, 128 (others: 5, 4, 4, 3)
  p.staged = !op.stat_max && stage_epilogue(p.e.vec2 != 0, p.nkb, BN) ? 1 : 0;
  const size_t epi_bytes = p.staged ? EPI_SMEM_BYTES : 0;
  int stages = (int)((227 * 1024 - 1024 - 256 - epi_bytes) / stage_bytes); if (stages > 6) stages = 6;
  MITB_CHECK(stages >= 2, "tma conv: tile does not fit shared memory");
  p.stages = stages;
  p.bar_off = (int)(stages * stage_bytes + epi_bytes);
  const size_t smem = stages * stage_bytes + epi_bytes + 2 * stages * 8 + 1024;
  const long total_tiles = mtiles * (p.npad / BN);
  const int grid = (int)(total_tiles < num_sms ? total_tiles : num_sms);      // persistent: one CTA per SM
  const int act_inst = op.stat_max ? ACT_NONE : (op.act == ACT_NONE || op.act == ACT_RELU || op.act == ACT_GELU || op.act == ACT_SILU) ? op.act : -1;
  const int sig = p.staged ? staged_epi_sig(act_inst, epi_sig(p.e)) : EPI_GENERIC;
  conv_trace(stem ? CK_STEM8 : CK_TMA, BN, 1, p.e.vec2, act_inst, reused, p.staged ? (p.e.vec4 ? 4 : 2) : 0, p.staged ? sig : -1);
  bool launched = false;
#define MITB_EPI_LAUNCH(A, S) if (!launched && sig == (S) && act_inst == (A)) { tma_kernel_launch<A, S>(BN, grid, smem, st, p); launched = true; }
  MITB_EPI_SIGS(MITB_EPI_LAUNCH)
#undef MITB_EPI_LAUNCH
  if (!launched) {
    switch (act_inst) {
      case ACT_NONE: tma_kernel_launch<ACT_NONE, EPI_GENERIC>(BN, grid, smem, st, p); break;
      case ACT_RELU: tma_kernel_launch<ACT_RELU, EPI_GENERIC>(BN, grid, smem, st, p); break;
      case ACT_GELU: tma_kernel_launch<ACT_GELU, EPI_GENERIC>(BN, grid, smem, st, p); break;
      case ACT_SILU: tma_kernel_launch<ACT_SILU, EPI_GENERIC>(BN, grid, smem, st, p); break;
      default: tma_kernel_launch<-1, EPI_GENERIC>(BN, grid, smem, st, p); break;
    }
  }
  count_launch();
  g_key_epoch = g_launch_epoch;
  CUDA_OK(cudaGetLastError());
#ifdef MITB_CONV_PHASES
  {
    unsigned long long ph[N_PHASES];
    CUDA_OK(cudaStreamSynchronize(st));
    CUDA_OK(cudaMemcpyFromSymbol(ph, g_conv_phases, sizeof(ph)));
    const unsigned long long zero[N_PHASES] = {};
    CUDA_OK(cudaMemcpyToSymbol(g_conv_phases, zero, sizeof(zero)));
    const int K = op.wt.ntaps * C + (two ? op.seg2.ntaps * op.seg2.C : 0);      // the GEMM shape tools/layer_times.py reports
    fprintf(stderr, "mitb_conv_phases M %d K %d N %d BN %d nkb %d ctas %d tiles %llu first_wait %llu main %llu wgmma_wait %llu epilogue %llu"
            " epi_chunk %llu epi_vec %llu epi_rows %llu act %d parts %d sig %d staged %d\n",
            N * op.Ho * op.Wo, K, op.out.C, BN, p.nkb, grid, ph[4], ph[0], ph[1], ph[2], ph[3], ph[5] / 128, ph[6] / 128, ph[7] / 128,
            act_inst, epi_sig(p.e), sig, p.staged ? (p.e.vec4 ? 4 : 2) : 0);
  }
#endif
}

}  // namespace mitb
