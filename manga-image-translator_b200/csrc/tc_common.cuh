// Device helpers shared by the wgmma convolution kernels (conv_tc.cu: register-gather producers; conv_tma.cu: TMA-fed
// operands): mbarrier / TMA / wgmma wrappers, the shared-memory matrix descriptor, the bf16 hi/mid split, the epilogue
// activations and the epilogue itself.  Included inside namespace mitb { namespace { ... } } of each translation unit.
#pragma once

// What the epilogue needs to know about the output side of a conv (ConvOp fields, see mitb_internal.h)
struct EpiParams {
  float* out; int oH, oW, out_cs, out_coff, Cout, out_planar, oy_mul, oy_add, ox_mul, ox_add;
  int Ho, Wo, M;                                              // logical output grid, rows of the GEMM
  const float* add0; int add0_cs, add0_coff, add0_planar;
  const float* add1; int add1_cs, add1_coff, add1_planar;
  const float* scale; const float* shift; const float* mul1; int act;
  float* stat_max; float* stat_sum; int* stat_idx; int stat_ld;     // fused log-softmax/argmax partials (vocabulary head)
  // split output (ConvOp::out_sv): bf16 hi / mid at [((n*os_Hp + y + os_pt)*os_Wp + x + os_pl)*os_pitch + os_coff + c] (null: none)
  uint16_t* os_hi; uint16_t* os_mid; int os_pitch, os_coff, os_Hp, os_Wp, os_pt, os_pl;
  const float* os_scale; const float* os_shift; int os_relu;  // consumer prologue applied before splitting
  float* partial; int npad;                                   // split-K: partial sums [splits][M][npad] (null: none)
  int vec2;                                                   // NHWC, even strides / offsets, 8-byte aligned operands, Cout even
  int vec4;                                                   // vec2 with strides / offsets / Cout multiples of 4, 16-byte aligned (8 for os_hi / os_mid)
};

inline void fill_epi(EpiParams& e, const ConvOp& op) {
  memset(&e, 0, sizeof(e));
  e.out = op.out.p; e.oH = op.out.H; e.oW = op.out.W; e.out_cs = op.out.cs; e.out_coff = op.out.coff; e.Cout = op.out.C;
  e.out_planar = op.out.planar; e.oy_mul = op.oy_mul; e.oy_add = op.oy_add; e.ox_mul = op.ox_mul; e.ox_add = op.ox_add;
  e.Ho = op.Ho; e.Wo = op.Wo; e.M = op.in.N * op.Ho * op.Wo;
  e.add0 = op.add0.p; e.add0_cs = op.add0.cs; e.add0_coff = op.add0.coff; e.add0_planar = op.add0.planar;
  e.add1 = op.add1.p; e.add1_cs = op.add1.cs; e.add1_coff = op.add1.coff; e.add1_planar = op.add1.planar;
  e.scale = op.scale; e.shift = op.shift; e.mul1 = op.mul1; e.act = op.act;
  e.stat_max = op.stat_max; e.stat_sum = op.stat_sum; e.stat_idx = op.stat_idx; e.stat_ld = op.stat_ld;
  if (op.out_sv.valid()) {
    const SplitView& o = op.out_sv;
    e.os_hi = o.hi; e.os_mid = o.mid; e.os_pitch = o.C; e.os_coff = op.out_sv_coff; e.os_Hp = o.Hp; e.os_Wp = o.Wp; e.os_pt = o.pt; e.os_pl = o.pl;
    e.os_scale = op.os_scale; e.os_shift = op.os_shift; e.os_relu = op.os_relu;
  }
  auto al8 = [](const void* q) { return ((uintptr_t)q & 7) == 0; };
  auto nhwc_ok = [&](const View& v) { return !v.p || (!v.planar && ((v.cs | v.coff) & 1) == 0 && al8(v.p)); };
  e.vec2 = !op.out.planar && op.out.C % 2 == 0 && nhwc_ok(op.out) && nhwc_ok(op.add0) && nhwc_ok(op.add1) && al8(op.scale) && al8(op.shift) &&
           al8(op.mul1) && al8(op.os_scale) && al8(op.os_shift) && (!e.os_hi || ((e.os_pitch | e.os_coff) & 1) == 0) &&
           (!e.os_hi || (((uintptr_t)e.os_hi | (uintptr_t)e.os_mid) & 3) == 0);
  auto al16 = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
  auto nhwc_ok4 = [&](const View& v) { return !v.p || (((v.cs | v.coff) & 3) == 0 && al16(v.p)); };
  e.vec4 = e.vec2 && op.out.C % 4 == 0 && nhwc_ok4(op.out) && nhwc_ok4(op.add0) && nhwc_ok4(op.add1) && al16(op.scale) && al16(op.shift) &&
           al16(op.mul1) && al16(op.os_scale) && al16(op.os_shift) && (!e.os_hi || ((e.os_pitch | e.os_coff) & 3) == 0) &&
           (!e.os_hi || (((uintptr_t)e.os_hi | (uintptr_t)e.os_mid) & 7) == 0);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded spin: a protocol bug traps (reported as a launch failure) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  long long t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 1023u) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000ll) __trap();          // ~2 s at 2 GHz: far beyond any legitimate wait
    }
  }
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* map, uint32_t bar, int x, int y) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_dst), "l"(map), "r"(bar), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma (warpgroup MMA, sm_90a): D[64 x N] (fp32, registers of the 128 threads of a warpgroup) += A[64 x 16] * B[16 x N],
// both operands K-major in shared memory.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across wgmma_wait / wgmma_fence
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, int accumulate);
template <> __device__ __forceinline__ void wgmma_bf16<32>(float (&d)[16], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
template <> __device__ __forceinline__ void wgmma_bf16<64>(float (&d)[32], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
template <> __device__ __forceinline__ void wgmma_bf16<96>(float (&d)[48], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %50, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
template <> __device__ __forceinline__ void wgmma_bf16<128>(float (&d)[64], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate) : "memory");
}

// wgmma shared-memory matrix descriptor: K-major operand, 128-byte swizzle, rows of 128 B, 8-row groups 1024 B apart.
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (unused for swizzled K-major, 1) | [32,46) stride byte
//   offset >> 4 (1024 >> 4) | [62,64) layout type 1 = SWIZZLE_128B.  A 16-element step along K inside the swizzle row is +32 B
//   of start address (+2 in the descriptor).
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}

// One K block (64 channels) of the bf16x3 product for this warpgroup: for each 16-wide k step Ah*Bh, Ah*Bm, Am*Bh
template <int BN>
__device__ __forceinline__ void wgmma_kblock_x3(float (&acc)[BN / 2], uint64_t dah, uint64_t dam, uint64_t dbh, uint64_t dbm, bool first) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint64_t adv = (uint64_t)(2 * k);
    wgmma_bf16<BN>(acc, dah + adv, dbh + adv, (first && k == 0) ? 0 : 1);
    wgmma_bf16<BN>(acc, dah + adv, dbm + adv, 1);
    wgmma_bf16<BN>(acc, dam + adv, dbh + adv, 1);
  }
}

// split 8 fp32 values into bf16 hi / mid packs (16 bytes each): 6 instructions per pair
// (F2FP pack-convert for hi, shift/mask to get hi back as fp32, two FADD for the remainder, F2FP for mid)
__device__ __forceinline__ void split8(const float (&v)[8], uint4& hi, uint4& mid) {
  uint32_t h[4], m[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __nv_bfloat162 hb = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);     // .x (low half) = v[2i]
    const uint32_t hbits = *reinterpret_cast<const uint32_t*>(&hb);
    const float h0 = __uint_as_float(hbits << 16), h1 = __uint_as_float(hbits & 0xffff0000u);
    const __nv_bfloat162 mb = __floats2bfloat162_rn(v[2 * i] - h0, v[2 * i + 1] - h1);
    h[i] = hbits;
    m[i] = *reinterpret_cast<const uint32_t*>(&mb);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  mid = make_uint4(m[0], m[1], m[2], m[3]);
}


// split 4 fp32 values into bf16 hi / mid packs (8 bytes each)
__device__ __forceinline__ void split4(const float4 v, uint2& hi, uint2& mid) {
  const __nv_bfloat162 h0 = __floats2bfloat162_rn(v.x, v.y), h1 = __floats2bfloat162_rn(v.z, v.w);
  const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&h0), b1 = *reinterpret_cast<const uint32_t*>(&h1);
  const __nv_bfloat162 m0 = __floats2bfloat162_rn(v.x - __uint_as_float(b0 << 16), v.y - __uint_as_float(b0 & 0xffff0000u));
  const __nv_bfloat162 m1 = __floats2bfloat162_rn(v.z - __uint_as_float(b1 << 16), v.w - __uint_as_float(b1 & 0xffff0000u));
  hi = make_uint2(b0, b1);
  mid = make_uint2(*reinterpret_cast<const uint32_t*>(&m0), *reinterpret_cast<const uint32_t*>(&m1));
}

// exact-erf GELU with erf from Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7): two MUFU + ~14 FP32 instructions instead of the
// ~35 of erff(); the GELU epilogue of the ConvNeXt fc1 layers is otherwise longer than their 2..8 K-block main loops
__device__ __forceinline__ float gelu_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.f)));
  float pl = fmaf(t, 1.061405429f, -1.453152027f);
  pl = fmaf(pl, t, 1.421413741f);
  pl = fmaf(pl, t, -0.284496736f);
  pl = fmaf(pl, t, 0.254829592f);
  pl *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(z * z * -1.44269504088896340736f));
  const float erf_abs = fmaf(-pl, e, 1.f);
  return 0.5f * x * (1.f + copysignf(erf_abs, x));
}

template <int ACT>
__device__ __forceinline__ float act_t(float v, int act_rt) {
  if (ACT == ACT_NONE) return v;
  if (ACT == ACT_RELU) return fmaxf(v, 0.f);
  if (ACT == ACT_GELU) return gelu_fast(v);
  if (ACT == ACT_SILU) return v / (1.f + expf(-v));
  return apply_act(v, act_rt);               // ACT == -1: rare activations, runtime switch
}


// split 2 fp32 values into packed bf16 hi / mid pairs
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& mid) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const uint32_t hb = *reinterpret_cast<const uint32_t*>(&h);
  const __nv_bfloat162 m = __floats2bfloat162_rn(a - __uint_as_float(hb << 16), b - __uint_as_float(hb & 0xffff0000u));
  hi = hb; mid = *reinterpret_cast<const uint32_t*>(&m);
}

// (max, first argmax, sum exp) partials of the vocabulary head: merge b into a
__device__ __forceinline__ void stat_merge(float& am, float& as, int& ai, float bm, float bs, int bi) {
  const float m = fmaxf(am, bm);
  if (m == -INFINITY) { ai = min(ai, bi); return; }
  as = as * expf(am - m) + bs * expf(bm - m);
  ai = am > bm ? ai : bm > am ? bi : min(ai, bi);
  am = m;
}

// Epilogue signature (EpiSig, mitb_internal.h) of a launch: a bitmask that a kernel can take as a template parameter
// (epilogue_staged declares, loads and tests only what its signature has).
inline int epi_sig(const EpiParams& e) {
  return (e.add0 ? EPI_ADD0 : 0) | (e.scale ? EPI_SCALE : 0) | (e.shift ? EPI_SHIFT : 0) | (e.mul1 ? EPI_MUL1 : 0) | (e.add1 ? EPI_ADD1 : 0) |
         (e.out ? EPI_OUT : 0) | (e.os_hi ? EPI_OS : 0) | (e.os_hi && e.os_scale ? EPI_OS_AFFINE : 0) |
         (e.os_hi && e.os_scale && e.os_relu ? EPI_OS_RELU : 0);
}
// does a launch of signature SIG have part BIT (rt: the run-time test, used by EPI_GENERIC only)
template <int SIG, int BIT> __device__ __forceinline__ bool epi_has(bool rt) {
  if constexpr (SIG == EPI_GENERIC) return rt;
  else return (SIG & BIT) != 0;
}

// The fused elementwise chain of two adjacent columns, v = acc (+add0) ; v = v*scale+shift ; act ; *mul1 ; +add1, and the split of
// its result into the consumer's bf16 hi / mid operands (after the consumer's prologue os_scale / os_shift / os_relu).  Every
// two-column epilogue calls these, so the fp32 operations and their order, which the outputs' bits depend on, live in one place.
// The products and sums are explicitly rounded: a signature with both scale and shift (or mul1 and add1) must not contract them
// into one FMA, so that every signature computes the bits of the generic chain.
template <int ACT, int SIG = EPI_GENERIC>
__device__ __forceinline__ void epi_chain2(const EpiParams& e, float& v0, float& v1, float2 a0, float2 sc, float2 sh, float2 m1, float2 a1) {
  if (epi_has<SIG, EPI_ADD0>(e.add0)) { v0 = __fadd_rn(v0, a0.x); v1 = __fadd_rn(v1, a0.y); }
  if (epi_has<SIG, EPI_SCALE>(e.scale)) { v0 = __fmul_rn(v0, sc.x); v1 = __fmul_rn(v1, sc.y); }
  if (epi_has<SIG, EPI_SHIFT>(e.shift)) { v0 = __fadd_rn(v0, sh.x); v1 = __fadd_rn(v1, sh.y); }
  v0 = act_t<ACT>(v0, e.act); v1 = act_t<ACT>(v1, e.act);
  if (epi_has<SIG, EPI_MUL1>(e.mul1)) { v0 = __fmul_rn(v0, m1.x); v1 = __fmul_rn(v1, m1.y); }
  if (epi_has<SIG, EPI_ADD1>(e.add1)) { v0 = __fadd_rn(v0, a1.x); v1 = __fadd_rn(v1, a1.y); }
}
template <int SIG = EPI_GENERIC>
__device__ __forceinline__ void epi_split2(const EpiParams& e, float v0, float v1, float2 s, float2 t, uint32_t& hi, uint32_t& mid) {
  if (epi_has<SIG, EPI_OS_AFFINE>(e.os_scale)) {
    v0 = fmaf(v0, s.x, t.x); v1 = fmaf(v1, s.y, t.y);
    if (epi_has<SIG, EPI_OS_RELU>(e.os_relu)) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
  }
  split2(v0, v1, hi, mid);
}

// Epilogue of one 128 x BN output tile from the wgmma accumulator fragments.  Warp w of warpgroup g holds rows
// 64 g + 16 (w % 4) + lane / 4 (registers 4j, 4j+1) and the row 8 below it (4j+2, 4j+3), columns 8 j + 2 (lane % 4) + {0, 1}:
// a warp store covers 8 rows x 32 contiguous bytes, whole sectors.  rowpix(r, nimg, oy, ox) maps tile row r to its output pixel
// (false: outside).  Modes: vocabulary-head row statistics, split-K partial sums, or the fused elementwise chain
// v = acc (+add0) ; v = v*scale+shift ; act ; *mul1 ; +add1 -> fp32 out and / or the consumer's bf16 hi / mid operands.
template <int ACT, int BN, class RowPix>
__device__ __forceinline__ void epilogue_tile(const EpiParams& e, const float (&acc)[BN / 2], int row0, int n0, int z, RowPix rowpix) {
  const int lane = threadIdx.x & 31;
  const int cl = 2 * (lane & 3);
  if (e.stat_max || e.partial) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int nimg = 0, oy = 0, ox = 0;
      const bool ok = rowpix(row0 + 8 * h, nimg, oy, ox);
      if (e.stat_max) {
        // online (max, first argmax, sum exp) per column half of the N tile over this thread's columns, then over the 4 lanes of
        // the row (model_48px_ctc.py:460-461); the logits never leave the registers
        constexpr int kHalf = ((BN / 16 + 1) / 2) * 16;
        float bm[2] = {-INFINITY, -INFINITY}, bs[2] = {0.f, 0.f}; int bi[2] = {0x7fffffff, 0x7fffffff};
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            const int cc = 8 * j + cl + q, c = n0 + cc, hf = cc < kHalf ? 0 : 1;
            if (c < e.Cout) {
              const float x = acc[4 * j + 2 * h + q] + (e.shift ? __ldg(e.shift + c) : 0.f);
              if (x > bm[hf]) { bs[hf] = bs[hf] * expf(bm[hf] - x) + 1.f; bm[hf] = x; bi[hf] = c; }
              else bs[hf] += expf(x - bm[hf]);
            }
          }
        }
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
#pragma unroll
          for (int o = 1; o <= 2; o <<= 1)
            stat_merge(bm[hf], bs[hf], bi[hf], __shfl_xor_sync(0xffffffffu, bm[hf], o), __shfl_xor_sync(0xffffffffu, bs[hf], o),
                       __shfl_xor_sync(0xffffffffu, bi[hf], o));
          if (ok && (lane & 3) == 0) {
            const size_t o = (((size_t)nimg * e.Ho + oy) * e.Wo + ox) * e.stat_ld + (n0 / BN) * 2 + hf;
            e.stat_max[o] = bm[hf]; e.stat_sum[o] = bs[hf]; e.stat_idx[o] = bi[hf];
          }
        }
        continue;
      }
      if (!ok) continue;
      // split-K partial: raw accumulators to partial[z][m][npad]
      float* dst = e.partial + ((size_t)z * e.M + ((size_t)nimg * e.Ho + oy) * e.Wo + ox) * e.npad + n0 + cl;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    }
    return;
  }
  // Fused elementwise chain.  The column-group loop is NOT unrolled: the body handles the group in r[0..3] and the registers
  // rotate down by one group per iteration.  Unrolled over BN / 8 groups with every runtime branch, the epilogue was tens of
  // thousands of instructions run once per tile, and fetching them, not the arithmetic or the stores, set its time.
  int nimg[2], oy[2], ox[2];
  bool ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    nimg[h] = oy[h] = ox[h] = 0;
    ok[h] = rowpix(row0 + 8 * h, nimg[h], oy[h], ox[h]);
  }
  float r[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) r[i] = acc[i];
  auto next_group = [&]() {
#pragma unroll
    for (int i = 0; i + 4 < BN / 2; ++i) r[i] = r[i + 4];
  };
  // two separate loops so that each keeps only its own row addresses live (registers are tight at BN = 128)
  if (e.vec2) {
    int opix[2], spix[2];                  // pixel indices of out / the split output in 32 bits, like e.M; element offsets in 64
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      opix[h] = (nimg[h] * e.oH + oy[h] * e.oy_mul + e.oy_add) * e.oW + ox[h] * e.ox_mul + e.ox_add;
      spix[h] = (nimg[h] * e.os_Hp + oy[h] + e.os_pt) * e.os_Wp + ox[h] + e.os_pl;
    }
#pragma unroll 1
    for (int j = 0; j < BN / 8; ++j) {
      const int c = n0 + 8 * j + cl;
      if (c < e.Cout) {
        // NHWC, even channel strides / offsets, 8-byte aligned operands, Cout even: columns c, c + 1 as one float2.  The loads of
        // the group (both rows) are issued before its first store: add0 / add1 may alias out, so the compiler cannot hoist them.
        const float2 z2 = make_float2(0.f, 0.f);
        const float2 sc = e.scale ? __ldg(reinterpret_cast<const float2*>(e.scale + c)) : z2;
        const float2 sh = e.shift ? __ldg(reinterpret_cast<const float2*>(e.shift + c)) : z2;
        const float2 m1 = e.mul1 ? __ldg(reinterpret_cast<const float2*>(e.mul1 + c)) : z2;
        float2 a0[2], a1[2];
        auto load_row = [&](int h) {
          a0[h] = ok[h] && e.add0 ? *reinterpret_cast<const float2*>(e.add0 + (size_t)opix[h] * e.add0_cs + e.add0_coff + c) : z2;
          a1[h] = ok[h] && e.add1 ? *reinterpret_cast<const float2*>(e.add1 + (size_t)opix[h] * e.add1_cs + e.add1_coff + c) : z2;
        };
        // both rows' residual loads ahead of the first store, except where the activation leaves no registers for them at BN = 128
        constexpr bool kBothRows = ACT != ACT_SILU && ACT != -1;
        if (kBothRows) { load_row(0); load_row(1); }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!kBothRows) load_row(h);
          if (!ok[h]) continue;
          float v0 = r[2 * h], v1 = r[2 * h + 1];
          epi_chain2<ACT>(e, v0, v1, a0[h], sc, sh, m1, a1[h]);
          if (e.out) *reinterpret_cast<float2*>(e.out + (size_t)opix[h] * e.out_cs + e.out_coff + c) = make_float2(v0, v1);
          if (e.os_hi) {                     // producer -> consumer fusion: store the consumer's bf16 hi / mid operands directly
            const float2 s = e.os_scale ? __ldg(reinterpret_cast<const float2*>(e.os_scale + c)) : z2;
            const float2 t = e.os_scale ? __ldg(reinterpret_cast<const float2*>(e.os_shift + c)) : z2;
            uint32_t hh, mm;
            epi_split2(e, v0, v1, s, t, hh, mm);
            const size_t so = (size_t)spix[h] * e.os_pitch + e.os_coff + c;
            *reinterpret_cast<uint32_t*>(e.os_hi + so) = hh;
            *reinterpret_cast<uint32_t*>(e.os_mid + so) = mm;
          }
        }
      }
      next_group();
    }
    return;
  }
  size_t opix[2], opl_pix[2], so[2];
  const size_t oplane = (size_t)e.oH * e.oW;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int py = oy[h] * e.oy_mul + e.oy_add, px = ox[h] * e.ox_mul + e.ox_add;
    opix[h] = ((size_t)nimg[h] * e.oH + py) * e.oW + px;
    opl_pix[h] = (size_t)py * e.oW + px;
    so[h] = e.os_hi ? ((size_t)(nimg[h] * e.os_Hp + oy[h] + e.os_pt) * e.os_Wp + ox[h] + e.os_pl) * e.os_pitch + e.os_coff : 0;
  }
#pragma unroll 1
  for (int j = 0; j < BN / 8; ++j) {
    const int c = n0 + 8 * j + cl;
    if (c < e.Cout) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!ok[h]) continue;
        auto at = [&](const float* b, int cs, int coff, int planar, int cc) -> const float* {
          return planar ? b + ((size_t)nimg[h] * cs + coff + cc) * oplane + opl_pix[h] : b + opix[h] * cs + coff + cc;
        };
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int cc = c + q;
          if (cc >= e.Cout) break;
          float x = r[2 * h + q];
          if (e.add0) x += *at(e.add0, e.add0_cs, e.add0_coff, e.add0_planar, cc);
          if (e.scale) x *= __ldg(e.scale + cc);
          if (e.shift) x += __ldg(e.shift + cc);
          x = act_t<ACT>(x, e.act);
          if (e.mul1) x *= __ldg(e.mul1 + cc);
          if (e.add1) x += *at(e.add1, e.add1_cs, e.add1_coff, e.add1_planar, cc);
          if (e.out) *const_cast<float*>(at(e.out, e.out_cs, e.out_coff, e.out_planar, cc)) = x;
          if (e.os_hi) {
            if (e.os_scale) { x = fmaf(x, __ldg(e.os_scale + cc), __ldg(e.os_shift + cc)); if (e.os_relu) x = fmaxf(x, 0.f); }
            const __nv_bfloat16 hb = __float2bfloat16_rn(x);
            const __nv_bfloat16 mb = __float2bfloat16_rn(x - __bfloat162float(hb));
            e.os_hi[so[h] + cc] = __bfloat16_as_ushort(hb); e.os_mid[so[h] + cc] = __bfloat16_as_ushort(mb);
          }
        }
      }
    }
    next_group();
  }
}
