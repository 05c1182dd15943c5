// cv2.bilateralFilter(img_u8c3, d=17, sigmaColor=80, sigmaSpace=80) -- the detector's CPU pre-filter
// (detection/dbnet_convnext.py:549, ~1 s per 2048x1536 page on the host) as a CUDA kernel.
//
// Semantics follow OpenCV's 8-bit 3-channel path (third-party, restated and checked against the installed cv2 4.13 in
// tests): radius 8, BORDER_REFLECT_101, neighbours = offsets with sqrt(i^2+j^2) <= 8 in row-major order, spatial weight
// float(exp(-0.5 r^2/sigma_s^2)), colour weight LUT float(exp(-0.5 k^2/sigma_c^2)) indexed by |db|+|dg|+|dr|,
// w = sw*cw, sums accumulated with fused multiply-add in neighbour order, result = cvRound(sum * (1/wsum)).
#include <math.h>
#include "mitb_internal.h"

namespace mitb {

constexpr int BR = 8, BTX = 32, BTY = 8, BMAXN = 225;
__constant__ float c_space_w[BMAXN];
__constant__ int8_t c_off_y[BMAXN], c_off_x[BMAXN];
__constant__ float c_color_w[768];
static int g_bilateral_n = 0;
static PerDeviceOnce g_bilateral_once;     // the __constant__ tables live per device

static void bilateral_init() {
  if (!g_bilateral_once.first()) return;
  float sw[BMAXN]; int8_t oy[BMAXN], ox[BMAXN]; float cw[768];
  const double gs = -0.5 / (80.0 * 80.0), gc = -0.5 / (80.0 * 80.0);
  int n = 0;
  for (int i = -BR; i <= BR; ++i)
    for (int j = -BR; j <= BR; ++j) {
      const double r = sqrt((double)i * i + (double)j * j);
      if (r > BR) continue;
      sw[n] = (float)exp(r * r * gs); oy[n] = (int8_t)i; ox[n] = (int8_t)j; ++n;
    }
  for (int k = 0; k < 768; ++k) cw[k] = (float)exp((double)k * k * gc);
  CUDA_OK(cudaMemcpyToSymbol(c_space_w, sw, sizeof(float) * n));
  CUDA_OK(cudaMemcpyToSymbol(c_off_y, oy, n));
  CUDA_OK(cudaMemcpyToSymbol(c_off_x, ox, n));
  CUDA_OK(cudaMemcpyToSymbol(c_color_w, cw, sizeof(cw)));
  g_bilateral_n = n;
}

__device__ __forceinline__ int reflect101(int i, int n) {
  if (n == 1) return 0;
  while (i < 0 || i >= n) { if (i < 0) i = -i; else i = 2 * n - 2 - i; }
  return i;
}

__global__ void __launch_bounds__(BTX * BTY) bilateral17_kernel(const uint8_t* img, int H, int W, uint8_t* out, int nn) {
  constexpr int TW = BTX + 2 * BR, TH = BTY + 2 * BR;
  __shared__ uchar4 tile[TH][TW];
  __shared__ float cw[768];
  const int x0 = blockIdx.x * BTX, y0 = blockIdx.y * BTY;
  const int tid = threadIdx.y * BTX + threadIdx.x;
  for (int i = tid; i < 768; i += BTX * BTY) cw[i] = c_color_w[i];
  for (int i = tid; i < TW * TH; i += BTX * BTY) {
    const int ty = i / TW, tx = i - ty * TW;
    const int gy = reflect101(y0 + ty - BR, H), gx = reflect101(x0 + tx - BR, W);
    const uint8_t* p = img + ((size_t)gy * W + gx) * 3;
    tile[ty][tx] = make_uchar4(p[0], p[1], p[2], 0);
  }
  __syncthreads();
  const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
  if (x >= W || y >= H) return;
  const uchar4 c = tile[threadIdx.y + BR][threadIdx.x + BR];
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, ws = 0.f;
  for (int k = 0; k < nn; ++k) {
    const uchar4 v = tile[threadIdx.y + BR + c_off_y[k]][threadIdx.x + BR + c_off_x[k]];
    const int d = abs((int)v.x - (int)c.x) + abs((int)v.y - (int)c.y) + abs((int)v.z - (int)c.z);
    const float w = __fmul_rn(c_space_w[k], cw[d]);
    s0 = __fmaf_rn((float)v.x, w, s0); s1 = __fmaf_rn((float)v.y, w, s1); s2 = __fmaf_rn((float)v.z, w, s2);
    ws = __fadd_rn(ws, w);
  }
  // OpenCV's own implementation (bilateral_filter.simd.hpp) multiplies by the reciprocal: w = 1 / wsum; b = cvRound(sum_b * w).
  // This is bit-exact against cv2 with IPP disabled on every machine.  The stock pip wheel routes 8-bit bilateralFilter through
  // Intel IPP, a closed-source kernel whose rounding differs from OpenCV's own in a few bytes per million AND between CPUs
  // (per-channel division on one host, something else again on another), so it cannot serve as a definition.
  const float inv = __fdiv_rn(1.f, ws);
  uint8_t* o = out + ((size_t)y * W + x) * 3;
  o[0] = (uint8_t)__float2int_rn(__fmul_rn(s0, inv));
  o[1] = (uint8_t)__float2int_rn(__fmul_rn(s1, inv));
  o[2] = (uint8_t)__float2int_rn(__fmul_rn(s2, inv));
}

void launch_bilateral17(const uint8_t* img, int h, int w, uint8_t* out, cudaStream_t st) {
  bilateral_init();
  dim3 block(BTX, BTY), grid((w + BTX - 1) / BTX, (h + BTY - 1) / BTY);
  ProfScope ps("bilateral17", 197.0 * 12 * h * w, 6.0 * h * w, st);
  bilateral17_kernel<<<grid, block, 0, st>>>(img, h, w, out, g_bilateral_n);
  count_launch();
  CUDA_OK(cudaGetLastError());
}

}  // namespace mitb
