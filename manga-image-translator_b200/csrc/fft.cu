// Real 2-D FFT for LaMa's FourierUnit (inpainting_lama_mpe.py:228, :252): torch.fft.rfftn / irfftn over (h, w),
// norm='ortho', on planar (NCHW) tensors, for ARBITRARY h, w (the bottleneck is (H/8) x (W/8): 256x192 for a
// 2048x1536 page, 320x240 at --inpainting-size 2560, odd sizes for odd pages).
//
// Shared-memory Stockham autosort FFT, mixed radix {4,2,3,5,7} plus a generic prime-radix stage, twiddles from a
// per-length table computed in double precision on the host.  2-D transform = row pass + column pass:
//   forward : rows   real->half-complex, two real rows packed into one complex FFT          (rfft_rows_kernel)
//             cols   complex FFT over h on tiles of 8 adjacent columns, writes the spectrum as
//                    interleaved planes c0_re, c0_im, c1_re, ...  (the "stack/permute/view" of :229-231) (fft_cols_kernel)
//   inverse : cols   reads the re/im planes (the inverse "view/permute/complex" of :245-249), inverse FFT over h
//             rows   half-complex->real for two rows per complex FFT, drops Im of the DC/Nyquist bins like C2R does,
//                    fuses the `x + fu(x)` residual of SpectralTransform (:305)
// The complex intermediate [planes][h][w/2+1] is written once and read once (L2 resident for LaMa sizes).
#include <math.h>
#include <mutex>
#include "mitb_internal.h"

namespace mitb {

constexpr int kMaxStages = 16;
struct FftDev { int n, nstages; int radix[kMaxStages]; const float2* tw; };
struct FftPlan { FftDev dev; };

FftTrace* g_fft_trace = nullptr;

static std::mutex g_plan_mu;
static std::map<std::pair<int, int>, FftPlan*> g_plans;    // (device, n)

FftPlan* fft_plan_get(int n) {
  int dev = 0; CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(g_plan_mu);
  auto key = std::make_pair(dev, n);
  auto it = g_plans.find(key);
  if (it != g_plans.end()) return it->second;
  MITB_CHECK(n >= 1 && n <= 4096, "fft length %d unsupported", n);
  FftPlan* p = new FftPlan();
  p->dev.n = n; p->dev.nstages = 0;
  int r = n;
  auto push = [&](int f) { MITB_CHECK(p->dev.nstages < kMaxStages, "too many fft stages"); p->dev.radix[p->dev.nstages++] = f; };
  while (r % 4 == 0) { push(4); r /= 4; }
  while (r % 2 == 0) { push(2); r /= 2; }
  for (int f = 3; f <= r; f += 2) while (r % f == 0) { push(f); r /= f; }
  std::vector<float2> tw(n);
  for (int i = 0; i < n; ++i) {
    double a = -2.0 * M_PI * (double)i / (double)n;
    tw[i] = make_float2((float)cos(a), (float)sin(a));
  }
  float2* d = nullptr;
  CUDA_OK(cudaMalloc(&d, sizeof(float2) * n));
  CUDA_OK(cudaMemcpy(d, tw.data(), sizeof(float2) * n, cudaMemcpyHostToDevice));
  p->dev.tw = d;
  g_plans[key] = p;
  return p;
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 twd(const float2* tw, int i, bool inv) { float2 t = __ldg(tw + i); if (inv) t.y = -t.y; return t; }

template <int R>
__device__ __forceinline__ void butterfly_small(const float2* x, float2* y, int q, int p, int s, int m, int n,
                                                const float2* tw, bool inv) {
  float2 a[R];
#pragma unroll
  for (int j = 0; j < R; ++j) a[j] = x[q + s * (p + j * m)];
  const int step = n / R;
#pragma unroll
  for (int k = 0; k < R; ++k) {
    float2 acc = a[0];
#pragma unroll
    for (int j = 1; j < R; ++j) acc = cadd(acc, cmul(a[j], twd(tw, ((j * k) % R) * step, inv)));
    if (k) acc = cmul(acc, twd(tw, s * p * k, inv));
    y[q + s * (R * p + k)] = acc;
  }
}

// FFT of `batch` sequences of length pl.n stored at X + b*ld; Y is scratch of the same shape.  Returns the buffer
// holding the natural-order result.  All threads of the CTA must call it.
__device__ float2* fft_smem(float2* X, float2* Y, int batch, int ld, const FftDev& pl, bool inv) {
  int ncur = pl.n, s = 1;
  const int n = pl.n;
  for (int st = 0; st < pl.nstages; ++st) {
    const int r = pl.radix[st];
    const int m = ncur / r;
    const int nb = n / r;
    for (int wi = threadIdx.x; wi < batch * nb; wi += blockDim.x) {
      const int b = wi / nb, bid = wi - b * nb;
      const int p = bid / s, q = bid - p * s;
      const float2* x = X + b * ld; float2* y = Y + b * ld;
      if (r == 4) {
        const float2 a0 = x[q + s * p], a1 = x[q + s * (p + m)], a2 = x[q + s * (p + 2 * m)], a3 = x[q + s * (p + 3 * m)];
        const float2 t0 = cadd(a0, a2), t1 = csub(a0, a2), t2 = cadd(a1, a3);
        float2 t3 = csub(a1, a3);
        t3 = inv ? make_float2(-t3.y, t3.x) : make_float2(t3.y, -t3.x);      // multiply by -i (fwd) / +i (inv)
        float2 o0 = cadd(t0, t2), o1 = cadd(t1, t3), o2 = csub(t0, t2), o3 = csub(t1, t3);
        if (p) { o1 = cmul(o1, twd(pl.tw, s * p, inv)); o2 = cmul(o2, twd(pl.tw, 2 * s * p, inv)); o3 = cmul(o3, twd(pl.tw, 3 * s * p, inv)); }
        y[q + s * (4 * p)] = o0; y[q + s * (4 * p + 1)] = o1; y[q + s * (4 * p + 2)] = o2; y[q + s * (4 * p + 3)] = o3;
      } else if (r == 2) {
        const float2 a0 = x[q + s * p], a1 = x[q + s * (p + m)];
        float2 o1 = csub(a0, a1);
        if (p) o1 = cmul(o1, twd(pl.tw, s * p, inv));
        y[q + s * (2 * p)] = cadd(a0, a1); y[q + s * (2 * p + 1)] = o1;
      } else if (r == 3) butterfly_small<3>(x, y, q, p, s, m, n, pl.tw, inv);
      else if (r == 5) butterfly_small<5>(x, y, q, p, s, m, n, pl.tw, inv);
      else if (r == 7) butterfly_small<7>(x, y, q, p, s, m, n, pl.tw, inv);
      else {
        const int step = n / r;
        for (int k = 0; k < r; ++k) {
          float2 acc = x[q + s * p];
          int jk = 0;
          for (int j = 1; j < r; ++j) {
            jk += k; if (jk >= r) jk -= r;
            acc = cadd(acc, cmul(x[q + s * (p + j * m)], twd(pl.tw, jk * step, inv)));
          }
          if (k) acc = cmul(acc, twd(pl.tw, s * p * k, inv));
          y[q + s * (r * p + k)] = acc;
        }
      }
    }
    __syncthreads();
    float2* t = X; X = Y; Y = t;
    ncur = m; s *= r;
  }
  return X;
}

// ---- forward rows: planar real [planes][h][w] -> tmp complex [planes][h][w2]
__global__ void __launch_bounds__(256) rfft_rows_kernel(const float* in, float2* tmp, int h, int w, int w2, int P, FftDev pl) {
  extern __shared__ float2 fsm[];
  float2* X = fsm; float2* Y = fsm + (size_t)P * w;
  const int plane = blockIdx.y;
  const int pair0 = blockIdx.x * P;
  const int npairs = (h + 1) / 2;
  const int np = min(P, npairs - pair0);
  const float* src = in + (size_t)plane * h * w;
  for (int i = threadIdx.x; i < np * w; i += blockDim.x) {
    const int b = i / w, x = i - b * w;
    const int ya = 2 * (pair0 + b), yb = ya + 1;
    X[b * w + x] = make_float2(src[(size_t)ya * w + x], yb < h ? src[(size_t)yb * w + x] : 0.f);
  }
  __syncthreads();
  const float2* Z = fft_smem(X, Y, np, w, pl, false);
  float2* dst = tmp + (size_t)plane * h * w2;
  for (int i = threadIdx.x; i < np * w2; i += blockDim.x) {
    const int b = i / w2, k = i - b * w2;
    const float2 z = Z[b * w + k], zc = Z[b * w + (k ? w - k : 0)];
    const int ya = 2 * (pair0 + b), yb = ya + 1;
    dst[(size_t)ya * w2 + k] = make_float2(0.5f * (z.x + zc.x), 0.5f * (z.y - zc.y));
    if (yb < h) dst[(size_t)yb * w2 + k] = make_float2(0.5f * (z.y + zc.y), -0.5f * (z.x - zc.x));
  }
}

// ---- columns: complex FFT over h on CB adjacent columns.
// forward: src = tmp complex, dst = interleaved re/im planes (scaled).  inverse: src = re/im planes, dst = tmp complex.
__global__ void __launch_bounds__(256) fft_cols_kernel(float2* tmp, float* spec, int h, int w2, int CB, FftDev pl, int inverse,
                                                       float scale) {
  extern __shared__ float2 fsm[];
  const int ld = h | 1;
  float2* X = fsm; float2* Y = fsm + (size_t)CB * ld;
  const int plane = blockIdx.y;
  const int kx0 = blockIdx.x * CB;
  const int nc = min(CB, w2 - kx0);
  float2* t = tmp + (size_t)plane * h * w2;
  float* re = spec + (size_t)(2 * plane) * h * w2; float* im = re + (size_t)h * w2;
  for (int i = threadIdx.x; i < nc * h; i += blockDim.x) {
    const int row = i / nc, col = i - row * nc;
    const size_t g = (size_t)row * w2 + kx0 + col;
    X[col * ld + row] = inverse ? make_float2(re[g], im[g]) : t[g];
  }
  __syncthreads();
  const float2* Z = fft_smem(X, Y, nc, ld, pl, inverse != 0);
  for (int i = threadIdx.x; i < nc * h; i += blockDim.x) {
    const int row = i / nc, col = i - row * nc;
    const size_t g = (size_t)row * w2 + kx0 + col;
    const float2 z = Z[col * ld + row];
    if (inverse) t[g] = z;
    else { re[g] = z.x * scale; im[g] = z.y * scale; }
  }
}

// ---- inverse rows: tmp complex [planes][h][w2] -> planar real [planes][h][w] (+ optional residual)
__global__ void __launch_bounds__(256) irfft_rows_kernel(const float2* tmp, float* out, const float* add, int h, int w, int w2,
                                                         int P, FftDev pl, float scale) {
  extern __shared__ float2 fsm[];
  float2* X = fsm; float2* Y = fsm + (size_t)P * w;
  const int plane = blockIdx.y;
  const int pair0 = blockIdx.x * P;
  const int npairs = (h + 1) / 2;
  const int np = min(P, npairs - pair0);
  const float2* src = tmp + (size_t)plane * h * w2;
  for (int i = threadIdx.x; i < np * w2; i += blockDim.x) {
    const int b = i / w2, k = i - b * w2;
    const int ya = 2 * (pair0 + b), yb = ya + 1;
    float2 A = src[(size_t)ya * w2 + k];
    float2 B = yb < h ? src[(size_t)yb * w2 + k] : make_float2(0.f, 0.f);
    if (k == 0 || 2 * k == w) { A.y = 0.f; B.y = 0.f; }            // C2R ignores Im of the DC / Nyquist bins
    X[b * w + k] = make_float2(A.x - B.y, A.y + B.x);              // A + iB
    if (k != 0 && 2 * k != w) X[b * w + (w - k)] = make_float2(A.x + B.y, -A.y + B.x);   // conj(A) + i conj(B)
  }
  __syncthreads();
  const float2* Z = fft_smem(X, Y, np, w, pl, true);
  float* dst = out + (size_t)plane * h * w;
  const float* res = add ? add + (size_t)plane * h * w : nullptr;
  for (int i = threadIdx.x; i < np * w; i += blockDim.x) {
    const int b = i / w, x = i - b * w;
    const int ya = 2 * (pair0 + b), yb = ya + 1;
    const float2 z = Z[b * w + x];
    const size_t ga = (size_t)ya * w + x, gb = (size_t)yb * w + x;
    dst[ga] = z.x * scale + (res ? res[ga] : 0.f);
    if (yb < h) dst[gb] = z.y * scale + (res ? res[gb] : 0.f);
  }
}

static PerDeviceOnce g_fft_attr;
static void fft_attrs() {
  if (!g_fft_attr.first()) return;
  CUDA_OK(cudaFuncSetAttribute(rfft_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  CUDA_OK(cudaFuncSetAttribute(irfft_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  CUDA_OK(cudaFuncSetAttribute(fft_cols_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
}

static const float* planar_base(const View& v, int* planes) {
  MITB_CHECK(v.planar, "fft expects planar views");
  MITB_CHECK(v.N == 1 || (v.cs == v.C && v.coff == 0), "fft expects contiguous planes");
  *planes = v.N * v.C;
  return v.p + (size_t)v.coff * v.H * v.W;
}

// test hook record: the two plans' radix sequences and the batching of the row and column passes
static void fft_trace(const FftPlan* ph, const FftPlan* pw, int P, int CB) {
  if (!g_fft_trace) return;
  FftTrace& t = *g_fft_trace;
  t = FftTrace();
  t.h_nst = ph->dev.nstages; t.w_nst = pw->dev.nstages;
  for (int s = 0; s < ph->dev.nstages; ++s) t.h_radix[s] = ph->dev.radix[s];
  for (int s = 0; s < pw->dev.nstages; ++s) t.w_radix[s] = pw->dev.radix[s];
  t.P = P; t.CB = CB;
}

static int pick_batch(int n, int per_elem_bytes, int want) {
  int b = want;
  while (b > 1 && (size_t)2 * b * (n | 1) * per_elem_bytes > 96 * 1024) b >>= 1;
  MITB_CHECK((size_t)2 * b * (n | 1) * per_elem_bytes <= 200 * 1024, "fft length %d too large for shared memory", n);
  return b;
}

void launch_rfft2(const View& in, const View& spec, float2* tmp, cudaStream_t st) {
  fft_attrs();
  int planes = 0, splanes = 0;
  const float* src = planar_base(in, &planes);
  float* dst = const_cast<float*>(planar_base(spec, &splanes));
  const int h = in.H, w = in.W, w2 = w / 2 + 1;
  MITB_CHECK(splanes == 2 * planes && spec.H == h && spec.W == w2, "rfft2 shape mismatch");
  FftPlan* pw = fft_plan_get(w); FftPlan* ph = fft_plan_get(h);
  const int P = pick_batch(w, 8, 8), CB = pick_batch(h, 8, 8);
  const int npairs = (h + 1) / 2;
  fft_trace(ph, pw, P, CB);
  // algorithmic: read the real planes once, write the half spectrum once; ~2.5 N log2 N flops per real plane
  ProfScope ps("fft_rfft2", 2.5 * planes * (double)h * w * log2((double)h * w), 4.0 * planes * ((double)h * w + 2.0 * h * w2), st);
  rfft_rows_kernel<<<dim3((npairs + P - 1) / P, planes), 256, (size_t)2 * P * w * sizeof(float2), st>>>(src, tmp, h, w, w2, P, pw->dev);
  count_launch();
  fft_cols_kernel<<<dim3((w2 + CB - 1) / CB, planes), 256, (size_t)2 * CB * (h | 1) * sizeof(float2), st>>>(
      tmp, dst, h, w2, CB, ph->dev, 0, (float)(1.0 / sqrt((double)h * (double)w)));
  count_launch();
  CUDA_OK(cudaGetLastError());
}

void launch_irfft2(const View& spec, const View& out, const View* add, float2* tmp, cudaStream_t st) {
  fft_attrs();
  int planes = 0, splanes = 0, aplanes = 0;
  float* src = const_cast<float*>(planar_base(spec, &splanes));
  float* dst = const_cast<float*>(planar_base(out, &planes));
  const float* res = add ? planar_base(*add, &aplanes) : nullptr;
  const int h = out.H, w = out.W, w2 = w / 2 + 1;
  MITB_CHECK(splanes == 2 * planes && spec.H == h && spec.W == w2, "irfft2 shape mismatch");
  MITB_CHECK(!add || (aplanes == planes && add->H == h && add->W == w), "irfft2 residual shape mismatch");
  FftPlan* pw = fft_plan_get(w); FftPlan* ph = fft_plan_get(h);
  const int P = pick_batch(w, 8, 8), CB = pick_batch(h, 8, 8);
  const int npairs = (h + 1) / 2;
  fft_trace(ph, pw, P, CB);
  ProfScope ps("fft_irfft2", 2.5 * planes * (double)h * w * log2((double)h * w),
               4.0 * planes * ((double)h * w * (add ? 2 : 1) + 2.0 * h * w2), st);
  fft_cols_kernel<<<dim3((w2 + CB - 1) / CB, planes), 256, (size_t)2 * CB * (h | 1) * sizeof(float2), st>>>(
      tmp, src, h, w2, CB, ph->dev, 1, 1.f);
  count_launch();
  irfft_rows_kernel<<<dim3((npairs + P - 1) / P, planes), 256, (size_t)2 * P * w * sizeof(float2), st>>>(
      tmp, dst, res, h, w, w2, P, pw->dev, (float)(1.0 / sqrt((double)h * (double)w)));
  count_launch();
  CUDA_OK(cudaGetLastError());
}

}  // namespace mitb
