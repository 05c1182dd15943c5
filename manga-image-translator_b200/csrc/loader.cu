// Load-time weight preparation: PyTorch state_dict tensors (device pointers) -> kernel layouts.
//   Conv2d          [Cout,Cin,kh,kw]  -> K-major [(tap,cin)][Cout padded to 4], taps row-major
//   ConvTranspose2d [Cin,Cout,k,k] s2 -> one K-major sub-kernel per output phase (py,px)
//   BatchNorm (eval)                  -> per-channel scale/shift
#include <math.h>
#include "mitb_internal.h"

namespace mitb {

static int round4(int x) { return (x + 3) & ~3; }

ConvW Loader::conv(const std::string& wname, int pad_y, int pad_x) {
  return conv_cat_cin({wname}, pad_y, pad_x);
}

ConvW Loader::conv_cat_cin(const std::vector<std::string>& wnames, int pad_y, int pad_x) {
  const mitb_tensor& t0 = W.get(wnames[0]);
  MITB_CHECK(t0.ndim == 4 || t0.ndim == 2, "%s: expected a conv/linear weight", wnames[0].c_str());
  const int Cout = (int)t0.shape[0];
  const int kh = t0.ndim == 4 ? (int)t0.shape[2] : 1, kw = t0.ndim == 4 ? (int)t0.shape[3] : 1;
  int Cin = 0;
  for (auto& nm : wnames) {
    const mitb_tensor& t = W.get(nm);
    MITB_CHECK((int)t.shape[0] == Cout && (t.ndim == 2 || ((int)t.shape[2] == kh && (int)t.shape[3] == kw)),
               "%s: incompatible with %s", nm.c_str(), wnames[0].c_str());
    Cin += (int)t.shape[1];
  }
  ConvW cw; cw.Cin = Cin; cw.Cout = Cout; cw.ntaps = kh * kw; cw.ldw = round4(Cout);
  MITB_CHECK(cw.ntaps <= kMaxTaps, "%s: kernel too large", wnames[0].c_str());
  std::vector<int> ky(cw.ntaps), kx(cw.ntaps);
  for (int t = 0; t < cw.ntaps; ++t) { ky[t] = t / kw; kx[t] = t % kw; cw.tdy[t] = (int8_t)(ky[t] - pad_y); cw.tdx[t] = (int8_t)(kx[t] - pad_x); }
  float* dst = blob.alloc_f((size_t)cw.ntaps * Cin * cw.ldw);
  // each source occupies a channel range [c0, c0+ci) of every tap: repack tap by tap
  int c0 = 0;
  if (wnames.size() == 1) {
    launch_repack(dst, t0.data, Cout, Cin, cw.ntaps, ky.data(), kx.data(), (long)Cin * kh * kw, (long)kh * kw, kw, 1, cw.ldw, st);
    cw.w = dst;
    conv_tc_prepare(cw, blob, st);
    return cw;
  }
  for (auto& nm : wnames) {
    const mitb_tensor& t = W.get(nm);
    const int ci = (int)t.shape[1];
    for (int tp = 0; tp < cw.ntaps; ++tp) {
      int one_ky = ky[tp], one_kx = kx[tp];
      launch_repack(dst + ((size_t)tp * Cin + c0) * cw.ldw, t.data, Cout, ci, 1, &one_ky, &one_kx,
                    (long)ci * kh * kw, (long)kh * kw, kw, 1, cw.ldw, st);
    }
    c0 += ci;
  }
  cw.w = dst;
  conv_tc_prepare(cw, blob, st);
  return cw;
}

// ConvTranspose2d stride 2: y = 2*i - pad + ky.  For output parity py, contributing ky satisfy (py + pad - ky) even;
// input offset dy = (py + pad - ky)/2 relative to i0 = floor(y/2).
ConvW Loader::convT_phase(const std::string& wname, int k, int pad, int py, int px) {
  const mitb_tensor& t = W.get(wname);
  MITB_CHECK(t.ndim == 4 && (int)t.shape[2] == k && (int)t.shape[3] == k, "%s: expected [Cin,Cout,%d,%d]", wname.c_str(), k, k);
  const int Cin = (int)t.shape[0], Cout = (int)t.shape[1];
  ConvW cw; cw.Cin = Cin; cw.Cout = Cout; cw.ldw = round4(Cout); cw.ntaps = 0;
  std::vector<int> ky, kx;
  for (int a = 0; a < k; ++a) {
    if (((py + pad - a) & 1) != 0) continue;
    for (int b = 0; b < k; ++b) {
      if (((px + pad - b) & 1) != 0) continue;
      ky.push_back(a); kx.push_back(b);
      cw.tdy[cw.ntaps] = (int8_t)((py + pad - a) / 2); cw.tdx[cw.ntaps] = (int8_t)((px + pad - b) / 2);
      ++cw.ntaps;
    }
  }
  MITB_CHECK(cw.ntaps > 0, "%s: empty transposed-conv phase", wname.c_str());
  float* dst = blob.alloc_f((size_t)cw.ntaps * Cin * cw.ldw);
  // src index: ci*(Cout*k*k) + co*(k*k) + ky*k + kx
  launch_repack(dst, t.data, Cout, Cin, cw.ntaps, ky.data(), kx.data(), (long)k * k, (long)Cout * k * k, k, 1, cw.ldw, st);
  cw.w = dst;
  conv_tc_prepare(cw, blob, st);
  return cw;
}

ConvW Loader::linear_rows(const std::string& wname, int r0, int nr) {
  const mitb_tensor& t = W.get(wname);
  MITB_CHECK(t.ndim == 2 && r0 + nr <= (int)t.shape[0], "%s: bad row slice", wname.c_str());
  const int Cin = (int)t.shape[1];
  ConvW cw; cw.Cin = Cin; cw.Cout = nr; cw.ntaps = 1; cw.ldw = round4(nr);
  float* dst = blob.alloc_f((size_t)Cin * cw.ldw);
  int z = 0;
  launch_repack(dst, t.data + (size_t)r0 * Cin, nr, Cin, 1, &z, &z, Cin, 1, 0, 0, cw.ldw, st);
  cw.w = dst;
  conv_tc_prepare(cw, blob, st);
  return cw;
}

const float* Loader::vec_slice(const std::string& name, int off, int n) {
  const mitb_tensor& t = W.get(name);
  float* d = blob.alloc_f(n + 4);
  CUDA_OK(cudaMemcpyAsync(d, t.data + off, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return d;
}

ConvW Loader::conv_padcin(const std::string& wname, int pad, int cin_pad) {
  const mitb_tensor& t = W.get(wname);
  MITB_CHECK(t.ndim == 4 && (int)t.shape[1] <= cin_pad, "%s: cannot pad input channels to %d", wname.c_str(), cin_pad);
  const int Cout = (int)t.shape[0], ci = (int)t.shape[1], kh = (int)t.shape[2], kw = (int)t.shape[3];
  ConvW cw; cw.Cin = cin_pad; cw.Cout = Cout; cw.ntaps = kh * kw; cw.ldw = round4(Cout);
  MITB_CHECK(cw.ntaps <= kMaxTaps, "%s: kernel too large", wname.c_str());
  float* dst = blob.alloc_f((size_t)cw.ntaps * cin_pad * cw.ldw);
  CUDA_OK(cudaMemsetAsync(dst, 0, sizeof(float) * cw.ntaps * cin_pad * cw.ldw, st));
  for (int tp = 0; tp < cw.ntaps; ++tp) {
    int ky = tp / kw, kx = tp % kw;
    cw.tdy[tp] = (int8_t)(ky - pad); cw.tdx[tp] = (int8_t)(kx - pad);
    launch_repack(dst + (size_t)tp * cin_pad * cw.ldw, t.data, Cout, ci, 1, &ky, &kx, (long)ci * kh * kw, (long)kh * kw, kw, 1, cw.ldw, st);
  }
  cw.w = dst;
  conv_tc_prepare(cw, blob, st);
  return cw;
}

ConvW Loader::cat_k(const ConvW& a, const ConvW& b) {
  MITB_CHECK(a.Cout == b.Cout && a.ldw == b.ldw && a.Cin % 64 == 0 && b.Cin % 64 == 0, "cat_k: incompatible weights");
  const int Ka = a.ntaps * a.Cin, Kb = b.ntaps * b.Cin;
  ConvW cw; cw.Cin = Ka + Kb; cw.Cout = a.Cout; cw.ntaps = 1; cw.ldw = a.ldw;
  float* dst = blob.alloc_f((size_t)(Ka + Kb) * cw.ldw);
  CUDA_OK(cudaMemcpyAsync(dst, a.w, (size_t)Ka * cw.ldw * sizeof(float), cudaMemcpyDeviceToDevice, st));
  CUDA_OK(cudaMemcpyAsync(dst + (size_t)Ka * cw.ldw, b.w, (size_t)Kb * cw.ldw * sizeof(float), cudaMemcpyDeviceToDevice, st));
  cw.w = dst;
  conv_tc_prepare(cw, blob, st);
  return cw;
}

const float* Loader::vec(const std::string& name) { return vec_tiled(name, 1); }

const float* Loader::vec_tiled(const std::string& name, int reps) {
  const mitb_tensor& t = W.get(name);
  size_t n = 1; for (int i = 0; i < t.ndim; ++i) n *= (size_t)t.shape[i];
  float* d = blob.alloc_f(n * reps + 4);
  for (int r = 0; r < reps; ++r) CUDA_OK(cudaMemcpyAsync(d + n * r, t.data, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return d;
}

void Loader::bn_fold(const std::string& p, float eps, const float** scale, const float** shift) {
  const mitb_tensor& tw = W.get(p + "weight");
  const int C = (int)tw.shape[0];
  std::vector<float> w(C), b(C), m(C), v(C), sc(C), sh(C);
  CUDA_OK(cudaMemcpy(w.data(), tw.data, C * sizeof(float), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(b.data(), W.get(p + "bias").data, C * sizeof(float), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(m.data(), W.get(p + "running_mean").data, C * sizeof(float), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(v.data(), W.get(p + "running_var").data, C * sizeof(float), cudaMemcpyDeviceToHost));
  for (int i = 0; i < C; ++i) {
    const double s = (double)w[i] / sqrt((double)v[i] + (double)eps);
    sc[i] = (float)s; sh[i] = (float)((double)b[i] - (double)m[i] * s);
  }
  float* ds = blob.alloc_f(C + 4); float* dh = blob.alloc_f(C + 4);
  CUDA_OK(cudaMemcpy(ds, sc.data(), C * sizeof(float), cudaMemcpyHostToDevice));
  CUDA_OK(cudaMemcpy(dh, sh.data(), C * sizeof(float), cudaMemcpyHostToDevice));
  *scale = ds; *shift = dh;
}

ConvW Loader::conv_bn(const std::string& wname, const std::string& p, int pad, float eps) {
  const mitb_tensor& t = W.get(wname);
  MITB_CHECK(t.ndim == 4, "%s: expected a Conv2d weight", wname.c_str());
  const int Cout = (int)t.shape[0], Cin = (int)t.shape[1], kh = (int)t.shape[2], kw = (int)t.shape[3];
  ConvW cw; cw.Cin = Cin; cw.Cout = Cout; cw.ntaps = kh * kw; cw.ldw = round4(Cout);
  MITB_CHECK(cw.ntaps <= kMaxTaps, "%s: kernel too large", wname.c_str());
  MITB_CHECK((int)W.get(p + "weight").shape[0] == Cout, "%s: BatchNorm has the wrong channel count", p.c_str());
  std::vector<int> ky(cw.ntaps), kx(cw.ntaps);
  for (int i = 0; i < cw.ntaps; ++i) { ky[i] = i / kw; kx[i] = i % kw; cw.tdy[i] = (int8_t)(ky[i] - pad); cw.tdx[i] = (int8_t)(kx[i] - pad); }
  const size_t n = (size_t)cw.ntaps * Cin * cw.ldw;
  float* dst = blob.alloc_f(n);
  launch_repack(dst, t.data, Cout, Cin, cw.ntaps, ky.data(), kx.data(), (long)Cin * kh * kw, (long)kh * kw, kw, 1, cw.ldw, st);
  const float* dscale; const float* dshift;
  bn_fold(p, eps, &dscale, &dshift);
  std::vector<float> sc(Cout), w(n);
  CUDA_OK(cudaStreamSynchronize(st));
  CUDA_OK(cudaMemcpy(sc.data(), dscale, Cout * sizeof(float), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(w.data(), dst, n * sizeof(float), cudaMemcpyDeviceToHost));
  for (size_t r = 0; r < n / cw.ldw; ++r)
    for (int co = 0; co < Cout; ++co) w[r * cw.ldw + co] *= sc[co];
  CUDA_OK(cudaMemcpy(dst, w.data(), n * sizeof(float), cudaMemcpyHostToDevice));
  cw.w = dst; cw.shift = dshift;
  conv_tc_prepare(cw, blob, st);
  return cw;
}

float Loader::scalar(const std::string& name) {
  float v = 0.f;
  CUDA_OK(cudaMemcpy(&v, W.get(name).data, sizeof(float), cudaMemcpyDeviceToHost));
  return v;
}

void Ctx::ensure_ws(size_t bytes) {
  if (bytes <= ws.cap) return;
  if (ws.base) CUDA_OK(cudaFree(ws.base));
  ws.base = nullptr; ws.cap = 0;
  const size_t want = bytes + (bytes >> 4) + (1 << 20);
  void* p = nullptr;
  CUDA_OK(cudaMalloc(&p, want));
  ws.base = (char*)p; ws.cap = want;
}

}  // namespace mitb
