// test_conv.cu — GPU self-test of the wgmma conv kernels against naive CUDA-core reference kernels
// (same bf16 inputs, fp32 accumulation). Run on an H100:  tests/native/bin/test_conv
// This is test infrastructure; the Python parity tests (tests/test_conv_gpu.py) compare against the oracle.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../include/opengenie_b200.h"

#define CK(x)                                                                          \
  do {                                                                                 \
    cudaError_t e = (x);                                                               \
    if (e != cudaSuccess) {                                                            \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__);   \
      exit(2);                                                                         \
    }                                                                                  \
  } while (0)

static void* g_ws = nullptr;
static size_t g_ws_bytes = 0;
static void* g_scratch = nullptr;       // weight-gradient split-K slabs
static size_t g_scratch_bytes = 0;
static uint32_t g_seed = 12345;
static float frand() {
  g_seed = g_seed * 1664525u + 1013904223u;
  return ((g_seed >> 8) & 0xFFFFFF) / float(0x1000000) * 2.f - 1.f;
}

__global__ void ref_fwd(const __nv_bfloat16* x0, int c0, int kt, int kh, int kw, int pt, int ph, int pw,
                        const __nv_bfloat16* x1, int c1, const __nv_bfloat16* w, int ldw, const float* b0,
                        const float* b1, float* out, int N, int T, int H, int W, int cout) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long total = (long long)N * T * H * W * cout;
  if (idx >= total) return;
  int co = idx % cout;
  long long v = idx / cout;
  int wv = v % W;
  int hv = (v / W) % H;
  int tv = (v / ((long long)W * H)) % T;
  int n = v / ((long long)W * H * T);
  float acc = 0.f;
  if (b0) acc += b0[co];
  if (b1) acc += b1[co];
  int tap = 0;
  for (int it = 0; it < kt; ++it)
    for (int ih = 0; ih < kh; ++ih)
      for (int iw = 0; iw < kw; ++iw, ++tap) {
        int t = tv + it - pt, h = hv + ih - ph, ww = wv + iw - pw;
        if (t < 0 || t >= T || h < 0 || h >= H || ww < 0 || ww >= W) continue;
        const __nv_bfloat16* xp = x0 + ((((long long)n * T + t) * H + h) * W + ww) * c0;
        const __nv_bfloat16* wp = w + (long long)co * ldw + (long long)tap * c0;
        for (int ci = 0; ci < c0; ++ci) acc += __bfloat162float(xp[ci]) * __bfloat162float(wp[ci]);
      }
  if (x1) {
    const __nv_bfloat16* xp = x1 + v * c1;
    const __nv_bfloat16* wp = w + (long long)co * ldw + (long long)kt * kh * kw * c0;
    for (int ci = 0; ci < c1; ++ci) acc += __bfloat162float(xp[ci]) * __bfloat162float(wp[ci]);
  }
  out[idx] = acc;
}

__global__ void ref_dgrad(const __nv_bfloat16* dy, int cout, const __nv_bfloat16* w, int ldw, int k_off, int kt,
                          int kh, int kw, int pt, int ph, int pw, float* dx, int N, int T, int H, int W, int cin) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long total = (long long)N * T * H * W * cin;
  if (idx >= total) return;
  int ci = idx % cin;
  long long v = idx / cin;
  int wv = v % W;
  int hv = (v / W) % H;
  int tv = (v / ((long long)W * H)) % T;
  int n = v / ((long long)W * H * T);
  float acc = 0.f;
  int tap = 0;
  for (int it = 0; it < kt; ++it)
    for (int ih = 0; ih < kh; ++ih)
      for (int iw = 0; iw < kw; ++iw, ++tap) {
        int t = tv - (it - pt), h = hv - (ih - ph), ww = wv - (iw - pw);
        if (t < 0 || t >= T || h < 0 || h >= H || ww < 0 || ww >= W) continue;
        const __nv_bfloat16* yp = dy + ((((long long)n * T + t) * H + h) * W + ww) * cout;
        for (int co = 0; co < cout; ++co)
          acc += __bfloat162float(yp[co]) * __bfloat162float(w[(long long)co * ldw + k_off + (long long)tap * cin + ci]);
      }
  dx[idx] = acc;
}

__global__ void ref_wgrad(const __nv_bfloat16* dy, int cout, const __nv_bfloat16* x, int cin, float* dw, int kt,
                          int kh, int kw, int pt, int ph, int pw, int N, int T, int H, int W) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  int ntaps = kt * kh * kw;
  long long total = (long long)cout * ntaps * cin;
  if (idx >= total) return;
  int ci = idx % cin;
  int tap = (idx / cin) % ntaps;
  int co = idx / ((long long)cin * ntaps);
  int it = tap / (kh * kw), ih = (tap / kw) % kh, iw = tap % kw;
  float acc = 0.f;
  for (int n = 0; n < N; ++n)
    for (int t = 0; t < T; ++t) {
      int ts = t + it - pt;
      if (ts < 0 || ts >= T) continue;
      for (int h = 0; h < H; ++h) {
        int hs = h + ih - ph;
        if (hs < 0 || hs >= H) continue;
        for (int ww = 0; ww < W; ++ww) {
          int ws = ww + iw - pw;
          if (ws < 0 || ws >= W) continue;
          acc += __bfloat162float(dy[((((long long)n * T + t) * H + h) * W + ww) * cout + co]) *
                 __bfloat162float(x[((((long long)n * T + ts) * H + hs) * W + ws) * cin + ci]);
        }
      }
    }
  dw[idx] = acc;
}

static __nv_bfloat16* dev_bf16(size_t n, float scale) {
  std::vector<__nv_bfloat16> h(n);
  for (size_t i = 0; i < n; ++i) h[i] = __float2bfloat16(frand() * scale);
  __nv_bfloat16* d;
  CK(cudaMalloc(&d, n * sizeof(__nv_bfloat16)));
  CK(cudaMemcpy(d, h.data(), n * sizeof(__nv_bfloat16), cudaMemcpyHostToDevice));
  return d;
}
static float* dev_f32(size_t n, float scale) {
  std::vector<float> h(n);
  for (size_t i = 0; i < n; ++i) h[i] = frand() * scale;
  float* d;
  CK(cudaMalloc(&d, n * sizeof(float)));
  CK(cudaMemcpy(d, h.data(), n * sizeof(float), cudaMemcpyHostToDevice));
  return d;
}

static bool compare(const char* name, const float* d_got, const float* d_ref, size_t n, float rtol, float atol) {
  std::vector<float> g(n), r(n);
  CK(cudaMemcpy(g.data(), d_got, n * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(r.data(), d_ref, n * 4, cudaMemcpyDeviceToHost));
  double max_abs = 0, max_ref = 0;
  size_t bad = 0, first_bad = 0;
  for (size_t i = 0; i < n; ++i) {
    double d = fabs((double)g[i] - r[i]);
    if (d > max_abs) max_abs = d;
    if (fabs(r[i]) > max_ref) max_ref = fabs(r[i]);
    if (!(d <= atol + rtol * fabs(r[i]))) {
      if (!bad) first_bad = i;
      ++bad;
    }
  }
  printf("  %-28s n=%zu max_abs_err=%.3e max|ref|=%.3e mismatches=%zu %s\n", name, n, max_abs, max_ref, bad,
         bad ? "FAIL" : "ok");
  if (bad) printf("    first mismatch at %zu: got %.6f ref %.6f\n", first_bad, g[first_bad], r[first_bad]);
  return bad == 0;
}

struct Case {
  int N, T, H, W, c0, c1, cout, kt, kh, kw, pt, ph, pw;
  bool bias;
};

static bool run_case(const Case& c, bool do_dgrad, bool do_wgrad) {
  printf("case N=%d T=%d H=%d W=%d c0=%d c1=%d cout=%d k=(%d,%d,%d) pad=(%d,%d,%d)\n", c.N, c.T, c.H, c.W, c.c0, c.c1,
         c.cout, c.kt, c.kh, c.kw, c.pt, c.ph, c.pw);
  bool ok = true;
  const long long V = (long long)c.N * c.T * c.H * c.W;
  const int ntaps = c.kt * c.kh * c.kw;
  const int ldw = ntaps * c.c0 + c.c1;
  __nv_bfloat16* x0 = dev_bf16(V * c.c0, 1.f);
  __nv_bfloat16* x1 = c.c1 ? dev_bf16(V * c.c1, 1.f) : nullptr;
  __nv_bfloat16* w = dev_bf16((size_t)c.cout * ldw, 0.05f);
  float* b0 = c.bias ? dev_f32(c.cout, 1.f) : nullptr;
  float* b1 = (c.bias && c.c1) ? dev_f32(c.cout, 1.f) : nullptr;
  float *out, *ref;
  CK(cudaMalloc(&out, V * c.cout * 4));
  CK(cudaMalloc(&ref, V * c.cout * 4));
  CK(cudaMemset(out, 0xFF, V * c.cout * 4));
  int r = og_conv3d_fwd(x0, c.c0, c.kt, c.kh, c.kw, c.pt, c.ph, c.pw, x1, c.c1, w, ldw, b0, b1, nullptr, out, 1, c.N, c.T, c.H,
                        c.W, c.cout, g_ws, g_ws_bytes, nullptr, 0);
  if (r != 0) {
    printf("  og_conv3d_fwd failed: %d %s\n", r, og_last_error());
    return false;
  }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    printf("  fwd kernel error: %s\n", cudaGetErrorString(e));
    exit(3);
  }
  {
    long long total = V * c.cout;
    ref_fwd<<<(unsigned)((total + 255) / 256), 256>>>(x0, c.c0, c.kt, c.kh, c.kw, c.pt, c.ph, c.pw, x1, c.c1, w, ldw,
                                                     b0, b1, ref, c.N, c.T, c.H, c.W, c.cout);
    CK(cudaDeviceSynchronize());
  }
  ok &= compare("fwd(fp32 out)", out, ref, V * c.cout, 1e-3f, 1e-3f);

  // bf16 output path
  {
    __nv_bfloat16* ob;
    CK(cudaMalloc(&ob, (V * c.cout + 64) * 2));
    CK(cudaMemset(ob, 0x7F, (V * c.cout + 64) * 2));
    r = og_conv3d_fwd(x0, c.c0, c.kt, c.kh, c.kw, c.pt, c.ph, c.pw, x1, c.c1, w, ldw, b0, b1, nullptr, ob, 0, c.N, c.T, c.H,
                      c.W, c.cout, g_ws, g_ws_bytes, nullptr, 0);
    CK(cudaDeviceSynchronize());
    std::vector<__nv_bfloat16> hb(V * c.cout + 64);
    std::vector<float> hr(V * c.cout);
    CK(cudaMemcpy(hb.data(), ob, hb.size() * 2, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(hr.data(), ref, V * c.cout * 4, cudaMemcpyDeviceToHost));
    size_t bad = 0;
    for (size_t i = 0; i < hr.size(); ++i) {
      float g = __bfloat162float(hb[i]);
      if (!(fabsf(g - hr[i]) <= 2e-3f + 8e-3f * fabsf(hr[i]))) ++bad;
    }
    for (size_t i = hr.size(); i < hb.size(); ++i)
      if (*reinterpret_cast<uint16_t*>(&hb[i]) != 0x7F7F) ++bad;  // wrote past the end
    printf("  %-28s mismatches=%zu %s\n", "fwd(bf16 out)", bad, bad ? "FAIL" : "ok");
    ok &= bad == 0;
    CK(cudaFree(ob));
  }

  if (do_dgrad && c.cout % 64 == 0) {
    __nv_bfloat16* dy = dev_bf16(V * c.cout, 1.f);
    float *dx, *dxr;
    CK(cudaMalloc(&dx, V * c.c0 * 4));
    CK(cudaMalloc(&dxr, V * c.c0 * 4));
    CK(cudaMemset(dx, 0xFF, V * c.c0 * 4));
    r = og_conv3d_dgrad(dy, c.cout, c.cout, w, ldw, 0, c.kt, c.kh, c.kw, c.pt, c.ph, c.pw, dx, 1, c.N, c.T, c.H, c.W,
                        c.c0, g_ws, g_ws_bytes, 0);
    if (r != 0) {
      printf("  og_conv3d_dgrad failed: %d %s\n", r, og_last_error());
      ok = false;
    } else {
      e = cudaDeviceSynchronize();
      if (e != cudaSuccess) {
        printf("  dgrad kernel error: %s\n", cudaGetErrorString(e));
        exit(3);
      }
      long long total = V * c.c0;
      ref_dgrad<<<(unsigned)((total + 255) / 256), 256>>>(dy, c.cout, w, ldw, 0, c.kt, c.kh, c.kw, c.pt, c.ph, c.pw,
                                                         dxr, c.N, c.T, c.H, c.W, c.c0);
      CK(cudaDeviceSynchronize());
      ok &= compare("dgrad(main segment)", dx, dxr, V * c.c0, 1e-3f, 1e-3f);
      // bf16 output (the product path): exercises the coalesced staged store, incl. partial last N tiles
      __nv_bfloat16* dxb;
      CK(cudaMalloc(&dxb, (V * c.c0 + 64) * 2));
      CK(cudaMemset(dxb, 0x7F, (V * c.c0 + 64) * 2));  // canary after the tensor
      r = og_conv3d_dgrad(dy, c.cout, c.cout, w, ldw, 0, c.kt, c.kh, c.kw, c.pt, c.ph, c.pw, dxb, 0, c.N, c.T, c.H, c.W,
                          c.c0, g_ws, g_ws_bytes, 0);
      CK(cudaDeviceSynchronize());
      std::vector<__nv_bfloat16> hb(V * c.c0 + 64);
      std::vector<float> hr(V * c.c0);
      CK(cudaMemcpy(hb.data(), dxb, hb.size() * 2, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(hr.data(), dxr, hr.size() * 4, cudaMemcpyDeviceToHost));
      size_t bad = 0;
      for (size_t i = 0; i < hr.size(); ++i)
        if (!(fabsf(__bfloat162float(hb[i]) - hr[i]) <= 2e-3f + 8e-3f * fabsf(hr[i]))) ++bad;
      for (size_t i = hr.size(); i < hb.size(); ++i)
        if (*reinterpret_cast<uint16_t*>(&hb[i]) != 0x7F7F) ++bad;  // wrote past the end
      printf("  %-28s mismatches=%zu %s\n", "dgrad(bf16 out + canary)", bad, bad ? "FAIL" : "ok");
      ok &= bad == 0;
      CK(cudaFree(dxb));
    }
    if (c.c1 && c.c1 % 64 == 0) {
      float *dx1, *dx1r;
      CK(cudaMalloc(&dx1, V * c.c1 * 4));
      CK(cudaMalloc(&dx1r, V * c.c1 * 4));
      r = og_conv3d_dgrad(dy, c.cout, c.cout, w, ldw, ntaps * c.c0, 1, 1, 1, 0, 0, 0, dx1, 1, c.N, c.T, c.H, c.W, c.c1, g_ws, g_ws_bytes, 0);
      if (r != 0) {
        printf("  og_conv3d_dgrad(shortcut) failed: %d %s\n", r, og_last_error());
        ok = false;
      } else {
        CK(cudaDeviceSynchronize());
        long long total = V * c.c1;
        ref_dgrad<<<(unsigned)((total + 255) / 256), 256>>>(dy, c.cout, w, ldw, ntaps * c.c0, 1, 1, 1, 0, 0, 0, dx1r,
                                                           c.N, c.T, c.H, c.W, c.c1);
        CK(cudaDeviceSynchronize());
        ok &= compare("dgrad(1x1x1 shortcut)", dx1, dx1r, V * c.c1, 1e-3f, 1e-3f);
      }
      CK(cudaFree(dx1));
      CK(cudaFree(dx1r));
    }
    if (do_wgrad && c.cout % 8 == 0) {
      float *dw, *dwr;
      size_t nw = (size_t)c.cout * ntaps * c.c0;
      CK(cudaMalloc(&dw, nw * 4));
      CK(cudaMalloc(&dwr, nw * 4));
      CK(cudaMemset(dw, 0, nw * 4));
      // weight gradient + bias gradient (column sums of dy) in one launch; og_colsum is the reference for the latter
      float *db, *dbr;
      CK(cudaMalloc(&db, c.cout * 4));
      CK(cudaMalloc(&dbr, c.cout * 4));
      CK(cudaMemset(db, 0, c.cout * 4));
      CK(cudaMemset(dbr, 0, c.cout * 4));
      r = og_conv3d_wgrad_bias(dy, c.cout, x0, c.c0, dw, (int64_t)ntaps * c.c0, c.kt, c.kh, c.kw, c.pt, c.ph, c.pw, c.N, c.T,
                               c.H, c.W, db, c.cout, g_scratch, g_scratch_bytes, 0);
      if (r == 0) r = og_colsum(dy, V, c.cout, c.cout, dbr, 0);
      if (r == 0) {
        CK(cudaDeviceSynchronize());
        ok &= compare("wgrad(bias gradient)", db, dbr, c.cout, 2e-3f, 5e-2f);
      }
      CK(cudaFree(db));
      CK(cudaFree(dbr));
      if (r != 0) {
        printf("  og_conv3d_wgrad failed: %d %s\n", r, og_last_error());
        ok = false;
      } else {
        e = cudaDeviceSynchronize();
        if (e != cudaSuccess) {
          printf("  wgrad kernel error: %s\n", cudaGetErrorString(e));
          exit(3);
        }
        ref_wgrad<<<(unsigned)((nw + 127) / 128), 128>>>(dy, c.cout, x0, c.c0, dwr, c.kt, c.kh, c.kw, c.pt, c.ph, c.pw,
                                                        c.N, c.T, c.H, c.W);
        CK(cudaDeviceSynchronize());
        // sums over up to ~1e4 voxels of O(1) products: scale tolerance with the magnitude
        ok &= compare("wgrad", dw, dwr, nw, 2e-3f, 5e-2f);
      }
      CK(cudaFree(dw));
      CK(cudaFree(dwr));
    }
    CK(cudaFree(dy));
    CK(cudaFree(dx));
    CK(cudaFree(dxr));
  }
  CK(cudaFree(x0));
  if (x1) CK(cudaFree(x1));
  CK(cudaFree(w));
  if (b0) CK(cudaFree(b0));
  if (b1) CK(cudaFree(b1));
  CK(cudaFree(out));
  CK(cudaFree(ref));
  return ok;
}

static void bench_case(const Case& c, int iters) {
  const long long V = (long long)c.N * c.T * c.H * c.W;
  const int ntaps = c.kt * c.kh * c.kw;
  const int ldw = ntaps * c.c0 + c.c1;
  __nv_bfloat16* x0 = dev_bf16(V * c.c0, 1.f);
  __nv_bfloat16* w = dev_bf16((size_t)c.cout * ldw, 0.05f);
  __nv_bfloat16* out;
  CK(cudaMalloc(&out, V * c.cout * 2));
  __nv_bfloat16* dy = dev_bf16(V * c.cout, 1.f);
  __nv_bfloat16* dx;
  CK(cudaMalloc(&dx, V * c.c0 * 2));
  float* dw;
  CK(cudaMalloc(&dw, (size_t)c.cout * ntaps * c.c0 * 4));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  double flop = 2.0 * V * c.cout * ntaps * c.c0;
  for (int which = 0; which < 3; ++which) {
    for (int i = 0; i < iters + 2; ++i) {
      if (i == 2) CK(cudaEventRecord(e0));
      int r = 0;
      if (which == 0)
        r = og_conv3d_fwd(x0, c.c0, c.kt, c.kh, c.kw, c.pt, c.ph, c.pw, nullptr, 0, w, ldw, nullptr, nullptr, nullptr, out, 0,
                          c.N, c.T, c.H, c.W, c.cout, g_ws, g_ws_bytes, nullptr, 0);
      else if (which == 1)
        r = og_conv3d_dgrad(dy, c.cout, c.cout, w, ldw, 0, c.kt, c.kh, c.kw, c.pt, c.ph, c.pw, dx, 0, c.N, c.T, c.H,
                            c.W, c.c0, g_ws, g_ws_bytes, 0);
      else
        r = og_conv3d_wgrad(dy, c.cout, x0, c.c0, dw, (int64_t)ntaps * c.c0, c.kt, c.kh, c.kw, c.pt, c.ph, c.pw, c.N,
                            c.T, c.H, c.W, g_scratch, g_scratch_bytes, 0);
      if (r) {
        printf("bench launch failed: %s\n", og_last_error());
        return;
      }
    }
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    ms /= iters;
    printf("bench %-5s N=%d %dx%dx%d c=%d->%d k=%d: %.3f ms  %.1f TFLOP/s\n",
           which == 0 ? "fwd" : which == 1 ? "dgrad" : "wgrad", c.N, c.T, c.H, c.W, c.c0, c.cout, c.kt, ms,
           flop / ms * 1e-9);
  }
  CK(cudaFree(x0)); CK(cudaFree(w)); CK(cudaFree(out)); CK(cudaFree(dy)); CK(cudaFree(dx)); CK(cudaFree(dw));
}

int main(int argc, char** argv) {
  int dev_count = 0;
  CK(cudaGetDeviceCount(&dev_count));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  printf("device: %s sm_%d%d SMs=%d\n", prop.name, prop.major, prop.minor, prop.multiProcessorCount);
  g_ws_bytes = (size_t)256 << 20;
  CK(cudaMalloc(&g_ws, g_ws_bytes));
  g_scratch_bytes = (size_t)64 << 20;
  CK(cudaMalloc(&g_scratch, g_scratch_bytes));
  bool quick = argc > 1 && !strcmp(argv[1], "quick");
  std::vector<Case> cases = {
      // N  T  H   W   c0   c1  cout kt kh kw pt ph pw bias
      {1, 2, 8, 8, 64, 0, 64, 1, 1, 1, 0, 0, 0, false},      // smallest: pure GEMM, 1 tile
      {1, 2, 8, 8, 64, 0, 64, 3, 3, 3, 1, 1, 1, false},      // 3x3x3 symmetric, halo entirely by OOB fill
      {2, 4, 16, 16, 128, 0, 128, 3, 3, 3, 1, 1, 1, true},   // multi-tile, 2 k-blocks per tap
      {2, 4, 16, 16, 128, 0, 128, 3, 3, 3, 2, 1, 1, true},   // causal time padding (front only)
      {2, 4, 16, 16, 128, 64, 256, 3, 3, 3, 1, 1, 1, true},  // fused 1x1x1 shortcut segment, N tile 256
      {1, 4, 8, 8, 512, 0, 512, 3, 3, 3, 1, 1, 1, false},    // deep K, small M (N tile shrinks)
      {2, 2, 16, 16, 64, 0, 18, 1, 1, 1, 0, 0, 0, true},     // Cout=18 (encoder head): masked scalar epilogue
      {1, 2, 64, 64, 128, 0, 3, 3, 3, 3, 2, 1, 1, true},     // Cout=3 (decoder tail), W=64 box
      {1, 4, 32, 32, 256, 0, 1024, 3, 3, 3, 2, 1, 1, true},  // up-conv shape (N heavy)
      {2, 8, 32, 32, 64, 0, 64, 1, 1, 1, 0, 0, 0, true},     // 1x1x1, many short tiles (2 k-blocks): epilogue-bound
      {1, 1, 1, 16384, 128, 0, 64, 1, 1, 1, 0, 0, 0, true},  // flattened im2col GEMM view (1,1,1,M)
      {1, 1, 1, 4100, 128, 0, 64, 1, 1, 1, 0, 0, 0, false},  // M not a multiple of the tile: partial boxes
      {3, 4, 8, 8, 64, 0, 128, 3, 3, 3, 1, 1, 1, true},      // odd batch with 2-row-block tiles
      {1, 2, 16, 16, 64, 0, 320, 1, 1, 1, 0, 0, 0, true},    // Cout = 320: partial last 128-wide N tile, bf16 fast store
      {8, 16, 64, 64, 64, 64, 64, 3, 3, 3, 1, 1, 1, true},   // full tokenizer size: many persistent tiles per CTA
  };
  bool all_ok = true;
  const bool bench_only = argc > 1 && !strcmp(argv[1], "benchonly");
  for (size_t i = 0; i < cases.size() && !bench_only; ++i) {
    if (quick && i > 3) break;
    all_ok &= run_case(cases[i], true, true);
  }
  printf("RESULT: %s\n", all_ok ? "ALL PASS" : "FAILURES");
  if (bench_only) {
    const int it = argc > 2 ? atoi(argv[2]) : 1;
    const int which = argc > 3 ? atoi(argv[3]) : 0;
    if (which == 0 || which == 1) bench_case({8, 16, 64, 64, 128, 0, 128, 3, 3, 3, 1, 1, 1, false}, it);
    if (which == 0 || which == 2) bench_case({8, 4, 8, 8, 512, 0, 512, 3, 3, 3, 1, 1, 1, false}, it);
    if (which == 3) bench_case({8, 8, 16, 16, 256, 0, 256, 3, 3, 3, 1, 1, 1, false}, it);
  }
  if (argc > 1 && !strcmp(argv[1], "bench")) {
    bench_case({8, 16, 64, 64, 128, 0, 128, 3, 3, 3, 1, 1, 1, false}, 5);
    bench_case({8, 16, 32, 32, 256, 0, 256, 3, 3, 3, 1, 1, 1, false}, 5);
    bench_case({8, 8, 16, 16, 256, 0, 256, 3, 3, 3, 1, 1, 1, false}, 10);
    bench_case({8, 4, 8, 8, 512, 0, 512, 3, 3, 3, 1, 1, 1, false}, 10);
    bench_case({8, 16, 32, 32, 256, 0, 1024, 3, 3, 3, 2, 1, 1, false}, 5);
  }
  return all_ok ? 0 : 1;
}
