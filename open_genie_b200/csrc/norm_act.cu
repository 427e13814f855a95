// norm_act.cu — GroupNorm / AdaptiveGroupNorm + activation on NDHWC bf16 tensors, forward and backward.
//
// These are HBM-bound passes (SURVEY.md §8d: 2+2 bytes per element), so the design is about traffic:
//   * statistics: ONE read of x  -> per-(sample, group) sum / sum-of-squares (fp32 partials, fp64 combine)
//   * apply     : one read + one write; the whole GN / AdaGN / affine / SiLU chain is folded into a
//                 per-(sample, channel) scale A and shift B:
//                     y = act(x * A[n][c] + B[n][c])
//                 A = rstd * gamma * s,  B = (beta - mean * rstd * gamma) * s + a        (s, a: AdaGN)
//                 (og_gn_act_fwd derives A, B inside the apply launch; og_gn_finalize + og_affine_act_fwd are
//                 the two-launch form kept for (C/G) % 8 != 0)
//   * backward  : one reduce pass (dy, x) -> per-(n,c) sums, then one apply pass
//                     dx = P[n][c] * dpre + Q[n][c] * x + R[n][c]  (+ add)
//                 whose prologue turns the sums into P, Q, R and the parameter gradients (og_gn_act_bwd)
//
// Replaces F.group_norm / nn.GroupNorm + nn.SiLU (genie/module/video.py:607-608,622-623, blueprint
// 'group_norm'+'silu' tokenizer.py:75-79,163-167), AdaptiveGroupNorm.forward (genie/module/norm.py:55-69)
// and the GroupNorm of the ST-block FFN (genie/module/misc.py:93), plus their autograd backward.
#include "og_host.cuh"
#include "og_ptx.cuh"

namespace og {
extern std::atomic<uint64_t> g_launches;

// sigmoid through the hardware tanh (one MUFU op instead of ex2 + an IEEE divide): these passes run at
// ~1.6 T elements/s when HBM-bound, which leaves ~20 issue slots per element — the exp/divide form alone used half.
// tanh.approx.f32 is documented to about 2^-11 relative error, so sigmoid is within 2^-12 and SiLU within |x| 2^-12
// (absolute): inside the bf16 rounding at the scale of the tensors these kernels write, but not per element in the
// negative tail. Measured on an H100 over every bf16 input in [-40, 40] (tests/test_gpu_norm_act_paths.py), SiLU and its
// derivative are within 0.82 bf16 ulps of the exact value for x >= -8 and 2.4 ulps for -12 <= x < -8; below -12, where
// |silu(x)| < 7.4e-5, the relative error reaches 100 % (up to 256 ulps), an absolute error below 1e-4.
__device__ __forceinline__ float sigmoid_f(float x) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * x));
  return fmaf(t, 0.5f, 0.5f);
}
__device__ __forceinline__ float tanh_fast(float x) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(x));
  return t;
}
// With h = pre/2 and t = tanh(h):  silu(pre) = h (1 + t),  silu'(pre) = (1 + w)/2 with w = t + h (1 - t^2).
// The hot loops fold the 1/2 into the per-channel scale/shift (h = x*A/2 + B/2) and into the output scale, which
// leaves 3 operations per element forward and 5 backward around the single MUFU op.
__device__ __forceinline__ float silu_from_half(float h) { return fmaf(h, tanh_fast(h), h); }
__device__ __forceinline__ float silu_grad2_from_half(float h) {  // 2 * silu'(2h) - 1  (= w above)
  const float t = tanh_fast(h);
  return fmaf(h, fmaf(-t, t, 1.f), t);
}
__device__ __forceinline__ float silu_f(float x) { return x * sigmoid_f(x); }
__device__ __forceinline__ float silu_grad_f(float x) {
  const float s = sigmoid_f(x);
  return s * fmaf(x, 1.f - s, 1.f);
}

// Activation codes shared by every pass: 0 identity, 1 SiLU, 2 LeakyReLU(0.01) (nn.LeakyReLU() of the discriminators,
// genie/module/image.py:124-137, discriminator.py:97), 3 ReLU (VGG16 features of the perceptual loss, loss.py:46).
// SiLU passes work on h = pre/2 (coefficients pre-halved by the caller, see above); the others on pre itself.
static constexpr float kLeakySlope = 0.01f;
__device__ __forceinline__ float act_fwd_val(float v, int act) {   // v = h for SiLU, pre otherwise
  if (act == 1) return silu_from_half(v);
  if (act == 2) return v > 0.f ? v : kLeakySlope * v;
  if (act == 3) return fmaxf(v, 0.f);
  return v;
}
// e such that dpre = e * (act == 1 ? 1/2 : 1): SiLU returns 2*dpre (its callers fold the 1/2 into the coefficients)
__device__ __forceinline__ float act_bwd_e(float d, float v, int act) {
  if (act == 1) return fmaf(d, silu_grad2_from_half(v), d);
  if (act == 2) return v > 0.f ? d : kLeakySlope * d;
  if (act == 3) return v > 0.f ? d : 0.f;
  return d;
}

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]);
  u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]);
  u.w = pack_bf16x2(f[6], f[7]);
  return u;
}

// ------------------------------------------------------------------------------------------------
// statistics: grid (chunks, N); block 256. Thread -> (channel vector cv, row lane rl).
// ------------------------------------------------------------------------------------------------
static constexpr int kStatRows = 16;  // granularity of the row ranges handed to a block. (It was 256: the 512-channel
// 4x8x8 stage has V = 256 rows per sample, i.e. ONE block per sample = 8 CTAs on 132 SMs, each walking 64 dependent
// iterations — 62 such launches per pass made the low-resolution stages cost as much as the 16x64x64 ones.)

// grid (blocks_per_sample, N); each block owns a contiguous row range of one sample and keeps fp32 partial
// sums in registers over the whole range (4 independent 16-byte loads in flight per thread), then one
// shared-memory and one global fp64 atomic per group.
__global__ void __launch_bounds__(256, 6) og_gn_stats_kernel(const uint4* __restrict__ x, long long V, int C, int G,
                                                          long long rows_per_block, double* __restrict__ sums) {
  const int cvs = C >> 3;  // channel vectors per row (host guarantees cvs <= 256)
  const int n = blockIdx.y;
  const long long r_begin = (long long)blockIdx.x * rows_per_block;
  const long long r_end = (r_begin + rows_per_block < V) ? r_begin + rows_per_block : V;
  __shared__ double sh[64 * 2];
  for (int i = threadIdx.x; i < 2 * G; i += 256) sh[i] = 0.0;
  __syncthreads();
  const int lanes = 256 / cvs;
  const int cv = threadIdx.x % cvs, rl = threadIdx.x / cvs;
  float ts = 0.f, tss = 0.f;
  if (rl < lanes && r_begin < V) {
    const uint4* base = x + (long long)n * V * cvs + cv;
    float s = 0.f, ss = 0.f;
    long long r = r_begin + rl;
    for (; r + 7LL * lanes < r_end; r += 8LL * lanes) {
      uint4 u[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) u[k] = __ldg(base + (r + (long long)k * lanes) * cvs);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        float f[8];
        unpack8(u[k], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          s += f[i];
          ss = fmaf(f[i], f[i], ss);
        }
      }
    }
    for (; r < r_end; r += lanes) {
      float f[8];
      unpack8(__ldg(base + r * cvs), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s += f[i];
        ss = fmaf(f[i], f[i], ss);
      }
    }
    if (G > 1) {
      const int g = (cv * 8) / (C / G);
      atomicAdd(&sh[2 * g], (double)s);
      atomicAdd(&sh[2 * g + 1], (double)ss);
    } else {
      ts = s;
      tss = ss;
    }
  }
  if (G == 1) {
    // one group: shuffle-reduce per warp, 8 partials per block (256 threads hammering one shared fp64 atomic
    // serialise into a CAS loop that costs more than the whole streaming pass)
    double ds = (double)ts, dss = (double)tss;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      ds += __shfl_xor_sync(0xffffffffu, ds, off);
      dss += __shfl_xor_sync(0xffffffffu, dss, off);
    }
    if ((threadIdx.x & 31) == 0) {
      atomicAdd(&sh[0], ds);
      atomicAdd(&sh[1], dss);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * G; i += 256) atomicAdd(&sums[(long long)n * G * 2 + i], sh[i]);
}

// (C/G) % 8 != 0 (GroupNorm(16, 64), GroupNorm(32, 96), ...): an 8-channel vector may span groups, so every thread keeps
// fp32 partials per channel and adds each channel into its own group's shared fp64 sums. Same grid and thread mapping
// as og_gn_stats_kernel; a separate kernel so that the one the product's (C/G) % 8 == 0 layers run stays as it is.
__global__ void __launch_bounds__(256) og_gn_stats_split_kernel(const uint4* __restrict__ x, long long V, int C, int G,
                                                                long long rows_per_block, double* __restrict__ sums) {
  const int cvs = C >> 3;  // host guarantees cvs <= 256
  const int n = blockIdx.y;
  const long long r_begin = (long long)blockIdx.x * rows_per_block;
  const long long r_end = (r_begin + rows_per_block < V) ? r_begin + rows_per_block : V;
  __shared__ double sh[64 * 2];
  for (int i = threadIdx.x; i < 2 * G; i += 256) sh[i] = 0.0;
  __syncthreads();
  const int lanes = 256 / cvs;
  const int cv = threadIdx.x % cvs, rl = threadIdx.x / cvs;
  if (rl < lanes && r_begin < V) {
    const uint4* base = x + (long long)n * V * cvs + cv;
    float s[8] = {0, 0, 0, 0, 0, 0, 0, 0}, ss[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (long long r = r_begin + rl; r < r_end; r += lanes) {
      float f[8];
      unpack8(__ldg(base + r * cvs), f);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        s[k] += f[k];
        ss[k] = fmaf(f[k], f[k], ss[k]);
      }
    }
    const int cpg = C / G;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int g = (cv * 8 + k) / cpg;
      atomicAdd(&sh[2 * g], (double)s[k]);
      atomicAdd(&sh[2 * g + 1], (double)ss[k]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * G; i += 256) atomicAdd(&sums[(long long)n * G * 2 + i], sh[i]);
}

// finalize: one thread per (n, c)
__global__ void og_gn_finalize_kernel(const double* __restrict__ sums, int N, int C, int G, double inv_count, float eps,
                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                      const float* __restrict__ cond_scale, const float* __restrict__ cond_shift,
                                      float* __restrict__ A, float* __restrict__ B, float* __restrict__ mean_rstd) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * C) return;
  const int n = idx / C, c = idx - n * C;
  const int g = c / (C / G);
  const double s = sums[((long long)n * G + g) * 2], ss = sums[((long long)n * G + g) * 2 + 1];
  const double mean = s * inv_count;
  double var = ss * inv_count - mean * mean;
  if (var < 0) var = 0;
  const float rstd = (float)(1.0 / sqrt(var + (double)eps));
  const float mu = (float)mean;
  const float ga = gamma ? gamma[c] : 1.f, be = beta ? beta[c] : 0.f;
  float a = rstd * ga;
  float b = be - mu * rstd * ga;
  if (cond_scale) {
    const float sc = cond_scale[idx];
    a *= sc;
    b *= sc;
  }
  if (cond_shift) b += cond_shift[idx];
  A[idx] = a;
  B[idx] = b;
  if (c == g * (C / G)) {
    mean_rstd[((long long)n * G + g) * 2] = mu;
    mean_rstd[((long long)n * G + g) * 2 + 1] = rstd;
  }
}

// ------------------------------------------------------------------------------------------------
// apply: y = act(x*A + B). grid-stride over 8-channel vectors.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) og_affine_act_fwd_kernel(const uint4* __restrict__ x, const float* __restrict__ A,
                                                                const float* __restrict__ B, uint4* __restrict__ y,
                                                                long long V, int C, long long total_vec, int act) {
  const int cvs = C >> 3;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total_vec;
       i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % cvs);
    const long long row = i / cvs;
    const int n = (int)(row / V);
    const float4* a4 = reinterpret_cast<const float4*>(A + (long long)n * C + cv * 8);
    const float4* b4 = reinterpret_cast<const float4*>(B + (long long)n * C + cv * 8);
    const float4 a0 = __ldg(a4), a1 = __ldg(a4 + 1), b0 = __ldg(b4), b1 = __ldg(b4 + 1);
    const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    float f[8];
    unpack8(__ldg(x + i), f);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float pre = fmaf(f[k], av[k], bv[k]);
      f[k] = act == 1 ? silu_f(pre) : act_fwd_val(pre, act);
    }
    y[i] = pack8(f);
  }
}

// ------------------------------------------------------------------------------------------------
// GELU (nn.GELU(), exact erf form) of the SpaceTimeAttention FFN's hidden layers: a = GELU(u), du = da * GELU'(u).
// Flat grid-stride over 8-element vectors. Phi(u) is taken as erfc(-u/sqrt 2)/2, which keeps its relative accuracy in
// the negative tail: u * Phi(u) stays exact to a few fp32 ulps until it underflows (to -0 below u ~ -14).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float gelu_cdf(float u) { return 0.5f * erfcf(-0.70710678118654752f * u); }

__global__ void __launch_bounds__(256) og_gelu_fwd_kernel(const uint4* __restrict__ u, uint4* __restrict__ a,
                                                          long long nvec) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * blockDim.x) {
    float f[8];
    unpack8(__ldg(u + i), f);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = f[k] * gelu_cdf(f[k]);
    a[i] = pack8(f);
  }
}

// GELU'(u) = Phi(u) + u phi(u), phi(u) = exp(-u^2/2) / sqrt(2 pi)
__global__ void __launch_bounds__(256) og_gelu_bwd_kernel(const uint4* __restrict__ da, const uint4* __restrict__ u,
                                                          uint4* __restrict__ du, long long nvec) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * blockDim.x) {
    float g[8], f[8];
    unpack8(__ldg(da + i), g);
    unpack8(__ldg(u + i), f);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float pdf = 0.39894228040143268f * expf(-0.5f * f[k] * f[k]);
      g[k] *= fmaf(f[k], pdf, gelu_cdf(f[k]));
    }
    du[i] = pack8(g);
  }
}

// ------------------------------------------------------------------------------------------------
// backward reduce: S[n][c] = (sum_v dpre, sum_v dpre * x), dpre = dy * act'(x*A+B)
// grid (chunks, N), block 256; same thread mapping as the stats kernel.
// ------------------------------------------------------------------------------------------------
template <int ACT>
__global__ void __launch_bounds__(256, 3)
    og_affine_act_bwd_reduce_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x,
                                    const float* __restrict__ A, const float* __restrict__ B, long long V, int C,
                                    int /*act: template parameter ACT*/, long long rows_per_block, float* __restrict__ S,
                                    float* __restrict__ partials) {
  constexpr int act = ACT;  // compile-time: the per-element switch cost 20 % of the backward pass as a runtime value
  const int cvs = C >> 3;  // host guarantees cvs <= 256
  const int n = blockIdx.y;
  const long long r_begin = (long long)blockIdx.x * rows_per_block;
  const long long r_end = (r_begin + rows_per_block < V) ? r_begin + rows_per_block : V;
  __shared__ float part[256 * 16];  // per-thread partial sums (s1[8], s2[8])
  const int lanes = 256 / cvs;
  const int cv = threadIdx.x % cvs, rl = threadIdx.x / cvs;
  if (rl < lanes && r_begin < V) {
    // act: h = pre/2 = x*(A/2) + B/2 and e = dy (1 + w) = 2 dpre (see silu_grad2_from_half); sums halved at the end
    float av[8], bv[8];
    const float cs = act == 1 ? 0.5f : 1.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      av[k] = cs * A[(long long)n * C + cv * 8 + k];
      bv[k] = cs * B[(long long)n * C + cv * 8 + k];
    }
    float s1[8] = {0, 0, 0, 0, 0, 0, 0, 0}, s2[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const long long base = (long long)n * V * cvs + cv;
    auto accum = [&](const uint4& uxv, const uint4& udv) {
      float fx[8], fd[8];
      unpack8(uxv, fx);
      unpack8(udv, fd);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float e = act ? act_bwd_e(fd[k], fmaf(fx[k], av[k], bv[k]), act) : fd[k];
        s1[k] += e;
        s2[k] = fmaf(e, fx[k], s2[k]);
      }
    };
    long long r = r_begin + rl;
    for (; r + 3LL * lanes < r_end; r += 4LL * lanes) {
      uint4 ux[4], ud[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        ux[j] = __ldg(x + base + (r + (long long)j * lanes) * cvs);
        ud[j] = __ldg(dy + base + (r + (long long)j * lanes) * cvs);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) accum(ux[j], ud[j]);
    }
    for (; r < r_end; r += lanes) accum(__ldg(x + base + r * cvs), __ldg(dy + base + r * cvs));
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      s1[k] *= cs;
      s2[k] *= cs;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      part[threadIdx.x * 16 + k] = s1[k];
      part[threadIdx.x * 16 + 8 + k] = s2[k];
    }
  } else {
#pragma unroll
    for (int k = 0; k < 16; ++k) part[threadIdx.x * 16 + k] = 0.f;
  }
  __syncthreads();
  // thread index == rl * cvs + cv: sum the row lanes of every channel (no contended shared atomics). With several blocks
  // per sample each block stores its sums as a partial, added up in block order by sum_partials (reproducible); a single
  // block per sample adds into S itself.
  for (int i = threadIdx.x; i < 2 * C; i += 256) {
    const int c = i >> 1, which = i & 1;
    float a = 0.f;
    for (int l = 0; l < lanes; ++l) a += part[(l * cvs + (c >> 3)) * 16 + which * 8 + (c & 7)];
    if (partials)
      partials[((long long)n * gridDim.x + blockIdx.x) * 2 * C + i] = a;
    else
      S[(long long)n * C * 2 + i] += a;
  }
}

// dgamma[c] += sum_n s T2, dbeta[c] += sum_n s T1 (s = cond_scale[n][c] or 1), one thread per channel walking the samples
// in order: reproducible, no atomics.
__global__ void __launch_bounds__(256)
    og_gn_param_grads_kernel(const float* __restrict__ S, const float* __restrict__ mean_rstd,
                             const float* __restrict__ cond_scale, int N, int C, int G, float* __restrict__ dgamma,
                             float* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int g = c / (C / G);
  float dg = 0.f, db = 0.f;
  for (int n = 0; n < N; ++n) {
    const float mu = mean_rstd[((long long)n * G + g) * 2], rstd = mean_rstd[((long long)n * G + g) * 2 + 1];
    const float s1 = S[((long long)n * C + c) * 2], s2 = S[((long long)n * C + c) * 2 + 1];
    const float sc = cond_scale ? cond_scale[(long long)n * C + c] : 1.f;
    dg += sc * (rstd * (s2 - mu * s1));
    db += sc * s1;
  }
  if (dgamma) dgamma[c] += dg;
  if (dbeta) dbeta[c] += db;
}

static int launch_param_grads(const float* S, const float* mean_rstd, const float* cond_scale, int N, int C, int G,
                              float* dgamma, float* dbeta, cudaStream_t stream) {
  if (!dgamma && !dbeta) return OG_OK;
  og_gn_param_grads_kernel<<<(C + 255) / 256, 256, 0, stream>>>(S, mean_rstd, cond_scale, N, C, G, dgamma, dbeta);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

// backward finalize: one block per sample n, 256 threads.
//   T1 = S1, T2 = rstd*(S2 - mean*S1);  g' = gamma*s
//   m1_g = sum_{c in g} g' T1 / M,  m2_g = sum_{c in g} g' T2 / M     (M = V * C/G)
//   P = A,  Q = -rstd^2 m2,  R = rstd (m2 rstd mean - m1)
//   dscale[n][c] = gamma T2 + beta T1, dshift[n][c] = T1 (dgamma / dbeta: og_gn_param_grads_kernel)
__global__ void __launch_bounds__(256)
    og_gn_bwd_finalize_kernel(const float* __restrict__ S, const float* __restrict__ mean_rstd,
                              const float* __restrict__ gamma, const float* __restrict__ beta,
                              const float* __restrict__ cond_scale, int C, int G, double inv_M, float* __restrict__ Q,
                              float* __restrict__ R, float* __restrict__ dgamma, float* __restrict__ dbeta,
                              float* __restrict__ dcond_scale, float* __restrict__ dcond_shift) {
  const int n = blockIdx.x;
  __shared__ double m1s[64], m2s[64];
  const int cpg = C / G;
  // group sums in a fixed order (reproducible): one thread per group walks its channels
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    const float mu = mean_rstd[((long long)n * G + g) * 2], rstd = mean_rstd[((long long)n * G + g) * 2 + 1];
    double a1 = 0.0, a2 = 0.0;
    for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
      const float s1 = S[((long long)n * C + c) * 2], s2 = S[((long long)n * C + c) * 2 + 1];
      const float gp = (gamma ? gamma[c] : 1.f) * (cond_scale ? cond_scale[(long long)n * C + c] : 1.f);
      a1 += (double)(gp * s1);
      a2 += (double)(gp * (rstd * (s2 - mu * s1)));
    }
    m1s[g] = a1;
    m2s[g] = a2;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const float mu = mean_rstd[((long long)n * G + g) * 2], rstd = mean_rstd[((long long)n * G + g) * 2 + 1];
    const float s1 = S[((long long)n * C + c) * 2], s2 = S[((long long)n * C + c) * 2 + 1];
    const float t1 = s1, t2 = rstd * (s2 - mu * s1);
    const float ga = gamma ? gamma[c] : 1.f, be = beta ? beta[c] : 0.f;
    if (dcond_scale) dcond_scale[(long long)n * C + c] = ga * t2 + be * t1;
    if (dcond_shift) dcond_shift[(long long)n * C + c] = t1;
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const float mu = mean_rstd[((long long)n * G + g) * 2], rstd = mean_rstd[((long long)n * G + g) * 2 + 1];
    const float m1 = (float)(m1s[g] * inv_M), m2 = (float)(m2s[g] * inv_M);
    Q[(long long)n * C + c] = -rstd * rstd * m2;
    R[(long long)n * C + c] = rstd * (m2 * rstd * mu - m1);
  }
}

// backward apply: dx = P*dpre + Q*x + R (+ add)
__global__ void __launch_bounds__(256)
    og_affine_act_bwd_apply_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x,
                                   const float* __restrict__ A, const float* __restrict__ B,
                                   const float* __restrict__ Q, const float* __restrict__ R,
                                   const uint4* __restrict__ add, uint4* __restrict__ dx, long long V, int C,
                                   long long total_vec, int act) {
  const int cvs = C >> 3;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total_vec;
       i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % cvs);
    const long long row = i / cvs;
    const int n = (int)(row / V);
    const long long o = (long long)n * C + cv * 8;
    float fx[8], fd[8], fa[8];
    unpack8(__ldg(x + i), fx);
    unpack8(__ldg(dy + i), fd);
    if (add) unpack8(__ldg(add + i), fa);
    float out[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float a = __ldg(A + o + k), b = __ldg(B + o + k);
      const float dpre = act == 1 ? fd[k] * silu_grad_f(fmaf(fx[k], a, b)) : act_bwd_e(fd[k], fmaf(fx[k], a, b), act);
      float v = a * dpre;
      if (Q) v += __ldg(Q + o + k) * fx[k] + __ldg(R + o + k);
      if (add) v += fa[k];
      out[k] = v;
    }
    dx[i] = pack8(out);
  }
}


// ------------------------------------------------------------------------------------------------
// fused finalize + apply (forward): grid (blocks_per_sample, N), block 256, thread -> (channel vector, row lane).
// Every thread derives the scale/shift of its own 8 channels from the fp64 group sums (a handful of flops),
// so the stand-alone finalize launch and the per-element coefficient loads disappear; block 0 of each
// sample stores A, B and (mean, rstd) for the backward pass.
// ------------------------------------------------------------------------------------------------
template <int ACT>
__global__ void __launch_bounds__(256, 4)
    og_gn_act_fwd_kernel(const uint4* __restrict__ x, const double* __restrict__ sums, const float* __restrict__ gamma,
                         const float* __restrict__ beta, const float* __restrict__ cond_scale,
                         const float* __restrict__ cond_shift, float* __restrict__ A, float* __restrict__ B,
                         float* __restrict__ mean_rstd, uint4* __restrict__ y, long long V, int C, int G,
                         double inv_count, float eps, int /*act: template parameter ACT*/, long long rows_per_block) {
  constexpr int act = ACT;  // compile-time: the per-element switch cost 20 % of the backward pass as a runtime value
  const int cvs = C >> 3;
  const int n = blockIdx.y;
  const long long r_begin = (long long)blockIdx.x * rows_per_block;
  const long long r_end = (r_begin + rows_per_block < V) ? r_begin + rows_per_block : V;
  const int lanes = 256 / cvs;
  const int cv = threadIdx.x % cvs, rl = threadIdx.x / cvs;
  if (rl >= lanes || r_begin >= V) return;
  float av[8], bv[8];
  const long long o = (long long)n * C + cv * 8;
  {
    const int cpg = C / G;
    const int g = (cv * 8) / cpg;
    const double s = sums[((long long)n * G + g) * 2], ss = sums[((long long)n * G + g) * 2 + 1];
    const double mean = s * inv_count;
    double var = ss * inv_count - mean * mean;
    if (var < 0) var = 0;
    const float rstd = (float)(1.0 / sqrt(var + (double)eps));
    const float mu = (float)mean;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float ga = gamma ? gamma[cv * 8 + k] : 1.f, be = beta ? beta[cv * 8 + k] : 0.f;
      float a = rstd * ga, b = be - mu * rstd * ga;
      if (cond_scale) {
        const float sc = cond_scale[o + k];
        a *= sc;
        b *= sc;
      }
      if (cond_shift) b += cond_shift[o + k];
      av[k] = a;
      bv[k] = b;
    }
    if (blockIdx.x == 0 && rl == 0) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        A[o + k] = av[k];
        B[o + k] = bv[k];
      }
      if ((cv * 8) % cpg == 0) {
        mean_rstd[((long long)n * G + g) * 2] = mu;
        mean_rstd[((long long)n * G + g) * 2 + 1] = rstd;
      }
    }
  }
  if (act == 1) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      av[k] *= 0.5f;
      bv[k] *= 0.5f;
    }
  }
  const long long base = (long long)n * V * cvs + cv;
  long long r = r_begin + rl;
  for (; r + 3LL * lanes < r_end; r += 4LL * lanes) {
    uint4 u[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) u[j] = __ldg(x + base + (r + (long long)j * lanes) * cvs);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float f[8];
      unpack8(u[j], f);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float h = fmaf(f[k], av[k], bv[k]);
        f[k] = act_fwd_val(h, act);
      }
      y[base + (r + (long long)j * lanes) * cvs] = pack8(f);
    }
  }
  for (; r < r_end; r += lanes) {
    float f[8];
    unpack8(__ldg(x + base + r * cvs), f);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float h = fmaf(f[k], av[k], bv[k]);
      f[k] = act_fwd_val(h, act);
    }
    y[base + r * cvs] = pack8(f);
  }
}

// ------------------------------------------------------------------------------------------------
// fused finalize + apply (backward): every block re-derives the per-group means m1, m2 of its sample from
// S (2*C floats, L2-resident), each thread the P/Q/R of its 8 channels; block 0 of the sample also emits
// dgamma / dbeta / dcond. Optionally accumulates the per-channel column sum of dx (the bias gradient of
// the convolution that produced x).
// ------------------------------------------------------------------------------------------------
template <int ACT>
__global__ void __launch_bounds__(256, 3)
    og_gn_act_bwd_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x, const float* __restrict__ A,
                         const float* __restrict__ B, const float* __restrict__ S, const float* __restrict__ mean_rstd,
                         const float* __restrict__ gamma, const float* __restrict__ beta,
                         const float* __restrict__ cond_scale, const uint4* __restrict__ add, uint4* __restrict__ dx,
                         float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dcond_scale,
                         float* __restrict__ dcond_shift, float* __restrict__ dx_colsum, long long V, int C, int G,
                         double inv_M, int /*act: template parameter ACT*/, long long rows_per_block,
                         float* __restrict__ partials) {
  constexpr int act = ACT;  // compile-time: the per-element switch cost 20 % of the backward pass as a runtime value
  const int cvs = C >> 3;
  const int n = blockIdx.y;
  const long long r_begin = (long long)blockIdx.x * rows_per_block;
  const long long r_end = (r_begin + rows_per_block < V) ? r_begin + rows_per_block : V;
  const int lanes = 256 / cvs;
  const int cv = threadIdx.x % cvs, rl = threadIdx.x / cvs;
  const int cpg = C / G;
  __shared__ double m1s[64], m2s[64];
  extern __shared__ float cs_s[];  // [256][8] per-thread column sums of dx (only when dx_colsum)
  if (dx_colsum)
    for (int i = threadIdx.x; i < 256 * 8; i += 256) cs_s[i] = 0.f;
  __syncthreads();
  if (S) {
    // group sums in a fixed order (reproducible): one thread per group walks its channels
    for (int g = threadIdx.x; g < G; g += 256) {
      const float mu = mean_rstd[((long long)n * G + g) * 2], rstd = mean_rstd[((long long)n * G + g) * 2 + 1];
      double a1 = 0.0, a2 = 0.0;
      for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
        const float s1 = S[((long long)n * C + c) * 2], s2 = S[((long long)n * C + c) * 2 + 1];
        const float gp = (gamma ? gamma[c] : 1.f) * (cond_scale ? cond_scale[(long long)n * C + c] : 1.f);
        a1 += (double)(gp * s1);
        a2 += (double)(gp * (rstd * (s2 - mu * s1)));
      }
      m1s[g] = a1;
      m2s[g] = a2;
    }
    for (int c = threadIdx.x; c < C; c += 256) {
      const int g = c / cpg;
      const float mu = mean_rstd[((long long)n * G + g) * 2], rstd = mean_rstd[((long long)n * G + g) * 2 + 1];
      const float s1 = S[((long long)n * C + c) * 2], s2 = S[((long long)n * C + c) * 2 + 1];
      const float t1 = s1, t2 = rstd * (s2 - mu * s1);
      const float ga = gamma ? gamma[c] : 1.f, be = beta ? beta[c] : 0.f;
      if (blockIdx.x == 0) {
        if (dcond_scale) dcond_scale[(long long)n * C + c] = ga * t2 + be * t1;
        if (dcond_shift) dcond_shift[(long long)n * C + c] = t1;
      }
    }
  }
  __syncthreads();
  const bool active = rl < lanes && r_begin < V;
  if (active) {
    float av[8], bv[8], qv[8], rv[8], cs[8];
    const long long o = (long long)n * C + cv * 8;
    {
      const float4 a0 = __ldg(reinterpret_cast<const float4*>(A + o)), a1 = __ldg(reinterpret_cast<const float4*>(A + o) + 1);
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(B + o)), b1 = __ldg(reinterpret_cast<const float4*>(B + o) + 1);
      av[0] = a0.x; av[1] = a0.y; av[2] = a0.z; av[3] = a0.w; av[4] = a1.x; av[5] = a1.y; av[6] = a1.z; av[7] = a1.w;
      bv[0] = b0.x; bv[1] = b0.y; bv[2] = b0.z; bv[3] = b0.w; bv[4] = b1.x; bv[5] = b1.y; bv[6] = b1.z; bv[7] = b1.w;
    }
    if (act == 1) {  // h = pre/2 and e = 2 dpre below: fold both halves into the coefficients
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        av[k] *= 0.5f;
        bv[k] *= 0.5f;
      }
    }
    float q = 0.f, rr = 0.f;
    if (S) {
      const int g = (cv * 8) / cpg;
      const float mu = mean_rstd[((long long)n * G + g) * 2], rstd = mean_rstd[((long long)n * G + g) * 2 + 1];
      const float m1 = (float)(m1s[g] * inv_M), m2 = (float)(m2s[g] * inv_M);
      q = -rstd * rstd * m2;
      rr = rstd * (m2 * rstd * mu - m1);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      qv[k] = q;
      rv[k] = rr;
      cs[k] = 0.f;
    }
    const long long base = (long long)n * V * cvs + cv;
    auto body = [&](const uint4& ux, const uint4& ud, const uint4& ua, long long idx) {
      float fx[8], fd[8], fa[8], out[8];
      unpack8(ux, fx);
      unpack8(ud, fd);
      if (add) unpack8(ua, fa);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float e = act ? act_bwd_e(fd[k], fmaf(fx[k], av[k], bv[k]), act) : fd[k];
        float v = fmaf(av[k], e, fmaf(qv[k], fx[k], rv[k]));
        if (add) v += fa[k];
        out[k] = v;
        cs[k] += v;
      }
      dx[idx] = pack8(out);
    };
    long long r = r_begin + rl;
    for (; r + (long long)lanes < r_end; r += 2LL * lanes) {
      const long long i0 = base + r * cvs, i1 = base + (r + lanes) * cvs;
      const uint4 x0 = __ldg(x + i0), d0 = __ldg(dy + i0), x1 = __ldg(x + i1), d1 = __ldg(dy + i1);
      uint4 a0 = make_uint4(0, 0, 0, 0), a1 = a0;
      if (add) {
        a0 = __ldg(add + i0);
        a1 = __ldg(add + i1);
      }
      body(x0, d0, a0, i0);
      body(x1, d1, a1, i1);
    }
    for (; r < r_end; r += lanes) {
      const long long i0 = base + r * cvs;
      uint4 a0 = make_uint4(0, 0, 0, 0);
      if (add) a0 = __ldg(add + i0);
      body(__ldg(x + i0), __ldg(dy + i0), a0, i0);
    }
    if (dx_colsum) {
#pragma unroll
      for (int k = 0; k < 8; ++k) cs_s[threadIdx.x * 8 + k] = cs[k];
    }
  }
  if (dx_colsum) {
    // one partial per block, added up in block order by sum_partials (reproducible); a single block adds directly
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += 256) {
      float a = 0.f;
      for (int l = 0; l < lanes; ++l) a += cs_s[(l * cvs + (i >> 3)) * 8 + (i & 7)];
      if (partials)
        partials[((long long)blockIdx.y * gridDim.x + blockIdx.x) * C + i] = a;
      else
        dx_colsum[i] += a;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// AdaptiveGroupNorm conditioning (genie/module/norm.py:58-66): cbar = mean_{t,h,w}(cond); scale = W_s cbar + b_s;
// shift = W_a cbar + b_a. One block per sample; replaces a mean reduction, two GEMVs and their bias adds (and, backward,
// two GEMVs, two outer products and two bias reductions) that used to run as ~10 small library launches per layer.
// cond: fp32 rows [N][V][D] (channels-last), D <= 64.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    og_adagn_cond_fwd_kernel(const float* __restrict__ cond, long long V, int D, const float* __restrict__ Ws,
                             const float* __restrict__ bs, const float* __restrict__ Wa, const float* __restrict__ ba,
                             int C, float* __restrict__ cbar, float* __restrict__ scale, float* __restrict__ shift) {
  const int n = blockIdx.x;
  __shared__ float part[256];
  __shared__ float cb[64];
  const float* cp = cond + (long long)n * V * D;
  // thread t owns channel d = t % D of rows t / D, t / D + 256 / D ... (coalesced: consecutive threads, consecutive floats)
  const int per = 256 / D;                 // row lanes
  const int d = threadIdx.x % D, rl = threadIdx.x / D;
  float a = 0.f;
  if (rl < per)
    for (long long r = rl; r < V; r += per) a += cp[r * D + d];
  part[threadIdx.x] = rl < per ? a : 0.f;
  __syncthreads();
  if (threadIdx.x < D) {
    float t = 0.f;
    for (int l = 0; l < per; ++l) t += part[l * D + threadIdx.x];
    t /= (float)V;
    cb[threadIdx.x] = t;
    cbar[n * D + threadIdx.x] = t;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += 256) {
    float s = bs ? bs[c] : 0.f, h = ba ? ba[c] : 0.f;
    for (int k = 0; k < D; ++k) {
      s = fmaf(Ws[c * D + k], cb[k], s);
      if (Wa) h = fmaf(Wa[c * D + k], cb[k], h);
    }
    scale[(long long)n * C + c] = s;
    if (shift) shift[(long long)n * C + c] = h;
  }
}

// backward, one launch: grid (C/64 + N): blocks [0, C/64) own 64 output channels each and write dWs, dbs, dWa, dba for
// them (sum over the N samples, no atomics); block C/64 + n writes dcbar of sample n and broadcasts it over the voxels.
__global__ void __launch_bounds__(256)
    og_adagn_cond_bwd_kernel(const float* __restrict__ dscale, const float* __restrict__ dshift,
                             const float* __restrict__ cbar, const float* __restrict__ Ws, const float* __restrict__ Wa,
                             int N, long long V, int D, int C, float* __restrict__ dWs, float* __restrict__ dbs,
                             float* __restrict__ dWa, float* __restrict__ dba, float* __restrict__ dcond) {
  const int cblocks = (C + 63) / 64;
  if ((int)blockIdx.x < cblocks) {
    // (c, k) pairs of this block: 64 channels x D
    for (int i = threadIdx.x; i < 64 * D; i += 256) {
      const int c = blockIdx.x * 64 + i / D, k = i % D;
      if (c >= C) continue;
      float gs = 0.f, ga = 0.f;
      for (int n = 0; n < N; ++n) {
        const float cb = cbar[n * D + k];
        gs = fmaf(dscale[(long long)n * C + c], cb, gs);
        if (dshift) ga = fmaf(dshift[(long long)n * C + c], cb, ga);
      }
      dWs[c * D + k] = gs;
      if (dWa) dWa[c * D + k] = ga;
    }
    for (int i = threadIdx.x; i < 64; i += 256) {
      const int c = blockIdx.x * 64 + i;
      if (c >= C) continue;
      float gs = 0.f, ga = 0.f;
      for (int n = 0; n < N; ++n) {
        gs += dscale[(long long)n * C + c];
        if (dshift) ga += dshift[(long long)n * C + c];
      }
      if (dbs) dbs[c] = gs;
      if (dba) dba[c] = ga;
    }
    return;
  }
  if (!dcond) return;
  // dcbar[n][k] = sum_c dscale[n][c] Ws[c][k] + dshift[n][c] Wa[c][k];  dcond[n][v][k] = dcbar[n][k] / V   (one block per n)
  __shared__ float dcb[64];
  {
    const int n = (int)blockIdx.x - cblocks;
    // warp w reduces k = w, w + 8, ...
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int k = warp; k < D; k += 8) {
      float a = 0.f;
      for (int c = lane; c < C; c += 32) {
        a = fmaf(dscale[(long long)n * C + c], Ws[c * D + k], a);
        if (dshift && Wa) a = fmaf(dshift[(long long)n * C + c], Wa[c * D + k], a);
      }
      for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      if (lane == 0) dcb[k] = a / (float)V;
    }
    __syncthreads();
    float* dp = dcond + (long long)n * V * D;
    for (long long i = threadIdx.x; i < V * D; i += 256) dp[i] = dcb[i % D];
  }
}

// (blocks_per_sample, N) grid of ~per_sm blocks per SM; every block owns a contiguous range of whole
// kStatRows-row groups of one sample.
static dim3 reduce_grid(int N, long long V, long long* rows_per_block, int per_sm = 4) {
  long long groups = (V + kStatRows - 1) / kStatRows;
  long long want = ((long long)per_sm * num_sms() + N - 1) / N;
  if (want < 1) want = 1;
  if (want > groups) want = groups;
  const long long gpb = (groups + want - 1) / want;
  *rows_per_block = gpb * kStatRows;
  return dim3((unsigned)((groups + gpb - 1) / gpb), (unsigned)N);
}

// reduce_grid, with at most as many blocks as the workspace holds partials of `floats_per_block` floats (at least one
// block per sample; then the blocks add into the output directly)
static dim3 partial_grid(int N, long long V, long long floats_per_block, void* workspace, size_t workspace_bytes,
                         long long* rows_per_block) {
  dim3 grid = reduce_grid(N, V, rows_per_block, 6);
  const long long fit = workspace ? (long long)(workspace_bytes / sizeof(float)) / floats_per_block : 0;
  if ((long long)grid.x * grid.y > fit) {
    long long want = fit / N;
    if (want < 1) want = 1;
    const long long groups = (V + kStatRows - 1) / kStatRows;
    const long long gpb = (groups + want - 1) / want;
    *rows_per_block = gpb * kStatRows;
    grid.x = (unsigned)((groups + gpb - 1) / gpb);
  }
  return grid;
}

static int ew_grid(long long total, int block) {
  long long g = (total + block - 1) / block;
  long long cap = (long long)num_sms() * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace og

using namespace og;

extern "C" int og_gn_stats(const void* x, int N, int64_t V, int C, int G, double* sums, og_stream_t stream) {
  OG_REQUIRE(x && sums, "gn_stats: null pointer");
  OG_REQUIRE(C % 8 == 0 && G >= 1 && G <= 64 && C % G == 0, "gn_stats: need C%%8==0, 1<=G<=64, C%%G==0 (C=%d G=%d)", C,
             G);
  OG_REQUIRE(C <= 2048, "gn_stats: C=%d > 2048", C);
  long long rpb;
  const dim3 grid = reduce_grid(N, V, &rpb, 6);
  if ((C / G) % 8 == 0)
    og_gn_stats_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint4*>(x), V, C, G, rpb, sums);
  else
    og_gn_stats_split_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint4*>(x), V, C, G, rpb,
                                                                      sums);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_gn_finalize(const double* sums, int N, int C, int G, int64_t V, float eps, const float* gamma,
                              const float* beta, const float* cond_scale, const float* cond_shift, float* A, float* B,
                              float* mean_rstd, og_stream_t stream) {
  OG_REQUIRE(sums && A && B && mean_rstd, "gn_finalize: null pointer");
  OG_REQUIRE(C >= 1 && G >= 1 && G <= 64 && C % G == 0, "gn_finalize: need 1<=G<=64, C%%G==0 (C=%d G=%d)", C, G);
  const double inv_count = 1.0 / ((double)V * (C / G));
  const int total = N * C;
  og_gn_finalize_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
      sums, N, C, G, inv_count, eps, gamma, beta, cond_scale, cond_shift, A, B, mean_rstd);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_affine_act_fwd(const void* x, const float* A, const float* B, void* y, int N, int64_t V, int C,
                                 int act, og_stream_t stream) {
  OG_REQUIRE(x && A && B && y, "affine_act_fwd: null pointer");
  OG_REQUIRE(C % 8 == 0, "affine_act_fwd: C=%d must be a multiple of 8", C);
  OG_REQUIRE(act >= 0 && act <= 3, "affine_act_fwd: unknown activation code %d", act);
  const long long total = (long long)N * V * (C / 8);
  og_affine_act_fwd_kernel<<<ew_grid(total, 256), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const uint4*>(x), A, B, reinterpret_cast<uint4*>(y), V, C, total, act);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_affine_act_bwd_reduce(const void* dy, const void* x, const float* A, const float* B, int act,
                                        float* S, int N, int64_t V, int C, void* workspace, size_t workspace_bytes,
                                        og_stream_t stream) {
  OG_REQUIRE(dy && x && A && B && S, "affine_act_bwd_reduce: null pointer");
  OG_REQUIRE(C % 8 == 0 && C <= 2048, "affine_act_bwd_reduce: C=%d must be a multiple of 8 and <= 2048", C);
  long long rpb;
  const dim3 grid = partial_grid(N, V, 2LL * C, workspace, workspace_bytes, &rpb);
  float* partials = grid.x > 1 ? reinterpret_cast<float*>(workspace) : nullptr;
#define OG_LAUNCH(ACT)                                                                                  \
  og_affine_act_bwd_reduce_kernel<ACT><<<grid, 256, 0, (cudaStream_t)stream>>>(                          \
      reinterpret_cast<const uint4*>(dy), reinterpret_cast<const uint4*>(x), A, B, V, C, act, rpb, S, partials)
  OG_REQUIRE(act >= 0 && act <= 3, "affine_act_bwd_reduce: unknown activation code %d", act);
  if (act == 0) OG_LAUNCH(0); else if (act == 1) OG_LAUNCH(1); else if (act == 2) OG_LAUNCH(2); else OG_LAUNCH(3);
#undef OG_LAUNCH
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  if (partials) return sum_partials(partials, N, (int)grid.x, 2LL * C, 2LL * C, 2LL * C, S, (cudaStream_t)stream);
  return OG_OK;
}

extern "C" int og_gn_bwd_finalize(const float* S, const float* mean_rstd, const float* gamma, const float* beta,
                                  const float* cond_scale, int N, int C, int G, int64_t V, float* Q, float* R,
                                  float* dgamma, float* dbeta, float* dcond_scale, float* dcond_shift,
                                  og_stream_t stream) {
  OG_REQUIRE(S && mean_rstd && Q && R, "gn_bwd_finalize: null pointer");
  OG_REQUIRE(G >= 1 && G <= 64 && C >= 1 && C % G == 0, "gn_bwd_finalize: need 1<=G<=64, C%%G==0 (C=%d G=%d)", C, G);
  const double inv_M = 1.0 / ((double)V * (C / G));
  og_gn_bwd_finalize_kernel<<<N, 256, 0, (cudaStream_t)stream>>>(S, mean_rstd, gamma, beta, cond_scale, C, G, inv_M, Q,
                                                                 R, dgamma, dbeta, dcond_scale, dcond_shift);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return launch_param_grads(S, mean_rstd, cond_scale, N, C, G, dgamma, dbeta, (cudaStream_t)stream);
}

extern "C" int og_affine_act_bwd_apply(const void* dy, const void* x, const float* A, const float* B, const float* Q,
                                       const float* R, const void* add, void* dx, int act, int N, int64_t V, int C,
                                       og_stream_t stream) {
  OG_REQUIRE(dy && x && A && B && dx, "affine_act_bwd_apply: null pointer");
  OG_REQUIRE((Q == nullptr) == (R == nullptr), "affine_act_bwd_apply: Q and R must both be given or both NULL");
  OG_REQUIRE(C % 8 == 0, "affine_act_bwd_apply: C=%d must be a multiple of 8", C);
  OG_REQUIRE(act >= 0 && act <= 3, "affine_act_bwd_apply: unknown activation code %d", act);
  const long long total = (long long)N * V * (C / 8);
  og_affine_act_bwd_apply_kernel<<<ew_grid(total, 256), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const uint4*>(dy), reinterpret_cast<const uint4*>(x), A, B, Q, R,
      reinterpret_cast<const uint4*>(add), reinterpret_cast<uint4*>(dx), V, C, total, act);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_gn_act_fwd(const void* x, const double* sums, const float* gamma, const float* beta,
                             const float* cond_scale, const float* cond_shift, float eps, int G, int act, void* y,
                             float* A, float* B, float* mean_rstd, int N, int64_t V, int C, og_stream_t stream) {
  OG_REQUIRE(x && sums && y && A && B && mean_rstd, "gn_act_fwd: null pointer");
  OG_REQUIRE(C % 8 == 0 && C <= 2048 && G >= 1 && G <= 64 && C % G == 0 && (C / G) % 8 == 0,
             "gn_act_fwd: need C%%8==0, C<=2048, G<=64, (C/G)%%8==0 (C=%d G=%d)", C, G);
  long long rpb;
  const dim3 grid = reduce_grid(N, V, &rpb, 8);
  const double inv_count = 1.0 / ((double)V * (C / G));
#define OG_LAUNCH(ACT)                                                                                  \
  og_gn_act_fwd_kernel<ACT><<<grid, 256, 0, (cudaStream_t)stream>>>(                                     \
      reinterpret_cast<const uint4*>(x), sums, gamma, beta, cond_scale, cond_shift, A, B, mean_rstd,     \
      reinterpret_cast<uint4*>(y), V, C, G, inv_count, eps, act, rpb)
  OG_REQUIRE(act >= 0 && act <= 3, "gn_act_fwd: unknown activation code %d", act);
  if (act == 0) OG_LAUNCH(0); else if (act == 1) OG_LAUNCH(1); else if (act == 2) OG_LAUNCH(2); else OG_LAUNCH(3);
#undef OG_LAUNCH
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_gn_act_bwd(const void* dy, const void* x, const float* A, const float* B, const float* S,
                             const float* mean_rstd, const float* gamma, const float* beta, const float* cond_scale,
                             int G, int act, const void* add, void* dx, float* dgamma, float* dbeta,
                             float* dcond_scale, float* dcond_shift, float* dx_colsum, int N, int64_t V, int C,
                             void* workspace, size_t workspace_bytes, og_stream_t stream) {
  OG_REQUIRE(dy && x && A && B && dx, "gn_act_bwd: null pointer");
  OG_REQUIRE((S == nullptr) == (mean_rstd == nullptr), "gn_act_bwd: S and mean_rstd must both be given or both NULL");
  OG_REQUIRE(C % 8 == 0 && C <= 2048 && G >= 1 && G <= 64 && C % G == 0 && (C / G) % 8 == 0,
             "gn_act_bwd: need C%%8==0, C<=2048, G<=64, (C/G)%%8==0 (C=%d G=%d)", C, G);
  long long rpb;
  // with dx_colsum: one C-wide partial per block in the workspace (the grid shrinks to what fits; one block adds directly)
  const dim3 grid = dx_colsum ? partial_grid(N, V, (long long)C, workspace, workspace_bytes, &rpb) : reduce_grid(N, V, &rpb, 6);
  float* partials = (dx_colsum && (long long)grid.x * grid.y > 1) ? reinterpret_cast<float*>(workspace) : nullptr;
  OG_REQUIRE(!dx_colsum || N == 1 || (workspace && workspace_bytes >= (size_t)N * C * sizeof(float)),
             "gn_act_bwd: dx_colsum over N=%d samples needs a workspace of at least N*C floats", N);
  const double inv_M = 1.0 / ((double)V * (C / G));
#define OG_LAUNCH(ACT)                                                                                                    \
  og_gn_act_bwd_kernel<ACT><<<grid, 256, dx_colsum ? 256 * 8 * sizeof(float) : 0, (cudaStream_t)stream>>>(                \
      reinterpret_cast<const uint4*>(dy), reinterpret_cast<const uint4*>(x), A, B, S, mean_rstd, gamma, beta, cond_scale, \
      reinterpret_cast<const uint4*>(add), reinterpret_cast<uint4*>(dx), dgamma, dbeta, dcond_scale, dcond_shift,         \
      dx_colsum, V, C, G, inv_M, act, rpb, partials)
  OG_REQUIRE(act >= 0 && act <= 3, "gn_act_bwd: unknown activation code %d", act);
  if (act == 0) OG_LAUNCH(0); else if (act == 1) OG_LAUNCH(1); else if (act == 2) OG_LAUNCH(2); else OG_LAUNCH(3);
#undef OG_LAUNCH
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  int rc = OG_OK;
  if (partials) rc = sum_partials(partials, 1, (int)(grid.x * grid.y), C, C, C, dx_colsum, (cudaStream_t)stream);
  if (rc != OG_OK) return rc;
  if (S) return launch_param_grads(S, mean_rstd, cond_scale, N, C, G, dgamma, dbeta, (cudaStream_t)stream);
  return OG_OK;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int og_gelu_fwd(const void* u, void* a, int64_t rows, int C, og_stream_t stream) {
  OG_REQUIRE(u && a, "gelu_fwd: null pointer");
  OG_REQUIRE(C > 0 && C % 8 == 0, "gelu_fwd: C=%d must be a positive multiple of 8", C);
  OG_REQUIRE(rows > 0, "gelu_fwd: empty problem (rows=%lld)", (long long)rows);
  OG_REQUIRE(aligned16(u) && aligned16(a), "gelu_fwd: u and a must be 16-byte aligned");
  const long long nvec = rows * (C / 8);
  og_gelu_fwd_kernel<<<ew_grid(nvec, 256), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint4*>(u),
                                                                          reinterpret_cast<uint4*>(a), nvec);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_gelu_bwd(const void* da, const void* u, void* du, int64_t rows, int C, og_stream_t stream) {
  OG_REQUIRE(da && u && du, "gelu_bwd: null pointer");
  OG_REQUIRE(C > 0 && C % 8 == 0, "gelu_bwd: C=%d must be a positive multiple of 8", C);
  OG_REQUIRE(rows > 0, "gelu_bwd: empty problem (rows=%lld)", (long long)rows);
  OG_REQUIRE(aligned16(da) && aligned16(u) && aligned16(du), "gelu_bwd: da, u and du must be 16-byte aligned");
  const long long nvec = rows * (C / 8);
  og_gelu_bwd_kernel<<<ew_grid(nvec, 256), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const uint4*>(da), reinterpret_cast<const uint4*>(u), reinterpret_cast<uint4*>(du), nvec);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_adagn_cond_fwd(const float* cond, int N, int64_t V, int D, const float* w_scale, const float* b_scale,
                                 const float* w_shift, const float* b_shift, int C, float* cbar, float* scale, float* shift,
                                 og_stream_t stream) {
  OG_REQUIRE(cond && w_scale && cbar && scale && N > 0 && V > 0, "adagn_cond_fwd: bad arguments");
  OG_REQUIRE(D >= 1 && D <= 64 && C >= 1, "adagn_cond_fwd: dim_cond=%d must be in [1, 64]", D);
  OG_REQUIRE((w_shift != nullptr) == (shift != nullptr), "adagn_cond_fwd: w_shift and shift go together");
  og_adagn_cond_fwd_kernel<<<N, 256, 0, (cudaStream_t)stream>>>(cond, V, D, w_scale, b_scale, w_shift, b_shift, C, cbar,
                                                               scale, shift);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_adagn_cond_bwd(const float* dscale, const float* dshift, const float* cbar, const float* w_scale,
                                 const float* w_shift, int N, int64_t V, int D, int C, float* dw_scale, float* db_scale,
                                 float* dw_shift, float* db_shift, float* dcond, og_stream_t stream) {
  OG_REQUIRE(dscale && cbar && w_scale && dw_scale && N > 0 && V > 0, "adagn_cond_bwd: bad arguments");
  OG_REQUIRE(D >= 1 && D <= 64 && C >= 1, "adagn_cond_bwd: dim_cond=%d must be in [1, 64]", D);
  const int blocks = (C + 63) / 64 + (dcond ? N : 0);
  og_adagn_cond_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(dscale, dshift, cbar, w_scale, w_shift, N, V, D, C,
                                                                    dw_scale, db_scale, dw_shift, db_shift, dcond);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}
