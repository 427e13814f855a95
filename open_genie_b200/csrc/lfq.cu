// lfq.cu — Lookup-Free Quantization: sign quantise, bit-packed indices, straight-through output and the
// entropy + commitment loss, forward and backward, WITHOUT materialising the (tokens x 2^D) softmax.
//
// Reference: LookupFreeQuantization.forward, genie/module/quantization.py:77-133 (entropy(): 17-28).
// The reference builds p = softmax(2*beta * x . C^T) over all 2^D codes (2.1 GB of fp32 at D=18, N=2048).
// Because every code is a sign pattern, the softmax factorises exactly:
//       p[n][j] = prod_d  sigmoid(+-4*beta*x[n][d])           (sign = bit d of j, MSB first, line 72)
// and with j = (hi << D2) | lo it is an outer product  p[n][hi][lo] = a[n][hi] * b[n][lo]  of two short
// vectors (2^D1 and 2^D2 entries, D1 = ceil(D/2)). Hence
//   * per-sample entropy  -sum_j p log(max(p, eps))  is evaluated pair by pair in registers, skipping
//     whole rows whose largest product is below eps (they contribute the closed form -log(eps) * mass);
//     the clamp is kept exactly as in the reference (it does not factorise);
//   * the batch-mean distribution is the (2^D1 x N) x (N x 2^D2) product A^T B / N  (fp32 CUDA-core GEMM:
//     these are probabilities, bf16 tensor cores would cost the 1e-3 parity);
//   * backward needs, per token, sum_j p_j G_j c_jd with G = dL/dp: the per-sample part is again a
//     pair loop, the batch part reduces to two more small GEMMs (U = B G2^T, V = A G2).
// The op is bound by SFU/FP32 throughput, not HBM: algorithmic bytes are N*D*(4+2+8) only.
#include "og_host.cuh"
#include "og_ptx.cuh"

namespace og {
extern std::atomic<uint64_t> g_launches;

static constexpr int kLfqThreads = 128;
static constexpr int kMaxD = 20;
static constexpr float kEps = 1e-6f;

struct LfqDims {
  int D, D1, D2, H, L;  // H = 2^D1 (high half), L = 2^D2
};

__device__ __forceinline__ float block_sum(float v, float* ws) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += ws[i];
  return t;
}

// builds a[0..H) and b[0..L) for one token in shared memory; returns tanh-like (sp - sm) in sh_t
__device__ __forceinline__ void build_ab(const float* __restrict__ xr, const LfqDims d, float beta, float* sp,
                                         float* sm, float* a, float* b) {
  if (threadIdx.x < d.D) {
    const float t = 4.f * beta * xr[threadIdx.x];
    sp[threadIdx.x] = 1.f / (1.f + expf(-t));
    sm[threadIdx.x] = 1.f / (1.f + expf(t));
  }
  __syncthreads();
  for (int h = threadIdx.x; h < d.H; h += blockDim.x) {
    float v = 1.f;
    for (int i = 0; i < d.D1; ++i) v *= ((h >> (d.D1 - 1 - i)) & 1) ? sp[i] : sm[i];
    a[h] = v;
  }
  for (int l = threadIdx.x; l < d.L; l += blockDim.x) {
    float v = 1.f;
    for (int i = 0; i < d.D2; ++i) v *= ((l >> (d.D2 - 1 - i)) & 1) ? sp[d.D1 + i] : sm[d.D1 + i];
    b[l] = v;
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// forward, one block per token
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLfqThreads)
    og_lfq_fwd_kernel(const float* __restrict__ x, int ldx, const LfqDims d, float beta, int training,
                      float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_bf16, int ld_bf16,
                      long long* __restrict__ idx, float* __restrict__ A, float* __restrict__ B,
                      float* __restrict__ stats /* [0]=sum H_n, [1]=sum (x-q)^2 */) {
  extern __shared__ float sh[];
  float* sp = sh;
  float* sm = sp + 32;
  float* ws = sm + 32;
  float* a = ws + 32;
  float* b = a + d.H;
  const long long n = blockIdx.x;
  const float* xr = x + n * ldx;

  // quantise / indices / straight-through output (lines 97-101)
  float commit = 0.f;
  if (threadIdx.x < 32) {
    long long bits = 0;
    if (threadIdx.x == 0) {
      for (int i = 0; i < d.D; ++i) bits |= (long long)(xr[i] > 0.f) << (d.D - 1 - i);
      idx[n] = bits;
    }
    for (int i = threadIdx.x; i < ld_bf16 || i < d.D; i += 32) {
      float code = 0.f;
      if (i < d.D) {
        const float v = xr[i];
        const float q = (v > 0.f) ? 1.f : ((v < 0.f) ? -1.f : 0.f);
        // training: x + (sign(x) - x), evaluated in this order like the reference's STE (not bit-equal to sign(x))
        code = training ? __fadd_rn(v, __fsub_rn(q, v)) : q;
        commit += (v - q) * (v - q);
        if (out_f32) out_f32[n * d.D + i] = code;
      }
      if (out_bf16 && i < ld_bf16) out_bf16[n * ld_bf16 + i] = __float2bfloat16_rn(code);
    }
  }
  if (!training) return;

  build_ab(xr, d, beta, sp, sm, a, b);
  for (int h = threadIdx.x; h < d.H; h += blockDim.x) A[n * d.H + h] = a[h];
  for (int l = threadIdx.x; l < d.L; l += blockDim.x) B[n * d.L + l] = b[l];

  float bmax = 0.f, bsum = 0.f, asum = 0.f;
  for (int l = 0; l < d.L; ++l) {
    bmax = fmaxf(bmax, b[l]);
    bsum += b[l];
  }
  for (int h = 0; h < d.H; ++h) asum += a[h];
  const float log_eps = logf(kEps);
  float acc = 0.f;
  for (int h = 0; h < d.H; ++h) {
    const float ah = a[h];
    if (ah * bmax < kEps) continue;  // block-uniform
    for (int l = threadIdx.x; l < d.L; l += blockDim.x) {
      const float p = ah * b[l];
      if (p >= kEps) acc += p * (logf(p) - log_eps);
    }
  }
  const float tot = block_sum(acc, ws);
  const float csum = block_sum(commit, ws);
  if (threadIdx.x == 0) {
    atomicAdd(&stats[0], -(log_eps * (asum * bsum) + tot));
    atomicAdd(&stats[1], csum);
  }
}

// entropy of the batch-mean distribution + G2 = dL/d(avg) (scaled) ; single block, then final loss
__global__ void __launch_bounds__(1024)
    og_lfq_avg_kernel(const float* __restrict__ avg, long long ncodes, long long ntok, int D, float w_commit,
                      float w_entropy, float w_div, float* __restrict__ g2, float* __restrict__ stats,
                      float* __restrict__ loss) {
  __shared__ float ws[32];
  const float log_eps = logf(kEps);
  float acc = 0.f;
  const float gs = w_entropy * w_div / (float)ntok;
  for (long long j = threadIdx.x; j < ncodes; j += blockDim.x) {
    const float p = avg[j];
    const float lp = logf(fmaxf(p, kEps));
    acc += p * lp;
    if (g2) g2[j] = -(lp + (p >= kEps ? 1.f : 0.f)) * gs;
  }
  const float tot = block_sum(acc, ws);
  if (threadIdx.x == 0) {
    const float h_avg = -tot;
    stats[2] = h_avg;
    const float inp_ent = stats[0] / (float)ntok;
    const float commit = stats[1] / ((float)ntok * (float)D);
    loss[0] = (inp_ent + w_div * h_avg) * w_entropy + commit * w_commit;
  }
  (void)log_eps;
}

// ------------------------------------------------------------------------------------------------
// generic small fp32 GEMM on CUDA cores: C[i][j] = alpha * sum_k X[i*sxi + k*sxk] * Y[j*syj + k*syk]
// 64x64 tile, 16-deep, 256 threads (4x4 per thread).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    og_sgemm_kernel(const float* __restrict__ X, long long sxi, long long sxk, const float* __restrict__ Y,
                    long long syj, long long syk, float* __restrict__ C, long long ldc, int M, int N, int K,
                    float alpha) {
  __shared__ float xs[16][65];
  __shared__ float ys[16][65];
  const int i0 = blockIdx.y * 64, j0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4] = {};
  // no split-K: every output is one block's fixed-order sum (reproducible), at the price of only 64 tiles for the
  // 512 x 512 batch-mean code distribution
  const int k_begin = 0;
  const int k_end = K;
  for (int k0 = k_begin; k0 < k_end; k0 += 16) {
    for (int e = threadIdx.x; e < 64 * 16; e += 256) {
      int kk, ii;
      if (sxk == 1) { kk = e & 15; ii = e >> 4; } else { ii = e & 63; kk = e >> 6; }
      const int gi = i0 + ii, gk = k0 + kk;
      xs[kk][ii] = (gi < M && gk < k_end) ? X[gi * sxi + gk * sxk] : 0.f;
      int kj, jj;
      if (syk == 1) { kj = e & 15; jj = e >> 4; } else { jj = e & 63; kj = e >> 6; }
      const int gj = j0 + jj, gk2 = k0 + kj;
      ys[kj][jj] = (gj < N && gk2 < k_end) ? Y[gj * syj + gk2 * syk] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float xv[4], yv[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) xv[r] = xs[kk][ty * 4 + r];
#pragma unroll
      for (int c = 0; c < 4; ++c) yv[c] = ys[kk][tx * 4 + c];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(xv[r], yv[c], acc[r][c]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int gi = i0 + ty * 4 + r, gj = j0 + tx * 4 + c;
      if (gi < M && gj < N) C[gi * ldc + gj] = alpha * acc[r][c];
    }
}

// ------------------------------------------------------------------------------------------------
// backward, one block per token
//   dx[d] = gl * 2 beta * ( M[d] - Gbar * tanh[d] ) + gl * w_c * 2 (x - q) / (N D) + dout[d]
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLfqThreads)
    og_lfq_bwd_kernel(const float* __restrict__ x, int ldx, const LfqDims d, float beta, long long ntok,
                      float w_commit, float w_entropy, const float* __restrict__ U, const float* __restrict__ Vm,
                      const float* __restrict__ gloss, const float* __restrict__ dout, int ld_dout,
                      float* __restrict__ dx_f32, __nv_bfloat16* __restrict__ dx_bf16, int ld_dx) {
  extern __shared__ float sh[];
  float* sp = sh;
  float* sm = sp + 32;
  float* ws = sm + 32;
  float* red = ws + 32;  // [kMaxD + 1] reduced sums
  float* a = red + 32;
  float* b = a + d.H;
  const long long n = blockIdx.x;
  const float* xr = x + n * ldx;
  build_ab(xr, d, beta, sp, sm, a, b);

  float bmax = 0.f;
  for (int l = 0; l < d.L; ++l) bmax = fmaxf(bmax, b[l]);
  const float log_eps = logf(kEps);

  // per-sample part: val = p (log p - log eps + 1) over pairs with p >= eps
  float m[kMaxD];
#pragma unroll
  for (int i = 0; i < kMaxD; ++i) m[i] = 0.f;
  float w1 = 0.f;
  for (int h = 0; h < d.H; ++h) {
    const float ah = a[h];
    if (ah * bmax < kEps) continue;
    for (int l = threadIdx.x; l < d.L; l += blockDim.x) {
      const float p = ah * b[l];
      if (p >= kEps) {
        const float val = p * (logf(p) - log_eps + 1.f);
        w1 += val;
#pragma unroll
        for (int i = 0; i < kMaxD; ++i) {
          if (i < d.D) {
            const int bit = (i < d.D1) ? ((h >> (d.D1 - 1 - i)) & 1) : ((l >> (d.D - 1 - i)) & 1);
            m[i] += bit ? val : -val;
          }
        }
      }
    }
  }
  // batch part: Gbar2 = sum_h a_h U_h ; M2[d<D1] = sum_h a_h c_hd U_h ; M2[d>=D1] = sum_l b_l c_ld V_l
  float g2bar = 0.f;
  float m2[kMaxD];
#pragma unroll
  for (int i = 0; i < kMaxD; ++i) m2[i] = 0.f;
  for (int h = threadIdx.x; h < d.H; h += blockDim.x) {
    const float au = a[h] * U[n * d.H + h];
    g2bar += au;
#pragma unroll
    for (int i = 0; i < kMaxD; ++i)
      if (i < d.D1) m2[i] += ((h >> (d.D1 - 1 - i)) & 1) ? au : -au;
  }
  for (int l = threadIdx.x; l < d.L; l += blockDim.x) {
    const float bv = b[l] * Vm[n * d.L + l];
#pragma unroll
    for (int i = 0; i < kMaxD; ++i)
      if (i >= d.D1 && i < d.D) m2[i] += ((l >> (d.D - 1 - i)) & 1) ? bv : -bv;
  }
  const float w1s = block_sum(w1, ws);
  const float g2s = block_sum(g2bar, ws);
  const float gl = gloss ? *gloss : 1.f;
  const float we_n = w_entropy / (float)ntok;
  const float gbar = -we_n * (log_eps + w1s) + g2s;
#pragma unroll
  for (int i = 0; i < kMaxD; ++i) {
    if (i < d.D) {
      const float m1s = block_sum(m[i], ws);
      const float m2s = block_sum(m2[i], ws);
      if (threadIdx.x == 0) red[i] = -we_n * (log_eps * (sp[i] - sm[i]) + m1s) + m2s;
    }
  }
  __syncthreads();
  if (threadIdx.x < d.D) {
    const int i = threadIdx.x;
    const float v = xr[i];
    const float q = (v > 0.f) ? 1.f : ((v < 0.f) ? -1.f : 0.f);
    float g = gl * 2.f * beta * (red[i] - gbar * (sp[i] - sm[i]));
    g += gl * w_commit * 2.f * (v - q) / ((float)ntok * (float)d.D);
    if (dout) g += dout[n * ld_dout + i];
    if (dx_f32) dx_f32[n * ld_dx + i] = g;
    if (dx_bf16) dx_bf16[n * ld_dx + i] = __float2bfloat16_rn(g);
  }
  if (dx_bf16)
    for (int i = d.D + threadIdx.x; i < ld_dx; i += blockDim.x) dx_bf16[n * ld_dx + i] = __float2bfloat16_rn(0.f);
  if (dx_f32)
    for (int i = d.D + threadIdx.x; i < ld_dx; i += blockDim.x) dx_f32[n * ld_dx + i] = 0.f;
}

static LfqDims make_dims(int D) {
  LfqDims d;
  d.D = D;
  d.D1 = (D + 1) / 2;
  d.D2 = D / 2;
  d.H = 1 << d.D1;
  d.L = 1 << d.D2;
  return d;
}

static int launch_sgemm(const float* X, long long sxi, long long sxk, const float* Y, long long syj, long long syk,
                        float* C, long long ldc, int M, int N, int K, float alpha, cudaStream_t s) {
  dim3 grid((N + 63) / 64, (M + 63) / 64);
  og_sgemm_kernel<<<grid, 256, 0, s>>>(X, sxi, sxk, Y, syj, syk, C, ldc, M, N, K, alpha);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

}  // namespace og

using namespace og;

extern "C" size_t og_lfq_workspace_bytes(int64_t ntok, int D) {
  if (D < 1 || D > kMaxD) return 0;
  const LfqDims d = make_dims(D);
  // A, B, U, V (per token) + avg, g2 (per code) + stats[4]
  return sizeof(float) * ((size_t)ntok * (d.H + d.L) * 2 + ((size_t)1 << D) * 2 + 4);
}

/* Workspace layout (floats): A[ntok*H] B[ntok*L] U[ntok*H] V[ntok*L] avg[2^D] g2[2^D] stats[4] */
extern "C" int og_lfq_fwd(const float* x, int ldx, int64_t ntok, int D, float beta, int training, float w_commit,
                          float w_entropy, float w_div, float* out_f32, void* out_bf16, int ld_bf16, int64_t* idx,
                          float* loss, void* workspace, og_stream_t stream) {
  OG_REQUIRE(x && idx && ntok > 0, "lfq_fwd: bad arguments");
  OG_REQUIRE(D >= 1 && D <= kMaxD, "lfq_fwd: codebook_dim=%d outside [1,%d]", D, kMaxD);
  OG_REQUIRE(!training || (loss && workspace), "lfq_fwd: training needs loss and workspace");
  cudaStream_t s = (cudaStream_t)stream;
  const LfqDims d = make_dims(D);
  float* ws = reinterpret_cast<float*>(workspace);
  float *A = nullptr, *B = nullptr, *avg = nullptr, *g2 = nullptr, *stats = nullptr;
  if (training) {
    A = ws;
    B = A + ntok * d.H;
    float* U = B + ntok * d.L;
    float* V = U + ntok * d.H;
    avg = V + ntok * d.L;
    g2 = avg + ((size_t)1 << D);
    stats = g2 + ((size_t)1 << D);
    OG_CHECK_CUDA(cudaMemsetAsync(stats, 0, 4 * sizeof(float), s));
  }
  const size_t smem = sizeof(float) * (96 + d.H + d.L);
  og_lfq_fwd_kernel<<<(unsigned)ntok, kLfqThreads, smem, s>>>(x, ldx, d, beta, training, out_f32,
                                                             (__nv_bfloat16*)out_bf16, ld_bf16, (long long*)idx, A, B,
                                                             stats);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  if (!training) return OG_OK;
  // avg[h][l] = (1/N) sum_n A[n][h] B[n][l]
  int r = launch_sgemm(A, 1, d.H, B, 1, d.L, avg, d.L, d.H, d.L, (int)ntok, 1.f / (float)ntok, s);
  if (r != OG_OK) return r;
  og_lfq_avg_kernel<<<1, 1024, 0, s>>>(avg, (long long)1 << D, ntok, D, w_commit, w_entropy, w_div, g2, stats, loss);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_lfq_bwd(const float* x, int ldx, int64_t ntok, int D, float beta, float w_commit, float w_entropy,
                          const float* gloss, const float* dout, int ld_dout, float* dx_f32, void* dx_bf16, int ld_dx,
                          void* workspace, og_stream_t stream) {
  OG_REQUIRE(x && workspace && (dx_f32 || dx_bf16) && ld_dx >= D, "lfq_bwd: bad arguments");
  OG_REQUIRE(D >= 1 && D <= kMaxD, "lfq_bwd: codebook_dim=%d outside [1,%d]", D, kMaxD);
  cudaStream_t s = (cudaStream_t)stream;
  const LfqDims d = make_dims(D);
  float* ws = reinterpret_cast<float*>(workspace);
  float* A = ws;
  float* B = A + ntok * d.H;
  float* U = B + ntok * d.L;
  float* V = U + ntok * d.H;
  float* avg = V + ntok * d.L;
  float* g2 = avg + ((size_t)1 << D);
  (void)avg;
  // U[n][h] = sum_l B[n][l] g2[h][l] ;  V[n][l] = sum_h A[n][h] g2[h][l]
  int r = launch_sgemm(B, d.L, 1, g2, d.L, 1, U, d.H, (int)ntok, d.H, d.L, 1.f, s);
  if (r != OG_OK) return r;
  r = launch_sgemm(A, d.H, 1, g2, 1, d.L, V, d.L, (int)ntok, d.L, d.H, 1.f, s);
  if (r != OG_OK) return r;
  const size_t smem = sizeof(float) * (128 + d.H + d.L);
  og_lfq_bwd_kernel<<<(unsigned)ntok, kLfqThreads, smem, s>>>(x, ldx, d, beta, ntok, w_commit, w_entropy, U, V, gloss,
                                                             dout, ld_dout, dx_f32, (__nv_bfloat16*)dx_bf16, ld_dx);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}
