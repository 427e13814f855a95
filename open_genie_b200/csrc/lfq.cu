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
//
// Several codebooks (num_codebook = C > 1, quantization.py:52,74,90): token n's C*D inputs are C rows r = n*C + c of
// D inputs each, quantised independently. The reference's codebook repeats each of the 2^D sign codes C times, so
// its softmax gives every code q_j / C, C times over, where q is the row's factorised distribution above. Hence
//   H(p) = H_{C eps}(q) + log C   per row,   and   H(avg_c) = H_{C eps}(mean_n q_(n,c)) + log C   per codebook,
// i.e. the kernels below run per row with the clamp at eps' = C * eps, the batch mean (and U, V) once per codebook,
// and the loss adds the constant (1 + w_div) log C. With C = 1 every formula is the single-codebook one.
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
// forward, one block per row r = n * C + c (token n, codebook c)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLfqThreads)
    og_lfq_fwd_kernel(const float* __restrict__ x, int ldx, const LfqDims d, int C, float eps, float beta,
                      int training, float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_bf16, int ld_bf16,
                      long long* __restrict__ idx, float* __restrict__ A, float* __restrict__ B,
                      float* __restrict__ stats /* [0]=sum H_r, [1]=sum (x-q)^2 */) {
  extern __shared__ float sh[];
  float* sp = sh;
  float* sm = sp + 32;
  float* ws = sm + 32;
  float* a = ws + 32;
  float* b = a + d.H;
  const long long r = blockIdx.x;
  const long long n = r / C;
  const int col0 = (int)(r - n * C) * d.D;  // this row's first column in the token's C*D
  const float* xr = x + n * ldx + col0;
  // the last codebook's row also zero-fills the bf16 pad columns [C*D, ld_bf16)
  const int ncol = (col0 + d.D == C * d.D && ld_bf16 - col0 > d.D) ? ld_bf16 - col0 : d.D;

  // quantise / indices / straight-through output (lines 97-101)
  float commit = 0.f;
  if (threadIdx.x < 32) {
    long long bits = 0;
    if (threadIdx.x == 0) {
      for (int i = 0; i < d.D; ++i) bits |= (long long)(xr[i] > 0.f) << (d.D - 1 - i);
      idx[r] = bits;
    }
    for (int i = threadIdx.x; i < ncol; i += 32) {
      float code = 0.f;
      if (i < d.D) {
        const float v = xr[i];
        const float q = (v > 0.f) ? 1.f : ((v < 0.f) ? -1.f : 0.f);
        // training: x + (sign(x) - x), evaluated in this order like the reference's STE (not bit-equal to sign(x))
        code = training ? __fadd_rn(v, __fsub_rn(q, v)) : q;
        commit += (v - q) * (v - q);
        if (out_f32) out_f32[r * d.D + i] = code;
      }
      if (out_bf16 && col0 + i < ld_bf16) out_bf16[n * ld_bf16 + col0 + i] = __float2bfloat16_rn(code);
    }
  }
  if (!training) return;

  build_ab(xr, d, beta, sp, sm, a, b);
  for (int h = threadIdx.x; h < d.H; h += blockDim.x) A[r * d.H + h] = a[h];
  for (int l = threadIdx.x; l < d.L; l += blockDim.x) B[r * d.L + l] = b[l];

  float bmax = 0.f, bsum = 0.f, asum = 0.f;
  for (int l = 0; l < d.L; ++l) {
    bmax = fmaxf(bmax, b[l]);
    bsum += b[l];
  }
  for (int h = 0; h < d.H; ++h) asum += a[h];
  const float log_eps = logf(eps);
  float acc = 0.f;
  for (int h = 0; h < d.H; ++h) {
    const float ah = a[h];
    if (ah * bmax < eps) continue;  // block-uniform
    for (int l = threadIdx.x; l < d.L; l += blockDim.x) {
      const float p = ah * b[l];
      if (p >= eps) acc += p * (logf(p) - log_eps);
    }
  }
  const float tot = block_sum(acc, ws);
  const float csum = block_sum(commit, ws);
  if (threadIdx.x == 0) {
    atomicAdd(&stats[0], -(log_eps * (asum * bsum) + tot));
    atomicAdd(&stats[1], csum);
  }
}

// entropy of each codebook's batch-mean distribution + G2 = dL/d(avg) (scaled); single block, then the final loss
//   loss = w_e (sum_r H_r / R + w_div mean_c H(avg_c) + (1 + w_div) log C) + w_c sum (x - q)^2 / (R D)
__global__ void __launch_bounds__(1024)
    og_lfq_avg_kernel(const float* __restrict__ avg, long long ncodes, int C, long long nrow, int D, float eps,
                      float w_commit, float w_entropy, float w_div, float* __restrict__ g2, float* __restrict__ stats,
                      float* __restrict__ loss) {
  __shared__ float ws[32];
  const float gs = w_entropy * w_div / (float)nrow;
  float h_sum = 0.f;
  for (int c = 0; c < C; ++c) {
    const float* avg_c = avg + c * ncodes;
    float acc = 0.f;
    for (long long j = threadIdx.x; j < ncodes; j += blockDim.x) {
      const float p = avg_c[j];
      const float lp = logf(fmaxf(p, eps));
      acc += p * lp;
      if (g2) g2[c * ncodes + j] = -(lp + (p >= eps ? 1.f : 0.f)) * gs;
    }
    h_sum += -block_sum(acc, ws);
  }
  if (threadIdx.x == 0) {
    const float h_avg = h_sum / (float)C;
    stats[2] = h_avg;
    const float inp_ent = stats[0] / (float)nrow;
    const float commit = stats[1] / ((float)nrow * (float)D);
    float ent = inp_ent + w_div * h_avg;
    if (C > 1) ent += (1.f + w_div) * logf((float)C);  // the duplicated codes; no gradient
    loss[0] = ent * w_entropy + commit * w_commit;
  }
}

// ------------------------------------------------------------------------------------------------
// generic small fp32 GEMM on CUDA cores: C[i][j] = alpha * sum_k X[i*sxi + k*sxk] * Y[j*syj + k*syk]
// 64x64 tile, 16-deep, 256 threads (4x4 per thread). Batched over blockIdx.z (one codebook each): X, Y and C
// start sxz, syz and scz elements further per batch.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    og_sgemm_kernel(const float* __restrict__ X, long long sxi, long long sxk, long long sxz,
                    const float* __restrict__ Y, long long syj, long long syk, long long syz, float* __restrict__ C,
                    long long ldc, long long scz, int M, int N, int K, float alpha) {
  __shared__ float xs[16][65];
  __shared__ float ys[16][65];
  X += blockIdx.z * sxz;
  Y += blockIdx.z * syz;
  C += blockIdx.z * scz;
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
// backward, one block per row r = n * C + c (token n, codebook c), R = N C rows
//   dx[d] = gl * 2 beta * ( M[d] - Gbar * tanh[d] ) + gl * w_c * 2 (x - q) / (R D) + dout[d]
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLfqThreads)
    og_lfq_bwd_kernel(const float* __restrict__ x, int ldx, const LfqDims d, int C, float eps, float beta,
                      long long nrow, float w_commit, float w_entropy, const float* __restrict__ U,
                      const float* __restrict__ Vm, const float* __restrict__ gloss, const float* __restrict__ dout,
                      int ld_dout, float* __restrict__ dx_f32, __nv_bfloat16* __restrict__ dx_bf16, int ld_dx) {
  extern __shared__ float sh[];
  float* sp = sh;
  float* sm = sp + 32;
  float* ws = sm + 32;
  float* red = ws + 32;  // [kMaxD + 1] reduced sums
  float* a = red + 32;
  float* b = a + d.H;
  const long long r = blockIdx.x;
  const long long n = r / C;
  const int col0 = (int)(r - n * C) * d.D;
  const float* xr = x + n * ldx + col0;
  build_ab(xr, d, beta, sp, sm, a, b);

  float bmax = 0.f;
  for (int l = 0; l < d.L; ++l) bmax = fmaxf(bmax, b[l]);
  const float log_eps = logf(eps);

  // per-sample part: val = p (log p - log eps + 1) over pairs with p >= eps
  float m[kMaxD];
#pragma unroll
  for (int i = 0; i < kMaxD; ++i) m[i] = 0.f;
  float w1 = 0.f;
  for (int h = 0; h < d.H; ++h) {
    const float ah = a[h];
    if (ah * bmax < eps) continue;
    for (int l = threadIdx.x; l < d.L; l += blockDim.x) {
      const float p = ah * b[l];
      if (p >= eps) {
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
    const float au = a[h] * U[r * d.H + h];
    g2bar += au;
#pragma unroll
    for (int i = 0; i < kMaxD; ++i)
      if (i < d.D1) m2[i] += ((h >> (d.D1 - 1 - i)) & 1) ? au : -au;
  }
  for (int l = threadIdx.x; l < d.L; l += blockDim.x) {
    const float bv = b[l] * Vm[r * d.L + l];
#pragma unroll
    for (int i = 0; i < kMaxD; ++i)
      if (i >= d.D1 && i < d.D) m2[i] += ((l >> (d.D - 1 - i)) & 1) ? bv : -bv;
  }
  const float w1s = block_sum(w1, ws);
  const float g2s = block_sum(g2bar, ws);
  const float gl = gloss ? *gloss : 1.f;
  const float we_n = w_entropy / (float)nrow;
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
    g += gl * w_commit * 2.f * (v - q) / ((float)nrow * (float)d.D);
    if (dout) g += dout[n * ld_dout + col0 + i];
    if (dx_f32) dx_f32[n * ld_dx + col0 + i] = g;
    if (dx_bf16) dx_bf16[n * ld_dx + col0 + i] = __float2bfloat16_rn(g);
  }
  if (col0 + d.D != C * d.D) return;  // the last codebook's row zeroes the pad columns [C*D, ld_dx)
  if (dx_bf16)
    for (int i = C * d.D + threadIdx.x; i < ld_dx; i += blockDim.x) dx_bf16[n * ld_dx + i] = __float2bfloat16_rn(0.f);
  if (dx_f32)
    for (int i = C * d.D + threadIdx.x; i < ld_dx; i += blockDim.x) dx_f32[n * ld_dx + i] = 0.f;
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

static int launch_sgemm(const float* X, long long sxi, long long sxk, long long sxz, const float* Y, long long syj,
                        long long syk, long long syz, float* C, long long ldc, long long scz, int M, int N, int K,
                        int batch, float alpha, cudaStream_t s) {
  dim3 grid((N + 63) / 64, (M + 63) / 64, batch);
  og_sgemm_kernel<<<grid, 256, 0, s>>>(X, sxi, sxk, sxz, Y, syj, syk, syz, C, ldc, scz, M, N, K, alpha);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

// Workspace (floats), R = ntok * C rows: A[R*H] B[R*L] U[R*H] V[R*L] avg[C*2^D] g2[C*2^D] stats[4]
static size_t lfq_workspace_floats(int64_t ntok, const LfqDims& d, int C) {
  const size_t rows = (size_t)ntok * (size_t)C;
  return rows * (size_t)(d.H + d.L) * 2 + ((size_t)C << d.D) * 2 + 4;
}

struct LfqWorkspace {
  float *A, *B, *U, *V, *avg, *g2, *stats;
};

static LfqWorkspace lfq_workspace(void* workspace, int64_t ntok, const LfqDims& d, int C) {
  const size_t rows = (size_t)ntok * (size_t)C;
  LfqWorkspace w;
  w.A = reinterpret_cast<float*>(workspace);
  w.B = w.A + rows * d.H;
  w.U = w.B + rows * d.L;
  w.V = w.U + rows * d.H;
  w.avg = w.V + rows * d.L;
  w.g2 = w.avg + ((size_t)C << d.D);
  w.stats = w.g2 + ((size_t)C << d.D);
  return w;
}

// forward on validated arguments: 1 + 3 launches in training (stats memset, rows, batch means, entropy + loss)
static int lfq_fwd(const float* x, int ldx, int64_t ntok, int D, int C, float beta, int training, float w_commit,
                   float w_entropy, float w_div, float* out_f32, void* out_bf16, int ld_bf16, int64_t* idx,
                   float* loss, void* workspace, cudaStream_t s) {
  const LfqDims d = make_dims(D);
  const float eps = kEps * (float)C;
  const long long nrow = (long long)ntok * C;
  LfqWorkspace w = {};
  if (training) {
    w = lfq_workspace(workspace, ntok, d, C);
    OG_CHECK_CUDA(cudaMemsetAsync(w.stats, 0, 4 * sizeof(float), s));
  }
  const size_t smem = sizeof(float) * (96 + d.H + d.L);
  og_lfq_fwd_kernel<<<(unsigned)nrow, kLfqThreads, smem, s>>>(x, ldx, d, C, eps, beta, training, out_f32,
                                                              (__nv_bfloat16*)out_bf16, ld_bf16, (long long*)idx, w.A,
                                                              w.B, w.stats);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  if (!training) return OG_OK;
  // avg_c[h][l] = (1/N) sum_n A[n*C+c][h] B[n*C+c][l], one batch per codebook
  const long long ncodes = 1LL << D;
  int r = launch_sgemm(w.A, 1, (long long)C * d.H, d.H, w.B, 1, (long long)C * d.L, d.L, w.avg, d.L, ncodes, d.H,
                       d.L, (int)ntok, C, 1.f / (float)ntok, s);
  if (r != OG_OK) return r;
  og_lfq_avg_kernel<<<1, 1024, 0, s>>>(w.avg, ncodes, C, nrow, D, eps, w_commit, w_entropy, w_div, w.g2, w.stats,
                                       loss);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

// backward on validated arguments: 3 launches (U, V, rows)
static int lfq_bwd(const float* x, int ldx, int64_t ntok, int D, int C, float beta, float w_commit, float w_entropy,
                   const float* gloss, const float* dout, int ld_dout, float* dx_f32, void* dx_bf16, int ld_dx,
                   void* workspace, cudaStream_t s) {
  const LfqDims d = make_dims(D);
  const float eps = kEps * (float)C;
  const long long nrow = (long long)ntok * C;
  const LfqWorkspace w = lfq_workspace(workspace, ntok, d, C);
  const long long ncodes = 1LL << D;
  // per codebook c, over its rows r = n*C + c:  U[r][h] = sum_l B[r][l] g2_c[h][l] ;  V[r][l] = sum_h A[r][h] g2_c[h][l]
  int r = launch_sgemm(w.B, (long long)C * d.L, 1, d.L, w.g2, d.L, 1, ncodes, w.U, (long long)C * d.H, d.H, (int)ntok,
                       d.H, d.L, C, 1.f, s);
  if (r != OG_OK) return r;
  r = launch_sgemm(w.A, (long long)C * d.H, 1, d.H, w.g2, 1, d.L, ncodes, w.V, (long long)C * d.L, d.L, (int)ntok, d.L,
                   d.H, C, 1.f, s);
  if (r != OG_OK) return r;
  const size_t smem = sizeof(float) * (128 + d.H + d.L);
  og_lfq_bwd_kernel<<<(unsigned)nrow, kLfqThreads, smem, s>>>(x, ldx, d, C, eps, beta, nrow, w_commit, w_entropy,
                                                              w.U, w.V, gloss, dout, ld_dout, dx_f32,
                                                              (__nv_bfloat16*)dx_bf16, ld_dx);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

}  // namespace og

using namespace og;

extern "C" size_t og_lfq_workspace_bytes(int64_t ntok, int D) {
  if (D < 1 || D > kMaxD) return 0;
  return sizeof(float) * lfq_workspace_floats(ntok, make_dims(D), 1);
}

extern "C" int og_lfq_fwd(const float* x, int ldx, int64_t ntok, int D, float beta, int training, float w_commit,
                          float w_entropy, float w_div, float* out_f32, void* out_bf16, int ld_bf16, int64_t* idx,
                          float* loss, void* workspace, og_stream_t stream) {
  OG_REQUIRE(x && idx && ntok > 0, "lfq_fwd: bad arguments");
  OG_REQUIRE(D >= 1 && D <= kMaxD, "lfq_fwd: codebook_dim=%d outside [1,%d]", D, kMaxD);
  OG_REQUIRE(!training || (loss && workspace), "lfq_fwd: training needs loss and workspace");
  return lfq_fwd(x, ldx, ntok, D, 1, beta, training, w_commit, w_entropy, w_div, out_f32, out_bf16, ld_bf16, idx, loss,
                 workspace, (cudaStream_t)stream);
}

extern "C" int og_lfq_bwd(const float* x, int ldx, int64_t ntok, int D, float beta, float w_commit, float w_entropy,
                          const float* gloss, const float* dout, int ld_dout, float* dx_f32, void* dx_bf16, int ld_dx,
                          void* workspace, og_stream_t stream) {
  OG_REQUIRE(x && workspace && (dx_f32 || dx_bf16) && ld_dx >= D, "lfq_bwd: bad arguments");
  OG_REQUIRE(D >= 1 && D <= kMaxD, "lfq_bwd: codebook_dim=%d outside [1,%d]", D, kMaxD);
  return lfq_bwd(x, ldx, ntok, D, 1, beta, w_commit, w_entropy, gloss, dout, ld_dout, dx_f32, dx_bf16, ld_dx, workspace,
                 (cudaStream_t)stream);
}

// rows r = n * C + c index the grid and must fit an int; each codebook is one SGEMM batch (grid z <= 65535)
static constexpr int kMaxCodebooks = 65535;
static bool lfq_rows_fit(int64_t ntok, int C) {
  return ntok > 0 && C >= 1 && C <= kMaxCodebooks && ntok <= INT_MAX / C;
}

extern "C" size_t og_lfq_multi_workspace_bytes(int64_t ntok, int D, int n_codebook) {
  if (D < 1 || D > kMaxD || !lfq_rows_fit(ntok, n_codebook)) return 0;
  return sizeof(float) * lfq_workspace_floats(ntok, make_dims(D), n_codebook);
}

extern "C" int og_lfq_multi_fwd(const float* x, int ldx, int64_t ntok, int D, int n_codebook, float beta, int training,
                                float w_commit, float w_entropy, float w_div, float* out_f32, void* out_bf16,
                                int ld_bf16, int64_t* idx, float* loss, void* workspace, og_stream_t stream) {
  const int C = n_codebook;
  OG_REQUIRE(x && idx, "lfq_multi_fwd: bad arguments");
  OG_REQUIRE(D >= 1 && D <= kMaxD, "lfq_multi_fwd: codebook_dim=%d outside [1,%d]", D, kMaxD);
  OG_REQUIRE(lfq_rows_fit(ntok, C), "lfq_multi_fwd: ntok=%lld, n_codebook=%d: need ntok >= 1, n_codebook in [1,%d] "
             "and ntok * n_codebook <= %d", (long long)ntok, C, kMaxCodebooks, INT_MAX);
  OG_REQUIRE((long long)ldx >= (long long)C * D, "lfq_multi_fwd: ldx=%d < n_codebook * codebook_dim", ldx);
  OG_REQUIRE(!out_bf16 || (long long)ld_bf16 >= (long long)C * D,
             "lfq_multi_fwd: ld_bf16=%d < n_codebook * codebook_dim", ld_bf16);
  OG_REQUIRE(!training || (loss && workspace), "lfq_multi_fwd: training needs loss and workspace");
  return lfq_fwd(x, ldx, ntok, D, C, beta, training, w_commit, w_entropy, w_div, out_f32, out_bf16, ld_bf16, idx, loss,
                 workspace, (cudaStream_t)stream);
}

extern "C" int og_lfq_multi_bwd(const float* x, int ldx, int64_t ntok, int D, int n_codebook, float beta,
                                float w_commit, float w_entropy, const float* gloss, const float* dout, int ld_dout,
                                float* dx_f32, void* dx_bf16, int ld_dx, void* workspace, og_stream_t stream) {
  const int C = n_codebook;
  OG_REQUIRE(x && workspace && (dx_f32 || dx_bf16), "lfq_multi_bwd: bad arguments");
  OG_REQUIRE(D >= 1 && D <= kMaxD, "lfq_multi_bwd: codebook_dim=%d outside [1,%d]", D, kMaxD);
  OG_REQUIRE(lfq_rows_fit(ntok, C), "lfq_multi_bwd: ntok=%lld, n_codebook=%d: need ntok >= 1, n_codebook in [1,%d] "
             "and ntok * n_codebook <= %d", (long long)ntok, C, kMaxCodebooks, INT_MAX);
  const long long cd = (long long)C * D;
  OG_REQUIRE(ldx >= cd && ld_dx >= cd && (!dout || ld_dout >= cd),
             "lfq_multi_bwd: ldx=%d, ld_dx=%d, ld_dout=%d: each must be >= n_codebook * codebook_dim", ldx, ld_dx,
             ld_dout);
  return lfq_bwd(x, ldx, ntok, D, C, beta, w_commit, w_entropy, gloss, dout, ld_dout, dx_f32, dx_bf16, ld_dx, workspace,
                 (cudaStream_t)stream);
}
