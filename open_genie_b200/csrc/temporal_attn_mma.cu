// temporal_attn_mma.cu — tensor-core form of the temporal (causal, T <= 16, d_head = 64) attention.
//
// STATUS: checked by tests/test_gpu_attention.py, tests/test_gpu_attention_paths.py and the full-size LatentAction /
// Dynamics parity tests; always used for d_head = 64, T <= 16 (temporal_mma_enabled in attention_rows.cu), the per-lane
// kernels there cover the other shapes.
// SASS: LDSM / HMMA.16816.F32.BF16.
//
// Why: one (batch, pixel, head) task is a 16 x 16 x 64 score tile and a 16 x 64 x 16 value product. The per-lane
// dot-product kernels spend ~2.5 K instructions per task and run ~4x above their HBM roofline time; with
// mma.sync.m16n8k16 the same task is 16 HMMA instructions forward (40 backward). wgmma is the wrong tool here:
// its M = 64 warpgroup tiles would need 4 unrelated tasks packed block-diagonally.
//
// Reference semantics: TemporalAttention.forward -> Attention.forward (genie/module/attention.py:309-371,
// 199-239): SDPA(q, k, v, is_causal=True, scale = n_head * d_head**-0.5) per pixel over t, optional (B, T, C)
// conditioning K/V broadcast over pixels (kv_bcast).
//
// Layouts. Rows of a task are staged with 16-byte loads into shared memory with a 144-byte pitch (bank-conflict
// free for ldmatrix); the fragment conventions and helpers are in temporal_mma_frag.cuh.
#include "og_host.cuh"
#include "og_ptx.cuh"
#include "temporal_mma_frag.cuh"

namespace og {
extern std::atomic<uint64_t> g_launches;

namespace tmma {
constexpr int kT = 16;
constexpr int kMat = kT * kPitch;           // one staged 16 x 64 matrix: 2304 B
constexpr int kPPitch = 48;                 // bytes per row of the 16 x 16 bf16 P / dS tiles (32 data + 16 pad)
constexpr int kPMat = kT * kPPitch;         // 768 B

// stage T rows of 64 bf16 (row pitch `pitch_elems` in global memory) into a 16 x 144-byte tile; rows >= T are zero
__device__ __forceinline__ void stage_rows(uint8_t* dst, const __nv_bfloat16* src, long long pitch_elems, int T,
                                           int lane) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = lane + 32 * i, r = idx >> 3, ch = idx & 7;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r < T) v = __ldg(reinterpret_cast<const uint4*>(src + (long long)r * pitch_elems) + ch);
    *reinterpret_cast<uint4*>(dst + r * kPitch + ch * 16) = v;
  }
}

// scores of one task: s[nt][.] = (Q K^T) fragments (unscaled)
__device__ __forceinline__ void scores(float (&s)[2][4], const uint8_t* qs, const uint8_t* ks, int lane) {
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) s[nt][e] = 0.f;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t a[4];
    load_a(a, qs, kk * 16, lane);
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      uint32_t b[2];
      load_b_rows(b, ks, nt * 8, kk * 16, lane);
      mma16816(s[nt], a, b[0], b[1]);
    }
  }
}

// causal softmax over the fragments; returns un-normalised p (in place) and the inverse row sums of rows g, g+8
__device__ __forceinline__ void causal_softmax(float (&s)[2][4], int T, float scale, int lane, float& inv0, float& inv1) {
  const int g = lane >> 2, q = lane & 3;
  float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int col = nt * 8 + q * 2 + e;
      s[nt][e] = (col <= g && col < T) ? s[nt][e] * scale : -INFINITY;
      s[nt][2 + e] = (col <= g + 8 && col < T) ? s[nt][2 + e] * scale : -INFINITY;
      m0 = fmaxf(m0, s[nt][e]);
      m1 = fmaxf(m1, s[nt][2 + e]);
    }
  m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
  m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
  m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
  m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
  if (g >= T) m0 = 0.f;       // padded query rows: everything masked, keep the arithmetic finite
  if (g + 8 >= T) m1 = 0.f;
  float l0 = 0.f, l1 = 0.f;
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      s[nt][e] = __expf(s[nt][e] - m0);
      s[nt][2 + e] = __expf(s[nt][2 + e] - m1);
      l0 += s[nt][e];
      l1 += s[nt][2 + e];
    }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  inv0 = l0 > 0.f ? 1.f / l0 : 0.f;
  inv1 = l1 > 0.f ? 1.f / l1 : 0.f;
}

struct Task {
  long long p;
  int b, h;
};
__device__ __forceinline__ Task decode(long long task, long long P, int nh) {
  Task t;
  t.p = task % P;
  const long long bh = task / P;
  t.h = (int)(bh % nh);
  t.b = (int)(bh / nh);
  return t;
}

// write a [16 rows][64 cols] fp32 fragment set (8 n-tiles) as bf16 into a staged tile (row pitch kPitch)
__device__ __forceinline__ void frags_to_tile(uint8_t* tile, const float (&o)[8][4], float sc0, float sc1, int lane) {
  const int g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    *reinterpret_cast<uint32_t*>(tile + g * kPitch + (nt * 8 + q * 2) * 2) = pack_bf16x2(o[nt][0] * sc0, o[nt][1] * sc0);
    *reinterpret_cast<uint32_t*>(tile + (g + 8) * kPitch + (nt * 8 + q * 2) * 2) =
        pack_bf16x2(o[nt][2] * sc1, o[nt][3] * sc1);
  }
}

// store T rows of a staged bf16 tile to global rows of pitch `pitch_elems` (+ optional bf16 residual, added in fp32)
__device__ __forceinline__ void tile_to_global(const uint8_t* tile, __nv_bfloat16* dst, const __nv_bfloat16* res,
                                               long long pitch_elems, int T, int lane) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = lane + 32 * i, r = idx >> 3, ch = idx & 7;
    if (r >= T) continue;
    uint4 v = *reinterpret_cast<const uint4*>(tile + r * kPitch + ch * 16);
    if (res) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(res + (long long)r * pitch_elems) + ch);
      const __nv_bfloat162* a = reinterpret_cast<const __nv_bfloat162*>(&v);
      const __nv_bfloat162* b = reinterpret_cast<const __nv_bfloat162*>(&u);
      uint32_t w[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 fa = __bfloat1622float2(a[e]), fb = __bfloat1622float2(b[e]);
        w[e] = pack_bf16x2(fa.x + fb.x, fa.y + fb.y);
      }
      v = make_uint4(w[0], w[1], w[2], w[3]);
    }
    *(reinterpret_cast<uint4*>(dst + (long long)r * pitch_elems) + ch) = v;
  }
}

__global__ void __launch_bounds__(128)
    og_temporal_attn_fwd_mma_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                    const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ res,
                                    __nv_bfloat16* __restrict__ out, int B, int T, long long P, int C, int nh,
                                    float scale, int kv_bcast) {
  extern __shared__ __align__(16) uint8_t smem_t[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint8_t* qs = smem_t + warp * 3 * kMat;
  uint8_t* ks = qs + kMat;
  uint8_t* vs = ks + kMat;
  const long long ntask = (long long)B * P * nh;
  const long long nw = (long long)gridDim.x * 4, w = (long long)blockIdx.x * 4 + warp;
  const long long per = (ntask + nw - 1) / nw;
  const long long t_begin = w * per, t_end = t_begin + per < ntask ? t_begin + per : ntask;
  const long long qpitch = P * (long long)C;
  for (long long task = t_begin; task < t_end; ++task) {
    const Task tk = decode(task, P, nh);
    const long long q0 = (((long long)tk.b * T) * P + tk.p) * C + tk.h * kD;   // row t adds t * P * C
    const long long k0 = kv_bcast ? ((long long)tk.b * T) * C + tk.h * kD : q0;
    const long long kpitch = kv_bcast ? (long long)C : qpitch;
    __syncwarp();
    stage_rows(qs, q + q0, qpitch, T, lane);
    stage_rows(ks, k + k0, kpitch, T, lane);
    stage_rows(vs, v + k0, kpitch, T, lane);
    __syncwarp();
    float s[2][4];
    scores(s, qs, ks, lane);
    float inv0, inv1;
    causal_softmax(s, T, scale, lane, inv0, inv1);
    uint32_t pa[4];
    pack_a(pa, s);
    float o[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) o[nt][e] = 0.f;
      uint32_t b[2];
      load_b_cols(b, vs, nt * 8, lane);
      mma16816(o[nt], pa, b[0], b[1]);
    }
    __syncwarp();  // every lane is done reading Q: reuse its tile as the output staging
    frags_to_tile(qs, o, inv0, inv1, lane);
    __syncwarp();
    tile_to_global(qs, out + q0, res ? res + q0 : nullptr, qpitch, T, lane);
  }
}

__global__ void __launch_bounds__(128)
    og_temporal_attn_bwd_mma_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                    const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ dout,
                                    __nv_bfloat16* __restrict__ dq, __nv_bfloat16* __restrict__ dk,
                                    __nv_bfloat16* __restrict__ dv, float* __restrict__ dk_b, float* __restrict__ dv_b,
                                    int B, int T, long long P, int C, int nh, float scale, int kv_bcast) {
  extern __shared__ __align__(16) uint8_t smem_t[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kPerWarp = 4 * kMat + 2 * kPMat;
  uint8_t* qs = smem_t + warp * kPerWarp;
  uint8_t* ks = qs + kMat;
  uint8_t* vs = ks + kMat;
  uint8_t* dos = vs + kMat;
  uint8_t* ps = dos + kMat;     // P  bf16 [query][key], pitch kPPitch
  uint8_t* dss = ps + kPMat;    // dS bf16 [query][key]
  const int g = lane >> 2, qd = lane & 3;
  const long long ntask = (long long)B * P * nh;
  const long long nw = (long long)gridDim.x * 4, w = (long long)blockIdx.x * 4 + warp;
  const long long per = (ntask + nw - 1) / nw;
  const long long t_begin = w * per, t_end = t_begin + per < ntask ? t_begin + per : ntask;
  const long long qpitch = P * (long long)C;
  // broadcast-K/V gradient accumulators (fragments: rows = keys g, g+8; cols = nt*8 + 2 qd + e), kept across the
  // pixels of one (b, h)
  float dk_acc[8][4], dv_acc[8][4];
#pragma unroll
  for (int nt = 0; nt < 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) dk_acc[nt][e] = dv_acc[nt][e] = 0.f;
  long long acc_bh = -1;
  auto flush = [&]() {
    if (acc_bh < 0) return;
    const int hh = (int)(acc_bh % nh), bb = (int)(acc_bh / nh);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = g + (e >> 1) * 8, col = nt * 8 + qd * 2 + (e & 1);
        if (row < T) {
          const long long o = ((long long)bb * T + row) * C + hh * kD + col;
          atomicAdd(dk_b + o, dk_acc[nt][e]);
          atomicAdd(dv_b + o, dv_acc[nt][e]);
        }
        dk_acc[nt][e] = dv_acc[nt][e] = 0.f;
      }
  };
  for (long long task = t_begin; task < t_end; ++task) {
    const Task tk = decode(task, P, nh);
    const long long q0 = (((long long)tk.b * T) * P + tk.p) * C + tk.h * kD;
    const long long k0 = kv_bcast ? ((long long)tk.b * T) * C + tk.h * kD : q0;
    const long long kpitch = kv_bcast ? (long long)C : qpitch;
    const long long bh = (long long)tk.b * nh + tk.h;
    if (kv_bcast && bh != acc_bh) {
      flush();
      acc_bh = bh;
    }
    __syncwarp();
    stage_rows(qs, q + q0, qpitch, T, lane);
    stage_rows(ks, k + k0, kpitch, T, lane);
    stage_rows(vs, v + k0, kpitch, T, lane);
    stage_rows(dos, dout + q0, qpitch, T, lane);
    __syncwarp();
    // P = softmax(scale * Q K^T) (normalised, fp32 fragments)
    float p[2][4];
    scores(p, qs, ks, lane);
    float inv0, inv1;
    causal_softmax(p, T, scale, lane, inv0, inv1);
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      p[nt][0] *= inv0;
      p[nt][1] *= inv0;
      p[nt][2] *= inv1;
      p[nt][3] *= inv1;
    }
    // dP = dO V^T
    float dp[2][4];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) dp[nt][e] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t a[4];
      load_a(a, dos, kk * 16, lane);
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        uint32_t b[2];
        load_b_rows(b, vs, nt * 8, kk * 16, lane);
        mma16816(dp[nt], a, b[0], b[1]);
      }
    }
    // delta = sum_s P dP per query row ; dS = P (dP - delta) * scale
    float d0 = 0.f, d1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      d0 += p[nt][0] * dp[nt][0] + p[nt][1] * dp[nt][1];
      d1 += p[nt][2] * dp[nt][2] + p[nt][3] * dp[nt][3];
    }
    d0 += __shfl_xor_sync(0xffffffffu, d0, 1);
    d0 += __shfl_xor_sync(0xffffffffu, d0, 2);
    d1 += __shfl_xor_sync(0xffffffffu, d1, 1);
    d1 += __shfl_xor_sync(0xffffffffu, d1, 2);
    float ds[2][4];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      ds[nt][0] = p[nt][0] * (dp[nt][0] - d0) * scale;
      ds[nt][1] = p[nt][1] * (dp[nt][1] - d0) * scale;
      ds[nt][2] = p[nt][2] * (dp[nt][2] - d1) * scale;
      ds[nt][3] = p[nt][3] * (dp[nt][3] - d1) * scale;
    }
    // P and dS tiles [query][key] for the transposed products
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      const int col = (nt * 8 + qd * 2) * 2;
      *reinterpret_cast<uint32_t*>(ps + g * kPPitch + col) = pack_bf16x2(p[nt][0], p[nt][1]);
      *reinterpret_cast<uint32_t*>(ps + (g + 8) * kPPitch + col) = pack_bf16x2(p[nt][2], p[nt][3]);
      *reinterpret_cast<uint32_t*>(dss + g * kPPitch + col) = pack_bf16x2(ds[nt][0], ds[nt][1]);
      *reinterpret_cast<uint32_t*>(dss + (g + 8) * kPPitch + col) = pack_bf16x2(ds[nt][2], ds[nt][3]);
    }
    // dQ = dS K   (A = dS fragments, B[k = key][n = d] = K[key][d])
    uint32_t dsa[4];
    pack_a(dsa, ds);
    float acc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[nt][e] = 0.f;
      uint32_t b[2];
      load_b_cols(b, ks, nt * 8, lane);
      mma16816(acc[nt], dsa, b[0], b[1]);
    }
    __syncwarp();  // P / dS tiles complete; all lanes are past their last read of the K fragments above
    // A fragments of P^T and dS^T: transposed 8x8 blocks of the [query][key] tiles
    uint32_t pta[4], dsta[4];
    {
      const int r = (lane & 7) + ((lane >> 4) & 1) * 8, c = ((lane >> 3) & 1) * 8;
      ldsm_x4_trans(pta, smem_u32(ps + r * kPPitch + c * 2));
      ldsm_x4_trans(dsta, smem_u32(dss + r * kPPitch + c * 2));
    }
    // dV = P^T dO, dK = dS^T Q
    float dvf[8][4], dkf[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) dvf[nt][e] = dkf[nt][e] = 0.f;
      uint32_t b[2];
      load_b_cols(b, dos, nt * 8, lane);
      mma16816(dvf[nt], pta, b[0], b[1]);
      load_b_cols(b, qs, nt * 8, lane);
      mma16816(dkf[nt], dsta, b[0], b[1]);
    }
    __syncwarp();  // every lane is done with the staged Q / K / V / dO: reuse the tiles for the outputs
    frags_to_tile(qs, acc, 1.f, 1.f, lane);
    if (kv_bcast) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          dk_acc[nt][e] += dkf[nt][e];
          dv_acc[nt][e] += dvf[nt][e];
        }
    } else {
      frags_to_tile(ks, dkf, 1.f, 1.f, lane);
      frags_to_tile(vs, dvf, 1.f, 1.f, lane);
    }
    __syncwarp();
    tile_to_global(qs, dq + q0, nullptr, qpitch, T, lane);
    if (!kv_bcast) {
      tile_to_global(ks, dk + q0, nullptr, qpitch, T, lane);
      tile_to_global(vs, dv + q0, nullptr, qpitch, T, lane);
    }
  }
  if (kv_bcast) flush();
}

}  // namespace tmma

// launchers used by og_temporal_attn_fwd / og_temporal_attn_bwd (attention_rows.cu) for d_head = 64, T <= 16
int launch_temporal_fwd_mma(const void* q, const void* k, const void* v, const void* residual, void* out, int B, int T,
                            long long P, int C, int n_head, float scale, int kv_bcast, cudaStream_t stream) {
  const long long ntask = (long long)B * P * n_head;
  long long grid = (ntask + 3) / 4;
  if (grid > (long long)num_sms() * 12) grid = (long long)num_sms() * 12;
  const size_t smem = (size_t)4 * 3 * tmma::kMat;
  tmma::og_temporal_attn_fwd_mma_kernel<<<(unsigned)grid, 128, smem, stream>>>(
      (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)residual,
      (__nv_bfloat16*)out, B, T, P, C, n_head, scale, kv_bcast);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

int launch_temporal_bwd_mma(const void* q, const void* k, const void* v, const void* dout, void* dq, void* dk, void* dv,
                            float* dk_b, float* dv_b, int B, int T, long long P, int C, int n_head, float scale,
                            int kv_bcast, cudaStream_t stream) {
  const long long ntask = (long long)B * P * n_head;
  long long grid = (ntask + 3) / 4;
  if (grid > (long long)num_sms() * 4) grid = (long long)num_sms() * 4;
  const size_t smem = (size_t)4 * (4 * tmma::kMat + 2 * tmma::kPMat);
  tmma::og_temporal_attn_bwd_mma_kernel<<<(unsigned)grid, 128, smem, stream>>>(
      (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)dout,
      (__nv_bfloat16*)dq, (__nv_bfloat16*)dk, (__nv_bfloat16*)dv, dk_b, dv_b, B, T, P, C, n_head, scale, kv_bcast);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

}  // namespace og
