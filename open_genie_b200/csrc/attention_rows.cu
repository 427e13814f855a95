// attention_rows.cu — the bandwidth-bound parts of the factored space-time attention:
//   * fused RoPE + LayerNorm (forward / backward) on NDHWC rows
//   * LayerNorm alone on the same rows (attention with embed=False, where the reference's embed is nn.Identity): the
//     same kernel bodies, templated on kRope, so the og_ln_rows_* kernels are the og_rope_ln_* ones minus the rotation
//     and the kRope = true instantiations compile to the same instructions as before the flag existed.
//     Registers (sm_90a, no spills): og_ln_rows_fwd_kernel 64, og_ln_rows_fwd_vec_kernel<1, 2, 4> 40 / 64 / 116,
//     og_ln_rows_bwd_kernel 190, og_ln_rows_bwd_vec_kernel<1, 2, 4> 72 / 128 / 248.
//   * temporal (causal, T <= 32) attention per pixel and head, forward / backward, on CUDA cores
//
// Reference (genie/module/attention.py, HEAD-valid configuration — SURVEY.md §7 H6):
//   qry = embed(qry)  -> RotaryEmbedding over the FULL channel dim, interleaved pairs, fp32 angles (48-94)
//   qry = norm(qry)   -> nn.LayerNorm(n_head*d_head)                                              (219-220)
//   q = k = v = qry   (to_q/to_k/to_v are Identity; with a temporal cond: k = to_k(cond), v = to_v(cond))
//   SDPA(q, k, v, is_causal, scale = n_head * d_head**-0.5)                                       (195, 229-234)
// Spatial sequences run over (h w) of one frame, temporal ones over t of one pixel. In NDHWC memory both
// are ROW-WISE operations on the same [B*T*H*W][C] matrix — only the position index of a row differs —
// so no 'b c t h w -> (b h w) t c' transposition copy is ever made (the reference makes two per block).
#include "og_host.cuh"
#include "og_ptx.cuh"

namespace og {
extern std::atomic<uint64_t> g_launches;

static constexpr int kMaxPairsPerLane = 16;  // C <= 1024

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------
// RoPE + LayerNorm forward: one warp per row. Lane l owns channel pairs l, l+32, ...
// pos(row) = (row / pos_div) % pos_mod   (spatial: div 1, mod H*W ; temporal: div H*W, mod T)
// ------------------------------------------------------------------------------------------------
template <bool kRope>
__device__ __forceinline__ void rope_ln_fwd_rows(const __nv_bfloat162* __restrict__ x, const float* __restrict__ freq,
                                                 const float* __restrict__ gamma, const float* __restrict__ beta,
                                                 float eps, __nv_bfloat162* __restrict__ y, long long rows, int C,
                                                 long long pos_div, int pos_mod) {
  const int lane = threadIdx.x & 31;
  const int pairs = C >> 1;
  const int ppl = (pairs + 31) >> 5;
  const long long warp0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long row = warp0; row < rows; row += nwarps) {
    const float pos = kRope ? (float)((row / pos_div) % pos_mod) : 0.f;
    float r0[kMaxPairsPerLane], r1[kMaxPairsPerLane];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxPairsPerLane; ++j) {
      const int p = lane + 32 * j;
      if (j < ppl && p < pairs) {
        const float2 v = __bfloat1622float2(x[row * pairs + p]);
        if constexpr (kRope) {
          float sn, cs;
          sincosf(pos * __ldg(freq + p), &sn, &cs);
          r0[j] = v.x * cs - v.y * sn;
          r1[j] = v.y * cs + v.x * sn;
        } else {
          r0[j] = v.x;
          r1[j] = v.y;
        }
        s += r0[j] + r1[j];
      } else {
        r0[j] = r1[j] = 0.f;
      }
    }
    const float mean = warp_sum(s) / (float)C;
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxPairsPerLane; ++j) {
      const int p = lane + 32 * j;
      if (j < ppl && p < pairs) {
        const float a = r0[j] - mean, b = r1[j] - mean;
        ss += a * a + b * b;
      }
    }
    const float rstd = rsqrtf(warp_sum(ss) / (float)C + eps);
#pragma unroll
    for (int j = 0; j < kMaxPairsPerLane; ++j) {
      const int p = lane + 32 * j;
      if (j < ppl && p < pairs) {
        const float o0 = (r0[j] - mean) * rstd * __ldg(gamma + 2 * p) + __ldg(beta + 2 * p);
        const float o1 = (r1[j] - mean) * rstd * __ldg(gamma + 2 * p + 1) + __ldg(beta + 2 * p + 1);
        y[row * pairs + p] = __floats2bfloat162_rn(o0, o1);
      }
    }
  }
}

__global__ void __launch_bounds__(256)
    og_rope_ln_fwd_kernel(const __nv_bfloat162* __restrict__ x, const float* __restrict__ freq,
                          const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                          __nv_bfloat162* __restrict__ y, long long rows, int C, long long pos_div, int pos_mod) {
  rope_ln_fwd_rows<true>(x, freq, gamma, beta, eps, y, rows, C, pos_div, pos_mod);
}

__global__ void __launch_bounds__(256)
    og_ln_rows_fwd_kernel(const __nv_bfloat162* __restrict__ x, const float* __restrict__ gamma,
                          const float* __restrict__ beta, float eps, __nv_bfloat162* __restrict__ y, long long rows,
                          int C) {
  rope_ln_fwd_rows<false>(x, nullptr, gamma, beta, eps, y, rows, C, 1, 1);
}

// Vector form of the forward pass for C % 256 == 0 (same lane -> channel mapping as the vector backward below:
// lane l owns the 4 consecutive pairs [128 j + 4 l, +4) of chunk j, i.e. one 16-byte load / store per chunk).
template <int NCH, bool kRope>
__device__ __forceinline__ void rope_ln_fwd_vec_rows(const uint4* __restrict__ x, const float* __restrict__ freq,
                                                     const float* __restrict__ gamma, const float* __restrict__ beta,
                                                     float eps, uint4* __restrict__ y, long long rows,
                                                     long long pos_div, int pos_mod, const float4* __restrict__ tab) {
  constexpr int NP = 4 * NCH;
  constexpr int C = 256 * NCH;
  constexpr int VPR = 32 * NCH;
  const int lane = threadIdx.x & 31;
  const long long warp0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  float fq[NP], gm0[NP], gm1[NP], bt0[NP], bt1[NP];
#pragma unroll
  for (int j = 0; j < NCH; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int p = 128 * j + 4 * lane + e;
      if constexpr (kRope) fq[4 * j + e] = __ldg(freq + p);
      gm0[4 * j + e] = __ldg(gamma + 2 * p);
      gm1[4 * j + e] = __ldg(gamma + 2 * p + 1);
      bt0[4 * j + e] = __ldg(beta + 2 * p);
      bt1[4 * j + e] = __ldg(beta + 2 * p + 1);
    }
  for (long long row = warp0; row < rows; row += nwarps) {
    const int ipos = kRope ? (int)((row / pos_div) % pos_mod) : 0;
    const float pos = (float)ipos;
    const long long vb = row * VPR + lane;
    uint4 ux[NCH];
#pragma unroll
    for (int j = 0; j < NCH; ++j) ux[j] = __ldg(x + vb + 32 * j);
    // (cos, sin) of this row's position: from the precomputed table (og_rope_table: the same sincosf values, computed
    // once per (frequencies, sequence length) instead of once per element — the '2d' angles reach ~4000 rad, where
    // sincosf takes its slow range-reduction path and made this pass SM-bound at 0.4 of the HBM roofline)
    float tcs[NP], tsn[NP];
    if (kRope && tab) {
      const float4* tr = tab + (long long)ipos * (C / 4);      // row of C/2 (cos, sin) pairs = C/4 float4
#pragma unroll
      for (int j = 0; j < NCH; ++j) {
        const float4 t0 = __ldg(tr + 64 * j + 2 * lane), t1 = __ldg(tr + 64 * j + 2 * lane + 1);
        tcs[4 * j] = t0.x; tsn[4 * j] = t0.y; tcs[4 * j + 1] = t0.z; tsn[4 * j + 1] = t0.w;
        tcs[4 * j + 2] = t1.x; tsn[4 * j + 2] = t1.y; tcs[4 * j + 3] = t1.z; tsn[4 * j + 3] = t1.w;
      }
    }
    float r0[NP], r1[NP];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&ux[j]);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * j + e;
        const float2 v = __bfloat1622float2(h[e]);
        if constexpr (kRope) {
          float sn, cs;
          if (tab) {
            sn = tsn[i];
            cs = tcs[i];
          } else {
            sincosf(pos * fq[i], &sn, &cs);
          }
          r0[i] = v.x * cs - v.y * sn;
          r1[i] = v.y * cs + v.x * sn;
        } else {
          r0[i] = v.x;
          r1[i] = v.y;
        }
        s += r0[i] + r1[i];
      }
    }
    const float mean = warp_sum(s) / (float)C;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NP; ++i) {
      const float a = r0[i] - mean, b = r1[i] - mean;
      ss += a * a + b * b;
    }
    const float rstd = rsqrtf(warp_sum(ss) / (float)C + eps);
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      uint4 o;
      uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * j + e;
        ow[e] = pack_bf16x2((r0[i] - mean) * rstd * gm0[i] + bt0[i], (r1[i] - mean) * rstd * gm1[i] + bt1[i]);
      }
      y[vb + 32 * j] = o;
    }
  }
}

template <int NCH>
__global__ void __launch_bounds__(256)
    og_rope_ln_fwd_vec_kernel(const uint4* __restrict__ x, const float* __restrict__ freq,
                              const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                              uint4* __restrict__ y, long long rows, long long pos_div, int pos_mod,
                              const float4* __restrict__ tab) {
  rope_ln_fwd_vec_rows<NCH, true>(x, freq, gamma, beta, eps, y, rows, pos_div, pos_mod, tab);
}

template <int NCH>
__global__ void __launch_bounds__(256)
    og_ln_rows_fwd_vec_kernel(const uint4* __restrict__ x, const float* __restrict__ gamma,
                              const float* __restrict__ beta, float eps, uint4* __restrict__ y, long long rows) {
  rope_ln_fwd_vec_rows<NCH, false>(x, nullptr, gamma, beta, eps, y, rows, 1, 1, nullptr);
}

// backward: g = g0 (+ g1 + g2) ; dx = R^T LN'(g) (+ add). dgamma / dbeta accumulated per lane over the
// warp's rows, then shared + global atomics once per block.
template <bool kRope>
__device__ __forceinline__ void rope_ln_bwd_rows(const __nv_bfloat162* __restrict__ x, const float* __restrict__ freq,
                                                 const float* __restrict__ gamma, float eps,
                                                 const __nv_bfloat162* __restrict__ g0,
                                                 const __nv_bfloat162* __restrict__ g1,
                                                 const __nv_bfloat162* __restrict__ g2,
                                                 const __nv_bfloat162* __restrict__ add,
                                                 __nv_bfloat162* __restrict__ dx, float* __restrict__ dgamma,
                                                 float* __restrict__ dbeta, long long rows, int C, long long pos_div,
                                                 int pos_mod) {
  extern __shared__ float sh[];  // [2][C]
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) sh[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int pairs = C >> 1;
  const int ppl = (pairs + 31) >> 5;
  const long long warp0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  float dg0[kMaxPairsPerLane], dg1[kMaxPairsPerLane], db0[kMaxPairsPerLane], db1[kMaxPairsPerLane];
#pragma unroll
  for (int j = 0; j < kMaxPairsPerLane; ++j) dg0[j] = dg1[j] = db0[j] = db1[j] = 0.f;
  for (long long row = warp0; row < rows; row += nwarps) {
    const float pos = kRope ? (float)((row / pos_div) % pos_mod) : 0.f;
    float r0[kMaxPairsPerLane], r1[kMaxPairsPerLane], sn[kMaxPairsPerLane], cs[kMaxPairsPerLane];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxPairsPerLane; ++j) {
      const int p = lane + 32 * j;
      if (j < ppl && p < pairs) {
        const float2 v = __bfloat1622float2(x[row * pairs + p]);
        if constexpr (kRope) {
          sincosf(pos * __ldg(freq + p), &sn[j], &cs[j]);
          r0[j] = v.x * cs[j] - v.y * sn[j];
          r1[j] = v.y * cs[j] + v.x * sn[j];
        } else {
          r0[j] = v.x;
          r1[j] = v.y;
        }
        s += r0[j] + r1[j];
      } else {
        r0[j] = r1[j] = sn[j] = cs[j] = 0.f;
      }
    }
    const float mean = warp_sum(s) / (float)C;
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxPairsPerLane; ++j) {
      const int p = lane + 32 * j;
      if (j < ppl && p < pairs) {
        r0[j] -= mean;
        r1[j] -= mean;
        ss += r0[j] * r0[j] + r1[j] * r1[j];
      }
    }
    const float rstd = rsqrtf(warp_sum(ss) / (float)C + eps);
    float gh0[kMaxPairsPerLane], gh1[kMaxPairsPerLane];
    float m1 = 0.f, m2 = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxPairsPerLane; ++j) {
      const int p = lane + 32 * j;
      if (j < ppl && p < pairs) {
        float2 g = __bfloat1622float2(g0[row * pairs + p]);
        if (g1) {
          const float2 t = __bfloat1622float2(g1[row * pairs + p]);
          g.x += t.x;
          g.y += t.y;
        }
        if (g2) {
          const float2 t = __bfloat1622float2(g2[row * pairs + p]);
          g.x += t.x;
          g.y += t.y;
        }
        const float xh0 = r0[j] * rstd, xh1 = r1[j] * rstd;
        db0[j] += g.x;
        db1[j] += g.y;
        dg0[j] += g.x * xh0;
        dg1[j] += g.y * xh1;
        gh0[j] = g.x * __ldg(gamma + 2 * p);
        gh1[j] = g.y * __ldg(gamma + 2 * p + 1);
        m1 += gh0[j] + gh1[j];
        m2 += gh0[j] * xh0 + gh1[j] * xh1;
        r0[j] = xh0;
        r1[j] = xh1;
      } else {
        gh0[j] = gh1[j] = 0.f;
      }
    }
    m1 = warp_sum(m1) / (float)C;
    m2 = warp_sum(m2) / (float)C;
#pragma unroll
    for (int j = 0; j < kMaxPairsPerLane; ++j) {
      const int p = lane + 32 * j;
      if (j < ppl && p < pairs) {
        const float d0 = rstd * (gh0[j] - m1 - r0[j] * m2);
        const float d1 = rstd * (gh1[j] - m1 - r1[j] * m2);
        float o0 = kRope ? d0 * cs[j] + d1 * sn[j] : d0;   // R^T
        float o1 = kRope ? -d0 * sn[j] + d1 * cs[j] : d1;
        if (add) {
          const float2 t = __bfloat1622float2(add[row * pairs + p]);
          o0 += t.x;
          o1 += t.y;
        }
        dx[row * pairs + p] = __floats2bfloat162_rn(o0, o1);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < kMaxPairsPerLane; ++j) {
    const int p = lane + 32 * j;
    if (j < ppl && p < pairs) {
      atomicAdd(&sh[2 * p], dg0[j]);
      atomicAdd(&sh[2 * p + 1], dg1[j]);
      atomicAdd(&sh[C + 2 * p], db0[j]);
      atomicAdd(&sh[C + 2 * p + 1], db1[j]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    atomicAdd(&dgamma[i], sh[i]);
    atomicAdd(&dbeta[i], sh[C + i]);
  }
}

__global__ void __launch_bounds__(256)
    og_rope_ln_bwd_kernel(const __nv_bfloat162* __restrict__ x, const float* __restrict__ freq,
                          const float* __restrict__ gamma, float eps, const __nv_bfloat162* __restrict__ g0,
                          const __nv_bfloat162* __restrict__ g1, const __nv_bfloat162* __restrict__ g2,
                          const __nv_bfloat162* __restrict__ add, __nv_bfloat162* __restrict__ dx,
                          float* __restrict__ dgamma, float* __restrict__ dbeta, long long rows, int C,
                          long long pos_div, int pos_mod) {
  rope_ln_bwd_rows<true>(x, freq, gamma, eps, g0, g1, g2, add, dx, dgamma, dbeta, rows, C, pos_div, pos_mod);
}

__global__ void __launch_bounds__(256)
    og_ln_rows_bwd_kernel(const __nv_bfloat162* __restrict__ x, const float* __restrict__ gamma, float eps,
                          const __nv_bfloat162* __restrict__ g0, const __nv_bfloat162* __restrict__ g1,
                          const __nv_bfloat162* __restrict__ g2, const __nv_bfloat162* __restrict__ add,
                          __nv_bfloat162* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta,
                          long long rows, int C) {
  rope_ln_bwd_rows<false>(x, nullptr, gamma, eps, g0, g1, g2, add, dx, dgamma, dbeta, rows, C, 1, 1);
}

// Vector form of the backward pass for C % 256 == 0: lane l owns the 4 consecutive channel pairs
// [128 j + 4 l, +4) of chunk j (one 16-byte load per tensor and chunk instead of four 4-byte ones) and the
// per-lane arrays are sized by the template, not by the C <= 1024 maximum: 216 -> ~128 registers, two resident
// blocks per SM and 4x the bytes in flight. Same arithmetic as the scalar kernel above.
template <int NCH, bool kRope>
__device__ __forceinline__ void rope_ln_bwd_vec_rows(const uint4* __restrict__ x, const float* __restrict__ freq,
                                                     const float* __restrict__ gamma, float eps,
                                                     const uint4* __restrict__ g0, const uint4* __restrict__ g1,
                                                     const uint4* __restrict__ g2, const uint4* __restrict__ add,
                                                     uint4* __restrict__ dx, float* __restrict__ dgamma,
                                                     float* __restrict__ dbeta, long long rows, long long pos_div,
                                                     int pos_mod, const float4* __restrict__ tab) {
  constexpr int NP = 4 * NCH;      // pairs per lane
  constexpr int C = 256 * NCH;
  constexpr int VPR = 32 * NCH;    // uint4 vectors per row
  extern __shared__ float sh[];    // [2][C]
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) sh[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warp0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  float fq[NP], gm0[NP], gm1[NP];
#pragma unroll
  for (int j = 0; j < NCH; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int p = 128 * j + 4 * lane + e;
      if constexpr (kRope) fq[4 * j + e] = __ldg(freq + p);
      gm0[4 * j + e] = __ldg(gamma + 2 * p);
      gm1[4 * j + e] = __ldg(gamma + 2 * p + 1);
    }
  float dg0[NP], dg1[NP], db0[NP], db1[NP];
#pragma unroll
  for (int i = 0; i < NP; ++i) dg0[i] = dg1[i] = db0[i] = db1[i] = 0.f;
  auto unpack = [](const uint4& u, float (&a)[4], float (&b)[4]) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 t = __bfloat1622float2(h[e]);
      a[e] = t.x;
      b[e] = t.y;
    }
  };
  for (long long row = warp0; row < rows; row += nwarps) {
    const int ipos = kRope ? (int)((row / pos_div) % pos_mod) : 0;
    const float pos = (float)ipos;
    const long long vb = row * VPR + lane;
    uint4 ux[NCH], ug[NCH];
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      ux[j] = __ldg(x + vb + 32 * j);
      ug[j] = __ldg(g0 + vb + 32 * j);
    }
    float r0[NP], r1[NP], sn[NP], cs[NP];
    if (kRope && tab) {   // see og_rope_ln_fwd_vec_kernel
      const float4* tr = tab + (long long)ipos * (C / 4);
#pragma unroll
      for (int j = 0; j < NCH; ++j) {
        const float4 t0 = __ldg(tr + 64 * j + 2 * lane), t1 = __ldg(tr + 64 * j + 2 * lane + 1);
        cs[4 * j] = t0.x; sn[4 * j] = t0.y; cs[4 * j + 1] = t0.z; sn[4 * j + 1] = t0.w;
        cs[4 * j + 2] = t1.x; sn[4 * j + 2] = t1.y; cs[4 * j + 3] = t1.z; sn[4 * j + 3] = t1.w;
      }
    }
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      float a[4], b[4];
      unpack(ux[j], a, b);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * j + e;
        if constexpr (kRope) {
          if (!tab) sincosf(pos * fq[i], &sn[i], &cs[i]);
          r0[i] = a[e] * cs[i] - b[e] * sn[i];
          r1[i] = b[e] * cs[i] + a[e] * sn[i];
        } else {
          r0[i] = a[e];
          r1[i] = b[e];
        }
        s += r0[i] + r1[i];
      }
    }
    const float mean = warp_sum(s) / (float)C;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NP; ++i) {
      r0[i] -= mean;
      r1[i] -= mean;
      ss += r0[i] * r0[i] + r1[i] * r1[i];
    }
    const float rstd = rsqrtf(warp_sum(ss) / (float)C + eps);
    float gh0[NP], gh1[NP];
    float m1 = 0.f, m2 = 0.f;
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      float ga[4], gb[4];
      unpack(ug[j], ga, gb);
      if (g1) {
        float ta[4], tb[4];
        unpack(__ldg(g1 + vb + 32 * j), ta, tb);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          ga[e] += ta[e];
          gb[e] += tb[e];
        }
      }
      if (g2) {
        float ta[4], tb[4];
        unpack(__ldg(g2 + vb + 32 * j), ta, tb);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          ga[e] += ta[e];
          gb[e] += tb[e];
        }
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * j + e;
        const float xh0 = r0[i] * rstd, xh1 = r1[i] * rstd;
        db0[i] += ga[e];
        db1[i] += gb[e];
        dg0[i] = fmaf(ga[e], xh0, dg0[i]);
        dg1[i] = fmaf(gb[e], xh1, dg1[i]);
        gh0[i] = ga[e] * gm0[i];
        gh1[i] = gb[e] * gm1[i];
        m1 += gh0[i] + gh1[i];
        m2 += gh0[i] * xh0 + gh1[i] * xh1;
        r0[i] = xh0;
        r1[i] = xh1;
      }
    }
    m1 = warp_sum(m1) / (float)C;
    m2 = warp_sum(m2) / (float)C;
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      float aa[4] = {0.f, 0.f, 0.f, 0.f}, ab[4] = {0.f, 0.f, 0.f, 0.f};
      if (add) unpack(__ldg(add + vb + 32 * j), aa, ab);
      uint4 o;
      uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * j + e;
        const float d0 = rstd * (gh0[i] - m1 - r0[i] * m2);
        const float d1 = rstd * (gh1[i] - m1 - r1[i] * m2);
        const float o0 = (kRope ? d0 * cs[i] + d1 * sn[i] : d0) + aa[e];   // R^T
        const float o1 = (kRope ? -d0 * sn[i] + d1 * cs[i] : d1) + ab[e];
        ow[e] = pack_bf16x2(o0, o1);
      }
      dx[vb + 32 * j] = o;
    }
  }
#pragma unroll
  for (int j = 0; j < NCH; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int p = 128 * j + 4 * lane + e, i = 4 * j + e;
      atomicAdd(&sh[2 * p], dg0[i]);
      atomicAdd(&sh[2 * p + 1], dg1[i]);
      atomicAdd(&sh[C + 2 * p], db0[i]);
      atomicAdd(&sh[C + 2 * p + 1], db1[i]);
    }
  __syncthreads();
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    atomicAdd(&dgamma[i], sh[i]);
    atomicAdd(&dbeta[i], sh[C + i]);
  }
}

template <int NCH>
__global__ void __launch_bounds__(256, (NCH <= 2 ? 2 : 1))
    og_rope_ln_bwd_vec_kernel(const uint4* __restrict__ x, const float* __restrict__ freq,
                              const float* __restrict__ gamma, float eps, const uint4* __restrict__ g0,
                              const uint4* __restrict__ g1, const uint4* __restrict__ g2,
                              const uint4* __restrict__ add, uint4* __restrict__ dx, float* __restrict__ dgamma,
                              float* __restrict__ dbeta, long long rows, long long pos_div, int pos_mod,
                              const float4* __restrict__ tab) {
  rope_ln_bwd_vec_rows<NCH, true>(x, freq, gamma, eps, g0, g1, g2, add, dx, dgamma, dbeta, rows, pos_div, pos_mod,
                                  tab);
}

template <int NCH>
__global__ void __launch_bounds__(256, (NCH <= 2 ? 2 : 1))
    og_ln_rows_bwd_vec_kernel(const uint4* __restrict__ x, const float* __restrict__ gamma, float eps,
                              const uint4* __restrict__ g0, const uint4* __restrict__ g1,
                              const uint4* __restrict__ g2, const uint4* __restrict__ add, uint4* __restrict__ dx,
                              float* __restrict__ dgamma, float* __restrict__ dbeta, long long rows) {
  rope_ln_bwd_vec_rows<NCH, false>(x, nullptr, gamma, eps, g0, g1, g2, add, dx, dgamma, dbeta, rows, 1, 1, nullptr);
}

// ------------------------------------------------------------------------------------------------
// temporal attention, one warp per (batch b, pixel p, head h). T <= 32, d = 64 (lane owns 2 dims... no:
// lane t owns QUERY row t). K/V rows of the sequence sit in shared memory (broadcast reads).
// q rows: q[((b*T + t)*P + p)*C + h*64 ...]; kv either the same layout (kv_bcast = 0) or [b][t][C]
// broadcast over pixels (kv_bcast = 1: the latent-action conditioning, attention.py:362-363).
// ------------------------------------------------------------------------------------------------
// Work distribution shared by both kernels: tasks are ordered (b, h, pixel) with the PIXEL fastest and every warp
// owns one contiguous range of them, so consecutive tasks of a warp share (b, h): the broadcast-K/V gradient can
// then be accumulated in registers across the whole range and flushed with one set of atomics per (b, h) change
// instead of one per pixel (8192 atomics per address before). When T <= 16 a warp runs TWO tasks at once, one per
// half-warp (lane = sub * 16 + t), so no lane idles on the short sequences the models use (T = 16).
struct TaskRange {
  long long begin, end;
};
__device__ __forceinline__ TaskRange warp_task_range(long long ntask, int tpw) {
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  const long long w = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  long long per = (ntask + nw - 1) / nw;
  per = (per + tpw - 1) / tpw * tpw;
  TaskRange r;
  r.begin = w * per;
  r.end = r.begin + per < ntask ? r.begin + per : ntask;
  return r;
}

template <int D>
__global__ void __launch_bounds__(128)
    og_temporal_attn_fwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ res,
                                __nv_bfloat16* __restrict__ out, int B, int T, long long P, int C, int nh, float scale,
                                int kv_bcast) {
  extern __shared__ __nv_bfloat16 smem_bf[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __nv_bfloat16* ks = smem_bf + warp * (2 * 32 * D);
  __nv_bfloat16* vs = ks + 32 * D;
  const int tpad = T <= 16 ? 16 : 32, tpw = 32 / tpad;
  const int sub = lane / tpad, t = lane % tpad;
  const long long ntask = (long long)B * P * nh;
  const TaskRange tr = warp_task_range(ntask, tpw);
  for (long long base = tr.begin; base < tr.end; base += tpw) {
    __syncwarp();
    // stage K, V rows of the warp's tpw tasks: smem row = sub * tpad + t, D*2 bytes each (one 4-byte word per lane)
    for (int rs = 0; rs < tpw; ++rs) {
      const long long task = base + rs;
      if (task >= tr.end) break;  // warp-uniform
      const long long pp = task % P, bh = task / P;  // decoded once per task, not per row
      const int hh = (int)(bh % nh), bb = (int)(bh / nh);
      for (int rt = 0; rt < T; ++rt) {
        const int r = rs * tpad + rt;
        const long long kr = kv_bcast ? ((long long)bb * T + rt) * C + hh * D : (((long long)bb * T + rt) * P + pp) * C + hh * D;
        const uint32_t* ksrc = reinterpret_cast<const uint32_t*>(k + kr);
        const uint32_t* vsrc = reinterpret_cast<const uint32_t*>(v + kr);
        for (int w = lane; w < D / 2; w += 32) {
          reinterpret_cast<uint32_t*>(ks + r * D)[w] = __ldg(ksrc + w);
          reinterpret_cast<uint32_t*>(vs + r * D)[w] = __ldg(vsrc + w);
        }
      }
    }
    __syncwarp();
    const long long task = base + sub;
    if (t < T && task < tr.end) {
      const long long p = task % P, bh = task / P;
      const int h = (int)(bh % nh), b = (int)(bh / nh);
      const __nv_bfloat16* kt = ks + sub * tpad * D;
      const __nv_bfloat16* vt = vs + sub * tpad * D;
      const long long qr = (((long long)b * T + t) * P + p) * C + h * D;
      float qf[D], o[D];
#pragma unroll
      for (int i = 0; i < D; i += 2) {
        const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(q + qr + i));
        qf[i] = f.x * scale;
        qf[i + 1] = f.y * scale;
        o[i] = o[i + 1] = 0.f;
      }
      float m = -INFINITY, l = 0.f;
      for (int s = 0; s <= t; ++s) {
        float sc = 0.f;
#pragma unroll
        for (int i = 0; i < D; i += 2) {
          const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(kt + s * D + i));
          sc = fmaf(qf[i], f.x, sc);
          sc = fmaf(qf[i + 1], f.y, sc);
        }
        const float mn = fmaxf(m, sc);
        const float corr = __expf(m - mn), pw = __expf(sc - mn);
        l = l * corr + pw;
#pragma unroll
        for (int i = 0; i < D; i += 2) {
          const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(vt + s * D + i));
          o[i] = fmaf(pw, f.x, o[i] * corr);
          o[i + 1] = fmaf(pw, f.y, o[i + 1] * corr);
        }
        m = mn;
      }
      const float inv = 1.f / l;
#pragma unroll
      for (int i = 0; i < D; i += 2) {
        float a = o[i] * inv, c2 = o[i + 1] * inv;
        if (res) {
          const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(res + qr + i));
          a += f.x;
          c2 += f.y;
        }
        *reinterpret_cast<__nv_bfloat162*>(out + qr + i) = __floats2bfloat162_rn(a, c2);
      }
    }
  }
}

// backward: recompute P; lane t owns query row t for dQ, lane s owns key row s for dK / dV.
template <int D>
__global__ void __launch_bounds__(128)
    og_temporal_attn_bwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ dout,
                                __nv_bfloat16* __restrict__ dq, __nv_bfloat16* __restrict__ dk,
                                __nv_bfloat16* __restrict__ dv, float* __restrict__ dk_b, float* __restrict__ dv_b,
                                int B, int T, long long P, int C, int nh, float scale, int kv_bcast) {
  extern __shared__ __nv_bfloat16 smem_bf[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // per warp: K, V, Q, dO rows (bf16, row = sub * tpad + t) + P and dS matrices (fp32 [32][33], row = sub * tpad + t)
  __nv_bfloat16* ks = smem_bf + warp * (4 * 32 * D);
  __nv_bfloat16* vs = ks + 32 * D;
  __nv_bfloat16* qs = vs + 32 * D;
  __nv_bfloat16* dos = qs + 32 * D;
  float* fbase = reinterpret_cast<float*>(smem_bf + 4 * (4 * 32 * D)) + warp * (2 * 32 * 33);
  float* Pm = fbase;
  float* dS = fbase + 32 * 33;
  const int tpad = T <= 16 ? 16 : 32, tpw = 32 / tpad;
  const int sub = lane / tpad, t = lane % tpad;
  const long long ntask = (long long)B * P * nh;
  const TaskRange tr = warp_task_range(ntask, tpw);
  // broadcast-K/V gradient accumulators of key row `t`, kept across tasks that share (b, h)
  float dkv[D], dvv[D];
#pragma unroll
  for (int i = 0; i < D; ++i) dkv[i] = dvv[i] = 0.f;
  long long acc_bh = -1;
  auto flush = [&]() {
    if (acc_bh >= 0 && t < T) {
      const int hh = (int)(acc_bh % nh), bb = (int)(acc_bh / nh);
      const long long kr = ((long long)bb * T + t) * C + hh * D;
#pragma unroll
      for (int i = 0; i < D; ++i) {
        atomicAdd(dk_b + kr + i, dkv[i]);
        atomicAdd(dv_b + kr + i, dvv[i]);
        dkv[i] = dvv[i] = 0.f;
      }
    }
  };
  for (long long base = tr.begin; base < tr.end; base += tpw) {
    __syncwarp();
    for (int rs = 0; rs < tpw; ++rs) {
      const long long task = base + rs;
      if (task >= tr.end) break;  // warp-uniform
      const long long pp = task % P, bh = task / P;  // decoded once per task, not per row
      const int hh = (int)(bh % nh), bb = (int)(bh / nh);
      for (int rt = 0; rt < T; ++rt) {
        const int r = rs * tpad + rt;
        const long long qr = (((long long)bb * T + rt) * P + pp) * C + hh * D;
        const long long kr = kv_bcast ? ((long long)bb * T + rt) * C + hh * D : qr;
        for (int w = lane; w < D / 2; w += 32) {
          reinterpret_cast<uint32_t*>(ks + r * D)[w] = __ldg(reinterpret_cast<const uint32_t*>(k + kr) + w);
          reinterpret_cast<uint32_t*>(vs + r * D)[w] = __ldg(reinterpret_cast<const uint32_t*>(v + kr) + w);
          reinterpret_cast<uint32_t*>(qs + r * D)[w] = __ldg(reinterpret_cast<const uint32_t*>(q + qr) + w);
          reinterpret_cast<uint32_t*>(dos + r * D)[w] = __ldg(reinterpret_cast<const uint32_t*>(dout + qr) + w);
        }
      }
    }
    __syncwarp();
    const long long task = base + sub;
    const bool live = t < T && task < tr.end;
    const long long p = live ? task % P : 0, bh = live ? task / P : 0;
    const int h = (int)(bh % nh), b = (int)(bh / nh);
    const int r0 = sub * tpad;  // first smem row of this half-warp's task
    // phase 1: row t: scores, softmax, dP, dS ; dQ
    if (live) {
      float sc[32];
      float m = -INFINITY;
      for (int s = 0; s <= t; ++s) {
        float a = 0.f;
#pragma unroll
        for (int i = 0; i < D; i += 2) {
          const float2 fq = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(qs + (r0 + t) * D + i));
          const float2 fk = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ks + (r0 + s) * D + i));
          a = fmaf(fq.x, fk.x, a);
          a = fmaf(fq.y, fk.y, a);
        }
        sc[s] = a * scale;
        m = fmaxf(m, sc[s]);
      }
      float l = 0.f;
      for (int s = 0; s <= t; ++s) {
        sc[s] = __expf(sc[s] - m);
        l += sc[s];
      }
      const float inv = 1.f / l;
      // dP[s] = dO_t . V_s ; delta = sum_s P dP
      float dp[32];
      float delta = 0.f;
      for (int s = 0; s <= t; ++s) {
        sc[s] *= inv;
        float a = 0.f;
#pragma unroll
        for (int i = 0; i < D; i += 2) {
          const float2 fo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(dos + (r0 + t) * D + i));
          const float2 fv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(vs + (r0 + s) * D + i));
          a = fmaf(fo.x, fv.x, a);
          a = fmaf(fo.y, fv.y, a);
        }
        dp[s] = a;
        delta = fmaf(sc[s], a, delta);
      }
      float dqv[D];
#pragma unroll
      for (int i = 0; i < D; ++i) dqv[i] = 0.f;
      for (int s = 0; s < T; ++s) {
        float pv = 0.f, ds = 0.f;
        if (s <= t) {
          pv = sc[s];
          ds = sc[s] * (dp[s] - delta) * scale;
#pragma unroll
          for (int i = 0; i < D; i += 2) {
            const float2 fk = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ks + (r0 + s) * D + i));
            dqv[i] = fmaf(ds, fk.x, dqv[i]);
            dqv[i + 1] = fmaf(ds, fk.y, dqv[i + 1]);
          }
        }
        Pm[(r0 + t) * 33 + s] = pv;
        dS[(r0 + t) * 33 + s] = ds;
      }
      const long long qr = (((long long)b * T + t) * P + p) * C + h * D;
#pragma unroll
      for (int i = 0; i < D; i += 2)
        *reinterpret_cast<__nv_bfloat162*>(dq + qr + i) = __floats2bfloat162_rn(dqv[i], dqv[i + 1]);
    }
    __syncwarp();
    // phase 2: key row s (= t of this lane): dK_s = sum_t' dS[t'][s] Q_t' ; dV_s = sum_t' P[t'][s] dO_t'
    if (kv_bcast && live && bh != acc_bh) {
      flush();
      acc_bh = bh;
    }
    if (live) {
      const int s = t;
      if (!kv_bcast) {
#pragma unroll
        for (int i = 0; i < D; ++i) dkv[i] = dvv[i] = 0.f;
      }
      for (int tt = s; tt < T; ++tt) {
        const float ds = dS[(r0 + tt) * 33 + s], pv = Pm[(r0 + tt) * 33 + s];
#pragma unroll
        for (int i = 0; i < D; i += 2) {
          const float2 fq = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(qs + (r0 + tt) * D + i));
          const float2 fo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(dos + (r0 + tt) * D + i));
          dkv[i] = fmaf(ds, fq.x, dkv[i]);
          dkv[i + 1] = fmaf(ds, fq.y, dkv[i + 1]);
          dvv[i] = fmaf(pv, fo.x, dvv[i]);
          dvv[i + 1] = fmaf(pv, fo.y, dvv[i + 1]);
        }
      }
      if (!kv_bcast) {
        const long long kr = (((long long)b * T + s) * P + p) * C + h * D;
#pragma unroll
        for (int i = 0; i < D; i += 2) {
          *reinterpret_cast<__nv_bfloat162*>(dk + kr + i) = __floats2bfloat162_rn(dkv[i], dkv[i + 1]);
          *reinterpret_cast<__nv_bfloat162*>(dv + kr + i) = __floats2bfloat162_rn(dvv[i], dvv[i + 1]);
        }
      }
    }
  }
  if (kv_bcast) flush();
}

// mma.sync m16n8k16 path (temporal_attn_mma.cu) for d_head = 64, T <= 16; the per-lane kernels above cover d_head = 32
// and T in (16, 32].
int launch_temporal_fwd_mma(const void* q, const void* k, const void* v, const void* residual, void* out, int B, int T,
                            long long P, int C, int n_head, float scale, int kv_bcast, cudaStream_t stream);
int launch_temporal_bwd_mma(const void* q, const void* k, const void* v, const void* dout, void* dq, void* dk, void* dv,
                            float* dk_b, float* dv_b, int B, int T, long long P, int C, int n_head, float scale,
                            int kv_bcast, cudaStream_t stream);
static bool temporal_mma_enabled(int D, int T, int C) {
  return D == 64 && T <= 16 && C % 8 == 0;
}

static int row_grid(long long rows, int warps_per_block) {
  long long g = (rows + warps_per_block - 1) / warps_per_block;
  long long cap = (long long)num_sms() * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace og

using namespace og;

extern "C" int og_rope_ln_fwd(const void* x, const float* freq, const float* gamma, const float* beta, float eps,
                              void* y, int64_t rows, int C, int64_t pos_div, int pos_mod, const float* cos_sin,
                              og_stream_t stream) {
  OG_REQUIRE(!cos_sin || (reinterpret_cast<uintptr_t>(cos_sin) & 15) == 0, "rope_ln_fwd: cos_sin must be 16-byte aligned");
  OG_REQUIRE(x && freq && gamma && beta && y && rows > 0, "rope_ln_fwd: bad arguments");
  OG_REQUIRE(C % 2 == 0 && C <= 2 * 32 * kMaxPairsPerLane, "rope_ln_fwd: C=%d must be even and <= 1024", C);
  if ((C == 256 || C == 512 || C == 1024) &&
      ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0) {
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = row_grid(rows, 8);
    if (C == 256)
      og_rope_ln_fwd_vec_kernel<1><<<grid, 256, 0, st>>>((const uint4*)x, freq, gamma, beta, eps, (uint4*)y, rows, pos_div, pos_mod, (const float4*)cos_sin);
    else if (C == 512)
      og_rope_ln_fwd_vec_kernel<2><<<grid, 256, 0, st>>>((const uint4*)x, freq, gamma, beta, eps, (uint4*)y, rows, pos_div, pos_mod, (const float4*)cos_sin);
    else
      og_rope_ln_fwd_vec_kernel<4><<<grid, 256, 0, st>>>((const uint4*)x, freq, gamma, beta, eps, (uint4*)y, rows, pos_div, pos_mod, (const float4*)cos_sin);
    OG_CHECK_CUDA(cudaGetLastError());
    g_launches.fetch_add(1);
    return OG_OK;
  }
  og_rope_ln_fwd_kernel<<<row_grid(rows, 8), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat162*)x, freq, gamma, beta, eps, (__nv_bfloat162*)y, rows, C, pos_div, pos_mod);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

// tab[pos][p] = (cos, sin)(pos * freq[p]) — exactly the values the passes would compute per element
__global__ void og_rope_table_kernel(const float* __restrict__ freq, int npos, int pairs, float2* __restrict__ tab) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npos * pairs) return;
  const int pos = i / pairs, p = i - pos * pairs;
  float sn, cs;
  sincosf((float)pos * __ldg(freq + p), &sn, &cs);
  tab[i] = make_float2(cs, sn);
}

extern "C" int og_rope_table(const float* freq, int npos, int C, float* table, og_stream_t stream) {
  OG_REQUIRE(freq && table && npos > 0 && C > 0 && C % 2 == 0, "rope_table: bad arguments");
  const int total = npos * (C / 2);
  og_rope_table_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(freq, npos, C / 2, (float2*)table);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_rope_ln_bwd(const void* x, const float* freq, const float* gamma, float eps, const void* g0,
                              const void* g1, const void* g2, const void* add, void* dx, float* dgamma, float* dbeta,
                              int64_t rows, int C, int64_t pos_div, int pos_mod, const float* cos_sin,
                              og_stream_t stream) {
  OG_REQUIRE(!cos_sin || (reinterpret_cast<uintptr_t>(cos_sin) & 15) == 0, "rope_ln_bwd: cos_sin must be 16-byte aligned");
  OG_REQUIRE(x && freq && gamma && g0 && dx && dgamma && dbeta && rows > 0, "rope_ln_bwd: bad arguments");
  OG_REQUIRE(C % 2 == 0 && C <= 2 * 32 * kMaxPairsPerLane, "rope_ln_bwd: C=%d must be even and <= 1024", C);
  int grid = row_grid(rows, 8);
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(g0) | reinterpret_cast<uintptr_t>(g1) |
                        reinterpret_cast<uintptr_t>(g2) | reinterpret_cast<uintptr_t>(add) |
                        reinterpret_cast<uintptr_t>(dx)) & 15) == 0;
  if (vec_ok && (C == 256 || C == 512 || C == 1024)) {
    if (grid > num_sms() * 4) grid = num_sms() * 4;  // 2 resident blocks per SM, 2 waves; bounds the dgamma/dbeta atomics
    cudaStream_t st = (cudaStream_t)stream;
    const size_t shb = 2 * C * sizeof(float);
#define OG_ROPE_BWD(NCH)                                                                                          \
    og_rope_ln_bwd_vec_kernel<NCH><<<grid, 256, shb, st>>>((const uint4*)x, freq, gamma, eps, (const uint4*)g0,     \
                                                           (const uint4*)g1, (const uint4*)g2, (const uint4*)add,  \
                                                           (uint4*)dx, dgamma, dbeta, rows, pos_div, pos_mod,       \
                                                           (const float4*)cos_sin)
    if (C == 256) OG_ROPE_BWD(1);
    else if (C == 512) OG_ROPE_BWD(2);
    else OG_ROPE_BWD(4);
#undef OG_ROPE_BWD
    OG_CHECK_CUDA(cudaGetLastError());
    g_launches.fetch_add(1);
    return OG_OK;
  }
  if (grid > num_sms() * 2) grid = num_sms() * 2;  // fewer blocks -> fewer dgamma/dbeta atomics
  og_rope_ln_bwd_kernel<<<grid, 256, 2 * C * sizeof(float), (cudaStream_t)stream>>>(
      (const __nv_bfloat162*)x, freq, gamma, eps, (const __nv_bfloat162*)g0, (const __nv_bfloat162*)g1,
      (const __nv_bfloat162*)g2, (const __nv_bfloat162*)add, (__nv_bfloat162*)dx, dgamma, dbeta, rows, C, pos_div,
      pos_mod);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

// LayerNorm-only passes (attention without a rotary embedding): the RoPE passes' kernels and dispatch, no rotation.
extern "C" int og_ln_rows_fwd(const void* x, const float* gamma, const float* beta, float eps, void* y, int64_t rows,
                              int C, og_stream_t stream) {
  OG_REQUIRE(x && gamma && beta && y && rows > 0, "ln_rows_fwd: bad arguments");
  OG_REQUIRE(C >= 2 && C % 2 == 0 && C <= 2 * 32 * kMaxPairsPerLane, "ln_rows_fwd: C=%d must be even and in [2, 1024]",
             C);
  const uintptr_t align = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y);
  OG_REQUIRE((align & 3) == 0, "ln_rows_fwd: x and y must be 4-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = row_grid(rows, 8);
  if ((C == 256 || C == 512 || C == 1024) && (align & 15) == 0) {
    if (C == 256)
      og_ln_rows_fwd_vec_kernel<1><<<grid, 256, 0, st>>>((const uint4*)x, gamma, beta, eps, (uint4*)y, rows);
    else if (C == 512)
      og_ln_rows_fwd_vec_kernel<2><<<grid, 256, 0, st>>>((const uint4*)x, gamma, beta, eps, (uint4*)y, rows);
    else
      og_ln_rows_fwd_vec_kernel<4><<<grid, 256, 0, st>>>((const uint4*)x, gamma, beta, eps, (uint4*)y, rows);
  } else {
    og_ln_rows_fwd_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat162*)x, gamma, beta, eps, (__nv_bfloat162*)y, rows, C);
  }
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_ln_rows_bwd(const void* x, const float* gamma, float eps, const void* g0, const void* g1,
                              const void* g2, const void* add, void* dx, float* dgamma, float* dbeta, int64_t rows,
                              int C, og_stream_t stream) {
  OG_REQUIRE(x && gamma && g0 && dx && dgamma && dbeta && rows > 0, "ln_rows_bwd: bad arguments");
  OG_REQUIRE(C >= 2 && C % 2 == 0 && C <= 2 * 32 * kMaxPairsPerLane, "ln_rows_bwd: C=%d must be even and in [2, 1024]",
             C);
  const uintptr_t align = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(g0) |
                          reinterpret_cast<uintptr_t>(g1) | reinterpret_cast<uintptr_t>(g2) |
                          reinterpret_cast<uintptr_t>(add) | reinterpret_cast<uintptr_t>(dx);
  OG_REQUIRE((align & 3) == 0, "ln_rows_bwd: x, g0, g1, g2, add and dx must be 4-byte aligned");
  OG_REQUIRE((((reinterpret_cast<uintptr_t>(dgamma) | reinterpret_cast<uintptr_t>(dbeta))) & 3) == 0,
             "ln_rows_bwd: dgamma and dbeta must be 4-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  int grid = row_grid(rows, 8);
  const size_t shb = 2 * C * sizeof(float);
  if ((C == 256 || C == 512 || C == 1024) && (align & 15) == 0) {
    if (grid > num_sms() * 4) grid = num_sms() * 4;  // as og_rope_ln_bwd
#define OG_LN_BWD(NCH)                                                                                                \
    og_ln_rows_bwd_vec_kernel<NCH><<<grid, 256, shb, st>>>((const uint4*)x, gamma, eps, (const uint4*)g0,              \
                                                           (const uint4*)g1, (const uint4*)g2, (const uint4*)add,      \
                                                           (uint4*)dx, dgamma, dbeta, rows)
    if (C == 256) OG_LN_BWD(1);
    else if (C == 512) OG_LN_BWD(2);
    else OG_LN_BWD(4);
#undef OG_LN_BWD
  } else {
    if (grid > num_sms() * 2) grid = num_sms() * 2;
    og_ln_rows_bwd_kernel<<<grid, 256, shb, st>>>(
        (const __nv_bfloat162*)x, gamma, eps, (const __nv_bfloat162*)g0, (const __nv_bfloat162*)g1,
        (const __nv_bfloat162*)g2, (const __nv_bfloat162*)add, (__nv_bfloat162*)dx, dgamma, dbeta, rows, C);
  }
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_temporal_attn_fwd(const void* q, const void* k, const void* v, const void* residual, void* out, int B,
                                    int T, int64_t P, int C, int n_head, float scale, int kv_bcast,
                                    og_stream_t stream) {
  OG_REQUIRE(q && k && v && out, "temporal_attn_fwd: null pointer");
  OG_REQUIRE(T >= 1 && T <= 32, "temporal_attn_fwd: T=%d must be in [1,32]", T);
  OG_REQUIRE(B >= 1 && P >= 1, "temporal_attn_fwd: empty problem (B=%d, P=%lld)", B, (long long)P);
  OG_REQUIRE(n_head >= 1 && C % n_head == 0, "temporal_attn_fwd: C=%d not divisible by n_head=%d", C, n_head);
  const int D = C / n_head;
  if (D != 32 && D != 64) {
    set_error("temporal_attn_fwd: d_head=%d not supported (32 or 64)", D);
    return OG_ERR_UNSUPPORTED_SHAPE;
  }
  if (temporal_mma_enabled(D, T, C))
    return launch_temporal_fwd_mma(q, k, v, residual, out, B, T, P, C, n_head, scale, kv_bcast, (cudaStream_t)stream);
  const long long ntask = (long long)B * P * n_head;
  long long grid = (ntask + 3) / 4;
  if (grid > (long long)num_sms() * 16) grid = (long long)num_sms() * 16;
  const size_t smem = (size_t)4 * 2 * 32 * D * 2;
  if (D == 64)
    og_temporal_attn_fwd_kernel<64><<<(unsigned)grid, 128, smem, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)residual,
        (__nv_bfloat16*)out, B, T, P, C, n_head, scale, kv_bcast);
  else
    og_temporal_attn_fwd_kernel<32><<<(unsigned)grid, 128, smem, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)residual,
        (__nv_bfloat16*)out, B, T, P, C, n_head, scale, kv_bcast);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_temporal_attn_bwd(const void* q, const void* k, const void* v, const void* dout, void* dq, void* dk,
                                    void* dv, float* dk_bcast, float* dv_bcast, int B, int T, int64_t P, int C,
                                    int n_head, float scale, int kv_bcast, og_stream_t stream) {
  OG_REQUIRE(q && k && v && dout && dq, "temporal_attn_bwd: null pointer");
  OG_REQUIRE(kv_bcast ? (dk_bcast && dv_bcast) : (dk && dv), "temporal_attn_bwd: missing dk/dv buffers");
  OG_REQUIRE(T >= 1 && T <= 32, "temporal_attn_bwd: T=%d must be in [1,32]", T);
  OG_REQUIRE(B >= 1 && P >= 1, "temporal_attn_bwd: empty problem (B=%d, P=%lld)", B, (long long)P);
  OG_REQUIRE(n_head >= 1 && C % n_head == 0, "temporal_attn_bwd: C=%d not divisible by n_head=%d", C, n_head);
  const int D = C / n_head;
  if (D != 32 && D != 64) {
    set_error("temporal_attn_bwd: d_head=%d not supported (32 or 64)", D);
    return OG_ERR_UNSUPPORTED_SHAPE;
  }
  if (temporal_mma_enabled(D, T, C))
    return launch_temporal_bwd_mma(q, k, v, dout, dq, dk, dv, dk_bcast, dv_bcast, B, T, P, C, n_head, scale, kv_bcast,
                                   (cudaStream_t)stream);
  const long long ntask = (long long)B * P * n_head;
  long long grid = (ntask + 3) / 4;
  if (grid > (long long)num_sms() * 8) grid = (long long)num_sms() * 8;
  const size_t smem = (size_t)4 * 4 * 32 * D * 2 + (size_t)4 * 2 * 32 * 33 * 4;
  cudaStream_t s = (cudaStream_t)stream;
  if (D == 64) {
    static bool attr = false;
    if (!attr) {
      OG_CHECK_CUDA(cudaFuncSetAttribute(og_temporal_attn_bwd_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
      attr = true;
    }
    og_temporal_attn_bwd_kernel<64><<<(unsigned)grid, 128, smem, s>>>(
        (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)dout,
        (__nv_bfloat16*)dq, (__nv_bfloat16*)dk, (__nv_bfloat16*)dv, dk_bcast, dv_bcast, B, T, P, C, n_head, scale,
        kv_bcast);
  } else {
    static bool attr = false;
    if (!attr) {
      OG_CHECK_CUDA(cudaFuncSetAttribute(og_temporal_attn_bwd_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
      attr = true;
    }
    og_temporal_attn_bwd_kernel<32><<<(unsigned)grid, 128, smem, s>>>(
        (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)dout,
        (__nv_bfloat16*)dq, (__nv_bfloat16*)dk, (__nv_bfloat16*)dv, dk_bcast, dv_bcast, B, T, P, C, n_head, scale,
        kv_bcast);
  }
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}
