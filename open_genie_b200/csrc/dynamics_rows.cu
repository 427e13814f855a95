// dynamics_rows.cu — the row-wise pieces of DynamicsModel (genie/dynamics.py):
//   * token + action embedding sum        tok_emb(tokens) + act_emb(act_id)[:, :, None, None]      (dynamics.py:34-38, 55)
//   * masked cross-entropy on the logits   cross_entropy(logits[mask], tokens[mask])                (dynamics.py:89-97)
// Both are HBM-bound gathers / reductions; the 512 -> vocab head itself runs on the conv GEMM kernel.
#include "og_host.cuh"
#include "og_ptx.cuh"

namespace og {
extern std::atomic<uint64_t> g_launches;

// out[row][c] = bf16(tok_w[tok[row]][c] + act_w[act[row / rows_per_act]][c])      (8 channels per thread)
__global__ void og_embed_add_fwd_kernel(const long long* __restrict__ tok, const long long* __restrict__ act,
                                        const float* __restrict__ tok_w, const float* __restrict__ act_w,
                                        __nv_bfloat16* __restrict__ out, long long rows, long long rows_per_act, int C,
                                        int tok_vocab, int act_vocab) {
  const int cv = C >> 3;
  const long long total = rows * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / cv;
    const int c = (int)(i % cv) * 8;
    const long long t = tok[row], a = act[row / rows_per_act];
    if (t < 0 || t >= tok_vocab || a < 0 || a >= act_vocab) {
      // nn.Embedding raises a device-side assert on an out-of-range index (dynamics.py:34-38); so does this kernel
      if (c == 0) printf("og_embed_add_fwd: index out of range (token %lld / vocab %d, action %lld / vocab %d)\n", t,
                         tok_vocab, a, act_vocab);
      __trap();
    }
    const float4* tp = reinterpret_cast<const float4*>(tok_w + t * C + c);
    const float4* ap = reinterpret_cast<const float4*>(act_w + a * C + c);
    const float4 t0 = __ldg(tp), t1 = __ldg(tp + 1), a0 = __ldg(ap), a1 = __ldg(ap + 1);
    uint4 u;
    u.x = pack_bf16x2(t0.x + a0.x, t0.y + a0.y);
    u.y = pack_bf16x2(t0.z + a0.z, t0.w + a0.w);
    u.z = pack_bf16x2(t1.x + a1.x, t1.y + a1.y);
    u.w = pack_bf16x2(t1.z + a1.z, t1.w + a1.w);
    *reinterpret_cast<uint4*>(out + row * C + c) = u;
  }
}

// d_tok_w[tok[row]] += dy[row] ; d_act_w[act[...]] += dy[row]   (fp32 atomics; vocab rows are few and hot)
__global__ void og_embed_add_bwd_kernel(const long long* __restrict__ tok, const long long* __restrict__ act,
                                        const __nv_bfloat16* __restrict__ dy, float* __restrict__ d_tok_w,
                                        float* __restrict__ d_act_w, long long rows, long long rows_per_act, int C,
                                        int tok_vocab, int act_vocab) {
  const int cv = C >> 3;
  const long long total = rows * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / cv;
    const int c = (int)(i % cv) * 8;
    long long t = tok[row], a = act[row / rows_per_act];
    t = t < 0 ? 0 : (t >= tok_vocab ? tok_vocab - 1 : t);
    a = a < 0 ? 0 : (a >= act_vocab ? act_vocab - 1 : a);
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(dy + row * C + c));
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = __bfloat1622float2(h[k]);
      atomicAdd(d_tok_w + t * C + c + 2 * k, f.x);
      atomicAdd(d_tok_w + t * C + c + 2 * k + 1, f.y);
      atomicAdd(d_act_w + a * C + c + 2 * k, f.x);
      atomicAdd(d_act_w + a * C + c + 2 * k + 1, f.y);
    }
  }
}

// masked cross entropy, one warp per row. stats[0] += sum_{masked rows} (lse - logit[target]) ; stats[1] += count
__global__ void og_masked_ce_fwd_kernel(const __nv_bfloat16* __restrict__ logits, const long long* __restrict__ target,
                                        const unsigned char* __restrict__ mask, long long rows, int V,
                                        float* __restrict__ row_lse, float* __restrict__ stats) {
  const int lane = threadIdx.x & 31;
  const long long w0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  float loss_acc = 0.f, cnt = 0.f;
  for (long long row = w0; row < rows; row += nw) {
    if (!mask[row]) continue;
    const __nv_bfloat16* lp = logits + row * V;
    float m = -INFINITY;
    for (int j = lane; j < V; j += 32) m = fmaxf(m, __bfloat162float(lp[j]));
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int j = lane; j < V; j += 32) s += __expf(__bfloat162float(lp[j]) - m);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float lse = m + __logf(s);
    if (lane == 0) {
      const long long t = target[row];
      if (t < 0 || t >= V) {  // F.cross_entropy raises a device-side assert on a target outside [0, V) (dynamics.py:97)
        printf("og_masked_ce_fwd: target %lld out of range [0, %d)\n", t, V);
        __trap();
      }
      row_lse[row] = lse;
      loss_acc += lse - __bfloat162float(lp[t]);
      cnt += 1.f;
    }
  }
  if (lane == 0 && cnt > 0.f) {
    atomicAdd(&stats[0], loss_acc);
    atomicAdd(&stats[1], cnt);
  }
}

// dlogits[row][j] = mask ? g/count * (softmax_j - [j == target]) : 0
__global__ void og_masked_ce_bwd_kernel(const __nv_bfloat16* __restrict__ logits, const long long* __restrict__ target,
                                        const unsigned char* __restrict__ mask, const float* __restrict__ row_lse,
                                        const float* __restrict__ stats, const float* __restrict__ gloss,
                                        __nv_bfloat16* __restrict__ dlogits, long long rows, int V) {
  const float g = (gloss ? *gloss : 1.f) / fmaxf(stats[1], 1.f);
  const long long total = rows * V;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / V;
    const int j = (int)(i % V);
    float v = 0.f;
    if (mask[row]) {
      long long t = target[row];
      t = t < 0 ? 0 : (t >= V ? V - 1 : t);
      v = g * (__expf(__bfloat162float(logits[i]) - row_lse[row]) - (j == t ? 1.f : 0.f));
    }
    dlogits[i] = __float2bfloat16_rn(v);
  }
}


// ------------------------------------------------------------------------------------------------
// MaskGIT sampling (DynamicsModel.generate, genie/dynamics.py:101-165)
//
// In the reference loop the transformer input `tok_id` is packed ONCE before the loop and never updated (lines
// 128-134), so every iteration sees the same logits; only the multinomial draws differ. The GPU form therefore
// evaluates the transformer once, turns the last frame's logits into per-position CDFs once (og_softmax_cdf), and runs
// ALL sampling iterations in one launch (og_maskgit_sample: one CTA per batch row; per iteration inverse-CDF draw ->
// confidence -> mask already-predicted positions to -inf -> top-k -> scatter into code / mask).
// ------------------------------------------------------------------------------------------------

// logits[row][j] * inv_temp in fp32, for bf16 or fp32 logits
__device__ __forceinline__ float scaled_logit(const void* __restrict__ logits, int logits_f32, long long i,
                                              float inv_temp) {
  return (logits_f32 ? reinterpret_cast<const float*>(logits)[i]
                     : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(logits)[i])) * inv_temp;
}

// cdf[row][j] = sum_{i<=j} softmax(logits[row] * inv_temp)[i], fp32; one warp per row. row_stats[row] = (max, 1/sum):
// prob[j] = expf(logit[j] * inv_temp - max) * (1/sum) is the exact fp32 value the CDF is summed from.
__global__ void og_softmax_cdf_kernel(const void* __restrict__ logits, int logits_f32, long long rows, int V, float inv_temp,
                                      float* __restrict__ cdf, float2* __restrict__ row_stats) {
  const int lane = threadIdx.x & 31;
  const long long w0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long row = w0; row < rows; row += nw) {
    auto at = [&](int j) -> float { return scaled_logit(logits, logits_f32, row * V + j, inv_temp); };
    float m = -INFINITY;
    for (int j = lane; j < V; j += 32) m = fmaxf(m, at(j));
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int j = lane; j < V; j += 32) s += expf(at(j) - m);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float inv = 1.f / s;
    if (row_stats && lane == 0) row_stats[row] = make_float2(m, inv);
    float carry = 0.f;
    for (int j0 = 0; j0 < V; j0 += 32) {
      const int j = j0 + lane;
      float p = j < V ? expf(at(j) - m) * inv : 0.f;
      for (int o = 1; o < 32; o <<= 1) {  // inclusive warp scan
        const float t = __shfl_up_sync(0xffffffffu, p, o);
        if (lane >= o) p += t;
      }
      p += carry;
      // Each lane sums its prefix in a different order, so two adjacent sums can come out in the wrong order (at
      // logits of standard deviation 4, most rows of 1024 have such a step). A running maximum makes every row
      // non-decreasing, which the inverse-CDF search needs; since the exact prefix sums are non-decreasing, no entry
      // moves further from its exact value than the largest error of the sums before it. carry is at most every p of
      // the next chunk.
      for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_up_sync(0xffffffffu, p, o);
        if (lane >= o) p = fmaxf(p, t);
      }
      if (j < V) cdf[row * V + j] = p;
      carry = __shfl_sync(0xffffffffu, p, 31);
    }
  }
}

// One CTA (1024 threads) per batch row; P = h*w positions (P <= 4096).
__global__ void __launch_bounds__(1024)
    og_maskgit_sample_kernel(const float* __restrict__ cdf, const void* __restrict__ logits, int logits_f32,
                             float inv_temp, const float2* __restrict__ row_stats, const float* __restrict__ uniforms,
                             const int* __restrict__ schedule, int steps, int B, int P, int V, long long* __restrict__ code,
                             unsigned char* __restrict__ mask) {
  extern __shared__ unsigned char smem_mg[];
  int Pp = 1;
  while (Pp < P) Pp <<= 1;
  float* key = reinterpret_cast<float*>(smem_mg);           // [Pp] confidence
  int* val = reinterpret_cast<int*>(key + Pp);              // [Pp] position
  int* pred = val + Pp;                                     // [P] sampled token of every position
  __shared__ int remaining;
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {
    int r = 0;
    for (int p = 0; p < P; ++p) r += mask[(long long)b * P + p] ? 1 : 0;
    remaining = r;
  }
  __syncthreads();
  for (int s = 0; s < steps; ++s) {
    if (remaining == 0) break;                              // `if mask.sum() == 0: break` (line 137)
    const int k = schedule[s];
    // draw + confidence (lines 143-151)
    for (int p = threadIdx.x; p < Pp; p += blockDim.x) {
      float c = -INFINITY;
      if (p < P) {
        const long long r = (long long)b * P + p;
        const float* row = cdf + r * V;
        const float u = uniforms[((long long)s * B + b) * P + p] * row[V - 1];
        int lo = 0, hi = V - 1;                             // first j with cdf[j] > u
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (row[mid] > u) hi = mid; else lo = mid + 1;
        }
        pred[p] = lo;
        // confidence = prob[pred] (line 146), recomputed from the row's (max, 1/sum). The difference of two CDF
        // entries would carry an absolute error of about one ulp of the running sum, which reorders unlikely draws.
        const float2 st = row_stats[r];
        const float pr = expf(scaled_logit(logits, logits_f32, r * V + lo, inv_temp) - st.x) * st.y;
        c = mask[(long long)b * P + p] ? pr : -INFINITY;    // conf[~mask] = -inf (line 151)
      }
      key[p] = c;
      val[p] = p;
    }
    __syncthreads();
    // top-k: bitonic sort by (confidence descending, position ascending)
    for (int size = 2; size <= Pp; size <<= 1) {
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        for (int i = threadIdx.x; i < Pp; i += blockDim.x) {
          const int j = i ^ stride;
          if (j > i) {
            const bool desc = (i & size) == 0;
            const float ki = key[i], kj = key[j];
            const int vi = val[i], vj = val[j];
            const bool i_first = (ki > kj) || (ki == kj && vi < vj);   // i should precede j in descending order
            if (desc ? !i_first : i_first) {
              key[i] = kj; key[j] = ki;
              val[i] = vj; val[j] = vi;
            }
          }
        }
        __syncthreads();
      }
    }
    // scatter the k most confident predictions (lines 154-163)
    for (int i = threadIdx.x; i < k && i < Pp; i += blockDim.x) {
      const int p = val[i];
      if (p < P) {
        code[(long long)b * P + p] = pred[p];
        mask[(long long)b * P + p] = 0;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int r = 0;
      for (int p = 0; p < P; ++p) r += mask[(long long)b * P + p] ? 1 : 0;
      remaining = r;
    }
    __syncthreads();
  }
}

static int grid_for(long long total, int block, int per_sm) {
  long long g = (total + block - 1) / block;
  long long cap = (long long)num_sms() * per_sm;
  if (g > cap) g = cap;
  return (int)(g < 1 ? 1 : g);
}

}  // namespace og

using namespace og;

extern "C" int og_embed_add_fwd(const int64_t* tok, const int64_t* act, const float* tok_w, const float* act_w, void* out,
                                int64_t rows, int64_t rows_per_act, int C, int tok_vocab, int act_vocab,
                                og_stream_t stream) {
  OG_REQUIRE(tok && act && tok_w && act_w && out && rows > 0 && rows_per_act > 0, "embed_add_fwd: bad arguments");
  OG_REQUIRE(C % 8 == 0, "embed_add_fwd: C=%d must be a multiple of 8", C);
  og_embed_add_fwd_kernel<<<grid_for(rows * (C / 8), 256, 16), 256, 0, (cudaStream_t)stream>>>(
      (const long long*)tok, (const long long*)act, tok_w, act_w, (__nv_bfloat16*)out, rows, rows_per_act, C, tok_vocab,
      act_vocab);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_embed_add_bwd(const int64_t* tok, const int64_t* act, const void* dy, float* d_tok_w, float* d_act_w,
                                int64_t rows, int64_t rows_per_act, int C, int tok_vocab, int act_vocab,
                                og_stream_t stream) {
  OG_REQUIRE(tok && act && dy && d_tok_w && d_act_w && rows > 0, "embed_add_bwd: bad arguments");
  OG_REQUIRE(C % 8 == 0, "embed_add_bwd: C=%d must be a multiple of 8", C);
  og_embed_add_bwd_kernel<<<grid_for(rows * (C / 8), 256, 16), 256, 0, (cudaStream_t)stream>>>(
      (const long long*)tok, (const long long*)act, (const __nv_bfloat16*)dy, d_tok_w, d_act_w, rows, rows_per_act, C,
      tok_vocab, act_vocab);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_masked_ce_fwd(const void* logits, const int64_t* target, const uint8_t* mask, int64_t rows, int V,
                                float* row_lse, float* stats, og_stream_t stream) {
  OG_REQUIRE(logits && target && mask && row_lse && stats && rows > 0 && V > 0, "masked_ce_fwd: bad arguments");
  og_masked_ce_fwd_kernel<<<grid_for(rows, 8, 8), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)logits, (const long long*)target, mask, rows, V, row_lse, stats);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_masked_ce_bwd(const void* logits, const int64_t* target, const uint8_t* mask, const float* row_lse,
                                const float* stats, const float* gloss, void* dlogits, int64_t rows, int V,
                                og_stream_t stream) {
  OG_REQUIRE(logits && target && mask && row_lse && stats && dlogits, "masked_ce_bwd: bad arguments");
  og_masked_ce_bwd_kernel<<<grid_for(rows * V, 256, 16), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)logits, (const long long*)target, mask, row_lse, stats, gloss, (__nv_bfloat16*)dlogits, rows,
      V);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_softmax_cdf(const void* logits, int logits_f32, int64_t rows, int V, float inv_temp, float* cdf,
                              float* row_stats, og_stream_t stream) {
  OG_REQUIRE(logits && cdf && rows > 0 && V > 0, "softmax_cdf: bad arguments");
  og_softmax_cdf_kernel<<<grid_for(rows, 8, 8), 256, 0, (cudaStream_t)stream>>>(logits, logits_f32, rows, V, inv_temp, cdf,
                                                                               reinterpret_cast<float2*>(row_stats));
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_maskgit_sample(const float* cdf, const void* logits, int logits_f32, float inv_temp,
                                 const float* row_stats, const float* uniforms, const int* schedule, int steps, int B,
                                 int P, int V, int64_t* code, uint8_t* mask, og_stream_t stream) {
  OG_REQUIRE(cdf && logits && row_stats && uniforms && schedule && code && mask && steps > 0 && B > 0 && V > 0,
             "maskgit_sample: bad arguments");
  OG_REQUIRE(P > 0 && P <= 4096, "maskgit_sample: P=%d positions per frame must be in [1, 4096]", P);
  int Pp = 1;
  while (Pp < P) Pp <<= 1;
  const size_t smem = (size_t)Pp * 8 + (size_t)P * 4;
  static bool attr_set = false;
  if (!attr_set) {
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_maskgit_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    attr_set = true;
  }
  og_maskgit_sample_kernel<<<B, 1024, smem, (cudaStream_t)stream>>>(
      cdf, logits, logits_f32, inv_temp, reinterpret_cast<const float2*>(row_stats), uniforms, schedule, steps, B, P, V,
      (long long*)code, mask);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}
