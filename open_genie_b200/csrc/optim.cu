// optim.cu — fused multi-tensor AdamW on fp32 master weights, emitting the bf16 operand copy the
// conv kernels read, in ONE launch for the whole model (HBM-bound: 16 B read + 12..14 B written / param).
//
// Replaces torch.optim.AdamW as configured by VideoTokenizer.configure_optimizers
// (genie/tokenizer.py:437-442; defaults lr=1e-3, betas=(0.9,0.999), eps=1e-8, weight_decay=1e-2) and the
// fp32->bf16 weight cast that autocast would perform on every conv call (config/tokenize.yaml:78).
#include "og_host.cuh"
#include "og_ptx.cuh"

namespace og {
extern std::atomic<uint64_t> g_launches;

static constexpr int kChunk = 2048;  // elements per block-iteration

__global__ void __launch_bounds__(256)
    og_adamw_kernel(const og_adamw_tensor* __restrict__ table, const int* __restrict__ chunk_tensor,
                    const int* __restrict__ chunk_index, int num_chunks, float lr, float beta1, float beta2,
                    float eps, float weight_decay, float bc1_host, float bc2_host, const int* __restrict__ step_dev,
                    const float* __restrict__ lr_dev, const float* __restrict__ grad_scale) {
  const float gs = grad_scale ? *grad_scale : 1.f;
  // step count / learning rate may live in device memory so that a captured CUDA graph of the whole
  // training step stays valid across replays (host scalars would be frozen at capture time)
  float bc1 = bc1_host, bc2 = bc2_host;
  if (step_dev) {
    const float t = (float)(*step_dev);
    bc1 = 1.f - powf(beta1, t);
    bc2 = sqrtf(1.f - powf(beta2, t));
  }
  if (lr_dev) lr = *lr_dev;
  for (int ch = blockIdx.x; ch < num_chunks; ch += gridDim.x) {
    const og_adamw_tensor t = table[chunk_tensor[ch]];
    const long long base = (long long)chunk_index[ch] * kChunk;
    const bool vec = (base + kChunk <= t.n) && ((reinterpret_cast<uintptr_t>(t.p + base) & 15) == 0) && t.g &&
                     ((reinterpret_cast<uintptr_t>(t.g + base) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(t.m + base) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(t.v + base) & 15) == 0) && (t.row_len % 4 == 0) &&
                     // the bf16 copy goes out as 8-byte stores: 4 elements never straddle a row, and every row
                     // start must be 8-byte aligned
                     (!t.p_bf16 || (((reinterpret_cast<uintptr_t>(t.p_bf16) & 7) == 0) && t.dst_ld % 4 == 0));
    if (vec) {
      // 16-byte path: 4 parameters per thread-iteration, bf16 copy written as one 8-byte store
      for (int e = threadIdx.x * 4; e < kChunk; e += 256 * 4) {
        const long long i = base + e;
        float4 p4 = *reinterpret_cast<const float4*>(t.p + i);
        const float4 g4 = *reinterpret_cast<const float4*>(t.g + i);
        float4 m4 = *reinterpret_cast<const float4*>(t.m + i);
        float4 v4 = *reinterpret_cast<const float4*>(t.v + i);
        float* pp = &p4.x;
        const float* gp = &g4.x;
        float* mp = &m4.x;
        float* vp = &v4.x;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float g = gp[k] * gs;
          pp[k] *= (1.f - lr * weight_decay);
          mp[k] = beta1 * mp[k] + (1.f - beta1) * g;
          vp[k] = beta2 * vp[k] + (1.f - beta2) * g * g;
          pp[k] -= (lr / bc1) * (mp[k] / (sqrtf(vp[k]) / bc2 + eps));
        }
        *reinterpret_cast<float4*>(t.p + i) = p4;
        *reinterpret_cast<float4*>(t.m + i) = m4;
        *reinterpret_cast<float4*>(t.v + i) = v4;
        if (t.p_bf16) {
          const long long row = i / t.row_len, col = i - row * t.row_len;
          uint2 u;
          u.x = pack_bf16x2(p4.x, p4.y);
          u.y = pack_bf16x2(p4.z, p4.w);
          *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(t.p_bf16) + row * t.dst_ld + col) = u;
        }
      }
      continue;
    }
    for (int e = threadIdx.x; e < kChunk; e += 256) {
      const long long i = base + e;
      if (i >= t.n) break;
      float p = t.p[i];
      if (t.g) {
        const float g = t.g[i] * gs;
        float m = t.m[i], v = t.v[i];
        p *= (1.f - lr * weight_decay);
        m = beta1 * m + (1.f - beta1) * g;
        v = beta2 * v + (1.f - beta2) * g * g;
        const float denom = sqrtf(v) / bc2 + eps;  // bc2 = sqrt(1 - beta2^t)
        p -= (lr / bc1) * (m / denom);
        t.p[i] = p;
        t.m[i] = m;
        t.v[i] = v;
      }
      if (t.p_bf16) {
        const long long row = i / t.row_len, col = i - row * t.row_len;
        reinterpret_cast<__nv_bfloat16*>(t.p_bf16)[row * t.dst_ld + col] = __float2bfloat16_rn(p);
      }
    }
  }
}

}  // namespace og

using namespace og;

extern "C" int og_adamw_chunk_elems(void) { return kChunk; }

__global__ void og_adamw_tick_kernel(int* step) { *step += 1; }

extern "C" int og_adamw_tick(int* step_dev, og_stream_t stream) {
  OG_REQUIRE(step_dev, "adamw_tick: null pointer");
  og_adamw_tick_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step_dev);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_adamw_step(const og_adamw_tensor* table_dev, const int* chunk_tensor_dev, const int* chunk_index_dev,
                             int num_chunks, float lr, float beta1, float beta2, float eps, float weight_decay,
                             int step, const int* step_dev, const float* lr_dev, const float* grad_scale_dev,
                             og_stream_t stream) {
  OG_REQUIRE(table_dev && chunk_tensor_dev && chunk_index_dev && num_chunks > 0 && step >= 1,
             "adamw_step: bad arguments");
  const float bc1 = (float)(1.0 - pow((double)beta1, (double)step));
  const float bc2 = (float)sqrt(1.0 - pow((double)beta2, (double)step));
  int grid = num_sms() * 8;
  if (grid > num_chunks) grid = num_chunks;
  og_adamw_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(table_dev, chunk_tensor_dev, chunk_index_dev, num_chunks, lr,
                                                         beta1, beta2, eps, weight_decay, bc1, bc2, step_dev, lr_dev, grad_scale_dev);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}
