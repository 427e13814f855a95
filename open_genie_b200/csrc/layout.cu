// layout.cu — data-movement kernels around the conv stack (all HBM-bound, coalesced on the
// channel-contiguous side, 16-byte vectors where the channel count allows):
//   * NCDHW fp32 <-> NDHWC bf16/fp32 casts at the Python boundary (the reference keeps NCDHW fp32
//     everywhere; the product keeps NDHWC bf16 between kernels)
//   * depth-to-space-time pixel shuffle 'b (c p q r) t h w -> b c (t p) (h q) (w r)' and its inverse
//     (genie/module/video.py:403-408)
//   * mse_loss forward / backward (tokenizer.py:364, action.py:166), bias gradient (column sums)
#include "og_host.cuh"
#include "og_ptx.cuh"

namespace og {
extern std::atomic<uint64_t> g_launches;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static int ew_blocks(long long total, int block) {
  long long g = (total + block - 1) / block;
  long long cap = (long long)num_sms() * 32;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

// NCDHW f32 -> NDHWC (bf16 or f32), via a 32x32 smem transpose over (channel, voxel)
template <typename OutT>
__global__ void og_ncdhw_to_ndhwc_kernel(const float* __restrict__ x, OutT* __restrict__ y, int C, long long V) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const long long v0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i;
    const long long v = v0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && v < V) ? x[((long long)n * C + c) * V + v] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const long long v = v0 + i;
    const int c = c0 + threadIdx.x;
    if (c < C && v < V) {
      const float val = tile[threadIdx.x][i];
      if constexpr (sizeof(OutT) == 2)
        y[((long long)n * V + v) * C + c] = __float2bfloat16_rn(val);
      else
        y[((long long)n * V + v) * C + c] = val;
    }
  }
}

template <typename InT>
__global__ void og_ndhwc_to_ncdhw_kernel(const InT* __restrict__ x, float* __restrict__ y, int C, long long V) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const long long v0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const long long v = v0 + i;
    const int c = c0 + threadIdx.x;
    float val = 0.f;
    if (c < C && v < V) {
      if constexpr (sizeof(InT) == 2)
        val = __bfloat162float(x[((long long)n * V + v) * C + c]);
      else
        val = x[((long long)n * V + v) * C + c];
    }
    tile[i][threadIdx.x] = val;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i;
    const long long v = v0 + threadIdx.x;
    if (c < C && v < V) y[((long long)n * C + c) * V + v] = tile[threadIdx.x][i];
  }
}

// pixel shuffle. forward: x [N,T,H,W,c*p*q*r] -> y [N,T*p,H*q,W*r,c]; channel index of x = ((cc*p+pp)*q+qq)*r+rr
// One thread per (output voxel, 8-channel... ) the gather side is strided by p*q*r, so go scalar on x and
// vector on y: thread handles 8 consecutive output channels.
__global__ void og_pixel_shuffle_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int T,
                                        int H, int W, int c, int p, int q, int r, long long total_vec, int inverse) {
  const int cv = c >> 3;
  const int pqr = p * q * r;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total_vec;
       i += (long long)gridDim.x * blockDim.x) {
    const int v8 = (int)(i % cv);
    long long o = i / cv;  // output voxel index over [N, T*p, H*q, W*r]
    const int wo = (int)(o % (W * r));
    o /= (W * r);
    const int ho = (int)(o % (H * q));
    o /= (H * q);
    const int to = (int)(o % (T * p));
    const int n = (int)(o / (T * p));
    const int t = to / p, pp = to % p, h = ho / q, qq = ho % q, w = wo / r, rr = wo % r;
    const long long vin = (((long long)n * T + t) * H + h) * W + w;
    const int sub = (pp * q + qq) * r + rr;
    __nv_bfloat16* yp = y + ((((long long)n * T * p + to) * (H * q) + ho) * (long long)(W * r) + wo) * c + v8 * 8;
    const long long xb = vin * ((long long)c * pqr) + (long long)(v8 * 8) * pqr + sub;
    if (!inverse) {
      __nv_bfloat16 tmp[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) tmp[k] = x[xb + (long long)k * pqr];
      *reinterpret_cast<uint4*>(yp) = *reinterpret_cast<uint4*>(tmp);
    } else {
      // inverse: here `y` is the SHUFFLED tensor (read) and `x` the un-shuffled one (written)
      __nv_bfloat16 tmp[8];
      *reinterpret_cast<uint4*>(tmp) = *reinterpret_cast<const uint4*>(yp);
      __nv_bfloat16* xw = const_cast<__nv_bfloat16*>(x);
#pragma unroll
      for (int k = 0; k < 8; ++k) xw[xb + (long long)k * pqr] = tmp[k];
    }
  }
}

// Any channel count (REPR_TOK_DEC ends in out_channels = 3, genie/tokenizer.py:196-204): one thread per output element.
__global__ void og_pixel_shuffle_scalar_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int T,
                                               int H, int W, int c, int p, int q, int r, long long total, int inverse) {
  const int pqr = p * q * r;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(i % c);
    long long o = i / c;  // output voxel index over [N, T*p, H*q, W*r]
    const int wo = (int)(o % (W * r));
    o /= (W * r);
    const int ho = (int)(o % (H * q));
    o /= (H * q);
    const int to = (int)(o % (T * p));
    const int n = (int)(o / (T * p));
    const int t = to / p, pp = to % p, h = ho / q, qq = ho % q, w = wo / r, rr = wo % r;
    const long long vin = (((long long)n * T + t) * H + h) * W + w;
    const long long xi = vin * ((long long)c * pqr) + (long long)ch * pqr + (pp * q + qq) * r + rr;
    if (!inverse)
      y[i] = x[xi];
    else
      const_cast<__nv_bfloat16*>(x)[xi] = y[i];
  }
}

// Vector form for p*q*r in {2, 4, 8}: one thread owns 8 consecutive output channels of ONE input voxel, i.e. a
// contiguous run of 8*PQR input channels (PQR 16-byte loads), transposes the 8 x PQR block in registers and
// writes one 16-byte vector to each of the PQR output voxels. Loads and stores are both fully coalesced; the
// scalar kernel above gathers 2-byte elements PQR apart and ran ~20x below the HBM roofline.
template <int PQR>
__global__ void __launch_bounds__(256)
    og_pixel_shuffle_vec_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int T, int H, int W, int c, int p,
                                int q, int r, long long total, int inverse) {
  const int cv = c >> 3;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int oct = (int)(i % cv);
    long long vin = i / cv;
    const long long xoff = (vin * cv + oct) * PQR;  // in uint4 units: voxel row has cv*PQR vectors
    const int w = (int)(vin % W);
    vin /= W;
    const int h = (int)(vin % H);
    vin /= H;
    const int t = (int)(vin % T);
    const int n = (int)(vin / T);
    union Blk {
      uint4 v[PQR];
      unsigned short e[8 * PQR];
    };
    Blk a, b;
    if (!inverse) {
#pragma unroll
      for (int k = 0; k < PQR; ++k) a.v[k] = __ldg(x + xoff + k);
#pragma unroll
      for (int sub = 0; sub < PQR; ++sub)
#pragma unroll
        for (int cc = 0; cc < 8; ++cc) b.e[sub * 8 + cc] = a.e[cc * PQR + sub];
    }
#pragma unroll
    for (int sub = 0; sub < PQR; ++sub) {
      const int pp = sub / (q * r), qq = (sub / r) % q, rr = sub % r;
      const long long ov = (((long long)n * T * p + t * p + pp) * (H * q) + h * q + qq) * (long long)(W * r) + w * r + rr;
      if (!inverse)
        y[ov * cv + oct] = b.v[sub];
      else
        b.v[sub] = __ldg(y + ov * cv + oct);
    }
    if (inverse) {
#pragma unroll
      for (int sub = 0; sub < PQR; ++sub)
#pragma unroll
        for (int cc = 0; cc < 8; ++cc) a.e[cc * PQR + sub] = b.e[sub * 8 + cc];
      uint4* xw = const_cast<uint4*>(x);
#pragma unroll
      for (int k = 0; k < PQR; ++k) xw[xoff + k] = a.v[k];
    }
  }
}

// mse: rec NDHWC fp32 [N,V,C] vs target NCDHW fp32 [N,C,V]. loss_sum += sum (rec - tgt)^2
__global__ void og_mse_fwd_kernel(const float* __restrict__ rec, const float* __restrict__ tgt, int C, long long V,
                                  long long total, float* __restrict__ loss_sum) {
  float acc = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    // iterate in target (NCDHW) order: i = (n*C + c)*V + v  -> coalesced target reads; rec reads are
    // C-strided but C is tiny (3) so every sector is still fully used across the c-loop of neighbours
    const long long v = i % V;
    const long long nc = i / V;
    const int c = (int)(nc % C);
    const long long n = nc / C;
    const float d = rec[(n * V + v) * C + c] - tgt[i];
    acc = fmaf(d, d, acc);
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ float ws[32];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? ws[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) atomicAdd(loss_sum, v);
  }
}

// d_rec[n,v,c] = gscale * 2 (rec - tgt) / numel, written as bf16 NDHWC with cpad channels (zero padded)
__global__ void og_mse_bwd_kernel(const float* __restrict__ rec, const float* __restrict__ tgt,
                                  const float* __restrict__ gscale, float coef, int C, int cpad, long long V,
                                  long long total, __nv_bfloat16* __restrict__ drec) {
  const float g = (gscale ? *gscale : 1.f) * coef;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cpad);
    const long long nv = i / cpad;
    float val = 0.f;
    if (c < C) {
      const long long n = nv / V, v = nv % V;
      val = g * (rec[nv * C + c] - tgt[(n * C + c) * V + v]);
    }
    drec[i] = __float2bfloat16_rn(val);
  }
}

// column sums (bias gradient): out[c] += sum_rows x[row][c]; x bf16 [rows][ld], first C columns
__global__ void og_colsum_kernel(const __nv_bfloat16* __restrict__ x, long long rows, int C, int ld,
                                 float* __restrict__ out) {
  // block handles 256 rows x all columns; thread t -> column t (loop), coalesced along c
  const long long r0 = (long long)blockIdx.x * 256;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = 0.f;
    for (int r = 0; r < 256; ++r) {
      const long long row = r0 + r;
      if (row >= rows) break;
      acc += __bfloat162float(x[row * ld + c]);
    }
    atomicAdd(&out[c], acc);
  }
}

// vectorised column sums for ld % 8 == 0: grid (row blocks, column blocks of <= 2048 channels); a block owns
// a contiguous row range, thread -> (8-channel vector, row lane), fp32 partials in registers over the whole
// range with 4 independent 16-byte loads in flight, then shared atomics and one global atomic per channel.
__global__ void __launch_bounds__(256) og_colsum_vec_kernel(const uint4* __restrict__ x, long long rows, int C, int ld,
                                                            long long rows_per_block, float* __restrict__ out) {
  __shared__ float part[256 * 8];  // per-thread partial column sums
  const int c0 = blockIdx.y * 2048;
  const int cw = (ld - c0 < 2048) ? ld - c0 : 2048;  // columns of this block
  const int cvs = cw >> 3, ldv = ld >> 3;
  const int lanes = 256 / cvs;
  const int cv = threadIdx.x % cvs, rl = threadIdx.x / cvs;
  const long long r0 = (long long)blockIdx.x * rows_per_block;
  const long long rend = (r0 + rows_per_block < rows) ? r0 + rows_per_block : rows;
  if (rl < lanes && r0 < rows) {
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const uint4* base = x + (c0 >> 3) + cv;
    long long r = r0 + rl;
    for (; r + 3LL * lanes < rend; r += 4LL * lanes) {
      uint4 u[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) u[k] = __ldg(base + (r + (long long)k * lanes) * ldv);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u[k]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 t = __bfloat1622float2(h[i]);
          acc[2 * i] += t.x;
          acc[2 * i + 1] += t.y;
        }
      }
    }
    for (; r < rend; r += lanes) {
      const uint4 u = __ldg(base + r * ldv);
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 t = __bfloat1622float2(h[i]);
        acc[2 * i] += t.x;
        acc[2 * i + 1] += t.y;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) part[threadIdx.x * 8 + i] = acc[i];
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) part[threadIdx.x * 8 + i] = 0.f;
  }
  __syncthreads();
  // thread index == rl * cvs + cv: sum the row lanes of each column (no contended shared atomics)
  for (int c = threadIdx.x; c < cw; c += 256) {
    float a = 0.f;
    for (int l = 0; l < lanes; ++l) a += part[(l * cvs + (c >> 3)) * 8 + (c & 7)];
    if (c0 + c < C) atomicAdd(&out[c0 + c], a);
  }
}

// copy [rows][cs] -> [rows][cd] (cd >= cs zero padded, or cd < cs truncating); src f32 or bf16, dst bf16
template <typename InT>
__global__ void og_pad_channels_kernel(const InT* __restrict__ x, __nv_bfloat16* __restrict__ y, int cs, int cd,
                                       long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cd);
    const long long row = i / cd;
    float v = 0.f;
    if (c < cs) {
      if constexpr (sizeof(InT) == 2)
        v = __bfloat162float(x[row * cs + c]);
      else
        v = x[row * cs + c];
    }
    y[i] = __float2bfloat16_rn(v);
  }
}

// strided row copy with cast: dst[row*dst_ld + c] = bf16(src[row*src_ld + c]), c < cols
template <typename InT>
__global__ void og_copy_rows_kernel(const InT* __restrict__ src, long long src_ld, __nv_bfloat16* __restrict__ dst,
                                    long long dst_ld, int cols, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cols);
    const long long row = i / cols;
    float v;
    if constexpr (sizeof(InT) == 2)
      v = __bfloat162float(src[row * src_ld + c]);
    else
      v = src[row * src_ld + c];
    dst[row * dst_ld + c] = __float2bfloat16_rn(v);
  }
}

// out = a - b (bf16, 8 elements per thread): recovers the attention output o = y - x from the saved block output
__global__ void og_sub_rows_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ out,
                                   long long nvec) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * blockDim.x) {
    const uint4 ua = __ldg(a + i), ub = __ldg(b + i);
    const __nv_bfloat162* ha = reinterpret_cast<const __nv_bfloat162*>(&ua);
    const __nv_bfloat162* hb = reinterpret_cast<const __nv_bfloat162*>(&ub);
    uint4 r;
    uint32_t* rw = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 fa = __bfloat1622float2(ha[k]), fb = __bfloat1622float2(hb[k]);
      rw[k] = pack_bf16x2(fa.x - fb.x, fa.y - fb.y);
    }
    out[i] = r;
  }
}

}  // namespace og

using namespace og;

extern "C" int og_sub_rows(const void* a, const void* b, void* out, int64_t n, og_stream_t stream) {
  OG_REQUIRE(a && b && out && n > 0 && n % 8 == 0, "sub_rows: bad arguments (n must be a multiple of 8)");
  OG_REQUIRE(aligned16(a) && aligned16(b) && aligned16(out), "sub_rows: a, b and out must be 16-byte aligned");
  og_sub_rows_kernel<<<ew_blocks(n / 8, 256), 256, 0, (cudaStream_t)stream>>>((const uint4*)a, (const uint4*)b,
                                                                             (uint4*)out, n / 8);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_copy_rows_to_bf16(const void* src, int src_f32, int64_t src_ld, void* dst, int64_t dst_ld,
                                    int64_t rows, int cols, og_stream_t stream) {
  OG_REQUIRE(src && dst && rows > 0 && cols > 0, "copy_rows_to_bf16: bad arguments");
  const long long total = (long long)rows * cols;
  if (src_f32)
    og_copy_rows_kernel<float><<<ew_blocks(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const float*)src, src_ld, (__nv_bfloat16*)dst, dst_ld, cols, total);
  else
    og_copy_rows_kernel<__nv_bfloat16><<<ew_blocks(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)src, src_ld, (__nv_bfloat16*)dst, dst_ld, cols, total);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_ncdhw_f32_to_ndhwc(const float* x, void* y, int y_f32, int N, int C, int64_t V,
                                     og_stream_t stream) {
  OG_REQUIRE(x && y && N > 0 && C > 0 && V > 0, "ncdhw_to_ndhwc: bad arguments");
  dim3 grid((unsigned)((V + 31) / 32), (C + 31) / 32, N), block(32, 8);
  if (y_f32)
    og_ncdhw_to_ndhwc_kernel<float><<<grid, block, 0, (cudaStream_t)stream>>>(x, (float*)y, C, V);
  else
    og_ncdhw_to_ndhwc_kernel<__nv_bfloat16><<<grid, block, 0, (cudaStream_t)stream>>>(x, (__nv_bfloat16*)y, C, V);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_ndhwc_to_ncdhw_f32(const void* x, int x_f32, float* y, int N, int C, int64_t V,
                                     og_stream_t stream) {
  OG_REQUIRE(x && y && N > 0 && C > 0 && V > 0, "ndhwc_to_ncdhw: bad arguments");
  dim3 grid((unsigned)((V + 31) / 32), (C + 31) / 32, N), block(32, 8);
  if (x_f32)
    og_ndhwc_to_ncdhw_kernel<float><<<grid, block, 0, (cudaStream_t)stream>>>((const float*)x, y, C, V);
  else
    og_ndhwc_to_ncdhw_kernel<__nv_bfloat16><<<grid, block, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, y, C, V);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_pixel_shuffle3d(const void* x, void* y, int inverse, int N, int T, int H, int W, int c, int p,
                                  int q, int r, og_stream_t stream) {
  OG_REQUIRE(x && y, "pixel_shuffle3d: null pointer");
  OG_REQUIRE(c >= 1 && p >= 1 && q >= 1 && r >= 1, "pixel_shuffle3d: bad shape (c=%d p=%d q=%d r=%d)", c, p, q, r);
  OG_REQUIRE(N >= 1 && T >= 1 && H >= 1 && W >= 1, "pixel_shuffle3d: bad extents (N=%d T=%d H=%d W=%d)", N, T, H, W);
  // og_pixel_shuffle_kernel moves 8 channels of y as one 16-byte vector: a y off that alignment goes scalar
  if (c % 8 != 0 || !aligned16(y)) {
    const long long tot = (long long)N * T * p * H * q * W * r * c;
    og_pixel_shuffle_scalar_kernel<<<ew_blocks(tot, 256), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x, (__nv_bfloat16*)y, T, H, W, c, p, q, r, tot, inverse);
    OG_CHECK_CUDA(cudaGetLastError());
    g_launches.fetch_add(1);
    return OG_OK;
  }
  const long long total = (long long)N * T * p * H * q * W * r * (c / 8);
  // forward: x un-shuffled (read), y shuffled (written). inverse: y shuffled (read), x un-shuffled (written).
  const int pqr = p * q * r;
  const long long tv = (long long)N * T * H * W * (c / 8);
  const bool aligned = aligned16(x);   // y is 16-byte aligned here
  if (aligned && pqr == 8)
    og_pixel_shuffle_vec_kernel<8><<<ew_blocks(tv, 256), 256, 0, (cudaStream_t)stream>>>(
        (const uint4*)x, (uint4*)y, T, H, W, c, p, q, r, tv, inverse);
  else if (aligned && pqr == 4)
    og_pixel_shuffle_vec_kernel<4><<<ew_blocks(tv, 256), 256, 0, (cudaStream_t)stream>>>(
        (const uint4*)x, (uint4*)y, T, H, W, c, p, q, r, tv, inverse);
  else if (aligned && pqr == 2)
    og_pixel_shuffle_vec_kernel<2><<<ew_blocks(tv, 256), 256, 0, (cudaStream_t)stream>>>(
        (const uint4*)x, (uint4*)y, T, H, W, c, p, q, r, tv, inverse);
  else
    og_pixel_shuffle_kernel<<<ew_blocks(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x, (__nv_bfloat16*)y, T, H, W, c, p, q, r, total, inverse);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_mse_fwd(const float* rec_ndhwc, const float* tgt_ncdhw, int N, int C, int64_t V, float* loss_sum,
                          og_stream_t stream) {
  OG_REQUIRE(rec_ndhwc && tgt_ncdhw && loss_sum, "mse_fwd: null pointer");
  const long long total = (long long)N * C * V;
  og_mse_fwd_kernel<<<ew_blocks(total, 256), 256, 0, (cudaStream_t)stream>>>(rec_ndhwc, tgt_ncdhw, C, V, total,
                                                                            loss_sum);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_mse_bwd(const float* rec_ndhwc, const float* tgt_ncdhw, const float* gscale, int N, int C, int cpad,
                          int64_t V, void* drec, og_stream_t stream) {
  OG_REQUIRE(rec_ndhwc && tgt_ncdhw && drec && cpad >= C, "mse_bwd: bad arguments");
  const long long total = (long long)N * V * cpad;
  const float coef = (float)(2.0 / ((double)N * C * V));
  og_mse_bwd_kernel<<<ew_blocks(total, 256), 256, 0, (cudaStream_t)stream>>>(rec_ndhwc, tgt_ncdhw, gscale, coef, C,
                                                                            cpad, V, total, (__nv_bfloat16*)drec);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_colsum(const void* x, int64_t rows, int C, int ld, float* out, og_stream_t stream) {
  OG_REQUIRE(x && out && rows > 0 && C > 0 && ld >= C, "colsum: bad arguments (rows=%lld C=%d ld=%d)", (long long)rows,
             C, ld);
  if (ld % 8 == 0 && (ld <= 2048 || ld % 2048 == 0) && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const int col_blocks = (ld + 2047) / 2048;
    long long want = (4LL * num_sms() + col_blocks - 1) / col_blocks;
    long long groups = (rows + 63) / 64;
    if (want > groups) want = groups;
    if (want < 1) want = 1;
    const long long rpb = ((groups + want - 1) / want) * 64;
    dim3 grid((unsigned)((rows + rpb - 1) / rpb), col_blocks);
    og_colsum_vec_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint4*)x, rows, C, ld, rpb, out);
  } else {
    const unsigned blocks = (unsigned)((rows + 255) / 256);
    og_colsum_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, rows, C, ld, out);
  }
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_pad_channels(const void* x, int x_f32, void* y, int64_t rows, int cs, int cd, og_stream_t stream) {
  OG_REQUIRE(x && y && cs > 0 && cd > 0, "pad_channels: bad arguments");
  const long long total = (long long)rows * cd;
  if (x_f32)
    og_pad_channels_kernel<float><<<ew_blocks(total, 256), 256, 0, (cudaStream_t)stream>>>((const float*)x,
                                                                                        (__nv_bfloat16*)y, cs, cd, total);
  else
    og_pad_channels_kernel<__nv_bfloat16><<<ew_blocks(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x, (__nv_bfloat16*)y, cs, cd, total);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

// ------------------------------------------------------------------------------------------------
// BlurPooling3d (genie/module/video.py:487-537): the reference repeats ONE Pascal kernel over a conv with
// `num_groups` = G groups, so output channel o of group g = o / (C_out/G) equals blur(sum of the C_in/G input
// channels of group g) (SURVEY.md §8 a6). G = 1 is a dense conv: every output channel is blur(sum_c x[:, c]).
//   pass 1: s[v][g] = sum_{c in group g} x[v][c]       (fp32 [N*T*H*W][G])
//   pass 2: y[vo][o] = sum_taps blur[tap] * s[vo*stride + tap - pad][g(o)]   (bf16 NDHWC, 16-byte vectors)
// The adjoint (backward) is the same pair with the stencil transposed: g[vo][g] = sum_{o in group g} dy[vo][o], then
//   dx[v][c] = sum over (tap, vo) hitting v of blur[tap] * g[vo][g(c)].
// Each 16-byte vector of 8 channels lies inside one group ((C/G) % 8 == 0), so pass 2 writes whole vectors.
// ptxas -v (sm_90a, -O3): og_channel_sum_kernel 30 registers, og_group_sum_kernel 40, og_blur3d_fwd_kernel 48,
// og_blur3d_bwd_kernel 46; no spills, 0-byte stack frames.
// ------------------------------------------------------------------------------------------------
namespace og {

__global__ void og_channel_sum_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ s, long long rows, int C) {
  const int lane = threadIdx.x & 31;
  const long long w0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long r = w0; r < rows; r += nw) {
    float a = 0.f;
    for (int c = lane; c < C; c += 32) a += __bfloat162float(x[r * C + c]);
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) s[r] = a;
  }
}

// num_groups > 1: one thread per (row, group). A group is cg = C / G contiguous channels (cg % 8 == 0), so the sum of
// entry i = row * G + g reads cg / 8 whole 16-byte vectors starting at x + i * cg, and adds them in channel order.
__global__ void og_group_sum_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ s, long long n_sums, int cg) {
  const int nv = cg >> 3;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_sums;
       i += (long long)gridDim.x * blockDim.x) {
    const uint4* p = reinterpret_cast<const uint4*>(x) + i * nv;
    float a = 0.f;
    for (int v = 0; v < nv; ++v) {
      const uint4 u = __ldg(p + v);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[j]));
        a += f.x;
        a += f.y;
      }
    }
    s[i] = a;
  }
}

__device__ __forceinline__ float pascal(int k, int i) {  // binomial(k-1, i)
  float v = 1.f;
  for (int j = 0; j < i; ++j) v = v * (float)(k - 1 - j) / (float)(j + 1);
  return v;
}

// forward stencil + broadcast over the group: one thread per (output voxel, 8-channel vector)
__global__ void og_blur3d_fwd_kernel(const float* __restrict__ s, __nv_bfloat16* __restrict__ y, int T, int H, int W,
                                     int To, int Ho, int Wo, int k, int st, int sh, int sw, int Cout, float norm,
                                     long long total_vec, int kt, int pad_t, int pad, int G) {
  const int cv = Cout >> 3, gv = cv / G;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total_vec;
       i += (long long)gridDim.x * blockDim.x) {
    long long vo = i / cv;
    const int g = (int)(i - vo * cv) / gv;
    const int wo = (int)(vo % Wo);
    long long r = vo / Wo;
    const int ho = (int)(r % Ho);
    r /= Ho;
    const int to = (int)(r % To);
    const int n = (int)(r / To);
    float acc = 0.f;
    for (int it = 0; it < kt; ++it) {
      const int t = to * st + it - pad_t;
      if (t < 0 || t >= T) continue;
      for (int ih = 0; ih < k; ++ih) {
        const int h = ho * sh + ih - pad;
        if (h < 0 || h >= H) continue;
        for (int iw = 0; iw < k; ++iw) {
          const int w = wo * sw + iw - pad;
          if (w < 0 || w >= W) continue;
          acc += pascal(kt, it) * pascal(k, ih) * pascal(k, iw) * s[((((long long)n * T + t) * H + h) * W + w) * G + g];
        }
      }
    }
    acc *= norm;
    const uint32_t p2 = pack_bf16x2(acc, acc);
    reinterpret_cast<uint4*>(y)[i] = make_uint4(p2, p2, p2, p2);
  }
}

// adjoint stencil + broadcast over the group: one thread per (input voxel, 8-channel vector)
__global__ void og_blur3d_bwd_kernel(const float* __restrict__ g, __nv_bfloat16* __restrict__ dx, int T, int H, int W,
                                     int To, int Ho, int Wo, int k, int st, int sh, int sw, int Cin, float norm,
                                     long long total_vec, int kt, int pad_t, int pad, int G) {
  const int cv = Cin >> 3, gv = cv / G;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total_vec;
       i += (long long)gridDim.x * blockDim.x) {
    long long v = i / cv;
    const int grp = (int)(i - v * cv) / gv;
    const int w = (int)(v % W);
    long long r = v / W;
    const int h = (int)(r % H);
    r /= H;
    const int t = (int)(r % T);
    const int n = (int)(r / T);
    float acc = 0.f;
    for (int it = 0; it < kt; ++it) {
      const int tn = t + pad_t - it;
      if (tn < 0 || tn % st || tn / st >= To) continue;
      for (int ih = 0; ih < k; ++ih) {
        const int hn = h + pad - ih;
        if (hn < 0 || hn % sh || hn / sh >= Ho) continue;
        for (int iw = 0; iw < k; ++iw) {
          const int wn = w + pad - iw;
          if (wn < 0 || wn % sw || wn / sw >= Wo) continue;
          acc += pascal(kt, it) * pascal(k, ih) * pascal(k, iw) *
                 g[((((long long)n * To + tn / st) * Ho + hn / sh) * Wo + wn / sw) * G + grp];
        }
      }
    }
    acc *= norm;
    const uint32_t p2 = pack_bf16x2(acc, acc);
    reinterpret_cast<uint4*>(dx)[i] = make_uint4(p2, p2, p2, p2);
  }
}

}  // namespace og

static int blurpool_launch(const void* x, void* y, float* scratch, int backward, int N, int T, int H, int W, int cin,
                           int cout, int kt, int k, int st, int sh, int sw, int pad_t, int pad, og_stream_t stream,
                           int G = 1) {
  using namespace og;
  OG_REQUIRE(x && y && scratch, "blurpool: null pointer");
  OG_REQUIRE(cin % 8 == 0 && cout % 8 == 0 && k >= 1 && k <= 7 && kt >= 1 && kt <= 7, "blurpool: need C %% 8 == 0 and k <= 7");
  OG_REQUIRE(pad_t >= 0 && pad >= 0 && st >= 1 && sh >= 1 && sw >= 1, "blurpool: bad stride / padding");
  OG_REQUIRE(N >= 1 && T >= 1 && H >= 1 && W >= 1, "blurpool: bad extents (N=%d T=%d H=%d W=%d)", N, T, H, W);
  // checked before the division below, which truncates towards zero and would turn a negative span into one output
  OG_REQUIRE(T + 2 * pad_t >= kt && H + 2 * pad >= k && W + 2 * pad >= k,
             "blurpool: padded input smaller than the kernel (T=%d H=%d W=%d k=%d)", T, H, W, k);
  // the stencil kernels write 8 channels of y as one 16-byte vector
  OG_REQUIRE(aligned16(y), "blurpool: y must be 16-byte aligned");
  const int To = (T + 2 * pad_t - kt) / st + 1, Ho = (H + 2 * pad - k) / sh + 1, Wo = (W + 2 * pad - k) / sw + 1;
  OG_REQUIRE(To >= 1 && Ho >= 1 && Wo >= 1, "blurpool: empty output");
  auto row_sum = [](int kk) {
    float t = 0.f;
    for (int i = 0; i < kk; ++i) {
      float v = 1.f;
      for (int j = 0; j < i; ++j) v = v * (float)(kk - 1 - j) / (float)(j + 1);
      t += v;
    }
    return t;
  };
  const float norm = 1.f / (row_sum(kt) * row_sum(k) * row_sum(k));
  cudaStream_t s = (cudaStream_t)stream;
  if (!backward) {
    // x: [N,T,H,W,cin] -> y: [N,To,Ho,Wo,cout]; scratch: N*T*H*W*G floats
    const long long rows = (long long)N * T * H * W;
    if (G == 1)
      og_channel_sum_kernel<<<ew_blocks(rows, 8), 256, 0, s>>>((const __nv_bfloat16*)x, scratch, rows, cin);
    else
      og_group_sum_kernel<<<ew_blocks(rows * G, 256), 256, 0, s>>>((const __nv_bfloat16*)x, scratch, rows * G, cin / G);
    OG_CHECK_CUDA(cudaGetLastError());
    const long long total = (long long)N * To * Ho * Wo * (cout / 8);
    og_blur3d_fwd_kernel<<<ew_blocks(total, 256), 256, 0, s>>>(scratch, (__nv_bfloat16*)y, T, H, W, To, Ho, Wo, k, st, sh,
                                                              sw, cout, norm, total, kt, pad_t, pad, G);
  } else {
    // x: dy [N,To,Ho,Wo,cout] -> y: dx [N,T,H,W,cin]; scratch: N*To*Ho*Wo*G floats
    const long long rows = (long long)N * To * Ho * Wo;
    if (G == 1)
      og_channel_sum_kernel<<<ew_blocks(rows, 8), 256, 0, s>>>((const __nv_bfloat16*)x, scratch, rows, cout);
    else
      og_group_sum_kernel<<<ew_blocks(rows * G, 256), 256, 0, s>>>((const __nv_bfloat16*)x, scratch, rows * G, cout / G);
    OG_CHECK_CUDA(cudaGetLastError());
    const long long total = (long long)N * T * H * W * (cin / 8);
    og_blur3d_bwd_kernel<<<ew_blocks(total, 256), 256, 0, s>>>(scratch, (__nv_bfloat16*)y, T, H, W, To, Ho, Wo, k, st, sh,
                                                              sw, cin, norm, total, kt, pad_t, pad, G);
  }
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(2);
  return OG_OK;
}

extern "C" int og_blurpool3d(const void* x, void* y, float* scratch, int backward, int N, int T, int H, int W, int cin,
                             int cout, int k, int st, int sh, int sw, og_stream_t stream) {
  OG_REQUIRE((k & 1) == 1, "blurpool3d: odd kernel sizes only (k=%d)", k);
  return blurpool_launch(x, y, scratch, backward, N, T, H, W, cin, cout, k, k, st, sh, sw, (k - 1) / 2, (k - 1) / 2, stream);
}

extern "C" int og_blurpool3d_grouped(const void* x, void* y, float* scratch, int backward, int N, int T, int H, int W,
                                     int cin, int cout, int groups, int k, int st, int sh, int sw, og_stream_t stream) {
  using namespace og;
  OG_REQUIRE((k & 1) == 1, "blurpool3d_grouped: odd kernel sizes only (k=%d)", k);
  OG_REQUIRE(groups >= 1 && cin % groups == 0 && cout % groups == 0,
             "blurpool3d_grouped: groups=%d must divide cin=%d and cout=%d", groups, cin, cout);
  OG_REQUIRE((cin / groups) % 8 == 0 && (cout / groups) % 8 == 0,
             "blurpool3d_grouped: need (cin/groups) %% 8 == 0 and (cout/groups) %% 8 == 0 (cin=%d cout=%d groups=%d)",
             cin, cout, groups);
  OG_REQUIRE(x && y && scratch, "blurpool3d_grouped: null pointer");
  // the group sums read x in 16-byte vectors
  OG_REQUIRE(aligned16(x), "blurpool3d_grouped: x must be 16-byte aligned");
  OG_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 3) == 0, "blurpool3d_grouped: scratch must be 4-byte aligned");
  return blurpool_launch(x, y, scratch, backward, N, T, H, W, cin, cout, k, k, st, sh, sw, (k - 1) / 2, (k - 1) / 2,
                         stream, groups);
}

extern "C" int og_blurpool2d(const void* x, void* y, float* scratch, int backward, int N, int H, int W, int cin, int cout,
                             int k, int sh, int sw, int pad, og_stream_t stream) {
  return blurpool_launch(x, y, scratch, backward, N, 1, H, W, cin, cout, 1, k, 1, sh, sw, 0, pad, stream);
}


// ------------------------------------------------------------------------------------------------
// data path: decoded video frames -> model input
// ------------------------------------------------------------------------------------------------
namespace og {

// frames: uint8 [N][T][H][W][3] exactly as OpenCV's VideoCapture.read() hands them over (BGR unless bgr == 0).
// One thread per (n, t, h, w) pixel: the colour swap of cv2.cvtColor(BGR2RGB), the `/ 255.` and the
// 't h w c -> c t h w' rearrange of Platformer2D.load_video_slice (genie/module/data.py:196-234) in one pass.
//   out_kind 0: NCDHW fp32 (the reference's tensor format at every public method)
//   out_kind 1: NDHWC bf16, channel pitch cpad >= 3, zero padded (the internal activation format)
__global__ void og_frames_u8_to_video_kernel(const unsigned char* __restrict__ frames, int bgr, void* __restrict__ out,
                                             int out_kind, int cpad, long long V, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const unsigned char* px = frames + i * 3;
    // IEEE division, not a multiply by the reciprocal: bit-identical to the reference's `torch.stack(frames) / 255.`
    const float c0 = __fdiv_rn((float)px[bgr ? 2 : 0], 255.f);
    const float c1 = __fdiv_rn((float)px[1], 255.f);
    const float c2 = __fdiv_rn((float)px[bgr ? 0 : 2], 255.f);
    if (out_kind == 0) {
      const long long n = i / V, v = i - n * V;
      float* o = reinterpret_cast<float*>(out) + n * 3 * V + v;
      o[0] = c0;
      o[V] = c1;
      o[2 * V] = c2;
    } else {
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out) + i * cpad;
      o[0] = __float2bfloat16_rn(c0);
      o[1] = __float2bfloat16_rn(c1);
      o[2] = __float2bfloat16_rn(c2);
      for (int c = 3; c < cpad; ++c) o[c] = __float2bfloat16_rn(0.f);
    }
  }
}

}  // namespace og

extern "C" int og_frames_u8_to_video(const uint8_t* frames, int bgr, void* out, int out_kind, int cpad, int N, int T, int H,
                                     int W, og_stream_t stream) {
  using namespace og;
  OG_REQUIRE(frames && out, "frames_u8_to_video: null pointer");
  OG_REQUIRE(N > 0 && T > 0 && H > 0 && W > 0, "frames_u8_to_video: empty video");
  OG_REQUIRE(out_kind == 0 || (out_kind == 1 && cpad >= 3), "frames_u8_to_video: bad output format");
  const long long V = (long long)T * H * W, total = (long long)N * V;
  og_frames_u8_to_video_kernel<<<ew_blocks(total, 256), 256, 0, (cudaStream_t)stream>>>(frames, bgr, out, out_kind, cpad, V,
                                                                                       total);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

// ------------------------------------------------------------------------------------------------
// perceptual loss helpers (genie/module/loss.py:34-107): VGG16 feature extractor pieces that are not conv / ReLU
// ------------------------------------------------------------------------------------------------
namespace og {

// nn.MaxPool2d(kernel_size=2, stride=2) on NHWC bf16 (torchvision vgg16.features.{4,9,16,23}); H, W even or floor.
__global__ void og_maxpool2x2_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int H, int W, int Ho, int Wo, int cv,
                                     long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv);
    long long r = i / cv;
    const int wo = (int)(r % Wo);
    r /= Wo;
    const int ho = (int)(r % Ho);
    const long long n = r / Ho;
    const long long base = ((n * H + 2 * ho) * W + 2 * wo) * cv + c;
    const uint4 q[4] = {__ldg(x + base), __ldg(x + base + cv), __ldg(x + base + (long long)W * cv),
                        __ldg(x + base + (long long)W * cv + cv)};
    uint4 o;
    __nv_bfloat162* oh = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      __nv_bfloat162 m = reinterpret_cast<const __nv_bfloat162*>(&q[0])[e];
#pragma unroll
      // NaN-propagating, as nn.MaxPool2d: a NaN feature must reach the loss
      for (int k = 1; k < 4; ++k) m = __hmax2_nan(m, reinterpret_cast<const __nv_bfloat162*>(&q[k])[e]);
      oh[e] = m;
    }
    y[i] = o;
  }
}

// out[0] += sum (a - b)^2 over n bf16 elements (n % 8 == 0): the feature-space mse of the perceptual loss
__global__ void og_sqdiff_sum_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, long long nvec,
                                     float* __restrict__ out) {
  float acc = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const uint4 ua = __ldg(a + i), ub = __ldg(b + i);
    const __nv_bfloat162* ha = reinterpret_cast<const __nv_bfloat162*>(&ua);
    const __nv_bfloat162* hb = reinterpret_cast<const __nv_bfloat162*>(&ub);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 fa = __bfloat1622float2(ha[e]), fb = __bfloat1622float2(hb[e]);
      const float d0 = fa.x - fb.x, d1 = fa.y - fb.y;
      acc = fmaf(d0, d0, fmaf(d1, d1, acc));
    }
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(out, acc);
}

}  // namespace og

extern "C" int og_maxpool2x2(const void* x, void* y, int N, int H, int W, int C, og_stream_t stream) {
  using namespace og;
  OG_REQUIRE(x && y && N > 0 && H >= 2 && W >= 2, "maxpool2x2: bad arguments");
  OG_REQUIRE(C % 8 == 0, "maxpool2x2: C=%d must be a multiple of 8", C);
  OG_REQUIRE(aligned16(x) && aligned16(y), "maxpool2x2: x and y must be 16-byte aligned");
  const int Ho = H / 2, Wo = W / 2;
  const long long total = (long long)N * Ho * Wo * (C / 8);
  og_maxpool2x2_kernel<<<ew_blocks(total, 256), 256, 0, (cudaStream_t)stream>>>((const uint4*)x, (uint4*)y, H, W, Ho, Wo, C / 8,
                                                                               total);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_sqdiff_sum(const void* a, const void* b, int64_t n, float* out, og_stream_t stream) {
  using namespace og;
  OG_REQUIRE(a && b && out && n > 0 && n % 8 == 0, "sqdiff_sum: bad arguments (n %% 8 == 0)");
  OG_REQUIRE(aligned16(a) && aligned16(b), "sqdiff_sum: a and b must be 16-byte aligned");
  og_sqdiff_sum_kernel<<<ew_blocks(n / 8, 256), 256, 0, (cudaStream_t)stream>>>((const uint4*)a, (const uint4*)b, n / 8, out);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}
