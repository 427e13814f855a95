// og_host.cu — error reporting, TMA descriptor encoding, device queries, ABI housekeeping.
#include <stdarg.h>

#include <atomic>

#include "og_host.cuh"

namespace og {

static thread_local char g_err[512] = {0};
std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
  });
  return fn;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, const uint32_t* elem_strides, CUtensorMapSwizzle swizzle) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled is unavailable (no CUDA driver / GPU?)");
    return OG_ERR_CUDA;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = elem_strides ? elem_strides[i] : 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d): rank %d dims [%llu %llu %llu %llu %llu] box [%u %u %u %u %u]",
              (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
              (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
              (unsigned long long)(rank > 4 ? dims[4] : 0), box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0,
              rank > 3 ? box[3] : 0, rank > 4 ? box[4] : 0);
    return OG_ERR_CUDA;
  }
  return OG_OK;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

// One block per 32 consecutive outputs of one group: warp w adds the partials b = w, w + 8, ... in order, then the eight
// warp sums are added in warp order — a fixed summation tree, so the result does not depend on scheduling.
__global__ void __launch_bounds__(256)
    og_sum_partials_kernel(const float* __restrict__ partials, int nparts, long long width, long long row_len,
                           long long out_ld, float* __restrict__ out) {
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long i = (long long)blockIdx.x * 32 + lane;
  const long long g = blockIdx.y;
  float a = 0.f;
  if (i < width)
    for (int b = w; b < nparts; b += 8) a += __ldcg(partials + (g * nparts + b) * width + i);
  red[w][lane] = a;
  __syncthreads();
  if (w == 0 && i < width) {
    float t = red[0][lane];
    for (int k = 1; k < 8; ++k) t += red[k][lane];
    const long long o = g * width + i;
    out[o / row_len * out_ld + o % row_len] += t;
  }
}

int sum_partials(const float* partials, int groups, int nparts, long long width, long long row_len, long long out_ld,
                 float* out, cudaStream_t stream) {
  OG_REQUIRE(groups >= 1 && groups <= 65535 && nparts >= 1 && width >= 1 && row_len >= 1 && out_ld >= row_len,
             "sum_partials: bad shape");
  const long long bx = (width + 31) / 32;
  OG_REQUIRE(bx < (1LL << 31), "sum_partials: too wide");
  og_sum_partials_kernel<<<dim3((unsigned)bx, (unsigned)groups), 256, 0, stream>>>(partials, nparts, width, row_len, out_ld,
                                                                                   out);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

static int pow2_ceil(int v) {
  int p = 1;
  while (p < v) p *= 2;
  return p;
}

void choose_voxel_box(int vox, int N, int T, int H, int W, int* bw, int* bh, int* bt, int* bn) {
  int rem = vox;
  int w = pow2_ceil(W) < rem ? pow2_ceil(W) : rem;
  rem /= w;
  int h = pow2_ceil(H) < rem ? pow2_ceil(H) : rem;
  rem /= h;
  int t = pow2_ceil(T) < rem ? pow2_ceil(T) : rem;
  rem /= t;
  int n = rem;  // whatever is left spans samples
  if (n > 256) n = 256;
  *bw = w;
  *bh = h;
  *bt = t;
  *bn = n;
  (void)N;
}

}  // namespace og

extern "C" {
const char* og_last_error(void) { return og::g_err; }
int og_abi_version(void) { return 2; }
int og_compiled_sm(void) { return 90; }
uint64_t og_launch_count(void) { return og::g_launches.load(); }
}
