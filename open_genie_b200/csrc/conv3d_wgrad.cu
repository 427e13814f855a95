// conv3d_wgrad.cu — weight gradient of the stride-1 3-D convolution on the Hopper tensor cores (wgmma).
//
//   dW[co][tap][ci] += sum_v dY[v][co] * X[v + tap - pad][ci]          (v = voxel (n,t,h,w))
//
// As a GEMM the reduction dimension is the voxel index, and both operands are stored with the
// NON-reduced dimension contiguous (channels-last), i.e. both are "MN-major" wgmma operands:
//   A tile = dY box  : [co/64 panel][64 voxel rows][64 co]   (TMA 5-D box, 128-byte swizzle)
//   B tile = X  box  : [ci/64 panel][64 voxel rows][64 ci]   (same box shifted by the tap; OOB -> 0)
// so no transposed copy of activations or gradients is ever made. A CTA owns 128 output channels x 128 accumulator
// columns (one tap of a 128-wide Cin tile, or two taps of a 64-wide one), held in the registers of its MMA warpgroup;
// the dY tile of a k-step is loaded once and reused by every tap of the group. The voxel range is split across CTAs
// (split-K); each split stores its partial tile into its own slab of the caller's workspace and a fixed-order pass adds the
// slabs into dW (reproducible: no atomics across CTAs). Unsplit launches add straight into dW, which the caller zeroes.
// Optional fused bias gradient (og_conv3d_wgrad_bias): db[co] = sum_v dY[v][co] is the same GEMM against a column of
// ones — the CTAs of the LAST tap group issue one extra N = 16 MMA per k-step against a constant all-ones tile in shared
// memory (a tile of ones is invariant under the 128-byte swizzle, so any valid descriptor reads it correctly).
//
// Replaces autograd's conv3d weight-gradient reached from genie/module/video.py:192,609-629,599-603 and
// genie/module/attention.py:429-438 during loss.backward().
#include <stdlib.h>

#include "og_host.cuh"
#include "og_ptx.cuh"

namespace og {
extern std::atomic<uint64_t> g_launches;

struct WgradParams {
  int kt, kh, kw, pt, ph, pw;
  int ntaps, taps_per_group, num_groups, splitk;
  int block_n;  // ci tile (64 or 128)
  int bw_log2, bh_log2, bt_log2, bn_log2;
  int tiles_w, tiles_h, tiles_t;
  int num_ksteps;  // 64-voxel boxes in the whole tensor
  int cin, cout;
  float* dw;
  long long ld_dw;
  int a_stages, b_stages;
  int sx_t, sx_h, sx_w;  // X box start = dY box start * stride + tap offset (strided convolution; 1 otherwise)
  int vec_ok;  // dw rows 8-byte aligned: vector reductions
  float* dbias;     // optional: += column sums of dY for output channels < n_bias (the convolution's bias gradient)
  int n_bias;
  float* slabs;     // split-K > 1: [splitk][cout][ntaps * cin] partial dW, then [splitk][n_bias] partial db (workspace)
  int plain_store;  // OG_WGRAD_PLAIN_STORE=1: the ABI says "accumulates", so overwriting is opt-in (the Python side zeroes dw anyway)
};

static constexpr int kWThreads = 256;
static constexpr int kVox = 64;                 // voxels (K rows) per k-step
static constexpr int kPanelBytes = kVox * 128;  // one 64-channel panel of a box: 8 KiB
static constexpr int kWABytes = 2 * kPanelBytes;  // 128 output channels
static constexpr int kWBBytes = 2 * kPanelBytes;  // 128 accumulator columns
static constexpr int kWMaxStages = 12;

// Warp roles: warp 0 TMA producer, warps 1-3 idle (wgmma needs an aligned warpgroup), warps 4-7 the MMA warpgroup,
// which also runs the epilogue (accumulator fragments -> dW, or this split's slab of the workspace).
__global__ void __launch_bounds__(kWThreads, 1)
    og_conv_wgrad_kernel(const __grid_constant__ CUtensorMap mapDY, const __grid_constant__ CUtensorMap mapX,
                         const WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // One B stage holds the 128 accumulator columns of a k-step: a tap of a 128-wide Cin tile, or a PAIR of taps of a
  // 64-wide one back to back ([tap j panel][tap j+1 panel]). It is issued as a single wgmma of N = 128 whose
  // accumulator columns are the taps' blocks (columns of a missing second tap are computed from stale data and dropped).
  const int tap_bytes = (p.block_n / 64) * kPanelBytes;
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + p.a_stages * kWABytes;
  uint8_t* smem_ones = smem_b + p.b_stages * kWBBytes;   // 16 k-rows x 128 B of bf16 1.0 (bias-gradient operand), 1024-aligned
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_ones + 2048);
  uint64_t* full_a = bars;
  uint64_t* empty_a = bars + kWMaxStages;
  uint64_t* full_b = bars + 2 * kWMaxStages;
  uint64_t* empty_b = bars + 3 * kWMaxStages;

  const int warp = warp_idx_uniform();
  const int lane = threadIdx.x & 31;
  const int co0 = blockIdx.x * 128;
  const int ci0 = blockIdx.y * p.block_n;
  // tap group is the FAST index: the CTAs that stream the same voxel range (same split, different taps)
  // are co-scheduled, so dY / X tiles are fetched from DRAM once and hit in L2 for the other groups
  const int split = blockIdx.z / p.num_groups;
  const int group = blockIdx.z - split * p.num_groups;
  const int tap0 = group * p.taps_per_group;
  const int ntap = min(p.taps_per_group, p.ntaps - tap0);
  const bool do_bias = p.dbias != nullptr && blockIdx.y == 0 && group == p.num_groups - 1;
  // contiguous k-step range of this split
  const int ks_begin = (int)(((long long)p.num_ksteps * split) / p.splitk);
  const int ks_end = (int)(((long long)p.num_ksteps * (split + 1)) / p.splitk);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&mapDY);
    tma_prefetch_desc(&mapX);
    for (int s = 0; s < p.a_stages; ++s) {
      mbar_init(&full_a[s], 1);
      mbar_init(&empty_a[s], 4);
    }
    for (int s = 0; s < p.b_stages; ++s) {
      mbar_init(&full_b[s], 1);
      mbar_init(&empty_b[s], 4);
    }
    fence_mbar_init();
  }
  if (do_bias) {
    for (int i = threadIdx.x; i < 2048 / 4; i += kWThreads) reinterpret_cast<uint32_t*>(smem_ones)[i] = 0x3F803F80u;
    fence_proxy_async_smem();   // generic-proxy writes -> visible to the tensor core's async-proxy reads
  }
  __syncthreads();

  if (warp == 0) {
    {
      // whole warp runs the loop converged; one elected lane issues (see elect_one() in og_ptx.cuh)
      int sa = 0, sb = 0;
      uint32_t pha = 0, phb = 0;
      // The producer is ONE thread: keep its per-k-step instruction count tiny (no divisions in the loop).
      // tap offsets of this group, decoded once
      int off_w[2], off_h[2], off_t[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int tap = tap0 + (j < ntap ? j : 0);
        off_t[j] = tap / (p.kh * p.kw) - p.pt;
        off_h[j] = (tap / p.kw) % p.kh - p.ph;
        off_w[j] = tap % p.kw - p.pw;
      }
      // box coordinates of the first k-step, then advanced incrementally with carries
      const int per_sample = p.tiles_w * p.tiles_h * p.tiles_t;
      int tn = ks_begin / per_sample;
      int r = ks_begin - tn * per_sample;
      int tw = r % p.tiles_w;
      r /= p.tiles_w;
      int th = r % p.tiles_h;
      int tt = r / p.tiles_h;
      const int panels = p.block_n / 64;
      for (int ks = ks_begin; ks < ks_end; ++ks) {
        const int n = tn << p.bn_log2, w0 = tw << p.bw_log2, h0 = th << p.bh_log2, t0 = tt << p.bt_log2;
        mbar_wait(&empty_a[sa], pha ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full_a[sa], kWABytes);
          tma_load_5d(smem_a + sa * kWABytes, &mapDY, &full_a[sa], co0, w0, h0, t0, n);
          tma_load_5d(smem_a + sa * kWABytes + kPanelBytes, &mapDY, &full_a[sa], co0 + 64, w0, h0, t0, n);
        }
        __syncwarp();
        if (++sa == p.a_stages) {
          sa = 0;
          pha ^= 1;
        }
        mbar_wait(&empty_b[sb], phb ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full_b[sb], (uint32_t)(ntap * tap_bytes));
          uint8_t* dst = smem_b + sb * kWBBytes;
          for (int u = 0; u < ntap; ++u)
            for (int pp = 0; pp < panels; ++pp)
              tma_load_5d(dst + u * tap_bytes + pp * kPanelBytes, &mapX, &full_b[sb], ci0 + pp * 64,
                          w0 * p.sx_w + off_w[u], h0 * p.sx_h + off_h[u], t0 * p.sx_t + off_t[u], n);
        }
        __syncwarp();
        if (++sb == p.b_stages) {
          sb = 0;
          phb ^= 1;
        }
        if (++tw == p.tiles_w) {
          tw = 0;
          if (++th == p.tiles_h) {
            th = 0;
            if (++tt == p.tiles_t) {
              tt = 0;
              ++tn;
            }
          }
        }
      }
    }
    __syncwarp();
  } else if (warp >= 4) {
    const int q = warp & 3;
    float acc[2][64], accb[2][8];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[hh][i] = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) accb[hh][i] = 0.f;
    }
    const uint32_t ones_addr = smem_u32(smem_ones);
    int sa = 0, sb = 0, prev_a = -1, prev_b = -1;
    uint32_t pha = 0, phb = 0;
    for (int ks = ks_begin; ks < ks_end; ++ks) {
      mbar_wait(&full_a[sa], pha);
      mbar_wait(&full_b[sb], phb);
      const uint32_t a_addr = smem_u32(smem_a + sa * kWABytes);
      const uint32_t b_addr = smem_u32(smem_b + sb * kWBBytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kVox / 16; ++k) {
        // MN-major panels [panel][64 k-rows][128 B]: 16 k-rows = 2048 B, panel stride = 8192 B
        const uint64_t bdesc = gmma_desc_sw128(b_addr + k * 2048, kPanelBytes, 1024);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const uint64_t adesc = gmma_desc_sw128(a_addr + hh * kPanelBytes + k * 2048, kPanelBytes, 1024);
          wgmma_ss<128, 1, 1>(acc[hh], adesc, bdesc, 1);
          if (do_bias)   // db += dY^T . 1  (N = 16 columns of ones; every column holds the same sum)
            wgmma_ss<16, 1, 1>(accb[hh], adesc, gmma_desc_sw128(ones_addr, kPanelBytes, 1024), 1);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();   // the previous k-step's MMAs are done: its stages go back to the producer
      if (prev_a >= 0 && lane == 0) {
        mbar_arrive(&empty_a[prev_a]);
        mbar_arrive(&empty_b[prev_b]);
      }
      prev_a = sa;
      prev_b = sb;
      if (++sa == p.a_stages) {
        sa = 0;
        pha ^= 1;
      }
      if (++sb == p.b_stages) {
        sb = 0;
        phb ^= 1;
      }
    }
    wgmma_wait<0>();
    reg_fence(acc[0]);
    reg_fence(acc[1]);
    reg_fence(accb[0]);
    reg_fence(accb[1]);
    // epilogue straight from the fragments: row = output channel, column c = (tap c / block_n, ci c % block_n)
    const int c_lane = 2 * (lane & 3);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int co = co0 + hh * 64 + q * 16 + (lane >> 2) + rr * 8;
        if (co >= p.cout) continue;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = j * 8 + c_lane;
          const int tj = c / p.block_n, ci = ci0 + c - tj * p.block_n;
          if (tj >= ntap || ci >= p.cin) continue;
          float* dst = p.dw + (long long)co * p.ld_dw + (long long)(tap0 + tj) * p.cin + ci;
          const float v0 = acc[hh][4 * j + 2 * rr], v1 = acc[hh][4 * j + 2 * rr + 1];
          if (p.slabs) {   // this split's own slab: plain stores, every element of the tile is written
            float* sl = p.slabs + (long long)split * p.cout * p.ntaps * p.cin + ((long long)co * p.ntaps + tap0 + tj) * p.cin + ci;
            sl[0] = v0;
            if (ci + 1 < p.cin) sl[1] = v1;
          } else if (p.vec_ok && p.plain_store) {
            // one CTA owns this (co, tap, ci) block and the caller's buffer is freshly zeroed: plain stores
            *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
          } else if (p.vec_ok) {
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(v0), "f"(v1) : "memory");
          } else {
            atomicAdd(dst, v0);
            if (ci + 1 < p.cin) atomicAdd(dst + 1, v1);
          }
        }
        if (do_bias && (lane & 3) == 0 && co < p.n_bias) {
          if (p.slabs)
            p.slabs[(long long)p.splitk * p.cout * p.ntaps * p.cin + (long long)split * p.n_bias + co] = accb[hh][2 * rr];
          else
            p.dbias[co] += accb[hh][2 * rr];   // one CTA per channel when unsplit
        }
      }
    }
  }
}

}  // namespace og

// N,T,H,W: the dY grid (= output voxels). Ti,Hi,Wi / st,sh,sw: extents of x and the convolution strides.
static int launch_wgrad(const void* dy, int cout, const void* x, int cin, float* dw, int64_t ld_dw, int kt, int kh, int kw,
                        int pt, int ph, int pw, int N, int T, int H, int W, int Ti, int Hi, int Wi, int st, int sh, int sw,
                        void* workspace, size_t workspace_bytes, og_stream_t stream, float* dbias = nullptr,
                        int n_bias = 0) {
  using namespace og;
  OG_REQUIRE(dy && x && dw, "conv3d_wgrad: null pointer");
  OG_REQUIRE(!dbias || (n_bias > 0 && n_bias <= cout), "conv3d_wgrad: n_bias=%d must be in 1..cout", n_bias);
  OG_REQUIRE(cin > 0 && cin % 64 == 0, "conv3d_wgrad: cin=%d must be a multiple of 64", cin);
  OG_REQUIRE(cout > 0 && cout % 8 == 0, "conv3d_wgrad: cout=%d must be a multiple of 8 (TMA row stride)", cout);
  OG_REQUIRE(kt >= 1 && kh >= 1 && kw >= 1 && pt >= 0 && ph >= 0 && pw >= 0 && pt < kt && ph < kh && pw < kw,
             "conv3d_wgrad: bad kernel/padding");
  OG_REQUIRE(st >= 1 && sh >= 1 && sw >= 1 && st <= 8 && sh <= 8 && sw <= 8, "conv3d_wgrad: bad stride");
  int bw, bh, bt, bn;
  choose_voxel_box(kVox, N, T, H, W, &bw, &bh, &bt, &bn);
  WgradParams p;
  memset(&p, 0, sizeof(p));
  p.kt = kt; p.kh = kh; p.kw = kw; p.pt = pt; p.ph = ph; p.pw = pw;
  p.sx_t = st; p.sx_h = sh; p.sx_w = sw;
  p.ntaps = kt * kh * kw;
  p.block_n = (cin % 128 == 0) ? 128 : 64;
  p.taps_per_group = 128 / p.block_n;   // 128 accumulator columns per CTA
  if (p.taps_per_group > p.ntaps) p.taps_per_group = p.ntaps;
  p.num_groups = (p.ntaps + p.taps_per_group - 1) / p.taps_per_group;
  p.bw_log2 = ilog2(bw); p.bh_log2 = ilog2(bh); p.bt_log2 = ilog2(bt); p.bn_log2 = ilog2(bn);
  p.tiles_w = (W + bw - 1) / bw; p.tiles_h = (H + bh - 1) / bh; p.tiles_t = (T + bt - 1) / bt;
  p.num_ksteps = ((N + bn - 1) / bn) * p.tiles_w * p.tiles_h * p.tiles_t;
  p.cin = cin; p.cout = cout; p.dw = dw; p.ld_dw = ld_dw;
  const int co_tiles = (cout + 127) / 128;
  const int ci_tiles = cin / p.block_n;
  const int base_ctas = co_tiles * ci_tiles * p.num_groups;
  // split-K factor: fill whole waves (a partial last wave costs a full CTA duration), keep >= 4 k-steps per
  // CTA so pipeline fill and the epilogue reductions stay amortised, at most ~3 waves.
  const int sms = num_sms();
  int max_split = p.num_ksteps / 4;
  // split-K needs one dW (+ db) slab per split in the workspace
  const long long slab_floats = (long long)cout * p.ntaps * cin + (dbias ? n_bias : 0);
  const long long fit = workspace ? (long long)(workspace_bytes / sizeof(float)) / slab_floats : 0;
  if (max_split > fit) max_split = (int)fit;
  if (max_split < 1) max_split = 1;
  if (max_split > 128) max_split = 128;
  int splitk = 1;
  double best = -1.0;
  for (int s = 1; s <= max_split; ++s) {
    const long long total = (long long)base_ctas * s;
    const long long waves = (total + sms - 1) / sms;
    if (waves > 3 && s > 1) break;
    const double eff = (double)total / (double)(waves * sms);
    // prefer higher wave efficiency; among equals prefer fewer splits (fewer reductions)
    if (eff > best + 1e-9) {
      best = eff;
      splitk = s;
    }
  }
  p.splitk = splitk;
  p.slabs = splitk > 1 ? reinterpret_cast<float*>(workspace) : nullptr;
  {
    const char* ps = getenv("OG_WGRAD_PLAIN_STORE");
    p.plain_store = ps ? atoi(ps) : 0;
  }
  p.vec_ok = (ld_dw % 2 == 0) && (cin % 2 == 0) && ((reinterpret_cast<uintptr_t>(dw) & 7) == 0);
  p.dbias = dbias;
  p.n_bias = n_bias;
  // one A and one B stage per k-step (16 + 16 KiB)
  p.a_stages = p.b_stages = 6;
  const size_t smem_bytes = (size_t)p.a_stages * kWABytes + (size_t)p.b_stages * kWBBytes + 2048 /*ones*/ + 1024 + 512;

  CUtensorMap mapDY, mapX;
  {
    uint64_t dims[5] = {(uint64_t)cout, (uint64_t)W, (uint64_t)H, (uint64_t)T, (uint64_t)N};
    uint64_t str[4] = {(uint64_t)cout * 2, (uint64_t)W * cout * 2, (uint64_t)H * W * cout * 2,
                       (uint64_t)T * H * W * cout * 2};
    uint32_t box[5] = {64, (uint32_t)bw, (uint32_t)bh, (uint32_t)bt, (uint32_t)bn};
    int r = make_tmap_bf16(&mapDY, dy, 5, dims, str, box);
    if (r != OG_OK) return r;
  }
  {
    // strided convolution: the x box spans bw*sw positions traversed with element stride sw (see conv3d_igemm.cu)
    uint64_t dims[5] = {(uint64_t)cin, (uint64_t)Wi, (uint64_t)Hi, (uint64_t)Ti, (uint64_t)N};
    uint64_t str[4] = {(uint64_t)cin * 2, (uint64_t)Wi * cin * 2, (uint64_t)Hi * Wi * cin * 2,
                       (uint64_t)Ti * Hi * Wi * cin * 2};
    uint32_t box[5] = {64, (uint32_t)(bw * sw), (uint32_t)(bh * sh), (uint32_t)(bt * st), (uint32_t)bn};
    uint32_t es[5] = {1, (uint32_t)sw, (uint32_t)sh, (uint32_t)st, 1};
    OG_REQUIRE(box[1] <= 256 && box[2] <= 256 && box[3] <= 256, "conv3d_wgrad: strided box exceeds the TMA limit");
    int r = make_tmap_bf16(&mapX, x, 5, dims, str, box, es);
    if (r != OG_OK) return r;
  }
  static bool attr_set = false;
  if (!attr_set) {
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_conv_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  dim3 grid(co_tiles, ci_tiles, p.num_groups * p.splitk);  // z = split * num_groups + group
  og_conv_wgrad_kernel<<<grid, kWThreads, smem_bytes, (cudaStream_t)stream>>>(mapDY, mapX, p);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  if (p.slabs) {   // add the split slabs in split order
    const long long row = (long long)p.ntaps * cin, w = (long long)cout * row;
    int rc = sum_partials(p.slabs, 1, splitk, w, row, ld_dw, dw, (cudaStream_t)stream);
    if (rc == OG_OK && p.dbias)
      rc = sum_partials(p.slabs + (long long)splitk * w, 1, splitk, n_bias, n_bias, n_bias, p.dbias, (cudaStream_t)stream);
    if (rc != OG_OK) return rc;
  }
  return OG_OK;
}

extern "C" int og_conv3d_wgrad(const void* dy, int cout, const void* x, int cin, float* dw, int64_t ld_dw, int kt,
                               int kh, int kw, int pt, int ph, int pw, int N, int T, int H, int W, void* workspace,
                               size_t workspace_bytes, og_stream_t stream) {
  return launch_wgrad(dy, cout, x, cin, dw, ld_dw, kt, kh, kw, pt, ph, pw, N, T, H, W, T, H, W, 1, 1, 1, workspace,
                      workspace_bytes, stream);
}

// Weight gradient + bias gradient in one launch: dbias[c] += sum over voxels of dy[v][c] for c < n_bias (the bias
// gradient of the same nn.Conv3d); see the file header.
extern "C" int og_conv3d_wgrad_bias(const void* dy, int cout, const void* x, int cin, float* dw, int64_t ld_dw, int kt,
                                    int kh, int kw, int pt, int ph, int pw, int N, int T, int H, int W, float* dbias,
                                    int n_bias, void* workspace, size_t workspace_bytes, og_stream_t stream) {
  if (!dbias) {
    og::set_error("conv3d_wgrad_bias: dbias is NULL");
    return OG_ERR_INVALID_ARGUMENT;
  }
  return launch_wgrad(dy, cout, x, cin, dw, ld_dw, kt, kh, kw, pt, ph, pw, N, T, H, W, T, H, W, 1, 1, 1, workspace,
                      workspace_bytes, stream, dbias, n_bias);
}

// Weight gradient of the strided CausalConv3d (SpaceTimeDownsample): dy on the OUTPUT grid, x on the input grid
// [N,T,H,W,cin]; x boxes are strided TMA boxes. Geometry as og_conv3d_strided_fwd.
extern "C" int og_conv3d_strided_wgrad(const void* dy, int cout, const void* x, int cin, float* dw, int64_t ld_dw, int kt,
                                       int kh, int kw, int st, int sh, int sw, int pt, int ph, int pw, int N, int T, int H,
                                       int W, void* workspace, size_t workspace_bytes, og_stream_t stream) {
  const int To = (T + pt - kt) / st + 1, Ho = (H + 2 * ph - kh) / sh + 1, Wo = (W + 2 * pw - kw) / sw + 1;
  if (To < 1 || Ho < 1 || Wo < 1) {
    og::set_error("conv3d_strided_wgrad: empty output");
    return OG_ERR_INVALID_ARGUMENT;
  }
  return launch_wgrad(dy, cout, x, cin, dw, ld_dw, kt, kh, kw, pt, ph, pw, N, To, Ho, Wo, T, H, W, st, sh, sw, workspace,
                      workspace_bytes, stream);
}
