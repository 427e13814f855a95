// conv3d_wgrad.cu — weight gradient of the 3-D convolution on the Hopper tensor cores (wgmma).
//
//   dW[co][tap][ci] += sum_v dY[v][co] * X[v * stride + tap - pad][ci]          (v = voxel (n,t,h,w))
//
// As a GEMM the reduction dimension is the voxel index, and both operands are stored with the
// NON-reduced dimension contiguous (channels-last), i.e. both are "MN-major" wgmma operands:
//   A tile = dY box  : [co/64 panel][64 voxel rows][64 co]   (TMA 5-D box, 128-byte swizzle)
//   B tile = X  box  : [64-column panel][64 voxel rows][64 ci]   (the box shifted by the panel's tap; OOB -> 0)
// so no transposed copy of activations or gradients is ever made. The accumulator columns are the flattened (tap, ci)
// index of dW's [co][tap][ci] rows. A CTA tile is 128 output channels x 256 columns = four 64-column panels, each ONE
// TMA box of X shifted by its own tap (cin is a multiple of 64, so no panel straddles two taps). Two MMA warpgroups
// each own 64 output channels x all 256 columns (m64n256k16, 128 fp32 accumulators per thread), so the dY box of a
// k-step is loaded once for 256 columns.
//
// Work division (stream-K): the (tile, k-step) space, tile-major, is cut into equal contiguous shares, one per CTA of a
// persistent grid, so every SM gets the same number of k-steps whatever the tile count. A tile that lies inside one
// share is added straight into dW by its only owner. A tile cut by share boundaries has each of its segments stored in
// a workspace slot of the CTA that computed it (a share has at most two such segments: its first and its last), and a
// fixup pass adds the segments of each cut tile into dW in k order. No CTA waits on another and no sum depends on
// scheduling, so the result is bit-identical from run to run for a given SM count.
//
// Bias gradient (og_conv3d_wgrad_bias, the kBias instantiation): db[co] = sum_v dY[v][co] is the same GEMM against a
// column of ones. The tiles whose columns start at 0 issue four extra N = 16 MMAs per k-step against a constant all-ones
// tile in shared memory (a tile of ones is invariant under the 128-byte swizzle, so any valid descriptor reads it
// correctly). It is a compile-time variant so that the plain kernel issues nothing but the main MMAs: a runtime branch
// among them makes ptxas fence every wgmma with its own warpgroup.arrive.
//
// Replaces autograd's conv3d weight-gradient reached from genie/module/video.py:192,609-629,599-603 and
// genie/module/attention.py:429-438 during loss.backward().
#include "og_host.cuh"
#include "og_ptx.cuh"

namespace og {
extern std::atomic<uint64_t> g_launches;

static constexpr int kWThreads = 384;
static constexpr int kVox = 64;                   // voxels (K rows) per k-step
static constexpr int kPanelBytes = kVox * 128;    // one 64-channel panel of a box: 8 KiB
static constexpr int kTileM = 128;                // output channels per tile
static constexpr int kTileN = 256;                // accumulator columns per tile
static constexpr int kWABytes = 2 * kPanelBytes;  // dY: 128 output channels
static constexpr int kWBBytes = 4 * kPanelBytes;  // X: 256 accumulator columns
static constexpr int kWStages = 4;
static constexpr int kSlotFloats = kTileM * kTileN;

struct WgradParams {
  int kt, kh, kw, pt, ph, pw;
  int sx_t, sx_h, sx_w;  // X box start = dY box start * stride + tap offset (strided convolution; 1 otherwise)
  int bw_log2, bh_log2, bt_log2, bn_log2;
  int tiles_w, tiles_h, tiles_t;
  int num_ksteps;  // 64-voxel boxes in the whole tensor: the k-steps of every tile
  int cin, cout;
  int ncols;      // ntaps * cin: dW columns
  int col_tiles;  // 256-column tiles per 128-channel row tile (tile = co_tile * col_tiles + col_tile)
  long long units;  // tiles * num_ksteps
  int ctas;         // persistent grid = number of shares
  int granule;      // share boundaries are multiples of this many k-steps: 1, or num_ksteps (whole tiles, no workspace)
  int period;       // min(k-steps per share rounded up, num_ksteps): the order a segment is walked in (see the producer)
  float* dw;
  long long ld_dw;
  int vec_ok;   // dw rows 8-byte aligned: float2 accesses
  float* dbias;  // kBias: += column sums of dY for output channels < n_bias (the convolution's bias gradient)
  int n_bias;
  float* ws;  // cut tiles: [2 * ctas][kTileM][kTileN] partial dW, then [2 * ctas][kTileM] partial db
};

// First (tile-major) unit of share b; share b is [share_begin(b), share_begin(b + 1)).
__host__ __device__ __forceinline__ long long share_begin(const WgradParams& p, int b) {
  return (long long)b * (p.units / p.granule) / p.ctas * p.granule;
}

// The MMA warpgroups' side of one segment: nsteps k-steps from ring stage s, each one m64n256k16 per 16 voxels
// (+ kOnes: the bias gradient, m64n16k16 against the tile of ones). kOnes is a template argument so that no branch sits
// among the wgmmas: ptxas would then fence every wgmma with its own warpgroup.arrive.
template <bool kOnes>
__device__ __forceinline__ void wgrad_mma_steps(float (&acc)[128], float (&accb)[8], int nsteps, const uint8_t* smem_a,
                                                const uint8_t* smem_b, uint32_t ones_addr, uint64_t* full,
                                                uint64_t* empty, int& s, uint32_t& ph, int lane) {
  int prev = -1;
  for (int i = 0; i < nsteps; ++i) {
    mbar_wait(&full[s], ph);
    const uint32_t a_addr = smem_u32(smem_a + s * kWABytes);
    const uint32_t b_addr = smem_u32(smem_b + s * kWBBytes);
    wgmma_fence();
    // MN-major panels [panel][64 k-rows][128 B]: 16 k-rows = 2048 B, panel stride = 8192 B
    // the segment's first MMA overwrites the accumulators (scale-d 0): zeroing them in registers instead would put
    // non-wgmma definitions of the accumulators between two wgmma pipelines, which makes ptxas serialize them
#pragma unroll
    for (int k = 0; k < kVox / 16; ++k)
      wgmma_ss<256, 1, 1>(acc, gmma_desc_sw128(a_addr + k * 2048, kPanelBytes, 1024),
                          gmma_desc_sw128(b_addr + k * 2048, kPanelBytes, 1024), (i | k) != 0);
    if constexpr (kOnes) {   // db += dY^T . 1  (N = 16 columns of ones; every column holds the same sum)
#pragma unroll
      for (int k = 0; k < kVox / 16; ++k)
        wgmma_ss<16, 1, 1>(accb, gmma_desc_sw128(a_addr + k * 2048, kPanelBytes, 1024),
                           gmma_desc_sw128(ones_addr, kPanelBytes, 1024), (i | k) != 0);
    }
    wgmma_commit();
    wgmma_wait<1>();   // the previous k-step's MMAs are done: its stage goes back to the producer
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
    prev = s;
    if (++s == kWStages) {
      s = 0;
      ph ^= 1;
    }
  }
  wgmma_wait<0>();
  if (lane == 0) mbar_arrive(&empty[prev]);
}

// Warp roles: warp 0 TMA producer, warps 1-3 idle (wgmma needs aligned warpgroups), warps 4-7 and 8-11 the two MMA
// warpgroups (output channels 0-63 and 64-127 of the tile), which also run the epilogue of each segment.
template <bool kBias>
__global__ void __launch_bounds__(kWThreads, 1)
    og_conv_wgrad_kernel(const __grid_constant__ CUtensorMap mapDY, const __grid_constant__ CUtensorMap mapX,
                         const WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kWStages * kWABytes;
  uint8_t* smem_ones = smem_b + kWStages * kWBBytes;   // 16 k-rows x 128 B of bf16 1.0 (bias-gradient operand), 1024-aligned
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_ones + 2048);
  uint64_t* empty = full + kWStages;

  const int warp = warp_idx_uniform();
  const int lane = threadIdx.x & 31;
  const long long u_begin = share_begin(p, blockIdx.x), u_end = share_begin(p, blockIdx.x + 1);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&mapDY);
    tma_prefetch_desc(&mapX);
    for (int s = 0; s < kWStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);   // lane 0 of each MMA warp
    }
    fence_mbar_init();
  }
  if (kBias) {
    for (int i = threadIdx.x; i < 2048 / 4; i += kWThreads) reinterpret_cast<uint32_t*>(smem_ones)[i] = 0x3F803F80u;
    fence_proxy_async_smem();   // generic-proxy writes -> visible to the tensor core's async-proxy reads
  }
  __syncthreads();

  if (warp == 0) {
    // whole warp runs the loop converged; one elected lane issues (see elect_one() in og_ptx.cuh)
    int s = 0;
    uint32_t ph = 0;
    const int per_sample = p.tiles_w * p.tiles_h * p.tiles_t;
    long long clock = 0;   // k-steps this CTA has walked
    for (long long u = u_begin; u < u_end;) {
      const int tile = (int)(u / p.num_ksteps);
      const int k0 = (int)(u - (long long)tile * p.num_ksteps);
      const int k1 = (int)min((long long)p.num_ksteps, u_end - (long long)tile * p.num_ksteps);
      u += k1 - k0;
      const int co0 = (tile / p.col_tiles) * kTileM;
      const int c0 = (tile % p.col_tiles) * kTileN;
      // the X panels of this tile: channel and tap offset of each; panels past the last column are not loaded
      const int npan = min(4, (p.ncols - c0) / 64);
      int pci[4], off_w[4], off_h[4], off_t[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = c0 + 64 * (j < npan ? j : 0);
        const int tap = c / p.cin;
        pci[j] = c - tap * p.cin;
        off_t[j] = tap / (p.kh * p.kw) - p.pt;
        off_h[j] = (tap / p.kw) % p.kh - p.ph;
        off_w[j] = tap % p.kw - p.pw;
      }
      const uint32_t tx_bytes = (uint32_t)(kWABytes + npan * kPanelBytes);
      // Walk [k0, k1) from the k-step congruent to this CTA's step count modulo the period, then wrap around to k0.
      // Every CTA then streams the voxel range at the same offset within a period at the same time, whichever tile it
      // works on, so a box fetched from DRAM for one tile is still in L2 when the other tiles read it.
      int ks = k0 + (int)((clock - k0 % p.period + p.period) % p.period);
      if (ks >= k1) ks = k0;
      clock += k1 - k0;
      int tn, tw, th, tt;
      auto decode = [&](int k) {   // box coordinates of k-step k (divisions only at a segment start and its wrap)
        tn = k / per_sample;
        int r = k - tn * per_sample;
        tw = r % p.tiles_w;
        r /= p.tiles_w;
        th = r % p.tiles_h;
        tt = r / p.tiles_h;
      };
      decode(ks);
      for (int i = k0; i < k1; ++i) {
        const int n = tn << p.bn_log2, w0 = tw << p.bw_log2, h0 = th << p.bh_log2, t0 = tt << p.bt_log2;
        mbar_wait(&empty[s], ph ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full[s], tx_bytes);
          uint8_t* a = smem_a + s * kWABytes;
          tma_load_5d(a, &mapDY, &full[s], co0, w0, h0, t0, n);
          tma_load_5d(a + kPanelBytes, &mapDY, &full[s], co0 + 64, w0, h0, t0, n);
          uint8_t* b = smem_b + s * kWBBytes;
          for (int j = 0; j < npan; ++j)
            tma_load_5d(b + j * kPanelBytes, &mapX, &full[s], pci[j], w0 * p.sx_w + off_w[j], h0 * p.sx_h + off_h[j],
                        t0 * p.sx_t + off_t[j], n);
        }
        __syncwarp();
        if (++s == kWStages) {
          s = 0;
          ph ^= 1;
        }
        if (++ks == k1) {
          ks = k0;
          decode(ks);
        } else if (++tw == p.tiles_w) {
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
    const int wg = (warp >> 2) - 1;   // output channels 64 wg .. 64 wg + 63 of the tile
    const int q = warp & 3;
    const uint32_t ones_addr = smem_u32(smem_ones);
    const uint8_t* a_wg = smem_a + wg * kPanelBytes;
    float acc[128], accb[8];
    int s = 0;
    uint32_t ph = 0;
    for (long long u = u_begin; u < u_end;) {
      const bool first = u == u_begin;
      const int tile = (int)(u / p.num_ksteps);
      const int k0 = (int)(u - (long long)tile * p.num_ksteps);
      const int k1 = (int)min((long long)p.num_ksteps, u_end - (long long)tile * p.num_ksteps);
      u += k1 - k0;
      const int co0 = (tile / p.col_tiles) * kTileM;
      const int c0 = (tile % p.col_tiles) * kTileN;
      const bool bias_tile = kBias && c0 == 0;
      if (bias_tile)
        wgrad_mma_steps<true>(acc, accb, k1 - k0, a_wg, smem_b, ones_addr, full, empty, s, ph, lane);
      else
        wgrad_mma_steps<false>(acc, accb, k1 - k0, a_wg, smem_b, ones_addr, full, empty, s, ph, lane);
      reg_fence(acc);
      reg_fence(accb);
      // epilogue straight from the fragments: row r = output channel co0 + r, column c = dW column c0 + c
      const bool whole = k0 == 0 && k1 == p.num_ksteps;
      const int slot = 2 * blockIdx.x + (first ? 0 : 1);
      const int c_lane = 2 * (lane & 3);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int r = wg * 64 + q * 16 + (lane >> 2) + rr * 8;
        const int co = co0 + r;
        if (whole) {   // the only owner of this tile: add into dW (ncols is a multiple of 64, so c < ncols covers c + 1)
          if (co >= p.cout) continue;
          float* row = p.dw + (long long)co * p.ld_dw + c0 + c_lane;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            if (c0 + 8 * j + c_lane >= p.ncols) continue;
            const float v0 = acc[4 * j + 2 * rr], v1 = acc[4 * j + 2 * rr + 1];
            if (p.vec_ok) {
              float2* d = reinterpret_cast<float2*>(row + 8 * j);
              const float2 o = *d;
              *d = make_float2(o.x + v0, o.y + v1);
            } else {
              row[8 * j] += v0;
              row[8 * j + 1] += v1;
            }
          }
          if (bias_tile && (lane & 3) == 0 && co < p.n_bias) p.dbias[co] += accb[2 * rr];
        } else {   // one segment of a cut tile: this CTA's slot, every element written
          float* sl = p.ws + ((long long)slot * kTileM + r) * kTileN + c_lane;
#pragma unroll
          for (int j = 0; j < 32; ++j)
            *reinterpret_cast<float2*>(sl + 8 * j) = make_float2(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1]);
          if (bias_tile && (lane & 3) == 0)
            p.ws[(long long)2 * p.ctas * kSlotFloats + (long long)slot * kTileM + r] = accb[2 * rr];
        }
      }
    }
  }
}

// Finishes the tiles cut by share boundaries. Block (x, y) handles 1024 elements of the tile holding the start of share
// y + 1, unless that tile starts before share y (then the block of the earlier boundary handles it) or the boundary is
// a tile edge. The segments are added in share order, i.e. in k order, and the sum is added into dW.
__global__ void __launch_bounds__(256) og_wgrad_fixup_kernel(const WgradParams p) {
  const int b = blockIdx.y;   // the share holding the tile's first k-step
  const long long ub = share_begin(p, b + 1);
  const int tile = (int)(ub / p.num_ksteps);
  const long long t0 = (long long)tile * p.num_ksteps, t1 = t0 + p.num_ksteps;
  if (ub == t0 || share_begin(p, b) > t0) return;
  const int co0 = (tile / p.col_tiles) * kTileM, c0 = (tile % p.col_tiles) * kTileN;
  const int e = (blockIdx.x * 256 + threadIdx.x) * 4;   // element of the tile
  const int r = e / kTileN, c = e % kTileN;
  float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
  float sumb = 0.f;
  const bool bias = p.dbias && c0 == 0 && blockIdx.x == 0 && threadIdx.x < kTileM;
  for (int sh = b; sh < p.ctas; ++sh) {
    const long long sb = share_begin(p, sh);
    if (sb >= t1) break;
    const int slot = 2 * sh + (sb >= t0 ? 0 : 1);   // the share's first segment, or (for share b) its last
    const float4 v = __ldcg(reinterpret_cast<const float4*>(p.ws + (long long)slot * kSlotFloats + e));
    sum.x += v.x;
    sum.y += v.y;
    sum.z += v.z;
    sum.w += v.w;
    if (bias) sumb += __ldcg(p.ws + (long long)2 * p.ctas * kSlotFloats + (long long)slot * kTileM + threadIdx.x);
  }
  if (co0 + r < p.cout && c0 + c < p.ncols) {   // ncols is a multiple of 64: all four columns are in range
    float* d = p.dw + (long long)(co0 + r) * p.ld_dw + c0 + c;
    d[0] += sum.x;
    d[1] += sum.y;
    d[2] += sum.z;
    d[3] += sum.w;
  }
  if (bias && co0 + (int)threadIdx.x < p.n_bias) p.dbias[co0 + threadIdx.x] += sumb;
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
  p.bw_log2 = ilog2(bw); p.bh_log2 = ilog2(bh); p.bt_log2 = ilog2(bt); p.bn_log2 = ilog2(bn);
  p.tiles_w = (W + bw - 1) / bw; p.tiles_h = (H + bh - 1) / bh; p.tiles_t = (T + bt - 1) / bt;
  p.num_ksteps = ((N + bn - 1) / bn) * p.tiles_w * p.tiles_h * p.tiles_t;
  p.cin = cin; p.cout = cout; p.dw = dw; p.ld_dw = ld_dw;
  p.ncols = kt * kh * kw * cin;
  p.col_tiles = (p.ncols + kTileN - 1) / kTileN;
  const long long tiles = (long long)((cout + kTileM - 1) / kTileM) * p.col_tiles;
  p.units = tiles * p.num_ksteps;
  // One share per SM, each at least 4 k-steps long so that pipeline fill stays amortised. Each share may leave two
  // segments in the workspace; with less room, fewer shares, and without room for more shares than tiles, whole
  // tiles only (no workspace).
  const int sms = num_sms();
  p.ctas = (int)std::min<long long>(sms, std::max<long long>(1, p.units / 4));
  p.granule = 1;
  const size_t slot_bytes = (size_t)(kSlotFloats + (dbias ? kTileM : 0)) * sizeof(float);
  const long long fit = workspace ? (long long)(workspace_bytes / (2 * slot_bytes)) : 0;
  if (fit < p.ctas) {
    if (fit > tiles) {
      p.ctas = (int)fit;
    } else {
      p.granule = p.num_ksteps;
      p.ctas = (int)std::min<long long>(sms, tiles);
    }
  }
  p.period = (int)std::min<long long>(p.num_ksteps, (p.units + p.ctas - 1) / p.ctas);
  p.ws = reinterpret_cast<float*>(workspace);
  p.vec_ok = (ld_dw % 2 == 0) && ((reinterpret_cast<uintptr_t>(dw) & 7) == 0);
  p.dbias = dbias;
  p.n_bias = n_bias;
  const size_t smem_bytes = (size_t)kWStages * (kWABytes + kWBBytes) + 2048 /*ones*/ + 1024 + 512;

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
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_conv_wgrad_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem_bytes));
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_conv_wgrad_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem_bytes));
    attr_set = true;
  }
  if (dbias)
    og_conv_wgrad_kernel<true><<<p.ctas, kWThreads, smem_bytes, (cudaStream_t)stream>>>(mapDY, mapX, p);
  else
    og_conv_wgrad_kernel<false><<<p.ctas, kWThreads, smem_bytes, (cudaStream_t)stream>>>(mapDY, mapX, p);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  if (p.granule == 1 && p.ctas > 1) {
    og_wgrad_fixup_kernel<<<dim3(kSlotFloats / 1024, p.ctas - 1), 256, 0, (cudaStream_t)stream>>>(p);
    OG_CHECK_CUDA(cudaGetLastError());
    g_launches.fetch_add(1);
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
