// conv3d_igemm.cu — stride-1 3-D convolution forward and data-gradient as an implicit GEMM on the
// Hopper tensor cores (wgmma.mma_async, fp32 accumulators in registers), operands staged by TMA.
//
//   D[m][n] = sum_k A[m][k] * B[n][k]      m = output voxel (n,t,h,w), n = output channel,
//                                           k = (segment, tap, input channel)
//
// A is never materialised: one k-block = 64 channels of ONE filter tap, and the 128 voxels of an M tile
// form a (bw x bh x bt) box of the NDHWC activation tensor, so the A tile of tap (it,ih,iw) is the SAME
// box shifted by (it-pt, ih-ph, iw-pw) — a single 5-D TMA tile load whose out-of-bounds elements are
// zero-filled by the hardware. That zero fill *is* the convolution padding, including the causal
// (front-only) time padding of CausalConv3d: pt = kt-1 simply shifts the box start to negative t.
// The reference does this with an explicit F.pad copy followed by conv3d (genie/module/video.py:160-192).
//
// Forward uses K-major weights w[cout][k]; the data gradient reuses the SAME weight buffer as an
// MN-major B operand (k = cout rows of 64, n = cin contiguous) with mirrored taps, so no transposed
// weight copy ever exists.
//
// Warp roles (384 threads, 1 CTA / SM, persistent over work items; "ping-pong" consumers):
//   warpgroup 0  producer: warp 0 issues the TMA loads (one elected lane); warps 1-3 only complete the warpgroup.
//                It gives its registers to the consumers (setmaxnreg 40 / 232).
//   warpgroups 1, 2  consumers: the CTA's i-th work item belongs to consumer i % 2, which runs its whole wgmma main
//                loop (128 x BN accumulator = two m64 halves in registers, BN <= 128) and then its epilogue straight
//                from the accumulator fragments. The main loops run strictly in item order (see kOrderBar), so one
//                consumer's epilogue overlaps the other consumer's MMAs.
// Both consumers read ONE stage ring, filled in item order. A consumer steps its ring position over the k-blocks of
// the other consumer's items; since an mbarrier parity wait cannot tell phase k from k + 2, it may only wait on a
// `full` barrier once every earlier item's stages have been filled, which the ordering of the main loops guarantees.
//
// Wide tiles (WIDE = true, 128 voxels x 256 channels, for the layers with 256 or more output channels; launch_igemm
// says which): both consumers work on every item, consumer wg on tile rows 64wg..64wg+63 against the whole 256-column B
// tile (m64n256k16, 128 fp32 accumulators per thread). A stage is 16 KiB of A + 32 KiB of B, and the A box and B tile
// are read from shared memory once per 128 x 256 outputs instead of once per 128 x 128 (B) or twice (A, when two N tiles
// cover 256 channels). The epilogues then no longer overlap the other consumer's MMAs: only the producer runs ahead.
// The k-blocks are added in the same order as in the ping-pong kernel, so the output has the same bits.
//
// Swapped tiles (SWAP = true, for 128 output channels over many voxels): a layer with 128 output channels has no second
// N tile to widen, so the tile grows along the voxels instead, with the operands swapped: D^T[channel][voxel] =
// W[channel][k] . X[voxel][k]^T. The weights are the wgmma A operand (consumer wg: channels 64wg..64wg+63; in the data
// gradient they are MN-major and read with the A-transpose bit), and a 256-voxel activation box, K-major as it lands
// from TMA, is B (m64n256k16). The epilogue transposes the [channel][voxel] fragments with stmatrix.trans through a
// shared buffer so that every row store is a whole 256-byte NDHWC row.
#include "og_host.cuh"
#include "og_ptx.cuh"

namespace og {
extern std::atomic<uint64_t> g_launches;

// One K segment = a (sub)set of filter taps over one input tensor. Along every axis d the taps visited are
// tap0[d] + j*tstep[d] (j < n[d]) of a (.., kh, kw) filter, and the A box of tap j is the M-tile box shifted by
// sh0[d] + j*shstep[d]:
//   forward                 n = k, tap0 = 0, tstep = 1, sh0 = -pad, shstep = +1      (x[v*stride + tap - pad])
//   data gradient, stride 1 n = k, tap0 = 0, tstep = 1, sh0 = +pad, shstep = -1      (dy[v - (tap - pad)])
//   data gradient, stride s one launch per residue class of the input position: n = #taps of that class,
//                           tap0 = class, tstep = s, sh0 = e, shstep = -1            (see og_conv3d_strided_dgrad)
// axis order: 0 = t, 1 = h, 2 = w.
struct IgemmSeg {
  int cin_blocks;  // channels / 64
  int n[3], tap0[3], tstep[3], sh0[3], shstep[3];
  int kh, kw;      // filter extents (tap index = (it*kh + ih)*kw + iw)
};

struct IgemmParams {
  int nseg;
  IgemmSeg seg[2];
  int sx[3];       // A box start = M-tile start * sx + shift (forward strided convolution: sx = stride; else 1)
  int OT, OH, OW;  // extents of the OUTPUT tensor; M-tile voxel (t,h,w) is stored at (t*om[0]+oo[0], h*om[1]+oo[1], ...)
  int om[3], oo[3];
  int b_mn_major;  // 0: B tile is [n rows][64 k] (K-major); 1: B tile is [k rows][n] in 64-wide panels (MN-major)
  int block_n;     // wgmma N (16..128)
  int num_n_tiles, num_m_tiles;
  int bw_log2, bh_log2, bt_log2, bn_log2;  // M tile = 2^bw x 2^bh x 2^bt x 2^bn voxels (product 128)
  int tiles_w, tiles_h, tiles_t;           // M tiles along each axis (ceil)
  int N, T, H, W;
  int n_out;      // valid output channels
  long long ldo;  // output row stride in elements
  void* out;
  int out_f32;
  int vec_ok;  // rows are 16-byte aligned and n_out is a multiple of the vector width
  const float* bias0;
  const float* bias1;
  int num_stages;
  int num_kb;  // k-blocks per tile
  int fast_store;  // bf16 output, n_out % 64 == 0, block_n % 64 == 0: coalesced staged stores
  const __nv_bfloat16* residual;  // optional bf16 [voxels][n_out] added to the output (out = conv + bias + residual)
  // fused epilogue reduction (fast_store path, one sample per CTA tile):
  double* gn_sums;             // forward: [N][2] += (sum y, sum y^2) of the bf16-rounded output (GroupNorm(1,C) statistics)
  int splits;      // split-K factor (1 = none): each work item covers a k-block range of one tile
  float* ws;       // when splits > 1: `splits` fp32 slabs of [voxels][n_out]; every split item STORES its partial tile into
  long long ws_slab;  // its own slab ws[split*ws_slab + ...] (no atomics, no memset) and the finish pass adds the slabs
};


static constexpr int kBlockM = 128;
static constexpr int kBlockK = 64;                       // 64 bf16 = one 128-byte swizzle row
static constexpr int kABytes = kBlockM * kBlockK * 2;    // 16 KiB
// Deeper rings fit in shared memory now that the epilogue needs no fp32 tile, but on H100 they measured slower: at
// BN = 128, 3, 5 and 6 stages all ran the large forward and data-gradient shapes 5-20% slower than 4.
static constexpr int kMaxStages = 4;
static constexpr int kThreads = 384;
// per consumer: bias row of the N tile (BN <= 128 floats) + 4 warps x 4 KiB store staging + GroupNorm sums (2 doubles)
// + GroupNorm sums of each of the 128 tile rows (float2)
static constexpr int kConsumerTail = 512 + 4 * 4096 + 64 + 128 * 8;
// barriers (256), then the two consumers' tails
static constexpr int kTailBytes = 256 + 2 * kConsumerTail;
// wide tile (kWideN = 256 columns, both consumers on every item), per consumer: bias row of the N tile (256 floats) +
// 4 warps x 2 KiB store staging + GroupNorm sums (2 doubles) + GroupNorm sums of its 64 tile rows per column half (float2)
static constexpr int kWideN = 256;
static constexpr int kWideConsumerTail = 1024 + 4 * 2048 + 64 + 2 * 64 * 8;
static constexpr int kWideTailBytes = 256 + 2 * kWideConsumerTail;
// swapped tile (256 voxels x 128 channels): barriers, a [64 voxels][128 channels] bf16 transpose buffer shared by both
// consumers, GroupNorm sums (2 doubles)
static constexpr int kSwapVox = 256;
static constexpr int kSwapTailBytes = 256 + 64 * 256 + 64;
// named barriers: 0 = __syncthreads, 1 + wg = consumer wg's own epilogue, kOrderBar + wg = "consumer wg may start its
// next main loop" (bar.arrive by the other consumer after it has issued its item's last MMA, bar.sync by wg)
static constexpr int kOrderBar = 3;

struct TileCoord {
  int n0, t0, h0, w0;
};

__device__ __forceinline__ TileCoord decode_m_tile(const IgemmParams& p, int m_tile) {
  TileCoord c;
  int per_sample = p.tiles_w * p.tiles_h * p.tiles_t;
  const int tn = m_tile / per_sample;
  c.n0 = tn << p.bn_log2;
  int r = m_tile - tn * per_sample;
  int tw = r % p.tiles_w;
  r /= p.tiles_w;
  int th = r % p.tiles_h;
  int tt = r / p.tiles_h;
  c.w0 = tw << p.bw_log2;
  c.h0 = th << p.bh_log2;
  c.t0 = tt << p.bt_log2;
  return c;
}

// Output voxel (row index of the output tensor) of row `row` of the M tile at `tc`; false for rows of a partial box.
// (generalised store position: a strided data gradient writes one residue class of the input grid per launch)
__device__ __forceinline__ bool tile_row(const IgemmParams& p, const TileCoord& tc, int row, long long& vox) {
  const int dw = row & ((1 << p.bw_log2) - 1);
  const int dh = (row >> p.bw_log2) & ((1 << p.bh_log2) - 1);
  const int dt = (row >> (p.bw_log2 + p.bh_log2)) & ((1 << p.bt_log2) - 1);
  const int dn = row >> (p.bw_log2 + p.bh_log2 + p.bt_log2);
  const int vn = tc.n0 + dn, vt = tc.t0 + dt, vh = tc.h0 + dh, vw = tc.w0 + dw;
  vox = (((long long)vn * p.OT + vt * p.om[0] + p.oo[0]) * p.OH + vh * p.om[1] + p.oo[1]) * p.OW + vw * p.om[2] + p.oo[2];
  return vn < p.N && vt < p.T && vh < p.H && vw < p.W;
}

// bias0 + bias1 of output column col (0 past n_out), summed as the epilogues always have: (0 + bias0) + bias1
__device__ __forceinline__ float bias_at(const IgemmParams& p, int col) {
  float b = 0.f;
  if (col < p.n_out) {
    if (p.bias0) b += __ldg(p.bias0 + col);
    if (p.bias1) b += __ldg(p.bias1 + col);
  }
  return b;
}

__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// WIDE: 128 x 256 tiles, both consumers on every item (see the file header); BN = kWideN, unsplit launches with bf16
// staged stores only (launch_igemm). SWAP (with WIDE): 256 voxels x 128 output channels with the operands swapped,
// D^T[channel][voxel] = W[channel][k] . X[voxel][k]^T; the activation box (256 voxels) is the wgmma B operand.
template <int BN, int BMN, bool WIDE, bool SWAP = false>
__global__ void __launch_bounds__(kThreads, 1)
    og_conv_igemm_kernel(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
                         const __grid_constant__ CUtensorMap mapB, const IgemmParams p) {
  static_assert(!SWAP || WIDE, "the swapped tile is a wide tile");
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment: required by the 128-byte swizzle pattern shared by TMA and the wgmma descriptors
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int b_bytes = p.block_n * kBlockK * 2;                 // weights
  const int a_bytes = SWAP ? kSwapVox * kBlockK * 2 : kABytes;   // activation box
  const int stage_bytes = a_bytes + b_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.num_stages * stage_bytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + kMaxStages;

  const int warp = warp_idx_uniform();
  const int lane = threadIdx.x & 31;
  const int total_tiles = p.num_m_tiles * p.num_n_tiles * p.splits;  // work items

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&mapA0);
    if (p.nseg > 1) tma_prefetch_desc(&mapA1);
    tma_prefetch_desc(&mapB);
    for (int s = 0; s < p.num_stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], WIDE ? 8 : 4);   // one arrival per warp of the consumer(s) that used the stage
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================================== TMA producer =====================================
    // (all 32 lanes of warp 0 run the loop converged; one elected lane issues — see elect_one() in og_ptx.cuh)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int item = blockIdx.x; item < total_tiles; item += gridDim.x) {
        const int tile = item / p.splits, split = item - tile * p.splits;
        const int m_super = tile / p.num_n_tiles;
        const int n_tile = tile - m_super * p.num_n_tiles;
        const TileCoord tc = decode_m_tile(p, m_super);
        const int kb_begin = (int)(((long long)p.num_kb * split) / p.splits);
        const int kb_end = (int)(((long long)p.num_kb * (split + 1)) / p.splits);
        // position (segment, tap = (jt, jh, jw), channel block) of kb_begin: divisions once per work item,
        // then the single producer thread only increments with carries (its instruction count per k-block
        // is what bounds the pipeline when MMAs are short)
        const int nkb0 = p.seg[0].cin_blocks * p.seg[0].n[0] * p.seg[0].n[1] * p.seg[0].n[2];
        int sidx = (kb_begin >= nkb0 && p.nseg > 1) ? 1 : 0;
        IgemmSeg sg = p.seg[sidx];
        int rel = kb_begin - (sidx ? nkb0 : 0);
        int tapc = rel / sg.cin_blocks;
        int cb = rel - tapc * sg.cin_blocks;
        int jt = tapc / (sg.n[1] * sg.n[2]);
        int jh = (tapc / sg.n[2]) % sg.n[1];
        int jw = tapc % sg.n[2];
        const int aw0 = tc.w0 * p.sx[2], ah0 = tc.h0 * p.sx[1], at0 = tc.t0 * p.sx[0];
        for (int kb = kb_begin; kb < kb_end; ++kb) {
          const CUtensorMap* mapA = (sidx == 0) ? &mapA0 : &mapA1;
          const int dt = sg.sh0[0] + jt * sg.shstep[0], dh = sg.sh0[1] + jh * sg.shstep[1],
                    dw = sg.sh0[2] + jw * sg.shstep[2];
          mbar_wait(&empty[stage], phase ^ 1);
          // stage = [activation box][weights], or [weights][activation box] for the swapped tile (the weights are then
          // the wgmma A operand, whose m64 halves start 8 KiB apart)
          uint8_t* sa = smem + stage * stage_bytes + (SWAP ? b_bytes : 0);
          uint8_t* sb = smem + stage * stage_bytes + (SWAP ? 0 : a_bytes);
          if (elect_one()) {
            mbar_expect_tx(&full[stage], (uint32_t)stage_bytes);
            tma_load_5d(sa, mapA, &full[stage], cb * kBlockK, aw0 + dw, ah0 + dh, at0 + dt, tc.n0);
            if (!BMN) {
              tma_load_2d(sb, &mapB, &full[stage], kb * kBlockK, n_tile * p.block_n);
            } else {
              // w[co][tap][ci] as (ci, tap, co): one (64 ci, 1 tap, 64 co) box per 64-wide N panel
              const int tap = ((sg.tap0[0] + jt * sg.tstep[0]) * sg.kh + sg.tap0[1] + jh * sg.tstep[1]) * sg.kw +
                              sg.tap0[2] + jw * sg.tstep[2];
              for (int pp = 0; pp < p.block_n / 64; ++pp)
                tma_load_3d(sb + pp * (64 * 128), &mapB, &full[stage], n_tile * p.block_n + pp * 64, tap,
                            cb * kBlockK);
            }
          }
          __syncwarp();
          if (++stage == p.num_stages) {
            stage = 0;
            phase ^= 1;
          }
          if (++cb == sg.cin_blocks) {
            cb = 0;
            if (++jw == sg.n[2]) {
              jw = 0;
              if (++jh == sg.n[1]) {
                jh = 0;
                if (++jt == sg.n[0]) {  // next segment (the fused 1x1x1 shortcut)
                  sidx = 1;
                  sg = p.seg[1];
                  jt = jh = jw = 0;
                }
              }
            }
          }
        }
      }
    }
  } else if constexpr (SWAP) {
    // ====== swapped tile: consumer wg = output channels 64wg..64wg+63 x all 256 voxels (m64n256), then the epilogue ======
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = (warp >> 2) - 1;
    const int q = warp & 3;
    const int ct = threadIdx.x - 128;   // 0..255 over both consumers
    uint8_t* tbuf = reinterpret_cast<uint8_t*>(bars) + 256;                  // [64 voxels][128 channels] bf16, swizzled
    double* stat_s = reinterpret_cast<double*>(tbuf + 64 * 256);            // [2]
    // this thread's two channel rows: 64wg + 16q + lane/4 (+ 8)
    const int ch0 = 64 * wg + 16 * q + (lane >> 2);
    const float bias_lo = bias_at(p, ch0), bias_hi = bias_at(p, ch0 + 8);
    int stage = 0;
    uint32_t phase = 0;
    if (ct == 0) stat_s[0] = stat_s[1] = 0.0;
    for (int item = blockIdx.x; item < total_tiles; item += gridDim.x) {
      float acc[BN / 2];
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t w_addr = smem_u32(smem + stage * stage_bytes) + wg * 8192;   // this consumer's 64 channels
        const uint32_t x_addr = smem_u32(smem + stage * stage_bytes) + b_bytes;     // [256 voxels][64 k]
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) {
          // weights: K-major [128 channel rows][64 k] (forward), or MN-major [64 k rows][64 channels] per 64-channel
          // panel (data gradient: w[co][tap][ci] has ci contiguous), read with the A-transpose bit
          const uint64_t adesc = BMN ? gmma_desc_sw128(w_addr + k * 2048, 64 * 128, 1024)
                                     : gmma_desc_sw128(w_addr + k * 32, 16, 1024);
          wgmma_ss<BN, BMN, 0>(acc, adesc, gmma_desc_sw128(x_addr + k * 32, 16, 1024), 1);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == p.num_stages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (lane == 0) mbar_arrive(&empty[prev]);

      // ---- epilogue (no residual: host-checked): acc[4j + 2h8 + {0,1}] = channel ch0 + 8h8, voxels 8j + 2(lane%4) +
      //      {0,1}. Per 64-voxel chunk both consumers transpose their fragments + bias into tbuf with stmatrix.trans,
      //      then all 256 threads store whole 256-byte NDHWC rows. 16-byte chunk c of row r sits at chunk c ^ (r % 8):
      //      the 8 rows of one 8x8 matrix then fall in 8 different bank groups.
      const TileCoord tc = decode_m_tile(p, item);
      float fl_s = 0.f, fl_ss = 0.f;
#pragma unroll
      for (int vc = 0; vc < 4; ++vc) {
        named_bar_sync(1, 256);   // the previous chunk's rows have been read out of tbuf
#pragma unroll
        for (int jp = 0; jp < 4; ++jp) {
          const int j = 8 * vc + 2 * jp;   // matrices m = 0..3: (voxel group j + m/2, channel half m%2)
          const int m = lane >> 3, r = 16 * jp + 8 * (m >> 1) + (lane & 7), c16 = 8 * wg + 2 * q + (m & 1);
          stmatrix_x4_trans(smem_u32(tbuf + r * 256 + ((c16 ^ (r & 7)) << 4)),
                            pack_bf16x2(acc[4 * j] + bias_lo, acc[4 * j + 1] + bias_lo),
                            pack_bf16x2(acc[4 * j + 2] + bias_hi, acc[4 * j + 3] + bias_hi),
                            pack_bf16x2(acc[4 * j + 4] + bias_lo, acc[4 * j + 5] + bias_lo),
                            pack_bf16x2(acc[4 * j + 6] + bias_hi, acc[4 * j + 7] + bias_hi));
        }
        named_bar_sync(1, 256);
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const int idx = it * 256 + ct, r = idx >> 4, c16 = idx & 15;
          long long vox;
          if (!tile_row(p, tc, vc * 64 + r, vox)) continue;
          const uint4 u = *reinterpret_cast<const uint4*>(tbuf + r * 256 + ((c16 ^ (r & 7)) << 4));
          reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + vox * p.ldo)[c16] = u;
          if (p.gn_sums) {   // GroupNorm(1, C) sums of the bf16-rounded output
            const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float2 f = __bfloat1622float2(h[e]);
              fl_s += f.x + f.y;
              fl_ss = fmaf(f.x, f.x, fmaf(f.y, f.y, fl_ss));
            }
          }
        }
      }
      if (p.gn_sums) {   // all voxels of a tile belong to one sample (host-checked)
        for (int o = 16; o > 0; o >>= 1) {
          fl_s += __shfl_xor_sync(0xffffffffu, fl_s, o);
          fl_ss += __shfl_xor_sync(0xffffffffu, fl_ss, o);
        }
        if (lane == 0) {
          atomicAdd(&stat_s[0], (double)fl_s);
          atomicAdd(&stat_s[1], (double)fl_ss);
        }
        named_bar_sync(1, 256);
        if (ct == 0) {
          atomicAdd(&p.gn_sums[(long long)tc.n0 * 2], stat_s[0]);
          atomicAdd(&p.gn_sums[(long long)tc.n0 * 2 + 1], stat_s[1]);
          stat_s[0] = 0.0;
          stat_s[1] = 0.0;
        }
      }
    }
  } else if constexpr (WIDE) {
    // ================= wide tile: both consumers on every item, m64n256 each, then the epilogue =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = (warp >> 2) - 1;   // tile rows 64 wg .. 64 wg + 63
    const int q = warp & 3;           // wgmma rows 16q..16q+15 of this consumer's m64 half
    const int et = threadIdx.x - 128 * (wg + 1);
    const int epi_bar = 1 + wg;
    uint8_t* tail = reinterpret_cast<uint8_t*>(bars) + 256 + wg * kWideConsumerTail;
    float* bias_s = reinterpret_cast<float*>(tail);                        // [BN] bias0 + bias1 of the current N tile
    uint8_t* my_stage = tail + 1024 + q * 2048;                            // this warp's 16 rows x 128 B store staging
    double* stat_s = reinterpret_cast<double*>(tail + 1024 + 4 * 2048);   // [2]
    float2* row_s = reinterpret_cast<float2*>(tail + 1024 + 4 * 2048 + 64);   // [2 column halves][64 tile rows]
    const int cl = 2 * (lane & 3);
    int stage = 0;
    uint32_t phase = 0;
    float fl_s[2] = {0.f, 0.f}, fl_ss[2] = {0.f, 0.f};   // GroupNorm row sums of columns 0-127 and 128-255
    if (et == 0) stat_s[0] = stat_s[1] = 0.0;
    for (int item = blockIdx.x; item < total_tiles; item += gridDim.x) {
      const int m_super = item / p.num_n_tiles;
      const int n_tile = item - m_super * p.num_n_tiles;
      float acc[BN / 2];
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * stage_bytes) + wg * 8192;   // this consumer's 64 A rows
        const uint32_t b_addr = smem_u32(smem + stage * stage_bytes) + a_bytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) {
          const uint64_t bdesc = BMN ? gmma_desc_sw128(b_addr + k * 2048, 64 * 128, 1024)
                                     : gmma_desc_sw128(b_addr + k * 32, 16, 1024);
          wgmma_ss<BN, 0, BMN>(acc, gmma_desc_sw128(a_addr + k * 32, 16, 1024), bdesc, 1);
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous k-block's MMAs are done: its stage goes back to the producer
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == p.num_stages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (lane == 0) mbar_arrive(&empty[prev]);

      // ---- epilogue: acc[4j + 2h8 + {0,1}] = tile row 64 wg + 16q + lane/4 + 8h8, columns 8j + cl + {0,1}. Per
      //      64-column chunk: fragments (+ residual) + bias -> bf16 -> this warp's 16 swizzled staging rows (staging
      //      row lr = tile row 64 wg + 16q + lr) -> 128-byte row segments, 2 rows per lane and instruction.
      const TileCoord tc = decode_m_tile(p, m_super);
      const int col0 = n_tile * BN;
      named_bar_sync(epi_bar, 128);   // the previous tile's bias readers are done
      for (int j = et; j < BN; j += 128) bias_s[j] = bias_at(p, col0 + j);
      named_bar_sync(epi_bar, 128);
      long long my_vox;   // lanes L and L + 16: staging row L % 16
      const int my_ok = tile_row(p, tc, wg * 64 + q * 16 + (lane & 15), my_vox);
      __nv_bfloat16* outp = reinterpret_cast<__nv_bfloat16*>(p.out) + col0;
      const __nv_bfloat16* resp = p.residual + col0;
      const int chunk = lane & 7;
#pragma unroll
      for (int c = 0; c < BN; c += 64) {
        if (col0 + c >= p.n_out) break;   // partial last N tile (n_out % 64 == 0, so chunks are all-or-nothing)
        if (p.residual) {
#pragma unroll
          for (int it = 0; it < 4; ++it) {
            const int r = it * 4 + (lane >> 3);
            const long long rvox = __shfl_sync(0xffffffffu, my_vox, r);
            const int rok = __shfl_sync(0xffffffffu, my_ok, r);
            uint4 u = make_uint4(0u, 0u, 0u, 0u);
            if (rok) u = __ldg(reinterpret_cast<const uint4*>(resp + rvox * p.ldo + c + chunk * 8));
            *reinterpret_cast<uint4*>(my_stage + r * 128 + ((chunk ^ (r & 7)) << 4)) = u;
          }
          __syncwarp();
        }
#pragma unroll
        for (int h8 = 0; h8 < 2; ++h8) {
          const int lr = h8 * 8 + (lane >> 2);   // lr & 7 == lane >> 2
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = c / 8 + jj;
            uint32_t* w = reinterpret_cast<uint32_t*>(my_stage + lr * 128 + ((jj ^ (lane >> 2)) << 4)) + (lane & 3);
            float v0 = acc[4 * j + 2 * h8], v1 = acc[4 * j + 2 * h8 + 1];
            if (p.residual) {   // fp32 add before the single bf16 rounding
              const float2 r = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(w));
              v0 += r.x;
              v1 += r.y;
            }
            const float2 b = *reinterpret_cast<const float2*>(bias_s + c + 8 * jj + cl);
            *w = pack_bf16x2(v0 + b.x, v1 + b.y);
          }
        }
        __syncwarp();
        if (p.gn_sums && my_ok && lane < 16) {
          // GroupNorm(1, C) sums of the bf16-rounded output: lane L < 16 sums staging row L in the order of the
          // ping-pong epilogue, one row sum per 128-column half (that kernel's N tile), so the sums keep their bits
          const int hf = c >> 7;
#pragma unroll
          for (int jc = 0; jc < 4; ++jc) {
            const uint4 u0 = *reinterpret_cast<const uint4*>(my_stage + lane * 128 + ((jc ^ (lane & 7)) << 4));
            const uint4 u1 = *reinterpret_cast<const uint4*>(my_stage + lane * 128 + (((jc + 4) ^ (lane & 7)) << 4));
            const __nv_bfloat162* h0 = reinterpret_cast<const __nv_bfloat162*>(&u0);
            const __nv_bfloat162* h1 = reinterpret_cast<const __nv_bfloat162*>(&u1);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float2 f0 = __bfloat1622float2(h0[e]), f1 = __bfloat1622float2(h1[e]);
              fl_s[hf] += f0.x + f1.x;
              fl_ss[hf] = fmaf(f0.x, f0.x, fmaf(f1.x, f1.x, fl_ss[hf]));
              fl_s[hf] += f0.y + f1.y;
              fl_ss[hf] = fmaf(f0.y, f0.y, fmaf(f1.y, f1.y, fl_ss[hf]));
            }
          }
        }
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const int r = it * 4 + (lane >> 3);
          const long long rvox = __shfl_sync(0xffffffffu, my_vox, r);
          const int rok = __shfl_sync(0xffffffffu, my_ok, r);
          const uint4 u = *reinterpret_cast<const uint4*>(my_stage + r * 128 + ((chunk ^ (r & 7)) << 4));
          if (rok) *reinterpret_cast<uint4*>(outp + rvox * p.ldo + c + chunk * 8) = u;
        }
        __syncwarp();
      }
      if (p.gn_sums) {
        // flush this tile's sums (all rows of a CTA tile belong to one sample: host-checked). Warp q adds the row sums
        // of column half q / 2 over 32 consecutive tile rows, exactly as the ping-pong kernel does per N tile; the
        // double sum of those fp32 partials does not depend on their order.
        if (lane < 16) {
          row_s[q * 16 + lane] = make_float2(fl_s[0], fl_ss[0]);
          row_s[64 + q * 16 + lane] = make_float2(fl_s[1], fl_ss[1]);
        }
        named_bar_sync(epi_bar, 128);
        const float2 rs = row_s[(q >> 1) * 64 + (q & 1) * 32 + lane];
        float s = rs.x, ss = rs.y;
        for (int o = 16; o > 0; o >>= 1) {
          s += __shfl_xor_sync(0xffffffffu, s, o);
          ss += __shfl_xor_sync(0xffffffffu, ss, o);
        }
        if (lane == 0) {
          atomicAdd(&stat_s[0], (double)s);
          atomicAdd(&stat_s[1], (double)ss);
        }
        named_bar_sync(epi_bar, 128);
        if (et == 0) {
          atomicAdd(&p.gn_sums[(long long)tc.n0 * 2], stat_s[0]);
          atomicAdd(&p.gn_sums[(long long)tc.n0 * 2 + 1], stat_s[1]);
          stat_s[0] = 0.0;
          stat_s[1] = 0.0;
        }
        fl_s[0] = fl_s[1] = fl_ss[0] = fl_ss[1] = 0.f;
      }
    }
  } else {
    // ============================ consumers: wgmma main loop + epilogue ============================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = (warp >> 2) - 1;   // consumer 0 or 1: the CTA's items i with i % 2 == wg
    const int q = warp & 3;           // warp of the warpgroup: wgmma rows 16q..16q+15 of each m64 half
    const int et = threadIdx.x - 128 * (wg + 1);
    const int epi_bar = 1 + wg;
    uint8_t* tail = reinterpret_cast<uint8_t*>(bars) + 256 + wg * kConsumerTail;
    float* bias_s = reinterpret_cast<float*>(tail);                       // [BN] bias0 + bias1 of the current N tile
    uint8_t* my_stage = tail + 512 + q * 4096;                            // this warp's 32 rows x 128 B store staging
    double* stat_s = reinterpret_cast<double*>(tail + 512 + 4 * 4096);   // [2]
    float2* row_s = reinterpret_cast<float2*>(tail + 512 + 4 * 4096 + 64);   // [128] GroupNorm sums of each tile row
    const int cl = 2 * (lane & 3);   // first of the two columns this thread holds in every 8-column group
    int stage = 0;
    uint32_t phase = 0;
    float fl_s = 0.f, fl_ss = 0.f;
    if (et == 0) stat_s[0] = stat_s[1] = 0.0;
    named_bar_sync(epi_bar, 128);
    int i = 0;
    for (int item = blockIdx.x; item < total_tiles; item += gridDim.x, ++i) {
      const int tile = item / p.splits;
      const int split = item - tile * p.splits;
      const int nkb = (int)(((long long)p.num_kb * (split + 1)) / p.splits) -
                      (int)(((long long)p.num_kb * split) / p.splits);
      if ((i & 1) != wg) {   // the other consumer's item: step over its k-blocks of the ring
        stage += nkb;
        const int wraps = stage / p.num_stages;
        stage -= wraps * p.num_stages;
        phase ^= wraps & 1;
        continue;
      }
      const int m_super = tile / p.num_n_tiles;
      const int n_tile = tile - m_super * p.num_n_tiles;
      // wait until the other consumer has issued the previous item's last MMA, i.e. waited for all of its stages
      if (i > 0) named_bar_sync(kOrderBar + wg, 256);
      float acc[2][BN / 2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) acc[hh][j] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * stage_bytes);
        const uint32_t b_addr = a_addr + a_bytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) {
          // A: K-major, 128-byte rows, 8-row groups 1024 B apart; advance 16 elements = 32 B inside the row.
          // B: K-major [BN rows][64 k], or MN-major panels [BN/64][64 k-rows][128 B] (16 k-rows = 2048 B, panels 8 KiB apart)
          const uint64_t bdesc = BMN ? gmma_desc_sw128(b_addr + k * 2048, 64 * 128, 1024)
                                     : gmma_desc_sw128(b_addr + k * 32, 16, 1024);
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
            wgmma_ss<BN, 0, BMN>(acc[hh], gmma_desc_sw128(a_addr + hh * 8192 + k * 32, 16, 1024), bdesc, 1);
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous k-block's MMAs are done: its stage goes back to the producer
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == p.num_stages) {
          stage = 0;
          phase ^= 1;
        }
      }
      if (item + gridDim.x < total_tiles) named_bar_arrive(kOrderBar + (wg ^ 1), 256);   // the next item's turn
      wgmma_wait<0>();
      reg_fence(acc[0]);
      reg_fence(acc[1]);
      if (lane == 0) mbar_arrive(&empty[prev]);

      // ---- epilogue from the fragments: acc[hh][4j + 2h8 + {0,1}] = tile row hh*64 + 16q + lane/4 + 8h8,
      //      columns 8j + cl + {0,1}
      const TileCoord tc = decode_m_tile(p, m_super);
      const int col0 = n_tile * p.block_n;
      if (p.splits > 1) {
        // split-K: store this item's partial sums into its own slab of the fp32 workspace; bias / cast happen in the
        // finish pass
        float* ws = p.ws + (long long)split * p.ws_slab + col0;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int h8 = 0; h8 < 2; ++h8) {
            long long vox;
            if (!tile_row(p, tc, hh * 64 + q * 16 + (lane >> 2) + 8 * h8, vox)) continue;
            float* dst = ws + vox * p.ldo;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
              const int col = col0 + 8 * j + cl;
              const float v0 = acc[hh][4 * j + 2 * h8], v1 = acc[hh][4 * j + 2 * h8 + 1];
              if (p.vec_ok && col + 1 < p.n_out) {
                __stcg(reinterpret_cast<float2*>(dst + 8 * j + cl), make_float2(v0, v1));
              } else {
                if (col < p.n_out) dst[8 * j + cl] = v0;
                if (col + 1 < p.n_out) dst[8 * j + cl + 1] = v1;
              }
            }
          }
      } else if (p.fast_store) {
        // bf16 output, whole 64-column chunks: fragments (+ residual) + bias -> bf16 -> this warp's swizzled staging
        // rows -> the warp writes 4 full 128-byte row segments per instruction. Staging row lr (0..31) is tile row
        // (lr / 16) * 64 + 16q + lr % 16, so the 32 rows are exactly those whose fragments this warp holds.
        named_bar_sync(epi_bar, 128);   // the previous tile's bias readers are done
        for (int j = et; j < p.block_n; j += 128) bias_s[j] = bias_at(p, col0 + j);
        named_bar_sync(epi_bar, 128);
        long long my_vox;   // lane L: staging row L
        const int my_ok = tile_row(p, tc, (lane >> 4) * 64 + q * 16 + (lane & 15), my_vox);
        __nv_bfloat16* outp = reinterpret_cast<__nv_bfloat16*>(p.out) + col0;
        const __nv_bfloat16* resp = p.residual + col0;
        const int chunk = lane & 7;
#pragma unroll
        for (int c = 0; c < BN; c += 64) {
          if (col0 + c >= p.n_out) break;   // partial last N tile (n_out % 64 == 0, so chunks are all-or-nothing)
          if (p.residual) {   // the residual's row segments, coalesced, into the staging rows
#pragma unroll
            for (int it = 0; it < 8; ++it) {
              const int r = it * 4 + (lane >> 3);
              const long long rvox = __shfl_sync(0xffffffffu, my_vox, r);
              const int rok = __shfl_sync(0xffffffffu, my_ok, r);
              uint4 u = make_uint4(0u, 0u, 0u, 0u);
              if (rok) u = __ldg(reinterpret_cast<const uint4*>(resp + rvox * p.ldo + c + chunk * 8));
              *reinterpret_cast<uint4*>(my_stage + r * 128 + ((chunk ^ (r & 7)) << 4)) = u;
            }
            __syncwarp();
          }
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int h8 = 0; h8 < 2; ++h8) {
              const int lr = hh * 16 + h8 * 8 + (lane >> 2);   // lr & 7 == lane >> 2
#pragma unroll
              for (int jj = 0; jj < 8; ++jj) {
                const int j = c / 8 + jj;
                // the staging word of columns c + 8jj + cl + {0,1}: the residual is read from it and the output
                // written back to it by the same thread
                uint32_t* w = reinterpret_cast<uint32_t*>(my_stage + lr * 128 + ((jj ^ (lane >> 2)) << 4)) + (lane & 3);
                float v0 = acc[hh][4 * j + 2 * h8], v1 = acc[hh][4 * j + 2 * h8 + 1];
                if (p.residual) {   // fp32 add before the single bf16 rounding
                  const float2 r = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(w));
                  v0 += r.x;
                  v1 += r.y;
                }
                const float2 b = *reinterpret_cast<const float2*>(bias_s + c + 8 * jj + cl);
                *w = pack_bf16x2(v0 + b.x, v1 + b.y);
              }
            }
          __syncwarp();
          if (p.gn_sums && my_ok) {
            // GroupNorm(1, C) sums of the bf16-rounded output: lane L sums its staging row L, columns c + j and
            // c + 32 + j in turn (j < 32). Row by row in this order, then a warp sum over 32 consecutive tile rows
            // (below), the sums come out with the same bits whatever the warp layout of the accumulators.
#pragma unroll
            for (int jc = 0; jc < 4; ++jc) {
              const uint4 u0 = *reinterpret_cast<const uint4*>(my_stage + lane * 128 + ((jc ^ (lane & 7)) << 4));
              const uint4 u1 = *reinterpret_cast<const uint4*>(my_stage + lane * 128 + (((jc + 4) ^ (lane & 7)) << 4));
              const __nv_bfloat162* h0 = reinterpret_cast<const __nv_bfloat162*>(&u0);
              const __nv_bfloat162* h1 = reinterpret_cast<const __nv_bfloat162*>(&u1);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 f0 = __bfloat1622float2(h0[e]), f1 = __bfloat1622float2(h1[e]);
                fl_s += f0.x + f1.x;
                fl_ss = fmaf(f0.x, f0.x, fmaf(f1.x, f1.x, fl_ss));
                fl_s += f0.y + f1.y;
                fl_ss = fmaf(f0.y, f0.y, fmaf(f1.y, f1.y, fl_ss));
              }
            }
          }
#pragma unroll
          for (int it = 0; it < 8; ++it) {
            const int r = it * 4 + (lane >> 3);
            const long long rvox = __shfl_sync(0xffffffffu, my_vox, r);
            const int rok = __shfl_sync(0xffffffffu, my_ok, r);
            const uint4 u = *reinterpret_cast<const uint4*>(my_stage + r * 128 + ((chunk ^ (r & 7)) << 4));
            if (rok) *reinterpret_cast<uint4*>(outp + rvox * p.ldo + c + chunk * 8) = u;
          }
          __syncwarp();
        }
        if (p.gn_sums) {
          // flush this tile's GroupNorm sums (all rows of a CTA tile belong to one sample: host-checked). The row
          // sums go through shared memory so that warp w adds those of tile rows 32w .. 32w + 31.
          row_s[(lane >> 4) * 64 + q * 16 + (lane & 15)] = make_float2(fl_s, fl_ss);
          named_bar_sync(epi_bar, 128);
          const float2 rs = row_s[q * 32 + lane];
          fl_s = rs.x;
          fl_ss = rs.y;
          for (int o = 16; o > 0; o >>= 1) {
            fl_s += __shfl_xor_sync(0xffffffffu, fl_s, o);
            fl_ss += __shfl_xor_sync(0xffffffffu, fl_ss, o);
          }
          if (lane == 0) {
            atomicAdd(&stat_s[0], (double)fl_s);
            atomicAdd(&stat_s[1], (double)fl_ss);
          }
          named_bar_sync(epi_bar, 128);
          if (et == 0) {
            atomicAdd(&p.gn_sums[(long long)tc.n0 * 2], stat_s[0]);
            atomicAdd(&p.gn_sums[(long long)tc.n0 * 2 + 1], stat_s[1]);
            stat_s[0] = 0.0;
            stat_s[1] = 0.0;
          }
          fl_s = fl_ss = 0.f;
        }
      } else {
        // fp32 output, BN < 64 or n_out not a multiple of 64: masked stores straight from the fragments,
        // (acc + bias) + residual
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int h8 = 0; h8 < 2; ++h8) {
            long long vox;
            if (!tile_row(p, tc, hh * 64 + q * 16 + (lane >> 2) + 8 * h8, vox)) continue;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
              const int col = col0 + 8 * j + cl;
              if (col >= p.n_out) continue;
              const bool two = col + 1 < p.n_out;
              float f0 = acc[hh][4 * j + 2 * h8] + bias_at(p, col);
              float f1 = acc[hh][4 * j + 2 * h8 + 1] + bias_at(p, col + 1);
              if (p.residual) {
                f0 += __bfloat162float(p.residual[vox * p.ldo + col]);
                if (two) f1 += __bfloat162float(p.residual[vox * p.ldo + col + 1]);
              }
              if (p.out_f32) {
                float* o = reinterpret_cast<float*>(p.out) + vox * p.ldo + col;
                if (p.vec_ok && two) {
                  *reinterpret_cast<float2*>(o) = make_float2(f0, f1);
                } else {
                  o[0] = f0;
                  if (two) o[1] = f1;
                }
              } else {
                __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + vox * p.ldo + col;
                if (p.vec_ok && two) {
                  *reinterpret_cast<uint32_t*>(o) = pack_bf16x2(f0, f1);
                } else {
                  o[0] = __float2bfloat16_rn(f0);
                  if (two) o[1] = __float2bfloat16_rn(f1);
                }
              }
            }
          }
      }
    }
  }
}

// split-K finish: out = cast(ws + bias0 + bias1)
// Finish pass of a split-K launch: out = cast(sum of the `nslab` partial slabs + bias), and — optionally — the per-sample
// GroupNorm(1, C) sums of the bf16-rounded result (what og_gn_stats would compute in another pass over `out`).
// grid = (chunks, samples); `per_sample` = T*H*W*n_out elements.
template <int VEC>
__global__ void __launch_bounds__(256)
    og_splitk_finish_kernel(const float* __restrict__ ws, long long slab, int nslab, const float* __restrict__ bias0,
                            const float* __restrict__ bias1, void* __restrict__ out, int out_f32, int n_out,
                            long long per_sample, double* __restrict__ gn_sums) {
  const long long base = (long long)blockIdx.y * per_sample;
  float s = 0.f, ss = 0.f;
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * VEC; i < per_sample;
       i += (long long)gridDim.x * blockDim.x * VEC) {
    float v[VEC];
    if (VEC == 4) {
      const float4 a = __ldcg(reinterpret_cast<const float4*>(ws + base + i));
      v[0] = a.x; v[1 % VEC] = a.y; v[2 % VEC] = a.z; v[3 % VEC] = a.w;
      for (int k = 1; k < nslab; ++k) {
        const float4 b = __ldcg(reinterpret_cast<const float4*>(ws + (long long)k * slab + base + i));
        v[0] += b.x; v[1 % VEC] += b.y; v[2 % VEC] += b.z; v[3 % VEC] += b.w;
      }
    } else {
      v[0] = __ldcg(ws + base + i);
      for (int k = 1; k < nslab; ++k) v[0] += __ldcg(ws + (long long)k * slab + base + i);
    }
    const int col = (int)(i % n_out);
#pragma unroll
    for (int e = 0; e < VEC; ++e) {
      if (bias0) v[e] += __ldg(bias0 + col + e);
      if (bias1) v[e] += __ldg(bias1 + col + e);
    }
    if (out_f32) {
#pragma unroll
      for (int e = 0; e < VEC; ++e) reinterpret_cast<float*>(out)[base + i + e] = v[e];
    } else {
      __nv_bfloat16 h[VEC];
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        h[e] = __float2bfloat16_rn(v[e]);
        const float r = __bfloat162float(h[e]);
        s += r;
        ss = fmaf(r, r, ss);
      }
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out) + base + i;
      if (VEC == 4)
        *reinterpret_cast<uint2*>(o) = *reinterpret_cast<const uint2*>(h);
      else
        o[0] = h[0];
    }
  }
  if (gn_sums) {
    __shared__ float red[2][8];
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, off);
      ss += __shfl_xor_sync(0xffffffffu, ss, off);
    }
    if ((threadIdx.x & 31) == 0) {
      red[0][threadIdx.x >> 5] = s;
      red[1][threadIdx.x >> 5] = ss;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double a = 0.0, b = 0.0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
        a += (double)red[0][w];
        b += (double)red[1][w];
      }
      atomicAdd(gn_sums + 2 * blockIdx.y, a);
      atomicAdd(gn_sums + 2 * blockIdx.y + 1, b);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static int pick_block_n(int n_out, bool mn_major) {
  // The widest N tile that covers n_out, up to 128: the 128 x 128 fp32 accumulator is 128 registers per thread of the
  // one MMA warpgroup, the most that leaves room for addressing. Low tile counts are handled by split-K.
  int bn = 16;
  while (bn < n_out && bn < 128) bn *= 2;
  if (mn_major && bn < 64) bn = 64;
  return bn;
}

template <int BN, int BMN, bool WIDE = false, bool SWAP = false>
static int launch_igemm_kernel(int grid, size_t smem_bytes, cudaStream_t stream, const CUtensorMap& mapA0,
                               const CUtensorMap& mapA1, const CUtensorMap& mapB, const IgemmParams& p) {
  static bool attr_set = false;
  if (!attr_set) {
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_conv_igemm_kernel<BN, BMN, WIDE, SWAP>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  og_conv_igemm_kernel<BN, BMN, WIDE, SWAP><<<grid, kThreads, smem_bytes, stream>>>(mapA0, mapA1, mapB, p);
  OG_CHECK_CUDA(cudaGetLastError());
  return OG_OK;
}

struct IgemmLaunch {
  const void* a0 = nullptr;   // segment-0 input tensor (bf16 NDHWC), c0 channels, spatial extents aT x aH x aW
  int c0 = 0;
  int aT = 0, aH = 0, aW = 0;
  int astride[3] = {1, 1, 1};  // element stride of the A boxes along (t, h, w): forward strided convolution
  const void* a1 = nullptr;    // optional segment-1 tensor (the fused 1x1x1 shortcut), same extents as the output grid
  int c1 = 0;
  IgemmSeg segs[2];
  int nseg = 1;
  const void* w = nullptr;
  int ldw = 0, k_off = 0, b_mn_major = 0, b_rows = 0, b_ntaps = 0;
  const float* bias0 = nullptr;
  const float* bias1 = nullptr;
  const void* residual = nullptr;
  void* out = nullptr;
  int out_f32 = 0;
  int N = 0, T = 0, H = 0, W = 0;  // the M grid (voxels this launch computes)
  int OT = 0, OH = 0, OW = 0;      // output tensor extents (0 = same as the M grid)
  int om[3] = {1, 1, 1}, oo[3] = {0, 0, 0};
  int n_out = 0;
  void* workspace = nullptr;
  size_t workspace_bytes = 0;
  double* gn_sums = nullptr;
};

static IgemmSeg make_seg(int cin_blocks, int kt, int kh, int kw, int pt, int ph, int pw, int sgn) {
  IgemmSeg g;
  g.cin_blocks = cin_blocks;
  const int k[3] = {kt, kh, kw}, pd[3] = {pt, ph, pw};
  for (int d = 0; d < 3; ++d) {
    g.n[d] = k[d];
    g.tap0[d] = 0;
    g.tstep[d] = 1;
    g.sh0[d] = -sgn * pd[d];
    g.shstep[d] = sgn;
  }
  g.kh = kh;
  g.kw = kw;
  return g;
}

static int launch_igemm(const IgemmLaunch& L, cudaStream_t stream) {
  const int N = L.N, T = L.T, H = L.H, W = L.W, n_out = L.n_out;
  OG_REQUIRE(N > 0 && T > 0 && H > 0 && W > 0 && n_out > 0, "conv3d: empty problem");
  const bool plain = (L.OT == 0) && L.astride[0] == 1 && L.astride[1] == 1 && L.astride[2] == 1;
  // 128 output channels over many voxels: 256-voxel x 128-channel tiles with the operands swapped (see the kernel), when
  // there are at least four such tiles per SM (then the launch would not be split either). scripts/bench_conv_gemm.py,
  // ms per launch, ping-pong -> swapped, H100 SXM at 700 W: fwd 256->128 @16x64x64 1.464 -> 1.394, 128->128 + sc256
  // 0.797 -> 0.751, 128->128 0.720 -> 0.717; data gradient 128<-3 (the tail) 0.941 -> 0.566, 128<-128 0.722 -> 0.718.
  // With a residual it measured slower (fwd 128->128 0.726 -> 0.783: the residual tile is read in the unoverlapped
  // epilogue), so residual launches keep the ping-pong kernel.
  const bool swap = plain && !L.out_f32 && !L.residual && n_out == 128 &&
                    (long long)N * T * H * W >= 4LL * kSwapVox * num_sms();
  int bw, bh, bt, bn;
  choose_voxel_box(swap ? kSwapVox : kBlockM, N, T, H, W, &bw, &bh, &bt, &bn);
  IgemmParams p;
  memset(&p, 0, sizeof(p));
  p.nseg = L.nseg;
  p.num_kb = 0;
  for (int s = 0; s < L.nseg; ++s) {
    p.seg[s] = L.segs[s];
    p.num_kb += L.segs[s].cin_blocks * L.segs[s].n[0] * L.segs[s].n[1] * L.segs[s].n[2];
  }
  OG_REQUIRE(p.num_kb > 0, "conv3d: empty reduction");
  for (int d = 0; d < 3; ++d) {
    p.sx[d] = L.astride[d];
    p.om[d] = L.om[d];
    p.oo[d] = L.oo[d];
  }
  p.OT = L.OT ? L.OT : T;
  p.OH = L.OH ? L.OH : H;
  p.OW = L.OW ? L.OW : W;
  p.b_mn_major = L.b_mn_major;
  p.bw_log2 = ilog2(bw);
  p.bh_log2 = ilog2(bh);
  p.bt_log2 = ilog2(bt);
  p.bn_log2 = ilog2(bn);
  p.tiles_w = (W + bw - 1) / bw;
  p.tiles_h = (H + bh - 1) / bh;
  p.tiles_t = (T + bt - 1) / bt;
  p.N = N;
  p.T = T;
  p.H = H;
  p.W = W;
  p.num_m_tiles = ((N + bn - 1) / bn) * p.tiles_w * p.tiles_h * p.tiles_t;
  p.block_n = pick_block_n(n_out, L.b_mn_major != 0);
  p.num_n_tiles = (n_out + p.block_n - 1) / p.block_n;
  p.n_out = n_out;
  p.ldo = n_out;
  p.out = L.out;
  p.out_f32 = L.out_f32;
  p.vec_ok = L.out_f32 ? (n_out % 4 == 0) : (n_out % 8 == 0);
  p.bias0 = L.bias0;
  p.bias1 = L.bias1;
  p.residual = reinterpret_cast<const __nv_bfloat16*>(L.residual);
  p.fast_store = (!L.out_f32 && n_out % 64 == 0 && p.block_n % 64 == 0) ? 1 : 0;
  // split-K when the tiles cannot fill the machine and each has a long K loop: every split stores into its own fp32 slab
  // of the workspace, so the split shrinks to the slabs that fit and the launch runs unsplit below two
  p.splits = 1;
  if (plain) {
    const long long tiles = (long long)p.num_m_tiles * p.num_n_tiles;
    const size_t need = (size_t)N * T * H * W * n_out * sizeof(float);   // one slab
    if (tiles * 2 <= num_sms() && p.num_kb >= 32 && L.workspace && !L.residual) {
      int sp = (int)(num_sms() / tiles);
      if (sp > p.num_kb / 8) sp = p.num_kb / 8;
      if (sp > 16) sp = 16;
      if ((size_t)sp > L.workspace_bytes / need) sp = (int)(L.workspace_bytes / need);
      if (sp >= 2) {
        p.splits = sp;
        p.ws = reinterpret_cast<float*>(L.workspace);
        p.ws_slab = (long long)(need / sizeof(float));
      }
    }
  }
  // 128 x 256 tiles (both consumers on each item) for unsplit, plain launches with staged bf16 stores and >= 256 output
  // channels; everything else keeps the ping-pong kernel with BN <= 128. scripts/bench_conv_gemm.py, ms per launch,
  // ping-pong -> wide, H100 SXM at a 400 W power limit (two alternated runs agreed within a few percent):
  //   forward  256->1024 @16x32x32 4.02 -> 3.22, 256->2048 @8x16x16 0.99 -> 0.78, 512->4096 @4x8x8 0.58 -> 0.41,
  //            512->256 @8x16x16 0.213 -> 0.176, 256->256 @16x32x32 0.794 -> 0.757, +sc128 0.826 -> 0.781,
  //            128->256 @16x32x32 0.414 -> 0.398, 256->256 @8x16x16 0.108 -> 0.106
  //   data gradient (MN-major weights) 256<-1024 @16x32x32 3.56 -> 3.04, 256<-128 @16x64x64 1.77 -> 1.64,
  //            256<-256 @16x32x32 0.777 -> 0.743, 256<-256 @8x16x16 0.114 -> 0.102; but slower with 512 outputs
  //            (512<-256 @8x16x16 0.204 -> 0.224) and with 2048-channel dy boxes (256<-2048 @8x16x16 0.763 -> 0.886),
  //            so the data gradient takes the wide tile only for 256 outputs over at most 1024 channels.
  const bool wide = plain && p.splits == 1 && p.fast_store && n_out >= kWideN &&
                    (!L.b_mn_major || (n_out == kWideN && L.c0 <= 1024));
  if (wide) {
    p.block_n = kWideN;
    p.num_n_tiles = (n_out + kWideN - 1) / kWideN;
  }
  OG_REQUIRE(!swap || (p.splits == 1 && p.fast_store && p.num_n_tiles == 1), "conv3d: bad swapped-tile launch");
  const int stage_bytes = (swap ? kSwapVox * kBlockK * 2 : kABytes) + p.block_n * kBlockK * 2;
  const int tail_bytes = swap ? kSwapTailBytes : wide ? kWideTailBytes : kTailBytes;
  int stages = (227 * 1024 - 1024 /*align slack*/ - tail_bytes) / stage_bytes;
  if (stages > kMaxStages) stages = kMaxStages;
  p.num_stages = stages;
  const size_t smem_bytes = (size_t)stages * stage_bytes + 1024 + tail_bytes;

  // the fused GroupNorm sums need: staged bf16 stores, no split-K, every CTA tile inside one sample. Requested sums
  // that neither the epilogue nor the split-K finish pass can make come from og_gn_stats over the stored output; its
  // conditions are checked here, before anything is launched, so that a refused call leaves `out` untouched.
  const bool can_fuse = plain && p.fast_store && p.splits == 1 && bn == 1 && n_out <= 65536;
  const bool finish_did_stats = L.gn_sums && p.splits > 1 && !L.out_f32;
  const bool stats_pass = L.gn_sums && !can_fuse && !finish_did_stats;
  OG_REQUIRE(!stats_pass || (!L.out_f32 && plain && n_out % 8 == 0 && n_out <= 2048),
             "conv3d: GroupNorm statistics of this launch need a plain bf16 output with cout %% 8 == 0 and cout <= 2048 "
             "(cout=%d)", n_out);

  CUtensorMap mapA0, mapA1, mapB;
  {
    // forward strided convolution: the box spans bw*sw input positions and TMA traverses it with element stride sw,
    // landing exactly the bw voxels the tile needs (the hardware zero-fills the out-of-range ones: the padding)
    const int c0 = L.c0;
    const int st = L.astride[0], sh = L.astride[1], sw = L.astride[2];
    uint64_t dims[5] = {(uint64_t)c0, (uint64_t)L.aW, (uint64_t)L.aH, (uint64_t)L.aT, (uint64_t)N};
    uint64_t str[4] = {(uint64_t)c0 * 2, (uint64_t)L.aW * c0 * 2, (uint64_t)L.aH * L.aW * c0 * 2,
                       (uint64_t)L.aT * L.aH * L.aW * c0 * 2};
    uint32_t box[5] = {kBlockK, (uint32_t)(bw * sw), (uint32_t)(bh * sh), (uint32_t)(bt * st), (uint32_t)bn};
    uint32_t es[5] = {1, (uint32_t)sw, (uint32_t)sh, (uint32_t)st, 1};
    OG_REQUIRE(box[1] <= 256 && box[2] <= 256 && box[3] <= 256, "conv3d: strided box exceeds the TMA limit");
    int r = make_tmap_bf16(&mapA0, L.a0, 5, dims, str, box, es);
    if (r != OG_OK) return r;
  }
  if (L.nseg > 1) {
    const int c1 = L.c1;
    uint64_t dims[5] = {(uint64_t)c1, (uint64_t)W, (uint64_t)H, (uint64_t)T, (uint64_t)N};
    uint64_t str[4] = {(uint64_t)c1 * 2, (uint64_t)W * c1 * 2, (uint64_t)H * W * c1 * 2, (uint64_t)T * H * W * c1 * 2};
    uint32_t box[5] = {kBlockK, (uint32_t)bw, (uint32_t)bh, (uint32_t)bt, (uint32_t)bn};
    int r = make_tmap_bf16(&mapA1, L.a1, 5, dims, str, box);
    if (r != OG_OK) return r;
  } else {
    mapA1 = mapA0;
  }
  const __nv_bfloat16* wb = reinterpret_cast<const __nv_bfloat16*>(L.w) + L.k_off;
  if (!L.b_mn_major) {
    // rows = output channels, contiguous k
    uint64_t ktot = (uint64_t)p.num_kb * kBlockK;
    uint64_t dims[2] = {ktot, (uint64_t)n_out};
    uint64_t str[1] = {(uint64_t)L.ldw * 2};
    uint32_t box[2] = {kBlockK, (uint32_t)p.block_n};
    int r = make_tmap_bf16(&mapB, wb, 2, dims, str, box);
    if (r != OG_OK) return r;
  } else {
    // w[co][tap][ci] viewed as (ci, tap, co): a (64,1,64) box lands as one [64 co rows][64 ci] panel
    uint64_t dims[3] = {(uint64_t)n_out, (uint64_t)L.b_ntaps, (uint64_t)L.b_rows};
    uint64_t str[2] = {(uint64_t)n_out * 2, (uint64_t)L.ldw * 2};
    uint32_t box[3] = {64, 1, 64};
    int r = make_tmap_bf16(&mapB, wb, 3, dims, str, box);
    if (r != OG_OK) return r;
  }

  p.gn_sums = (L.gn_sums && can_fuse) ? L.gn_sums : nullptr;
  const int total_tiles = p.num_m_tiles * p.num_n_tiles * p.splits;
  int grid = num_sms();
  if (grid > total_tiles) grid = total_tiles;
  int rc;
  if (swap) {
    rc = p.b_mn_major ? launch_igemm_kernel<kSwapVox, 1, true, true>(grid, smem_bytes, stream, mapA0, mapA1, mapB, p)
                      : launch_igemm_kernel<kSwapVox, 0, true, true>(grid, smem_bytes, stream, mapA0, mapA1, mapB, p);
  } else if (wide) {
    rc = p.b_mn_major ? launch_igemm_kernel<kWideN, 1, true>(grid, smem_bytes, stream, mapA0, mapA1, mapB, p)
                      : launch_igemm_kernel<kWideN, 0, true>(grid, smem_bytes, stream, mapA0, mapA1, mapB, p);
  } else switch (p.block_n * 2 + p.b_mn_major) {
    case 16 * 2: rc = launch_igemm_kernel<16, 0>(grid, smem_bytes, stream, mapA0, mapA1, mapB, p); break;
    case 32 * 2: rc = launch_igemm_kernel<32, 0>(grid, smem_bytes, stream, mapA0, mapA1, mapB, p); break;
    case 64 * 2: rc = launch_igemm_kernel<64, 0>(grid, smem_bytes, stream, mapA0, mapA1, mapB, p); break;
    case 128 * 2: rc = launch_igemm_kernel<128, 0>(grid, smem_bytes, stream, mapA0, mapA1, mapB, p); break;
    case 64 * 2 + 1: rc = launch_igemm_kernel<64, 1>(grid, smem_bytes, stream, mapA0, mapA1, mapB, p); break;
    case 128 * 2 + 1: rc = launch_igemm_kernel<128, 1>(grid, smem_bytes, stream, mapA0, mapA1, mapB, p); break;
    default: OG_REQUIRE(false, "conv3d: no kernel for block_n=%d", p.block_n);
  }
  if (rc != OG_OK) return rc;
  g_launches.fetch_add(1);
  if (p.splits > 1) {
    const long long per_sample = (long long)T * H * W * n_out;
    double* gs = finish_did_stats ? L.gn_sums : nullptr;
    const int vec = (n_out % 4 == 0) ? 4 : 1;
    long long bx = (per_sample / vec + 255) / 256;
    const long long cap = ((long long)num_sms() * 8 + N - 1) / N;
    if (bx > cap) bx = cap;
    if (bx < 1) bx = 1;
    dim3 grid((unsigned)bx, (unsigned)N);
    if (vec == 4)
      og_splitk_finish_kernel<4><<<grid, 256, 0, stream>>>(p.ws, p.ws_slab, p.splits, L.bias0, L.bias1, L.out, L.out_f32,
                                                            n_out, per_sample, gs);
    else
      og_splitk_finish_kernel<1><<<grid, 256, 0, stream>>>(p.ws, p.ws_slab, p.splits, L.bias0, L.bias1, L.out, L.out_f32,
                                                            n_out, per_sample, gs);
    OG_CHECK_CUDA(cudaGetLastError());
    g_launches.fetch_add(1);
  }
  // requested statistics that could not be fused: run the stand-alone pass on the stored output
  if (stats_pass) {
    int r = og_gn_stats(L.out, N, (int64_t)T * H * W, n_out, 1, L.gn_sums, (og_stream_t)stream);
    if (r != OG_OK) return r;
  }
  return OG_OK;
}

}  // namespace og

extern "C" int og_conv3d_fwd(const void* x0, int c0, int kt, int kh, int kw, int pt, int ph, int pw, const void* x1,
                             int c1, const void* w, int ldw, const float* bias0, const float* bias1,
                             const void* residual, void* out, int out_f32, int N, int T, int H, int W, int cout,
                             void* workspace, size_t workspace_bytes, double* gn_sums, og_stream_t stream) {
  using namespace og;
  OG_REQUIRE(x0 && w && out, "conv3d_fwd: null pointer");
  OG_REQUIRE(c0 > 0 && c0 % 64 == 0, "conv3d_fwd: c0=%d must be a positive multiple of 64", c0);
  OG_REQUIRE(!x1 || (c1 > 0 && c1 % 64 == 0), "conv3d_fwd: c1=%d must be a multiple of 64", c1);
  OG_REQUIRE(kt >= 1 && kh >= 1 && kw >= 1 && pt >= 0 && ph >= 0 && pw >= 0 && pt < kt && ph < kh && pw < kw,
             "conv3d_fwd: bad kernel/padding (%d,%d,%d)/(%d,%d,%d)", kt, kh, kw, pt, ph, pw);
  const int ktot = kt * kh * kw * c0 + (x1 ? c1 : 0);
  OG_REQUIRE(ldw >= ktot && ldw % 8 == 0, "conv3d_fwd: ldw=%d must be >= %d and a multiple of 8", ldw, ktot);
  OG_REQUIRE(!gn_sums || !out_f32, "conv3d_fwd: gn_sums needs a bf16 output (out_f32 = 0)");
  IgemmLaunch L;
  L.a0 = x0; L.c0 = c0; L.aT = T; L.aH = H; L.aW = W;
  L.a1 = x1; L.c1 = c1;
  L.segs[0] = make_seg(c0 / 64, kt, kh, kw, pt, ph, pw, +1);
  L.segs[1] = make_seg(c1 / 64, 1, 1, 1, 0, 0, 0, +1);
  L.nseg = x1 ? 2 : 1;
  L.w = w; L.ldw = ldw;
  L.bias0 = bias0; L.bias1 = bias1; L.residual = residual;
  L.out = out; L.out_f32 = out_f32;
  L.N = N; L.T = T; L.H = H; L.W = W; L.n_out = cout;
  L.workspace = workspace; L.workspace_bytes = workspace_bytes;
  L.gn_sums = gn_sums;
  return launch_igemm(L, (cudaStream_t)stream);
}

extern "C" int og_conv3d_dgrad(const void* dy, int cout, int w_rows, const void* w, int ldw, int k_off, int kt, int kh,
                               int kw, int pt, int ph, int pw, void* dx, int dx_f32, int N, int T, int H, int W,
                               int cin, void* workspace, size_t workspace_bytes, og_stream_t stream) {
  using namespace og;
  OG_REQUIRE(dy && w && dx, "conv3d_dgrad: null pointer");
  OG_REQUIRE(cout > 0 && cout % 64 == 0, "conv3d_dgrad: cout=%d must be a multiple of 64", cout);
  OG_REQUIRE(cin > 0 && cin % 64 == 0, "conv3d_dgrad: cin=%d must be a multiple of 64", cin);
  OG_REQUIRE(k_off % 8 == 0 && ldw % 8 == 0, "conv3d_dgrad: k_off/ldw must be multiples of 8");
  OG_REQUIRE(w_rows > 0 && w_rows <= cout, "conv3d_dgrad: w_rows=%d must be in (0, cout]", w_rows);
  OG_REQUIRE(kt >= 1 && kh >= 1 && kw >= 1 && pt >= 0 && ph >= 0 && pw >= 0 && pt < kt && ph < kh && pw < kw,
             "conv3d_dgrad: bad kernel/padding (%d,%d,%d)/(%d,%d,%d)", kt, kh, kw, pt, ph, pw);
  OG_REQUIRE(k_off >= 0, "conv3d_dgrad: k_off=%d must be >= 0", k_off);
  const long long kend = (long long)k_off + (long long)kt * kh * kw * cin;
  OG_REQUIRE(ldw >= kend, "conv3d_dgrad: ldw=%d must be >= k_off + kt*kh*kw*cin = %lld", ldw, kend);
  IgemmLaunch L;
  L.a0 = dy; L.c0 = cout; L.aT = T; L.aH = H; L.aW = W;
  L.segs[0] = make_seg(cout / 64, kt, kh, kw, pt, ph, pw, -1);
  L.nseg = 1;
  L.w = w; L.ldw = ldw; L.k_off = k_off; L.b_mn_major = 1; L.b_rows = w_rows; L.b_ntaps = kt * kh * kw;
  L.out = dx; L.out_f32 = dx_f32;
  L.N = N; L.T = T; L.H = H; L.W = W; L.n_out = cin;
  L.workspace = workspace; L.workspace_bytes = workspace_bytes;
  return launch_igemm(L, (cudaStream_t)stream);
}

// Output extent of a strided convolution; 0 when the padded input is shorter than the kernel (truncating division
// would give such an input one output where F.conv3d raises).
static int out_extent(int in, int pad_front, int pad_back, int k, int s) {
  const int span = in + pad_front + pad_back - k;
  return span < 0 ? 0 : span / s + 1;
}

// Strided CausalConv3d forward (SpaceTimeDownsample, genie/module/video.py:457-483; geometry video.py:154-164: time is
// padded at the FRONT only by pt = kt-1 + (1-st), space symmetrically by (k-1)//2), as the SAME implicit GEMM: the A
// box of a tap is a strided TMA box (element strides = the convolution strides). No im2col buffer.
extern "C" int og_conv3d_strided_fwd(const void* x, int cin, int kt, int kh, int kw, int st, int sh, int sw, int pt, int ph,
                                     int pw, const void* w, int ldw, const float* bias, void* out, int out_f32, int N, int T,
                                     int H, int W, int cout, og_stream_t stream) {
  using namespace og;
  OG_REQUIRE(x && w && out, "conv3d_strided_fwd: null pointer");
  OG_REQUIRE(cin > 0 && cin % 64 == 0, "conv3d_strided_fwd: cin=%d must be a positive multiple of 64", cin);
  OG_REQUIRE(kt >= 1 && kh >= 1 && kw >= 1 && st >= 1 && sh >= 1 && sw >= 1 && st <= 8 && sh <= 8 && sw <= 8 && pt >= 0 &&
                 ph >= 0 && pw >= 0, "conv3d_strided_fwd: bad kernel / stride / padding");
  OG_REQUIRE(ldw >= kt * kh * kw * cin && ldw % 8 == 0, "conv3d_strided_fwd: bad ldw=%d", ldw);
  OG_REQUIRE(N > 0 && T > 0 && H > 0 && W > 0, "conv3d_strided_fwd: extents must be positive");
  const int To = out_extent(T, pt, 0, kt, st), Ho = out_extent(H, ph, ph, kh, sh), Wo = out_extent(W, pw, pw, kw, sw);
  OG_REQUIRE(To >= 1 && Ho >= 1 && Wo >= 1, "conv3d_strided_fwd: empty output (padded input smaller than the kernel)");
  IgemmLaunch L;
  L.a0 = x; L.c0 = cin; L.aT = T; L.aH = H; L.aW = W;
  L.astride[0] = st; L.astride[1] = sh; L.astride[2] = sw;
  L.segs[0] = make_seg(cin / 64, kt, kh, kw, pt, ph, pw, +1);
  L.nseg = 1;
  L.w = w; L.ldw = ldw;
  L.bias0 = bias;
  L.out = out; L.out_f32 = out_f32;
  L.N = N; L.T = To; L.H = Ho; L.W = Wo; L.n_out = cout;
  return launch_igemm(L, (cudaStream_t)stream);
}

// Data gradient of the strided convolution, without col2im: input position i receives dy[(i + pad - tap) / s] only from
// the taps with tap == (i + pad) mod s, so the input grid splits into st*sh*sw residue classes, each of which is a
// stride-1 implicit GEMM over dy with its own tap subset whose output rows are stored at stride s into dx.
// dy: bf16 [N,To,Ho,Wo,cout] (cout % 64 == 0, zero padded by the caller; w_rows real rows); dx: bf16 [N,T,H,W,cin].
extern "C" int og_conv3d_strided_dgrad(const void* dy, int cout, int w_rows, const void* w, int ldw, int kt, int kh, int kw,
                                       int st, int sh, int sw, int pt, int ph, int pw, void* dx, int N, int T, int H, int W,
                                       int cin, og_stream_t stream) {
  using namespace og;
  OG_REQUIRE(dy && w && dx, "conv3d_strided_dgrad: null pointer");
  OG_REQUIRE(cout > 0 && cout % 64 == 0 && cin > 0 && cin % 64 == 0, "conv3d_strided_dgrad: channels must be multiples of 64");
  OG_REQUIRE(w_rows > 0 && w_rows <= cout && ldw % 8 == 0 && ldw >= kt * kh * kw * cin,
             "conv3d_strided_dgrad: bad w_rows / ldw");
  OG_REQUIRE(kt >= 1 && kh >= 1 && kw >= 1 && st >= 1 && sh >= 1 && sw >= 1 && st <= 8 && sh <= 8 && sw <= 8 && pt >= 0 &&
                 ph >= 0 && pw >= 0, "conv3d_strided_dgrad: bad kernel / stride / padding");
  // checked before the memset below, whose size they give
  OG_REQUIRE(N > 0 && T > 0 && H > 0 && W > 0, "conv3d_strided_dgrad: extents must be positive");
  const int To = out_extent(T, pt, 0, kt, st), Ho = out_extent(H, ph, ph, kh, sh), Wo = out_extent(W, pw, pw, kw, sw);
  OG_REQUIRE(To >= 1 && Ho >= 1 && Wo >= 1, "conv3d_strided_dgrad: empty output (padded input smaller than the kernel)");
  const int k[3] = {kt, kh, kw}, s[3] = {st, sh, sw}, pd[3] = {pt, ph, pw}, in[3] = {T, H, W};
  bool any_empty = false;
  for (int d = 0; d < 3; ++d)
    if (k[d] < s[d]) any_empty = true;   // some residue classes have no tap: their rows of dx are zero
  if (any_empty) OG_CHECK_CUDA(cudaMemsetAsync(dx, 0, (size_t)N * T * H * W * cin * 2, (cudaStream_t)stream));
  for (int ct = 0; ct < st; ++ct)
    for (int ch = 0; ch < sh; ++ch)
      for (int cw = 0; cw < sw; ++cw) {
        const int cls[3] = {ct, ch, cw};
        IgemmLaunch L;
        L.segs[0].cin_blocks = cout / 64;
        L.segs[0].kh = kh;
        L.segs[0].kw = kw;
        int grid[3];
        bool empty = false;
        for (int d = 0; d < 3; ++d) {
          // class c: input positions i with (i + pad) mod s == c, i.e. i = s*a + r, r = (c - pad) mod s (>= 0)
          const int r = ((cls[d] - pd[d]) % s[d] + s[d]) % s[d];
          const int ntap = cls[d] < k[d] ? (k[d] - 1 - cls[d]) / s[d] + 1 : 0;
          grid[d] = in[d] > r ? (in[d] - r + s[d] - 1) / s[d] : 0;
          if (ntap == 0 || grid[d] == 0) empty = true;
          L.segs[0].n[d] = ntap;
          L.segs[0].tap0[d] = cls[d];
          L.segs[0].tstep[d] = s[d];
          L.segs[0].sh0[d] = (r + pd[d] - cls[d]) / s[d];   // exact: r + pad - c is a multiple of s
          L.segs[0].shstep[d] = -1;
          L.om[d] = s[d];
          L.oo[d] = r;
        }
        if (empty) continue;
        L.a0 = dy; L.c0 = cout; L.aT = To; L.aH = Ho; L.aW = Wo;
        L.nseg = 1;
        L.w = w; L.ldw = ldw; L.b_mn_major = 1; L.b_rows = w_rows; L.b_ntaps = kt * kh * kw;
        L.out = dx; L.out_f32 = 0;
        L.N = N; L.T = grid[0]; L.H = grid[1]; L.W = grid[2]; L.n_out = cin;
        L.OT = T; L.OH = H; L.OW = W;
        int rc = launch_igemm(L, (cudaStream_t)stream);
        if (rc != OG_OK) return rc;
      }
  return OG_OK;
}
