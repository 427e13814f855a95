// flash_attn.cu — spatial multi-head attention (non-causal, and causal below), FlashAttention-style, on the Hopper tensor cores (wgmma).
//
// Reference: F.scaled_dot_product_attention(q, k, v, scale = n_head * d_head**-0.5) reached from
// SpatialAttention.forward -> Attention.forward (genie/module/attention.py:279-307, 199-239), with
// q = k = v = LayerNorm(RoPE(x)) in the HEAD-valid configuration. Layout: [nseq][S][C] bf16 rows
// (one sequence = the H*W tokens of one frame, contiguous in NDHWC), head h = columns [h*d, h*d+d), d = 16, 64 or 128.
//
// Every kernel is one warpgroup (128 threads) owning a 64-row tile; thread 0 streams the other operand's 64-row tiles
// through a two-stage TMA ring (rows beyond S are zero-filled by TMA and masked). Accumulators live in registers in the
// wgmma fragment layout (og_ptx.cuh): a thread holds two rows, r0 = 16*warp + lane/4 and r0 + 8.
//
// Forward, one CTA per (sequence, head, 64-query tile), loop over 64-key tiles:
//   S  = Q K^T           wgmma, A = Q tile (K-major smem), B = K tile (K-major smem)
//   P  = exp(S*scale - m) online max / sum in registers (base 2 with the scale folded in)
//   O  = O*alpha + P V    wgmma, A = P straight from the S registers (bf16), B = V tile (MN-major: keys are the K dim)
// Backward recomputes P from the saved log-sum-exp in two passes, both recomputing S and dP = dO V^T:
//   MODE 0: one CTA per key tile j, streams the query tiles i, computes the transposed scores S^T = K Q^T and
//             dV_j += P^T dO_i,  dK_j += dS^T Q_i        (A = P^T / dS^T from registers, B = dO_i / Q_i MN-major)
//   MODE 1: one CTA per query tile i, streams the key tiles j:
//             dQ_i += dS K_j                             (A = dS from registers, B = K_j MN-major)
// with P = exp(S*scale - lse), dS = P * (dP - delta) * scale, delta = rowsum(dO * O).
// No atomics, no fp32 gradient buffers; outputs are bf16 in the activation layout.
//
// d_head = 128 (og_flash_attn_fwd_d128_kernel, og_flash_attn_bwd_d128_kernel<MODE>, og_attn_delta_d128_kernel): the
// same kernel bodies (flash_fwd / flash_bwd, templated on kH = d / 64). A 64 x 128 tile is two 64 x 64 half-tiles of
// the 128-byte swizzle, 8 KiB apart, each its own TMA box (a SWIZZLE_128B box is at most 64 bf16 wide) on the same
// mbarrier. The K-major score GEMMs walk 8 k16 slices, slices 4-7 from the second half. The MN-major B operands
// (V in P V, dO and Q in MODE 0, K in MODE 1) are taken one half at a time: one m64n64k16 per half and slice into its
// own m64n64 accumulator, through the same gemm_acc / descriptor as d = 64. That keeps one descriptor form for both
// widths and lets MODE 0 split the head columns between warpgroups; the issue count equals one m64n128k16 per slice
// with the atom stride in the descriptor.
//   forward: O as two m64n64 fragments (64 registers); smem Q + 2 x (K, V) = 80 KiB.
//   MODE 0: two warpgroups (256 threads) per key tile. Both compute the full S^T and dP^T (contracting over all 128
//           dims: the score GEMMs run twice), warpgroup w keeps dV and dK for head columns [64w, 64w + 64), so a
//           thread holds 2 x 32 accumulators as at d = 64. smem 2 + 2 x 2 tiles = 96 KiB.
//   MODE 1: one warpgroup, dQ as two m64n64 fragments.
//
// d_head = 16 (og_flash_attn_fwd_d16_kernel, og_flash_attn_bwd_d16_kernel<MODE>, og_attn_delta_d16_kernel): the same
// bodies at kDh = 16. A 64 x 16 tile is one 32-byte-wide TMA box with the 32-byte swizzle (2 KiB), read through
// gmma_desc_sw32: K-major for the score GEMMs (one k16 slice, 8-row groups 256 B apart), MN-major for the products
// with a register A operand, which issue m64n16k16 (wgmma_rs_n16; 8-row k groups 256 B apart, 512 B per k16 slice).
// The score tile is still m64n64, so the softmax is that of d = 64; O, dV, dK and dQ are one m64n16 fragment
// (8 registers). smem: forward 11 KiB, backward 13 KiB. The exponentials, not the MMAs, bound these kernels (one ex2
// per 64 MMA FLOP forward).
// Registers (nvcc 12.9, -O3, sm_90a; no spills): d = 64: fwd 98, MODE 0 168, MODE 1 122; d = 128: fwd 130,
// MODE 0 175 (256 threads), MODE 1 154; d = 16: fwd 66, MODE 0 128, MODE 1 98, delta 32.
//
// Dropout (og_flash_attn_dropout_fwd_kernel<d>, og_flash_attn_dropout_bwd_kernel<MODE, d>): the same bodies with kDrop
// set; the mask is attn_dropout.cuh's. The forward keeps the row max and sum of the undropped P (the lse it writes is
// the undropped one), zeroes the dropped P before P V and applies 1 / (1 - p) with 1 / l. MODE 0 feeds P Z^T to dV
// (1 / (1 - p) at the store) and masks dP^T; MODE 1 masks dP; the delta kernels are unchanged (O is the dropped output).
// With kDrop off the kernels are instruction-identical to those before dropout. Registers (no spills): d = 16: fwd 72,
// MODE 0 126, MODE 1 117; d = 64: fwd 130, MODE 0 182, MODE 1 154; d = 128: fwd 128, MODE 0 195, MODE 1 198.
//
// Causal (og_flash_attn_causal_fwd_kernel<d, drop>, og_flash_attn_causal_bwd_kernel<MODE, d, drop>; SDPA
// is_causal=True, key j <= query i): the same bodies with kCausal set. The forward and MODE 1 (query tile i) walk key
// tiles 0 .. i, MODE 0 (key tile j) walks query tiles j .. tiles - 1; the diagonal tile masks key > query (-inf in the
// forward, P = 0 in the backward) on top of the ragged-S mask. Dropout, when set, applies to what the causal mask keeps
// (the Philox mask is unchanged); the delta kernels are unchanged. Query tile i costs i + 1 key tiles, so blockIdx maps
// the longest items first: qt descending (forward, MODE 1) or j ascending (MODE 0) as the slowest index, (sequence,
// head) the fastest. With kCausal off the kernels are instruction-identical to those before the flag. Registers (no
// spills), without / with dropout: d = 16: fwd 66 / 72, MODE 0 106 / 152, MODE 1 98 / 130; d = 64: fwd 98 / 130,
// MODE 0 154 / 204, MODE 1 122 / 152; d = 128: fwd 138 / 130, MODE 0 160 / 207 (256 threads), MODE 1 154 / 220.
#include "og_host.cuh"
#include "og_ptx.cuh"
#include "attn_dropout.cuh"

namespace og {
extern std::atomic<uint64_t> g_launches;

static constexpr int kD = 64;            // width of one 64-column half of a head (the whole head at d_head = 64)
static constexpr int kTile = 64;         // rows per tile (queries or keys)
static constexpr int kTileBytes = kTile * kD * 2;  // 8 KiB: one 64 x 64 swizzled half-tile
static constexpr int kFaThreads = 128;

struct FaParams {
  int S, C, nh, nseq;
  int q_tiles, kv_tiles;
  float scale;
  __nv_bfloat16* out;  // [nseq][S][C]
  float* lse;          // [nseq][nh][S]
  const __nv_bfloat16* res;  // optional residual: out_res = attn + res (x = attn(x) + x, attention.py:470)
  __nv_bfloat16* out_res;
};

struct FaBwdParams {
  int S, C, nh, nseq, tiles;
  float scale;
  const float* lse;    // [nseq][nh][S]
  const float* delta;  // [nseq][nh][S]
  __nv_bfloat16* dq;
  __nv_bfloat16* dk;
  __nv_bfloat16* dv;
};

// S-fragment (m64n64 fp32) -> the bf16 A operand of the next wgmma, one k16 slice per kk (og_ptx.cuh layouts: the
// accumulator columns 16kk..16kk+15 of a thread's two rows are exactly its A fragment of that slice)
__device__ __forceinline__ void frag_to_a(const float (&x)[32], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    a[kk][0] = pack_bf16x2(x[8 * kk], x[8 * kk + 1]);
    a[kk][1] = pack_bf16x2(x[8 * kk + 2], x[8 * kk + 3]);
    a[kk][2] = pack_bf16x2(x[8 * kk + 4], x[8 * kk + 5]);
    a[kk][3] = pack_bf16x2(x[8 * kk + 6], x[8 * kk + 7]);
  }
}

// Geometry at head width kDh. d = 64, 128: kH 64-column halves with the 128-byte swizzle, outputs as kH m64n64
// fragments. d = 16: one 64 x 16 tile with the 32-byte swizzle (2 KiB), outputs as one m64n16 fragment.
template <int kDh>
struct FaGeo {
  static constexpr int kH = kDh >= kD ? kDh / kD : 1;   // accumulator fragments per output
  static constexpr int kN = kDh >= kD ? kD : kDh;       // fragment width (N of the MN-major products)
  static constexpr int kR = kN / 2;                     // fp32 registers per fragment and thread
  static constexpr int kTB = kTile * kDh * 2;           // one 64-row tile
};

// D = X Y^T over the kDh head dims, both tiles K-major. d = 64, 128: kH half-tiles [64 rows][64 d] with the 128-byte
// swizzle, kTileBytes apart (k16 slices 4c .. 4c + 3 come from half c). d = 16: one k16 slice of 32-byte rows.
template <int kDh>
__device__ __forceinline__ void gemm_rows(float (&d)[32], uint32_t x_addr, uint32_t y_addr) {
  if constexpr (kDh == 16) {
    wgmma_ss<64, 0, 0>(d, gmma_desc_sw32(x_addr, 16, 256), gmma_desc_sw32(y_addr, 16, 256), 0);
  } else {
    constexpr int kH = kDh / kD;
#pragma unroll
    for (int c = 0; c < kH; ++c)
#pragma unroll
      for (int k = 0; k < kD / 16; ++k)
        wgmma_ss<64, 0, 0>(d, gmma_desc_sw128(x_addr + c * kTileBytes + k * 32, 16, 1024),
                           gmma_desc_sw128(y_addr + c * kTileBytes + k * 32, 16, 1024), c > 0 || k > 0);
  }
}

// D += A Y: A from registers (64 rows x 64 k), Y a [64 k rows][kN d] tile read MN-major: a 64-wide half-tile with the
// 128-byte swizzle (m64n64k16), or a 16-wide tile with the 32-byte swizzle (m64n16k16, 512 B per k16 slice)
template <int kN>
__device__ __forceinline__ void gemm_acc(float (&d)[kN / 2], const uint32_t (&a)[4][4], uint32_t y_addr) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    if constexpr (kN == 16)
      wgmma_rs_n16<1>(d, a[kk], gmma_desc_sw32(y_addr + kk * 512, 2048, 256), 1);
    else
      wgmma_rs_n64<1>(d, a[kk], gmma_desc_sw128(y_addr + kk * 2048, 8192, 1024), 1);
  }
}

// 64 x kN fragment (times `sc`) -> bf16 rows of [nseq][S][C] (rows >= S dropped)
template <int kN>
__device__ __forceinline__ void store_frag(const float (&d)[kN / 2], float sc, __nv_bfloat16* base, long long row0,
                                           int S, int row_in_seq0, int C) {
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int r = warp * 16 + (lane >> 2) + rr * 8;
    if (row_in_seq0 + r >= S) continue;
    __nv_bfloat16* dst = base + (row0 + r) * C + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < kN / 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(d[4 * j + 2 * rr] * sc, d[4 * j + 2 * rr + 1] * sc);
  }
}

// rows row0 .. row0 + 63, head columns [h kDh, h kDh + kDh) of one sequence -> kH half-tiles, or one 16-wide tile
template <int kDh>
__device__ __forceinline__ void load_rows(uint8_t* dst, const CUtensorMap* map, uint64_t* bar, int h, int row0, int seq) {
  if constexpr (kDh == 16) {
    tma_load_3d(dst, map, bar, h * kDh, row0, seq);
  } else {
    constexpr int kH = kDh / kD;
#pragma unroll
    for (int c = 0; c < kH; ++c) tma_load_3d(dst + c * kTileBytes, map, bar, (h * kH + c) * kD, row0, seq);
  }
}

// Forward of one (sequence, head, 64-query tile) at head width kDh; O as kH fragments of 64 x kN.
template <int kDh, bool kDrop = false, bool kCausal = false>
__device__ __forceinline__ void flash_fwd(const CUtensorMap* mapQ, const CUtensorMap* mapK, const CUtensorMap* mapV,
                                          const FaParams& p, const DropParams* dr = nullptr) {
  using G = FaGeo<kDh>;
  constexpr int kTB = G::kTB, kH = G::kH, kN = G::kN, kR = G::kR;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                   // 1 tile
  uint8_t* sKV = smem + kTB;            // 2 stages x (K, V)
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + 4 * kTB);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;  // [2]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  int id = blockIdx.x;
  int qt;
  if constexpr (kCausal) {   // query tile qt reads qt + 1 key tiles: the longest are scheduled first
    const int nsh = p.nh * p.nseq;
    qt = p.q_tiles - 1 - id / nsh;
    id %= nsh;
  } else {
    qt = id % p.q_tiles;
    id /= p.q_tiles;
  }
  const int h = id % p.nh;
  const int seq = id / p.nh;
  const int q0 = qt * kTile;
  const int n_kv = kCausal ? qt + 1 : p.kv_tiles;   // key tiles 0 .. n_kv - 1

  if (tid == 0) {
    tma_prefetch_desc(mapQ);
    tma_prefetch_desc(mapK);
    tma_prefetch_desc(mapV);
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1);
    mbar_init(&kv_full[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(q_full, kTB);
    load_rows<kDh>(sQ, mapQ, q_full, h, q0, seq);
    for (int j = 0; j < 2 && j < n_kv; ++j) {
      mbar_expect_tx(&kv_full[j], 2 * kTB);
      load_rows<kDh>(sKV + j * 2 * kTB, mapK, &kv_full[j], h, j * kTile, seq);
      load_rows<kDh>(sKV + j * 2 * kTB + kTB, mapV, &kv_full[j], h, j * kTile, seq);
    }
  }
  // Online softmax in base 2 with the scale folded in: p = 2^(s*c - m), c = scale*log2(e). l is a per-thread partial
  // row sum (the quad's four partial sums are added once at the end).
  const float cl2 = p.scale * 1.4426950408889634f;
  float o[kH][kR];
#pragma unroll
  for (int c = 0; c < kH; ++c)
#pragma unroll
    for (int i = 0; i < kR; ++i) o[c][i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const uint32_t q_addr = smem_u32(sQ);
  uint2 dkey;
  if constexpr (kDrop) dkey = drop_key(dr->seed);
  mbar_wait(q_full, 0);
  for (int j = 0; j < n_kv; ++j) {
    const int st = j & 1;
    mbar_wait(&kv_full[st], (j >> 1) & 1);
    const uint32_t k_addr = smem_u32(sKV + st * 2 * kTB), v_addr = k_addr + kTB;
    float s[32];
    wgmma_fence();
    gemm_rows<kDh>(s, q_addr, k_addr);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    const int kv_valid = p.S - j * kTile;  // keys of this tile that exist (>= 64 except for the last tile)
    if (kv_valid < kTile) {
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if ((i >> 2) * 8 + 2 * (lane & 3) + (i & 1) >= kv_valid) s[i] = -INFINITY;
    }
    if constexpr (kCausal) {   // the diagonal tile: keys after the query are out (key 0 stays in every row)
      if (j == qt) {
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if ((i >> 2) * 8 + 2 * (lane & 3) + (i & 1) > warp * 16 + (lane >> 2) + 8 * ((i >> 1) & 1)) s[i] = -INFINITY;
      }
    }
    float alpha[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      float mt = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) mt = fmaxf(mt, fmaxf(s[4 * jj + 2 * rr], s[4 * jj + 2 * rr + 1]));
      mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 1));
      mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 2));
      const float mn = fmaxf(m[rr], mt * cl2);  // scale > 0; every tile has a valid key, so mn is finite
      alpha[rr] = ex2_approx(m[rr] - mn);
      m[rr] = mn;
      float ls = 0.f;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 4 * jj + 2 * rr + e;
          s[i] = ex2_approx(fmaf(s[i], cl2, -mn));
          ls += s[i];
        }
      }
      l[rr] = l[rr] * alpha[rr] + ls;
    }
    if constexpr (kDrop) {   // l keeps the undropped sum; P V takes the kept probabilities (1 / (1 - p) at the end)
      const uint32_t keep = drop_keep_tile<false>(q0 + warp * 16 + (lane >> 2), j * kTile + 2 * (lane & 3),
                                                  (uint64_t)seq * p.nh + h, dkey, dr->thresh);
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (!((keep >> i) & 1u)) s[i] = 0.f;
    }
#pragma unroll
    for (int c = 0; c < kH; ++c)
#pragma unroll
      for (int i = 0; i < kR; ++i) o[c][i] *= alpha[(i >> 1) & 1];
    uint32_t a[4][4];
    frag_to_a(s, a);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < kH; ++c) gemm_acc<kN>(o[c], a, v_addr + c * kTileBytes);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < kH; ++c) reg_fence(o[c]);
    __syncthreads();  // every warp is done with stage st
    if (tid == 0 && j + 2 < n_kv) {
      mbar_expect_tx(&kv_full[st], 2 * kTB);
      load_rows<kDh>(sKV + st * 2 * kTB, mapK, &kv_full[st], h, (j + 2) * kTile, seq);
      load_rows<kDh>(sKV + st * 2 * kTB + kTB, mapV, &kv_full[st], h, (j + 2) * kTile, seq);
    }
  }
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    l[rr] += __shfl_xor_sync(0xffffffffu, l[rr], 1);
    l[rr] += __shfl_xor_sync(0xffffffffu, l[rr], 2);
  }
  float inv[2] = {1.f / l[0], 1.f / l[1]};
  if constexpr (kDrop) {
    inv[0] *= dr->rscale;
    inv[1] *= dr->rscale;
  }
#pragma unroll
  for (int c = 0; c < kH; ++c)
#pragma unroll
    for (int i = 0; i < kR; ++i) o[c][i] *= inv[(i >> 1) & 1];
  const long long row0 = (long long)seq * p.S + q0;
#pragma unroll
  for (int c = 0; c < kH; ++c) store_frag<kN>(o[c], 1.f, p.out + h * kDh + c * kD, row0, p.S, q0, p.C);
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int r = warp * 16 + (lane >> 2) + rr * 8;
    if (q0 + r >= p.S) continue;
    if (p.res) {  // second output: attention + residual, added in fp32 before the rounding
#pragma unroll
      for (int c = 0; c < kH; ++c) {
        const long long off = (row0 + r) * p.C + h * kDh + c * kD + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < kN / 8; ++j) {
          const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.res + off + 8 * j));
          *reinterpret_cast<uint32_t*>(p.out_res + off + 8 * j) =
              pack_bf16x2(o[c][4 * j + 2 * rr] + t.x, o[c][4 * j + 2 * rr + 1] + t.y);
        }
      }
    }
    if (p.lse && (lane & 3) == 0)
      p.lse[((long long)seq * p.nh + h) * p.S + q0 + r] = (m[rr] + __log2f(l[rr])) * 0.6931471805599453f;
  }
}

__global__ void __launch_bounds__(kFaThreads)
    og_flash_attn_fwd_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                             const __grid_constant__ CUtensorMap mapV, const FaParams p) {
  flash_fwd<64>(&mapQ, &mapK, &mapV, p);
}

__global__ void __launch_bounds__(kFaThreads)
    og_flash_attn_fwd_d128_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                                  const __grid_constant__ CUtensorMap mapV, const FaParams p) {
  flash_fwd<128>(&mapQ, &mapK, &mapV, p);
}

__global__ void __launch_bounds__(kFaThreads)
    og_flash_attn_fwd_d16_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                                 const __grid_constant__ CUtensorMap mapV, const FaParams p) {
  flash_fwd<16>(&mapQ, &mapK, &mapV, p);
}

// with attention dropout (attn_dropout.cuh), d_head = kDh
template <int kDh>
__global__ void __launch_bounds__(kFaThreads)
    og_flash_attn_dropout_fwd_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                                     const __grid_constant__ CUtensorMap mapV, const FaParams p, const DropParams d) {
  flash_fwd<kDh, true>(&mapQ, &mapK, &mapV, p, &d);
}

// causal (SDPA is_causal=True: key j <= query i), without (kDrop false) or with dropout, d_head = kDh
template <int kDh, bool kDrop>
__global__ void __launch_bounds__(kFaThreads)
    og_flash_attn_causal_fwd_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                                    const __grid_constant__ CUtensorMap mapV, const FaParams p, const DropParams d) {
  flash_fwd<kDh, kDrop, true>(&mapQ, &mapK, &mapV, p, &d);
}

// ------------------------------------------------------------------------------------------------
// backward (see the file header). The softmax scale is applied once per output element of dK / dQ, not per score.
// kH = d_head / 64 at d = 64, 128 (1 at d = 16). MODE 0 at kH = 2 runs two warpgroups: both compute the full S^T and
// dP^T (contracting over all 128 head dims), warpgroup w keeps dV and dK for head columns [64 w, 64 w + 64). MODE 1
// keeps dQ as kH fragments.
// ------------------------------------------------------------------------------------------------
template <int MODE, int kDh, bool kDrop = false, bool kCausal = false>
__device__ __forceinline__ void flash_bwd(const CUtensorMap* mapQ, const CUtensorMap* mapK, const CUtensorMap* mapV,
                                          const CUtensorMap* mapDO, const FaBwdParams& p,
                                          const DropParams* dr = nullptr) {
  using G = FaGeo<kDh>;
  constexpr int kTB = G::kTB, kH = G::kH, kN = G::kN, kR = G::kR;
  constexpr int kNA = MODE == 0 ? 1 : kH;   // accumulator fragments per thread and output
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sFix = smem;                    // stationary pair: MODE 0: K_j, V_j ; MODE 1: Q_i, dO_i   (2 tiles)
  uint8_t* sStr = smem + 2 * kTB;          // streamed pair, 2 stages x (2 tiles)
  uint64_t* bars = reinterpret_cast<uint64_t*>(sStr + 4 * kTB);
  uint64_t* fix_full = bars;
  uint64_t* str_full = bars + 1;   // [2]
  const CUtensorMap* mapF0 = MODE == 0 ? mapK : mapQ;
  const CUtensorMap* mapF1 = MODE == 0 ? mapV : mapDO;
  const CUtensorMap* mapS0 = MODE == 0 ? mapQ : mapK;
  const CUtensorMap* mapS1 = MODE == 0 ? mapDO : mapV;

  const int tid = threadIdx.x, warp = (tid >> 5) & 3, lane = tid & 31;
  const int wg = MODE == 0 && kH == 2 ? tid >> 7 : 0;   // MODE 0 at d_head 128: the head-column half this thread owns
  int id = blockIdx.x;
  int own;   // MODE 0: kv tile ; MODE 1: q tile
  if constexpr (kCausal) {   // the longest first: MODE 0 key tile j reads tiles - j query tiles, MODE 1 query tile i
    const int nsh = p.nh * p.nseq;   // reads i + 1 key tiles
    own = MODE == 0 ? id / nsh : p.tiles - 1 - id / nsh;
    id %= nsh;
  } else {
    own = id % p.tiles;
    id /= p.tiles;
  }
  // streamed tiles it0 .. it0 + n_it - 1 (causal: MODE 0 the query tiles i >= j, MODE 1 the key tiles j <= i)
  const int it0 = kCausal && MODE == 0 ? own : 0;
  const int n_it = !kCausal ? p.tiles : MODE == 0 ? p.tiles - own : own + 1;
  const int h = id % p.nh;
  const int seq = id / p.nh;
  const long long stat0 = ((long long)seq * p.nh + h) * p.S;   // lse / delta row of this (sequence, head)

  if (tid == 0) {
    tma_prefetch_desc(mapQ);
    tma_prefetch_desc(mapK);
    tma_prefetch_desc(mapV);
    tma_prefetch_desc(mapDO);
    mbar_init(fix_full, 1);
    mbar_init(&str_full[0], 1);
    mbar_init(&str_full[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(fix_full, 2 * kTB);
    load_rows<kDh>(sFix, mapF0, fix_full, h, own * kTile, seq);
    load_rows<kDh>(sFix + kTB, mapF1, fix_full, h, own * kTile, seq);
    for (int it = 0; it < 2 && it < n_it; ++it) {
      mbar_expect_tx(&str_full[it], 2 * kTB);
      load_rows<kDh>(sStr + it * 2 * kTB, mapS0, &str_full[it], h, (it0 + it) * kTile, seq);
      load_rows<kDh>(sStr + it * 2 * kTB + kTB, mapS1, &str_full[it], h, (it0 + it) * kTile, seq);
    }
  }
  const float cl2 = p.scale * 1.4426950408889634f;
  const int r_base = warp * 16 + (lane >> 2);   // fragment rows r_base, r_base + 8
  const int c_base = 2 * (lane & 3);            // fragment columns 8j + c_base + {0, 1}
  // MODE 1: rows are queries of the own tile -> per-row lse / delta, loaded once
  float lse_r[2] = {0.f, 0.f}, delta_r[2] = {0.f, 0.f};
  if (MODE == 1) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int qrow = own * kTile + r_base + rr * 8;
      if (qrow < p.S) {
        lse_r[rr] = p.lse[stat0 + qrow] * 1.4426950408889634f;
        delta_r[rr] = p.delta[stat0 + qrow];
      }
    }
  }
  float acc0[kNA][kR], acc1[kNA][kR];   // MODE 0: dV, dK (head columns of half wg) ; MODE 1: dQ (acc1 unused)
#pragma unroll
  for (int c = 0; c < kNA; ++c)
#pragma unroll
    for (int i = 0; i < kR; ++i) acc0[c][i] = acc1[c][i] = 0.f;
  const uint32_t f0 = smem_u32(sFix), f1 = f0 + kTB;
  uint2 dkey;
  if constexpr (kDrop) dkey = drop_key(dr->seed);
  mbar_wait(fix_full, 0);
  for (int it = 0; it < n_it; ++it) {
    const int st = it & 1;
    mbar_wait(&str_full[st], (it >> 1) & 1);
    const uint32_t s0 = smem_u32(sStr + st * 2 * kTB), s1 = s0 + kTB;
    // MODE 0: s = S^T = K Q^T, dp = dP^T = V dO^T (rows = keys, columns = queries)
    // MODE 1: s = S   = Q K^T, dp = dP   = dO V^T (rows = queries, columns = keys)
    float s[32], dp[32];
    wgmma_fence();
    gemm_rows<kDh>(s, f0, s0);
    gemm_rows<kDh>(dp, f1, s1);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    reg_fence(dp);
    const int row_tile = own, col_tile = it0 + it;
    const bool rows_full = (row_tile + 1) * kTile <= p.S, cols_full = (col_tile + 1) * kTile <= p.S;
    uint32_t keep = 0;   // dropout: MODE 0 holds S^T (rows are keys), MODE 1 holds S
    if constexpr (kDrop)
      keep = drop_keep_tile<MODE == 0>(row_tile * kTile + r_base, col_tile * kTile + c_base, (uint64_t)seq * p.nh + h,
                                       dkey, dr->thresh);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = col_tile * kTile + 8 * j + c_base + e;
        float lse2c = 0.f, deltac = 0.f;
        if (MODE == 0 && col < p.S) {   // columns are queries
          lse2c = p.lse[stat0 + col] * 1.4426950408889634f;
          deltac = p.delta[stat0 + col];
        }
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int i = 4 * j + 2 * rr + e;
          const float lse2 = MODE == 0 ? lse2c : lse_r[rr], dl = MODE == 0 ? deltac : delta_r[rr];
          float pv = ex2_approx(fmaf(s[i], cl2, -lse2));
          if (!(rows_full && cols_full)) {
            const int row = row_tile * kTile + r_base + rr * 8;
            if (row >= p.S || col >= p.S) pv = 0.f;
          }
          if constexpr (kCausal) {   // the diagonal tile: no key after the query (MODE 0 rows are keys)
            const int rl = r_base + rr * 8, cl = 8 * j + c_base + e;
            if (row_tile == col_tile && (MODE == 0 ? rl > cl : cl > rl)) pv = 0.f;
          }
          if constexpr (kDrop) {   // dV takes P~ = P Z (1 / (1 - p) at the store); dS = P (dP Z - delta)
            const bool kp = (keep >> i) & 1u;
            s[i] = kp ? pv : 0.f;
            dp[i] = pv * ((kp ? dp[i] * dr->rscale : 0.f) - dl);
          } else {
            s[i] = pv;
            dp[i] = pv * (dp[i] - dl);
          }
        }
      }
    }
    uint32_t a_p[4][4], a_ds[4][4];
    frag_to_a(dp, a_ds);
    wgmma_fence();
    if (MODE == 0) {
      frag_to_a(s, a_p);
      gemm_acc<kN>(acc0[0], a_p, s1 + wg * kTileBytes);    // dV_j += P^T dO_i
      gemm_acc<kN>(acc1[0], a_ds, s0 + wg * kTileBytes);   // dK_j += dS^T Q_i
    } else {
#pragma unroll
      for (int c = 0; c < kNA; ++c) gemm_acc<kN>(acc0[c], a_ds, s0 + c * kTileBytes);   // dQ_i += dS K_j
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < kNA; ++c) {
      reg_fence(acc0[c]);
      reg_fence(acc1[c]);
    }
    __syncthreads();  // every warp is done with stage st
    if (tid == 0 && it + 2 < n_it) {
      mbar_expect_tx(&str_full[st], 2 * kTB);
      load_rows<kDh>(sStr + st * 2 * kTB, mapS0, &str_full[st], h, (it0 + it + 2) * kTile, seq);
      load_rows<kDh>(sStr + st * 2 * kTB + kTB, mapS1, &str_full[st], h, (it0 + it + 2) * kTile, seq);
    }
  }
  const long long row0 = (long long)seq * p.S + own * kTile;
  if (MODE == 0) {
    if constexpr (kDrop)
      store_frag<kN>(acc0[0], dr->rscale, p.dv + h * kDh + wg * kD, row0, p.S, own * kTile, p.C);
    else
      store_frag<kN>(acc0[0], 1.f, p.dv + h * kDh + wg * kD, row0, p.S, own * kTile, p.C);
    store_frag<kN>(acc1[0], p.scale, p.dk + h * kDh + wg * kD, row0, p.S, own * kTile, p.C);
  } else {
#pragma unroll
    for (int c = 0; c < kNA; ++c)
      store_frag<kN>(acc0[c], p.scale, p.dq + h * kDh + c * kD, row0, p.S, own * kTile, p.C);
  }
}

template <int MODE>
__global__ void __launch_bounds__(kFaThreads)
    og_flash_attn_bwd_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                             const __grid_constant__ CUtensorMap mapV, const __grid_constant__ CUtensorMap mapDO,
                             const FaBwdParams p) {
  flash_bwd<MODE, 64>(&mapQ, &mapK, &mapV, &mapDO, p);
}

template <int MODE>
__global__ void __launch_bounds__(MODE == 0 ? 2 * kFaThreads : kFaThreads)
    og_flash_attn_bwd_d128_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                                  const __grid_constant__ CUtensorMap mapV, const __grid_constant__ CUtensorMap mapDO,
                                  const FaBwdParams p) {
  flash_bwd<MODE, 128>(&mapQ, &mapK, &mapV, &mapDO, p);
}

template <int MODE>
__global__ void __launch_bounds__(kFaThreads)
    og_flash_attn_bwd_d16_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                                 const __grid_constant__ CUtensorMap mapV, const __grid_constant__ CUtensorMap mapDO,
                                 const FaBwdParams p) {
  flash_bwd<MODE, 16>(&mapQ, &mapK, &mapV, &mapDO, p);
}

template <int MODE, int kDh>
__global__ void __launch_bounds__(MODE == 0 && kDh == 128 ? 2 * kFaThreads : kFaThreads)
    og_flash_attn_dropout_bwd_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                                     const __grid_constant__ CUtensorMap mapV, const __grid_constant__ CUtensorMap mapDO,
                                     const FaBwdParams p, const DropParams d) {
  flash_bwd<MODE, kDh, true>(&mapQ, &mapK, &mapV, &mapDO, p, &d);
}

template <int MODE, int kDh, bool kDrop>
__global__ void __launch_bounds__(MODE == 0 && kDh == 128 ? 2 * kFaThreads : kFaThreads)
    og_flash_attn_causal_bwd_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                                    const __grid_constant__ CUtensorMap mapV, const __grid_constant__ CUtensorMap mapDO,
                                    const FaBwdParams p, const DropParams d) {
  flash_bwd<MODE, kDh, kDrop, true>(&mapQ, &mapK, &mapV, &mapDO, p, &d);
}

// delta[seq][h][s] = sum_d dO * O   (one warp per row, lanes over the head's 64 dims)
__global__ void og_attn_delta_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ d_o,
                                     float* __restrict__ delta, long long rows, int S, int C, int nh) {
  const int lane = threadIdx.x & 31;
  const long long w0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long t = w0; t < rows * nh; t += nw) {
    const int h = (int)(t % nh);
    const long long row = t / nh;
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(o + row * C + h * kD + lane * 2));
    const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(d_o + row * C + h * kD + lane * 2));
    float v = a.x * b.x + a.y * b.y;
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (lane == 0) delta[((row / S) * nh + h) * (long long)S + row % S] = v;
  }
}

// the same at d_head = 128: four consecutive dims per lane
__global__ void og_attn_delta_d128_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ d_o,
                                          float* __restrict__ delta, long long rows, int S, int C, int nh) {
  const int lane = threadIdx.x & 31;
  const long long w0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long t = w0; t < rows * nh; t += nw) {
    const int h = (int)(t % nh);
    const long long off = (t / nh) * C + h * 2 * kD + lane * 4;
    const uint2 ua = *reinterpret_cast<const uint2*>(o + off), ub = *reinterpret_cast<const uint2*>(d_o + off);
    const float2 a0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&ua.x));
    const float2 a1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&ua.y));
    const float2 b0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&ub.x));
    const float2 b1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&ub.y));
    float v = a0.x * b0.x + a0.y * b0.y + a1.x * b1.x + a1.y * b1.y;
    for (int off2 = 16; off2 > 0; off2 >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off2);
    const long long row = t / nh;
    if (lane == 0) delta[((row / S) * nh + h) * (long long)S + row % S] = v;
  }
}

// the same at d_head = 16: one thread per (row, head), its 16 dims as two 16-byte loads of each operand, summed in
// column order
__global__ void og_attn_delta_d16_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ d_o,
                                         float* __restrict__ delta, long long rows, int S, int C, int nh) {
  const long long n0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nt = (long long)gridDim.x * blockDim.x;
  for (long long t = n0; t < rows * nh; t += nt) {
    const int h = (int)(t % nh);
    const long long row = t / nh;
    const uint4* pa = reinterpret_cast<const uint4*>(o + row * C + h * 16);
    const uint4* pb = reinterpret_cast<const uint4*>(d_o + row * C + h * 16);
    float v = 0.f;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const uint4 ua = pa[c], ub = pb[c];
      const __nv_bfloat162* a2 = reinterpret_cast<const __nv_bfloat162*>(&ua);
      const __nv_bfloat162* b2 = reinterpret_cast<const __nv_bfloat162*>(&ub);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 a = __bfloat1622float2(a2[e]), b = __bfloat1622float2(b2[e]);
        v = fmaf(a.x, b.x, v);
        v = fmaf(a.y, b.y, v);
      }
    }
    delta[((row / S) * nh + h) * (long long)S + row % S] = v;
  }
}

// [nseq][S][C] rows; boxes of 64 rows by one 64-column half (128-byte swizzle) or, at d_head = 16, by one 16-column
// head (32-byte swizzle)
static int make_seq_map(CUtensorMap* m, const void* base, int nseq, int S, int C, int dh) {
  uint64_t dims[3] = {(uint64_t)C, (uint64_t)S, (uint64_t)nseq};
  uint64_t str[2] = {(uint64_t)C * 2, (uint64_t)S * C * 2};
  uint32_t box[3] = {dh == 16 ? 16u : (uint32_t)kD, kTile, 1};
  return make_tmap_bf16(m, base, 3, dims, str, box, nullptr,
                        dh == 16 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_128B);
}

}  // namespace og

using namespace og;

// d_head of C = n_head * d_head, or 0 when the head width has no kernel
static int flash_d_head(int C, int n_head) {
  if (n_head < 1) return 0;
  if (C == n_head * 64) return 64;
  if (C == n_head * 128) return 128;
  if (C == n_head * 16) return 16;
  return 0;
}

// the dropout kernels at d_head = kDh (shared memory as for the kernels without dropout)
template <int kDh>
static int flash_dropout_fwd_launch(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv,
                                    const FaParams& p, const DropParams& d, unsigned grid, cudaStream_t s) {
  const size_t smem_bytes = 5 * FaGeo<kDh>::kTB + 1024 + 64;
  static bool attr = false;
  if (!attr) {
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_flash_attn_dropout_fwd_kernel<kDh>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    attr = true;
  }
  og_flash_attn_dropout_fwd_kernel<kDh><<<grid, kFaThreads, smem_bytes, s>>>(mq, mk, mv, p, d);
  return OG_OK;
}

template <int kDh>
static int flash_dropout_bwd_launch(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv,
                                    const CUtensorMap& mdo, const FaBwdParams& p, const DropParams& d, unsigned grid,
                                    cudaStream_t s) {
  const size_t smem_bytes = 6 * FaGeo<kDh>::kTB + 1024 + 64;
  static bool attr = false;
  if (!attr) {
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_flash_attn_dropout_bwd_kernel<0, kDh>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_flash_attn_dropout_bwd_kernel<1, kDh>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    attr = true;
  }
  og_flash_attn_dropout_bwd_kernel<0, kDh><<<grid, kDh == 128 ? 2 * kFaThreads : kFaThreads, smem_bytes, s>>>(
      mq, mk, mv, mdo, p, d);
  OG_CHECK_CUDA(cudaGetLastError());
  og_flash_attn_dropout_bwd_kernel<1, kDh><<<grid, kFaThreads, smem_bytes, s>>>(mq, mk, mv, mdo, p, d);
  return OG_OK;
}

// the causal kernels at d_head = kDh, with dropout when `drop` is given (shared memory as without the mask)
template <int kDh>
static int flash_causal_fwd_launch(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv,
                                   const FaParams& p, const DropParams* drop, unsigned grid, cudaStream_t s) {
  const size_t smem_bytes = 5 * FaGeo<kDh>::kTB + 1024 + 64;
  static bool attr = false;
  if (!attr) {
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_flash_attn_causal_fwd_kernel<kDh, false>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_flash_attn_causal_fwd_kernel<kDh, true>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    attr = true;
  }
  if (drop)
    og_flash_attn_causal_fwd_kernel<kDh, true><<<grid, kFaThreads, smem_bytes, s>>>(mq, mk, mv, p, *drop);
  else
    og_flash_attn_causal_fwd_kernel<kDh, false><<<grid, kFaThreads, smem_bytes, s>>>(mq, mk, mv, p, DropParams{});
  return OG_OK;
}

template <int kDh, bool kDrop>
static int flash_causal_bwd_launch(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv,
                                   const CUtensorMap& mdo, const FaBwdParams& p, const DropParams& d, unsigned grid,
                                   cudaStream_t s) {
  const size_t smem_bytes = 6 * FaGeo<kDh>::kTB + 1024 + 64;
  static bool attr = false;
  if (!attr) {
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_flash_attn_causal_bwd_kernel<0, kDh, kDrop>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_flash_attn_causal_bwd_kernel<1, kDh, kDrop>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    attr = true;
  }
  og_flash_attn_causal_bwd_kernel<0, kDh, kDrop><<<grid, kDh == 128 ? 2 * kFaThreads : kFaThreads, smem_bytes, s>>>(
      mq, mk, mv, mdo, p, d);
  OG_CHECK_CUDA(cudaGetLastError());
  og_flash_attn_causal_bwd_kernel<1, kDh, kDrop><<<grid, kFaThreads, smem_bytes, s>>>(mq, mk, mv, mdo, p, d);
  return OG_OK;
}

template <int kDh>
static int flash_causal_bwd_launch(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv,
                                   const CUtensorMap& mdo, const FaBwdParams& p, const DropParams* drop, unsigned grid,
                                   cudaStream_t s) {
  return drop ? flash_causal_bwd_launch<kDh, true>(mq, mk, mv, mdo, p, *drop, grid, s)
              : flash_causal_bwd_launch<kDh, false>(mq, mk, mv, mdo, p, DropParams{}, grid, s);
}

// og_flash_attn_fwd, og_flash_attn_dropout_fwd when `drop` is given, og_flash_attn_causal_fwd when `causal` is set
static int flash_fwd_call(const void* q, const void* k, const void* v, void* out, const void* residual, void* out_res,
                          float* lse, int nseq, int S, int C, int n_head, float scale, const DropParams* drop,
                          og_stream_t stream, bool causal = false) {
  OG_REQUIRE(q && k && v && out, "flash_attn_fwd: null pointer");
  const int dh = flash_d_head(C, n_head);
  OG_REQUIRE(dh != 0, "flash_attn_fwd: needs d_head = 64, 128 or 16 (C=%d, n_head=%d)", C, n_head);
  OG_REQUIRE(nseq > 0 && S > 0, "flash_attn_fwd: empty problem");
  OG_REQUIRE(scale > 0.f, "flash_attn_fwd: scale must be positive (the row maximum is taken on raw scores)");
  FaParams p;
  p.S = S; p.C = C; p.nh = n_head; p.nseq = nseq;
  p.q_tiles = (S + kTile - 1) / kTile;
  p.kv_tiles = p.q_tiles;
  p.scale = scale;
  p.out = (__nv_bfloat16*)out;
  p.lse = lse;
  p.res = (const __nv_bfloat16*)residual;
  p.out_res = (__nv_bfloat16*)out_res;
  OG_REQUIRE(!residual || out_res, "flash_attn_fwd: residual given without out_res");
  CUtensorMap mq, mk, mv;
  int r;
  if ((r = make_seq_map(&mq, q, nseq, S, C, dh)) != OG_OK) return r;
  if ((r = make_seq_map(&mk, k, nseq, S, C, dh)) != OG_OK) return r;
  if ((r = make_seq_map(&mv, v, nseq, S, C, dh)) != OG_OK) return r;
  const long long grid = (long long)nseq * n_head * p.q_tiles;
  OG_REQUIRE(grid < (1LL << 31), "flash_attn_fwd: too many tiles");
  if (causal) {
    const int r2 = dh == 64    ? flash_causal_fwd_launch<64>(mq, mk, mv, p, drop, (unsigned)grid, (cudaStream_t)stream)
                   : dh == 128 ? flash_causal_fwd_launch<128>(mq, mk, mv, p, drop, (unsigned)grid, (cudaStream_t)stream)
                               : flash_causal_fwd_launch<16>(mq, mk, mv, p, drop, (unsigned)grid, (cudaStream_t)stream);
    if (r2 != OG_OK) return r2;
  } else if (drop) {
    const int r2 = dh == 64    ? flash_dropout_fwd_launch<64>(mq, mk, mv, p, *drop, (unsigned)grid, (cudaStream_t)stream)
                   : dh == 128 ? flash_dropout_fwd_launch<128>(mq, mk, mv, p, *drop, (unsigned)grid, (cudaStream_t)stream)
                               : flash_dropout_fwd_launch<16>(mq, mk, mv, p, *drop, (unsigned)grid, (cudaStream_t)stream);
    if (r2 != OG_OK) return r2;
  } else if (dh == 64) {
    const size_t smem_bytes = 5 * kTileBytes + 1024 + 64;
    static bool attr = false;
    if (!attr) {
      OG_CHECK_CUDA(cudaFuncSetAttribute(og_flash_attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem_bytes));
      attr = true;
    }
    og_flash_attn_fwd_kernel<<<(unsigned)grid, kFaThreads, smem_bytes, (cudaStream_t)stream>>>(mq, mk, mv, p);
  } else if (dh == 16) {
    const size_t smem_bytes = 5 * FaGeo<16>::kTB + 1024 + 64;   // Q, 2 x (K, V) at 2 KiB a tile
    og_flash_attn_fwd_d16_kernel<<<(unsigned)grid, kFaThreads, smem_bytes, (cudaStream_t)stream>>>(mq, mk, mv, p);
  } else {
    const size_t smem_bytes = 10 * kTileBytes + 1024 + 64;   // Q, 2 x (K, V) at 16 KiB a tile
    static bool attr = false;
    if (!attr) {
      OG_CHECK_CUDA(cudaFuncSetAttribute(og_flash_attn_fwd_d128_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem_bytes));
      attr = true;
    }
    og_flash_attn_fwd_d128_kernel<<<(unsigned)grid, kFaThreads, smem_bytes, (cudaStream_t)stream>>>(mq, mk, mv, p);
  }
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_flash_attn_fwd(const void* q, const void* k, const void* v, void* out, const void* residual,
                                 void* out_res, float* lse, int nseq, int S, int C, int n_head, float scale,
                                 og_stream_t stream) {
  return flash_fwd_call(q, k, v, out, residual, out_res, lse, nseq, S, C, n_head, scale, nullptr, stream);
}

extern "C" int og_flash_attn_dropout_fwd(const void* q, const void* k, const void* v, void* out, const void* residual,
                                         void* out_res, float* lse, int nseq, int S, int C, int n_head, float scale,
                                         float p, const uint64_t* seed, og_stream_t stream) {
  DropParams d;
  if (const int r = drop_params(p, seed, "flash_attn_dropout_fwd", &d)) return r;
  return flash_fwd_call(q, k, v, out, residual, out_res, lse, nseq, S, C, n_head, scale, &d, stream);
}

// og_flash_attn_bwd, og_flash_attn_dropout_bwd when `drop` is given, og_flash_attn_causal_bwd when `causal` is set
static int flash_bwd_call(const void* q, const void* k, const void* v, const void* out, const void* dout,
                          const float* lse, float* delta_ws, void* dq, void* dk, void* dv, int nseq, int S, int C,
                          int n_head, float scale, const DropParams* drop, og_stream_t stream, bool causal = false) {
  OG_REQUIRE(q && k && v && out && dout && lse && delta_ws && dq && dk && dv, "flash_attn_bwd: null pointer");
  const int dh = flash_d_head(C, n_head);
  OG_REQUIRE(dh != 0, "flash_attn_bwd: needs d_head = 64, 128 or 16 (C=%d, n_head=%d)", C, n_head);
  OG_REQUIRE(nseq > 0 && S > 0, "flash_attn_bwd: empty problem");
  OG_REQUIRE(scale > 0.f, "flash_attn_bwd: scale must be positive (as in the forward pass)");
  cudaStream_t s = (cudaStream_t)stream;
  const long long rows = (long long)nseq * S;
  {
    long long blocks = (rows * n_head + 7) / 8;
    if (blocks > (long long)num_sms() * 16) blocks = (long long)num_sms() * 16;
    if (dh == 64)
      og_attn_delta_kernel<<<(unsigned)blocks, 256, 0, s>>>((const __nv_bfloat16*)out, (const __nv_bfloat16*)dout,
                                                           delta_ws, rows, S, C, n_head);
    else if (dh == 16)
      og_attn_delta_d16_kernel<<<(unsigned)std::min((rows * n_head + 255) / 256, (long long)num_sms() * 16), 256, 0,
                                 s>>>(
          (const __nv_bfloat16*)out, (const __nv_bfloat16*)dout, delta_ws, rows, S, C, n_head);
    else
      og_attn_delta_d128_kernel<<<(unsigned)blocks, 256, 0, s>>>(
          (const __nv_bfloat16*)out, (const __nv_bfloat16*)dout, delta_ws, rows, S, C, n_head);
    OG_CHECK_CUDA(cudaGetLastError());
    g_launches.fetch_add(1);
  }
  FaBwdParams p;
  p.S = S; p.C = C; p.nh = n_head; p.nseq = nseq;
  p.tiles = (S + kTile - 1) / kTile;
  p.scale = scale;
  p.lse = lse;
  p.delta = delta_ws;
  p.dq = (__nv_bfloat16*)dq; p.dk = (__nv_bfloat16*)dk; p.dv = (__nv_bfloat16*)dv;
  CUtensorMap mq, mk, mv, mdo;
  int r;
  if ((r = make_seq_map(&mq, q, nseq, S, C, dh)) != OG_OK) return r;
  if ((r = make_seq_map(&mk, k, nseq, S, C, dh)) != OG_OK) return r;
  if ((r = make_seq_map(&mv, v, nseq, S, C, dh)) != OG_OK) return r;
  if ((r = make_seq_map(&mdo, dout, nseq, S, C, dh)) != OG_OK) return r;
  const long long grid = (long long)nseq * n_head * p.tiles;
  OG_REQUIRE(grid < (1LL << 31), "flash_attn_bwd: too many tiles");
  if (causal) {
    const int r2 = dh == 64    ? flash_causal_bwd_launch<64>(mq, mk, mv, mdo, p, drop, (unsigned)grid, s)
                   : dh == 128 ? flash_causal_bwd_launch<128>(mq, mk, mv, mdo, p, drop, (unsigned)grid, s)
                               : flash_causal_bwd_launch<16>(mq, mk, mv, mdo, p, drop, (unsigned)grid, s);
    if (r2 != OG_OK) return r2;
  } else if (drop) {
    const int r2 = dh == 64    ? flash_dropout_bwd_launch<64>(mq, mk, mv, mdo, p, *drop, (unsigned)grid, s)
                   : dh == 128 ? flash_dropout_bwd_launch<128>(mq, mk, mv, mdo, p, *drop, (unsigned)grid, s)
                               : flash_dropout_bwd_launch<16>(mq, mk, mv, mdo, p, *drop, (unsigned)grid, s);
    if (r2 != OG_OK) return r2;
  } else if (dh == 64) {
    const size_t smem_bytes = 6 * kTileBytes + 1024 + 64;
    static bool attr = false;
    if (!attr) {
      OG_CHECK_CUDA(cudaFuncSetAttribute(og_flash_attn_bwd_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem_bytes));
      OG_CHECK_CUDA(cudaFuncSetAttribute(og_flash_attn_bwd_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem_bytes));
      attr = true;
    }
    og_flash_attn_bwd_kernel<0><<<(unsigned)grid, kFaThreads, smem_bytes, s>>>(mq, mk, mv, mdo, p);
    OG_CHECK_CUDA(cudaGetLastError());
    og_flash_attn_bwd_kernel<1><<<(unsigned)grid, kFaThreads, smem_bytes, s>>>(mq, mk, mv, mdo, p);
  } else if (dh == 16) {
    const size_t smem_bytes = 6 * FaGeo<16>::kTB + 1024 + 64;   // 2 + 2 x 2 tiles of 2 KiB
    og_flash_attn_bwd_d16_kernel<0><<<(unsigned)grid, kFaThreads, smem_bytes, s>>>(mq, mk, mv, mdo, p);
    OG_CHECK_CUDA(cudaGetLastError());
    og_flash_attn_bwd_d16_kernel<1><<<(unsigned)grid, kFaThreads, smem_bytes, s>>>(mq, mk, mv, mdo, p);
  } else {
    const size_t smem_bytes = 12 * kTileBytes + 1024 + 64;   // 2 + 2 x 2 tiles of 16 KiB
    static bool attr = false;
    if (!attr) {
      OG_CHECK_CUDA(cudaFuncSetAttribute(og_flash_attn_bwd_d128_kernel<0>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
      OG_CHECK_CUDA(cudaFuncSetAttribute(og_flash_attn_bwd_d128_kernel<1>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
      attr = true;
    }
    og_flash_attn_bwd_d128_kernel<0><<<(unsigned)grid, 2 * kFaThreads, smem_bytes, s>>>(mq, mk, mv, mdo, p);
    OG_CHECK_CUDA(cudaGetLastError());
    og_flash_attn_bwd_d128_kernel<1><<<(unsigned)grid, kFaThreads, smem_bytes, s>>>(mq, mk, mv, mdo, p);
  }
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(2);
  return OG_OK;
}

extern "C" int og_flash_attn_bwd(const void* q, const void* k, const void* v, const void* out, const void* dout,
                                 const float* lse, float* delta_ws, void* dq, void* dk, void* dv, int nseq, int S,
                                 int C, int n_head, float scale, og_stream_t stream) {
  return flash_bwd_call(q, k, v, out, dout, lse, delta_ws, dq, dk, dv, nseq, S, C, n_head, scale, nullptr, stream);
}

extern "C" int og_flash_attn_dropout_bwd(const void* q, const void* k, const void* v, const void* out, const void* dout,
                                         const float* lse, float* delta_ws, void* dq, void* dk, void* dv, int nseq,
                                         int S, int C, int n_head, float scale, float p, const uint64_t* seed,
                                         og_stream_t stream) {
  DropParams d;
  if (const int r = drop_params(p, seed, "flash_attn_dropout_bwd", &d)) return r;
  return flash_bwd_call(q, k, v, out, dout, lse, delta_ws, dq, dk, dv, nseq, S, C, n_head, scale, &d, stream);
}

extern "C" int og_flash_attn_causal_fwd(const void* q, const void* k, const void* v, void* out, const void* residual,
                                        void* out_res, float* lse, int nseq, int S, int C, int n_head, float scale,
                                        float p, const uint64_t* seed, og_stream_t stream) {
  DropParams d;
  const DropParams* drop;
  if (const int r = drop_params_opt(p, seed, "flash_attn_causal_fwd", &d, &drop)) return r;
  return flash_fwd_call(q, k, v, out, residual, out_res, lse, nseq, S, C, n_head, scale, drop, stream, true);
}

extern "C" int og_flash_attn_causal_bwd(const void* q, const void* k, const void* v, const void* out, const void* dout,
                                        const float* lse, float* delta_ws, void* dq, void* dk, void* dv, int nseq,
                                        int S, int C, int n_head, float scale, float p, const uint64_t* seed,
                                        og_stream_t stream) {
  DropParams d;
  const DropParams* drop;
  if (const int r = drop_params_opt(p, seed, "flash_attn_causal_bwd", &d, &drop)) return r;
  return flash_bwd_call(q, k, v, out, dout, lse, delta_ws, dq, dk, dv, nseq, S, C, n_head, scale, drop, stream, true);
}
