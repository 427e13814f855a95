// temporal_attn_long.cu — temporal (causal or bidirectional, d_head = 16, 64 or 128) attention for clips of any length: FlashAttention-2
// on mma.sync m16n8k16, tiled over queries and keys, online softmax in fp32.
//
// STATUS: checked by tests/test_gpu_temporal_long.py (kernel level against float64 for T = 1 .. 1024, model level
// against the CPU oracle); ops._TimeAttnFn uses it for T > 32, the kernels of temporal_attn_mma.cu / attention_rows.cu
// keep T <= 32.
// SASS: LDGSTS / LDSM / HMMA.16816.F32.BF16.
//
// Reference semantics: as temporal_attn_mma.cu — SDPA(q, k, v, is_causal=True, scale) per pixel over t
// (genie/module/attention.py:347-371), K/V optionally (B, T, C) conditioning rows shared by all pixels (kv_bcast).
//
// Why mma.sync and not wgmma: one causal (pixel, head) sequence of T = 64 is ~0.5 MFLOP on ~32 KB of rows (~16 FLOP/B),
// far under the H100's ridge point; the work is moving rows, and 64 x 64 tiles of four independent warps (16 query or
// key rows each) need no warpgroup synchronisation. The fragment helpers are those of the T <= 16 kernels
// (temporal_mma_frag.cuh).
//
// Kernels (one CTA of 4 warps per 64-row tile of one (b, p, h) sequence; rows are 64-bit offsets
// ((b*T + t)*P + p)*C + h*64, so consecutive frames of a sequence are P*C elements apart):
//   og_temporal_attn_long_fwd_kernel      query tile i; key / value tiles j <= i through a double-buffered cp.async
//                                         ring (rows >= T zero-filled); only the diagonal tile is masked. P is rounded
//                                         to bf16 for P V. Writes out, optionally out_res = out + residual (added in
//                                         fp32, one rounding) and the fp32 log-sum-exp.
//   og_temporal_attn_long_bwd_dq_kernel   query tile i: delta = rowsum(dO * O) from the stored bf16 O (written to the
//                                         workspace for the next kernel), then dQ = sum_j dS_ij K_j over key tiles j <= i.
//   og_temporal_attn_long_bwd_dkdv_kernel key tile j: dV = sum_i P_ij^T dO_i, dK = sum_i dS_ij^T Q_i over query tiles
//                                         i >= j. With kv_bcast a CTA walks a contiguous chunk of the pixels of one
//                                         (b, h), accumulates in registers and adds the chunk into the fp32 outputs
//                                         with atomics.
// Both backward kernels recompute P = exp(scale * S - lse); dS = P (dP - delta). No atomics except the kv_bcast flush.
// Outputs are staged in shared memory and stored as whole row segments (128 bytes at D = 64).
//
// Head width D (template argument, 16, 64 or 128; ops._TimeAttnFn sends every T here at D = 16 and 128). Staged rows
// are 2D bytes plus 16 of padding (144 / 272 B, both an odd number of 16-byte units, so ldmatrix stays conflict free);
// tiles are 9 / 17 KiB, and shared memory at D = 128 is 85 KiB (forward), 119 KiB (dQ) and 103 KiB (dK / dV). The
// forward and dQ kernels keep their shape, with D / 8 n-tiles of accumulators per lane. The dK / dV kernel cannot hold
// dK and dV for 128 columns (16 rows x 128 columns x 2 = 128 accumulators per lane on top of S^T and dP^T): at D = 128 it runs 8
// warps, warps w and w + 4 own the same 16 key rows, both compute the full S^T and dP^T over the 128 dims, and each
// keeps dK / dV for one 64-column half, as at D = 64.
// At D = 16 rows are staged at a 48-byte pitch (3 x 16 B, conflict free as well) in 3 KiB tiles, a row leaves as two
// 16-byte chunks, the fp32 output staging exactly fills one ring stage, and the dK / dV kernel (4 warps) keeps two n8
// tiles of dK and dV per lane. Shared memory: 15 KiB (forward), 21 KiB (dQ), 19 KiB (dK / dV).
// Registers (nvcc 12.9, -O3, sm_90a; no spills): D = 64: fwd 128, dQ 167, dK/dV 230; D = 128: fwd 167, dQ 245,
// dK/dV 230 (256 threads); D = 16: fwd 72, dQ 94, dK/dV 135.
// Dropout (og_temporal_attn_long_dropout_{fwd,bwd_dq,bwd_dkdv}_kernel<D>): the same bodies with kDrop set, the mask of
// attn_dropout.cuh with sequence b * P + p (with kv_bcast too). The forward keeps the undropped row sum and lse; dQ
// masks dP; dK / dV takes P Z for dV (1 / (1 - p) at the store or the atomic flush) and masks dP^T. With kDrop off the
// kernels are instruction-identical to those before dropout. Registers (no spills): D = 16: fwd 78, dQ 127, dK/dV 168;
// D = 64: fwd 128, dQ 168, dK/dV 237; D = 128: fwd 168, dQ 240, dK/dV 238 (256 threads).
// Bidirectional (og_temporal_attn_bidir_{fwd,bwd_dq,bwd_dkdv}_kernel<D, drop>; SDPA is_causal=False over t, the
// reference TemporalAttention's default): the same bodies with kCausal off. The forward and dQ walk every key tile, dK /
// dV every query tile (also on the kv_bcast chunked path). Rows >= T are zero-filled, so a padded key would score 0,
// not -inf: the last key tile masks keys >= T explicitly (the causal kernels never reach them). Padded query rows need
// no mask in dK / dV: their Q, dO, lse and delta are zero-filled, so P^T dO and dS vanish there. With kCausal on the
// kernels are instruction-identical to those before the flag. Registers (no spills), without / with dropout: D = 16:
// fwd 72 / 80, dQ 92 / 128, dK/dV 80 / 128; D = 64: fwd 128 / 130, dQ 167 / 165, dK/dV 168 / 242; D = 128: fwd 167 /
// 168, dQ 246 / 233, dK/dV 234 / 254 (256 threads).
#include "og_host.cuh"
#include "og_ptx.cuh"
#include "temporal_mma_frag.cuh"
#include "attn_dropout.cuh"

namespace og {
extern std::atomic<uint64_t> g_launches;

namespace tlong {
using tmma::load_a;
using tmma::load_b_cols;
using tmma::load_b_rows;
using tmma::mma16816;
using tmma::pack_a;

constexpr int kTile = 64;                      // rows per query / key tile (16 per warp)
constexpr int kThreads = 128;
constexpr int kVecBytes = kTile * 4;           // 64 fp32 values (lse or delta of one query tile)
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// Shapes at head width D (16, 64 or 128)
template <int D>
struct Geo {
  static constexpr int kPitch = 2 * D + 16;            // staged bf16 row: 48 / 144 / 272 B (ldmatrix conflict free)
  static constexpr int kTileBytes = kTile * kPitch;    // one staged 64 x D tile: 3072 / 9216 / 17408 B
  static constexpr int kFPitch = 4 * D + 32;           // fp32 output staging row (float2 stores conflict free)
  static constexpr int kNT = D / 8;                    // 8-column n-tiles of a full-width fragment
  static constexpr int kDkdvThreads = D == 128 ? 256 : 128;  // dK / dV: one warp, or a warp pair, per 16 key rows
  static constexpr int kDkdvNT = D == 16 ? 2 : 8;      // dK / dV n-tiles a warp keeps (64 columns at D = 64, 128)
  static constexpr size_t kFwdSmem = 5 * (size_t)kTileBytes;                           // Q, 2 x (K, V)
  static constexpr size_t kDqSmem = 7 * (size_t)kTileBytes;                            // Q, dO, O, 2 x (K, V)
  static constexpr size_t kDkdvSmem = 6 * (size_t)kTileBytes + 4 * (size_t)kVecBytes;  // K, V, 2 x (Q, dO, lse, delta)
  static_assert(4 * 16 * kFPitch <= 2 * kTileBytes, "fp32 output staging must fit in one ring stage");
};

// 16- / 4-byte cp.async with zero fill: `valid` false reads nothing and writes zeros
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(valid ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// rows t0 .. t0+63 of a sequence (row pitch `pitch` elements) into a staged tile; rows >= T are zero.
// NTHR threads share the copy.
template <int D, int NTHR = kThreads>
__device__ __forceinline__ void load_tile(uint8_t* dst, const __nv_bfloat16* seq, long long pitch, int t0, int T,
                                          int tid) {
  constexpr int kCh = D / 8;   // 16-byte chunks per row
#pragma unroll
  for (int i = 0; i < kTile * kCh / NTHR; ++i) {
    const int idx = tid + NTHR * i, r = idx / kCh, ch = idx % kCh;
    const bool ok = t0 + r < T;
    cp_async16(smem_u32(dst + r * Geo<D>::kPitch + ch * 16), seq + (ok ? (long long)(t0 + r) * pitch : 0) + ch * 8,
               ok);
  }
}
// fp32 values t0 .. t0+63 of one sequence's lse / delta row; entries >= T are zero
__device__ __forceinline__ void load_vec(uint8_t* dst, const float* row, int t0, int T, int tid) {
  if (tid < kTile) {
    const bool ok = t0 + tid < T;
    cp_async4(smem_u32(dst + tid * 4), row + (ok ? t0 + tid : 0), ok);
  }
}

// acc = A_w B^T over the D head dims: A = 16 staged rows of this warp, B = the 64 rows of a staged tile
// (S = Q K^T, dP = dO V^T, S^T = K Q^T, dP^T = V dO^T); fragment [kc][half][.] covers columns 16 kc + 8 half ..
template <int D>
__device__ __forceinline__ void gemm_nt(float (&acc)[4][2][4], const uint8_t* a_rows, const uint8_t* b_rows, int lane) {
  constexpr int P = Geo<D>::kPitch;
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[c][hf][e] = 0.f;
#pragma unroll
  for (int kk = 0; kk < D / 16; ++kk) {
    uint32_t a[4];
    load_a<P>(a, a_rows, kk * 16, lane);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      uint32_t b[2];
      load_b_rows<P>(b, b_rows, nt * 8, kk * 16, lane);
      mma16816(acc[nt >> 1][nt & 1], a, b[0], b[1]);
    }
  }
}

// acc += X B: X = the 16 x 64 fragments `x` (rounded to bf16), B = columns n0 .. n0 + 8 NT - 1 of a staged 64-row
// tile whose rows are the k index (P V, dS K, P^T dO, dS^T Q)
template <int D, int NT>
__device__ __forceinline__ void gemm_nn_acc(float (&acc)[NT][4], const float (&x)[4][2][4], const uint8_t* b_tile,
                                            int n0, int lane) {
  constexpr int P = Geo<D>::kPitch;
#pragma unroll
  for (int kc = 0; kc < 4; ++kc) {
    uint32_t a[4];
    pack_a(a, x[kc]);
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      uint32_t b[2];
      load_b_cols<P>(b, b_tile + kc * 16 * P, n0 + nt * 8, lane);
      mma16816(acc[nt], a, b[0], b[1]);
    }
  }
}

// 16 x 8NT fp32 fragments (times sc0 / sc1 for rows g / g+8) as bf16 into columns n0 .. of a warp's 16 staged rows
template <int D, int NT>
__device__ __forceinline__ void frags_to_rows(uint8_t* rows, const float (&o)[NT][4], float sc0, float sc1, int n0,
                                              int lane) {
  constexpr int P = Geo<D>::kPitch;
  const int g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    *reinterpret_cast<uint32_t*>(rows + g * P + (n0 + nt * 8 + q * 2) * 2) = pack_bf16x2(o[nt][0] * sc0, o[nt][1] * sc0);
    *reinterpret_cast<uint32_t*>(rows + (g + 8) * P + (n0 + nt * 8 + q * 2) * 2) =
        pack_bf16x2(o[nt][2] * sc1, o[nt][3] * sc1);
  }
}
// 16-byte chunks ch0 .. ch0 + CH - 1 of a warp's 16 staged bf16 rows (sequence rows t0 ..) to global memory, rows >= T
// dropped
template <int D, int CH>
__device__ __forceinline__ void rows_to_global(const uint8_t* rows, __nv_bfloat16* seq, long long pitch, int t0, int T,
                                               int ch0, int lane) {
  constexpr int kRows = 32 / CH;   // rows per pass
#pragma unroll
  for (int it = 0; it < 16 / kRows; ++it) {
    const int r = lane / CH + kRows * it, ch = ch0 + lane % CH;
    if (t0 + r >= T) continue;
    *(reinterpret_cast<uint4*>(seq + (long long)(t0 + r) * pitch) + ch) =
        *reinterpret_cast<const uint4*>(rows + r * Geo<D>::kPitch + ch * 16);
  }
}

struct Seq {
  long long q0, k0, kpitch, task;
  int b, h;
};
// task = (b*nh + h)*P + p: the row of the lse / delta layout
__device__ __forceinline__ Seq decode(long long task, int T, long long P, int C, int nh, int D, int kv_bcast) {
  Seq s;
  s.task = task;
  const long long p = task % P, bh = task / P;
  s.h = (int)(bh % nh);
  s.b = (int)(bh / nh);
  s.q0 = ((long long)s.b * T * P + p) * C + (long long)s.h * D;
  s.k0 = kv_bcast ? (long long)s.b * T * C + (long long)s.h * D : s.q0;
  s.kpitch = kv_bcast ? (long long)C : P * C;
  return s;
}

// Kernel bodies, templated on the head width, on dropout (attn_dropout.cuh; without it they are the kernels as they
// were before dropout) and on the causal mask (kCausal false: bidirectional, every query sees all T keys). The
// __global__ wrappers follow each body.
template <int D, bool kDrop, bool kCausal = true>
__device__ __forceinline__ void long_fwd_body(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                     const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ res,
                                     __nv_bfloat16* __restrict__ out, __nv_bfloat16* __restrict__ out_res,
                                     float* __restrict__ lse, int B, int T, long long P, int C, int nh, float scale,
                                     int kv_bcast, int tiles, const DropParams* dr) {
  using G = Geo<D>;
  constexpr int kTileBytes = G::kTileBytes, kPitch = G::kPitch, kFPitch = G::kFPitch, kNT = G::kNT;
  extern __shared__ __align__(16) uint8_t smem_l[];
  uint8_t* qs = smem_l;
  uint8_t* ring = smem_l + kTileBytes;   // stage s: K at ring + 2 s kTileBytes, V right after
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, qd = lane & 3;
  const long long ntask = (long long)B * nh * P;
  const int i = tiles - 1 - (int)(blockIdx.x / ntask);   // the longest query tiles are scheduled first
  const Seq sq = decode(blockIdx.x % ntask, T, P, C, nh, D, kv_bcast);
  const long long qpitch = P * C;
  load_tile<D>(qs, q + sq.q0, qpitch, i * kTile, T, tid);
  load_tile<D>(ring, k + sq.k0, sq.kpitch, 0, T, tid);
  load_tile<D>(ring + kTileBytes, v + sq.k0, sq.kpitch, 0, T, tid);
  cp_async_commit();
  const float cl2 = scale * kLog2e;
  const int row0 = i * kTile + warp * 16 + g;   // this lane's query rows: row0, row0 + 8
  const uint8_t* qw = qs + warp * 16 * kPitch;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  uint2 dkey;
  uint64_t dz;
  if constexpr (kDrop) {
    dkey = drop_key(dr->seed);
    dz = ((uint64_t)sq.b * P + sq.task % P) * nh + sq.h;
  }
  float o[kNT][4];
#pragma unroll
  for (int nt = 0; nt < kNT; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[nt][e] = 0.f;
  const int jl = kCausal ? i : tiles - 1;   // the last key tile this query tile reads
  for (int j = 0; j <= jl; ++j) {
    cp_async_wait_all();
    __syncthreads();   // tile j has landed for every thread; every warp is done with tile j - 1
    if (j < jl) {
      uint8_t* nx = ring + ((j + 1) & 1) * 2 * kTileBytes;
      load_tile<D>(nx, k + sq.k0, sq.kpitch, (j + 1) * kTile, T, tid);
      load_tile<D>(nx + kTileBytes, v + sq.k0, sq.kpitch, (j + 1) * kTile, T, tid);
      cp_async_commit();
    }
    const uint8_t* ks = ring + (j & 1) * 2 * kTileBytes;
    float s[4][2][4];
    gemm_nt<D>(s, qw, ks, lane);
    // scores in the log2 domain; the diagonal tile masks keys after the query (bidirectional: the last tile masks the
    // zero-filled keys >= T, whose scores would be 0). Key 0 is in every row of tile 0, so the row maximum is finite
    // from the first tile on.
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int rr = e >> 1, col = j * kTile + nt * 8 + 2 * qd + (e & 1);
        float x = s[nt >> 1][nt & 1][e] * cl2;
        if (kCausal ? j == i && col > row0 + 8 * rr : j == jl && col >= T) x = -INFINITY;
        s[nt >> 1][nt & 1][e] = x;
        mx[rr] = fmaxf(mx[rr], x);
      }
    float alpha[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 1));
      mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 2));
      alpha[rr] = ex2_approx(m[rr] - mx[rr]);   // 0 on the first tile (m = -inf)
      m[rr] = mx[rr];
      l[rr] *= alpha[rr];
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int rr = e >> 1;
        const float p = ex2_approx(s[nt >> 1][nt & 1][e] - m[rr]);
        s[nt >> 1][nt & 1][e] = p;
        l[rr] += p;
      }
    if constexpr (kDrop) {   // l keeps the undropped sum; P V takes the kept probabilities (1 / (1 - p) at the end)
      const uint32_t keep = drop_keep_tile<false>(row0, j * kTile + 2 * qd, dz, dkey, dr->thresh);
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (!((keep >> (4 * nt + e)) & 1u)) s[nt >> 1][nt & 1][e] = 0.f;
    }
#pragma unroll
    for (int nt = 0; nt < kNT; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[nt][e] *= alpha[e >> 1];
    gemm_nn_acc<D, kNT>(o, s, ks + kTileBytes, 0, lane);
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
  // fp32 staging of the normalised output in the ring stage the loop no longer reads (its last tile, jl - 1, was
  // finished by every warp before the last barrier); each warp writes and reads only its own 16 rows
  uint8_t* st = ring + ((jl + 1) & 1) * 2 * kTileBytes + warp * 16 * kFPitch;
#pragma unroll
  for (int nt = 0; nt < kNT; ++nt)
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
      *reinterpret_cast<float2*>(st + (g + 8 * rr) * kFPitch + (nt * 8 + 2 * qd) * 4) =
          make_float2(o[nt][2 * rr] * inv[rr], o[nt][2 * rr + 1] * inv[rr]);
  __syncwarp();
  const int t_w = i * kTile + warp * 16;
  constexpr int kCh = D / 8, kRows = 32 / kCh;   // 8-column chunks per row, rows per pass
#pragma unroll
  for (int it = 0; it < 16 / kRows; ++it) {
    const int r = lane / kCh + kRows * it, ch = lane % kCh;
    if (t_w + r >= T) continue;
    const float4 a = *reinterpret_cast<const float4*>(st + r * kFPitch + ch * 32);
    const float4 c = *reinterpret_cast<const float4*>(st + r * kFPitch + ch * 32 + 16);
    const long long off = sq.q0 + (long long)(t_w + r) * qpitch + ch * 8;
    *reinterpret_cast<uint4*>(out + off) =
        make_uint4(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w), pack_bf16x2(c.x, c.y), pack_bf16x2(c.z, c.w));
    if (res) {   // second output: attention + residual, added in fp32 before the rounding
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(res + off));
      const __nv_bfloat162* rb = reinterpret_cast<const __nv_bfloat162*>(&u);
      const float2 r0 = __bfloat1622float2(rb[0]), r1 = __bfloat1622float2(rb[1]), r2 = __bfloat1622float2(rb[2]),
                   r3 = __bfloat1622float2(rb[3]);
      *reinterpret_cast<uint4*>(out_res + off) =
          make_uint4(pack_bf16x2(a.x + r0.x, a.y + r0.y), pack_bf16x2(a.z + r1.x, a.w + r1.y),
                     pack_bf16x2(c.x + r2.x, c.y + r2.y), pack_bf16x2(c.z + r3.x, c.w + r3.y));
    }
  }
  if (qd == 0) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
      if (row0 + 8 * rr < T) lse[sq.task * T + row0 + 8 * rr] = (m[rr] + __log2f(l[rr])) * kLn2;
  }
}

template <int D>
__global__ void __launch_bounds__(kThreads)
    og_temporal_attn_long_fwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                     const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ res,
                                     __nv_bfloat16* __restrict__ out, __nv_bfloat16* __restrict__ out_res,
                                     float* __restrict__ lse, int B, int T, long long P, int C, int nh, float scale,
                                     int kv_bcast, int tiles) {
  long_fwd_body<D, false>(q, k, v, res, out, out_res, lse, B, T, P, C, nh, scale, kv_bcast, tiles, nullptr);
}

template <int D>
__global__ void __launch_bounds__(kThreads)
    og_temporal_attn_long_dropout_fwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                     const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ res,
                                     __nv_bfloat16* __restrict__ out, __nv_bfloat16* __restrict__ out_res,
                                     float* __restrict__ lse, int B, int T, long long P, int C, int nh, float scale,
                                     int kv_bcast, int tiles, const DropParams d) {
  long_fwd_body<D, true>(q, k, v, res, out, out_res, lse, B, T, P, C, nh, scale, kv_bcast, tiles, &d);
}

template <int D, bool kDrop, bool kCausal = true>
__device__ __forceinline__ void long_dq_body(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                        const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ o,
                                        const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse,
                                        float* __restrict__ delta, __nv_bfloat16* __restrict__ dq, int B, int T,
                                        long long P, int C, int nh, float scale, int kv_bcast, int tiles, const DropParams* dr) {
  using G = Geo<D>;
  constexpr int kTileBytes = G::kTileBytes, kPitch = G::kPitch, kNT = G::kNT;
  extern __shared__ __align__(16) uint8_t smem_l[];
  uint8_t* qs = smem_l;
  uint8_t* dos = qs + kTileBytes;
  uint8_t* os = dos + kTileBytes;
  uint8_t* ring = os + kTileBytes;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, qd = lane & 3;
  const long long ntask = (long long)B * nh * P;
  const int i = tiles - 1 - (int)(blockIdx.x / ntask);
  const Seq sq = decode(blockIdx.x % ntask, T, P, C, nh, D, kv_bcast);
  const long long qpitch = P * C;
  load_tile<D>(qs, q + sq.q0, qpitch, i * kTile, T, tid);
  load_tile<D>(dos, dout + sq.q0, qpitch, i * kTile, T, tid);
  load_tile<D>(os, o + sq.q0, qpitch, i * kTile, T, tid);
  load_tile<D>(ring, k + sq.k0, sq.kpitch, 0, T, tid);
  load_tile<D>(ring + kTileBytes, v + sq.k0, sq.kpitch, 0, T, tid);
  cp_async_commit();
  const int t_w = i * kTile + warp * 16, row0 = t_w + g;
  const uint8_t* qw = qs + warp * 16 * kPitch;
  const uint8_t* dow = dos + warp * 16 * kPitch;
  // lse (log2 domain) of rows row0, row0 + 8; zero on rows >= T, whose Q and dO rows are zero: P stays finite there
  float lse2[2];
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) lse2[rr] = row0 + 8 * rr < T ? lse[sq.task * T + row0 + 8 * rr] * kLog2e : 0.f;
  cp_async_wait_all();
  __syncthreads();   // the rows of every tile are loaded by all four warps
  // delta = rowsum(dO * O) of this warp's rows: two lanes per row, D / 2 columns each
  float dsum;
  {
    const int r = lane >> 1, c0 = (lane & 1) * (D / 2);
    const uint8_t* dr = dow + r * kPitch + c0 * 2;
    const uint8_t* orow = os + (warp * 16 + r) * kPitch + c0 * 2;
    dsum = 0.f;
#pragma unroll
    for (int c = 0; c < D / 2; c += 2) {
      const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(dr + c * 2));
      const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(orow + c * 2));
      dsum = fmaf(a.x, b.x, dsum);
      dsum = fmaf(a.y, b.y, dsum);
    }
    dsum += __shfl_xor_sync(0xffffffffu, dsum, 1);
    if ((lane & 1) == 0 && t_w + r < T) delta[sq.task * T + t_w + r] = dsum;
  }
  const float dl[2] = {__shfl_sync(0xffffffffu, dsum, 2 * g), __shfl_sync(0xffffffffu, dsum, 2 * g + 16)};
  const float cl2 = scale * kLog2e;
  uint2 dkey;
  uint64_t dz;
  if constexpr (kDrop) {
    dkey = drop_key(dr->seed);
    dz = ((uint64_t)sq.b * P + sq.task % P) * nh + sq.h;
  }
  float acc[kNT][4];
#pragma unroll
  for (int nt = 0; nt < kNT; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[nt][e] = 0.f;
  const int jl = kCausal ? i : tiles - 1;
  for (int j = 0; j <= jl; ++j) {
    cp_async_wait_all();
    __syncthreads();
    if (j < jl) {
      uint8_t* nx = ring + ((j + 1) & 1) * 2 * kTileBytes;
      load_tile<D>(nx, k + sq.k0, sq.kpitch, (j + 1) * kTile, T, tid);
      load_tile<D>(nx + kTileBytes, v + sq.k0, sq.kpitch, (j + 1) * kTile, T, tid);
      cp_async_commit();
    }
    const uint8_t* ks = ring + (j & 1) * 2 * kTileBytes;
    const uint8_t* vs = ks + kTileBytes;
    float s[4][2][4], dp[4][2][4];
    gemm_nt<D>(s, qw, ks, lane);
    gemm_nt<D>(dp, dow, vs, lane);
    uint32_t keep = 0;
    if constexpr (kDrop) keep = drop_keep_tile<false>(row0, j * kTile + 2 * qd, dz, dkey, dr->thresh);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int rr = e >> 1, col = j * kTile + nt * 8 + 2 * qd + (e & 1);
        float p = ex2_approx(fmaf(s[nt >> 1][nt & 1][e], cl2, -lse2[rr]));
        // bidirectional: keys >= T are zero rows, with P = 2^-lse and dP = 0 they would add -P delta K
        if (kCausal ? j == i && col > row0 + 8 * rr : j == jl && col >= T) p = 0.f;
        if constexpr (kDrop) {   // dS = P (dP Z - delta)
          const float d = (keep >> (4 * nt + e)) & 1u ? dp[nt >> 1][nt & 1][e] * dr->rscale : 0.f;
          s[nt >> 1][nt & 1][e] = p * (d - dl[rr]);
        } else {
          s[nt >> 1][nt & 1][e] = p * (dp[nt >> 1][nt & 1][e] - dl[rr]);   // dS (without the scale)
        }
      }
    gemm_nn_acc<D, kNT>(acc, s, ks, 0, lane);
  }
  // dQ = scale * sum_j dS K_j; every read of this warp's Q rows is done, so they stage the output
  __syncwarp();
  uint8_t* qw_out = qs + warp * 16 * kPitch;
  frags_to_rows<D, kNT>(qw_out, acc, scale, scale, 0, lane);
  __syncwarp();
  rows_to_global<D, D / 8>(qw_out, dq + sq.q0, qpitch, t_w, T, 0, lane);
}

template <int D>
__global__ void __launch_bounds__(kThreads)
    og_temporal_attn_long_bwd_dq_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                        const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ o,
                                        const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse,
                                        float* __restrict__ delta, __nv_bfloat16* __restrict__ dq, int B, int T,
                                        long long P, int C, int nh, float scale, int kv_bcast, int tiles) {
  long_dq_body<D, false>(q, k, v, o, dout, lse, delta, dq, B, T, P, C, nh, scale, kv_bcast, tiles, nullptr);
}

template <int D>
__global__ void __launch_bounds__(kThreads)
    og_temporal_attn_long_dropout_bwd_dq_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                        const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ o,
                                        const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse,
                                        float* __restrict__ delta, __nv_bfloat16* __restrict__ dq, int B, int T,
                                        long long P, int C, int nh, float scale, int kv_bcast, int tiles, const DropParams d) {
  long_dq_body<D, true>(q, k, v, o, dout, lse, delta, dq, B, T, P, C, nh, scale, kv_bcast, tiles, &d);
}

// D = 64: warp w owns key rows 16 w .. 16 w + 15 and all 64 head columns of dK / dV.
// D = 128: eight warps; warps w and w + 4 own the same 16 key rows, each computes the full S^T and dP^T (over all 128
// dims) and keeps dK / dV for head columns [64 (w / 4), 64 (w / 4) + 64) only, so a lane holds 2 x 32 accumulators
// as at D = 64.
template <int D, bool kDrop, bool kCausal = true>
__device__ __forceinline__ void long_dkdv_body(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                          const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ dout,
                                          const float* __restrict__ lse, const float* __restrict__ delta,
                                          __nv_bfloat16* __restrict__ dk, __nv_bfloat16* __restrict__ dv,
                                          float* __restrict__ dk_b, float* __restrict__ dv_b, int B, int T,
                                          long long P, int C, int nh, float scale, int kv_bcast, int tiles,
                                          long long chunk, long long nchunk, const DropParams* dr) {
  using G = Geo<D>;
  constexpr int kTileBytes = G::kTileBytes, kPitch = G::kPitch, NTHR = G::kDkdvThreads;
  extern __shared__ __align__(16) uint8_t smem_l[];
  uint8_t* ks = smem_l;
  uint8_t* vs = ks + kTileBytes;
  uint8_t* ring = vs + kTileBytes;   // stage s: Q, dO, lse[64], delta[64]
  constexpr int kStage = 2 * kTileBytes + 2 * kVecBytes;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, qd = lane & 3;
  const int wr = warp & 3, half = warp >> 2;   // key-row group; head-column half (0 at D = 64)
  const int n0 = half * 64;
  const long long per_j = (long long)B * nh * nchunk;
  const int j = (int)(blockIdx.x / per_j);   // key tile; the longest (j = 0) are scheduled first
  const long long rest = blockIdx.x % per_j, bh = rest / nchunk;
  const long long p0 = (rest % nchunk) * chunk, p1 = p0 + chunk < P ? p0 + chunk : P;
  // query tiles i = i0 .. tiles - 1 per pixel: i0 = j, or 0 when bidirectional. Query rows >= T need no mask: their Q
  // and dO rows are zero-filled and so are their lse and delta, so P = 1 there but P^T dO = 0 and dS = 0.
  const int i0 = kCausal ? j : 0, nq = tiles - i0;
  const long long items = (p1 - p0) * nq;
  const Seq s0 = decode(bh * P + p0, T, P, C, nh, D, kv_bcast);
  const long long qpitch = P * C;
  auto load_item = [&](long long n, int stage) {
    const long long task = bh * P + p0 + n / nq;
    const int i = i0 + (int)(n % nq);
    const long long q0 = s0.q0 + (task - s0.task) * C;   // the pixels of one (b, h) are C elements apart
    uint8_t* st = ring + stage * kStage;
    load_tile<D, NTHR>(st, q + q0, qpitch, i * kTile, T, tid);
    load_tile<D, NTHR>(st + kTileBytes, dout + q0, qpitch, i * kTile, T, tid);
    load_vec(st + 2 * kTileBytes, lse + task * T, i * kTile, T, tid);
    load_vec(st + 2 * kTileBytes + kVecBytes, delta + task * T, i * kTile, T, tid);
  };
  load_tile<D, NTHR>(ks, k + s0.k0, s0.kpitch, j * kTile, T, tid);
  load_tile<D, NTHR>(vs, v + s0.k0, s0.kpitch, j * kTile, T, tid);
  load_item(0, 0);
  cp_async_commit();
  const float cl2 = scale * kLog2e;
  uint2 dkey;
  if constexpr (kDrop) dkey = drop_key(dr->seed);
  const int key0 = j * kTile + wr * 16 + g;   // this lane's key rows: key0, key0 + 8
  const uint8_t* kw = ks + wr * 16 * kPitch;
  const uint8_t* vw = vs + wr * 16 * kPitch;
  constexpr int kAN = G::kDkdvNT;
  float dka[kAN][4], dva[kAN][4];
#pragma unroll
  for (int nt = 0; nt < kAN; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) dka[nt][e] = dva[nt][e] = 0.f;
  for (long long n = 0; n < items; ++n) {
    cp_async_wait_all();
    __syncthreads();
    if (n + 1 < items) {
      load_item(n + 1, (int)((n + 1) & 1));
      cp_async_commit();
    }
    const uint8_t* st = ring + (int)(n & 1) * kStage;
    const uint8_t* qsn = st;
    const uint8_t* dosn = st + kTileBytes;
    const float* lse_s = reinterpret_cast<const float*>(st + 2 * kTileBytes);
    const float* del_s = reinterpret_cast<const float*>(st + 2 * kTileBytes + kVecBytes);
    const int i = i0 + (int)(n % nq);
    // transposed products: rows = this warp's keys, columns = the 64 queries of tile i
    float s[4][2][4], dp[4][2][4];
    gemm_nt<D>(s, kw, qsn, lane);
    gemm_nt<D>(dp, vw, dosn, lane);
    uint32_t keep = 0;   // dropout: rows are keys (S^T); the sequence is pixel p0 + n / nq of (b, h)
    if constexpr (kDrop)
      keep = drop_keep_tile<true>(key0, i * kTile + 2 * qd, ((uint64_t)s0.b * P + p0 + n / nq) * nh + s0.h, dkey,
                                  dr->thresh);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int c = nt * 8 + 2 * qd;
      const float2 ls = *reinterpret_cast<const float2*>(lse_s + c);
      const float2 dl = *reinterpret_cast<const float2*>(del_s + c);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int rr = e >> 1, ce = e & 1;
        float p = ex2_approx(fmaf(s[nt >> 1][nt & 1][e], cl2, -(ce ? ls.y : ls.x) * kLog2e));
        if (kCausal && i == j && i * kTile + c + ce < key0 + 8 * rr) p = 0.f;
        if constexpr (kDrop) {   // dV takes P~ = P Z (1 / (1 - p) at the flush); dS = P (dP Z - delta)
          const bool kp = (keep >> (4 * nt + e)) & 1u;
          s[nt >> 1][nt & 1][e] = kp ? p : 0.f;
          dp[nt >> 1][nt & 1][e] = p * ((kp ? dp[nt >> 1][nt & 1][e] * dr->rscale : 0.f) - (ce ? dl.y : dl.x));
        } else {
          s[nt >> 1][nt & 1][e] = p;
          dp[nt >> 1][nt & 1][e] = p * (dp[nt >> 1][nt & 1][e] - (ce ? dl.y : dl.x));
        }
      }
    }
    gemm_nn_acc<D, kAN>(dva, s, dosn, n0, lane);    // dV += P^T dO
    gemm_nn_acc<D, kAN>(dka, dp, qsn, n0, lane);    // dK += dS^T Q
  }
  const int t_w = j * kTile + wr * 16;
  if (!kv_bcast) {
    // every read of this warp's K / V rows is done (at D = 128 also by the partner warp, which reads all columns):
    // they stage the outputs
    if (D == 128) __syncthreads(); else __syncwarp();
    uint8_t* kw_out = ks + wr * 16 * kPitch;
    uint8_t* vw_out = vs + wr * 16 * kPitch;
    frags_to_rows<D, kAN>(kw_out, dka, scale, scale, n0, lane);
    if constexpr (kDrop)
      frags_to_rows<D, kAN>(vw_out, dva, dr->rscale, dr->rscale, n0, lane);
    else
      frags_to_rows<D, kAN>(vw_out, dva, 1.f, 1.f, n0, lane);
    __syncwarp();
    rows_to_global<D, kAN>(kw_out, dk + s0.q0, qpitch, t_w, T, half * 8, lane);
    rows_to_global<D, kAN>(vw_out, dv + s0.q0, qpitch, t_w, T, half * 8, lane);
  } else {
    // this chunk's sum over its pixels into the caller's fp32 [B][T][C] (unordered across chunks)
#pragma unroll
    for (int nt = 0; nt < kAN; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int t = key0 + 8 * (e >> 1);
        if (t >= T) continue;
        const long long off = ((long long)s0.b * T + t) * C + (long long)s0.h * D + n0 + nt * 8 + 2 * qd + (e & 1);
        atomicAdd(dk_b + off, dka[nt][e] * scale);
        if constexpr (kDrop)
          atomicAdd(dv_b + off, dva[nt][e] * dr->rscale);
        else
          atomicAdd(dv_b + off, dva[nt][e]);
      }
  }
}

template <int D>
__global__ void __launch_bounds__(Geo<D>::kDkdvThreads)
    og_temporal_attn_long_bwd_dkdv_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                          const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ dout,
                                          const float* __restrict__ lse, const float* __restrict__ delta,
                                          __nv_bfloat16* __restrict__ dk, __nv_bfloat16* __restrict__ dv,
                                          float* __restrict__ dk_b, float* __restrict__ dv_b, int B, int T,
                                          long long P, int C, int nh, float scale, int kv_bcast, int tiles,
                                          long long chunk, long long nchunk) {
  long_dkdv_body<D, false>(q, k, v, dout, lse, delta, dk, dv, dk_b, dv_b, B, T, P, C, nh, scale, kv_bcast, tiles, chunk,
                           nchunk, nullptr);
}

template <int D>
__global__ void __launch_bounds__(Geo<D>::kDkdvThreads)
    og_temporal_attn_long_dropout_bwd_dkdv_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                          const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ dout,
                                          const float* __restrict__ lse, const float* __restrict__ delta,
                                          __nv_bfloat16* __restrict__ dk, __nv_bfloat16* __restrict__ dv,
                                          float* __restrict__ dk_b, float* __restrict__ dv_b, int B, int T,
                                          long long P, int C, int nh, float scale, int kv_bcast, int tiles,
                                          long long chunk, long long nchunk, const DropParams d) {
  long_dkdv_body<D, true>(q, k, v, dout, lse, delta, dk, dv, dk_b, dv_b, B, T, P, C, nh, scale, kv_bcast, tiles, chunk,
                          nchunk, &d);
}

// bidirectional (SDPA is_causal=False over t), without (kDrop false) or with dropout
template <int D, bool kDrop>
__global__ void __launch_bounds__(kThreads)
    og_temporal_attn_bidir_fwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                      const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ res,
                                      __nv_bfloat16* __restrict__ out, __nv_bfloat16* __restrict__ out_res,
                                      float* __restrict__ lse, int B, int T, long long P, int C, int nh, float scale,
                                      int kv_bcast, int tiles, const DropParams d) {
  long_fwd_body<D, kDrop, false>(q, k, v, res, out, out_res, lse, B, T, P, C, nh, scale, kv_bcast, tiles, &d);
}

template <int D, bool kDrop>
__global__ void __launch_bounds__(kThreads)
    og_temporal_attn_bidir_bwd_dq_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                         const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ o,
                                         const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse,
                                         float* __restrict__ delta, __nv_bfloat16* __restrict__ dq, int B, int T,
                                         long long P, int C, int nh, float scale, int kv_bcast, int tiles,
                                         const DropParams d) {
  long_dq_body<D, kDrop, false>(q, k, v, o, dout, lse, delta, dq, B, T, P, C, nh, scale, kv_bcast, tiles, &d);
}

template <int D, bool kDrop>
__global__ void __launch_bounds__(Geo<D>::kDkdvThreads)
    og_temporal_attn_bidir_bwd_dkdv_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                           const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ dout,
                                           const float* __restrict__ lse, const float* __restrict__ delta,
                                           __nv_bfloat16* __restrict__ dk, __nv_bfloat16* __restrict__ dv,
                                           float* __restrict__ dk_b, float* __restrict__ dv_b, int B, int T,
                                           long long P, int C, int nh, float scale, int kv_bcast, int tiles,
                                           long long chunk, long long nchunk, const DropParams d) {
  long_dkdv_body<D, kDrop, false>(q, k, v, dout, lse, delta, dk, dv, dk_b, dv_b, B, T, P, C, nh, scale, kv_bcast,
                                  tiles, chunk, nchunk, &d);
}

}  // namespace tlong

}  // namespace og

using namespace og;

static bool long_aligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

namespace {
// the bidirectional kernels at head width D, with dropout when kDrop is set (shared memory as for the causal ones)
template <int D, bool kDrop>
int bidir_fwd(const void* q, const void* k, const void* v, void* out, const void* residual, void* out_res, float* lse,
              int B, int T, int64_t P, int C, int n_head, float scale, int kv_bcast, int tiles, long long grid,
              const DropParams& d, cudaStream_t stream) {
  using namespace og::tlong;
  static bool attr = false;
  if (!attr) {
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_temporal_attn_bidir_fwd_kernel<D, kDrop>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Geo<D>::kFwdSmem));
    attr = true;
  }
  og_temporal_attn_bidir_fwd_kernel<D, kDrop><<<(unsigned)grid, kThreads, Geo<D>::kFwdSmem, stream>>>(
      (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)residual,
      (__nv_bfloat16*)out, (__nv_bfloat16*)out_res, lse, B, T, P, C, n_head, scale, kv_bcast, tiles, d);
  OG_CHECK_CUDA(cudaGetLastError());
  return OG_OK;
}

template <int D, bool kDrop>
int bidir_bwd(const void* q, const void* k, const void* v, const void* out, const void* dout, const float* lse,
              float* delta_ws, void* dq, void* dk, void* dv, float* dk_bcast, float* dv_bcast, int B, int T, int64_t P,
              int C, int n_head, float scale, int kv_bcast, int tiles, long long chunk, long long nchunk,
              const DropParams& d, cudaStream_t s) {
  using namespace og::tlong;
  static bool attr = false;
  if (!attr) {
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_temporal_attn_bidir_bwd_dq_kernel<D, kDrop>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Geo<D>::kDqSmem));
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_temporal_attn_bidir_bwd_dkdv_kernel<D, kDrop>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Geo<D>::kDkdvSmem));
    attr = true;
  }
  const long long ntask = (long long)B * n_head * P;
  og_temporal_attn_bidir_bwd_dq_kernel<D, kDrop><<<(unsigned)(ntask * tiles), kThreads, Geo<D>::kDqSmem, s>>>(
      (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)out,
      (const __nv_bfloat16*)dout, lse, delta_ws, (__nv_bfloat16*)dq, B, T, P, C, n_head, scale, kv_bcast, tiles, d);
  OG_CHECK_CUDA(cudaGetLastError());
  const long long grid = (long long)B * n_head * nchunk * tiles;
  og_temporal_attn_bidir_bwd_dkdv_kernel<D, kDrop><<<(unsigned)grid, Geo<D>::kDkdvThreads, Geo<D>::kDkdvSmem, s>>>(
      (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)dout, lse,
      delta_ws, (__nv_bfloat16*)dk, (__nv_bfloat16*)dv, dk_bcast, dv_bcast, B, T, P, C, n_head, scale, kv_bcast, tiles,
      chunk, nchunk, d);
  OG_CHECK_CUDA(cudaGetLastError());
  return OG_OK;
}

template <int D>
int long_fwd(const void* q, const void* k, const void* v, void* out, const void* residual, void* out_res, float* lse,
             int B, int T, int64_t P, int C, int n_head, float scale, int kv_bcast, int tiles, long long grid,
             const DropParams* drop, cudaStream_t stream, bool causal) {
  using namespace og::tlong;
  if (!causal)
    return drop ? bidir_fwd<D, true>(q, k, v, out, residual, out_res, lse, B, T, P, C, n_head, scale, kv_bcast, tiles,
                                     grid, *drop, stream)
                : bidir_fwd<D, false>(q, k, v, out, residual, out_res, lse, B, T, P, C, n_head, scale, kv_bcast, tiles,
                                      grid, DropParams{}, stream);
  if (drop) {
    static bool dattr = false;
    if (!dattr) {
      OG_CHECK_CUDA(cudaFuncSetAttribute(og_temporal_attn_long_dropout_fwd_kernel<D>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Geo<D>::kFwdSmem));
      dattr = true;
    }
    og_temporal_attn_long_dropout_fwd_kernel<D><<<(unsigned)grid, kThreads, Geo<D>::kFwdSmem, stream>>>(
        (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)residual,
        (__nv_bfloat16*)out, (__nv_bfloat16*)out_res, lse, B, T, P, C, n_head, scale, kv_bcast, tiles, *drop);
    OG_CHECK_CUDA(cudaGetLastError());
    return OG_OK;
  }
  static bool attr = false;
  if (!attr) {   // above the 48 KiB default at D = 128
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_temporal_attn_long_fwd_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)Geo<D>::kFwdSmem));
    attr = true;
  }
  og_temporal_attn_long_fwd_kernel<D><<<(unsigned)grid, kThreads, Geo<D>::kFwdSmem, stream>>>(
      (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)residual,
      (__nv_bfloat16*)out, (__nv_bfloat16*)out_res, lse, B, T, P, C, n_head, scale, kv_bcast, tiles);
  OG_CHECK_CUDA(cudaGetLastError());
  return OG_OK;
}

template <int D>
int long_bwd(const void* q, const void* k, const void* v, const void* out, const void* dout, const float* lse,
             float* delta_ws, void* dq, void* dk, void* dv, float* dk_bcast, float* dv_bcast, int B, int T, int64_t P,
             int C, int n_head, float scale, int kv_bcast, int tiles, const DropParams* drop, cudaStream_t s,
             bool causal) {
  using namespace og::tlong;
  const long long ntask = (long long)B * n_head * P;
  // dK / dV: one pixel per CTA, or with kv_bcast contiguous pixel chunks of one (b, h), enough of them for ~4 CTAs
  // per SM
  long long chunk = 1, nchunk = P;
  if (kv_bcast) {
    const long long bht = (long long)B * n_head * tiles;
    long long want = ((long long)num_sms() * 4 + bht - 1) / bht;
    if (want < 1) want = 1;
    if (want > P) want = P;
    chunk = (P + want - 1) / want;
    nchunk = (P + chunk - 1) / chunk;
  }
  if (!causal) {   // dQ first: it also writes delta, which the dK / dV kernel reads
    const int r = drop ? bidir_bwd<D, true>(q, k, v, out, dout, lse, delta_ws, dq, dk, dv, dk_bcast, dv_bcast, B, T, P,
                                            C, n_head, scale, kv_bcast, tiles, chunk, nchunk, *drop, s)
                       : bidir_bwd<D, false>(q, k, v, out, dout, lse, delta_ws, dq, dk, dv, dk_bcast, dv_bcast, B, T,
                                             P, C, n_head, scale, kv_bcast, tiles, chunk, nchunk, DropParams{}, s);
    if (r != OG_OK) return r;
    g_launches.fetch_add(2);
    return OG_OK;
  }
  static bool attr = false, dattr = false;
  if (drop && !dattr) {
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_temporal_attn_long_dropout_bwd_dq_kernel<D>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Geo<D>::kDqSmem));
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_temporal_attn_long_dropout_bwd_dkdv_kernel<D>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Geo<D>::kDkdvSmem));
    dattr = true;
  }
  if (!drop && !attr) {
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_temporal_attn_long_bwd_dq_kernel<D>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Geo<D>::kDqSmem));
    OG_CHECK_CUDA(cudaFuncSetAttribute(og_temporal_attn_long_bwd_dkdv_kernel<D>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Geo<D>::kDkdvSmem));
    attr = true;
  }
  // dQ first: it also writes delta, which the dK / dV kernel reads
  if (drop)
    og_temporal_attn_long_dropout_bwd_dq_kernel<D><<<(unsigned)(ntask * tiles), kThreads, Geo<D>::kDqSmem, s>>>(
        (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)out,
        (const __nv_bfloat16*)dout, lse, delta_ws, (__nv_bfloat16*)dq, B, T, P, C, n_head, scale, kv_bcast, tiles,
        *drop);
  else
    og_temporal_attn_long_bwd_dq_kernel<D><<<(unsigned)(ntask * tiles), kThreads, Geo<D>::kDqSmem, s>>>(
        (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)out,
        (const __nv_bfloat16*)dout, lse, delta_ws, (__nv_bfloat16*)dq, B, T, P, C, n_head, scale, kv_bcast, tiles);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  const long long grid = (long long)B * n_head * nchunk * tiles;
  if (drop)
    og_temporal_attn_long_dropout_bwd_dkdv_kernel<D><<<(unsigned)grid, Geo<D>::kDkdvThreads, Geo<D>::kDkdvSmem, s>>>(
        (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)dout, lse,
        delta_ws, (__nv_bfloat16*)dk, (__nv_bfloat16*)dv, dk_bcast, dv_bcast, B, T, P, C, n_head, scale, kv_bcast,
        tiles, chunk, nchunk, *drop);
  else
    og_temporal_attn_long_bwd_dkdv_kernel<D><<<(unsigned)grid, Geo<D>::kDkdvThreads, Geo<D>::kDkdvSmem, s>>>(
        (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)dout, lse,
        delta_ws, (__nv_bfloat16*)dk, (__nv_bfloat16*)dv, dk_bcast, dv_bcast, B, T, P, C, n_head, scale, kv_bcast,
        tiles, chunk, nchunk);
  OG_CHECK_CUDA(cudaGetLastError());
  g_launches.fetch_add(1);
  return OG_OK;
}
}  // namespace

// og_temporal_attn_long_fwd, og_temporal_attn_long_dropout_fwd when `drop` is given, og_temporal_attn_bidir_fwd
// when `causal` is false
static int long_fwd_call(const void* q, const void* k, const void* v, void* out, const void* residual, void* out_res,
                         float* lse, int B, int T, int64_t P, int C, int n_head, float scale, int kv_bcast,
                         const DropParams* drop, og_stream_t stream, bool causal = true) {
  using namespace og::tlong;
  OG_REQUIRE(q && k && v && out && lse, "temporal_attn_long_fwd: null pointer");
  OG_REQUIRE(!residual == !out_res, "temporal_attn_long_fwd: residual and out_res must be given together");
  OG_REQUIRE(B >= 1 && T >= 1 && P >= 1, "temporal_attn_long_fwd: empty problem (B=%d, T=%d, P=%lld)", B, T,
             (long long)P);
  OG_REQUIRE(n_head >= 1 && C % n_head == 0, "temporal_attn_long_fwd: C=%d not divisible by n_head=%d", C, n_head);
  OG_REQUIRE(scale > 0.f, "temporal_attn_long_fwd: scale must be positive");
  const int dh = C / n_head;
  if (dh != 64 && dh != 128 && dh != 16) {
    set_error("temporal_attn_long_fwd: d_head=%d not supported (16, 64 or 128)", dh);
    return OG_ERR_UNSUPPORTED_SHAPE;
  }
  OG_REQUIRE(long_aligned(q) && long_aligned(k) && long_aligned(v) && long_aligned(out) && long_aligned(residual) &&
                 long_aligned(out_res),
             "temporal_attn_long_fwd: q, k, v, out, residual and out_res must be 16-byte aligned");
  const int tiles = (T + kTile - 1) / kTile;
  const long long grid = (long long)B * n_head * P * tiles;
  OG_REQUIRE(grid < (1LL << 31), "temporal_attn_long_fwd: too many tiles");
  const int r = dh == 64    ? long_fwd<64>(q, k, v, out, residual, out_res, lse, B, T, P, C, n_head, scale, kv_bcast,
                                           tiles, grid, drop, (cudaStream_t)stream, causal)
                 : dh == 128 ? long_fwd<128>(q, k, v, out, residual, out_res, lse, B, T, P, C, n_head, scale, kv_bcast,
                                             tiles, grid, drop, (cudaStream_t)stream, causal)
                             : long_fwd<16>(q, k, v, out, residual, out_res, lse, B, T, P, C, n_head, scale, kv_bcast,
                                            tiles, grid, drop, (cudaStream_t)stream, causal);
  if (r != OG_OK) return r;
  g_launches.fetch_add(1);
  return OG_OK;
}

extern "C" int og_temporal_attn_long_fwd(const void* q, const void* k, const void* v, void* out, const void* residual,
                                         void* out_res, float* lse, int B, int T, int64_t P, int C, int n_head,
                                         float scale, int kv_bcast, og_stream_t stream) {
  return long_fwd_call(q, k, v, out, residual, out_res, lse, B, T, P, C, n_head, scale, kv_bcast, nullptr, stream);
}

extern "C" int og_temporal_attn_long_dropout_fwd(const void* q, const void* k, const void* v, void* out,
                                                 const void* residual, void* out_res, float* lse, int B, int T,
                                                 int64_t P, int C, int n_head, float scale, int kv_bcast, float p,
                                                 const uint64_t* seed, og_stream_t stream) {
  DropParams d;
  if (const int r = drop_params(p, seed, "temporal_attn_long_dropout_fwd", &d)) return r;
  return long_fwd_call(q, k, v, out, residual, out_res, lse, B, T, P, C, n_head, scale, kv_bcast, &d, stream);
}

// og_temporal_attn_long_bwd, og_temporal_attn_long_dropout_bwd when `drop` is given, og_temporal_attn_bidir_bwd
// when `causal` is false
static int long_bwd_call(const void* q, const void* k, const void* v, const void* out, const void* dout,
                         const float* lse, float* delta_ws, void* dq, void* dk, void* dv, float* dk_bcast,
                         float* dv_bcast, int B, int T, int64_t P, int C, int n_head, float scale, int kv_bcast,
                         const DropParams* drop, og_stream_t stream, bool causal = true) {
  using namespace og::tlong;
  OG_REQUIRE(q && k && v && out && dout && lse && delta_ws && dq, "temporal_attn_long_bwd: null pointer");
  OG_REQUIRE(kv_bcast ? (dk_bcast && dv_bcast) : (dk && dv), "temporal_attn_long_bwd: missing dk/dv buffers");
  OG_REQUIRE(B >= 1 && T >= 1 && P >= 1, "temporal_attn_long_bwd: empty problem (B=%d, T=%d, P=%lld)", B, T,
             (long long)P);
  OG_REQUIRE(n_head >= 1 && C % n_head == 0, "temporal_attn_long_bwd: C=%d not divisible by n_head=%d", C, n_head);
  OG_REQUIRE(scale > 0.f, "temporal_attn_long_bwd: scale must be positive");
  const int dh = C / n_head;
  if (dh != 64 && dh != 128 && dh != 16) {
    set_error("temporal_attn_long_bwd: d_head=%d not supported (16, 64 or 128)", dh);
    return OG_ERR_UNSUPPORTED_SHAPE;
  }
  OG_REQUIRE(long_aligned(q) && long_aligned(k) && long_aligned(v) && long_aligned(out) && long_aligned(dout) &&
                 long_aligned(dq) && (kv_bcast || (long_aligned(dk) && long_aligned(dv))),
             "temporal_attn_long_bwd: q, k, v, out, dout, dq, dk and dv must be 16-byte aligned");
  const int tiles = (T + kTile - 1) / kTile;
  const long long ntask = (long long)B * n_head * P;
  OG_REQUIRE(ntask * tiles < (1LL << 31), "temporal_attn_long_bwd: too many tiles");
  if (dh == 16)
    return long_bwd<16>(q, k, v, out, dout, lse, delta_ws, dq, dk, dv, dk_bcast, dv_bcast, B, T, P, C, n_head, scale,
                        kv_bcast, tiles, drop, (cudaStream_t)stream, causal);
  return dh == 64 ? long_bwd<64>(q, k, v, out, dout, lse, delta_ws, dq, dk, dv, dk_bcast, dv_bcast, B, T, P, C,
                                 n_head, scale, kv_bcast, tiles, drop, (cudaStream_t)stream, causal)
                  : long_bwd<128>(q, k, v, out, dout, lse, delta_ws, dq, dk, dv, dk_bcast, dv_bcast, B, T, P, C,
                                  n_head, scale, kv_bcast, tiles, drop, (cudaStream_t)stream, causal);
}

extern "C" int og_temporal_attn_long_bwd(const void* q, const void* k, const void* v, const void* out,
                                         const void* dout, const float* lse, float* delta_ws, void* dq, void* dk,
                                         void* dv, float* dk_bcast, float* dv_bcast, int B, int T, int64_t P, int C,
                                         int n_head, float scale, int kv_bcast, og_stream_t stream) {
  return long_bwd_call(q, k, v, out, dout, lse, delta_ws, dq, dk, dv, dk_bcast, dv_bcast, B, T, P, C, n_head, scale,
                       kv_bcast, nullptr, stream);
}

extern "C" int og_temporal_attn_long_dropout_bwd(const void* q, const void* k, const void* v, const void* out,
                                                 const void* dout, const float* lse, float* delta_ws, void* dq,
                                                 void* dk, void* dv, float* dk_bcast, float* dv_bcast, int B, int T,
                                                 int64_t P, int C, int n_head, float scale, int kv_bcast, float p,
                                                 const uint64_t* seed, og_stream_t stream) {
  DropParams d;
  if (const int r = drop_params(p, seed, "temporal_attn_long_dropout_bwd", &d)) return r;
  return long_bwd_call(q, k, v, out, dout, lse, delta_ws, dq, dk, dv, dk_bcast, dv_bcast, B, T, P, C, n_head, scale,
                       kv_bcast, &d, stream);
}

extern "C" int og_temporal_attn_bidir_fwd(const void* q, const void* k, const void* v, void* out, const void* residual,
                                          void* out_res, float* lse, int B, int T, int64_t P, int C, int n_head,
                                          float scale, int kv_bcast, float p, const uint64_t* seed, og_stream_t stream) {
  DropParams d;
  const DropParams* drop;
  if (const int r = drop_params_opt(p, seed, "temporal_attn_bidir_fwd", &d, &drop)) return r;
  return long_fwd_call(q, k, v, out, residual, out_res, lse, B, T, P, C, n_head, scale, kv_bcast, drop, stream, false);
}

extern "C" int og_temporal_attn_bidir_bwd(const void* q, const void* k, const void* v, const void* out, const void* dout,
                                          const float* lse, float* delta_ws, void* dq, void* dk, void* dv,
                                          float* dk_bcast, float* dv_bcast, int B, int T, int64_t P, int C, int n_head,
                                          float scale, int kv_bcast, float p, const uint64_t* seed,
                                          og_stream_t stream) {
  DropParams d;
  const DropParams* drop;
  if (const int r = drop_params_opt(p, seed, "temporal_attn_bidir_bwd", &d, &drop)) return r;
  return long_bwd_call(q, k, v, out, dout, lse, delta_ws, dq, dk, dv, dk_bcast, dv_bcast, B, T, P, C, n_head, scale,
                       kv_bcast, drop, stream, false);
}
