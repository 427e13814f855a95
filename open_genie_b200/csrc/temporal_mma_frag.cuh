// temporal_mma_frag.cuh — mma.sync m16n8k16 fragment helpers shared by the temporal attention kernels
// (temporal_attn_mma.cu for T <= 16, temporal_attn_long.cu for longer clips).
//
// Staged matrices are rows of 64 bf16 in shared memory with a 144-byte pitch (128 data + 16 pad), which makes every
// ldmatrix below bank-conflict free. The loaders take the pitch as a template argument (default 144) so the tiled
// kernels can stage 128-wide rows at 272 bytes (256 data + 16 pad, 17 x 16 B: conflict free as well). Fragment conventions (PTX ISA, mma.m16n8k16 .row.col, bf16):
//   A (16x16): a0a1 = (g, 2q..), a2a3 = (g+8, 2q..), a4a5 = (g, 8+2q..), a6a7 = (g+8, 8+2q..)   g = lane/4, q = lane%4
//   B (16x8) : b0b1 = (k = 2q.., n = g), b2b3 = (k = 8+2q.., n = g)
//   C (16x8) : c0c1 = (g, 2q..), c2c3 = (g+8, 2q..)
// so the C fragments of a 16x16 product (two n-tiles) re-pack directly into the A fragment of the next one (pack_a).
#pragma once
#include "og_ptx.cuh"

namespace og {
namespace tmma {
constexpr int kD = 64;
constexpr int kPitch = 144;                 // bytes per staged row (128 data + 16 pad)

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2(uint32_t (&r)[2], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2_trans(uint32_t (&r)[2], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// A fragment (16 x 16 slice starting at column `col0`) of a staged row-major matrix
template <int Pitch = kPitch>
__device__ __forceinline__ void load_a(uint32_t (&a)[4], const uint8_t* m, int col0, int lane) {
  ldsm_x4(a, smem_u32(m + (lane & 15) * Pitch + (col0 + (lane >> 4) * 8) * 2));
}
// B fragment for  B[k][n] = M[n0 + n][k0 + k]  (rows of the staged matrix are the n index: Q K^T, dO V^T)
template <int Pitch = kPitch>
__device__ __forceinline__ void load_b_rows(uint32_t (&b)[2], const uint8_t* m, int n0, int k0, int lane) {
  ldsm_x2(b, smem_u32(m + (n0 + (lane & 7)) * Pitch + (k0 + ((lane >> 3) & 1) * 8) * 2));
}
// B fragment for  B[k][n] = M[k][n0 + n]  (rows of the staged matrix are the k index: P V, dS K, P^T dO, dS^T Q)
template <int Pitch = kPitch>
__device__ __forceinline__ void load_b_cols(uint32_t (&b)[2], const uint8_t* m, int n0, int lane) {
  ldsm_x2_trans(b, smem_u32(m + (lane & 15) * Pitch + n0 * 2));
}

// the C fragments of a 16 x 16 product (two n-tiles) as the bf16 A fragment of the next product
__device__ __forceinline__ void pack_a(uint32_t (&a)[4], const float (&c)[2][4]) {
  a[0] = pack_bf16x2(c[0][0], c[0][1]);
  a[1] = pack_bf16x2(c[0][2], c[0][3]);
  a[2] = pack_bf16x2(c[1][0], c[1][1]);
  a[3] = pack_bf16x2(c[1][2], c[1][3]);
}

}  // namespace tmma
}  // namespace og
