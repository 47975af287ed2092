// Activation-buffer layout of the tensor-core point kernel (point_tc.cu) and the byte offsets its epilogues and its
// fold1/conv1 prologue store at.  Host and device code: tests/test_tc_addressing_cpu.py checks the offsets on the CPU.
#pragma once
#include <stdint.h>

#include "tc_common.cuh"

namespace disn {
namespace ptc {

constexpr uint32_t X_TILE = 8192;          // 64 rows x 64 k x 2 B (SW128)
constexpr uint32_t X8_TILE = 4096;         // 64 rows x 64 k x 1 B (SW64)
constexpr uint32_t X_SLICE = 2 * X_TILE;   // one 64-wide K slice: [hi | lo] or [fp16 | e5m2 residual | e5m2 copy]

// The swizzle XOR touches bits 4-6 (SW128) or 4-5 (SW64) of a byte offset.  The bits below are the byte within the
// 16-byte chunk, and everything above (rows, 8-row groups, tiles, K slices; the buffer is 1024-B aligned) is a multiple
// of 128 or 64 that the XOR never carries into.  So a thread that always stores at the same row and the same byte of a
// chunk keeps one base per row, with the row's own XOR pattern already in bits 4-6 / 4-5, and XORs the chunk into it:
//   sw128_offset(row, c) + b == (sw128_row_base(row) + b) ^ (c << 4),  b < 16,
// and likewise for SW64; any multiple of 1024 (SW128) or 512 (SW64) can be added on either side.
__host__ __device__ constexpr uint32_t sw128_row_base(uint32_t row) { return (row >> 3) * 1024u + (row & 7u) * (128u + 16u); }
__host__ __device__ constexpr uint32_t sw64_row_base(uint32_t row) {
  return (row >> 3) * 512u + (row & 7u) * 64u + (((row >> 1) & 3u) << 4);
}

// Layer epilogue of thread (h, r0, cq): accumulator rows r0 + 8 e2, features 256 nb + 128 h + cq + 8 j (j = 0..15), that
// is K slice 4 nb + 2 h + j / 8 at k = cq + 8 (j % 8).  The thread keeps base16 and base8; each distinct j % 8 costs one
// XOR per epilogue, and nb, j / 8, e2 and the tile within the slice are immediates.
__host__ __device__ constexpr uint32_t epi_base16(uint32_t h, uint32_t r0, uint32_t cq) {
  return 2u * h * X_SLICE + sw128_row_base(r0) + 2u * cq;
}
__host__ __device__ constexpr uint32_t epi_base8(uint32_t h, uint32_t r0, uint32_t cq) {
  return 2u * h * X_SLICE + X_TILE + sw64_row_base(r0) + cq;
}
// fp16 / bf16 hi element pair (the bf16 lo pair is X_TILE further)
__host__ __device__ constexpr uint32_t epi_off16(uint32_t base16, int nb, int j, int e2) {
  return (base16 ^ ((uint32_t)(j & 7) << 4)) + (uint32_t)(4 * nb + (j >> 3)) * X_SLICE + (uint32_t)e2 * 1024u;
}
// e5m2 residual pair (the e5m2 copy is X8_TILE further)
__host__ __device__ constexpr uint32_t epi_off8(uint32_t base8, int nb, int j, int e2) {
  return (base8 ^ ((uint32_t)((j & 7) >> 1) << 4)) + 8u * (uint32_t)(j & 1) + (uint32_t)(4 * nb + (j >> 3)) * X_SLICE +
         (uint32_t)e2 * 512u;
}

// fold1/conv1 prologue of thread (p, q): point p, features 16 q + jj (jj = 0, 2, .., 14) of K slice 0
__host__ __device__ constexpr uint32_t pro_base16(uint32_t p, uint32_t q) { return sw128_row_base(p) ^ (q << 5); }
__host__ __device__ constexpr uint32_t pro_base8(uint32_t p, uint32_t q) { return X_TILE + (sw64_row_base(p) ^ (q << 4)); }
__host__ __device__ constexpr uint32_t pro_off16(uint32_t base16, int jj) {
  return (base16 ^ ((uint32_t)(jj >> 3) << 4)) + 2u * (uint32_t)(jj & 7);
}
__host__ __device__ constexpr uint32_t pro_off8(uint32_t base8, int jj) { return base8 + (uint32_t)jj; }

// number of stores whose offset differs from the one tc::sw128_offset / tc::sw64_offset give, over every thread and
// element of the epilogues and the prologue (0 when the formulas above are right)
__host__ __device__ constexpr int store_offset_mismatches() {
  int bad = 0;
  for (uint32_t h = 0; h < 2; ++h)
    for (uint32_t r0 = 0; r0 + 8 < 64; ++r0)
      for (uint32_t cq = 0; cq < 8; cq += 2) {
        const uint32_t b16 = epi_base16(h, r0, cq), b8 = epi_base8(h, r0, cq);
        for (int nb = 0; nb < 2; ++nb)
          for (int j = 0; j < 16; ++j)
            for (int e2 = 0; e2 < 2; ++e2) {
              const uint32_t col = 256u * nb + 128u * h + cq + 8u * j, row = r0 + 8u * e2, k = col & 63u;
              const uint32_t slice = (col >> 6) * X_SLICE;
              bad += epi_off16(b16, nb, j, e2) != slice + tc::sw128_offset(row, k >> 3) + 2u * (k & 7u);
              bad += epi_off8(b8, nb, j, e2) != slice + X_TILE + tc::sw64_offset(row, k >> 4) + (k & 15u);
            }
      }
  for (uint32_t p = 0; p < 64; ++p)
    for (uint32_t q = 0; q < 4; ++q)
      for (int jj = 0; jj < 16; jj += 2) {
        const uint32_t k = 16u * q + (uint32_t)jj;
        bad += pro_off16(pro_base16(p, q), jj) != tc::sw128_offset(p, k >> 3) + 2u * (k & 7u);
        bad += pro_off8(pro_base8(p, q), jj) != X_TILE + tc::sw64_offset(p, k >> 4) + (k & 15u);
      }
  return bad;
}

}  // namespace ptc
}  // namespace disn
