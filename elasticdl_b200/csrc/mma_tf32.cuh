// 3xTF32 on mma.sync.m16n8k8 (sm_80+), shared by the mma DeepFM tower (deepfm_tower_mma.cu) and the xDeepFM CIN
// (xdeepfm_cin.cu): an fp32 operand is split hi + lo in registers (both TF32) and a product is the sum of
// lo*hi + hi*lo + hi*hi, which carries fp32-grade accuracy with fp32 accumulation.
//
// Fragment coordinates (PTX ISA, m16n8k8 .tf32): gid = lane / 4, tig = lane % 4
//   A (16x8, row): a0 (gid, tig)  a1 (gid+8, tig)  a2 (gid, tig+4)  a3 (gid+8, tig+4)
//   B ( 8x8, col): b0 (k = tig, n = gid)  b1 (k = tig+4, n = gid)
//   C (16x8):      c0 (gid, 2 tig)  c1 (gid, 2 tig+1)  c2 (gid+8, 2 tig)  c3 (gid+8, 2 tig+1)
#pragma once
#include <cstdint>

namespace deepfm {

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void split(float x, uint32_t& hi, uint32_t& lo) {
  hi = to_tf32(x);
  lo = to_tf32(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// d += a * b with the operands split hi + lo (small terms first)
__device__ __forceinline__ void mma3(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                     const uint32_t (&bh)[2], const uint32_t (&bl)[2]) {
  mma_tf32(d, al, bh);
  mma_tf32(d, ah, bl);
  mma_tf32(d, ah, bh);
}

}  // namespace deepfm
