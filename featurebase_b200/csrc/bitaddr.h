// Byte offset of the bitmap word that holds an array element, for the two u16 elements packed in one 32-bit payload word.
// Written as mask + multiply-high so that ptxas emits LOP3 + LEA.HI (base folded into the LEA) instead of
// SHF.R + LOP3 + IADD: one instruction less per scattered / probed element in the array hot loops (checked with
// cuobjdump -sass; the identity itself is checked on the host by tests/test_stripe.py::test_word_offset_identity).
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define FBGPU_HD __host__ __device__ __forceinline__
#else
#define FBGPU_HD inline
#endif

namespace fbgpu {
FBGPU_HD uint32_t mulhi_u32(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}
// Shift / LEA forms, not IMAD.HI on the FMA pipe: IMAD.HI issues at half their rate (bench_micro/pipe_rates.cu), measured slower.
// w = (hi << 16) | lo.  4 * (lo >> 5)  and  4 * (hi >> 5)
FBGPU_HD uint32_t word_off_lo(uint32_t w) { return mulhi_u32(w & 0xffe0u, 1u << 29); }
FBGPU_HD uint32_t word_off_hi(uint32_t w) { return mulhi_u32(w & 0xffe00000u, 1u << 13); }
// sb: shared-space address of the bitmap
FBGPU_HD uint32_t word_addr_lo(uint32_t sb, uint32_t w) { return sb + word_off_lo(w); }
FBGPU_HD uint32_t word_addr_hi(uint32_t sb, uint32_t w) { return sb + word_off_hi(w); }
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ void pin_base(uint32_t& sb) { asm volatile("" : "+r"(sb)); }
#else
inline void pin_base(uint32_t&) {}
#endif
}  // namespace fbgpu
