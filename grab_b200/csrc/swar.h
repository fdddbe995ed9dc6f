// swar.h -- SIMD-within-a-register byte predicates, 4 bytes per 32-bit op.  __host__ __device__
// so the arithmetic can be brute-force checked on the CPU (tests/test_swar.py); the product only
// ever runs the device instantiation.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define SWAR_HD __host__ __device__ __forceinline__
#else
#define SWAR_HD inline
#endif

namespace gscan {

constexpr uint32_t kOnes = 0x01010101u, kHigh = 0x80808080u, kLow7 = 0x7f7f7f7fu;

// Bit 7 of every byte of the result is set where the byte of t MAY be zero: exact for the lowest
// zero byte, may over-report above it (borrow).  Non-zero result <=> t has a zero byte.
SWAR_HD uint32_t zero_bytes_superset(uint32_t t) { return (t - kOnes) & ~t; }

// Filter test on 4 positions at once: byte k of the result has bit 7 set (superset) where
// (w.byte[k] & m0) == v0 and (s.byte[k] & m1) == v1.
SWAR_HD uint32_t pair_test(uint32_t w, uint32_t s, uint32_t m0, uint32_t v0, uint32_t m1, uint32_t v1)
{
	uint32_t t = ((w & m0) ^ v0) | ((s & m1) ^ v1);
	return zero_bytes_superset(t);
}

// Exact range test on the low 7 bits: x7 = x & 0x7f7f7f7f; bit 7 of byte k set iff lo <= x7.byte[k] <= hi
// add_ge = (0x80-lo)*kOnes, add_gt = (0x7f-hi)*kOnes.  No carries cross bytes.
SWAR_HD uint32_t range7(uint32_t x7, uint32_t add_ge, uint32_t add_gt) { return (x7 + add_ge) & ~(x7 + add_gt); }

// Gathers bit 7 of the four bytes into bits 28..31 (byte 0 -> bit 28).  f must only have bits 7,15,23,31.
SWAR_HD uint32_t pack_top_nibble(uint32_t f) { return f * 0x00204081u; }

// positions (low 16 bits of w32 = own chunk, high 16 = following chunk) where at least n (1..17)
// consecutive one bits start
SWAR_HD uint32_t runs_at_least(uint32_t w, uint32_t n)
{
	uint32_t r1 = w, r2 = r1 & (r1 >> 1), r4 = r2 & (r2 >> 2), r8 = r4 & (r4 >> 4), r16 = r8 & (r8 >> 8);
	uint32_t acc = 0xffffffffu, sh = 0;
	if (n & 16) { acc &= r16; sh = 16; }
	if (n & 8) { acc &= r8 >> sh; sh += 8; }
	if (n & 4) { acc &= r4 >> sh; sh += 4; }
	if (n & 2) { acc &= r2 >> sh; sh += 2; }
	if (n & 1) { acc &= r1 >> sh; }
	return acc;
}

} // namespace gscan
