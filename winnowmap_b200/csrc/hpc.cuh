// Homopolymer compression of a packed slice (the is_hpc branch of mm_sketch, reference src/sketch.c:146-157): a run of
// one non-ambiguous code collapses into one symbol that sits at the run's LAST base; an ambiguous base is a symbol of its
// own.  Runs never cross the ends of the sketched slice.  The bit logic here is shared by the device front end
// (sketch.cu) and the host software warp of the tests.
#pragma once
#include <stdint.h>

// bits 0, 2, .., 62 of x -> bits 0 .. 31
__host__ __device__ __forceinline__ uint32_t wm_hpc_even_bits(uint64_t x)
{
	x &= 0x5555555555555555ULL;
	x = (x | x >> 1) & 0x3333333333333333ULL;
	x = (x | x >> 2) & 0x0f0f0f0f0f0f0f0fULL;
	x = (x | x >> 4) & 0x00ff00ff00ff00ffULL;
	x = (x | x >> 8) & 0x0000ffff0000ffffULL;
	x = (x | x >> 16) & 0x00000000ffffffffULL;
	return (uint32_t)x;
}

// Symbol ends among 32 bases: v / m are the 2-bit codes and ambiguity flags of bases b .. b + 31, v1 / m1 those of
// b + 1 .. b + 32.  Bit j is set when base b + j ends its symbol: the next base has another code, or either is ambiguous.
__host__ __device__ __forceinline__ uint32_t wm_hpc_ends32(uint64_t v, uint64_t v1, uint32_t m, uint32_t m1)
{
	const uint64_t d = v ^ v1;
	return wm_hpc_even_bits(d | d >> 1) | m | m1;
}

// the ends of group g (bases 32g .. 32g + 31) of a slice of len bases: nothing past the slice, and its last base ends a symbol
__host__ __device__ __forceinline__ uint32_t wm_hpc_clip(uint32_t e, int g, int len)
{
	const int n = len - 32 * g; // bases of the slice from the group's first one on
	if (n > 32) return e;
	return (n == 32 ? e : e & ((1u << n) - 1u)) | 1u << (n - 1);
}
