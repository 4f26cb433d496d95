// morton.cuh -- 64-bit 3-D Morton codes and the window query over a sorted code array (SURVEY.md 8f, row N3).
//
// Replaces src/common/morton_code.cpp (MortonCode64: constructor :43-63, decode :73-81, operator+ :131-146,
// Negate :118-129, operator- :160-163) and the five bindings of src/morton.cpp (morton_add :26-103,
// morton_subtract :106-183, morton_encode :185-239, morton_decode :253-310, morton_knn :324-414) of the reference.
// Integer work throughout: results are bit-identical.
// Layout of a code: bit 3 i + a holds bit i of coordinate a (a = 0: x); coordinates are 21-bit two's complement
// with the sign bit (bit 20 -> code bits 60 .. 62) stored INVERTED, so that unsigned order of the codes is the
// order of the signed coordinates along the curve.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pcu {

constexpr unsigned long long kMortonSigns = 0x7000000000000000ull;
constexpr unsigned long long kMortonX = 0x1249249249249249ull;   // every third bit: the x coordinate

__host__ __device__ __forceinline__ unsigned long long morton_split21(int x) {   // morton_code.cpp:13-26
    unsigned long long r = (unsigned long long)(long long)x;   // `uint64_t r = x` sign-extends a negative int32 like this
    r = (r | r << 32) & 0x1f00000000ffffull;
    r = (r | r << 16) & 0x1f0000ff0000ffull;
    r = (r | r << 8) & 0x100f00f00f00f00full;
    r = (r | r << 4) & 0x10c30c30c30c30c3ull;
    r = (r | r << 2) & 0x1249249249249249ull;
    return r;
}
__host__ __device__ __forceinline__ int morton_compact21(unsigned long long x) {   // :28-41
    unsigned long long d = x & 0x1249249249249249ull;
    d = (d | d >> 2) & 0x10c30c30c30c30c3ull;
    d = (d | d >> 4) & 0x100f00f00f00f00full;
    d = (d | d >> 8) & 0x1f0000ff0000ffull;
    d = (d | d >> 16) & 0x1f00000000ffffull;
    d = (d | d >> 32);
    d = (d & 0x100000ull) ? (d | 0xffe00000ull) : d;   // sign extension
    return (int)d;
}
__host__ __device__ __forceinline__ unsigned long long morton_encode3(int x, int y, int z) {   // :48-63
    // sign bit to bit 20; in the reference `x & 0x80000000` is unsigned (the literal does not fit an int), so the shift is logical
    x = (int)(((unsigned)x & 0x80000000u) >> 11 | ((unsigned)x & 0x0fffffu));
    y = (int)(((unsigned)y & 0x80000000u) >> 11 | ((unsigned)y & 0x0fffffu));
    z = (int)(((unsigned)z & 0x80000000u) >> 11 | ((unsigned)z & 0x0fffffu));
    const unsigned long long data = morton_split21(x) | morton_split21(y) << 1 | morton_split21(z) << 2;
    return data ^ kMortonSigns;
}
__host__ __device__ __forceinline__ void morton_decode3(unsigned long long code, int& x, int& y, int& z) {   // :73-81
    const unsigned long long d = code ^ kMortonSigns;
    x = morton_compact21(d);
    y = morton_compact21(d >> 1);
    z = morton_compact21(d >> 2);
}
__host__ __device__ __forceinline__ unsigned long long morton_add2(unsigned long long a, unsigned long long b) {   // :131-146
    const unsigned long long c1 = a ^ kMortonSigns, c2 = b ^ kMortonSigns;
    const unsigned long long ym = kMortonX << 1, zm = kMortonX << 2;
    const unsigned long long xs = (c1 | ~kMortonX) + (c2 & kMortonX);
    const unsigned long long ys = (c1 | ~ym) + (c2 & ym);
    const unsigned long long zs = (c1 | ~zm) + (c2 & zm);
    return ((xs & kMortonX) | (ys & ym) | (zs & zm)) ^ kMortonSigns;
}
__host__ __device__ __forceinline__ unsigned long long morton_negate(unsigned long long a) {   // :118-129 (no sign-bit inversion there)
    const unsigned long long ym = kMortonX << 1, zm = kMortonX << 2;
    const unsigned long long d = ~a;
    const unsigned long long xs = (d | ~kMortonX) + 1, ys = (d | ~ym) + 1, zs = (d | ~zm) + 1;
    return (xs & kMortonX) | (ys & ym) | (zs & zm);
}

}  // namespace pcu
