// The streak records of a compressed alignment (src/compressAlignment.cpp, formats src/compressAlignment.hpp:102-320): a
// streak is a run of len consecutive aligned marker pairs, stored as (skip0, skip1, len - 1) in 1, 2, 4, 8 or 16 bytes, where
// skip0 and skip1 are the ordinal steps from the last pair of the previous streak (from (0, 0) for the first streak).
#pragma once

#include <cstdint>

namespace shb {

// The bytes of the smallest format that holds the streak (src/compressAlignment.cpp:11-70).
__device__ __forceinline__ uint32_t compressedStreakBytes(int32_t skip0, int32_t skip1, uint32_t len)
{
    if(skip0 >= 0 && skip0 <= 3 && skip1 >= 0 && skip1 <= 3 && len <= 8) return 1;
    if(skip0 >= -8 && skip0 <= 7 && skip1 >= -8 && skip1 <= 7 && len <= 32) return 2;
    if(skip0 >= -512 && skip0 <= 511 && skip1 >= -512 && skip1 <= 511 && len <= 512) return 4;
    if(skip0 >= -524288 && skip0 <= 524287 && skip1 >= -524288 && skip1 <= 524287 && len <= 2097152) return 8;
    return 16;
}

// Writes the streak's record at out. Returns its size. It repeats the range tests of compressedStreakBytes: written in terms
// of it, alignmentWriteKernel compiles to different code.
__device__ __forceinline__ uint32_t writeCompressedStreak(uint8_t* out, int32_t skip0, int32_t skip1, uint32_t len)
{
    const uint64_t nm1 = len - 1;
    if(skip0 >= 0 && skip0 <= 3 && skip1 >= 0 && skip1 <= 3 && len <= 8) {
        out[0] = uint8_t(0u | (uint32_t(skip0) << 1) | (uint32_t(skip1) << 3) | (uint32_t(nm1) << 5));
        return 1;
    }
    uint64_t v; uint32_t bytes;
    if(skip0 >= -8 && skip0 <= 7 && skip1 >= -8 && skip1 <= 7 && len <= 32) {
        v = 1u | ((uint32_t(skip0) & 0xFu) << 3) | ((uint32_t(skip1) & 0xFu) << 7) | (uint32_t(nm1) << 11); bytes = 2;
    } else if(skip0 >= -512 && skip0 <= 511 && skip1 >= -512 && skip1 <= 511 && len <= 512) {
        v = 3u | ((uint32_t(skip0) & 0x3FFu) << 3) | ((uint32_t(skip1) & 0x3FFu) << 13) | (uint32_t(nm1) << 23); bytes = 4;
    } else if(skip0 >= -524288 && skip0 <= 524287 && skip1 >= -524288 && skip1 <= 524287 && len <= 2097152) {
        v = 5ull | ((uint64_t(int64_t(skip0)) & 0xFFFFFull) << 3) | ((uint64_t(int64_t(skip1)) & 0xFFFFFull) << 23) | (nm1 << 43); bytes = 8;
    } else {
        const uint32_t w[4] = {7u, uint32_t(skip0), uint32_t(skip1), uint32_t(nm1)};
        for(int i = 0; i < 16; i++) out[i] = uint8_t(w[i >> 2] >> (8 * (i & 3)));
        return 16;
    }
    for(uint32_t i = 0; i < bytes; i++) out[i] = uint8_t(v >> (8 * i));
    return bytes;
}

__host__ __device__ __forceinline__ uint32_t streakByte(const uint8_t* s, uint64_t i)
{
#ifdef __CUDA_ARCH__
    return __ldg(s + i);
#else
    return s[i];
#endif
}

// The streak record at s[pos], pos < end, as shasta::decompress reads it (src/compressAlignment.cpp:73-137); pos moves past
// it. Returns false when the record runs past end. The 2- and 4-byte records are read as whole 8-byte words: the 6 bytes
// after end must be readable.
__host__ __device__ __forceinline__ bool decodeStreak(const uint8_t* s, uint64_t& pos, uint64_t end, int32_t& skip0, int32_t& skip1,
                                                      uint32_t& len)
{
    const uint32_t c0 = streakByte(s, pos);
    if((c0 & 1u) == 0) {
        skip0 = (c0 >> 1) & 3; skip1 = (c0 >> 3) & 3; len = ((c0 >> 5) & 7u) + 1; pos += 1;
        return true;
    }
    const uint32_t tag = c0 & 7u;
    const uint32_t nb = tag == 1 ? 2 : tag == 3 ? 4 : tag == 5 ? 8 : 16;
    if(pos + nb > end) return false;
    uint64_t v = 0, w = 0;
    for(uint32_t b = 0; b < 8; b++) v |= uint64_t(streakByte(s, pos + b)) << (8 * b);
    if(nb == 16) {
        for(uint32_t b = 0; b < 8; b++) w |= uint64_t(streakByte(s, pos + 8 + b)) << (8 * b);
        skip0 = int32_t(uint32_t(v >> 32)); skip1 = int32_t(uint32_t(w)); len = uint32_t(w >> 32) + 1;
    } else {
        const int bits = nb == 2 ? 4 : nb == 4 ? 10 : 20;
        if(nb < 8) v &= (1ull << (8 * nb)) - 1;
        const uint64_t m = (1ull << bits) - 1, sign = 1ull << (bits - 1);
        const uint64_t f0 = (v >> 3) & m, f1 = (v >> (3 + bits)) & m;
        skip0 = int32_t(int64_t(f0 ^ sign) - int64_t(sign));
        skip1 = int32_t(int64_t(f1 ^ sign) - int64_t(sign));
        len = uint32_t(v >> (3 + 2 * bits)) + 1;
    }
    pos += nb;
    return true;
}

} // namespace shb
