// faiss_b200 -- device-side addressing of the stored IVF list layouts, shared by every kernel that reads or
// writes list entries: the appends and list copies (ivfpq_scan.cu), the scans (ivfsq_scan.cu) and the decoder
// (ivf_reconstruct.cu).  One owner per layout: a second copy of these formulas is a second place to get wrong.
#pragma once

#include <cuda_fp16.h>

#include <cstdint>

namespace fb200 {

// ---- interleaved-by-32 PQ layout (kernels.h): 8-bit codes with M in {16, 32} and 4-bit codes as M/2 nibble-pair
// bytes.  Byte b of the CPU code of list-relative vector v = 32 g + t, for codes of codeBytes (16 or 32) bytes, lives
// at this offset from the list's first code byte: group g, 16-byte column (j / 16), lane t, j = (b ^ t) mod codeBytes.
__device__ __forceinline__ int64_t ivfInterleavedByte(int64_t v, int b, int codeBytes) {
    const int t = (int)(v & 31);
    const int j = (b ^ t) & (codeBytes - 1);
    return (v >> 5) * 32 * codeBytes + (j >> 4) * 512 + t * 16 + (j & 15);
}

// ---- scalar-quantiser code fields (faiss/impl/scalar_quantizer/codecs.h).  Codecs: 0 = one byte per component
// (8bit, 8bit_uniform, 8bit_direct), 1 = nibbles (4bit, 4bit_uniform), 2 = 6-bit (3 bytes per 4 components),
// 3 = fp16.
enum { SQC_BYTE = 0, SQC_NIBBLE = 1, SQC_SIX = 2, SQC_HALF = 3 };

__device__ __forceinline__ float sq_u2f(unsigned c) { // exact for c < 2^23, no I2F
    return __uint_as_float(c | 0x4B000000u) - 8388608.f;
}

// component i of one code row, as a float: the integer code (exactly), or the fp16 value widened
template <int CODEC>
__device__ __forceinline__ float sq_row_comp(const uint8_t* __restrict__ cp, int i) {
    if (CODEC == SQC_BYTE) {
        return sq_u2f(__ldg(cp + i));
    } else if (CODEC == SQC_NIBBLE) {
        return sq_u2f(((unsigned)__ldg(cp + (i >> 1)) >> ((i & 1) << 2)) & 0xfu);
    } else if (CODEC == SQC_SIX) { // codecs.h:94-116
        const uint8_t* g = cp + (i >> 2) * 3;
        unsigned bits;
        switch (i & 3) {
            case 0:
                bits = __ldg(g) & 0x3fu;
                break;
            case 1:
                bits = ((unsigned)__ldg(g) >> 6) | (((unsigned)__ldg(g + 1) & 0xfu) << 2);
                break;
            case 2:
                bits = ((unsigned)__ldg(g + 1) >> 4) | (((unsigned)__ldg(g + 2) & 3u) << 4);
                break;
            default:
                bits = (unsigned)__ldg(g + 2) >> 2;
                break;
        }
        return sq_u2f(bits);
    } else {
        return __half2float(__ushort_as_half(__ldg(reinterpret_cast<const unsigned short*>(cp) + i)));
    }
}

} // namespace fb200
