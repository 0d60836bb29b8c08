// Philox4x32-10 (Salmon et al., SC'11), word 0 of the output block: the counter-based generator behind the device-drawn
// StVD discards.  Counter domains (word 2) keep the draws of the different users apart:
//   0: layer discard        (row, site, 0, 0)                                  csrc/stvd_layer.cu
//   1: input discard keys   (row, 0, 1, draw)                                  csrc/stvd.cu
//   2: input shuffle        (value, stream << 16 | scene, 2, draw << 8 | round)  csrc/stvd.cu
// numpy restatement: oracle/stvd_layer.py (philox4x32_10).
#pragma once
#include <stdint.h>

namespace vc {

__device__ __forceinline__ uint32_t philox_word0(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) {
            k0 += 0x9E3779B9u;
            k1 += 0xBB67AE85u;
        }
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0;
        c1 = lo1;
        c2 = n2;
        c3 = lo0;
    }
    return c0;
}

}  // namespace vc
