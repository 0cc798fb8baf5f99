// Philox4x32-10 (Salmon et al., SC'11): the counter-based generator of every random draw K7 and the PER sampler make.
#pragma once
#include <stdint.h>

__device__ __forceinline__ uint4 philox(uint4 c, uint2 k)
{
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u; k.y += 0xBB67AE85u;
    }
    return c;
}
