// philox.cuh -- one round of Random123's Philox-4x32-10, the counter-based generator of lisa.cu and pylisa.cu.  A draw
// runs ten rounds, bumping the key (k0, k1) by (0x9E3779B9, 0xBB67AE85) after each.
#pragma once

__device__ __forceinline__ void philox_round(unsigned &c0, unsigned &c1, unsigned &c2, unsigned &c3, unsigned k0, unsigned k1)
{
    const unsigned long long p0 = (unsigned long long)0xD2511F53u * c0, p1 = (unsigned long long)0xCD9E8D57u * c2;
    const unsigned n0 = (unsigned)(p1 >> 32) ^ c1 ^ k0, n1 = (unsigned)p1, n2 = (unsigned)(p0 >> 32) ^ c3 ^ k1, n3 = (unsigned)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
}
