// philox.cuh -- Philox4x32-10 (Salmon, Moraes, Dror and Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC 2011)
// as __host__ __device__ functions: the counter-based stream of the dynamic instability (skb_dynamic.cu), the same
// function on the host and on the device.  tests/dynamic_instability_reference.py restates it and checks the known
// answers of the paper's Random123 distribution.
//
// The stream of skb_flow_dynamic_instability (DESIGN.md §3.11): key = (seed low 32 bits, seed high 32 bits), counter =
// (draw index i, purpose, call counter low 32 bits, call counter high 32 bits); purpose 0 the catastrophe draw of fiber i
// (container order before the call), 1 the Poisson draw of chunk i, 2 the site pick i.  A draw is independent of the
// launch configuration and of how the fibers are partitioned.
#pragma once
#include <cstdint>

namespace skb {

constexpr uint32_t kPhiloxM0 = 0xD2511F53u, kPhiloxM1 = 0xCD9E8D57u; // round multipliers
constexpr uint32_t kPhiloxW0 = 0x9E3779B9u, kPhiloxW1 = 0xBB67AE85u; // Weyl key increments
enum DiPurpose : uint32_t { kDiCatastrophe = 0, kDiPoisson = 1, kDiPick = 2 };

struct Philox4 {
    uint32_t v[4];
};

__host__ __device__ inline Philox4 philox4x32_10(Philox4 c, uint32_t k0, uint32_t k1) {
    for (int r = 0; r < 10; ++r) {
        if (r > 0) {
            k0 += kPhiloxW0;
            k1 += kPhiloxW1;
        }
        const uint64_t p0 = (uint64_t)kPhiloxM0 * c.v[0], p1 = (uint64_t)kPhiloxM1 * c.v[2];
        const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
        c = Philox4{{hi1 ^ c.v[1] ^ k0, lo1, hi0 ^ c.v[3] ^ k1, lo0}};
    }
    return c;
}

// the uniform draw in [0, 1) of (i, purpose) in call `call` of stream `seed`: the top 53 bits of (w1 << 32 | w0)
__host__ __device__ inline double philox_uniform(uint64_t seed, uint64_t call, uint32_t i, uint32_t purpose) {
    const Philox4 w = philox4x32_10(Philox4{{i, purpose, (uint32_t)call, (uint32_t)(call >> 32)}}, (uint32_t)seed,
                                    (uint32_t)(seed >> 32));
    return (double)((((uint64_t)w.v[1] << 32) | w.v[0]) >> 11) * 0x1.0p-53;
}

} // namespace skb
