// philox.cuh -- the counter-based generator Philox4x32-10 (Salmon, Moraes, Dror and Shaw, "Parallel random numbers: as easy as
// 1, 2, 3", SC 2011) and the Box-Muller normals of mppi()'s noise (DESIGN.md 4.5.2), compiled for the sm_90a kernels (mppi.cu)
// and for the host harness (tests/host_harness/mppi_host.cpp).  Integer arithmetic only up to the uniforms, so the words are the
// same on both; the normals use the platform's log, sqrt, cos and sin (a few ulp apart between the two).
#pragma once
#include <stdint.h>
#include <math.h>
#include "quad_core.cuh"

namespace qs {

constexpr uint32_t kPhiloxM0 = 0xD2511F53u, kPhiloxM1 = 0xCD9E8D57u;   // multipliers
constexpr uint32_t kPhiloxW0 = 0x9E3779B9u, kPhiloxW1 = 0xBB67AE85u;   // key increments (golden ratio, sqrt(3) - 1)

QS_HD void mulhilo32(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
    const uint64_t p = (uint64_t)a * (uint64_t)b;
    hi = (uint32_t)(p >> 32);
    lo = (uint32_t)p;
}

// out = Philox4x32-10(ctr, key): ten rounds, the key bumped between rounds
QS_HD void philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) {
    uint32_t c0 = ctr[0], c1 = ctr[1], c2 = ctr[2], c3 = ctr[3], k0 = key[0], k1 = key[1];
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r > 0) {
            k0 += kPhiloxW0;
            k1 += kPhiloxW1;
        }
        uint32_t hi0, lo0, hi1, lo1;
        mulhilo32(kPhiloxM0, c0, hi0, lo0);
        mulhilo32(kPhiloxM1, c2, hi1, lo1);
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// u = (x + 0.5) 2^-53 in (0, 1] from the top 53 bits x of the 64-bit word (hi << 32) | lo
QS_HD double philox_uniform(uint32_t hi, uint32_t lo) {
    const uint64_t x = (((uint64_t)hi << 32) | (uint64_t)lo) >> 11;
    return ((double)x + 0.5) * 1.1102230246251565404e-16;                            // 2^-53
}

// Box-Muller: the uniforms of (w0, w1) and (w2, w3) -> sqrt(-2 ln u_a) (cos 2 pi u_b, sin 2 pi u_b)
QS_HD void box_muller(const uint32_t w[4], double& z0, double& z1) {
    const double ua = philox_uniform(w[0], w[1]), ub = philox_uniform(w[2], w[3]);
    const double r = sqrt(-2.0 * log(ua));
    const double a = (2.0 * 3.14159265358979323846) * ub;
    z0 = r * cos(a);
    z1 = r * sin(a);
}

}  // namespace qs
