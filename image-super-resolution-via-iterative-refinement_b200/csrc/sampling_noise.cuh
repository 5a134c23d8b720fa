// The sampler's random draw and the last line of p_sample (diffusion.py:169-174), shared by the posterior epilogue of the tile kernel
// (gemm_wgmma.cuh) and the windowed sampler's merge (window_kernels.cuh): both add sigma_t * z through the same device functions, so the two
// samplers round alike and a one-window canvas reproduces the plain sampler bit for bit.
#pragma once
#include <cstdint>

namespace sr3 {

// ---------------------------------------------------------------- Philox4x32-10 + Box-Muller
__device__ __forceinline__ void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
        const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
        c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
}
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
    const float u1 = (static_cast<float>(a) + 1.0f) * 2.3283064365386963e-10f;   // (0, 1]
    const float u2 = static_cast<float>(b) * 2.3283064365386963e-10f;            // [0, 1)
    const float r = sqrtf(-2.0f * logf(u1));
    float s, c;
    sincospif(2.0f * u2, &s, &c);
    z0 = r * c; z1 = r * s;
}

// z of the (up to four) channels of one pixel at timestep t: counter (pixel, sample index low, t, sample index high), key = seed.
// `sample` is the GLOBAL index of the image, `pix` the pixel's index in the image being sampled (for a windowed canvas: in the canvas).
__device__ __forceinline__ void sampling_noise4(unsigned long long seed, unsigned long long sample, uint32_t pix, int t, float (&z)[4]) {
    uint32_t ctr[4] = {pix, static_cast<uint32_t>(sample), static_cast<uint32_t>(t), static_cast<uint32_t>(sample >> 32)};
    philox4x32_10(ctr, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
    box_muller(ctr[0], ctr[1], z[0], z[1]);
    box_muller(ctr[2], ctr[3], z[2], z[3]);
}

// sigma_t = exp(0.5 * posterior_log_variance_clipped[t]) for t > 0, 0 at the last step; tab: the [5][T] schedule table, row 4 = log-variance
__device__ __forceinline__ float posterior_sigma(const float* tab, int T, int t) { return (t > 0) ? expf(0.5f * tab[4 * T + t]) : 0.0f; }
// x_{t-1} = mean + sigma_t * z, two separately rounded operations (never contracted into a fused multiply-add)
__device__ __forceinline__ float posterior_sample(float mean, float z, float sigma) { return __fadd_rn(mean, __fmul_rn(z, sigma)); }

}  // namespace sr3
