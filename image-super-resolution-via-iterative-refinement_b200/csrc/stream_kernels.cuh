// Continuous batching (sr3_stream_*): every slot of an engine's batch carries its own request at its own timestep.  The engine's step
// graph runs unchanged in its UNet.forward form (eps into eps_buf, noise level of image b = nl_buf[b]); one kernel after it applies the
// posterior update of p_sample (diffusion.py:169-174) slot by slot and advances the slot table:
//   slot_update_kernel  eps + x_t of every active slot -> x_{t-1} (x_state and the bf16 UNet input), t_s -= 1, nl_buf[s] for the next step
#pragma once
#include "aux_kernels.cuh"

namespace sr3 {

// One slot of a stream.  The host keeps an exact mirror: every request takes exactly T steps.
struct StreamSlot {
    int t;                        // timestep of the slot's next step while active; -1 once its request has finished
    int active;                   // 1: the slot runs a request
    unsigned long long sample;    // global sample index of the request (its Philox draws are keyed by it, as sample_offset + b is)
};

// The slot table is double-buffered: a launch reads `cur` in every block and block 0 writes the advanced table into `next`, which the
// following launch reads.  No block can see a half-advanced table.
struct SlotUpdate {
    const float* eps;             // the engine's eps_buf [B][C][H][W]
    float* x_state;               // [B][C][H][W]: x_t in, x_{t-1} out
    __nv_bfloat16* in_buf;        // the engine's NHWC bf16 UNet input: in_ld channels per pixel, x_t at [in_coff, in_coff + C)
    int in_ld, in_coff, lo_off;   // lo_off: precise mode, the low halves lo_off channels further; 0 = bf16 mode
    const float* tab;             // the engine's [5][tab_T] schedule table
    int tab_T;
    const float* nl_table;        // fp32(sqrt_alphas_cumprod_prev) [T + 1]
    float* nl_buf;                // [B]: noise level of each slot's next step
    const StreamSlot* cur;
    StreamSlot* next;
    unsigned long long seed;
    int B, C, H, W;
};

// One thread per (slot, pixel), all (<= 4) channels.  The arithmetic is final_epilogue's (gemm_wgmma.cuh) operation for operation: the
// same separately rounded products and differences, the same clamp, the same Philox draw at the same counter, the same bf16 split of
// x_{t-1}; so a slot reproduces the image the lockstep sampler computes for the same input, noise level and sample index bit for bit.
__global__ void __launch_bounds__(256) slot_update_kernel(const SlotUpdate p) {
    pdl_launch_dependents();
    pdl_wait();
    if (blockIdx.x == 0) {
        for (int s = threadIdx.x; s < p.B; s += blockDim.x) {
            StreamSlot e = p.cur[s];
            if (e.active) {
                e.t -= 1;
                if (e.t < 0) e.active = 0;
                else p.nl_buf[s] = p.nl_table[e.t + 1];      // the value the lockstep step at timestep e.t reads (embed_kernel)
            }
            p.next[s] = e;
        }
    }
    const long long plane = static_cast<long long>(p.H) * p.W;
    const long long total = plane * p.B;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int b = static_cast<int>(i / plane);
        const StreamSlot e = p.cur[b];
        if (!e.active) continue;
        const long long pix = i - b * plane;
        const int t = e.t;
        const float c1 = p.tab[t], c2 = p.tab[p.tab_T + t], pc1 = p.tab[2 * p.tab_T + t], pc2 = p.tab[3 * p.tab_T + t];
        const float sigma = posterior_sigma(p.tab, p.tab_T, t);
        float z[4] = {0.f, 0.f, 0.f, 0.f};
        if (t > 0) sampling_noise4(p.seed, e.sample, static_cast<uint32_t>(pix), t, z);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            if (c >= p.C) break;
            const long long idx = (static_cast<long long>(b) * p.C + c) * plane + pix;
            const float xt = p.x_state[idx];
            float x0 = __fsub_rn(__fmul_rn(c1, xt), __fmul_rn(c2, p.eps[idx]));
            x0 = fminf(fmaxf(x0, -1.0f), 1.0f);
            const float mean = __fadd_rn(__fmul_rn(pc1, x0), __fmul_rn(pc2, xt));
            const float xn = posterior_sample(mean, z[c], sigma);
            p.x_state[idx] = xn;
            __nv_bfloat16* ib = p.in_buf + (static_cast<long long>(b) * plane + pix) * p.in_ld + p.in_coff + c;
            const __nv_bfloat16 hi = __float2bfloat16_rn(xn);
            *ib = hi;
            if (p.lo_off) ib[p.lo_off] = __float2bfloat16_rn(xn - __bfloat162float(hi));
        }
    }
}

}  // namespace sr3
