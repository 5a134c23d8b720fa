// Continuous batching of windowed canvases (sr3_wstream_*): every request is a canvas of any size whose windows take one slot each of an
// engine's batch; all windows of a request run at the request's own timestep, windows of different requests share the batch.  The
// engine's step graph runs unchanged in its UNet.forward form (eps into eps_buf, noise level of slot s = nl_buf[s]); three kernels stand
// around it:
//   wstream_gather_kernel  crops of each slot's canvas x_t and condition -> the engine's bf16 NHWC input and fp32 x_state; nl_buf per slot
//   wstream_means_kernel   eps + x_t of every active slot -> its clipped posterior mean at its request's t (the means arena)
//   wstream_merge_kernel   the window means blended per canvas pixel, + sigma_t * z -> the canvas x_{t-1}; advances the request table
// Every request carries its own noise schedule (the engine's tables, or tables registered with sr3_wstream_add_schedule), so requests on
// different schedules share the batch: the three kernels read the schedule of each slot's request, never one of the step.
#pragma once
#include "aux_kernels.cuh"

namespace sr3 {

// One request: a canvas the caller owns, and the schedule it samples on.  The host keeps an exact mirror: a request on a schedule of
// T steps takes exactly T steps.
struct WStreamReq {
    int t;                        // timestep of the request's next step while active; -1 once it has finished
    int active;                   // 1: the request's windows run
    unsigned long long sample;    // global sample index (its Philox draws are keyed by it, as the windowed sampler's image 0 is)
    float* x;                     // canvas x_t [C][H][W], overwritten with x_{t-1} every step (borrowed)
    const float* cond;            // canvas condition [cond_c][H][W] (borrowed)
    int H, W, ny, nx;             // canvas size and window grid
    const float* tab;             // its schedule's [5][tab_T] table (sqrt_recip_ac, sqrt_recipm1_ac, post_coef1, post_coef2, post_logvar)
    const float* nl_table;        // its schedule's fp32(sqrt_alphas_cumprod_prev) [T + 1]
    int tab_T;                    // row stride of tab (>= the schedule's T)
};

// One slot: the window of a request it runs.  Written by the host only (admission and retirement).
struct WStreamSlot {
    int req;                      // request record, -1: idle
    int iy, ix;                   // window row and column in the request's grid
};

// The request table is double-buffered: every kernel of a step reads `cur`; block 0 of the merge writes the advanced table into `next`,
// which the following step reads.  Per-record geometry lives in fixed regions of `geo_stride` entries per record (a request has at most
// B windows, so ny, nx <= B): oy / ox / slot_of [rec][B], wy [rec][B][wh], wx [rec][B][ww] -- the windowed sampler's host-built tables.
struct WStreamStep {
    const WStreamReq* cur;
    WStreamReq* next;
    const WStreamSlot* slots;     // [B]
    const int* oy; const int* ox; const float* wy; const float* wx;
    const int* slot_of;           // [rec][B]: slot of window iy * nx + ix
    int B, C, cond_c, wh, ww;
    __nv_bfloat16* in_buf;        // the engine's NHWC input, in_ld channels per pixel: [cond | x_t | 0...] (+ low halves lo_off further)
    int in_ld, lo_off;
    float* x_state;               // the engine's [B][C][wh][ww]: x_t of every slot's window
    const float* eps;             // the engine's eps_buf [B][C][wh][ww]
    float* means;                 // [B][C][wh][ww]
    float* nl_buf;                // [B]
    unsigned long long seed;
};

// One thread per (slot, window pixel), every channel.  An active slot gets its window's crop of the canvas (the values window_gather_kernel
// writes for the same window: bf16 of x, and bf16 of x - bf16(x) in precise mode); an idle slot, or one whose request has finished, gets
// zeros, so it never carries non-finite values.  Block 0 sets nl_buf[s] = nl_table[t + 1] of the slot's request's schedule, the value the
// windowed sampler's step at t reads after sr3_engine_set_schedule of that schedule.
__global__ void __launch_bounds__(256) wstream_gather_kernel(const WStreamStep p) {
    pdl_launch_dependents();
    pdl_wait();
    if (blockIdx.x == 0) {
        for (int s = threadIdx.x; s < p.B; s += blockDim.x) {
            const int r = p.slots[s].req;
            if (r >= 0 && p.cur[r].active) p.nl_buf[s] = p.cur[r].nl_table[p.cur[r].t + 1];
        }
    }
    const int wplane = p.wh * p.ww;
    const int nch = p.cond_c + p.C;
    const long long total = static_cast<long long>(p.B) * wplane;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int s = static_cast<int>(i / wplane);
        const int wp = static_cast<int>(i - static_cast<long long>(s) * wplane);
        const WStreamSlot sl = p.slots[s];
        const WStreamReq* r = sl.req >= 0 ? p.cur + sl.req : nullptr;
        const bool on = r != nullptr && r->active;
        long long plane = 0, src = 0;
        const float* x = nullptr; const float* cond = nullptr;
        if (on) {
            const int y = p.oy[sl.req * p.B + sl.iy] + wp / p.ww, xx = p.ox[sl.req * p.B + sl.ix] + wp % p.ww;
            plane = static_cast<long long>(r->H) * r->W;
            src = static_cast<long long>(y) * r->W + xx;
            x = r->x; cond = r->cond;
        }
        __nv_bfloat16* dst = p.in_buf + (static_cast<long long>(s) * wplane + wp) * p.in_ld;
        for (int c0 = 0; c0 < nch; c0 += 2) {
            float v[2];
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const int c = c0 + k;
                v[k] = 0.f;
                if (c >= nch) continue;
                if (on) v[k] = c < p.cond_c ? cond[c * plane + src] : x[(c - p.cond_c) * plane + src];
                if (c >= p.cond_c) p.x_state[(static_cast<long long>(s) * p.C + (c - p.cond_c)) * wplane + wp] = v[k];
            }
            *reinterpret_cast<__nv_bfloat162*>(dst + c0) = __floats2bfloat162_rn(v[0], v[1]);
            if (p.lo_off) *reinterpret_cast<__nv_bfloat162*>(dst + c0 + p.lo_off) = __floats2bfloat162_rn(bf16_residual(v[0]), bf16_residual(v[1]));
        }
    }
}

// One thread per (slot, window pixel), every channel: final_epilogue's (gemm_wgmma.cuh) clipped posterior mean, operation for operation
// (the same separately rounded x0 = c1 x_t - c2 eps, clamp, mean = pc1 x0 + pc2 x_t), at the slot's request's own t.  This is the mean the
// windowed sampler's engine writes for the same window.  The coefficients are the request's schedule's.
__global__ void __launch_bounds__(256) wstream_means_kernel(const WStreamStep p) {
    pdl_launch_dependents();
    pdl_wait();
    const int wplane = p.wh * p.ww;
    const long long total = static_cast<long long>(p.B) * wplane;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int s = static_cast<int>(i / wplane);
        const int wp = static_cast<int>(i - static_cast<long long>(s) * wplane);
        const int r = p.slots[s].req;
        if (r < 0 || !p.cur[r].active) continue;
        const int t = p.cur[r].t;
        const float* tab = p.cur[r].tab;
        const int tT = p.cur[r].tab_T;
        const float c1 = tab[t], c2 = tab[tT + t], pc1 = tab[2 * tT + t], pc2 = tab[3 * tT + t];
        for (int c = 0; c < p.C; ++c) {
            const long long idx = (static_cast<long long>(s) * p.C + c) * wplane + wp;
            const float xt = p.x_state[idx];
            float x0 = __fsub_rn(__fmul_rn(c1, xt), __fmul_rn(c2, p.eps[idx]));
            x0 = fminf(fmaxf(x0, -1.0f), 1.0f);
            p.means[idx] = __fadd_rn(__fmul_rn(pc1, x0), __fmul_rn(pc2, xt));
        }
    }
}

// One thread per (slot, window pixel): a launch shape fixed by the engine, whatever the canvases.  The thread writes canvas pixel p only if
// its window OWNS p -- along each axis the window with the largest origin <= p, which covers p -- so every pixel of a running canvas is
// written exactly once.  The covering windows are accumulated as window_merge_kernel does (ascending window index, separately rounded
// products and sums, __fdiv_rn), with z keyed by (seed, the request's sample index, the pixel's index in its canvas, t): the windowed
// sampler's x_{t-1} of image 0 bit for bit; sigma_t is the request's schedule's.  Block 0 advances the request table into `next`.
__global__ void __launch_bounds__(256) wstream_merge_kernel(const WStreamStep p) {
    pdl_launch_dependents();
    pdl_wait();
    if (blockIdx.x == 0) {
        for (int k = threadIdx.x; k < p.B; k += blockDim.x) {
            WStreamReq e = p.cur[k];
            if (e.active && --e.t < 0) e.active = 0;
            p.next[k] = e;
        }
    }
    const int wplane = p.wh * p.ww;
    const long long total = static_cast<long long>(p.B) * wplane;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int s = static_cast<int>(i / wplane);
        const int wp = static_cast<int>(i - static_cast<long long>(s) * wplane);
        const WStreamSlot sl = p.slots[s];
        if (sl.req < 0) continue;
        const WStreamReq* r = p.cur + sl.req;
        if (!r->active) continue;
        const int* oy = p.oy + sl.req * p.B;
        const int* ox = p.ox + sl.req * p.B;
        const int ny = r->ny, nx = r->nx;
        const int y = oy[sl.iy] + wp / p.ww, x = ox[sl.ix] + wp % p.ww;
        if ((sl.iy + 1 < ny && oy[sl.iy + 1] <= y) || (sl.ix + 1 < nx && ox[sl.ix + 1] <= x)) continue;    // a later window owns it
        const float* wy = p.wy + static_cast<long long>(sl.req) * p.B * p.wh;
        const float* wx = p.wx + static_cast<long long>(sl.req) * p.B * p.ww;
        const int* slot_of = p.slot_of + sl.req * p.B;
        float num[4] = {0.f, 0.f, 0.f, 0.f}, den = 0.f;
        for (int iy = 0; iy < ny; ++iy) {
            const int dy = y - oy[iy];
            if (dy < 0 || dy >= p.wh) continue;
            const float wyv = wy[iy * p.wh + dy];
            for (int ix = 0; ix < nx; ++ix) {
                const int dx = x - ox[ix];
                if (dx < 0 || dx >= p.ww) continue;
                const float w = __fmul_rn(wyv, wx[ix * p.ww + dx]);
                const float* m = p.means + static_cast<long long>(slot_of[iy * nx + ix]) * p.C * wplane + dy * p.ww + dx;
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (c < p.C) num[c] = __fadd_rn(num[c], __fmul_rn(w, m[c * wplane]));
                den = __fadd_rn(den, w);
            }
        }
        const int t = r->t;
        const float sigma = posterior_sigma(r->tab, r->tab_T, t);
        const long long plane = static_cast<long long>(r->H) * r->W;
        const long long pix = static_cast<long long>(y) * r->W + x;
        float z[4] = {0.f, 0.f, 0.f, 0.f};
        if (t > 0) sampling_noise4(p.seed, r->sample, static_cast<uint32_t>(pix), t, z);
        float* xo = r->x;
#pragma unroll
        for (int c = 0; c < 4; ++c)
            if (c < p.C) xo[c * plane + pix] = posterior_sample(__fdiv_rn(num[c], den), z[c], sigma);
    }
}

}  // namespace sr3
