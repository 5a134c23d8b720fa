// Windowed sampling (sr3_windowed_*): a canvas of any size is denoised by overlapping windows of a size the UNet plan supports, and the
// windows are merged INSIDE every reverse step -- the canvas keeps one x_t and draws one noise value per pixel; the windows contribute
// their posterior means only.  Two kernels stand around the engine's step graph:
//   window_gather_kernel  crops of the canvas x_t and of the condition -> the engine's bf16 NHWC input buffer and fp32 x_state
//   window_merge_kernel   weighted average of the window means per canvas pixel, + sigma_t * z -> the canvas x_{t-1} (and a snapshot)
//   window_solver_merge_kernel   the DPM-Solver++(2M) form of the merge: the windows' means are their clipped x0 (the engine runs with
//                         pc1 = 1, pc2 = 0), blended alike, then x_{k-1} = A x_k + B x0 + C x0_prev; x0 is kept for the next step
#pragma once
#include "aux_kernels.cuh"

namespace sr3 {

// Canvas [B][C][H][W] covered by ny x nx windows of wh x ww per image; window n of the list = image n / (ny nx), row (n / nx) % ny,
// column n % nx.  Blend weight of window pixel (y, x) = wy[iy][y] * wx[ix][x] (host-built from the geometry alone).
struct WindowGeom {
    int B, C, H, W;
    int wh, ww, ny, nx;
    const int* oy; const int* ox;        // [ny], [nx] window origins
    const float* wy; const float* wx;    // [ny][wh], [nx][ww]
};

// Device-resident control block of a canvas: what changes between launches of its captured step graph.  `step` is advanced by
// step_begin_kernel exactly like an engine's; of its fields the canvas uses t_cur / t_next, use_noise_buf, seed and sample_offset.
struct WindowCtl {
    StepCtl step;
    float* snapshots;        // optional [snapshot_cap][B][C][H][W]
    int snapshot_cap;
    int T;                   // n_timestep of the schedule (decides which steps are snapshots)
};

struct WindowGather {
    WindowGeom g;
    const float* cond;       // canvas condition [B][cond_c][H][W] (nullptr when cond_c == 0)
    const float* x;          // canvas x_t [B][C][H][W]
    int first, n_total, Bw;  // this pass runs windows [first, first + Bw) of n_total; slots past the end repeat the last window
    __nv_bfloat16* in_buf;   // engine input, NHWC, in_ld channels per pixel: [cond | x_t | 0...] (+ the low halves lo_off further, precise mode)
    int in_ld, cond_c, lo_off;
    float* x_state;          // engine state [Bw][C][wh][ww]: the x_t the posterior epilogue reads
    const WindowCtl* wctl;
    StepCtl* ectl;           // the engine's control block: its next step runs at the canvas's current timestep
};

// One thread per (slot, window row, group of 4 pixels along W) and per pair of channels.  A group is read with one 16-byte load per channel
// when the canvas rows keep it aligned (W % 4 == 0 and a window origin that is a multiple of 4); any other origin or canvas width falls
// back to four scalar loads of the same values.  Writes are always aligned: ww is a power of two >= 4.
__global__ void __launch_bounds__(256) window_gather_kernel(const WindowGather p) {
    pdl_launch_dependents();
    pdl_wait();
    const WindowGeom& g = p.g;
    if (blockIdx.x == 0 && threadIdx.x == 0) p.ectl->t_next = p.wctl->step.t_cur;
    const int nch = p.cond_c + g.C;
    const int qpr = g.ww >> 2;
    const long long cplane = static_cast<long long>(g.H) * g.W;
    const int wplane = g.wh * g.ww;
    const int per = g.ny * g.nx;
    const long long total = static_cast<long long>(p.Bw) * g.wh * qpr;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int q = static_cast<int>(i % qpr);
        const int y = static_cast<int>((i / qpr) % g.wh);
        const int slot = static_cast<int>(i / (static_cast<long long>(qpr) * g.wh));
        const int n = min(p.first + slot, p.n_total - 1);
        const int b = n / per, iy = (n % per) / g.nx, ix = n % g.nx;
        const int cx = g.ox[ix] + 4 * q;
        const long long src_row = static_cast<long long>(g.oy[iy] + y) * g.W + cx;
        const bool vec = ((g.W | cx) & 3) == 0;
        const long long wpix = static_cast<long long>(slot) * wplane + y * g.ww + 4 * q;
        for (int c0 = 0; c0 < nch; c0 += 2) {
            float v[2][4];
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const int c = c0 + k;
                if (c >= nch) { v[k][0] = v[k][1] = v[k][2] = v[k][3] = 0.f; continue; }
                const float* src = (c < p.cond_c ? p.cond + (static_cast<long long>(b) * p.cond_c + c) * cplane
                                                 : p.x + (static_cast<long long>(b) * g.C + (c - p.cond_c)) * cplane) + src_row;
                if (vec) {
                    const float4 f = *reinterpret_cast<const float4*>(src);
                    v[k][0] = f.x; v[k][1] = f.y; v[k][2] = f.z; v[k][3] = f.w;
                } else {
#pragma unroll
                    for (int j = 0; j < 4; ++j) v[k][j] = src[j];
                }
                if (c >= p.cond_c)
                    *reinterpret_cast<float4*>(p.x_state + (static_cast<long long>(slot) * g.C + (c - p.cond_c)) * wplane + y * g.ww + 4 * q) =
                        make_float4(v[k][0], v[k][1], v[k][2], v[k][3]);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                __nv_bfloat16* dst = p.in_buf + (wpix + j) * p.in_ld + c0;
                *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(v[0][j], v[1][j]);
                if (p.lo_off) *reinterpret_cast<__nv_bfloat162*>(dst + p.lo_off) = __floats2bfloat162_rn(bf16_residual(v[0][j]), bf16_residual(v[1][j]));
            }
        }
    }
}

struct WindowMerge {
    WindowGeom g;
    const float* means;      // window-mean arena [B * ny * nx][C][wh][ww]: every window covering a merged pixel must be present
    float* x;                // canvas state, overwritten with x_{t-1}
    const float* noise;      // canvas-shaped z of this step (read when step.use_noise_buf)
    const float* tab;        // the engine's [5][tab_T] schedule table
    int tab_T;
    const WindowCtl* ctl;
    const int* band;         // optional [B][2]: only rows [y0, y1) of image b are merged (a rank's band); nullptr: every row
    int band_rows;           // max over images of y1 - y0 (the launch covers B x band_rows x W pixels)
};

// The weighted sum of the means of the windows covering canvas pixel `pix` of image b (num[c], c < C) and the sum of their weights (den):
// windows in ascending index, separately rounded multiplies and adds, so the sum does not depend on the launch shape or on how many
// windows a pass ran.
__device__ __forceinline__ void blend_window_means(const WindowGeom& g, const float* means, int b, long long pix, float (&num)[4], float& den) {
    const int wplane = g.wh * g.ww;
    const int y = static_cast<int>(pix / g.W), x = static_cast<int>(pix - static_cast<long long>(y) * g.W);
    num[0] = num[1] = num[2] = num[3] = 0.f; den = 0.f;
    for (int iy = 0; iy < g.ny; ++iy) {
        const int dy = y - g.oy[iy];
        if (dy < 0 || dy >= g.wh) continue;
        const float wyv = g.wy[iy * g.wh + dy];
        for (int ix = 0; ix < g.nx; ++ix) {
            const int dx = x - g.ox[ix];
            if (dx < 0 || dx >= g.ww) continue;
            const float w = __fmul_rn(wyv, g.wx[ix * g.ww + dx]);
            const float* m = means + (static_cast<long long>(b) * g.ny + iy) * g.nx * g.C * wplane + static_cast<long long>(ix) * g.C * wplane + dy * g.ww + dx;
#pragma unroll
            for (int c = 0; c < 4; ++c)
                if (c < g.C) num[c] = __fadd_rn(num[c], __fmul_rn(w, m[c * wplane]));
            den = __fadd_rn(den, w);
        }
    }
}

// Snapshot slot of the step at t: p_sample_loop keeps x_{t-1} whenever t % (1 | T / 10) == 0 (diffusion.py:179-199), first kept image
// first; nullptr when the step keeps none.
__device__ __forceinline__ float* window_snapshot(const WindowCtl* ctl, int t, long long canvas_elems) {
    const int inter = 1 | (ctl->T / 10);
    const int slot = (ctl->T - 1) / inter - t / inter;
    return (ctl->snapshots != nullptr && t % inter == 0 && slot < ctl->snapshot_cap) ? ctl->snapshots + slot * canvas_elems : nullptr;
}

// One thread per canvas pixel, all (<= 4) channels: the Philox draw of a pixel yields the z of its channels.  The covering windows are found
// from the two per-axis origin tables and accumulated in ascending window index with separately rounded multiplies and adds, so the sum is
// the same whatever the launch shape and however many windows a pass ran: no atomics, repeat runs are bit identical.  With a band table
// a pixel outside its image's band is neither read nor written, so a rank that holds only the means covering its band computes that band.
__global__ void __launch_bounds__(256) window_merge_kernel(const WindowMerge p) {
    pdl_launch_dependents();
    pdl_wait();
    const WindowGeom& g = p.g;
    const StepCtl ctl = p.ctl->step;
    const int t = ctl.t_cur;
    const float sigma = posterior_sigma(p.tab, p.tab_T, t);
    const long long plane = static_cast<long long>(g.H) * g.W;
    float* snap = window_snapshot(p.ctl, t, plane * g.C * g.B);
    const long long bplane = p.band ? static_cast<long long>(p.band_rows) * g.W : plane;
    const long long total = bplane * g.B;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int b = static_cast<int>(i / bplane);
        long long pix = i - b * bplane;
        if (p.band) {
            pix += static_cast<long long>(p.band[2 * b]) * g.W;
            if (pix >= static_cast<long long>(p.band[2 * b + 1]) * g.W) continue;
        }
        float num[4], den;
        blend_window_means(g, p.means, b, pix, num, den);
        float z[4] = {0.f, 0.f, 0.f, 0.f};
        if (t > 0) {
            if (ctl.use_noise_buf) {
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (c < g.C) z[c] = p.noise[(static_cast<long long>(b) * g.C + c) * plane + pix];
            } else {
                sampling_noise4(ctl.seed, ctl.sample_offset + b, static_cast<uint32_t>(pix), t, z);
            }
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            if (c < g.C) {
                const long long idx = (static_cast<long long>(b) * g.C + c) * plane + pix;
                const float xn = posterior_sample(__fdiv_rn(num[c], den), z[c], sigma);
                p.x[idx] = xn;
                if (snap) snap[idx] = xn;
            }
        }
    }
}

struct WindowSolverMerge {
    WindowMerge m;           // geometry, means arena (the windows' clipped x0), canvas x_k, control block, band; noise and tab unused
    float* x0_prev;          // canvas-shaped x0 of the previous step, overwritten with this step's (zero before the first step)
    const float* coef;       // [3][stride]: A, B, C of step index k = t
    int stride;
};

// DPM-Solver++(2M) (data prediction, multistep) on the canvas: x0 is the blend of the windows' clipped x0 (window_merge_kernel's blend and
// division), then x_{k-1} = (A x_k + B x0) + C x0_prev in that order with separately rounded operations, and x0_prev = x0.  No noise.  The
// update is linear and the blend weights sum to 1, so blending x0 and then stepping is stepping every window and blending the results.
__global__ void __launch_bounds__(256) window_solver_merge_kernel(const WindowSolverMerge p) {
    pdl_launch_dependents();
    pdl_wait();
    const WindowGeom& g = p.m.g;
    const int t = p.m.ctl->step.t_cur;
    const float A = p.coef[t], B = p.coef[p.stride + t], Cc = p.coef[2 * p.stride + t];
    const long long plane = static_cast<long long>(g.H) * g.W;
    float* snap = window_snapshot(p.m.ctl, t, plane * g.C * g.B);
    const long long total = plane * g.B;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int b = static_cast<int>(i / plane);
        const long long pix = i - b * plane;
        float num[4], den;
        blend_window_means(g, p.m.means, b, pix, num, den);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            if (c < g.C) {
                const long long idx = (static_cast<long long>(b) * g.C + c) * plane + pix;
                const float x0 = __fdiv_rn(num[c], den);
                const float xn = __fadd_rn(__fadd_rn(__fmul_rn(A, p.m.x[idx]), __fmul_rn(B, x0)), __fmul_rn(Cc, p.x0_prev[idx]));
                p.x0_prev[idx] = x0;
                p.m.x[idx] = xn;
                if (snap) snap[idx] = xn;
            }
        }
    }
}

}  // namespace sr3
