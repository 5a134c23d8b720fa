// Kernels of the TRAINING path (reference: model/model.py:48-58 optimize_parameters, model/sr3_modules/diffusion.py:221-246 p_losses):
// everything the backward pass needs that is not the forward tile kernel.
//
//   * data gradients of every conv are the forward tile kernel (gemm_wgmma.cuh) on re-packed weights (mirrored taps for 3x3 stride 1,
//     the four output-parity phases for the stride-2 Downsample conv, a 4x4 stride-2 kernel for nearest-2x + conv3x3), packed by pack_entry
//     (the end of this file), which also packs every forward weight;
//   * weight gradients are a wgmma GEMM that contracts over PIXELS with both operands MN-major (wgrad_kernel);
//   * GroupNorm + SiLU (+ Dropout) backward, bias / FiLM / noise-MLP gradients, attention backward, loss gradient, Adam.
#pragma once
#include "aux_kernels.cuh"

namespace sr3 {

// ------------------------------------------------------------------------------------------------ weight gradient (wgmma, MN-major operands)
//     dW[co][tap][ci] = sum over pixels p of  dY[p][co] * X[p + tap][ci]
// The contraction runs over PIXELS.  With NHWC activations both operands are MN-major (channels contiguous): a TMA box {64 channels, 8 x 8
// pixels} with the 128-byte swizzle IS the canonical MN-major layout of a wgmma shared-memory operand: one 128 B row = 64 channels of one
// pixel, 8 pixels = one 1024 B atom, and a K step of 16 pixels is two atoms.  A tap is the X box shifted (TMA zero fill = padding); the
// stride-2 conv reads X through the parity view of the forward kernel.
// One CTA = (128 output channels, 64 input channels, a group of <= 3 taps, a slice of the 8x8-pixel patches): warpgroup g owns output
// channels [64 g, 64 g + 64) and holds <= 3 accumulators of 64 x 64 fp32 in registers, written as a partial tile into
// ws[slice][co][tap][ci]; wgrad_reduce_kernel sums the slices (fixed order: deterministic) and writes the parameter gradient in the
// reference's OIHW layout.
constexpr int WGRAD_THREADS = 288;                      // warps 0..7: two consumer warpgroups, warp 8: TMA producer
constexpr int WGRAD_STAGES = 4;
constexpr int WGRAD_STAGE_BYTES = 16384 + 3 * 8192;     // dY: 2 panels of 64 co x 64 px | X: 3 taps x (64 px x 64 ci)
constexpr int WGRAD_SMEM_BYTES = 1024 + WGRAD_STAGES * WGRAD_STAGE_BYTES + 256;
constexpr int WGRAD_MAX_TAPS = 9;

struct WgradTap { int dchan, dw, p, dh; };
struct WgradParams {
    CUtensorMap dy_map;      // 5-D bf16 (Cout, OW, 1, OH, B), box {64, 8, 1, 8, 1}
    CUtensorMap x_map;       // 5-D bf16 view of X, box {64, 8, 1, 8, 1}
    float* ws;               // partial tiles: ws[slice * ws_slice_stride + co * ws_row_stride + tap * Cin + ci]  (default [slices][co_pad][ntaps][Cin])
    long long ws_slice_stride, ws_row_stride;
    int Cin, co_pad, cout_valid, OH, OW, B;   // OH, OW: the patch grid in pixels (8 for a 4x4 output: one patch, zero outside the image)
    int ntaps, taps_per_cta;
    int patches;             // B * (OH/8) * (OW/8)
    int slices;
    WgradTap taps[WGRAD_MAX_TAPS];
};

__global__ void __launch_bounds__(WGRAD_THREADS, 1) wgrad_kernel(const __grid_constant__ WgradParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    const uint32_t bar_base = base + WGRAD_STAGES * WGRAD_STAGE_BYTES;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (WGRAD_STAGES + s); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_ci = p.Cin / 64;
    const int co0 = (blockIdx.x / n_ci) * 128, ci0 = (blockIdx.x % n_ci) * 64;
    const int tap0 = blockIdx.y * p.taps_per_cta;
    const int nt = min(p.taps_per_cta, p.ntaps - tap0);
    const int slice = blockIdx.z;
    const int it_begin = static_cast<int>((static_cast<long long>(p.patches) * slice) / p.slices);
    const int it_end = static_cast<int>((static_cast<long long>(p.patches) * (slice + 1)) / p.slices);
    const int iters = it_end - it_begin;
    const int tiles_w = p.OW / 8, tiles_h = p.OH / 8;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.dy_map);
        tma_prefetch_desc(&p.x_map);
        for (int s = 0; s < WGRAD_STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 2); }   // empty: one arrive per warpgroup
        fence_mbar_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();

    if (warp == 8) {
        int s = 0;
        uint32_t ph = 0;
        for (int it = it_begin; it < it_end; ++it) {
            const int b = it / (tiles_w * tiles_h);
            const int r = it % (tiles_w * tiles_h);
            const int w0 = (r % tiles_w) * 8, h0 = (r / tiles_w) * 8;
            mbar_wait(empty_bar(s), ph ^ 1u);
            if (elect_one_sync()) {
                const uint32_t dst = base + s * WGRAD_STAGE_BYTES;
                mbar_arrive_expect_tx(full_bar(s), 16384 + nt * 8192);
                tma_load_5d(dst, &p.dy_map, full_bar(s), co0, w0, 0, h0, b);
                tma_load_5d(dst + 8192, &p.dy_map, full_bar(s), co0 + 64, w0, 0, h0, b);
                for (int t = 0; t < nt; ++t) {       // X box of tap t; out-of-image pixels arrive as zeros (= padding)
                    const WgradTap& tp = p.taps[tap0 + t];
                    tma_load_5d(dst + 16384 + t * 8192, &p.x_map, full_bar(s), ci0 + tp.dchan, w0 + tp.dw, tp.p, h0 + tp.dh, b);
                }
            }
            __syncwarp();
            if (++s == WGRAD_STAGES) { s = 0; ph ^= 1u; }
        }
    } else if (warp < 8) {
        // warpgroup g: output channels [co0 + 64 g, co0 + 64 g + 64); one 64 x 64 accumulator per tap (each tap's X box is one MN panel)
        const int g = warp >> 2;
        const bool leader = (threadIdx.x & 127) == 0;
        float acc[3][32];
#pragma unroll
        for (int t = 0; t < 3; ++t)
#pragma unroll
            for (int j = 0; j < 32; ++j) acc[t][j] = 0.f;
        int s = 0, prev = -1;
        uint32_t ph = 0;
        for (int it = 0; it < iters; ++it) {
            mbar_wait(full_bar(s), ph);
            const uint32_t st = base + s * WGRAD_STAGE_BYTES;
            // one branch-free wgmma chain per tap count (a branch between two wgmma makes ptxas re-fence or serialise them)
            auto issue = [&](auto nt_c) {
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {                   // 16 pixels = two 8-pixel atoms per wgmma
                    const uint64_t adesc = wgmma_desc_sw128(st + g * 8192 + kk * 2048, 1024, 1024);
#pragma unroll
                    for (int t = 0; t < decltype(nt_c)::value; ++t)
                        Wgmma<64>::template mma<1, 1>(acc[t], adesc, wgmma_desc_sw128(st + 16384 + t * 8192 + kk * 2048, 1024, 1024), (it | kk) != 0);
                }
                wgmma_commit();
            };
            if (nt == 3) issue(std::integral_constant<int, 3>{});
            else if (nt == 2) issue(std::integral_constant<int, 2>{});
            else issue(std::integral_constant<int, 1>{});
            if (prev >= 0) {
                wgmma_wait<1>();
                mbar_arrive_if(empty_bar(prev), leader);
            }
            prev = s;
            if (++s == WGRAD_STAGES) { s = 0; ph ^= 1u; }
        }
        wgmma_wait<0>();
#pragma unroll
        for (int t = 0; t < 3; ++t) wgmma_fence_regs(acc[t]);
        // register j of a thread: output channel row 16 (warp % 4) + lane / 4 + 8 ((j / 2) % 2), input channel 8 (j / 4) + 2 (lane % 4) + j % 2
#pragma unroll
        for (int t = 0; t < 3; ++t) {
            if (t >= nt) continue;
#pragma unroll
            for (int j = 0; j < 32; j += 2) {
                const int co = co0 + 64 * g + 16 * (warp & 3) + (lane >> 2) + 8 * ((j >> 1) & 1);
                if (co >= p.cout_valid) continue;               // padded rows of the 128-row tile (Cout = 64 / 3): nobody reads them
                const int ci = 8 * (j >> 2) + 2 * (lane & 3);
                *reinterpret_cast<float2*>(p.ws + slice * p.ws_slice_stride + co * p.ws_row_stride + static_cast<long long>(tap0 + t) * p.Cin + ci0 + ci) =
                    make_float2(acc[t][j], acc[t][j + 1]);
            }
        }
    }
}

// grad[co][ci][tap] (OIHW) = gscale * sum over slices of ws[slice][co][tap][ci]   (ci < cin_valid, co < cout_valid).
// One block per (co, chunk of input channels): its eight warps are split into `sw` slice lanes x 8/sw groups of 32 input channels (sw = 8, 4,
// 2 or 1 by the slice count, so no warp idles); a warp sums its slices for every tap of its 32 channels (coalesced 128 B rows, nine independent
// loads in flight), the partial sums meet in shared memory laid out [ci][tap] = the OIHW order, are added in warp order (deterministic) and
// written as one contiguous span.  (Finalising inside wgrad_kernel by the last-arriving CTA of a tile was measured slower: its 4-byte stores
// at a 36-byte stride and the serial tail cost more than the launch they save.)
// first index i in [0, n) with ends[i] > b  (ends ascending): which table entry owns block b
__device__ __forceinline__ int find_entry(const int* __restrict__ ends, int n, int b) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(&ends[mid]) > b) hi = mid; else lo = mid + 1;
    }
    return lo;
}
// Table-driven: ONE launch reduces the partial tiles of every weight-gradient kernel that ran since the last flush (the layers of a gradient
// bucket): blocks find their entry by its block-offset range.
struct WgradReduceDesc {
    const float* ws; float* grad;
    int slices, co_pad, ntaps, Cin, cout_valid, cin_valid, sw, blocks_x;
    int block_begin, block_end;            // this entry's blocks inside the flush it belongs to are [block_begin, block_end) minus the flush's first block
};
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const WgradReduceDesc* __restrict__ tab, const int* __restrict__ block_ends, int first, int count, int block_base,
                                                           float gscale) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float sm[8][32 * WGRAD_MAX_TAPS];
    const WgradReduceDesc d = tab[first + find_entry(block_ends + first, count, block_base + blockIdx.x)];
    const int lb = block_base + blockIdx.x - d.block_begin;
    const int bx = lb % d.blocks_x, co = lb / d.blocks_x;
    const int sw = d.sw, ntaps = d.ntaps;
    const int groups = 8 / sw;                       // 32-channel groups per block
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int grp = w / sw, sl = w % sw;
    const int ci0 = bx * 32 * groups;
    const int ci = ci0 + grp * 32 + lane;
    const long long sstride = static_cast<long long>(d.co_pad) * ntaps * d.Cin;
    float acc[WGRAD_MAX_TAPS];
#pragma unroll
    for (int t = 0; t < WGRAD_MAX_TAPS; ++t) acc[t] = 0.f;
    if (ci < d.cin_valid) {
        const float* s = d.ws + static_cast<long long>(co) * ntaps * d.Cin + ci;
        for (int k = sl; k < d.slices; k += sw) {
#pragma unroll
            for (int t = 0; t < WGRAD_MAX_TAPS; ++t)
                if (t < ntaps) acc[t] += __ldcg(&s[k * sstride + static_cast<long long>(t) * d.Cin]);
        }
    }
#pragma unroll
    for (int t = 0; t < WGRAD_MAX_TAPS; ++t)
        if (t < ntaps) sm[w][lane * ntaps + t] = acc[t];
    __syncthreads();
    const int nci = min(32 * groups, d.cin_valid - ci0);
    float* g = d.grad + (static_cast<long long>(co) * d.cin_valid + ci0) * ntaps;
    for (int i = threadIdx.x; i < nci * ntaps; i += blockDim.x) {
        const int gi = i / (32 * ntaps), r = i - gi * 32 * ntaps;      // channel group, position inside its [32][ntaps] slab
        float a = 0.f;
        for (int k = 0; k < sw; ++k) a += sm[gi * sw + k][r];
        g[i] = a * gscale;
    }
}

// ------------------------------------------------------------------------------------------------ GroupNorm (+SiLU, +Dropout) backward
// forward (unet.py:80-91):  xh = (x - mean_g) rstd_g,  y = gamma xh + beta,  a = drop(silu(y));   given dA:
//   d   = dA * drop' * silu'(y)                     S1[b][c] = sum_p d,   S2[b][c] = sum_p d xh          (pass 1: gn_bwd_reduce_kernel)
//   dx  = rstd_g (gamma d - m1_g - xh m2_g),        m1_g = sum_{c in g} gamma_c S1 / n,  m2_g = sum_{c in g} gamma_c S2 / n   (pass 2)
//   dgamma_c = sum_b S2[b][c],  dbeta_c = sum_b S1[b][c]
struct GnBwdParams {
    PrepParams f;            // the forward op (sources, statistics, gamma / beta, groups, HW, silu, eps); B = images
    const float* dA;         // [B][HW][C]
    const DropSpec* drop;    // optional
    float* sums;             // [B][C][2], zero before pass 1
    const float* add;        // optional fp32 [B][HW][add_ld]: gradient reaching x along another path (residual / shortcut conv), added to dx
    int add_ld;
    float* dst0; int acc0; __nv_bfloat16* dst0_b; float* gsum0; int gsum_ld0;    // gradient of source 0: [B][HW][C0]; acc: dst += ; gsum[b * ld + c] += column sums
    float* dst1; int acc1; __nv_bfloat16* dst1_b; float* gsum1; int gsum_ld1;    // source 1 (skip connection)
    const float* mr;         // [B][groups][2] (mean, rstd) saved by the forward's GroupNorm apply (prep_kernel's save_mr)
    float* dgamma; float* dbeta; float gscale;   // pass 2, block (0, 0): dgamma[c] = gscale sum_b S2[b][c], dbeta[c] = gscale sum_b S1[b][c]
};

// shared memory: gm[groups] | gr[groups] | m1[groups] | m2[groups] | red[2*C] floats
__host__ __device__ constexpr int gn_bwd_smem_bytes(int C, int groups) { return 4 * groups * 4 + 2 * C * 4; }

template <bool APPLY>
__global__ void __launch_bounds__(512) gn_bwd_kernel(const GnBwdParams p) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float smf[];
    const PrepParams& f = p.f;
    const int C = f.C0 + f.C1;
    const int gs = C / f.groups;
    float* gm = smf;
    float* gr = gm + f.groups;
    float* m1 = gr + f.groups;
    float* m2 = m1 + f.groups;
    float* red = m2 + f.groups;                    // [2C]
    const int b = blockIdx.y;
    for (int g = threadIdx.x; g < f.groups; g += blockDim.x) {
        gm[g] = __ldcg(&p.mr[(static_cast<long long>(b) * f.groups + g) * 2]);
        gr[g] = __ldcg(&p.mr[(static_cast<long long>(b) * f.groups + g) * 2 + 1]);
    }
    __syncthreads();
    if (APPLY) {
        if (blockIdx.x == 0 && blockIdx.y == 0 && (p.dgamma != nullptr || p.dbeta != nullptr)) {
            for (int c = threadIdx.x; c < C; c += blockDim.x) {
                float a = 0.f, q = 0.f;
                for (int bb = 0; bb < f.B; ++bb) { a += __ldcg(&p.sums[(static_cast<long long>(bb) * C + c) * 2]); q += __ldcg(&p.sums[(static_cast<long long>(bb) * C + c) * 2 + 1]); }
                if (p.dgamma) p.dgamma[c] = q * p.gscale;
                if (p.dbeta) p.dbeta[c] = a * p.gscale;
            }
        }
        // group means of gamma * S1, gamma * S2
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            const float g = __ldg(&f.gamma[c]);
            red[c] = g * __ldcg(&p.sums[(static_cast<long long>(b) * C + c) * 2]);
            red[C + c] = g * __ldcg(&p.sums[(static_cast<long long>(b) * C + c) * 2 + 1]);
        }
        __syncthreads();
        const float inv = 1.0f / (static_cast<float>(gs) * static_cast<float>(f.HW));
        for (int g = threadIdx.x; g < f.groups; g += blockDim.x) {
            float a = 0.f, q = 0.f;
            for (int j = 0; j < gs; ++j) { a += red[g * gs + j]; q += red[C + g * gs + j]; }
            m1[g] = a * inv; m2[g] = q * inv;
        }
        __syncthreads();
    } else {
        for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) red[c] = 0.f;
        __syncthreads();
    }
    const int vpp = C >> 2;
    const int kpix = blockDim.x / vpp;
    const int c = (threadIdx.x % vpp) << 2;
    const int lp = threadIdx.x / vpp;
    float mu[4], rs[4], ga[4], be[4], mm1[4], mm2[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int g = (c + j) / gs;
        mu[j] = gm[g]; rs[j] = gr[g]; ga[j] = __ldg(&f.gamma[c + j]); be[j] = __ldg(&f.beta[c + j]);
        mm1[j] = APPLY ? m1[g] : 0.f; mm2[j] = APPLY ? m2[g] : 0.f;
    }
    const bool from0 = c < f.C0;
    const float* src = from0 ? f.src0 + c : f.src1 + (c - f.C0);
    const int cs = from0 ? f.C0 : f.C1;
    const int pix0 = blockIdx.x * f.pix_per_block;
    const int pix1 = min(pix0 + f.pix_per_block, f.HW);
    const long long img = static_cast<long long>(b) * f.HW;
    float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f}, cs4[4] = {0.f, 0.f, 0.f, 0.f};
    float* dst = from0 ? p.dst0 : p.dst1;
    __nv_bfloat16* dst_b = from0 ? p.dst0_b : p.dst1_b;
    const int acc = from0 ? p.acc0 : p.acc1;
    const int cl = from0 ? c : c - f.C0;
    if (threadIdx.x < vpp * kpix) {
        constexpr int U = 1;                          // (U = 4 measured slower: 124 registers per thread halve the resident blocks)
        for (int pix = pix0 + lp; pix < pix1; pix += kpix * U) {
            float4 xv[U], dv[U], av[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int pp = pix + u * kpix;
                if (pp < pix1) {
                    xv[u] = __ldg(reinterpret_cast<const float4*>(src + (img + pp) * cs));
                    dv[u] = __ldcg(reinterpret_cast<const float4*>(p.dA + (img + pp) * C + c));
                    if (APPLY && p.add) av[u] = __ldcg(reinterpret_cast<const float4*>(p.add + (img + pp) * p.add_ld + c));
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int pp = pix + u * kpix;
                if (pp >= pix1) continue;
                const float x4[4] = {xv[u].x, xv[u].y, xv[u].z, xv[u].w};
                float d4[4] = {dv[u].x, dv[u].y, dv[u].z, dv[u].w};
                if (p.drop && p.drop->p > 0.f) {
                    float sc[4];
                    drop_scale4(*p.drop, b, c, pp, C, f.HW, sc);
#pragma unroll
                    for (int j = 0; j < 4; ++j) d4[j] *= sc[j];
                }
                float out[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float xh = (x4[j] - mu[j]) * rs[j];
                    float d = d4[j];
                    if (f.silu) {
                        const float y = ga[j] * xh + be[j];
                        const float sg = 1.0f / (1.0f + __expf(-y));
                        d *= sg * (1.0f + y * (1.0f - sg));
                    }
                    if (APPLY) out[j] = rs[j] * (ga[j] * d - mm1[j] - xh * mm2[j]);
                    else { s1[j] += d; s2[j] += d * xh; }
                }
                if (APPLY) {
                    if (p.add) { out[0] += av[u].x; out[1] += av[u].y; out[2] += av[u].z; out[3] += av[u].w; }
                    if (dst) {
                        float4* dp = reinterpret_cast<float4*>(dst + (img + pp) * cs + cl);
                        if (acc) { const float4 o = *dp; out[0] += o.x; out[1] += o.y; out[2] += o.z; out[3] += o.w; }
                        *dp = make_float4(out[0], out[1], out[2], out[3]);
                    }
                    if (dst_b) *reinterpret_cast<uint2*>(dst_b + (img + pp) * cs + cl) = pack_bf16x4(out[0], out[1], out[2], out[3]);
#pragma unroll
                    for (int j = 0; j < 4; ++j) cs4[j] += out[j];
                }
            }
        }
    }
    // block reduction over the pixel lanes that share a channel column, then one atomic per (image, channel)
    if (APPLY) {
        if (p.gsum0 == nullptr && p.gsum1 == nullptr) return;       // (block-uniform)
        __syncthreads();
        for (int i = threadIdx.x; i < C; i += blockDim.x) red[i] = 0.f;
        __syncthreads();
        if (threadIdx.x < vpp * kpix) {
#pragma unroll
            for (int j = 0; j < 4; ++j) atomicAdd(&red[c + j], cs4[j]);
        }
        __syncthreads();
        for (int i = threadIdx.x; i < C; i += blockDim.x) {
            float* g2 = (i < f.C0) ? p.gsum0 : p.gsum1;
            if (g2) atomicAdd(&g2[static_cast<long long>(b) * ((i < f.C0) ? p.gsum_ld0 : p.gsum_ld1) + ((i < f.C0) ? i : i - f.C0)], red[i]);
        }
    } else {
        if (threadIdx.x < vpp * kpix) {
#pragma unroll
            for (int j = 0; j < 4; ++j) { atomicAdd(&red[c + j], s1[j]); atomicAdd(&red[C + c + j], s2[j]); }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < C; i += blockDim.x) {
            atomicAdd(&p.sums[(static_cast<long long>(b) * C + i) * 2], red[i]);
            atomicAdd(&p.sums[(static_cast<long long>(b) * C + i) * 2 + 1], red[C + i]);
        }
    }
}

// bias gradient from per-image channel sums: db[c] = gscale * sum_b gsum[b * ld + c]   (up to two destinations share it: conv2 + shortcut conv)
__global__ void __launch_bounds__(256) bias_grad_kernel(const float* __restrict__ gsum, int ld, float* __restrict__ d0, float* __restrict__ d1, int B, int C, float gscale) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float a = 0.f;
    for (int b = 0; b < B; ++b) a += gsum[static_cast<long long>(b) * ld + c];
    if (d0) d0[c] = a * gscale;
    if (d1) d1[c] = a * gscale;
}

// Elementwise gradient plumbing without a GroupNorm in front: out = a (+ b), optional accumulate into dst, bf16 copy and per-(image, channel)
// sums.  Tensors [B][HW][C] fp32.
__global__ void __launch_bounds__(256) grad_combine_kernel(const float* __restrict__ a, const float* __restrict__ b2, float* __restrict__ dst, int acc,
                                                           __nv_bfloat16* __restrict__ dst_b, float* __restrict__ gsum, int B, int HW, int C, int pix_per_block) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float red[];
    const int b = blockIdx.y;
    const int vpp = C >> 2, kpix = blockDim.x / vpp;
    for (int i = threadIdx.x; i < C; i += blockDim.x) red[i] = 0.f;
    __syncthreads();
    const int c = (threadIdx.x % vpp) << 2, lp = threadIdx.x / vpp;
    const int pix0 = blockIdx.x * pix_per_block, pix1 = min(pix0 + pix_per_block, HW);
    float cs4[4] = {0.f, 0.f, 0.f, 0.f};
    if (threadIdx.x < vpp * kpix) {
        for (int pix = pix0 + lp; pix < pix1; pix += kpix) {
            const long long o = (static_cast<long long>(b) * HW + pix) * C + c;
            float4 v = __ldcg(reinterpret_cast<const float4*>(a + o));
            if (b2) { const float4 w = __ldcg(reinterpret_cast<const float4*>(b2 + o)); v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w; }
            if (dst) {
                if (acc) { const float4 w = *reinterpret_cast<const float4*>(dst + o); v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w; }
                *reinterpret_cast<float4*>(dst + o) = v;
            }
            if (dst_b) *reinterpret_cast<uint2*>(dst_b + o) = pack_bf16x4(v.x, v.y, v.z, v.w);
            cs4[0] += v.x; cs4[1] += v.y; cs4[2] += v.z; cs4[3] += v.w;
        }
        if (gsum) {
#pragma unroll
            for (int j = 0; j < 4; ++j) atomicAdd(&red[c + j], cs4[j]);
        }
    }
    if (gsum) {
        __syncthreads();
        for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(&gsum[static_cast<long long>(b) * C + i], red[i]);
    }
}

// ------------------------------------------------------------------------------------------------ FiLM + noise-level MLP backward
// film[b][j] = Wf[j] . tau[b] + bf[j] + cb[j]  (unet.py:34-50 bias-only FiLM, cb = block1 conv bias folded in).  dfilm [B][F] = per-image
// channel sums of the gradient of block1's conv output.   dWf[j][i] = sum_b dfilm[b][j] tau[b][i];  dbf[j] = dcb[j] = sum_b dfilm[b][j];
// dtau[b][i] = sum_j Wf[j][i] dfilm[b][j]  (atomics into a zeroed dtau).
__global__ void __launch_bounds__(256) film_bwd_kernel(const float* __restrict__ wf, const float* __restrict__ tau, const float* __restrict__ dfilm,
                                                       float* __restrict__ dwf, float* __restrict__ dbf, float* __restrict__ dcb, float* __restrict__ dtau,
                                                       int F, int inner, int B, float gscale) {
    extern __shared__ float sm[];
    float* ts = sm;                 // [B][inner]
    float* dts = sm + B * inner;    // [B][inner] partial dtau of this block
    for (int i = threadIdx.x; i < B * inner; i += blockDim.x) { ts[i] = tau[i]; dts[i] = 0.f; }
    __syncthreads();
    const int j0 = blockIdx.x * 64;
    for (int idx = threadIdx.x; idx < 64 * inner; idx += blockDim.x) {
        const int jl = idx / inner, i = idx % inner, j = j0 + jl;
        if (j >= F) continue;
        float acc = 0.f;
        const float w = wf[static_cast<long long>(j) * inner + i];
        for (int b = 0; b < B; ++b) {
            const float d = dfilm[static_cast<long long>(b) * F + j];
            acc += d * ts[b * inner + i];
            atomicAdd(&dts[b * inner + i], w * d);
        }
        dwf[static_cast<long long>(j) * inner + i] = acc * gscale;
    }
    for (int jl = threadIdx.x; jl < 64; jl += blockDim.x) {
        const int j = j0 + jl;
        if (j >= F) continue;
        float a = 0.f;
        for (int b = 0; b < B; ++b) a += dfilm[static_cast<long long>(b) * F + j];
        dbf[j] = a * gscale; dcb[j] = a * gscale;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < B * inner; i += blockDim.x) atomicAdd(&dtau[i], dts[i]);
}
// The shared part of the noise-level MLP's backward: pe and pre recomputed from the noise level, dpre = d pre from dtau.  Shared memory
// (embed_bwd_smem) holds pe [B][inner], pre [B][hid], dpre [B][hid], dt [B][inner] in that order; returns with all of it written.
__device__ __forceinline__ void embed_bwd_dpre(const float* __restrict__ nl, const float* __restrict__ w1, const float* __restrict__ b1,
                                               const float* __restrict__ w2, const float* __restrict__ dtau, float* sm, int inner, int B) {
    const int hid = 4 * inner;
    float* pe = sm;                       // [B][inner]
    float* pre = pe + B * inner;          // [B][hid]
    float* dpre = pre + B * hid;          // [B][hid]
    float* dt = dpre + B * hid;           // [B][inner]
    const int count = inner / 2;
    for (int idx = threadIdx.x; idx < B * inner; idx += blockDim.x) {
        const int b = idx / inner, j = idx % inner;
        const int jj = j < count ? j : j - count;
        const float e = nl[b] * expf(-9.210340371976184f * (static_cast<float>(jj) / static_cast<float>(count)));
        pe[idx] = j < count ? sinf(e) : cosf(e);
        dt[idx] = dtau[idx];
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < B * hid; idx += blockDim.x) {
        const int b = idx / hid, j = idx % hid;
        float a = b1[j];
        for (int i = 0; i < inner; ++i) a += w1[j * inner + i] * pe[b * inner + i];
        pre[idx] = a;
    }
    __syncthreads();
    // dh = W2^T dtau;  dpre = dh * swish'(pre)
    for (int idx = threadIdx.x; idx < B * hid; idx += blockDim.x) {
        const int b = idx / hid, j = idx % hid;
        float a = 0.f;
        for (int o = 0; o < inner; ++o) a += w2[o * hid + j] * dt[b * inner + o];
        const float x = pre[idx], sg = 1.0f / (1.0f + expf(-x));
        dpre[idx] = a * sg * (1.0f + x * (1.0f - sg));
    }
    __syncthreads();
}
// tau = W2 swish(W1 pe + b1) + b2 (unet.py:177-184): one block, everything in shared memory.  pe / pre are recomputed from the noise level.
__global__ void __launch_bounds__(256) embed_bwd_kernel(const float* __restrict__ nl, const float* __restrict__ w1, const float* __restrict__ b1,
                                                        const float* __restrict__ w2, const float* __restrict__ dtau, float* __restrict__ dw1, float* __restrict__ db1,
                                                        float* __restrict__ dw2, float* __restrict__ db2, int inner, int B, float gscale) {
    extern __shared__ float sm[];
    const int hid = 4 * inner;
    float* pe = sm;                       // [B][inner]
    float* pre = pe + B * inner;          // [B][hid]
    float* dpre = pre + B * hid;          // [B][hid]
    float* dt = dpre + B * hid;           // [B][inner]
    embed_bwd_dpre(nl, w1, b1, w2, dtau, sm, inner, B);
    for (int idx = threadIdx.x; idx < inner * hid; idx += blockDim.x) {     // dW2[o][j] = sum_b dtau[b][o] swish(pre[b][j])
        const int o = idx / hid, j = idx % hid;
        float a = 0.f;
        for (int b = 0; b < B; ++b) { const float x = pre[b * hid + j]; a += dt[b * inner + o] * (x / (1.0f + expf(-x))); }
        dw2[idx] = a * gscale;
    }
    for (int o = threadIdx.x; o < inner; o += blockDim.x) { float a = 0.f; for (int b = 0; b < B; ++b) a += dt[b * inner + o]; db2[o] = a * gscale; }
    for (int idx = threadIdx.x; idx < hid * inner; idx += blockDim.x) {     // dW1[j][i] = sum_b dpre[b][j] pe[b][i]
        const int j = idx / inner, i = idx % inner;
        float a = 0.f;
        for (int b = 0; b < B; ++b) a += dpre[b * hid + j] * pe[b * inner + i];
        dw1[idx] = a * gscale;
    }
    for (int j = threadIdx.x; j < hid; j += blockDim.x) { float a = 0.f; for (int b = 0; b < B; ++b) a += dpre[b * hid + j]; db1[j] = a * gscale; }
}
// Gradient of the noise level itself (unet.py:18-31 PositionalEncoding, the MLP's input): dPE[b] = W1^T dpre[b] (dpre as embed_bwd_kernel
// forms it), then dnl[b] = sum_i dPE[b][i] dPE_i/dnl with PE_i = sin(nl f_i) for i < inner/2 (derivative cos(nl f_i) f_i), cos(nl f_i) for
// the other half (-sin(nl f_i) f_i), f_i = exp(-ln(1e4) (i mod inner/2) / (inner/2)).  One block (shared memory as embed_bwd_kernel), one
// warp per image.  Unscaled: the caller's upstream gradient carries any scale.
__global__ void __launch_bounds__(256) noise_level_bwd_kernel(const float* __restrict__ nl, const float* __restrict__ w1, const float* __restrict__ b1,
                                                              const float* __restrict__ w2, const float* __restrict__ dtau, float* __restrict__ dnl, int inner,
                                                              int B) {
    extern __shared__ float sm[];
    const int hid = 4 * inner, count = inner / 2;
    const float* dpre = sm + B * inner + B * hid;
    embed_bwd_dpre(nl, w1, b1, w2, dtau, sm, inner, B);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
    for (int b = warp; b < B; b += nwarp) {
        float acc = 0.f;
        for (int i = lane; i < inner; i += 32) {
            float d = 0.f;
            for (int j = 0; j < hid; ++j) d += w1[j * inner + i] * dpre[b * hid + j];
            const int ii = i < count ? i : i - count;
            const float f = expf(-9.210340371976184f * (static_cast<float>(ii) / static_cast<float>(count)));
            const float e = nl[b] * f;
            acc += d * (i < count ? cosf(e) : -sinf(e)) * f;
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) dnl[b] = acc;
    }
}

// ------------------------------------------------------------------------------------------------ attention backward (unet.py:129-139)
// The four matrix products run on the tensor cores (train_plan.inc, bwd_attention); these are the small kernels between them.
// softmax backward, in place on dP: dS = P * (dP - sum_k P dP) * scale; rows / segments as softmax_kernel
__global__ void __launch_bounds__(256) softmax_bwd_kernel(const __nv_bfloat16* __restrict__ P, float* __restrict__ dP, __nv_bfloat16* __restrict__ dS_b, long long rows, int L, int seg,
                                                          float scale) {
    pdl_launch_dependents();
    pdl_wait();
    const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const int k0 = (static_cast<int>(row % L) / seg) * seg;
    const __nv_bfloat16* pr = P + row * L;
    float* d = dP + row * L;
    float dot = 0.f;
    for (int k = k0 + lane; k < k0 + seg; k += 32) dot += __bfloat162float(pr[k]) * d[k];
#pragma unroll
    for (int o = 16; o; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    for (int k = lane; k < L; k += 32) {
        const float v = (k >= k0 && k < k0 + seg) ? __bfloat162float(pr[k]) * (d[k] - dot) * scale : 0.f;
        d[k] = v;
        if (dS_b) dS_b[row * L + k] = __float2bfloat16_rn(v);
    }
}
// bf16 matrix transpose, batched: dst[z][c][r] = src[z][r * src_ld + c]  (r < R, c < Cc); one 32x32 tile per block
__global__ void __launch_bounds__(256) transpose_bf16_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst, int R, int Cc, long long src_ld,
                                                             long long src_z, long long dst_z) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ __nv_bfloat16 t[32][33];
    const int z = blockIdx.z, r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int i = ty; i < 32; i += 8)
        if (r0 + i < R && c0 + tx < Cc) t[i][tx] = src[z * src_z + (r0 + i) * src_ld + c0 + tx];
    __syncthreads();
    for (int i = ty; i < 32; i += 8)
        if (c0 + i < Cc && r0 + tx < R) dst[z * dst_z + static_cast<long long>(c0 + i) * R + r0 + tx] = t[tx][i];
}
// fp32 [rows][C] -> bf16 (gradient operands of the tile / wgrad kernels)
__global__ void __launch_bounds__(256) cast_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n4) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const float4 v = __ldcg(reinterpret_cast<const float4*>(src) + i);
        reinterpret_cast<uint2*>(dst)[i] = pack_bf16x4(v.x, v.y, v.z, v.w);
    }
}

// ------------------------------------------------------------------------------------------------ loss + its gradient
// L1Loss / MSELoss(reduction='sum') of (noise, eps) (diffusion.py:84-90, 245).  d loss / d eps = sign(eps - noise) (L1) or 2 (eps - noise) (L2),
// written UNSCALED (exactly representable for L1) as bf16 NHWC with `ld` channels per pixel (the padded A operand of the final conv's
// data / weight gradient); every parameter gradient is multiplied by the scalar reaching the loss (1 / (b c h w), model.py:50-53) when it is
// written.  bias_sum [C] += sum of the gradient (final conv bias).
__global__ void __launch_bounds__(256) loss_grad_kernel(const float* __restrict__ noise, const float* __restrict__ eps, int B, int C, int H, int W, int l2,
                                                        double* __restrict__ loss, __nv_bfloat16* __restrict__ deps, int ld, float* __restrict__ bias_sum) {
    const long long n = static_cast<long long>(B) * C * H * W;
    double acc = 0.0;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const float d = eps[i] - noise[i];
        acc += l2 ? static_cast<double>(d) * d : static_cast<double>(fabsf(d));
        const float g = l2 ? 2.0f * d : (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
        long long r = i;
        const int w = static_cast<int>(r % W); r /= W;
        const int h = static_cast<int>(r % H); r /= H;
        const int c = static_cast<int>(r % C);
        const int b = static_cast<int>(r / C);
        deps[((static_cast<long long>(b) * H + h) * W + w) * ld + c] = __float2bfloat16_rn(g);
        if ((H * W) & 31) {                            // a 4x4 image: (b, c) changes inside a warp
            atomicAdd(&bias_sum[c], g);
            continue;
        }
        float gs = g;                                  // H * W is a multiple of 32: the lanes of a warp share (b, c)
#pragma unroll
        for (int o = 16; o; o >>= 1) gs += __shfl_xor_sync(0xffffffffu, gs, o);
        if ((threadIdx.x & 31) == 0) atomicAdd(&bias_sum[c], gs);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __shared__ double ws[8];
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < 8; ++i) t += ws[i];
        atomicAdd(loss, t);
    }
}
// The backward of UNet.forward alone, from an upstream gradient g = d(anything) / d eps (fp32 NCHW [B][C][H][W]), loaded in place of
// loss_grad_kernel's loss gradient: bf16 NHWC with `ld` channels per pixel (the padded A operand of the final conv's data / weight
// gradient; the padding channels and padded images are not touched and stay zero) and bias_sum [C] += its sums, taken from the unrounded
// fp32 values.
__global__ void __launch_bounds__(256) grad_load_kernel(const float* __restrict__ g_in, int B, int C, int H, int W, __nv_bfloat16* __restrict__ deps,
                                                        int ld, float* __restrict__ bias_sum) {
    const long long n = static_cast<long long>(B) * C * H * W;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const float g = g_in[i];
        long long r = i;
        const int w = static_cast<int>(r % W); r /= W;
        const int h = static_cast<int>(r % H); r /= H;
        const int c = static_cast<int>(r % C);
        const int b = static_cast<int>(r / C);
        deps[((static_cast<long long>(b) * H + h) * W + w) * ld + c] = __float2bfloat16_rn(g);
        if ((H * W) & 31) {                            // a 4x4 image: (b, c) changes inside a warp
            atomicAdd(&bias_sum[c], g);
            continue;
        }
        float gs = g;                                  // H * W is a multiple of 32: the lanes of a warp share (b, c)
#pragma unroll
        for (int o = 16; o; o >>= 1) gs += __shfl_xor_sync(0xffffffffu, gs, o);
        if ((threadIdx.x & 31) == 0) atomicAdd(&bias_sum[c], gs);
    }
}
// The input gradient: channels [0, C) of the fp32 NHWC data gradient of the first conv (ld channels per pixel) -> fp32 NCHW [B][C][H][W]
__global__ void __launch_bounds__(256) input_grad_store_kernel(const float* __restrict__ src, int B, int C, int H, int W, int ld, float* __restrict__ dst) {
    const long long n = static_cast<long long>(B) * C * H * W;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        long long r = i;
        const int w = static_cast<int>(r % W); r /= W;
        const int h = static_cast<int>(r % H); r /= H;
        const int c = static_cast<int>(r % C);
        const int b = static_cast<int>(r / C);
        dst[i] = src[((static_cast<long long>(b) * H + h) * W + w) * ld + c];
    }
}
__global__ void scale_vec_kernel(const float* __restrict__ src, float* __restrict__ dst, int n, float s) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i] * s;
}

// ------------------------------------------------------------------------------------------------ Adam (model/model.py:39-40: torch.optim.Adam defaults)
// One launch over a table of tensors: p -= lr * m_hat / (sqrt(v_hat) + eps), torch's formulation (bias corrections as scalars).
struct AdamTensor { float* p; const float* g; float* m; float* v; long long n; };
__global__ void __launch_bounds__(256) adam_kernel(const AdamTensor* __restrict__ tab, int n_tensors, float lr, float beta1, float beta2, float eps,
                                                   float bc1, float bc2_sqrt, float grad_scale) {
    for (int t = blockIdx.y; t < n_tensors; t += gridDim.y) {
        const AdamTensor a = tab[t];
        for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < a.n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
            const float g = a.g[i] * grad_scale;
            const float m = beta1 * a.m[i] + (1.0f - beta1) * g;
            const float v = beta2 * a.v[i] + (1.0f - beta2) * g * g;
            a.m[i] = m; a.v[i] = v;
            const float denom = sqrtf(v) / bc2_sqrt + eps;
            a.p[i] = a.p[i] - (lr / bc1) * (m / denom);
        }
    }
}

// ------------------------------------------------------------------------------------------------ weight packing
// Every packed copy of an fp32 parameter is one PackDesc, and pack_entry is the only code that writes one: the forward K-major conv weights,
// the folded Upsample phases, the data-gradient weights of the training plan, plain fp32 copies of the GroupNorm / bias / Linear parameters
// and the fused block2 + res_conv bias.  pack_all_kernel walks the whole table in one launch (the training loop's re-pack after every
// optimizer step: ~470 copies); pack_one_kernel packs one entry (loading a single parameter, sr3_test_conv_ex).
// One thread per work item, grid-strided; the item order keeps both the reads and the writes of a warp coalesced.
struct PackDesc {
    int type;                 // 0 fp32 copy, 1 forward conv weight, 2 stride-1 data-gradient weight, 3 Downsample data-gradient phases,
                              // 4 Upsample data-gradient 4x4 kernel, 5 folded Upsample forward phases, 6 dst = src + src2 (fused bias)
    int Cout, Cin, k, ld, k_off, rows_pad;
    int tap_stride;           // types 1, 2: columns between consecutive taps of a dst row (cin_pad / cout_pad)
    int lo_off;               // types 1, 5, precise mode: the low halves bf16(v - bf16(v)) sit lo_off elements after the high halves; else 0
    const float* src; const float* src2;
    void* dst;
    long long n;              // type 0 / 6: elements;  type 5: element stride between the four phase matrices
};
__device__ __forceinline__ void pack_entry(const PackDesc& d, long long i0, long long stride) {
    __nv_bfloat16* db = static_cast<__nv_bfloat16*>(d.dst);
    switch (d.type) {
    case 0: { float* o = static_cast<float*>(d.dst); for (long long i = i0; i < d.n; i += stride) o[i] = d.src[i]; break; }
    case 6: { float* o = static_cast<float*>(d.dst); for (long long i = i0; i < d.n; i += stride) o[i] = d.src[i] + d.src2[i]; break; }
    case 1: {
        // OIHW -> K-major: dst[o][k_off + (r*k+s)*tap_stride + c]; one item per (o, c), c fastest
        const int taps = d.k * d.k;
        const long long total = static_cast<long long>(d.Cout) * d.Cin;
        for (long long i = i0; i < total; i += stride) {
            const int c = static_cast<int>(i % d.Cin), o = static_cast<int>(i / d.Cin);
            const float* sp = d.src + i * taps;
            for (int t = 0; t < taps; ++t) {
                const float v = sp[t];
                const long long di = static_cast<long long>(o) * d.ld + d.k_off + t * d.tap_stride + c;
                db[di] = __float2bfloat16_rn(v);
                if (d.lo_off) db[di + d.lo_off] = __float2bfloat16_rn(bf16_residual(v));
            }
        }
        break;
    }
    case 2: {
        // data gradient of a stride-1 conv: dX = conv(dY, W') with W'[ci][((k-1-r)*k + (k-1-s)) * tap_stride + co] = W[co][ci][r][s];
        // one item per (c, o), o fastest
        const int taps = d.k * d.k;
        const long long total = static_cast<long long>(d.Cout) * d.Cin;
        for (long long i = i0; i < total; i += stride) {
            const int o = static_cast<int>(i % d.Cout), c = static_cast<int>(i / d.Cout);
            const float* sp = d.src + (static_cast<long long>(o) * d.Cin + c) * taps;
            __nv_bfloat16* dp = db + static_cast<long long>(c) * d.ld + o;
            for (int t = 0; t < taps; ++t) dp[(taps - 1 - t) * d.tap_stride] = __float2bfloat16_rn(sp[t]);     // (k-1-r)*k + (k-1-s) = k*k-1 - (r*k+s)
        }
        break;
    }
    case 3: {
        // data gradient of the stride-2 Downsample conv (unet.py:68-74) as four output-parity phases on the low-resolution dY grid: input
        // pixel (2i+py, 2j+px) receives, through tap offset (py-1+a, px-1+b) of dY, kernel row R(py,a), column R(px,b) with R(0,0) = none,
        // R(0,1) = 1, R(1,0) = 2, R(1,1) = 0.   dst[phase][ci][(a*2+b)*Cout + co], phases rows_pad rows apart
        const long long total = 4LL * d.Cin * 4 * d.Cout;
        for (long long i = i0; i < total; i += stride) {
            long long r = i;
            const int o = static_cast<int>(r % d.Cout); r /= d.Cout;
            const int ab = static_cast<int>(r % 4); r /= 4;
            const int c = static_cast<int>(r % d.Cin);
            const int ph = static_cast<int>(r / d.Cin);
            const int py = ph >> 1, px = ph & 1, a = ab >> 1, b = ab & 1;
            const int rr = py == 0 ? (a == 1 ? 1 : -1) : (a == 0 ? 2 : 0);
            const int ss = px == 0 ? (b == 1 ? 1 : -1) : (b == 0 ? 2 : 0);
            const float v = (rr < 0 || ss < 0) ? 0.f : d.src[((static_cast<long long>(o) * d.Cin + c) * 3 + rr) * 3 + ss];
            db[(static_cast<long long>(ph) * d.rows_pad + c) * (4LL * d.Cout) + ab * d.Cout + o] = __float2bfloat16_rn(v);
        }
        break;
    }
    case 4: {
        // data gradient of Upsample (nearest 2x -> conv3x3, unet.py:58-65): dX[i][j] = sum_{u,v in 0..3} K[u][v] dY[2i-1+u][2j-1+v],
        // K[u][v][ci][co] = sum over (e, r): e + 2 - r = u, (f, s): f + 2 - s = v of W[co][ci][r][s]  (e, f in {0,1}: the 2x2 replicated
        // pixels).   dst[ci][(u*4+v)*Cout + co]
        const long long total = static_cast<long long>(d.Cin) * 16 * d.Cout;
        for (long long i = i0; i < total; i += stride) {
            long long r = i;
            const int o = static_cast<int>(r % d.Cout); r /= d.Cout;
            const int uv = static_cast<int>(r % 16);
            const int c = static_cast<int>(r / 16);
            const int u = uv >> 2, v = uv & 3;
            float acc = 0.f;
            for (int e = 0; e < 2; ++e) {
                const int rr = e + 2 - u;
                if (rr < 0 || rr > 2) continue;
                for (int f = 0; f < 2; ++f) {
                    const int ss = f + 2 - v;
                    if (ss < 0 || ss > 2) continue;
                    acc += d.src[((static_cast<long long>(o) * d.Cin + c) * 3 + rr) * 3 + ss];
                }
            }
            db[static_cast<long long>(c) * (16LL * d.Cout) + uv * d.Cout + o] = __float2bfloat16_rn(acc);
        }
        break;
    }
    case 5: {
        // the four phase convs of a folded nearest-2x -> conv3x3: for output parity py the kernel rows that land on low-res row offset a are
        // R(0,0)={0}, R(0,1)={1,2}, R(1,0)={0,1}, R(1,1)={2} (same for columns); summed in fp32, rounded once.   dst[phase][o][(a*2+b)*Cin + c]
        const long long total = 4LL * d.Cout * d.Cin * 4;
        for (long long i = i0; i < total; i += stride) {
            long long r = i;
            const int c = static_cast<int>(r % d.Cin); r /= d.Cin;
            const int ab = static_cast<int>(r % 4); r /= 4;
            const int o = static_cast<int>(r % d.Cout);
            const int ph = static_cast<int>(r / d.Cout);
            const int py = ph >> 1, px = ph & 1, a = ab >> 1, b = ab & 1;
            const int r0 = (py == 0) ? (a == 0 ? 0 : 1) : (a == 0 ? 0 : 2), r1 = (py == 0) ? (a == 0 ? 0 : 2) : (a == 0 ? 1 : 2);
            const int s0 = (px == 0) ? (b == 0 ? 0 : 1) : (b == 0 ? 0 : 2), s1 = (px == 0) ? (b == 0 ? 0 : 2) : (b == 0 ? 1 : 2);
            float acc = 0.f;
            for (int rr = r0; rr <= r1; ++rr)
                for (int ss = s0; ss <= s1; ++ss) acc += d.src[((static_cast<long long>(o) * d.Cin + c) * 3 + rr) * 3 + ss];
            const long long di = ph * d.n + static_cast<long long>(o) * d.ld + ab * d.Cin + c;
            db[di] = __float2bfloat16_rn(acc);
            if (d.lo_off) db[di + d.lo_off] = __float2bfloat16_rn(bf16_residual(acc));
        }
        break;
    }
    default: break;
    }
}
// 256-thread blocks for one entry, in proportion to its work: ~8 (o, c) pairs (x k*k taps) or 32 plain elements per thread
inline int pack_entry_blocks(const PackDesc& d) {
    long long items;
    switch (d.type) {
        case 0: case 6: items = (d.n + 3) / 4; break;
        case 1: case 2: items = 1LL * d.Cout * d.Cin; break;
        case 3: items = 2LL * d.Cin * d.Cout; break;
        default: items = 4LL * d.Cin * d.Cout; break;
    }
    const long long nb = (items + 256 * 8 - 1) / (256 * 8);
    return static_cast<int>(nb < 1 ? 1 : (nb > 4096 ? 4096 : nb));
}
// block_ends[e] = one past the last block of entry e (pack_entry_blocks(tab[e]) blocks each)
__global__ void __launch_bounds__(256) pack_all_kernel(const PackDesc* __restrict__ tab, const int* __restrict__ block_ends, int n_entries) {
    const int e = find_entry(block_ends, n_entries, blockIdx.x);
    const int b0 = e == 0 ? 0 : __ldg(&block_ends[e - 1]), nb = __ldg(&block_ends[e]) - b0;
    const PackDesc d = tab[e];
    pack_entry(d, (blockIdx.x - b0) * static_cast<long long>(blockDim.x) + threadIdx.x, static_cast<long long>(nb) * blockDim.x);
}
__global__ void __launch_bounds__(256) pack_one_kernel(const __grid_constant__ PackDesc d) {
    pack_entry(d, blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x, static_cast<long long>(gridDim.x) * blockDim.x);
}

}  // namespace sr3
