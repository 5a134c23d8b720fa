// Bandwidth-bound helper kernels of the SR3 step (everything that is not a tensor-core tile):
// GroupNorm apply (+SiLU) with channel concat, fp32->bf16 cast / nearest 2x upsample, row softmax,
// noise-level embedding MLP + FiLM projections, layout conversion at the API boundary.  (Weight packing: pack_entry, train_kernels.cuh.)
#pragma once
#include "gemm_wgmma.cuh"

namespace sr3 {

__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }

__device__ __forceinline__ uint2 pack_bf16x4(float a, float b, float c, float d) {
    __nv_bfloat162 lo = __floats2bfloat162_rn(a, b), hi = __floats2bfloat162_rn(c, d);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&lo);
    u.y = *reinterpret_cast<uint32_t*>(&hi);
    return u;
}
// precise mode: the part of x that bf16(x) loses, itself rounded to bf16 (x ~ hi + lo to ~2^-17 relative)
__device__ __forceinline__ float bf16_residual(float x) { return x - __bfloat162float(__float2bfloat16_rn(x)); }
__device__ __forceinline__ uint2 pack_bf16x4_residual(float a, float b, float c, float d) {
    return pack_bf16x4(bf16_residual(a), bf16_residual(b), bf16_residual(c), bf16_residual(d));
}
// One 4-channel vector of a bf16 operand tensor: `o` = element offset of the high halves; precise mode (lo_off != 0) also stores the low halves
__device__ __forceinline__ void store_operand4(__nv_bfloat16* base, long long o, long long lo_off, float a, float b, float c, float d) {
    *reinterpret_cast<uint2*>(base + o) = pack_bf16x4(a, b, c, d);
    if (lo_off) *reinterpret_cast<uint2*>(base + o + lo_off) = pack_bf16x4_residual(a, b, c, d);
}

// ------------------------------------------------------------------------------------------------ dropout (unet.py:86, block2 only)
// keep-mask of element (b, c, pixel) of a [B][HW][C] tensor: either an injected mask (tests: the reference's own masks, uint8 NCHW) or
// Philox4x32-10 keyed by (seed; vector index, layer).  Forward and backward evaluate the same function.
struct DropSpec {
    const unsigned char* mask;     // optional [B][C][HW] (1 = keep)
    float p;                       // drop probability; 0 = no dropout
    unsigned int layer;
    unsigned long long seed;
};
__device__ __forceinline__ void drop_scale4(const DropSpec& d, int b, int c, int pix, int C, int HW, float (&s)[4]) {
    const float keep_scale = 1.0f / (1.0f - d.p);
    if (d.mask) {
#pragma unroll
        for (int j = 0; j < 4; ++j) s[j] = d.mask[(static_cast<long long>(b) * C + c + j) * HW + pix] ? keep_scale : 0.f;
        return;
    }
    const unsigned long long vec = (static_cast<unsigned long long>(b) * HW + pix) * (C >> 2) + (c >> 2);
    uint32_t ctr[4] = {static_cast<uint32_t>(vec), static_cast<uint32_t>(vec >> 32), d.layer, 0x5d0u};
    philox4x32_10(ctr, static_cast<uint32_t>(d.seed), static_cast<uint32_t>(d.seed >> 32));
#pragma unroll
    for (int j = 0; j < 4; ++j) s[j] = (static_cast<float>(ctr[j]) * 2.3283064365386963e-10f >= d.p) ? keep_scale : 0.f;
}

// ---------------------------------------------------------------------------------------------
// GroupNorm apply: a = [silu]( (x - mean_g) * rstd_g * gamma_c + beta_c ), x = concat(src0, src1) along channels.
// Statistics come from the per-(image, channel) sums the producing GEMM epilogues accumulated.
// reference: nn.GroupNorm(groups, C, eps=1e-5) + Swish of Block (unet.py:80-91), torch.cat of unet.py:255.
struct PrepParams {
    const float* src0; const float* src1;
    const double* st0; const double* st1;   // [B][C0][2], [B][C1][2]: fp64 (sum, sumsq) of the producing epilogues
    int C0, C1;
    const float* gamma; const float* beta;
    int groups, HW, pix_per_block, silu;
    float eps;
    __nv_bfloat16* out_a;                   // [B][HW][C0+C1]
    __nv_bfloat16* out_raw;                 // optional bf16(x), same shape
    int B;                                  // images (the GroupNorm backward reads it)
    int precise;                            // 1: operands are (hi | lo) pairs -- out rows are 2 (C0+C1) wide, low halves C0+C1 elements behind
    const DropSpec* drop;                   // training-mode forward only: Dropout after the SiLU (unet.py:86); nullptr otherwise
    float* save_mr;                         // training-mode forward only: [B][groups][2] (mean, rstd) kept for the backward; nullptr otherwise
};

// Per-(image, channel) scale / shift of a GroupNorm from the fp64 channel sums: y = x * sc[c] + sh[c].
// sc / sh: [C] floats each, CONTIGUOUS ([2C] floats = [C] doubles of scratch) in shared memory; gm / gr: [groups] each.
// All channel sums are fetched in ONE parallel round trip (a thread per channel), then reduced per group from shared memory.
// Ends with a __syncthreads().
__device__ __forceinline__ void groupnorm_scale_shift(const PrepParams& p, int b, float* sc, float* sh, float* gm, float* gr) {
    const int C = p.C0 + p.C1;
    const int gs = C / p.groups;
    // The [2C]-float sc/sh area holds C doubles: first all the sums, then (after the group means are known) all the sums of squares.  The two
    // rounds re-read the statistics from L2 instead of caching (sum, sumsq) pairs in registers: the streaming loop that follows decides the
    // kernel's register count, and 40 extra registers here cost the 128x128-level launches a third of their resident blocks (24 vs 15 us).
    double* scratch = reinterpret_cast<double*>(sc);
    const double inv = 1.0 / (static_cast<double>(gs) * static_cast<double>(p.HW));
    for (int c = threadIdx.x; c < C; c += blockDim.x)
        scratch[c] = (c < p.C0) ? __ldcg(p.st0 + (static_cast<long long>(b) * p.C0 + c) * 2) : __ldcg(p.st1 + (static_cast<long long>(b) * p.C1 + (c - p.C0)) * 2);
    __syncthreads();
    double gmean = 0.0;
    for (int g = threadIdx.x; g < p.groups; g += blockDim.x) {        // groups <= blockDim.x: one iteration
        double s = 0.0;
        for (int j = 0; j < gs; ++j) s += scratch[g * gs + j];
        gmean = s * inv;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x)
        scratch[c] = (c < p.C0) ? __ldcg(p.st0 + (static_cast<long long>(b) * p.C0 + c) * 2 + 1) : __ldcg(p.st1 + (static_cast<long long>(b) * p.C1 + (c - p.C0)) * 2 + 1);
    __syncthreads();
    for (int g = threadIdx.x; g < p.groups; g += blockDim.x) {
        double q = 0.0;
        for (int j = 0; j < gs; ++j) q += scratch[g * gs + j];
        double var = q * inv - gmean * gmean;               // fp64: no cancellation problem for |mean| >> std
        if (var < 0.0) var = 0.0;
        gm[g] = static_cast<float>(gmean);
        gr[g] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(p.eps)));
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const int g = c / gs;
        const float k = gr[g] * __ldg(&p.gamma[c]);
        sc[c] = k; sh[c] = __ldg(&p.beta[c]) - gm[g] * k;
    }
    __syncthreads();
}

// Block size = (C/4) * k threads: every thread owns ONE 4-channel column for the whole kernel (scale / shift live in
// registers, no shared-memory or integer-division traffic in the streaming loop) and walks pixels k at a time.
// DROP: training-mode forward of a block2 (Dropout after the SiLU); a separate instantiation keeps the Philox code out of the sampler's kernel
template <bool DROP>
__global__ void __launch_bounds__(512) prep_kernel(const PrepParams p) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float sm[];
    const int C = p.C0 + p.C1;
    float* sc = sm;              // [C] scale
    float* sh = sm + C;          // [C] shift
    float* gm = sm + 2 * C;      // [groups] mean
    float* gr = gm + p.groups;   // [groups] rstd
    const int b = blockIdx.y;
    groupnorm_scale_shift(p, b, sc, sh, gm, gr);
    if (p.save_mr != nullptr && blockIdx.x == 0) {
        for (int g = threadIdx.x; g < p.groups; g += blockDim.x) {
            p.save_mr[(static_cast<long long>(b) * p.groups + g) * 2] = gm[g];
            p.save_mr[(static_cast<long long>(b) * p.groups + g) * 2 + 1] = gr[g];
        }
    }
    const int vpp = C >> 2;                       // 4-channel vectors per pixel
    const int kpix = blockDim.x / vpp;            // pixels covered by the block per step
    const int c = (threadIdx.x % vpp) << 2;       // this thread's channels (constant)
    const int lp = threadIdx.x / vpp;             // this thread's pixel lane
    float k4[4], s4[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { k4[j] = sc[c + j]; s4[j] = sh[c + j]; }
    const bool from0 = c < p.C0;
    const float* src = from0 ? p.src0 + c : p.src1 + (c - p.C0);
    const int cs = from0 ? p.C0 : p.C1;
    const int pix0 = blockIdx.x * p.pix_per_block;
    const int pix1 = min(pix0 + p.pix_per_block, p.HW);
    const long long img = static_cast<long long>(b) * p.HW;
    constexpr int U = 4;                          // independent 16-byte loads in flight per thread
    for (int pix = pix0 + lp; pix < pix1; pix += kpix * U) {
        float4 x[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int pp = pix + u * kpix;
            if (pp < pix1) x[u] = __ldg(reinterpret_cast<const float4*>(src + (img + pp) * cs));
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int pp = pix + u * kpix;
            if (pp < pix1) {
                float y0 = x[u].x * k4[0] + s4[0], y1 = x[u].y * k4[1] + s4[1], y2 = x[u].z * k4[2] + s4[2], y3 = x[u].w * k4[3] + s4[3];
                if (p.silu) { y0 = silu_f(y0); y1 = silu_f(y1); y2 = silu_f(y2); y3 = silu_f(y3); }
                if (DROP && p.drop->p > 0.f) {
                    float ds[4];
                    drop_scale4(*p.drop, b, c, pp, C, p.HW, ds);
                    y0 *= ds[0]; y1 *= ds[1]; y2 *= ds[2]; y3 *= ds[3];
                }
                const long long o = (img + pp) * (p.precise ? 2 * C : C) + c;
                const long long lo_off = p.precise ? C : 0;
                store_operand4(p.out_a, o, lo_off, y0, y1, y2, y3);
                if (p.out_raw) store_operand4(p.out_raw, o, lo_off, x[u].x, x[u].y, x[u].z, x[u].w);
            }
        }
    }
}

// fp32 NHWC -> bf16 NHWC, optionally nearest-2x upsampled (nn.Upsample(scale_factor=2,'nearest'), unet.py:58-65)
__global__ void __launch_bounds__(256) cast_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int B, int H, int W,
                                                   int C, int up) {
    pdl_launch_dependents();
    pdl_wait();
    const int OH = H * up, OW = W * up;
    const long long total = static_cast<long long>(B) * OH * OW * (C >> 2);
    const int vpp = C >> 2;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int v = static_cast<int>(i % vpp);
        long long pix = i / vpp;
        const int ow = static_cast<int>(pix % OW); pix /= OW;
        const int oh = static_cast<int>(pix % OH);
        const int b = static_cast<int>(pix / OH);
        const long long sp = (static_cast<long long>(b) * H + oh / up) * W + ow / up;
        const float4 x = __ldg(reinterpret_cast<const float4*>(src + sp * C + (v << 2)));
        *reinterpret_cast<uint2*>(dst + i * 4) = pack_bf16x4(x.x, x.y, x.z, x.w);
    }
}

// Row softmax over keys (torch.softmax(attn, -1), unet.py:136): S fp32 [rows][L] -> P bf16 [rows][L].
// Rows are grouped in segments of `seg` tokens; a row only attends to the keys of its own segment (two 64-token images share
// one 128-row attention batch); keys outside get probability 0.
struct SoftmaxParams { const float* S; __nv_bfloat16* P; long long rows; int L, seg, precise; };
__global__ void __launch_bounds__(256) softmax_kernel(const float* __restrict__ S, __nv_bfloat16* __restrict__ P, long long rows, int L,
                                                      int seg, int precise) {
    pdl_launch_dependents();
    pdl_wait();
    const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const int r_in = static_cast<int>(row % L);
    const int k0 = (r_in / seg) * seg;
    const float* s = S + row * L;
    __nv_bfloat16* pr = P + row * (precise ? 2 * L : L);
    float m = -INFINITY;
    for (int k = k0 + lane; k < k0 + seg; k += 32) m = fmaxf(m, s[k]);
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float sum = 0.f;
    for (int k = k0 + lane; k < k0 + seg; k += 32) sum += expf(s[k] - m);
#pragma unroll
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.0f / sum;
    for (int k = lane; k < L; k += 32) {
        const float v = (k >= k0 && k < k0 + seg) ? expf(s[k] - m) * inv : 0.f;
        pr[k] = __float2bfloat16_rn(v);
        if (precise) pr[L + k] = __float2bfloat16_rn(bf16_residual(v));
    }
}

// Start of a step: clear the GroupNorm statistics arena and advance the device-side timestep.
__global__ void __launch_bounds__(256) step_begin_kernel(float4* stats, long long n4, StepCtl* ctl) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4; i += static_cast<long long>(gridDim.x) * blockDim.x)
        stats[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const int t = ctl->t_next;
        ctl->t_cur = t;
        ctl->t_next = t - 1;
    }
}

// PositionalEncoding + noise_level_mlp (unet.py:18-31, 177-184): one block per image -> tau[b][inner].
struct EmbedParams {
    const StepCtl* ctl;
    const float* nl_table;   // fp32(sqrt_alphas_cumprod_prev) [T+1]
    const float* nl_buf;     // [B]
    const float* w1; const float* b1;   // [4*inner][inner]
    const float* w2; const float* b2;   // [inner][4*inner]
    float* tau;              // [B][inner]
    int inner;
};
__global__ void __launch_bounds__(256) embed_kernel(const EmbedParams p) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float sm[];
    const int inner = p.inner, hid = 4 * inner;
    float* pe = sm;            // [inner]
    float* h = sm + inner;     // [hid]
    const int b = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
    const float nl = p.ctl->nl_from_table ? p.nl_table[p.ctl->t_cur + 1] : p.nl_buf[b];
    const int count = inner / 2;
    for (int j = threadIdx.x; j < inner; j += blockDim.x) {
        const int jj = j < count ? j : j - count;
        const float step = static_cast<float>(jj) / static_cast<float>(count);
        const float e = nl * expf(-9.210340371976184f * step);
        pe[j] = j < count ? sinf(e) : cosf(e);
    }
    __syncthreads();
    // one warp per output row (coalesced weights + shuffle reduction); 8 rows are in flight per warp so the L2 latency of the
    // weight loads is paid once per batch of rows, not once per row
    constexpr int R = 8;
    for (int j0 = warp * R; j0 < hid; j0 += nwarp * R) {
        float a[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            a[r] = 0.f;
            if (j0 + r < hid)
                for (int i = lane; i < inner; i += 32) a[r] += __ldg(&p.w1[(j0 + r) * inner + i]) * pe[i];
        }
#pragma unroll
        for (int r = 0; r < R; ++r) {
#pragma unroll
            for (int o = 16; o; o >>= 1) a[r] += __shfl_xor_sync(0xffffffffu, a[r], o);
            if (lane == 0 && j0 + r < hid) { const float t = a[r] + p.b1[j0 + r]; h[j0 + r] = t / (1.0f + expf(-t)); }
        }
    }
    __syncthreads();
    for (int j0 = warp * R; j0 < inner; j0 += nwarp * R) {
        float a[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            a[r] = 0.f;
            if (j0 + r < inner)
                for (int i = lane; i < hid; i += 32) a[r] += __ldg(&p.w2[(j0 + r) * hid + i]) * h[i];
        }
#pragma unroll
        for (int r = 0; r < R; ++r) {
#pragma unroll
            for (int o = 16; o; o >>= 1) a[r] += __shfl_xor_sync(0xffffffffu, a[r], o);
            if (lane == 0 && j0 + r < inner) p.tau[b * inner + j0 + r] = a[r] + p.b2[j0 + r];
        }
    }
}

// All FeatureWiseAffine projections at once (unet.py:34-50, bias-only form) + the block1 conv bias folded in:
// film[b][j] = Wf[j] . tau[b] + bf[j] + cbias[j],  j over the concatenated Cout of every ResnetBlock.
// A block owns 64 outputs: their weight rows are staged (coalesced) in padded smem, tau in chunks of `chunk` images (any batch fits).
__global__ void __launch_bounds__(256) film_kernel(const float* __restrict__ wf, const float* __restrict__ bf, const float* __restrict__ cbias,
                                                   const float* __restrict__ tau, float* __restrict__ film, int F, int inner, int B, int chunk) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float sm[];
    float* ws = sm;                          // [64][inner + 1]
    float* ts = sm + 64 * (inner + 1);       // [chunk][inner]
    const int j0 = blockIdx.x * 64;
    for (int i = threadIdx.x; i < 64 * inner; i += blockDim.x) {
        const int r = i / inner, c = i % inner;
        ws[r * (inner + 1) + c] = (j0 + r < F) ? __ldg(&wf[static_cast<long long>(j0 + r) * inner + c]) : 0.f;
    }
    const int jl = threadIdx.x & 63, bq = threadIdx.x >> 6;
    const int j = j0 + jl;
    const float base = j < F ? bf[j] + cbias[j] : 0.f;
    const float* w = ws + jl * (inner + 1);
    for (int b0 = 0; b0 < B; b0 += chunk) {
        const int nb = min(chunk, B - b0);
        __syncthreads();                     // (the previous chunk's tau is no longer read)
        for (int i = threadIdx.x; i < nb * inner; i += blockDim.x) ts[i] = __ldg(&tau[static_cast<long long>(b0) * inner + i]);
        __syncthreads();
        if (j >= F) continue;
        for (int b = bq; b < nb; b += 4) {
            float a = base;
            const float* t = ts + b * inner;
            for (int i = 0; i < inner; ++i) a += w[i] * t[i];
            film[static_cast<long long>(b0 + b) * F + j] = a;
        }
    }
}

// API boundary: NCHW fp32 (reference layout) -> bf16 NHWC channel slice of the UNet input buffer (+ optional fp32 NCHW copy).
__global__ void __launch_bounds__(256) load_nchw_kernel(const float* __restrict__ src, int B, int C, int H, int W, __nv_bfloat16* __restrict__ in_buf,
                                                        int in_C, int coff, float* __restrict__ copy, int lo_off) {
    const long long total = static_cast<long long>(B) * C * H * W;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        long long r = i;
        const int w = static_cast<int>(r % W); r /= W;
        const int h = static_cast<int>(r % H); r /= H;
        const int c = static_cast<int>(r % C);
        const int b = static_cast<int>(r / C);
        const float v = src[i];
        const long long di = ((static_cast<long long>(b) * H + h) * W + w) * in_C + coff + c;
        in_buf[di] = __float2bfloat16_rn(v);
        if (lo_off) in_buf[di + lo_off] = __float2bfloat16_rn(bf16_residual(v));
        if (copy) copy[i] = v;
    }
}

// q_sample (diffusion.py:212-219) fused with the input load: x_noisy = g * x0 + sqrt(1 - g^2) * noise, written as bf16 into the
// UNet input buffer (channels [coff, coff+C)); g = continuous_sqrt_alpha_cumprod of the image.
__global__ void __launch_bounds__(256) q_sample_load_kernel(const float* __restrict__ x0, const float* __restrict__ noise, const float* __restrict__ gamma,
                                                            int B, int C, int H, int W, __nv_bfloat16* __restrict__ in_buf, int in_C, int coff, int lo_off) {
    const long long total = static_cast<long long>(B) * C * H * W;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        long long r = i;
        const int w = static_cast<int>(r % W); r /= W;
        const int h = static_cast<int>(r % H); r /= H;
        const int c = static_cast<int>(r % C);
        const int b = static_cast<int>(r / C);
        const float g = gamma[b];
        const float v = __fadd_rn(__fmul_rn(g, x0[i]), __fmul_rn(sqrtf(__fsub_rn(1.0f, __fmul_rn(g, g))), noise[i]));
        const long long di = ((static_cast<long long>(b) * H + h) * W + w) * in_C + coff + c;
        in_buf[di] = __float2bfloat16_rn(v);
        if (lo_off) in_buf[di + lo_off] = __float2bfloat16_rn(bf16_residual(v));
    }
}

// L1Loss / MSELoss with reduction='sum' (diffusion.py:84-90, 245): loss += sum |noise - eps| (or squared), double accumulation
__global__ void __launch_bounds__(256) loss_sum_kernel(const float* __restrict__ noise, const float* __restrict__ eps, long long n, int l2,
                                                       double* __restrict__ out) {
    double acc = 0.0;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const float d = noise[i] - eps[i];
        acc += l2 ? static_cast<double>(d) * d : static_cast<double>(fabsf(d));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __shared__ double ws[8];
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < 8; ++i) t += ws[i];
        atomicAdd(out, t);
    }
}

// tensor2img of the reference (core/metrics.py:8-34) on the device: clamp to [lo, hi] -> (x - lo) / (hi - lo) -> * 255 -> round half to even
// -> uint8, laid out HWC.  `n` images [n][C][H][W] are tiled like torchvision.utils.make_grid(nrow, padding=2, pad_value=0) when n > 1
// (grid of ncol x nrow cells of (H+2) x (W+2) pixels plus a 2-pixel border); n == 1: plain [H][W][C].
// Per-image form: n == 1 and gridDim.y images, image blockIdx.y read from src [y][C][H][W] and written to its own dst [y][H][W][C]
// (what tensor2img(sr[i]) gives for every i of a batch); the grid form launches gridDim.y == 1.
__global__ void __launch_bounds__(256) tensor2img_kernel(const float* __restrict__ src, unsigned char* __restrict__ dst, int n, int C, int H, int W,
                                                         int ncol, int GH, int GW, float lo, float hi) {
    const long long total = static_cast<long long>(GH) * GW * C;
    src += blockIdx.y * (static_cast<long long>(C) * H * W);
    dst += blockIdx.y * total;
    const int pad = n > 1 ? 2 : 0;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c = static_cast<int>(i % C);
        const int gx = static_cast<int>((i / C) % GW);
        const int gy = static_cast<int>(i / (static_cast<long long>(C) * GW));
        float v = 0.f;                                               // pad_value 0 (already in [0, 1] units)
        bool inside = true;
        int img = 0, y = gy, x = gx;
        if (n > 1) {
            const int cy = (gy - pad) / (H + pad), cx = (gx - pad) / (W + pad);
            y = (gy - pad) - cy * (H + pad); x = (gx - pad) - cx * (W + pad);
            img = cy * ncol + cx;
            inside = gy >= pad && gx >= pad && y < H && x < W && img < n && cx < ncol;
        }
        if (inside) {
            float t = src[((static_cast<long long>(img) * C + c) * H + y) * W + x];
            t = fminf(fmaxf(t, lo), hi);
            v = __fdiv_rn(__fsub_rn(t, lo), __fsub_rn(hi, lo));
        }
        dst[i] = static_cast<unsigned char>(rintf(__fmul_rn(v, 255.0f)));
    }
}

// sum of squared differences of two uint8 images (calculate_psnr, core/metrics.py:42-50): exact in integers.
// Per-pair form: gridDim.y pairs of n elements each, pair blockIdx.y summed into out[blockIdx.y] (integer atomics: order-independent).
__global__ void __launch_bounds__(256) ssd_u8_kernel(const unsigned char* __restrict__ a, const unsigned char* __restrict__ b, long long n,
                                                     unsigned long long* __restrict__ out) {
    a += blockIdx.y * n;
    b += blockIdx.y * n;
    out += blockIdx.y;
    unsigned long long acc = 0;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int d = static_cast<int>(a[i]) - static_cast<int>(b[i]);
        acc += static_cast<unsigned long long>(d * d);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0 && acc) atomicAdd(out, acc);
}

// ssim of the reference (core/metrics.py:52-72), everything in fp64: the 11x11 window outer(g, g) of cv2.getGaussianKernel(11, 1.5), applied
// as an 11-tap horizontal then an 11-tap vertical pass to the five moments x, y, x^2, y^2, xy, only where the window fits the image
// (filter2D(...)[5:-5, 5:-5] keeps exactly those pixels); sigma = E[x^2] - mu^2; every channel of an HWC image filtered on its own.
// Pair blockIdx.z of [n][H][W][C]; a CTA owns an SSIM_TH x SSIM_TW tile of the (H-10) x (W-10) valid region across all channels and writes
// the sum of its map values to partial[pair][tile]; ssim_finish_kernel adds the tiles in order.  The split depends on (H, W, C) only, so a
// pair's value does not depend on the batch it is scored in.
constexpr int SSIM_TH = 16, SSIM_TW = 32, SSIM_THREADS = 256, SSIM_TAPS = 11;
struct SsimWindow { double g[SSIM_TAPS]; };

template <typename T>
__global__ void __launch_bounds__(SSIM_THREADS) ssim_kernel(const T* __restrict__ a, const T* __restrict__ b, int H, int W, int C, const SsimWindow win,
                                                            double* __restrict__ partial) {
    constexpr int R = SSIM_TH + SSIM_TAPS - 1;                  // input rows a tile's vertical pass reads
    __shared__ double hs[5][R][SSIM_TW];                        // horizontal pass: the five moments per (input row, output column)
    __shared__ double ws[SSIM_THREADS / 32];
    constexpr double C1 = (0.01 * 255) * (0.01 * 255), C2 = (0.03 * 255) * (0.03 * 255);
    const int Hv = H - (SSIM_TAPS - 1), Wv = W - (SSIM_TAPS - 1);
    const int x0 = blockIdx.x * SSIM_TW, y0 = blockIdx.y * SSIM_TH;
    const long long img = blockIdx.z * (static_cast<long long>(H) * W * C);
    a += img;
    b += img;
    double acc = 0.0;
    for (int c = 0; c < C; ++c) {
        for (int i = threadIdx.x; i < R * SSIM_TW; i += SSIM_THREADS) {
            const int r = i / SSIM_TW, j = i % SSIM_TW;
            double m[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
            if (y0 + r < H && x0 + j < Wv) {
                const long long p = (static_cast<long long>(y0 + r) * W + x0 + j) * C + c;
#pragma unroll
                for (int k = 0; k < SSIM_TAPS; ++k) {
                    const double u = static_cast<double>(a[p + k * C]), v = static_cast<double>(b[p + k * C]), w = win.g[k];
                    m[0] += w * u; m[1] += w * v; m[2] += w * (u * u); m[3] += w * (v * v); m[4] += w * (u * v);
                }
            }
#pragma unroll
            for (int q = 0; q < 5; ++q) hs[q][r][j] = m[q];
        }
        __syncthreads();
        for (int i = threadIdx.x; i < SSIM_TH * SSIM_TW; i += SSIM_THREADS) {
            const int r = i / SSIM_TW, j = i % SSIM_TW;
            if (y0 + r >= Hv || x0 + j >= Wv) continue;
            double m[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
            for (int k = 0; k < SSIM_TAPS; ++k) {
#pragma unroll
                for (int q = 0; q < 5; ++q) m[q] += win.g[k] * hs[q][r + k][j];
            }
            // explicit roundings (no contraction): for x == y both factors of the ratio are bit-identical, so the map is exactly 1
            const double mu1_sq = __dmul_rn(m[0], m[0]), mu2_sq = __dmul_rn(m[1], m[1]), mu1_mu2 = __dmul_rn(m[0], m[1]);
            const double s1 = __dsub_rn(m[2], mu1_sq), s2 = __dsub_rn(m[3], mu2_sq), s12 = __dsub_rn(m[4], mu1_mu2);
            const double num = __dmul_rn(__dadd_rn(__dmul_rn(2.0, mu1_mu2), C1), __dadd_rn(__dmul_rn(2.0, s12), C2));
            const double den = __dmul_rn(__dadd_rn(__dadd_rn(mu1_sq, mu2_sq), C1), __dadd_rn(__dadd_rn(s1, s2), C2));
            acc += __ddiv_rn(num, den);
        }
        __syncthreads();
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < SSIM_THREADS / 32; ++i) t += ws[i];
        partial[(static_cast<long long>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = t;
    }
}

// ssim_map.mean() per pair: the pair's `tiles` partial sums added in tile order, over `count` = (H-10) (W-10) C map values
__global__ void __launch_bounds__(128) ssim_finish_kernel(const double* __restrict__ partial, int tiles, double count, int n, double* __restrict__ out) {
    const int pair = blockIdx.x * blockDim.x + threadIdx.x;
    if (pair >= n) return;
    double t = 0.0;
    for (int i = 0; i < tiles; ++i) t += partial[static_cast<long long>(pair) * tiles + i];
    out[pair] = t / count;
}

// One pass of Pillow's 8-bit resampler (src/libImaging/Resample.c, ImagingResampleHorizontal_8bpc / Vertical_8bpc) with host-built
// integer coefficient tables: out = clip8((2^21 + sum_k in[first + k] * coef[k]) >> 22).  `axis_stride` / `line_stride` / `img_stride` are in
// elements of the uint8 input [img][line][axis][C]; one thread per output element (img, line, o, c).
// Output: uint8 [img][..][C] with the same structure (dst_u8) and / or float CHW planes (dst_f32: ToTensor /255, optional flip along W,
// * (max - min) + min -- data/util.py:74-83) -- only meaningful for the LAST pass (vertical), where line = x and o = y.
__global__ void __launch_bounds__(256) resample_u8_kernel(const unsigned char* __restrict__ src, unsigned char* __restrict__ dst_u8, float* __restrict__ dst_f32,
                                                          int n_img, int n_line, int n_out, int C, long long in_axis_stride, long long in_line_stride,
                                                          long long in_img_stride, long long out_axis_stride, long long out_line_stride, long long out_img_stride,
                                                          const int* __restrict__ bounds, const int* __restrict__ coef, int ksize, int flip, float vmin, float vmax) {
    const long long total = static_cast<long long>(n_img) * n_line * n_out * C;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c = static_cast<int>(i % C);
        const int line = static_cast<int>((i / C) % n_line);
        const int o = static_cast<int>((i / (static_cast<long long>(C) * n_line)) % n_out);
        const int img = static_cast<int>(i / (static_cast<long long>(C) * n_line * n_out));
        const int first = bounds[2 * o], n = bounds[2 * o + 1];
        const unsigned char* sp = src + img * in_img_stride + line * in_line_stride + first * in_axis_stride + c;
        int acc = 1 << 21;
        for (int k = 0; k < n; ++k) acc += static_cast<int>(sp[k * in_axis_stride]) * coef[o * ksize + k];
        int v = acc >> 22;
        v = v < 0 ? 0 : (v > 255 ? 255 : v);
        if (dst_u8) dst_u8[img * out_img_stride + line * out_line_stride + o * out_axis_stride + c] = static_cast<unsigned char>(v);
        if (dst_f32) {                                 // last (vertical) pass: o = y, line = x; CHW planes of n_out x n_line
            const int x = flip ? (n_line - 1 - line) : line;
            const float t = __fdiv_rn(static_cast<float>(v), 255.0f);
            dst_f32[((static_cast<long long>(img) * C + c) * n_out + o) * n_line + x] = __fadd_rn(__fmul_rn(t, __fsub_rn(vmax, vmin)), vmin);
        }
    }
}

}  // namespace sr3
