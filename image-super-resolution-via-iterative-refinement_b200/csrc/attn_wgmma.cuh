// attn_wgmma.cuh -- the core of SelfAttention (reference model/sr3_modules/unet.py:129-139) as ONE tensor-core kernel:
//
//   S = q k^T / sqrt(C)   (wgmma, accumulator in registers)   -> row softmax in registers (unnormalised exp, bf16) -> shared memory
//   O = P v               (wgmma, P is the A operand straight from shared memory)                -> O / rowsum -> bf16 [token][C]
//
// One CTA = (attention batch z, 128 query rows, DN of the C output channels); it recomputes S for its query rows (0.27 GFLOP per
// image at 16x16: cheaper than a second launch) so that 2 * C/DN CTAs per image run instead of 2.  n_head = 1 in every reference
// config, so the head dimension is C (512): S needs all of it (K loop over C); O's columns are split across CTAs.  Key count
// Lt <= 256 (16x16 = 256 tokens; two 8x8 images share a 128-token batch with a block-diagonal mask, as in softmax_kernel); longer
// sequences (32x32 mid block of the 64->512 config, larger images) run attn_long_kernel (attn_long_wgmma.cuh).
//
// Operands (both produced by tile-kernel launches): qk [nz*Lt][2C] bf16 (q = columns [0,C), k = [C,2C)), vT [nz*C][Lt] bf16.
// Warp roles: 8 = TMA producer, 0..7 = two warpgroups, each owning 64 query rows: S (64 x Lt) and O (64 x DN) in registers.
#pragma once
#include <cuda_bf16.h>
#include <cuda.h>
#include "gemm_wgmma.cuh"

namespace sr3 {

constexpr int ATTN_THREADS = 288;
constexpr int ATTN_PRODUCER_WARP = 8;
constexpr int ATTN_STAGES = 3;
constexpr int ATTN_STAGE_BYTES = 16384 + 32768;          // A: 128 rows x 64 | B: up to 256 rows x 64 (bf16, 128B-swizzled)
constexpr int ATTN_P_BYTES = 65536;                      // P: 128 rows x up to 256 keys, as K chunks of 64
constexpr int ATTN_SMEM_BYTES = 1024 + GEMM_HDR_BYTES + ATTN_STAGES * ATTN_STAGE_BYTES + ATTN_P_BYTES;   // header: barriers

struct AttnParams {
    CUtensorMap qk_map;      // 2-D bf16 [nz*Lt rows][2C], box {64, 128}
    CUtensorMap vt_map;      // 2-D bf16 [nz*C rows][Lt], box {64, 128}
    __nv_bfloat16* out;      // [nz*Lt][C]
    int C, Lt, HW, dn, nz;
    float scale_log2e;       // log2(e) / sqrt(C)
};

// One (attention batch z, query tile qt, channel slice dc) unit for Lt = LT keys and DN output channels: the body of attn_kernel (one
// unit per CTA).  `pm` points at the parameters in the kernel parameter space (TMA descriptors are addressed through it).
template <int LT, int DN>
__device__ __forceinline__ void attn_unit_t(const AttnParams& p, const AttnParams* pm, const uint32_t base_in, uint8_t* base_ptr_in,
                                            const int qt, const int dc, const int z) {
    const uint32_t bar_base = base_in;                                 // header (gemm_wgmma.cuh)
    const uint32_t base = base_in + GEMM_HDR_BYTES;
    uint8_t* base_ptr = base_ptr_in + GEMM_HDR_BYTES;
    const uint32_t p_base = base + ATTN_STAGES * ATTN_STAGE_BYTES;
    uint8_t* p_ptr = base_ptr + ATTN_STAGES * ATTN_STAGE_BYTES;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (ATTN_STAGES + s); };

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int kc1 = p.C / 64;        // K chunks of S = q k^T
    constexpr int kc3 = LT / 64;     // K chunks of O = P v

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&pm->qk_map);
        tma_prefetch_desc(&pm->vt_map);
        for (int s = 0; s < ATTN_STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 2); }   // empty: one arrive per warpgroup
        fence_mbar_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();                  // q, k, vT come from the two preceding launches

    if (warp == ATTN_PRODUCER_WARP) {
        // ------------------------------------------------------------ TMA producer
        int s = 0;
        uint32_t ph = 0;
        for (int it = 0; it < kc1 + kc3; ++it) {
            mbar_wait(empty_bar(s), ph ^ 1u);
            if (elect_one_sync()) {
                const uint32_t dst = base + s * ATTN_STAGE_BYTES;
                if (it < kc1) {
                    mbar_arrive_expect_tx(full_bar(s), 16384 + LT * 128);
                    tma_load_2d(dst, &pm->qk_map, full_bar(s), it * 64, z * LT + qt * 128);
                    for (int j = 0; j < LT / 128; ++j)
                        tma_load_2d(dst + 16384 + j * 16384, &pm->qk_map, full_bar(s), p.C + it * 64, z * LT + j * 128);
                } else {
                    mbar_arrive_expect_tx(full_bar(s), DN * 128);
                    for (int j = 0; j < DN / 128; ++j)
                        tma_load_2d(dst + 16384 + j * 16384, &pm->vt_map, full_bar(s), (it - kc1) * 64, z * p.C + dc * DN + j * 128);
                }
            }
            __syncwarp();
            if (++s == ATTN_STAGES) { s = 0; ph ^= 1u; }
        }
    } else if (warp < ATTN_PRODUCER_WARP) {
        // ------------------------------------------------------------ warpgroup g: query rows [64 g, 64 g + 64) of the tile
        const int g = warp >> 2;
        const int wq = warp & 3;
        const bool leader = (threadIdx.x & 127) == 0;
        int s = 0, prev = -1;
        uint32_t ph = 0;
        auto release_prev = [&]() {                        // the stage before the one just committed has been read
            if (prev >= 0) {
                wgmma_wait<1>();
                mbar_arrive_if(empty_bar(prev), leader);
            }
            prev = s;
            if (++s == ATTN_STAGES) { s = 0; ph ^= 1u; }
        };
        float sacc[LT / 2];
        for (int it = 0; it < kc1; ++it) {
            mbar_wait(full_bar(s), ph);
            wgmma_fence();
            const uint32_t st = base + s * ATTN_STAGE_BYTES;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                Wgmma<LT>::template mma<0, 0>(sacc, wgmma_desc_sw128(st + g * 8192 + kk * 32, 16, 1024), wgmma_desc_sw128(st + 16384 + kk * 32, 16, 1024),
                                              (it | kk) != 0);
            wgmma_commit();
            release_prev();
        }
        wgmma_wait<0>();
        wgmma_fence_regs(sacc);
        // thread rows: h = 0 / 1 -> row 16 wq + lane / 4 + 8 h of this warpgroup; key of register j: 8 (j / 4) + 2 (lane % 4) + j % 2
        int rows[2], segs[2];
        float mx[2] = {-3.0e38f, -3.0e38f}, sum[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            rows[h] = 64 * g + 16 * wq + (lane >> 2) + 8 * h;
            segs[h] = (qt * 128 + rows[h]) / p.HW;         // image inside the batch (block-diagonal mask)
        }
#pragma unroll
        for (int j = 0; j < LT / 2; ++j) {
            const int h = (j >> 1) & 1, key = 8 * (j >> 2) + 2 * (lane & 3) + (j & 1);
            if (key / p.HW == segs[h]) mx[h] = fmaxf(mx[h], sacc[j]);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        }
        const float mxs[2] = {mx[0] * p.scale_log2e, mx[1] * p.scale_log2e};
#pragma unroll
        for (int j = 0; j < LT / 2; j += 2) {
            const int h = (j >> 1) & 1, key = 8 * (j >> 2) + 2 * (lane & 3);
            const float x0 = exp2f(fmaf(sacc[j], p.scale_log2e, -mxs[h])), x1 = exp2f(fmaf(sacc[j + 1], p.scale_log2e, -mxs[h]));
            const float e0 = (key / p.HW == segs[h]) ? x0 : 0.f, e1 = ((key + 1) / p.HW == segs[h]) ? x1 : 0.f;
            sum[h] += e0 + e1;
            // K chunk of 64 keys = 128 B per row; 16-byte units XOR-swizzled with the row (128B swizzle)
            const int r = rows[h];
            uint8_t* dst = p_ptr + (key >> 6) * 16384 + (r >> 3) * 1024 + (r & 7) * 128 + ((((key & 63) >> 3) ^ (r & 7)) << 4) + (key & 7) * 2;
            *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(e0, e1);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
            sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
        }
        fence_proxy_async_smem();                          // P was written through the generic proxy, wgmma reads it through the async proxy
        asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory");   // the warpgroup's 64 rows of P are complete

        float oacc[DN / 2];
        for (int kc = 0; kc < kc3; ++kc) {
            mbar_wait(full_bar(s), ph);
            wgmma_fence();
            const uint32_t st = base + s * ATTN_STAGE_BYTES;
            const uint32_t pa = p_base + kc * 16384 + g * 8192;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                Wgmma<DN>::template mma<0, 0>(oacc, wgmma_desc_sw128(pa + kk * 32, 16, 1024), wgmma_desc_sw128(st + 16384 + kk * 32, 16, 1024),
                                              (kc | kk) != 0);
            wgmma_commit();
            release_prev();
        }
        wgmma_wait<0>();
        wgmma_fence_regs(oacc);
        if (prev >= 0) mbar_arrive_if(empty_bar(prev), leader);
        const float inv[2] = {1.0f / sum[0], 1.0f / sum[1]};
#pragma unroll
        for (int j = 0; j < DN / 2; j += 2) {
            const int h = (j >> 1) & 1, col = 8 * (j >> 2) + 2 * (lane & 3);
            __nv_bfloat16* o = p.out + (static_cast<long long>(z) * LT + qt * 128 + rows[h]) * p.C + dc * DN + col;
            *reinterpret_cast<__nv_bfloat162*>(o) = __floats2bfloat162_rn(oacc[j] * inv[h], oacc[j + 1] * inv[h]);
        }
    }
    __syncthreads();
}

__device__ __forceinline__ void attn_unit(const AttnParams& p, const AttnParams* pm, const uint32_t base, uint8_t* base_ptr, const int qt,
                                          const int dc, const int z) {
    if (p.Lt == 256) {
        if (p.dn == 256) attn_unit_t<256, 256>(p, pm, base, base_ptr, qt, dc, z);
        else attn_unit_t<256, 128>(p, pm, base, base_ptr, qt, dc, z);
    } else {
        if (p.dn == 256) attn_unit_t<128, 256>(p, pm, base, base_ptr, qt, dc, z);
        else attn_unit_t<128, 128>(p, pm, base, base_ptr, qt, dc, z);
    }
}

__global__ void __launch_bounds__(ATTN_THREADS, 1) attn_kernel(const __grid_constant__ AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    const int n_dc = p.C / p.dn;
    attn_unit(p, &p, base, smem_raw + (base - raw), blockIdx.x / n_dc, blockIdx.x % n_dc, blockIdx.y);
}

}  // namespace sr3
