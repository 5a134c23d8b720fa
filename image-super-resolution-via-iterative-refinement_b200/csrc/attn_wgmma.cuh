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
// Warp roles, as in the tile kernel (gemm_wgmma.cuh): warps 0..7 are two consumer warpgroups, each owning 64 query rows with S (64 x Lt)
// and then O (64 x DN) in registers; warps 8..11 are the producer warpgroup, of which warp 8 issues the TMA loads.  384 threads start at
// 168 registers each; after the set-up the producer warpgroup drops to 40 and the consumers rise to 232 (setmaxnreg), so the 128-float
// S row block of Lt = 256 and the 128-float O block of DN = 256 stay in registers instead of spilling.
// DN (64, 128 or 256 of the C output channels per CTA) is picked per shape on the host (make_attn_op): it only decides which CTA
// computes which columns, not how any column is summed.
#pragma once
#include <cuda_bf16.h>
#include <cuda.h>
#include "gemm_wgmma.cuh"

namespace sr3 {

constexpr int ATTN_THREADS = 384;
constexpr int ATTN_CONSUMER_WARPS = 8;
constexpr int ATTN_PRODUCER_WARP = 8;
constexpr int ATTN_CONSUMER_REGS = 232;
constexpr int ATTN_PRODUCER_REGS = 40;
static_assert(ATTN_CONSUMER_WARPS * 32 * ATTN_CONSUMER_REGS + (ATTN_THREADS - ATTN_CONSUMER_WARPS * 32) * ATTN_PRODUCER_REGS <= 65536, "register file");
static_assert(ATTN_THREADS == 384 && ATTN_PRODUCER_WARP == ATTN_CONSUMER_WARPS, "setmaxnreg acts on whole warpgroups: 2 consumer + 1 producer");
constexpr int ATTN_STAGES = 3;
constexpr int ATTN_STAGE_BYTES = 16384 + 32768;          // A: 128 rows x 64 | B: up to 256 rows x 64 (bf16, 128B-swizzled)
constexpr int ATTN_P_BYTES = 65536;                      // P: 128 rows x up to 256 keys, as K chunks of 64
constexpr int ATTN_SMEM_BYTES = 1024 + GEMM_HDR_BYTES + ATTN_STAGES * ATTN_STAGE_BYTES + ATTN_P_BYTES;   // header: barriers

struct AttnParams {
    CUtensorMap qk_map;      // 2-D bf16 [nz*Lt rows][2C], box {64, 128}
    CUtensorMap vt_map;      // 2-D bf16 [nz*C rows][Lt], box {64, min(dn, 128)}
    __nv_bfloat16* out;      // [nz*Lt][C]
    int C, Lt, HW, dn, nz;
    float scale_log2e;       // log2(e) / sqrt(C)
};

// One CTA = one (attention batch z, query tile qt, channel slice dc) unit for Lt = LT keys and DN output channels.
template <int LT, int DN>
__global__ void __launch_bounds__(ATTN_THREADS, 1) attn_kernel(const __grid_constant__ AttnParams p) {
    static_assert((LT == 128 || LT == 256) && (DN == 64 || DN == 128 || DN == 256), "attn_kernel shape");
    constexpr int VB = DN < 128 ? DN : 128;                            // rows of one vT box (vt_map)
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t bar_base = (raw + 1023u) & ~1023u;                  // header (gemm_wgmma.cuh): barriers
    const uint32_t base = bar_base + GEMM_HDR_BYTES;
    uint8_t* base_ptr = smem_raw + (base - raw);
    const int n_dc = p.C / DN;
    const int qt = blockIdx.x / n_dc, dc = blockIdx.x % n_dc, z = blockIdx.y;
    const uint32_t p_base = base + ATTN_STAGES * ATTN_STAGE_BYTES;
    uint8_t* p_ptr = base_ptr + ATTN_STAGES * ATTN_STAGE_BYTES;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (ATTN_STAGES + s); };

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int kc1 = p.C / 64;        // K chunks of S = q k^T
    constexpr int kc3 = LT / 64;     // K chunks of O = P v

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.qk_map);
        tma_prefetch_desc(&p.vt_map);
        for (int s = 0; s < ATTN_STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 2); }   // empty: one arrive per warpgroup
        fence_mbar_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();                  // q, k, vT come from the two preceding launches

    // The warp roles split here.  No block-wide barrier may follow: warps 9..11 have nothing more to do, and named barriers 2 / 3 count
    // the 128 threads of one consumer warpgroup.
    if (warp >= ATTN_CONSUMER_WARPS) {
        setmaxnreg_dec<ATTN_PRODUCER_REGS>();
        if (warp != ATTN_PRODUCER_WARP) return;
        // ------------------------------------------------------------ TMA producer warp (converged; one elected lane issues)
        int s = 0;
        uint32_t ph = 0;
        for (int it = 0; it < kc1 + kc3; ++it) {
            mbar_wait(empty_bar(s), ph ^ 1u);
            if (elect_one_sync()) {
                const uint32_t dst = base + s * ATTN_STAGE_BYTES;
                if (it < kc1) {
                    mbar_arrive_expect_tx(full_bar(s), 16384 + LT * 128);
                    tma_load_2d(dst, &p.qk_map, full_bar(s), it * 64, z * LT + qt * 128);
                    for (int j = 0; j < LT / 128; ++j)
                        tma_load_2d(dst + 16384 + j * 16384, &p.qk_map, full_bar(s), p.C + it * 64, z * LT + j * 128);
                } else {
                    mbar_arrive_expect_tx(full_bar(s), DN * 128);
                    for (int j = 0; j < DN / VB; ++j)
                        tma_load_2d(dst + 16384 + j * VB * 128, &p.vt_map, full_bar(s), (it - kc1) * 64, z * p.C + dc * DN + j * VB);
                }
            }
            __syncwarp();
            if (++s == ATTN_STAGES) { s = 0; ph ^= 1u; }
        }
    } else {
        setmaxnreg_inc<ATTN_CONSUMER_REGS>();
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
        // Block-diagonal mask: key and row are in the same image iff key / HW == row / HW, i.e. 0 <= key - HW (row / HW) < HW.  With the
        // lane's part of the key folded into seg0, that is one unsigned compare of a constant per register instead of a division.  A
        // masked logit becomes -inf: the row maximum skips it and its exponential is exactly 0, as a masked P must be.
        int rows[2], seg0[2];
        float mx[2] = {-3.0e38f, -3.0e38f}, sum[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            rows[h] = 64 * g + 16 * wq + (lane >> 2) + 8 * h;
            seg0[h] = (qt * 128 + rows[h]) / p.HW * p.HW - 2 * (lane & 3);   // first key of the row's image, less the lane's key offset
        }
        auto same_image = [&](int jkey, int h) { return static_cast<unsigned>(jkey - seg0[h]) < static_cast<unsigned>(p.HW); };
#pragma unroll
        for (int j = 0; j < LT / 2; ++j) {
            const int h = (j >> 1) & 1;
            if (!same_image(8 * (j >> 2) + (j & 1), h)) sacc[j] = -INFINITY;
            mx[h] = fmaxf(mx[h], sacc[j]);
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
            const float e0 = exp2f(fmaf(sacc[j], p.scale_log2e, -mxs[h])), e1 = exp2f(fmaf(sacc[j + 1], p.scale_log2e, -mxs[h]));
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
}

}  // namespace sr3
