// attn_long_wgmma.cuh -- the core of SelfAttention for MORE than 256 tokens per image, as one tensor-core kernel with a streaming
// (online) softmax: no token x token matrix leaves the SM.
//
// attn_kernel (attn_wgmma.cuh) holds a whole row block of S in registers, which stops at 256 keys.  Here a CTA owns the same unit
// (attention batch z, 128 query rows, 128 of the C output channels) and walks the keys in blocks of 128, in ascending order:
//
//   S_blk = q k_blk^T            (wgmma, 64 x 128 per warpgroup in registers; K loop over C in 64-channel chunks)
//   m' = max(m, rowmax(S_blk));  a = 2^((m - m') scale);  l = a l + rowsum(2^((S_blk - m') scale));  O = a O
//   P~ = bf16(2^((S_blk - m') scale))  -> shared memory (128-byte swizzle, the A operand of the next wgmma)
//   O += P~ v_blk                (wgmma, 64 x 128 per warpgroup in registers)
//
// and after the last block stores O / l as bf16 [token][C].  scale = log2(e) / sqrt(C); the row sum l is taken from the unrounded
// exponentials, as in attn_kernel.  Key blocks are visited in one fixed order and nothing is accumulated with atomics: repeat launches
// are bit-identical.
//
// Registers: 64 (S block) + 64 (O) fp32 per thread is what fits under the 168-register cap of 288 threads, hence 128 keys x 128
// channels.  n_head = 1, so each of the C / 128 CTAs of a query tile recomputes S: the kernel executes (2 C / 128 + 2) Lt^2 128 FLOP
// per image where the algorithm needs 4 Lt^2 C (2.5x at C = 512, 4.5x at C = 1024).
// Shared memory: the q tile (128 x C bf16: 128 KB at C = 512, 256 KB at C = 1024) does not fit beside the stage ring for every
// config, so it is never resident: every S stage carries its 64-channel chunk of q next to the chunk of k.  Per key block a CTA
// pulls 128 C 2 (q) + 128 C 2 (k) + 128 128 2 (v) bytes through TMA, all of it from L2 after the first CTA of a query tile.
//
// The MMA issue order is S(0), then per key block: softmax(kb), P.v(kb), S(kb + 1) -- the P.v group and the next S group are in flight
// together and the one wait per block (wgmma_wait<0>) sits in front of the softmax, which is also where O is rescaled.
#pragma once
#include "attn_wgmma.cuh"

namespace sr3 {

constexpr int ATTNL_THREADS = 288;                       // two consumer warpgroups + the TMA producer warp (ATTN_PRODUCER_WARP)
constexpr int ATTNL_KB = 128;                            // keys per block
constexpr int ATTNL_DN = 128;                            // output channels per CTA
constexpr int ATTNL_STAGES = 5;
constexpr int ATTNL_STAGE_BYTES = 16384 + 16384;         // S stage: q chunk 128 x 64 | k chunk 128 x 64; P.v stage: - | vT 128 channels x 64 keys
constexpr int ATTNL_P_BYTES = 128 * ATTNL_KB * 2;        // P~: 128 rows x 128 keys, as two K chunks of 64
constexpr int ATTNL_SMEM_BYTES = 1024 + GEMM_HDR_BYTES + ATTNL_STAGES * ATTNL_STAGE_BYTES + ATTNL_P_BYTES;

__global__ void __launch_bounds__(ATTNL_THREADS, 1) attn_long_kernel(const __grid_constant__ AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t bar_base = (raw + 1023u) & ~1023u;                  // header: barriers
    const uint32_t base = bar_base + GEMM_HDR_BYTES;
    const uint32_t p_base = base + ATTNL_STAGES * ATTNL_STAGE_BYTES;
    uint8_t* p_ptr = smem_raw + (p_base - raw);
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (ATTNL_STAGES + s); };

    const int n_dc = p.C / ATTNL_DN;
    const int qt = blockIdx.x / n_dc, dc = blockIdx.x % n_dc, z = blockIdx.y;
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int kc1 = p.C / 64;                 // K chunks of S = q k^T
    constexpr int kc3 = ATTNL_KB / 64;        // K chunks of O += P v
    const int nb = p.Lt / ATTNL_KB;           // key blocks

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.qk_map);
        tma_prefetch_desc(&p.vt_map);
        for (int s = 0; s < ATTNL_STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 2); }   // empty: one arrive per warpgroup
        fence_mbar_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();                  // q, k, vT come from the preceding launch

    if (warp == ATTN_PRODUCER_WARP) {
        // ------------------------------------------------------------ TMA producer: S(0), then P.v(kb), S(kb + 1) for every key block
        int s = 0;
        uint32_t ph = 0;
        auto stage = [&](bool is_s, int kb, int c) {
            mbar_wait(empty_bar(s), ph ^ 1u);
            if (elect_one_sync()) {
                const uint32_t dst = base + s * ATTNL_STAGE_BYTES;
                if (is_s) {
                    mbar_arrive_expect_tx(full_bar(s), 32768);
                    tma_load_2d(dst, &p.qk_map, full_bar(s), c * 64, z * p.Lt + qt * 128);
                    tma_load_2d(dst + 16384, &p.qk_map, full_bar(s), p.C + c * 64, z * p.Lt + kb * ATTNL_KB);
                } else {
                    mbar_arrive_expect_tx(full_bar(s), 16384);
                    tma_load_2d(dst + 16384, &p.vt_map, full_bar(s), kb * ATTNL_KB + c * 64, z * p.C + dc * ATTNL_DN);
                }
            }
            __syncwarp();
            if (++s == ATTNL_STAGES) { s = 0; ph ^= 1u; }
        };
        for (int c = 0; c < kc1; ++c) stage(true, 0, c);
        for (int kb = 0; kb < nb; ++kb) {
            for (int c = 0; c < kc3; ++c) stage(false, kb, c);
            if (kb + 1 < nb)
                for (int c = 0; c < kc1; ++c) stage(true, kb + 1, c);
        }
    } else {
        // ------------------------------------------------------------ warpgroup g: query rows [64 g, 64 g + 64) of the tile
        const int g = warp >> 2;
        const int wq = warp & 3;
        const bool leader = (threadIdx.x & 127) == 0;
        int s = 0, prev = 0;
        bool have_prev = false;
        uint32_t ph = 0;
        auto release_prev = [&]() {                        // the stage before the one just committed has been read (branch-free)
            wgmma_wait<1>();
            mbar_arrive_if(empty_bar(prev), leader && have_prev);
            prev = s; have_prev = true;
            if (++s == ATTNL_STAGES) { s = 0; ph ^= 1u; }
        };
        // O is not zero-initialised (its first wgmma overwrites it): ptxas schedules such stores into the pipeline stage of S(0) and
        // then serialises every wgmma of the kernel (C7515)
        float sacc[ATTNL_KB / 2], oacc[ATTNL_DN / 2];
        auto s_block = [&](int chunks) {                   // S = q k_blk^T over `chunks` stages (0: no further block)
            for (int it = 0; it < chunks; ++it) {
                mbar_wait(full_bar(s), ph);
                wgmma_fence();
                const uint32_t st = base + s * ATTNL_STAGE_BYTES;
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)
                    Wgmma<ATTNL_KB>::template mma<0, 0>(sacc, wgmma_desc_sw128(st + g * 8192 + kk * 32, 16, 1024),
                                                        wgmma_desc_sw128(st + 16384 + kk * 32, 16, 1024), (it | kk) != 0);
                wgmma_commit();
                release_prev();
            }
        };
        // thread rows: h = 0 / 1 -> row 16 wq + lane / 4 + 8 h of this warpgroup; key of register j: 8 (j / 4) + 2 (lane % 4) + j % 2
        int rows[2];
        uint8_t* prow[2];
        float mrun[2] = {-3.0e38f, -3.0e38f}, sum[2] = {0.f, 0.f};     // running row max (raw logits) and this thread's share of the row sum
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = rows[h] = 64 * g + 16 * wq + (lane >> 2) + 8 * h;
            prow[h] = p_ptr + (r >> 3) * 1024 + (r & 7) * 128 + (lane & 3) * 4;
        }

        s_block(kc1);
        for (int kb = 0; kb < nb; ++kb) {
            wgmma_wait<0>();                               // S(kb) and P.v(kb - 1): sacc and oacc are ours, the P buffer is free again
            wgmma_fence_regs(sacc);
            wgmma_fence_regs(oacc);
            float mx[2] = {mrun[0], mrun[1]};
#pragma unroll
            for (int j = 0; j < ATTNL_KB / 2; ++j) mx[(j >> 1) & 1] = fmaxf(mx[(j >> 1) & 1], sacc[j]);
            float alpha[2], mxs[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
                mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
                alpha[h] = exp2f((mrun[h] - mx[h]) * p.scale_log2e);   // first block: 2^(-huge) = 0 on sum = 0; O is not read (its first wgmma does not accumulate)
                mrun[h] = mx[h];
                mxs[h] = mx[h] * p.scale_log2e;
                sum[h] *= alpha[h];
            }
#pragma unroll
            for (int j = 0; j < ATTNL_KB / 2; j += 2) {
                const int h = (j >> 1) & 1, key = 8 * (j >> 2);        // + 2 (lane % 4): folded into prow
                const float e0 = exp2f(fmaf(sacc[j], p.scale_log2e, -mxs[h])), e1 = exp2f(fmaf(sacc[j + 1], p.scale_log2e, -mxs[h]));
                sum[h] += e0 + e1;
                // K chunk of 64 keys = 128 B per row; 16-byte units XOR-swizzled with the row (128B swizzle)
                uint8_t* dst = prow[h] + (key >> 6) * 16384 + ((((key & 63) >> 3) ^ (rows[h] & 7)) << 4);
                *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(e0, e1);
            }
#pragma unroll
            for (int j = 0; j < ATTNL_DN / 2; ++j) oacc[j] *= alpha[(j >> 1) & 1];
            fence_proxy_async_smem();                      // P was written through the generic proxy, wgmma reads it through the async proxy
            asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory");   // the warpgroup's 64 rows of P are complete

            for (int kc = 0; kc < kc3; ++kc) {
                mbar_wait(full_bar(s), ph);
                wgmma_fence();
                const uint32_t st = base + s * ATTNL_STAGE_BYTES;
                const uint32_t pa = p_base + kc * 16384 + g * 8192;
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)
                    Wgmma<ATTNL_DN>::template mma<0, 0>(oacc, wgmma_desc_sw128(pa + kk * 32, 16, 1024),
                                                        wgmma_desc_sw128(st + 16384 + kk * 32, 16, 1024), (kb | kc | kk) != 0);
                wgmma_commit();
                release_prev();
            }
            s_block(kb + 1 < nb ? kc1 : 0);
        }
        wgmma_wait<0>();
        wgmma_fence_regs(oacc);
        float inv[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
            sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
            inv[h] = 1.0f / sum[h];
        }
#pragma unroll
        for (int j = 0; j < ATTNL_DN / 2; j += 2) {
            const int h = (j >> 1) & 1, col = 8 * (j >> 2) + 2 * (lane & 3);
            __nv_bfloat16* o = p.out + (static_cast<long long>(z) * p.Lt + qt * 128 + rows[h]) * p.C + dc * ATTNL_DN + col;
            *reinterpret_cast<__nv_bfloat162*>(o) = __floats2bfloat162_rn(oacc[j] * inv[h], oacc[j + 1] * inv[h]);
        }
    }
}

}  // namespace sr3
