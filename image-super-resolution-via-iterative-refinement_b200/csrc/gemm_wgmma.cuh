// Implicit-GEMM tile kernel for sm_90a (wgmma + TMA), the one tensor-core kernel of the SR3 path.
//
//   D[(MH x 128) pixels x BLOCK_N] = sum over stages, taps   A_tap[128 x 64] * B_tap[BLOCK_N x 64]^T     (bf16 -> fp32 in registers)
//
// * A pipeline stage holds ONE activation tile fetched by one 5-D TMA box from an NHWC bf16 tensor (out-of-image pixels are
//   zero-filled by TMA = conv padding; no im2col buffer exists) plus 1..3 weight tiles.  For a 3x3 stride-1 conv the
//   box is a "tall halo": 8 pixels wide, (rows + 2) high, shifted horizontally by the tap column dw.  The three vertical
//   taps of that column are then just three wgmma descriptors whose start address is shifted by whole 8-pixel rows
//   (1024 B = one 128-byte-swizzle atom), so every activation byte that enters shared memory feeds 3 taps x BLOCK_N outputs,
//   and with MH = 2 two 128-row halves share the halo and the weights.
// * The generic form (MH = 1, one tap per stage, box = any 128 rows of a 5-D view) covers stride-2 convs (row / column parity
//   folded into the view), 1x1 convs, the 8x8 levels and the attention matrix products.
// * B rows are output channels (or keys / head-dim for attention) of a K-major bf16 matrix, 2-D TMA box {64, BLOCK_N}.
// * The stage table is built on the host (engine.cu): 3x3 taps, the 1x1 residual conv accumulated into the same
//   tile and channel concats are all just more stages.
// * Persistent CTAs (one per SM) walk a contiguous range of tiles.  Warp 8 = TMA producer (its warpgroup runs on 40 registers per thread
//   so that the consumers get 232, see GEMM_THREADS); warps 0..7 = two consumer warpgroups that
//   issue the wgmma of their share of the tile (MH = 2: one 128-row half each; MH = 1: one half of the columns each; tiles of at most
//   32 columns: warpgroup 0 alone) and then run the epilogue on it: accumulator -> per-warp 32 x 32 transposition in shared memory ->
//   bias / FiLM -> residual (TMA prefetched into smem) -> fp32 tile staged in swizzled smem and written by TMA store (and/or bf16
//   direct stores) -> per-(image, channel) GroupNorm partial sums, accumulated in registers across tiles.
//   Ping-pong schedule (PP, 256x64 / 128x128 / 128x64 tiles): instead each warpgroup owns every other tile of the CTA's range and the two
//   take turns at the MMAs (named barriers 2 and 3), so the epilogue of one tile runs while the tensor cores work on the next.
// * A warpgroup's m64 wgmma pair covers 128 rows with the 8-row groups interleaved (instruction i reads groups 2g + i at a 2048 B group
//   stride), so that warp q of the group holds exactly rows [32 q, 32 q + 32): the 32-row unit of the epilogue, of its TMA boxes and of
//   the statistics.
// * The last UNet conv (Cout = 3) uses the posterior epilogue: eps -> x0 -> clamp -> posterior mean -> + sigma_t * z
//   (model/sr3_modules/diffusion.py:141-174 of the reference) and writes x_{t-1} straight into the next step's input.
#pragma once
#include <cuda.h>
#include <type_traits>
#include "ptx.cuh"
#include "sampling_noise.cuh"

namespace sr3 {

struct OutSpec {
    long long sZ, sB, sH, sW, off;   // element strides: gemm-batch, image, row, column; constant offset
};

// Device-resident control block: everything that changes between launches of the (captured) step graph.
struct StepCtl {
    int t_cur;            // timestep of the running step
    int t_next;           // timestep the next step_begin will load
    int nl_from_table;    // 1: noise level = sqrt_alphas_cumprod_prev[t+1] (sampling); 0: read nl_buf[b]
    int out_mode;         // 0: write eps (UNet.forward); 1: posterior update (p_sample)
    int use_noise_buf;    // 1: z from noise_buf; 0: Philox
    int write_mean;       // 1: also store the posterior mean (p_mean_variance)
    int clip;             // clip_denoised
    int update_state;     // 1: write x_{t-1} into x_state and the UNet input buffer
    unsigned long long seed;
    unsigned long long sample_offset;   // global index of image 0 (multi-GPU sharding keeps streams rank independent)
};

struct PostParams {
    const float* tab;         // [5][T]: sqrt_recip_ac, sqrt_recipm1_ac, post_coef1, post_coef2, post_logvar_clipped
    int T;
    int H, W, C;              // image geometry, C = sample channels (3)
    float* x_state;           // [B,C,H,W] fp32 NCHW
    float* eps_out;           // [B,C,H,W]
    float* mean_out;          // [B,C,H,W]
    const float* noise_buf;   // [B,C,H,W]
    __nv_bfloat16* in_buf;    // NHWC bf16 UNet input, channel stride in_C, x_t lives at channels [in_coff, in_coff+C)
    int in_C, in_coff;
    int in_lo_off;            // precise mode: the low halves (x - bf16(x)) live in_lo_off channels further; 0 = bf16 mode
};

// One pipeline stage of the K loop (host-built table, copied to shared memory by the kernel): up to three K slabs
// (64 channels each).  Tall-halo stages load ONE activation box that serves all taps (a_multi = 0); generic stages load one
// box per slab (a_multi = 1) -- grouping slabs only amortises the mbarrier handshake.
struct StageTap {
    int a_chan;      // channel coordinate (dim 0) of the A box
    int dw, dh, p;   // box shift along W', H' and the parity coordinate
    int b_col;       // B column (K coordinate)
    int a_off;       // byte offset of this tap's first row inside the A stage buffer (multiple of 1024)
};
struct StageDesc {
    int ntaps;       // K slabs in this stage (1..3)
    int a_multi;     // 1: every tap has its own A box (loaded at a_off), 0: one box (tap 0's coordinates) shared by all taps
    int a_sel;       // which A tensor map
    int pad0;
    StageTap tap[3];
    int pad1, pad2;  // 96 bytes = 6 x int4
};

struct GemmParams {
    CUtensorMap a_map[2];
    CUtensorMap b_map;
    CUtensorMap out_map;     // fp32 output, 5-D {N, W, 1, H, B|Z}, box {32, w_sub, 1, h_sub, 1}: one warp's 32 rows x 32 columns
    CUtensorMap res_map;     // fp32 residual, same geometry
    const StageDesc* ktab;   // [num_k]
    int num_k;
    int a_stage_bytes;       // bytes reserved for activation boxes per stage (multiple of 1024)
    int a_box_bytes;         // bytes of ONE activation box (what a single TMA load delivers)
    int a_half_off;          // byte offset between the two 128-row halves inside the A buffer (MH = 2)
    int b_taps;              // weight tiles reserved per stage (max ntaps)
    int tiles_w, tiles_h, tiles_b;
    int n_tiles, nz;         // persistent schedule: tile = m_tile + tiles_m * (n_tile + n_tiles * z); CTA c owns a contiguous range
    int tma_epi;             // 1: fp32 output / residual go through smem + TMA (out_map / res_map)
    int epi_c4_is_z;         // 5th coordinate of out_map / res_map: gemm-batch z (1) or image index (0)
    int ksplit;              // split-K factor: ksplit CTAs share one output tile, partial sums meet in `ws` (fp32, same addressing as out_f32)
    float* ws;               // zero between launches (the finalising CTA clears what it reads)
    unsigned int* counters;  // [tiles] arrival counters (monotonic: +ksplit per launch)
    const void* pf_ptr;      // weights of the NEXT tile-kernel launch: pulled into L2 while this launch runs (they would otherwise be
    long long pf_bytes;      // first-touch HBM reads on the critical path of every pipeline stage of that launch)
    int w_box, h_box, b_box; // pixel patch of one tile: w_box * h_box * b_box == MH * 128 (all powers of two)
    int w_shift, h_shift;    // log2(w_box), log2(h_box): the epilogue splits a tile row into (w, h, image) with shifts, not divisions
    int a_zstep, b_zrows;
    int stages;
    // epilogue
    int mode;                // 0 normal, 1 final conv (eps / posterior)
    int OW, OH, OB, n_valid;
    float scale;
    const float* bias;
    const float* bias2;      // per-image bias (FiLM + conv bias), bias2[img * bias2_stride + n]
    int bias2_stride;
    const float* resid;
    OutSpec rs;
    float* out_f32;
    OutSpec os;
    __nv_bfloat16* out_bf16;
    OutSpec hs;
    // columns >= t_col0 are stored TRANSPOSED instead: out_t[(img / t_per) * t_rows + (n - t_col0)][(img % t_per) * OH*OW + oh*OW + ow]
    // (the v third of the qkv projection lands directly as the K-major B operand v^T of O = P v)
    __nv_bfloat16* out_t;
    int t_col0, t_rows, t_ld, t_per;
    double* stats;           // [B][stats_C][2] (sum, sumsq) in fp64, channel offset stats_coff (see stats_quantize)
    int stats_C, stats_coff;
    const StepCtl* ctl;
    PostParams post;
    // z_phase = 1: the gemm-batch index z = 2*py + px is the output phase of a folded (nearest-2x -> conv3x3): taps shift by (py, px) input
    // pixels, weights of phase z start at row z * b_zrows, the tile lands at output pixel (2h + py, 2w + px) -- out_map is then
    // {2N (px, n), W, 2 (py), H, B} and plain stores add (py * z_off_hi + px * z_off_lo) elements
    int z_phase;
    long long z_off_hi, z_off_lo;
    // Precise mode (fp32-level accuracy on the bf16 tensor cores): every operand is a pair hi = bf16(x), lo = bf16(x - hi) and a product is
    // hi*hi + hi*lo + lo*hi (the dropped lo*lo term is ~2^-18 relative).  The K loop runs `passes` = 3 times over the SAME stage table:
    // pass 1 reads the low weights (B column + lo_b_col), pass 2 the low activations (A channel + lo_a_chan[source]).  Low halves of
    // bf16 outputs go lo_out_off elements (lo_t_off for the transposed store) behind the high halves.  passes = 1: plain bf16.
    int passes, lo_b_col, lo_a_chan[2];
    long long lo_out_off, lo_t_off;
};

// warps 0..7: two consumer warpgroups (MMA + epilogue); warps 8..11: the producer warpgroup, of which warp 8 issues the TMA loads.
// A block of 384 threads starts at 168 registers per thread (a sub-partition's 16384 registers over its three warps).  After the set-up
// the producer warpgroup gives all but 40 back and the consumers take them (setmaxnreg): 2 x 128 x 232 + 128 x 40 = 64512 <= 65536, so
// the accumulator and the epilogue of the widest tiles stay in registers.
constexpr int GEMM_THREADS = 384;
constexpr int GEMM_EPI_WARPS = 8;
constexpr int GEMM_PRODUCER_WARP = 8;
constexpr int GEMM_CONSUMER_REGS = 232;
constexpr int GEMM_PRODUCER_REGS = 40;
static_assert(GEMM_EPI_WARPS * 32 * GEMM_CONSUMER_REGS + (GEMM_THREADS - GEMM_EPI_WARPS * 32) * GEMM_PRODUCER_REGS <= 65536, "register file");
static_assert(GEMM_THREADS == 384 && GEMM_PRODUCER_WARP == GEMM_EPI_WARPS, "setmaxnreg acts on whole warpgroups: 2 consumer + 1 producer");
constexpr int GEMM_MAX_STAGES = 8;
// per epilogue warp: 4 KB staging (accumulator transposition, then the fp32 chunk for the TMA store) [+ 2 x 4 KB residual staging when the layer has one]
__host__ __device__ constexpr int gemm_epi_warp_bytes(bool resid) { return resid ? 12288 : 4096; }
__host__ __device__ constexpr int gemm_epi_bytes(bool resid) { return GEMM_EPI_WARPS * gemm_epi_warp_bytes(resid); }
constexpr int GEMM_MAX_K = 160;              // stages per tile (<= 3 K slabs each); the table is sized per launch
// Shared-memory header (first 2 KB of the 1024-aligned region): the mbarriers, in [0, 512).  They need less than 2 KB, but the size
// enters gemm_aux_bytes and so the stage counts the planner picks: shrinking it changes plans, and with them results and speed.
constexpr int GEMM_HDR_BYTES = 2048;
// Tiles of at most 32 columns (MH = 1) are computed by warpgroup 0 alone; every other tile is shared by both consumer warpgroups.
__host__ __device__ constexpr bool gemm_single_wg(int block_n, int mh) { return mh == 1 && block_n <= 32; }
// Ping-pong schedule: each consumer warpgroup owns whole tiles (local tiles g, g + 2, ... of the CTA's range), their MMA phases take
// turns through two named barriers, so one warpgroup's epilogue runs while the other one feeds the tensor cores.  Shapes it exists for:
__host__ __device__ constexpr bool gemm_pingpong_ok(int block_n, int mh) { return (mh == 2 && block_n == 64) || (mh == 1 && (block_n == 64 || block_n == 128)); }
constexpr int GEMM_ORDER_BAR = 2;            // named barriers 2 (warpgroup 0's turn) and 3 (warpgroup 1's turn); 1 is the split-K pass
// arrivals that release a pipeline stage: one per warpgroup that reads it
__host__ __device__ constexpr int gemm_stage_readers(int block_n, int mh, bool pp) { return (pp || gemm_single_wg(block_n, mh)) ? 1 : 2; }
__host__ __device__ constexpr int gemm_aux_bytes(int num_k) {
    return GEMM_HDR_BYTES + ((num_k * 96 + 127) / 128) * 128 /*stage table*/ + GEMM_EPI_WARPS * 2 * 32 * 4 /*per-warp bias staging*/;
}

__host__ __device__ constexpr int gemm_stage_bytes(int block_n, int a_stage_bytes, int b_taps) { return a_stage_bytes + b_taps * block_n * 128; }
__host__ __device__ constexpr int gemm_smem_bytes(int block_n, int a_stage_bytes, int b_taps, int stages, bool resid, int num_k) {
    return stages * gemm_stage_bytes(block_n, a_stage_bytes, b_taps) + gemm_epi_bytes(resid) + 1024 /*align slack*/ + gemm_aux_bytes(num_k);
}

// GroupNorm statistics are accumulated with fp64 atomics.  Every contribution is first rounded to a multiple of 2^-20, so as long as
// a sum stays below 2^33 (|x|_rms < 180 over a 512x512 channel) every addition is EXACT: the result does not depend on the order in
// which the CTAs arrive -- repeat runs are bit identical -- and E[x^2] - mean^2 is evaluated in fp64 by the consumer (no fp32
// cancellation for |mean| >> std).  The rounding itself is unbiased and ~1e-6 absolute per contribution, far below eps = 1e-5.
__device__ __forceinline__ double stats_quantize(double v) { return rint(v * 1048576.0) * (1.0 / 1048576.0); }

// Transposing warp reduction: every lane holds v[0..31] (one row, 32 columns); afterwards lane l returns the sum over the
// 32 lanes (rows) of column l.  31 shuffles instead of 32 x 5.
__device__ __forceinline__ float warp_column_sums(float (&v)[32]) {
    const uint32_t lane = lane_id();
#pragma unroll
    for (int half = 16; half >= 1; half >>= 1) {
        const bool up = (lane & half) != 0;
#pragma unroll
        for (int j = 0; j < half; ++j) {
            const float keep = up ? v[j + half] : v[j];
            const float send = up ? v[j] : v[j + half];
            v[j] = keep + __shfl_xor_sync(0xffffffffu, send, half);
        }
    }
    return v[0];
}

__device__ __forceinline__ long long out_index(const OutSpec& s, int z, int img, int oh, int ow) {
    return s.off + static_cast<long long>(z) * s.sZ + static_cast<long long>(img) * s.sB + static_cast<long long>(oh) * s.sH +
           static_cast<long long>(ow) * s.sW;
}

// reference: predict_start_from_noise + clamp + q_posterior + p_sample noise add (diffusion.py:141-174)
__device__ __forceinline__ void final_epilogue(const GemmParams& p, const float (&eps)[4], int img, int oh, int ow) {
    const PostParams& q = p.post;
    const StepCtl ctl = *p.ctl;
    const long long plane = static_cast<long long>(q.H) * q.W;
    const long long pix = static_cast<long long>(oh) * q.W + ow;
    if (ctl.out_mode == 0) {
        for (int c = 0; c < q.C; ++c) q.eps_out[(static_cast<long long>(img) * q.C + c) * plane + pix] = eps[c];
        return;
    }
    const int t = ctl.t_cur;
    const float c1 = q.tab[t], c2 = q.tab[q.T + t], pc1 = q.tab[2 * q.T + t], pc2 = q.tab[3 * q.T + t];
    const float sigma = posterior_sigma(q.tab, q.T, t);
    float z[4] = {0.f, 0.f, 0.f, 0.f};
    if (t > 0) {
        if (ctl.use_noise_buf) {
            for (int c = 0; c < q.C; ++c) z[c] = q.noise_buf[(static_cast<long long>(img) * q.C + c) * plane + pix];
        } else {
            // (sampling_noise4 of sampling_noise.cuh, spelled out: this kernel's code is kept instruction for instruction)
            uint32_t ctr[4] = {static_cast<uint32_t>(pix), static_cast<uint32_t>(ctl.sample_offset + img), static_cast<uint32_t>(t),
                               static_cast<uint32_t>((ctl.sample_offset + img) >> 32)};
            philox4x32_10(ctr, static_cast<uint32_t>(ctl.seed), static_cast<uint32_t>(ctl.seed >> 32));
            box_muller(ctr[0], ctr[1], z[0], z[1]);
            box_muller(ctr[2], ctr[3], z[2], z[3]);
        }
    }
    for (int c = 0; c < q.C; ++c) {
        const long long idx = (static_cast<long long>(img) * q.C + c) * plane + pix;
        const float xt = q.x_state[idx];
        float x0 = __fsub_rn(__fmul_rn(c1, xt), __fmul_rn(c2, eps[c]));
        if (ctl.clip) x0 = fminf(fmaxf(x0, -1.0f), 1.0f);
        const float mean = __fadd_rn(__fmul_rn(pc1, x0), __fmul_rn(pc2, xt));
        if (ctl.write_mean) q.mean_out[idx] = mean;
        const float xn = posterior_sample(mean, z[c], sigma);
        if (ctl.update_state) {
            q.x_state[idx] = xn;
            __nv_bfloat16* ib = q.in_buf + (static_cast<long long>(img) * plane + pix) * q.in_C + q.in_coff + c;
            const __nv_bfloat16 hi = __float2bfloat16_rn(xn);
            *ib = hi;
            if (q.in_lo_off) ib[q.in_lo_off] = __float2bfloat16_rn(xn - __bfloat162float(hi));
        }
    }
}

// CTA-local set-up of one tile-kernel launch: stage table -> shared memory, TMA descriptor prefetch, mbarrier initialisation.
// Must be followed by a block-wide barrier.
__device__ __forceinline__ void gemm_stage_setup(const GemmParams& p, const GemmParams* pm, const uint32_t base, uint8_t* base_ptr, const int block_n,
                                                 const int mh, const bool pp) {
    const int stages = p.stages;
    const int stage_bytes = p.a_stage_bytes + p.b_taps * block_n * 128;
    const bool use_res_tma = p.tma_epi && p.resid != nullptr && p.ksplit <= 1;
    const int epi_bytes = GEMM_EPI_WARPS * gemm_epi_warp_bytes(use_res_tma);
    uint8_t* aux_ptr = base_ptr + GEMM_HDR_BYTES + stages * stage_bytes + epi_bytes;
    {
        const int4* src = reinterpret_cast<const int4*>(p.ktab);
        int4* dst = reinterpret_cast<int4*>(aux_ptr);
        for (int i = threadIdx.x; i < p.num_k * 6; i += blockDim.x) dst[i] = __ldg(&src[i]);
    }
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&pm->a_map[0]);
        tma_prefetch_desc(&pm->a_map[1]);
        tma_prefetch_desc(&pm->b_map);
        if (p.tma_epi) { tma_prefetch_desc(&pm->out_map); tma_prefetch_desc(&pm->res_map); }
        const uint32_t bar_base = base;
        const uint32_t consumers = gemm_stage_readers(block_n, mh, pp);
        for (int s = 0; s < stages; ++s) {
            mbar_init(bar_base + 8u * s, 1);                                     // full
            mbar_init(bar_base + 8u * (GEMM_MAX_STAGES + s), consumers);         // empty: one arrive per consumer warpgroup that reads it
        }
        for (int w = 0; w < 2 * GEMM_EPI_WARPS; ++w) mbar_init(bar_base + 8u * (2 * GEMM_MAX_STAGES + w), 1);   // residual tiles
        fence_mbar_init();
    }
}

// Accumulator chunk -> rows: this warp's 32 rows x CW columns of chunk CL of the warpgroup accumulator go through the warp's 4 KB
// staging buffer (float4 index XOR-swizzled with the row: conflict-free both ways) and come back as lane = row, v[j] = column j.
// CL is a template argument so that only chunk CL's registers are read: the chunk is dead afterwards.
template <int WN, int CW, int CL>
__device__ __forceinline__ void acc_chunk_rows(const float (&acc)[2][WN / 2], float* buf, float (&v)[32]) {
    static_assert(CW <= 32 && (CL + 1) * CW <= WN, "accumulator chunk");
    const int lane = static_cast<int>(lane_id());
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
        for (int j = (CL * CW) / 2; j < ((CL + 1) * CW) / 2; j += 2) {
            const int r = (lane >> 2) + 8 * i + 16 * ((j >> 1) & 1);
            const int cc = 8 * (j >> 2) - CL * CW + 2 * (lane & 3);
            *reinterpret_cast<float2*>(buf + r * 32 + (cc ^ ((r & 7) << 2))) = make_float2(acc[i][j], acc[i][j + 1]);
        }
    }
    __syncwarp();
#pragma unroll
    for (int c4 = 0; c4 < CW / 4; ++c4) {
        const float4 x = *reinterpret_cast<const float4*>(buf + lane * 32 + ((4 * c4) ^ ((lane & 7) << 2)));
        v[4 * c4] = x.x; v[4 * c4 + 1] = x.y; v[4 * c4 + 2] = x.z; v[4 * c4 + 3] = x.w;
    }
}

// f(std::integral_constant<int, I>{}) for I = 0 .. N-1: the body sees its index as a compile-time constant.
template <int N, int I = 0, typename F>
__device__ __forceinline__ void static_for(F&& f) {
    if constexpr (I < N) {
        f(std::integral_constant<int, I>{});
        static_for<N, I + 1>(f);
    }
}

// One lane's fp64 GroupNorm running sums over N 32-column chunks of one image: chunk c is column n0 + (ch0 + c) * 32 + lane.
// stats_quantize rounds a sum once per flush, so where a run ends is part of the result: a run ends when the image or the column
// block changes, and at the end of the op.
template <int N>
struct StatRun {
    double sum[N], sq[N];
    int img = -1, n0 = -1;
    __device__ __forceinline__ StatRun() { clear(); }
    __device__ __forceinline__ void clear() {
#pragma unroll
        for (int c = 0; c < N; ++c) { sum[c] = 0.0; sq[c] = 0.0; }
    }
    __device__ __forceinline__ void flush(const GemmParams& p, const int ch0, const int lane) {
        if (img >= 0 && img < p.OB) {
#pragma unroll
            for (int c = 0; c < N; ++c) {
                const int n = n0 + (ch0 + c) * 32 + lane;
                if (n < p.n_valid) {
                    double* st = p.stats + (static_cast<long long>(img) * p.stats_C + p.stats_coff + n) * 2;
                    red_add_f64_global(st, stats_quantize(sum[c]));
                    red_add_f64_global(st + 1, stats_quantize(sq[c]));
                }
            }
        }
        clear();
    }
    // the next contributions belong to image `im`, column block `nb0`
    __device__ __forceinline__ void start(const GemmParams& p, const int im, const int nb0, const int ch0, const int lane) {
        if (im != img || nb0 != n0) { flush(p, ch0, lane); img = im; n0 = nb0; }
    }
    __device__ __forceinline__ void add(const int c, const double s, const double q) {
#pragma unroll
        for (int cc = 0; cc < N; ++cc)
            if (cc == c) { sum[cc] += s; sq[cc] += q; }
    }
};

// Persistent, warp-specialised tile loop of gemm_tile_kernel (see the file header).  `p` lives in the kernel parameter space and `pm`
// points at it (TMA descriptors are addressed through it).  `base` / `base_ptr`: 1024-aligned start of the CTA's dynamic shared memory
// (header first).
// PP = false: cooperative schedule, both warpgroups share every tile.  PP = true: ping-pong schedule (gemm_pingpong_ok shapes, no split-K):
// warpgroup g owns the CTA's local tiles g, g + 2, ... with an accumulator of the whole tile, and the warpgroups issue their MMAs in
// turn (order barrier GEMM_ORDER_BAR + g), so the stage ring is consumed strictly in order, one warpgroup per stage.
template <int BLOCK_N, int MH, bool PP = false>
__device__ __forceinline__ void gemm_tile_body(const GemmParams& p, const GemmParams* pm, const uint32_t base, uint8_t* base_ptr,
                                               const int cta, const int ncta) {
    static_assert(!PP || gemm_pingpong_ok(BLOCK_N, MH), "ping-pong tile shape");
    constexpr int B_BYTES = BLOCK_N * 128;
    constexpr bool SINGLE = !PP && gemm_single_wg(BLOCK_N, MH);
    constexpr int WN = (PP || SINGLE || MH == 2) ? BLOCK_N : BLOCK_N / 2;   // accumulator columns of one warpgroup
    constexpr int AH = PP ? MH : 1;                                     // 128-row halves in one warpgroup's accumulator
    constexpr int CW = WN < 32 ? WN : 32;                               // columns of one epilogue chunk
    constexpr int NCH = BLOCK_N >= 32 ? BLOCK_N / 32 : 1;               // 32-column chunks per 128-row half
    constexpr int NITEMS = MH * NCH;                                    // work items (half, chunk) per tile
    constexpr int OWN = PP ? NITEMS : SINGLE ? 1 : NITEMS / 2;          // items held by one warpgroup's accumulator
    constexpr int NSTAT = PP ? NCH : OWN;                               // chunks of one GroupNorm run (ping-pong: one run per half)
    static_assert(WN % CW == 0 && AH * WN <= 128, "accumulator shape");

    const int stages = p.stages;
    const int stage_bytes = p.a_stage_bytes + p.b_taps * B_BYTES;            // multiple of 1024
    const bool use_res_tma = p.tma_epi && p.resid != nullptr && p.ksplit <= 1;
    const int epi_warp_bytes = gemm_epi_warp_bytes(use_res_tma);
    const int epi_bytes = GEMM_EPI_WARPS * epi_warp_bytes;
    const uint32_t bar_base = base;                                          // header
    const uint32_t stage_base = base + GEMM_HDR_BYTES;
    uint8_t* stage_ptr = base_ptr + GEMM_HDR_BYTES;
    const uint32_t epi_base = stage_base + stages * stage_bytes;
    // barriers: full[8] empty[8] res_full[8 warps][2]
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (GEMM_MAX_STAGES + s); };
    auto res_bar = [&](int w, int b) { return bar_base + 8u * (2 * GEMM_MAX_STAGES + 2 * w + b); };   // w in [0, 8)
    uint8_t* aux_ptr = stage_ptr + stages * stage_bytes + epi_bytes;
    // with ~227 KB of shared memory per CTA there is no L1 left: anything re-read per iteration must live in smem
    StageDesc* ktab_s = reinterpret_cast<StageDesc*>(aux_ptr);
    float* bias_s = reinterpret_cast<float*>(aux_ptr + ((p.num_k * 96 + 127) / 128) * 128);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int tiles_m = p.tiles_w * p.tiles_h * p.tiles_b;
    const int ksplit = p.ksplit > 1 ? p.ksplit : 1;
    const int total_tiles = tiles_m * p.n_tiles * p.nz * ksplit;      // split index fastest: the CTAs of one output tile run together
    const int num_kt = p.num_k * (p.passes > 1 ? p.passes : 1);       // stages per tile (precise mode: three passes over the table)
    gemm_stage_setup(p, pm, base, base_ptr, BLOCK_N, MH, PP);
    __syncthreads();
    if (warp == 2 && lane == 0 && p.pf_bytes > 0) {                   // L2 prefetch of this CTA's slice of the next layer's weights
        long long chunk = ((p.pf_bytes + ncta - 1) / ncta + 15) & ~15ll;
        const long long off = chunk * cta;
        if (off < p.pf_bytes) {
            if (off + chunk > p.pf_bytes) chunk = (p.pf_bytes - off) & ~15ll;
            const char* src = static_cast<const char*>(p.pf_ptr) + off;
            for (long long done = 0; done < chunk; done += 65536) {
                const unsigned int n = static_cast<unsigned int>(chunk - done < 65536 ? chunk - done : 65536);
                if (n >= 16) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src + done), "r"(n) : "memory");
            }
        }
    }
    pdl_launch_dependents();  // the next kernel may be scheduled onto SMs as our CTAs retire ...
    pdl_wait();               // ... and we touch upstream activations / statistics only after the previous kernel completed

    auto decode = [&](int tile_s, int& w0, int& h0, int& b0, int& n0, int& z) {
        const int tile = tile_s / ksplit;
        const int tm = tile % tiles_m;          // m fastest: a CTA's consecutive tiles share the weight slab and mostly the image
        const int r = tile / tiles_m;
        const int nt = r % p.n_tiles;
        z = r / p.n_tiles;
        const int tw = tm % p.tiles_w;
        const int th = (tm / p.tiles_w) % p.tiles_h;
        const int tb = tm / (p.tiles_w * p.tiles_h);
        w0 = tw * p.w_box; h0 = th * p.h_box; b0 = tb * p.b_box + z * p.a_zstep; n0 = nt * BLOCK_N;
    };
    // contiguous tile range of this CTA (balanced to +-1 tile)
    const int tile_begin = static_cast<int>((static_cast<long long>(total_tiles) * cta) / ncta);
    const int tile_end = static_cast<int>((static_cast<long long>(total_tiles) * (cta + 1)) / ncta);

    // The warp roles split here.  No block-wide barrier may follow: warps 9..11 have nothing more to do, and named barriers 1..3 count the
    // 256 consumer threads only.
    if (warp >= GEMM_EPI_WARPS) {
        setmaxnreg_dec<GEMM_PRODUCER_REGS>();
        if (warp == GEMM_PRODUCER_WARP) {
            // ---------------------------------------------------- TMA producer warp (converged; one elected lane issues)
            int s = 0;
            uint32_t ph = 0;
            for (int tile = tile_begin; tile < tile_end; ++tile) {
                int w0, h0, b0, n0, z;
                decode(tile, w0, h0, b0, n0, z);
                const int brow = n0 + z * p.b_zrows;
                const int zdw = p.z_phase ? (z & 1) : 0, zdh = p.z_phase ? (z >> 1) : 0;
                const int sp = tile % ksplit;
                const int k0 = (num_kt * sp) / ksplit, k1 = (num_kt * (sp + 1)) / ksplit;
                for (int k = k0; k < k1; ++k) {
                    mbar_wait(empty_bar(s), ph ^ 1u);
                    if (elect_one_sync()) {
                        const int pass = k / p.num_k;
                        const StageDesc& e = ktab_s[k - pass * p.num_k];
                        const int a_lo = (pass == 2) ? p.lo_a_chan[e.a_sel] : 0, b_lo = (pass == 1) ? p.lo_b_col : 0;
                        const uint32_t a_dst = stage_base + s * stage_bytes;
                        const int na = e.a_multi ? e.ntaps : 1;
                        mbar_arrive_expect_tx(full_bar(s), na * p.a_box_bytes + e.ntaps * B_BYTES);
                        for (int t = 0; t < na; ++t)
                            tma_load_5d(a_dst + (e.a_multi ? e.tap[t].a_off : 0), &pm->a_map[e.a_sel], full_bar(s), e.tap[t].a_chan + a_lo, w0 + e.tap[t].dw + zdw, e.tap[t].p,
                                        h0 + e.tap[t].dh + (e.a_multi ? zdh : 0), b0);     // tall halo boxes always start one row above the tile
                        for (int t = 0; t < e.ntaps; ++t)
                            tma_load_2d(a_dst + p.a_stage_bytes + t * B_BYTES, &pm->b_map, full_bar(s), e.tap[t].b_col + b_lo, brow);
                    }
                    __syncwarp();
                    if (++s == stages) { s = 0; ph ^= 1u; }
                }
            }
        }
    } else {
        setmaxnreg_inc<GEMM_CONSUMER_REGS>();
        // ---------------------------------------------------- consumers: warpgroup g issues the wgmma of its share of the tile, then
        // every warp runs the epilogue of its 32-row quadrant q of that share, one 32-column chunk (item) at a time
        const int g = warp >> 2;
        const int q = warp & 3;
        const int ew = warp;                                                // 0..7
        const bool mma_wg = !SINGLE || g == 0;                              // (the warpgroups that hold items)
        const int own0 = (SINGLE || PP) ? 0 : g * OWN;                      // items [own0, own0 + OWN) are in this warpgroup's accumulator
        const int ch0 = PP ? 0 : own0 % NCH;                                // item own0 + ii = accumulator chunk ii = tile chunk ch0 + ii
        const int acc_half = (MH == 2 && !PP) ? g : 0;
        const int acc_c0 = (MH == 1 && !SINGLE && !PP) ? g * WN : 0;        // first accumulator column inside the tile
        const uint32_t out_smem = epi_base + ew * epi_warp_bytes;           // 4 KB
        const uint32_t res_smem = out_smem + 4096;                          // 2 x 4 KB (layers with a residual only)
        uint8_t* out_ptr = stage_ptr + stages * stage_bytes + ew * epi_warp_bytes;
        uint8_t* res_ptr = out_ptr + 4096;
        const bool use_out_tma = p.tma_epi && p.out_f32 != nullptr;
        uint32_t res_phase = 0;        // bit b = parity of res_bar(ew, b)
        uint32_t res_count = 0;        // residual chunks consumed so far
        uint32_t bias_slot = 0;        // alternating bias staging slot
        bool out_pending = false;      // a bulk store from the staging buffer may still be reading it
        int s = 0;                     // stage ring position
        uint32_t ph = 0;
        // GroupNorm partial sums of this lane's column in the warp's OWN chunks, kept across the tiles of one (image, column block).
        // (All items of a warp's share of a tile lie in one image: a warp's 32 rows never straddle images.  Ping-pong: the two halves of
        // a tile may be two images, so a run covers the NCH chunks of one half.)
        StatRun<NSTAT> st_own;
        for (int tile = tile_begin + (PP ? g : 0); tile < tile_end; tile += (PP ? 2 : 1)) {
            float acc[AH][2][WN / 2];
            int w0, h0, b0, n0, z;
            decode(tile, w0, h0, b0, n0, z);
            if constexpr (PP) {        // every tile of the range streams num_kt stages: this tile's first stage is number li * num_kt
                const long long pos = static_cast<long long>(tile - tile_begin) * num_kt;
                s = static_cast<int>(pos % stages);
                ph = static_cast<uint32_t>((pos / stages) & 1);
            }
            // geometry of a work item: rows of `half`, columns of `ch`
            auto item_geom = [&](int item, int qq, int& half, int& ch, int& sw, int& sh, int& c4) {
                half = item / NCH; ch = item % NCH;
                const int r0 = half * 128 + qq * 32;
                sw = r0 & (p.w_box - 1);
                sh = (r0 >> p.w_shift) & (p.h_box - 1);
                const int sb = r0 >> (p.w_shift + p.h_shift);
                c4 = p.epi_c4_is_z ? z : (b0 + sb);
            };
            auto request_resid = [&](int item) {                   // lane 0 only
                int half, ch, sw, sh, c4;
                item_geom(item, q, half, ch, sw, sh, c4);
                const uint32_t b = res_count & 1;
                mbar_arrive_expect_tx(res_bar(ew, b), 4096);
                tma_load_5d(res_smem + b * 4096, &pm->res_map, res_bar(ew, b), n0 + ch * 32, w0 + sw, 0, h0 + sh, c4);
            };
            // bias (+ per-image FiLM bias) of this lane's column of an item
            auto item_bias = [&](int item, int qq) {
                float bv = 0.f;
                const int half = item / NCH, ch = item % NCH;
                const int img = b0 + ((half * 128 + qq * 32) >> (p.w_shift + p.h_shift));
                const int n = n0 + ch * 32 + lane;
                if (n < p.n_valid) {
                    if (p.bias) bv += __ldg(&p.bias[n]);
                    if (p.bias2) bv += __ldcg(&p.bias2[static_cast<long long>(img < p.OB ? img : 0) * p.bias2_stride + n]);   // written by this step's FiLM kernel: L2 only
                }
                return bv;
            };
            // where a (half, chunk) unit's rows sit in a split-K partial tile: laid out [chunk][j][row] so that the 32 lanes (consecutive
            // rows) of one store / load instruction touch 512 contiguous bytes; WJ = float4 stride between the j-th and (j+1)-th quad of a row
            constexpr int WJ = MH * 128;
            auto ws_row = [&](int item, int qq) {
                return (static_cast<long long>(item % NCH) * 8 * WJ + (item / NCH) * 128 + qq * 32 + lane) * 4;
            };
            if (use_res_tma && mma_wg && lane == 0) request_resid(own0);     // overlaps the main loop
            // the bias of every item of this warp is fetched now (there is no L1, an L2 round trip per item would sit on the critical
            // path) and broadcast through smem when the item is processed
            float bvs[OWN] = {};
            if constexpr (BLOCK_N != 16) {
                if (mma_wg) {
#pragma unroll
                    for (int ii = 0; ii < OWN; ++ii) bvs[ii] = item_bias(own0 + ii, q);
                }
            }
            const int sp = tile % ksplit;
            if (mma_wg) {
                // ------------------------------------------------ main loop: this warpgroup's share of the tile
                const int k0 = (num_kt * sp) / ksplit, k1 = (num_kt * (sp + 1)) / ksplit;
                int zrow_off = 0;                                           // folded-upsample phase py: vertical taps one halo row further down
                if (p.z_phase) {
                    const int zz = (tile / ksplit) / (tiles_m * p.n_tiles);
                    zrow_off = (zz >> 1) * 1024;
                }
                const uint32_t a_base = stage_base + acc_half * p.a_half_off;
                const uint32_t b_base = stage_base + p.a_stage_bytes + acc_c0 * 128;
                const int li = tile - tile_begin;                           // (ping-pong) local tile index: li % 2 == g
                if (PP && li > 0) asm volatile("bar.sync %0, 256;" ::"r"(GEMM_ORDER_BAR + g) : "memory");   // our turn to issue MMAs
                int prev = -1;
                for (int k = k0; k < k1; ++k) {
                    mbar_wait(full_bar(s), ph);
                    const StageDesc& e = ktab_s[k % p.num_k];
                    // The MMAs of a stage are one branch-free chain with a compile-time tap count: a branch between two wgmma (a loop
                    // over a count read from shared memory) makes ptxas re-fence before every tap or serialise them.  The count is
                    // broadcast from lane 0 so that ptxas knows the switch below is warp-uniform.
                    const int ntaps = __shfl_sync(0xffffffffu, e.ntaps, 0);
                    auto issue = [&](auto nt_c) {
                        wgmma_fence();
#pragma unroll
                        for (int t = 0; t < decltype(nt_c)::value; ++t) {
                            const uint32_t a_addr = a_base + s * stage_bytes + e.tap[t].a_off + (e.a_multi ? 0 : zrow_off);
                            const uint32_t b_addr = b_base + s * stage_bytes + t * B_BYTES;
#pragma unroll
                            for (int kk = 0; kk < 4; ++kk) {   // 4 x K(16) = 64 channels; +32 B inside the 128 B swizzle row
                                const uint64_t bdesc = wgmma_desc_sw128(b_addr + kk * 32, 16, 1024);
#pragma unroll
                                for (int hh = 0; hh < AH; ++hh)    // (ping-pong, MH = 2: both 128-row halves share the B slab)
#pragma unroll
                                    for (int i = 0; i < 2; ++i)    // row groups 2 g' + i, g' = 0..7
                                        Wgmma<WN>::template mma<0, 0>(acc[hh][i],
                                                                      wgmma_desc_sw128(a_addr + hh * p.a_half_off + i * 1024 + kk * 32, 16, 2048),
                                                                      bdesc, ((k - k0) | t | kk) != 0);
                            }
                        }
                        wgmma_commit();
                    };
                    if (ntaps == 3) issue(std::integral_constant<int, 3>{});
                    else if (ntaps == 2) issue(std::integral_constant<int, 2>{});
                    else issue(std::integral_constant<int, 1>{});
                    if (stages == 1) {                                      // nothing can be loaded ahead: free the only stage now
                        wgmma_wait<0>();
                        mbar_arrive_if(empty_bar(s), (threadIdx.x & 127) == 0);
                    } else {
                        if (prev >= 0) {                                    // the stage before this one has been read
                            wgmma_wait<1>();
                            mbar_arrive_if(empty_bar(prev), (threadIdx.x & 127) == 0);
                        }
                        prev = s;
                    }
                    if (++s == stages) { s = 0; ph ^= 1u; }
                }
                // every MMA of the tile is issued: the other warpgroup may issue those of the next tile (if the CTA has one)
                if (PP && tile + 1 < tile_end) asm volatile("bar.arrive %0, 256;" ::"r"(GEMM_ORDER_BAR + (g ^ 1)) : "memory");
                wgmma_wait<0>();
#pragma unroll
                for (int hh = 0; hh < AH; ++hh) {
                    wgmma_fence_regs(acc[hh][0]);
                    wgmma_fence_regs(acc[hh][1]);
                }
                if (prev >= 0) mbar_arrive_if(empty_bar(prev), (threadIdx.x & 127) == 0);
            }
            // pass 0 reads the accumulator.  With split-K it only stores this CTA's partial tile into its slice of `ws`;
            // once all `ksplit` CTAs of the output tile have arrived at the tile's counter, pass 1 runs in EVERY one of them on a
            // 1/ksplit share of the tile's 32x32 units: sum the partials (fixed order: deterministic) and do the real epilogue.
            // (All CTAs of the grid are resident -- at most one (tile, split) pair per SM -- so the spin wait cannot deadlock.)
            const int npass = (!PP && ksplit > 1) ? 2 : 1;                 // (the host never splits a ping-pong launch)
            constexpr long long SLICE = static_cast<long long>(MH) * 128 * BLOCK_N;       // floats per partial tile
#pragma unroll 1
            for (int pass = 0; pass < npass; ++pass) {
            if (pass == 1) {
                __threadfence();
                asm volatile("bar.sync 1, 256;" ::: "memory");
                if (ew == 0 && lane == 0) {
                    unsigned int* ctr = p.counters + tile / ksplit;
                    const unsigned int old = atomicAdd(ctr, 1u);
                    const unsigned int target = (old / ksplit + 1u) * ksplit;              // the counter only ever grows
                    spin_wait_reached(ctr, target);
                    __threadfence();
                }
                __syncwarp();
                asm volatile("bar.sync 1, 256;" ::: "memory");
            }
            const bool to_ws = (!PP && ksplit > 1 && pass == 0);
            // the epilogue of one item (half, chunk) in quadrant qq: `fetch(v)` brings this lane's row of the item's 32x32 chunk (lane = row,
            // v[j] = column j), which is then finished in place; `add_stats(cs, cq)` takes the GroupNorm sums of this lane's column
            auto epi_item = [&](const int item, const int qq, const float bv, const bool last, auto&& fetch, auto&& add_stats) {
                int half, ch, sw, sh, c4;
                item_geom(item, qq, half, ch, sw, sh, c4);
                const int row = half * 128 + qq * 32 + lane;
                const int w = row & (p.w_box - 1);
                const int h = (row >> p.w_shift) & (p.h_box - 1);
                const int bb = row >> (p.w_shift + p.h_shift);
                const int ow = w0 + w, oh = h0 + h, img = b0 + bb;
                const bool row_ok = (ow < p.OW) && (oh < p.OH) && (img < p.OB);
                float v[32];
                if constexpr (BLOCK_N == 16) {
                    fetch(v);
                    if (row_ok) {
                        float eps[4] = {0.f, 0.f, 0.f, 0.f};
                        for (int c = 0; c < p.post.C; ++c) eps[c] = v[c] + __ldg(&p.bias[c]);
                        final_epilogue(p, eps, img, oh, ow);
                    }
                } else {
                    const int nb = n0 + ch * 32;
                    float* bs = bias_s + (ew * 2 + (bias_slot++ & 1u)) * 32;
                    bs[lane] = bv;
                    __syncwarp();
                    if (use_res_tma) {
                        ++res_count;                             // this item is residual request number res_count
                        if (!last && lane == 0) request_resid(item + 1);   // other buffer: freed one item ago
                    }
                    fetch(v);
                    const float ep_scale = p.scale;
                    const bool full = (nb + 32 <= p.n_valid);
#pragma unroll
                    for (int j4 = 0; j4 < 8; ++j4) {               // bias broadcast: 8 x LDS.128 (the slot is 128 B aligned)
                        const float4 bq = reinterpret_cast<const float4*>(bs)[j4];
                        const float bb4[4] = {bq.x, bq.y, bq.z, bq.w};
#pragma unroll
                        for (int jj = 0; jj < 4; ++jj) {
                            const int j = 4 * j4 + jj;
                            float x = v[j] * ep_scale + bb4[jj];
                            if (!full && nb + j >= p.n_valid) x = 0.f;
                            v[j] = x;
                        }
                    }
                    if (use_res_tma) {
                        const uint32_t b = (res_count - 1) & 1;
                        mbar_wait(res_bar(ew, b), (res_phase >> b) & 1u);
                        res_phase ^= (1u << b);
                        const uint8_t* rp = res_ptr + b * 4096 + lane * 128;
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const float4 r = *reinterpret_cast<const float4*>(rp + ((j ^ (lane & 7)) << 4));
                            v[4 * j] += r.x; v[4 * j + 1] += r.y; v[4 * j + 2] += r.z; v[4 * j + 3] += r.w;
                        }
                        __syncwarp();                            // everyone is done with the buffer before it is re-requested
                    } else if (row_ok && p.resid) {
                        const long long ro = out_index(p.rs, z, img, oh, ow);
                        for (int j = 0; j < 32; ++j)
                            if (nb + j < p.n_valid) v[j] += __ldcg(&p.resid[ro + nb + j]);
                    }
                    if (use_out_tma) {
                        if (out_pending) {                       // the previous bulk store must have finished reading the staging buffer
                            if (lane == 0) tma_store_wait_read<0>();
                            __syncwarp();
                        }
                        uint8_t* op = out_ptr + lane * 128;
#pragma unroll
                        for (int j = 0; j < 8; ++j)
                            *reinterpret_cast<float4*>(op + ((j ^ (lane & 7)) << 4)) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                        fence_proxy_async_smem();
                        __syncwarp();
                        if (lane == 0) {
                            if (p.z_phase) tma_store_5d(&pm->out_map, out_smem, (z & 1) * p.n_valid + nb, w0 + sw, z >> 1, h0 + sh, c4);
                            else tma_store_5d(&pm->out_map, out_smem, nb, w0 + sw, 0, h0 + sh, c4);
                            tma_store_commit();
                        }
                        out_pending = true;
                    } else if (row_ok && p.out_f32) {
                        const long long oo = out_index(p.os, z, img, oh, ow) + (p.z_phase ? (z >> 1) * p.z_off_hi + (z & 1) * p.z_off_lo : 0);
                        if (full) {
                            float4* o4 = reinterpret_cast<float4*>(p.out_f32 + oo + nb);
#pragma unroll
                            for (int j = 0; j < 8; ++j) o4[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                        } else {
                            for (int j = 0; j < 32; ++j)
                                if (nb + j < p.n_valid) p.out_f32[oo + nb + j] = v[j];
                        }
                    }
                    if (p.out_t && nb >= p.t_col0) {
                        if (ow < p.OW && oh < p.OH && nb + 32 <= p.n_valid) {          // padded images too: their (finite) values are multiplied by P = 0 later
                            __nv_bfloat16* tp = p.out_t + (static_cast<long long>(img / p.t_per) * p.t_rows + (nb - p.t_col0)) * p.t_ld +
                                                (img % p.t_per) * (p.OH * p.OW) + oh * p.OW + ow;
#pragma unroll
                            for (int j = 0; j < 32; ++j) {                                                              // lanes = consecutive tokens
                                const __nv_bfloat16 hi = __float2bfloat16_rn(v[j]);
                                tp[static_cast<long long>(j) * p.t_ld] = hi;
                                if (p.lo_t_off) tp[static_cast<long long>(j) * p.t_ld + p.lo_t_off] = __float2bfloat16_rn(v[j] - __bfloat162float(hi));
                            }
                        }
                    } else if (row_ok && p.out_bf16) {
                        const long long ho = out_index(p.hs, z, img, oh, ow);
                        if (full) {
                            uint4* o4 = reinterpret_cast<uint4*>(p.out_bf16 + ho + nb);
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                __nv_bfloat162 h0v = __floats2bfloat162_rn(v[8 * j], v[8 * j + 1]);
                                __nv_bfloat162 h1v = __floats2bfloat162_rn(v[8 * j + 2], v[8 * j + 3]);
                                __nv_bfloat162 h2v = __floats2bfloat162_rn(v[8 * j + 4], v[8 * j + 5]);
                                __nv_bfloat162 h3v = __floats2bfloat162_rn(v[8 * j + 6], v[8 * j + 7]);
                                uint4 uu;
                                uu.x = *reinterpret_cast<uint32_t*>(&h0v); uu.y = *reinterpret_cast<uint32_t*>(&h1v);
                                uu.z = *reinterpret_cast<uint32_t*>(&h2v); uu.w = *reinterpret_cast<uint32_t*>(&h3v);
                                o4[j] = uu;
                            }
                        } else {
                            for (int j = 0; j < 32; ++j)
                                if (nb + j < p.n_valid) p.out_bf16[ho + nb + j] = __float2bfloat16_rn(v[j]);
                        }
                        if (p.lo_out_off) {                       // precise mode: low halves
                            __nv_bfloat16* lp = p.out_bf16 + ho + nb + p.lo_out_off;
                            if (full) {
                                uint4* o4 = reinterpret_cast<uint4*>(lp);
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                    float r[8];
#pragma unroll
                                    for (int u = 0; u < 8; ++u) r[u] = v[8 * j + u] - __bfloat162float(__float2bfloat16_rn(v[8 * j + u]));
                                    __nv_bfloat162 h0v = __floats2bfloat162_rn(r[0], r[1]), h1v = __floats2bfloat162_rn(r[2], r[3]);
                                    __nv_bfloat162 h2v = __floats2bfloat162_rn(r[4], r[5]), h3v = __floats2bfloat162_rn(r[6], r[7]);
                                    uint4 uu;
                                    uu.x = *reinterpret_cast<uint32_t*>(&h0v); uu.y = *reinterpret_cast<uint32_t*>(&h1v);
                                    uu.z = *reinterpret_cast<uint32_t*>(&h2v); uu.w = *reinterpret_cast<uint32_t*>(&h3v);
                                    o4[j] = uu;
                                }
                            } else {
                                for (int j = 0; j < 32; ++j)
                                    if (nb + j < p.n_valid) lp[j] = __float2bfloat16_rn(v[j] - __bfloat162float(__float2bfloat16_rn(v[j])));
                            }
                        }
                    }
                    if (p.stats) {
                        double cs, cq;
                        if (use_out_tma) {
                            // the 32x32 tile sits in the (swizzled) staging buffer: lane c walks down column c -- conflict free, and a
                            // third of the instructions of the shuffle transposition below
                            const unsigned int okm = __ballot_sync(0xffffffffu, row_ok);
                            const uint8_t* colp = out_ptr + ((lane & 3) << 2);
                            const int cq4 = lane >> 2;
                            // shifted sums: the fp32 partial sums run over x - x[row 0] (values of the size of the spread, not of the
                            // mean), the shift is put back in fp64:  sum x = a + n s,  sum x^2 = q + 2 s a + n s^2
                            const float sft = *reinterpret_cast<const float*>(colp + (cq4 << 4));
                            float a0 = 0.f, a1 = 0.f, q0 = 0.f, q1 = 0.f;
                            if (okm == 0xffffffffu) {            // (warp-uniform) the usual case: no padded pixel / image in this chunk
#pragma unroll
                                for (int r = 0; r < 32; r += 2) {
                                    const float x0 = *reinterpret_cast<const float*>(colp + r * 128 + ((cq4 ^ (r & 7)) << 4)) - sft;
                                    const float x1 = *reinterpret_cast<const float*>(colp + (r + 1) * 128 + ((cq4 ^ ((r + 1) & 7)) << 4)) - sft;
                                    a0 += x0; q0 = fmaf(x0, x0, q0);
                                    a1 += x1; q1 = fmaf(x1, x1, q1);
                                }
                            } else {
#pragma unroll
                                for (int r = 0; r < 32; r += 2) {
                                    float x0 = *reinterpret_cast<const float*>(colp + r * 128 + ((cq4 ^ (r & 7)) << 4)) - sft;
                                    float x1 = *reinterpret_cast<const float*>(colp + (r + 1) * 128 + ((cq4 ^ ((r + 1) & 7)) << 4)) - sft;
                                    if (!((okm >> r) & 1u)) x0 = 0.f;
                                    if (!((okm >> (r + 1)) & 1u)) x1 = 0.f;
                                    a0 += x0; q0 = fmaf(x0, x0, q0);
                                    a1 += x1; q1 = fmaf(x1, x1, q1);
                                }
                            }
                            const double n_ok = static_cast<double>(__popc(okm)), ds = static_cast<double>(sft);
                            const double da = static_cast<double>(a0 + a1), dq = static_cast<double>(q0 + q1);
                            cs = da + n_ok * ds;
                            cq = dq + 2.0 * ds * da + n_ok * ds * ds;
                        } else {
                            float s2[32];
#pragma unroll
                            for (int j = 0; j < 32; ++j) {
                                const float x = row_ok ? v[j] : 0.f;
                                v[j] = x; s2[j] = x * x;
                            }
                            cs = static_cast<double>(warp_column_sums(v));
                            cq = static_cast<double>(warp_column_sums(s2));
                        }
                        add_stats(cs, cq);
                    }
                }
            };
            if (pass == 0) {
                if (mma_wg) {
                    if (!PP && p.stats && !to_ws) st_own.start(p, b0 + ((acc_half * 128 + q * 32) >> (p.w_shift + p.h_shift)), n0, ch0, lane);
                    static_for<OWN>([&](auto ii_c) {             // compile-time ii: accumulator chunk ii is dead once it has been staged
                        constexpr int ii = decltype(ii_c)::value;
                        constexpr int AHI = PP ? ii / NCH : 0, ACL = PP ? ii % NCH : ii;   // accumulator half and chunk of item ii
                        if constexpr (PP) {                      // a new half may be a new image: its own GroupNorm run
                            if (ACL == 0 && p.stats) st_own.start(p, b0 + ((AHI * 128 + q * 32) >> (p.w_shift + p.h_shift)), n0, 0, lane);
                        }
                        auto stage_acc = [&](float (&v)[32]) {
                            if (out_pending) {                   // the staging buffer is about to be overwritten by the transposition
                                if (lane == 0) tma_store_wait_read<0>();
                                __syncwarp();
                            }
                            acc_chunk_rows<WN, CW, ACL>(acc[AHI], reinterpret_cast<float*>(out_ptr), v);
                        };
                        if (to_ws) {                             // split-K: park the partial sums
                            float v[32];
                            stage_acc(v);
                            float4* dst = reinterpret_cast<float4*>(p.ws + static_cast<long long>(tile) * SLICE + ws_row(own0 + ii, q));
#pragma unroll
                            for (int j = 0; j < 8; ++j) __stcg(dst + j * WJ, make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]));
                        } else {
                            epi_item(own0 + ii, q, bvs[ii], ii + 1 == OWN, stage_acc, [&](double cs, double cq) { st_own.add(PP ? ACL : ii, cs, cq); });
                        }
                    });
                }
            } else {
                // units u = item * 4 + quadrant with u % ksplit == sp, dealt round-robin to the eight warps.  A split-K CTA owns exactly one
                // (tile, split) pair, so the statistics run of its units ends with the tile.
                StatRun<NCH> st_ws;
#pragma unroll 1
                for (int it = sp + ksplit * ew; it < NITEMS * 4; it += ksplit * GEMM_EPI_WARPS) {
                    const int item = it >> 2, qq = it & 3;
                    if (p.stats) st_ws.start(p, b0 + (((item / NCH) * 128 + qq * 32) >> (p.w_shift + p.h_shift)), n0, 0, lane);
                    epi_item(item, qq, BLOCK_N != 16 ? item_bias(item, qq) : 0.f, true,
                             [&](float (&v)[32]) {               // sum the ksplit partial tiles (L2 resident), split 0 first
                                 const float* src0 = p.ws + static_cast<long long>(tile - sp) * SLICE + ws_row(item, qq);
#pragma unroll
                                 for (int j = 0; j < 32; ++j) v[j] = 0.f;
                                 for (int s2 = 0; s2 < ksplit; ++s2) {
                                     const float4* src = reinterpret_cast<const float4*>(src0 + s2 * SLICE);
#pragma unroll
                                     for (int j = 0; j < 8; ++j) {
                                         const float4 r = __ldcg(src + j * WJ);
                                         v[4 * j] += r.x; v[4 * j + 1] += r.y; v[4 * j + 2] += r.z; v[4 * j + 3] += r.w;
                                     }
                                 }
                             },
                             [&](double cs, double cq) { st_ws.add(item % NCH, cs, cq); });
                }
                if (p.stats) st_ws.flush(p, 0, lane);
            }
            }       // pass
        }           // tiles
        if (p.stats) st_own.flush(p, ch0, lane);
        if (use_out_tma && out_pending && lane == 0) tma_store_wait_read<0>();     // smem must outlive the reads of the last bulk stores
    }
}

template <int BLOCK_N, int MH, bool PP = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tile_kernel(const __grid_constant__ GemmParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    gemm_tile_body<BLOCK_N, MH, PP>(p, &p, base, smem_raw + (base - raw), blockIdx.x, gridDim.x);
}

}  // namespace sr3
