// step_megakernel.cuh -- one reverse-diffusion step (UNet forward + posterior update) as ONE persistent cooperative launch.
//
// The per-layer kernels of a step (reference: one p_sample call, model/sr3_modules/diffusion.py:151-174, i.e. UNet.forward of
// unet.py:235-259 + the posterior arithmetic) used to be ~158 dependent launches whose fixed cost (launch gap, prologue, first TMA
// round trip, drain: 8-17 us each) was a quarter of the step at batch 16 and nearly all of it for a 2-image shard.  Here one CTA per
// SM stays resident for the whole step and walks a host-built op list; the only grid-wide dependencies (an op reads what ALL CTAs of
// the previous op wrote: activations through TMA, GroupNorm sums) are grid barriers (~1 us) instead of kernel boundaries:
//
//     for op in ops:  [grid barrier]  ->  gemm tile loop | GroupNorm apply | fused attention | row softmax | embedding + FiLM | ...
//
// mbarriers live in a fixed shared-memory header and are recycled per op, parameter blocks (incl. TMA descriptors) live in global
// memory and are copied into the header by every CTA.
#pragma once
#include "aux_kernels.cuh"
#include "attn_wgmma.cuh"

namespace sr3 {

enum MegaOpType : int { MOP_GEMM = 0, MOP_PREP = 1, MOP_ATTN = 2, MOP_SOFTMAX = 3, MOP_EMBED_FILM = 4, MOP_ZERO = 5 };

struct MegaOp {
    int type;
    int variant;        // gemm: BLOCK_N | (MH << 16) | (ping-pong << 24)
    int sync_before;    // 1: grid barrier before this op (it reads what other CTAs wrote in earlier ops)
    int param_bytes;
    long long param_off;    // byte offset of the parameter block inside the blob (128-byte aligned)
    long long pad;
};

struct SoftmaxParams { const float* S; __nv_bfloat16* P; long long rows; int L, seg, precise; };
struct ZeroParams { float4* ptr; long long n4; };
struct EmbedFilmParams {
    EmbedParams e;                          // ctl, nl_table, nl_buf, MLP weights, tau (unused here), inner
    const float* wf; const float* bf; const float* cbias;   // FiLM projections [F][inner], [F], block1 conv bias [F]
    float* film;                            // [B][F]
    int F, B;
};

struct MegaParams {
    const MegaOp* ops;
    int n_ops;
    const uint8_t* blob;
    unsigned long long* bar;                // grid-barrier counter (monotonic)
    unsigned long long* prof;               // [n_ops + 1][4] globaltimer stamps of CTA 0 (nullptr: off): op start (previous op done),
                                            // barrier arrived + set-up done, barrier passed, body done
    StepCtl* ctl;
};

// ---------------------------------------------------------------------------------------------------------------- grid barrier
struct GridBarrier {
    unsigned long long* ctr;
    unsigned long long target;              // thread 0 only
    unsigned int n;
    __device__ __forceinline__ void init(unsigned long long* c, unsigned int ncta) {
        ctr = c; n = ncta; target = 0;
        if (threadIdx.x == 0) {
            // every launch starts with the counter at a multiple of n; nobody passes barrier 1 before all CTAs have read it
            const unsigned long long v = ld_acquire_gpu_u64(c);
            target = v - (v % ncta);
        }
    }
    // Split barrier.  arrive(): all threads of the CTA; everything this CTA wrote before is published.  wait(): returns once every CTA has
    // arrived; what they published is visible to all threads of this CTA afterwards.  CTA-local set-up of the next op goes in between.
    __device__ __forceinline__ void arrive() {
        __syncthreads();
        if (threadIdx.x == 0) {
            target += n;
            __threadfence();
            red_release_gpu_add_u64(ctr, 1ull);
        }
    }
    __device__ __forceinline__ void wait(int tag) {
        if (threadIdx.x == 0) {
            uint64_t t0 = 0;
            for (uint32_t spins = 0;; ++spins) {
                if (ld_acquire_gpu_u64(ctr) >= target) break;
                if ((spins & 4095u) == 4095u) {
                    const uint64_t now = globaltimer_ns();
                    if (t0 == 0) t0 = now;
                    if (now - t0 > 4000000000ull) {
                        printf("sr3: grid barrier timeout cta=%d op=%d counter=%llu target=%llu\n", blockIdx.x, tag, ld_acquire_gpu_u64(ctr), target);
                        __trap();
                    }
                }
            }
            __threadfence();
        }
        __syncthreads();
        fence_proxy_async_all();            // what other CTAs wrote with st.global is about to be read through TMA
    }
};

// ---------------------------------------------------------------------------------------------------------------- GroupNorm apply
// Same arithmetic as prep_kernel (aux_kernels.cuh) for the 288-thread CTAs of the step kernel: a CTA owns a contiguous range of
// (image, pixel block) items; scale / shift are rebuilt when the image changes.  Loads are L2-coherent (.cg): the data was produced
// earlier in the same launch.
__device__ __noinline__ void prep_body(const PrepParams& p, float* sm, const int cta, const int ncta) {
    const int C = p.C0 + p.C1;
    float* sc = sm;
    float* sh = sm + C;
    float* gm = sm + 2 * C;
    float* gr = gm + p.groups;
    const int nth = static_cast<int>(blockDim.x);
    const int vpp = C >> 2;                                  // 4-channel vectors per pixel
    const bool wide = vpp > nth;                             // more vectors than threads: a thread walks several (table stays in smem)
    const int kpix = wide ? 1 : nth / vpp;
    const bool active = wide || static_cast<int>(threadIdx.x) < vpp * kpix;
    const int c = wide ? 0 : (threadIdx.x % vpp) << 2;
    const int lp = wide ? 0 : threadIdx.x / vpp;
    // this CTA's share: a contiguous range of the B x HW pixels (whole multiples of the kpix pixels a pass of the block covers)
    const long long total = static_cast<long long>(p.B) * p.HW;
    const long long units = (total + kpix - 1) / kpix;
    const long long g0 = (units * cta / ncta) * kpix;
    long long g1 = (units * (cta + 1) / ncta) * kpix;
    if (g1 > total) g1 = total;
    const bool from0 = c < p.C0;
    const float* src = from0 ? p.src0 + c : p.src1 + (c - p.C0);
    const int cs = from0 ? p.C0 : p.C1;
    float k4[4] = {0.f, 0.f, 0.f, 0.f}, s4[4] = {0.f, 0.f, 0.f, 0.f};
    constexpr int U = 6;
    const int orow = p.precise ? 2 * C : C;
    const long long lo_off = p.precise ? C : 0;
    for (long long g = g0; g < g1;) {
        const int b = static_cast<int>(g / p.HW);
        const long long img = static_cast<long long>(b) * p.HW;
        const int pix0 = static_cast<int>(g - img);
        const int pix1 = static_cast<int>((g1 - img) < p.HW ? (g1 - img) : p.HW);
        g = img + pix1;
        __syncthreads();                             // everyone is done with the previous image's table
        groupnorm_scale_shift(p, b, sc, sh, gm, gr);
        if (!active) continue;
        if (wide) {
            for (int pix = pix0; pix < pix1; ++pix) {
                for (int v = threadIdx.x; v < vpp; v += nth) {
                    const int cc = v << 2;
                    const float4 x = (cc < p.C0) ? __ldcg(reinterpret_cast<const float4*>(p.src0 + (img + pix) * p.C0 + cc))
                                                 : __ldcg(reinterpret_cast<const float4*>(p.src1 + (img + pix) * p.C1 + (cc - p.C0)));
                    const float4 kk = *reinterpret_cast<const float4*>(sc + cc), ss = *reinterpret_cast<const float4*>(sh + cc);
                    float y0 = x.x * kk.x + ss.x, y1 = x.y * kk.y + ss.y, y2 = x.z * kk.z + ss.z, y3 = x.w * kk.w + ss.w;
                    if (p.silu) { y0 = silu_f(y0); y1 = silu_f(y1); y2 = silu_f(y2); y3 = silu_f(y3); }
                    const long long o = (img + pix) * orow + cc;
                    store_operand4(p.out_a, o, lo_off, y0, y1, y2, y3);
                    if (p.out_raw) store_operand4(p.out_raw, o, lo_off, x.x, x.y, x.z, x.w);
                }
            }
            continue;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) { k4[j] = sc[c + j]; s4[j] = sh[c + j]; }
        // software pipeline: the loads of batch i+1 are in flight while batch i is normalised and stored (2 x U x 16 B per thread)
        float4 cur[U], nxt[U];
        int pix = pix0 + lp;
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int pp = pix + u * kpix;
            if (pp < pix1) cur[u] = __ldcg(reinterpret_cast<const float4*>(src + (img + pp) * cs));
        }
        while (pix < pix1) {
            const int npix = pix + kpix * U;
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int pp = npix + u * kpix;
                if (pp < pix1) nxt[u] = __ldcg(reinterpret_cast<const float4*>(src + (img + pp) * cs));
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int pp = pix + u * kpix;
                if (pp < pix1) {
                    float y0 = cur[u].x * k4[0] + s4[0], y1 = cur[u].y * k4[1] + s4[1], y2 = cur[u].z * k4[2] + s4[2], y3 = cur[u].w * k4[3] + s4[3];
                    if (p.silu) { y0 = silu_f(y0); y1 = silu_f(y1); y2 = silu_f(y2); y3 = silu_f(y3); }
                    const long long o = (img + pp) * orow + c;
                    store_operand4(p.out_a, o, lo_off, y0, y1, y2, y3);
                    if (p.out_raw) store_operand4(p.out_raw, o, lo_off, cur[u].x, cur[u].y, cur[u].z, cur[u].w);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) cur[u] = nxt[u];
            pix = npix;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------- row softmax
__device__ __noinline__ void softmax_body(const SoftmaxParams& p, const int cta, const int ncta) {
    const int nwarp = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (long long row = static_cast<long long>(cta) * nwarp + warp; row < p.rows; row += static_cast<long long>(ncta) * nwarp) {
        const int r_in = static_cast<int>(row % p.L);
        const int k0 = (r_in / p.seg) * p.seg;
        const float* s = p.S + row * p.L;
        __nv_bfloat16* pr = p.P + row * (p.precise ? 2 * p.L : p.L);
        float m = -INFINITY;
        for (int k = k0 + lane; k < k0 + p.seg; k += 32) m = fmaxf(m, __ldcg(&s[k]));
#pragma unroll
        for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        float sum = 0.f;
        for (int k = k0 + lane; k < k0 + p.seg; k += 32) sum += expf(__ldcg(&s[k]) - m);
#pragma unroll
        for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        const float inv = 1.0f / sum;
        for (int k = lane; k < p.L; k += 32) {
            const float v = (k >= k0 && k < k0 + p.seg) ? expf(__ldcg(&s[k]) - m) * inv : 0.f;
            pr[k] = __float2bfloat16_rn(v);
            if (p.precise) pr[p.L + k] = __float2bfloat16_rn(bf16_residual(v));
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------- embedding + FiLM
// PositionalEncoding + noise_level_mlp (unet.py:18-31,177-184) and this CTA's share of the FeatureWiseAffine projections
// (unet.py:34-50, bias-only form, block1's conv bias folded in).  Every CTA recomputes tau (32 K MACs per distinct noise level: cheaper
// than a grid barrier); during sampling all images share the step's noise level, so tau is computed once.
// Shared memory it uses on ncta CTAs: pe, h, tau of every image and the CTA's share of the FiLM weight rows (padded rows).
__host__ __device__ constexpr long long embed_film_smem_bytes(int B, int inner, int F, int ncta) {
    return 4ll * (5ll * inner + static_cast<long long>(B) * inner + static_cast<long long>((F + ncta - 1) / ncta) * (inner + 1));
}
__device__ __noinline__ void embed_film_body(const EmbedFilmParams& p, float* sm, const int t_step, const int cta, const int ncta) {
    const int inner = p.e.inner, hid = 4 * inner, B = p.B;
    const int from_table = p.e.ctl->nl_from_table;
    const int n_tau = from_table ? 1 : B;
    float* pe = sm;                         // [inner]
    float* h = pe + inner;                  // [hid]
    float* tau = h + hid;                   // [n_tau][inner]
    float* wrow = tau + B * inner;          // [rows_here][inner + 1]
    const int tid = threadIdx.x, nth = blockDim.x;
    const int warp = tid >> 5, lane = tid & 31, nwarp = nth >> 5;
    const int r0 = static_cast<int>(static_cast<long long>(p.F) * cta / ncta), r1 = static_cast<int>(static_cast<long long>(p.F) * (cta + 1) / ncta);
    const int rows = r1 - r0;
    for (int i = tid; i < rows * inner; i += nth) {           // coalesced staging of this CTA's FiLM weight rows
        const int r = i / inner, cc = i % inner;
        wrow[r * (inner + 1) + cc] = __ldg(&p.wf[static_cast<long long>(r0 + r) * inner + cc]);
    }
    const int count = inner / 2;
    for (int ti = 0; ti < n_tau; ++ti) {
        const float nl = from_table ? p.e.nl_table[t_step + 1] : p.e.nl_buf[ti];
        __syncthreads();
        for (int j = tid; j < inner; j += nth) {
            const int jj = j < count ? j : j - count;
            const float step = static_cast<float>(jj) / static_cast<float>(count);
            const float e = nl * expf(-9.210340371976184f * step);
            pe[j] = j < count ? sinf(e) : cosf(e);
        }
        __syncthreads();
        for (int j = warp; j < hid; j += nwarp) {             // one warp per output row: coalesced weights + shuffle reduction
            float a = 0.f;
            for (int i = lane; i < inner; i += 32) a += __ldg(&p.e.w1[j * inner + i]) * pe[i];
#pragma unroll
            for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
            if (lane == 0) { const float t = a + __ldg(&p.e.b1[j]); h[j] = t / (1.0f + expf(-t)); }
        }
        __syncthreads();
        for (int j = warp; j < inner; j += nwarp) {
            float a = 0.f;
            for (int i = lane; i < hid; i += 32) a += __ldg(&p.e.w2[j * hid + i]) * h[i];
#pragma unroll
            for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
            if (lane == 0) tau[ti * inner + j] = a + __ldg(&p.e.b2[j]);
        }
    }
    __syncthreads();
    for (int idx = tid; idx < rows * B; idx += nth) {
        const int r = idx % rows, b = idx / rows;
        const int j = r0 + r;
        const float* w = wrow + r * (inner + 1);
        const float* t = tau + (from_table ? 0 : b) * inner;
        float a = __ldg(&p.bf[j]) + __ldg(&p.cbias[j]);
        for (int i = 0; i < inner; ++i) a += w[i] * t[i];
        p.film[static_cast<long long>(b) * p.F + j] = a;
    }
}

// ---------------------------------------------------------------------------------------------------------------- the step kernel
// (not inlined: every tile variant / op body gets its own register allocation instead of sharing the step kernel's)
constexpr int MEGA_VARIANT_PP = 1 << 24;
template <int BN, int MH, bool PP = false>
__device__ __noinline__ void mega_gemm(const uint8_t* hdr_params, const uint8_t* gparams, uint32_t base, uint8_t* base_ptr, int cta, int ncta) {
    gemm_tile_body<BN, MH, true, PP>(*reinterpret_cast<const GemmParams*>(hdr_params), reinterpret_cast<const GemmParams*>(gparams), base, base_ptr,
                                 cta, ncta);
}

__device__ __noinline__ void mega_attn(const AttnParams& ap, const AttnParams* gp, uint32_t base, uint8_t* base_ptr, int qt, int dc, int z) {
    attn_unit<true>(ap, gp, base, base_ptr, qt, dc, z);
}

__global__ void __launch_bounds__(GEMM_THREADS, 1) step_kernel(const __grid_constant__ MegaParams mp) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* base_ptr = smem_raw + (base - raw);
    uint8_t* hdr_params = base_ptr + HDR_PARAMS;
    uint8_t* op_smem = base_ptr + GEMM_HDR_BYTES;
    volatile int* t_slot = reinterpret_cast<volatile int*>(base_ptr + HDR_SCALARS + 8);
    const int cta = blockIdx.x, ncta = gridDim.x;

    if (threadIdx.x == 0) {
        for (int i = 0; i < HDR_NUM_BARS; ++i) mbar_init(base + 8u * i, 1);      // valid objects: every op starts by invalidating them
        fence_mbar_init();
        *t_slot = mp.ctl->t_next;                                                // this step's timestep (CTA 0 advances it at the very end)
    }
    GridBarrier gb;
    gb.init(mp.bar, ncta);
    __syncthreads();
    const int t_step = *t_slot;

    for (int i = 0; i < mp.n_ops; ++i) {
        const MegaOp op = mp.ops[i];
        const uint8_t* gparams = mp.blob + op.param_off;
        const bool stamp = mp.prof && cta == 0 && threadIdx.x == 0;
        if (stamp) mp.prof[4 * i] = globaltimer_ns();
        if (op.sync_before) gb.arrive();         // (starts with a __syncthreads: the previous op is finished in this CTA)
        // CTA-local set-up, overlapped with the other CTAs still arriving: parameter block -> shared-memory header, and for a tile op its
        // stage table / descriptor prefetch / mbarrier recycling
        for (int w = threadIdx.x; w < (op.param_bytes >> 2); w += blockDim.x)
            reinterpret_cast<uint32_t*>(hdr_params)[w] = __ldg(reinterpret_cast<const uint32_t*>(gparams) + w);
        __syncthreads();
        if (op.type == MOP_GEMM) {
            if (threadIdx.x == 0) reinterpret_cast<GemmParams*>(hdr_params)->t_fixed = t_step;
            gemm_stage_setup(*reinterpret_cast<const GemmParams*>(hdr_params), reinterpret_cast<const GemmParams*>(gparams), base, base_ptr,
                             op.variant & 0xffff, (op.variant >> 16) & 0xff, (op.variant & MEGA_VARIANT_PP) != 0, true);
        }
        if (stamp) mp.prof[4 * i + 1] = globaltimer_ns();
        if (op.sync_before) gb.wait(i); else __syncthreads();
        if (stamp) mp.prof[4 * i + 2] = globaltimer_ns();
        switch (op.type) {
            case MOP_GEMM: {
                switch (op.variant) {
                    case 16 | (1 << 16): mega_gemm<16, 1>(hdr_params, gparams, base, base_ptr, cta, ncta); break;
                    case 16 | (2 << 16): mega_gemm<16, 2>(hdr_params, gparams, base, base_ptr, cta, ncta); break;
                    case 32 | (1 << 16): mega_gemm<32, 1>(hdr_params, gparams, base, base_ptr, cta, ncta); break;
                    case 64 | (1 << 16): mega_gemm<64, 1>(hdr_params, gparams, base, base_ptr, cta, ncta); break;
                    case 64 | (2 << 16): mega_gemm<64, 2>(hdr_params, gparams, base, base_ptr, cta, ncta); break;
                    case 128 | (1 << 16): mega_gemm<128, 1>(hdr_params, gparams, base, base_ptr, cta, ncta); break;
                    case 128 | (2 << 16): mega_gemm<128, 2>(hdr_params, gparams, base, base_ptr, cta, ncta); break;
                    case 64 | (2 << 16) | MEGA_VARIANT_PP: mega_gemm<64, 2, true>(hdr_params, gparams, base, base_ptr, cta, ncta); break;
                    case 64 | (1 << 16) | MEGA_VARIANT_PP: mega_gemm<64, 1, true>(hdr_params, gparams, base, base_ptr, cta, ncta); break;
                    case 128 | (1 << 16) | MEGA_VARIANT_PP: mega_gemm<128, 1, true>(hdr_params, gparams, base, base_ptr, cta, ncta); break;
                    default: if (threadIdx.x == 0) printf("sr3: step kernel: unsupported tile variant %x\n", op.variant); __trap();
                }
                break;
            }
            case MOP_PREP:
                prep_body(*reinterpret_cast<const PrepParams*>(hdr_params), reinterpret_cast<float*>(op_smem), cta, ncta);
                break;
            case MOP_ATTN: {
                const AttnParams& ap = *reinterpret_cast<const AttnParams*>(hdr_params);
                const int n_dc = ap.C / ap.dn, per_z = (ap.Lt / 128) * n_dc, units = per_z * ap.nz;
                for (int u = cta; u < units; u += ncta) {
                    const int z = u / per_z, r = u % per_z;
                    mega_attn(ap, reinterpret_cast<const AttnParams*>(gparams), base, base_ptr, r / n_dc, r % n_dc, z);
                }
                break;
            }
            case MOP_SOFTMAX:
                softmax_body(*reinterpret_cast<const SoftmaxParams*>(hdr_params), cta, ncta);
                break;
            case MOP_EMBED_FILM:
                embed_film_body(*reinterpret_cast<const EmbedFilmParams*>(hdr_params), reinterpret_cast<float*>(op_smem), t_step, cta, ncta);
                break;
            case MOP_ZERO: {
                const ZeroParams& zp = *reinterpret_cast<const ZeroParams*>(hdr_params);
                for (long long j = static_cast<long long>(cta) * blockDim.x + threadIdx.x; j < zp.n4; j += static_cast<long long>(ncta) * blockDim.x)
                    zp.ptr[j] = make_float4(0.f, 0.f, 0.f, 0.f);
                break;
            }
            default: break;
        }
        if (stamp) mp.prof[4 * i + 3] = globaltimer_ns();
        // Publication of this op's global writes: the next arrive() is __syncthreads + (thread 0) __threadfence + release -- cumulative over
        // the writes of the whole CTA, as in cooperative-groups grid.sync; each thread orders its own generic writes against later
        // async-proxy (TMA) accesses itself.
        fence_proxy_async_all();
        __syncthreads();
    }
    if (cta == 0 && threadIdx.x == 0) {
        if (mp.prof) mp.prof[4 * mp.n_ops] = globaltimer_ns();
        mp.ctl->t_cur = t_step;               // what the per-layer path's step_begin_kernel does at the start of a step
        mp.ctl->t_next = t_step - 1;
    }
}

}  // namespace sr3
