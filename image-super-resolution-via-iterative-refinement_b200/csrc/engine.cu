// Host side of libsr3_b200.so: builds the per-step kernel plan of the SR3 UNet + posterior update for one
// (config, batch), owns device buffers / packed weights / TMA descriptors, captures the step as a CUDA graph and exposes
// the C ABI declared in include/sr3_b200.h.  Reference call sites are cited in the header next to each entry point.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/sr3_b200.h"
#include "aux_kernels.cuh"
#include "attn_wgmma.cuh"
#include "attn_long_wgmma.cuh"
#include "train_kernels.cuh"
#include "window_kernels.cuh"

using namespace sr3;
typedef __nv_bfloat16 bf16;

namespace {

thread_local std::string g_err;

std::string fmt(const char* f, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, f);
    vsnprintf(buf, sizeof(buf), f, ap);
    va_end(ap);
    return std::string(buf);
}
#define CK(expr)                                                                                                  \
    do {                                                                                                          \
        cudaError_t e_ = (expr);                                                                                  \
        if (e_ != cudaSuccess) throw std::runtime_error(fmt("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e_))); \
    } while (0)
#define REQUIRE(cond, ...)                                                 \
    do {                                                                   \
        if (!(cond)) throw std::runtime_error(fmt(__VA_ARGS__));           \
    } while (0)

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    REQUIRE(p != nullptr && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available from the driver");
    fn = reinterpret_cast<EncodeTiledFn>(p);
    return fn;
}

CUtensorMap encode_map(int rank, const void* ptr, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                       CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16) {
    CUtensorMap m;
    cuuint64_t gd[5], gs[4];
    cuuint32_t bx[5], es[5];
    for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
    for (int i = 0; i < rank - 1; ++i) gs[i] = strides_bytes[i];
    // a box may be larger than the tensor extent (halo rows of small images): TMA zero-fills / clips the out-of-range part
    for (int i = 0; i < rank; ++i) REQUIRE(box[i] >= 1 && box[i] <= 256, "TMA box %u out of range (axis %d)", box[i], i);
    REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA base not 16B aligned");
    for (int i = 0; i < rank - 1; ++i) REQUIRE(strides_bytes[i] % 16 == 0 && strides_bytes[i] > 0, "TMA stride %llu (axis %d) must be a positive multiple of 16", (unsigned long long)strides_bytes[i], i + 1);
    CUresult r = get_encode_fn()(&m, dtype, rank, const_cast<void*>(ptr), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                 CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d) rank=%d dims=%llu,%llu box=%u,%u", (int)r, rank,
            (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    return m;
}

// 5-D source view of an A operand: dims (C', W', P, H', Bn), byte strides of dims 1..4
struct ASrc {
    const void* ptr = nullptr;
    int C = 0, W = 1, P = 1, H = 1, Bn = 1;
    long long sW = 0, sP = 0, sH = 0, sB = 0;
};
ASrc nhwc_src(const void* ptr, int Bn, int H, int W, int C) {
    ASrc a; a.ptr = ptr; a.C = C; a.W = W; a.P = 1; a.H = H; a.Bn = Bn;
    a.sW = 2LL * C; a.sP = 2LL * W * C; a.sH = 2LL * W * C; a.sB = 2LL * H * W * C;
    return a;
}
// stride-2 view of an NHWC tensor: (2C, W/2, 2, H/2, B)
ASrc nhwc_stride2_src(const void* ptr, int Bn, int H, int W, int C) {
    ASrc a; a.ptr = ptr; a.C = 2 * C; a.W = W / 2; a.P = 2; a.H = H / 2; a.Bn = Bn;
    a.sW = 4LL * C; a.sP = 2LL * W * C; a.sH = 4LL * W * C; a.sB = 2LL * H * W * C;
    return a;
}
// batched row-major matrices [nb][rows][K] (row stride ld elements)
ASrc matrix_src(const void* ptr, int nb, int rows, int K, long long ld, long long batch_stride_elems) {
    ASrc a; a.ptr = ptr; a.C = K; a.W = rows; a.P = 1; a.H = 1; a.Bn = nb;
    a.sW = 2LL * ld; a.sP = 2LL * ld * rows; a.sH = 2LL * ld * rows; a.sB = 2LL * batch_stride_elems;
    if (nb == 1) a.sB = a.sH;
    return a;
}

struct KSlab { int a_sel, a_chan, dw, dh, p, b_col; };

struct GemmDesc {
    ASrc a[2];
    int n_a = 1;
    const void* b_ptr = nullptr;
    long long b_rows = 0; int b_K = 0;            // B matrix [b_rows][b_K] bf16 row-major
    std::vector<KSlab> slabs;
    int block_n = 128;
    int w_box = 16, h_box = 8, b_box = 1;         // output pixel patch of one tile (mh * 128 rows)
    int mh = 1;                                   // 128-row accumulator halves per tile
    int pingpong = 0;                             // 1: ping-pong schedule (each consumer warpgroup owns whole tiles; never split)
    int tall = 0;                                 // 3x3 stride-1 "tall halo" mode: A box = 8 x (rows + 2) pixels, vertical taps share it
    int a_box_w = 0, a_box_h = 0, a_box_b = 0;    // TMA box of the A operand (0: same as the tile patch)
    int a_half_off = 0;
    bool b_is_param = false;                      // B operand is a packed weight matrix (constant within a step): eligible for L2 prefetch
    int ksplit_max = 1;                           // split-K allowed up to this factor (image convs with few output tiles)
    int tiles_w = 1, tiles_h = 1, tiles_b = 1, n_tiles = 1, nz = 1;
    int a_zstep = 0, b_zrows = 0;
    int z_phase = 0; long long z_off_hi = 0, z_off_lo = 0;   // nz = 4 output phases of a folded upsample conv (gemm_wgmma.cuh)
    int passes = 1, lo_b_col = 0, lo_a_chan[2] = {0, 0};      // precise mode: three passes over the stage table (gemm_wgmma.cuh)
    long long lo_out_off = 0, lo_t_off = 0;
    // epilogue
    int mode = 0, OW = 0, OH = 1, OB = 1, n_valid = 0;
    int out_imgs = 0;                             // images the fp32 output / residual tensors hold (0: at least every image the tiles cover)
    float scale = 1.f;
    const float* bias = nullptr; const float* bias2 = nullptr; int bias2_stride = 0;
    const float* resid = nullptr; OutSpec rs{};
    float* out_f32 = nullptr; OutSpec os{};
    bf16* out_bf16 = nullptr; OutSpec hs{};
    bf16* out_t = nullptr; int t_col0 = 0, t_rows = 0, t_ld = 0, t_per = 1;   // transposed bf16 store of columns >= t_col0
    double* stats = nullptr; int stats_C = 0, stats_coff = 0;
    const StepCtl* ctl = nullptr; PostParams post{};
};

OutSpec nhwc_out(int H, int W, int C, long long off = 0) {
    OutSpec s; s.sZ = 0; s.sB = 1LL * H * W * C; s.sH = 1LL * W * C; s.sW = C; s.off = off; return s;
}

constexpr int SMEM_LIMIT = 232448;   // 227 KB opt-in maximum per CTA on sm_90
int pick_stages(int block_n, int a_stage_bytes, int b_taps, bool resid, int num_k) {
    int s = GEMM_MAX_STAGES;
    if (const char* e = getenv("SR3_STAGES")) s = atoi(e);
    if (s > GEMM_MAX_STAGES) s = GEMM_MAX_STAGES;
    while (s > 1 && gemm_smem_bytes(block_n, a_stage_bytes, b_taps, s, resid, num_k) > SMEM_LIMIT) --s;
    if (s < 1) s = 1;
    return s;
}
int current_device() { int dev = 0; CK(cudaGetDevice(&dev)); return dev; }
int num_sms() {
    static std::map<int, int> cache;               // per device: a process may hold engines on several GPUs
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    const int dev = current_device();
    auto it = cache.find(dev);
    if (it != cache.end()) return it->second;
    int n = 0;
    CK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    cache[dev] = n;
    return n;
}
// cudaFuncSetAttribute is per device: remember which devices already have the opt-in shared-memory size of a kernel family
bool first_use_on_device(std::vector<int>& seen) {
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    const int dev = current_device();
    for (int d : seen) if (d == dev) return false;
    seen.push_back(dev);
    return true;
}
// Every kernel of the step is launched with programmatic stream serialization (PDL): its prologue overlaps the tail of the
// previous kernel; the kernels call griddepcontrol.wait before touching upstream data.
template <typename... KArgs, typename... Args>
void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    CK(cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...));
}
// Split-K layers: the `ksplit` CTAs that share an output tile are consecutive blocks and wait for each other inside the kernel.  They are
// launched as ONE THREAD-BLOCK CLUSTER (cluster dimension = ksplit): the hardware gang-schedules a cluster, so the partners are co-resident
// by construction -- no assumption about what else occupies the device (other engines / streams, NCCL, library kernels), inside or outside
// graph capture, and the launch keeps its programmatic-dependent-launch edge.
constexpr int MAX_CLUSTER_SPLIT = 8;               // portable cluster size limit
template <int BN, int MH, bool PP = false>
void launch_gemm_bn(const GemmParams& p, dim3 grid, int smem, cudaStream_t st) {
    if (p.ksplit == 1) { launch_k(gemm_tile_kernel<BN, MH, PP>, grid, dim3(GEMM_THREADS), (size_t)smem, st, p); return; }
    REQUIRE(!PP, "a ping-pong tile launch cannot be split");
    REQUIRE(p.ksplit <= MAX_CLUSTER_SPLIT && grid.x % p.ksplit == 0, "split-K factor %d does not form clusters of grid %u", p.ksplit, grid.x);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = dim3(GEMM_THREADS); cfg.dynamicSmemBytes = (size_t)smem; cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)p.ksplit; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 2;
    CK(cudaLaunchKernelEx(&cfg, gemm_tile_kernel<BN, MH>, p));
}
void init_gemm_attrs() {
    static std::vector<int> seen;
    if (!first_use_on_device(seen)) return;
    CK(cudaFuncSetAttribute(gemm_tile_kernel<16, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    CK(cudaFuncSetAttribute(gemm_tile_kernel<16, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    CK(cudaFuncSetAttribute(gemm_tile_kernel<32, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    CK(cudaFuncSetAttribute(gemm_tile_kernel<64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    CK(cudaFuncSetAttribute(gemm_tile_kernel<64, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    CK(cudaFuncSetAttribute(gemm_tile_kernel<128, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    CK(cudaFuncSetAttribute(gemm_tile_kernel<128, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    CK(cudaFuncSetAttribute(gemm_tile_kernel<256, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    CK(cudaFuncSetAttribute(gemm_tile_kernel<64, 2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    CK(cudaFuncSetAttribute(gemm_tile_kernel<64, 1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    CK(cudaFuncSetAttribute(gemm_tile_kernel<128, 1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
}

// How many clusters of `c` tile-kernel CTAs (one CTA per SM: they use the whole shared memory) the device holds at once; a cluster lives
// inside one GPC, so this is less than SMs / c.  Split-K factors are chosen so that all clusters of a layer run in one wave.
int cluster_capacity(int c) {
    static std::map<std::pair<int, int>, int> cache;
    static std::mutex mu;
    if (c <= 1) return num_sms();
    init_gemm_attrs();
    std::lock_guard<std::mutex> lock(mu);
    const std::pair<int, int> key(current_device(), c);
    auto it = cache.find(key);
    if (it != cache.end()) return it->second;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(c * 32); cfg.blockDim = dim3(GEMM_THREADS); cfg.dynamicSmemBytes = SMEM_LIMIT;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)c; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, gemm_tile_kernel<64, 1>, &cfg) != cudaSuccess || n <= 0) {
        cudaGetLastError();
        n = 8 * ((num_sms() / 8) / c);               // eight GPCs of equal size, conservatively
    }
    cache[key] = n;
    return n;
}
// largest split-K factor <= want whose clusters all fit the device together with `tiles` output tiles
int fit_split(int want, long long tiles) {
    if (want > MAX_CLUSTER_SPLIT) want = MAX_CLUSTER_SPLIT;
    while (want > 1 && cluster_capacity(want) < tiles) --want;
    return want;
}

struct DevAllocs {
    std::vector<void*> ptrs;
    long long bytes = 0;
    void* alloc(size_t n, bool zero = true) {
        void* p = nullptr;
        if (n == 0) n = 16;
        CK(cudaMalloc(&p, n));
        if (zero) CK(cudaMemset(p, 0, n));
        ptrs.push_back(p);
        bytes += (long long)n;
        return p;
    }
    ~DevAllocs() { for (void* p : ptrs) cudaFree(p); }
};

typedef std::function<void(cudaStream_t)> Op;
struct GemmHandle { std::shared_ptr<GemmParams> p; const void* w_ptr = nullptr; long long w_bytes = 0; bool w_is_param = false; int bn = 0, mh = 0; };
static thread_local std::vector<GemmHandle>* g_gemm_registry = nullptr;   // set by the engine while it builds its plan
// what the most recent sr3_test_conv_ex of this thread launched (sr3_tile_schedule with no engine)
struct LastTestConv { sr3_gemm_geometry geo{}; int schedule = -1; int out_hwc[3] = {0, 0, 0}; };
static thread_local LastTestConv g_last_test_conv;

// Turns a GemmDesc into a launchable op (encodes the TMA maps, uploads the K-slab table).  `geo` / `schedule` (optional) receive the variant,
// launch shape and schedule (0 cooperative, 1 ping-pong) that were actually chosen, after every host-side override and cap.
Op make_gemm_op(const GemmDesc& d, DevAllocs& mem, sr3_gemm_geometry* geo = nullptr, int* schedule = nullptr) {
    REQUIRE(d.w_box * d.h_box * d.b_box == 128 * d.mh, "tile box must cover %d rows", 128 * d.mh);
    REQUIRE(!d.slabs.empty(), "gemm without K slabs");
    GemmParams p;
    memset(&p, 0, sizeof(p));
    const int abw = d.a_box_w ? d.a_box_w : d.w_box, abh = d.a_box_h ? d.a_box_h : d.h_box, abb = d.a_box_b ? d.a_box_b : d.b_box;
    p.a_stage_bytes = abw * abh * abb * 128;
    REQUIRE(p.a_stage_bytes % 1024 == 0, "A box must be a whole number of swizzle atoms");
    for (int i = 0; i < 2; ++i) {
        const ASrc& a = d.a[i < d.n_a ? i : 0];
        REQUIRE(a.C % 64 == 0, "A channels (%d) must be a multiple of 64", a.C);
        const uint64_t dims[5] = {(uint64_t)a.C, (uint64_t)a.W, (uint64_t)a.P, (uint64_t)a.H, (uint64_t)a.Bn};
        const uint64_t str[4] = {(uint64_t)a.sW, (uint64_t)a.sP, (uint64_t)a.sH, (uint64_t)a.sB};
        const uint32_t box[5] = {64u, (uint32_t)abw, 1u, (uint32_t)abh, (uint32_t)abb};
        p.a_map[i] = encode_map(5, a.ptr, dims, str, box);
    }
    {
        REQUIRE(d.b_K % 64 == 0, "B K extent must be a multiple of 64");
        const uint64_t dims[2] = {(uint64_t)d.b_K, (uint64_t)d.b_rows};
        const uint64_t str[1] = {2ull * d.b_K};
        const uint32_t box[2] = {64u, (uint32_t)d.block_n};
        REQUIRE(d.b_rows >= d.block_n, "B rows %lld < block_n %d", d.b_rows, d.block_n);
        p.b_map = encode_map(2, d.b_ptr, dims, str, box);
    }
    // stage table.  Tall mode: the three vertical taps (dh = -1, 0, +1) of one (source, channel chunk, dw) share one halo box.
    // Generic mode: up to three consecutive K slabs of the same source are grouped into a stage (one box each).
    std::vector<StageDesc> tab;
    int b_taps = 1, a_boxes = 1;
    for (size_t i = 0; i < d.slabs.size(); ++i) {
        const KSlab& k = d.slabs[i];
        REQUIRE(k.a_sel < d.n_a, "slab refers to missing A source");
        StageDesc e; memset(&e, 0, sizeof(e));
        e.a_sel = k.a_sel; e.ntaps = 1;
        e.tap[0].a_chan = k.a_chan; e.tap[0].dw = k.dw; e.tap[0].dh = k.dh; e.tap[0].p = k.p; e.tap[0].b_col = k.b_col;
        if (d.tall) {
            // all vertical taps (dh) of this (source, channel chunk, dw) share the halo box: 3 for a 3x3 conv, 2 for a phase of a
            // folded upsample conv, 1 for the 1x1 shortcut
            bool first = true;
            int nt = 0;
            for (const KSlab& o : d.slabs) {
                if (o.a_sel != k.a_sel || o.a_chan != k.a_chan || o.dw != k.dw) continue;
                if (&o < &k) { first = false; break; }
                REQUIRE(nt < 3 && o.p == 0 && o.dh >= -1 && o.dh <= 1, "bad tall tap group");
                e.tap[nt] = e.tap[0];
                e.tap[nt].dh = -1;                        // the box always starts one row above the tile
                e.tap[nt].b_col = o.b_col;
                e.tap[nt].a_off = (o.dh + 1) * 1024;
                ++nt;
            }
            if (!first) continue;                         // folded into the stage of the group's first slab
            e.ntaps = nt;
            if (nt > b_taps) b_taps = nt;
        } else {
            e.a_multi = 1;
            int n = 1;
            while (n < 3 && i + n < d.slabs.size() && d.slabs[i + n].a_sel == k.a_sel) ++n;
            e.ntaps = n;
            for (int t = 0; t < n; ++t) {
                const KSlab& o = d.slabs[i + t];
                e.tap[t].a_chan = o.a_chan; e.tap[t].dw = o.dw; e.tap[t].dh = o.dh; e.tap[t].p = o.p; e.tap[t].b_col = o.b_col;
                e.tap[t].a_off = t * p.a_stage_bytes;     // boxes back to back (p.a_stage_bytes still holds ONE box here)
            }
            if (n > b_taps) b_taps = n;
            if (n > a_boxes) a_boxes = n;
            i += n - 1;
        }
        tab.push_back(e);
    }
    p.a_box_bytes = p.a_stage_bytes;
    p.a_stage_bytes = p.a_box_bytes * a_boxes;
    REQUIRE((int)tab.size() <= GEMM_MAX_K, "gemm with %d stages per tile (max %d)", (int)tab.size(), GEMM_MAX_K);
    StageDesc* dtab = static_cast<StageDesc*>(mem.alloc(tab.size() * sizeof(StageDesc), false));
    CK(cudaMemcpy(dtab, tab.data(), tab.size() * sizeof(StageDesc), cudaMemcpyHostToDevice));
    p.ktab = dtab; p.num_k = (int)tab.size();
    p.b_taps = b_taps; p.a_half_off = d.a_half_off;
    p.tiles_w = d.tiles_w; p.tiles_h = d.tiles_h; p.tiles_b = d.tiles_b;
    p.w_box = d.w_box; p.h_box = d.h_box; p.b_box = d.b_box;
    {
        auto lg = [](int v) { int l = 0; while ((1 << l) < v) ++l; return l; };
        REQUIRE((d.w_box & (d.w_box - 1)) == 0 && (d.h_box & (d.h_box - 1)) == 0, "tile box %dx%d must be powers of two", d.w_box, d.h_box);
        p.w_shift = lg(d.w_box); p.h_shift = lg(d.h_box);
    }
    p.a_zstep = d.a_zstep; p.b_zrows = d.b_zrows;
    p.n_tiles = d.n_tiles; p.nz = d.nz;
    p.mode = d.mode; p.OW = d.OW; p.OH = d.OH; p.OB = d.OB; p.n_valid = d.n_valid; p.scale = d.scale;
    p.bias = d.bias; p.bias2 = d.bias2; p.bias2_stride = d.bias2_stride;
    p.resid = d.resid; p.rs = d.rs; p.out_f32 = d.out_f32; p.os = d.os; p.out_bf16 = d.out_bf16; p.hs = d.hs;
    p.out_t = d.out_t; p.t_col0 = d.t_col0; p.t_rows = d.t_rows; p.t_ld = d.t_ld; p.t_per = d.t_per > 0 ? d.t_per : 1;
    p.stats = d.stats; p.stats_C = d.stats_C; p.stats_coff = d.stats_coff; p.ctl = d.ctl; p.post = d.post;
    p.z_phase = d.z_phase; p.z_off_hi = d.z_off_hi; p.z_off_lo = d.z_off_lo;
    p.passes = d.passes; p.lo_b_col = d.lo_b_col; p.lo_a_chan[0] = d.lo_a_chan[0]; p.lo_a_chan[1] = d.lo_a_chan[1];
    p.lo_out_off = d.lo_out_off; p.lo_t_off = d.lo_t_off;
    if (d.stats) REQUIRE((d.w_box * d.h_box) % 32 == 0, "stats need whole warps per image");
    // fp32 output / residual through smem + TMA: one 32-row x 32-column box per epilogue warp
    p.tma_epi = (d.mode == 0 && (d.out_f32 || d.resid)) ? 1 : 0;
    if (p.tma_epi) {
        const int w_sub = d.w_box < 32 ? d.w_box : 32, h_sub = 32 / w_sub;
        REQUIRE(d.w_box % w_sub == 0 && (d.h_box % h_sub == 0 || d.h_box == 1) && (h_sub == 1 || (128 / w_sub) % h_sub == 0), "tile box %dx%d cannot be split into per-warp boxes", d.w_box, d.h_box);
        auto mk = [&](const float* ptr, const OutSpec& o, bool& c4z) {
            c4z = (o.sB == 0 && o.sZ != 0);
            const long long s4 = c4z ? o.sZ : o.sB;
            const uint64_t n4 = c4z ? (uint64_t)d.nz : d.out_imgs ? (uint64_t)d.out_imgs : (uint64_t)(d.tiles_b * d.b_box > d.OB ? d.tiles_b * d.b_box : d.OB);
            uint64_t dims[5] = {(uint64_t)d.n_valid, (uint64_t)d.OW, 1ull, (uint64_t)d.OH, n4};
            uint64_t str[4];
            str[0] = (uint64_t)o.sW * 4;
            str[1] = str[0] * d.OW;
            str[2] = d.OH > 1 ? (uint64_t)o.sH * 4 : str[1];
            str[3] = s4 != 0 ? (uint64_t)s4 * 4 : str[2] * d.OH;
            if (d.z_phase) {      // {2N (px, n), W, 2 (py), H, B}: phase (py, px) is coordinate 2 and an offset of px * N in coordinate 0
                REQUIRE(d.z_off_lo == d.n_valid && o.sW == 2 * d.n_valid, "phase-batched output must be NHWC with 2x the width");
                dims[0] = 2ull * d.n_valid; dims[2] = 2ull; str[1] = (uint64_t)d.z_off_hi * 4;
            }
            const uint32_t box[5] = {32u, (uint32_t)w_sub, 1u, (uint32_t)h_sub, 1u};
            REQUIRE(d.n_valid >= 32, "TMA epilogue needs at least 32 output columns");
            return encode_map(5, ptr + o.off, dims, str, box, CU_TENSOR_MAP_DATA_TYPE_FLOAT32);
        };
        bool zo = false, zr = false;
        if (d.out_f32) p.out_map = mk(d.out_f32, d.os, zo);
        if (d.resid) p.res_map = mk(d.resid, d.rs, zr);
        if (d.out_f32 && d.resid) REQUIRE(zo == zr, "output and residual must share the batch coordinate");
        if (!d.out_f32) p.out_map = p.res_map;
        if (!d.resid) p.res_map = p.out_map;
        p.epi_c4_is_z = (d.out_f32 ? zo : zr) ? 1 : 0;
    } else {
        p.out_map = p.b_map; p.res_map = p.b_map;
    }
    // split-K: when the output has too few tiles to occupy the SMs, `ksplit` CTAs share a tile, each streams a slice of K and parks its
    // partial tile in `ws`; every one of them then finalises a 1/ksplit share of the tile (gemm_wgmma.cuh, epilogue pass 1).
    // One (tile, split) pair per SM at most: all CTAs are co-resident, which the in-kernel wait relies on.
    p.ksplit = 1;
    {
        const int tiles = d.tiles_w * d.tiles_h * d.tiles_b * d.n_tiles * d.nz;
        const int ks = d.ksplit_max;
        if (ks > 1 && !d.pingpong && d.mode == 0 && d.out_f32 && d.block_n >= 32 && d.n_valid % 32 == 0) {
            int want = num_sms() / tiles;                  // CTAs per tile that still fit one wave
            if (want > ks) want = ks;
            if (want > p.num_k * d.passes / 2) want = p.num_k * d.passes / 2;    // at least two stages per slice
            const int units = d.mh * (d.block_n / 32) * 4; // 32x32 units of a tile: every split finalises at least one
            if (want > units) want = units;
            want = fit_split(want, tiles);
            if (want > 1) {
                p.ksplit = want;
                p.ws = static_cast<float*>(mem.alloc((size_t)tiles * want * d.mh * 128 * d.block_n * sizeof(float), false));
                p.counters = static_cast<unsigned int*>(mem.alloc((size_t)tiles * sizeof(unsigned int)));
            }
        }
    }
    const int total_tiles = d.tiles_w * d.tiles_h * d.tiles_b * d.n_tiles * d.nz * p.ksplit;
    int ctas = total_tiles < num_sms() ? total_tiles : num_sms();
    if (const char* e = getenv("SR3_MAX_CTAS")) { int v = atoi(e); if (v > 0 && v < ctas) ctas = v; }
    // the split-K partners of a tile wait for each other inside the kernel: a CTA that owned two splits of one tile would wait for itself
    REQUIRE(p.ksplit == 1 || ctas == total_tiles, "split-K launch needs one CTA per (tile, split) pair: %d CTAs for %d (SR3_MAX_CTAS with a split tile)", ctas, total_tiles);
    const dim3 grid(ctas, 1, 1);
    const int bn = d.block_n;
    const int mh = d.mh;
    const bool res_smem = p.tma_epi && d.resid != nullptr && p.ksplit <= 1;
    p.stages = pick_stages(d.block_n, p.a_stage_bytes, p.b_taps, res_smem, p.num_k);
    const int smem = gemm_smem_bytes(bn, p.a_stage_bytes, p.b_taps, p.stages, res_smem, p.num_k);
    REQUIRE(smem <= SMEM_LIMIT, "gemm shared memory %d exceeds the limit", smem);
    init_gemm_attrs();
    REQUIRE((bn == 16 || bn == 32 || bn == 64 || bn == 128 || bn == 256) && (mh == 1 || (mh == 2 && bn <= 128 && bn != 32)), "unsupported tile %dx%d", 128 * mh, bn);
    const bool pp = d.pingpong != 0;
    REQUIRE(!pp || (gemm_pingpong_ok(bn, mh) && p.ksplit == 1 && d.mode == 0), "no ping-pong form of tile %dx%d (split %d)", 128 * mh, bn, p.ksplit);
    if (geo) {
        geo->tall = d.tall; geo->mh = mh; geo->block_n = bn; geo->h_box = d.h_box; geo->b_box = d.b_box;
        geo->ksplit = p.ksplit; geo->stages = p.stages; geo->ctas = ctas; geo->tiles = total_tiles / p.ksplit; geo->res_smem = res_smem ? 1 : 0;
    }
    if (schedule) *schedule = pp ? 1 : 0;
    std::shared_ptr<GemmParams> sp = std::make_shared<GemmParams>(p);
    if (g_gemm_registry) {
        GemmHandle h; h.p = sp; h.w_ptr = d.b_ptr; h.w_bytes = 2LL * d.b_rows * d.b_K; h.w_is_param = d.b_is_param; h.bn = bn; h.mh = mh;
        g_gemm_registry->push_back(h);
    }
    return [sp, grid, bn, mh, pp, smem](cudaStream_t st) {
        const GemmParams& p = *sp;
        if (pp) {
            if (mh == 2) launch_gemm_bn<64, 2, true>(p, grid, smem, st);
            else if (bn == 64) launch_gemm_bn<64, 1, true>(p, grid, smem, st);
            else launch_gemm_bn<128, 1, true>(p, grid, smem, st);
            return;
        }
        switch (bn) {
            case 16: if (mh == 2) launch_gemm_bn<16, 2>(p, grid, smem, st); else launch_gemm_bn<16, 1>(p, grid, smem, st); break;
            case 32: launch_gemm_bn<32, 1>(p, grid, smem, st); break;
            case 64: if (mh == 2) launch_gemm_bn<64, 2>(p, grid, smem, st); else launch_gemm_bn<64, 1>(p, grid, smem, st); break;
            case 128: if (mh == 2) launch_gemm_bn<128, 2>(p, grid, smem, st); else launch_gemm_bn<128, 1>(p, grid, smem, st); break;
            default: launch_gemm_bn<256, 1>(p, grid, smem, st); break;
        }
    };
}

// Fused attention core: S = q k^T / sqrt(C), softmax, O = P v in one launch.  qk [nz*Lt][2C], vT [nz*C][Lt], out [nz*Lt][C].
// Up to 256 tokens a row block of S stays in registers (attn_wgmma.cuh); above, the keys stream through in blocks of 128 with a
// running maximum (attn_long_wgmma.cuh), and an attention batch is then always one image.
bool attn_fusable(int Lt, int C) { return Lt >= 128 && Lt % 128 == 0 && C % 128 == 0 && C >= 128; }

Op make_attn_op(const bf16* qk, const bf16* vT, bf16* out, int nz, int Lt, int HW, int C) {
    REQUIRE(attn_fusable(Lt, C) && Lt % HW == 0, "attention shape Lt=%d HW=%d C=%d is not supported by the fused kernel", Lt, HW, C);
    REQUIRE(Lt <= 256 || HW == Lt, "attention over %d tokens per batch takes one image per batch (HW=%d)", Lt, HW);
    AttnParams p;
    memset(&p, 0, sizeof(p));
    {
        const uint64_t dims[2] = {(uint64_t)2 * C, (uint64_t)nz * Lt};
        const uint64_t str[1] = {(uint64_t)2 * C * 2};
        const uint32_t box[2] = {64u, 128u};
        p.qk_map = encode_map(2, qk, dims, str, box);
    }
    {
        const uint64_t dims[2] = {(uint64_t)Lt, (uint64_t)nz * C};
        const uint64_t str[1] = {(uint64_t)Lt * 2};
        const uint32_t box[2] = {64u, 128u};
        p.vt_map = encode_map(2, vT, dims, str, box);
    }
    p.out = out; p.C = C; p.Lt = Lt; p.HW = HW; p.nz = nz;
    p.dn = (C % 256 == 0) ? 256 : 128;
    p.scale_log2e = 1.4426950408889634f / sqrtf((float)C);
    if (Lt > 256) {
        p.dn = ATTNL_DN;
        static std::vector<int> seen_long;
        if (first_use_on_device(seen_long)) CK(cudaFuncSetAttribute(attn_long_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATTNL_SMEM_BYTES));
        const dim3 grid((Lt / 128) * (C / ATTNL_DN), nz, 1);
        return [p, grid](cudaStream_t st) { launch_k(attn_long_kernel, grid, dim3(ATTN_THREADS), ATTNL_SMEM_BYTES, st, p); };
    }
    static std::vector<int> seen;
    if (first_use_on_device(seen)) CK(cudaFuncSetAttribute(attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATTN_SMEM_BYTES));
    const dim3 grid((Lt / 128) * (C / p.dn), nz, 1);
    return [p, grid](cudaStream_t st) { launch_k(attn_kernel, grid, dim3(ATTN_THREADS), ATTN_SMEM_BYTES, st, p); };
}

void pick_image_box(int W, int H, int& w_box, int& h_box, int& b_box);
int pick_block_n(int cout);
// SR3_PINGPONG: -1 unset (the byte model chooses the schedule), 0 cooperative only, 1 ping-pong wherever the tile shape has that form
int pingpong_knob() {
    const char* e = getenv("SR3_PINGPONG");
    return e ? (atoi(e) != 0 ? 1 : 0) : -1;
}

// Geometry of an image conv: the "tall halo" form for 3x3 stride-1 convs at >= 16x16, else a plain 128-pixel patch per tap.
// The tile shape (rows x BLOCK_N) and the split-K factor are chosen by a byte model of the per-CTA critical path: a CTA ingests
// stages x (A box + B boxes) through TMA at a fixed rate, runs ceil(tiles * split / SMs) waves, and a split tile costs an extra
// partial-tile store + reload + a grid-level handshake (`tools/gpu_layer_profile.py --sweep` times every candidate per layer).
// Bt: images the tiles must cover (tiles_b = ceil(Bt / b_box); images past the A tensor's batch load as zeros).
void conv_geometry(GemmDesc& d, int OW, int OH, int Bt, int cout, bool has_resid = false, int nz = 1) {
    const int npass = d.passes > 1 ? d.passes : 1;
    bool tall_ok = OW >= 8 && OH >= 16, has3 = false;
    for (const KSlab& k : d.slabs) { if (k.p != 0) tall_ok = false; if (k.dh != 0) has3 = true; }
    tall_ok = tall_ok && has3 && (OH >= 32 || Bt % 2 == 0);
    const int sms = num_sms();
    // Schedule.  SR3_PINGPONG (tests / A-B timing): 1 = ping-pong wherever the tile shape has that form (the model ranks the ping-pong
    // shapes), 0 = cooperative everywhere; a tile forced by SR3_TALL_BN / SR3_TALL_MH / SR3_BLOCK_N keeps the forced shape and, unless
    // SR3_PINGPONG=1, the cooperative form.  Unset: every cooperative tile and every ping-pong tile compete, each charged its epilogue.
    const int pp_knob = pingpong_knob();
    const bool pp_force = pp_knob == 1, pp_auto = pp_knob < 0;
    const bool shape_forced = getenv("SR3_TALL_BN") || getenv("SR3_TALL_MH") || getenv("SR3_BLOCK_N");
    // Epilogue of one 32x32 output item (transposition, bias / FiLM, residual, TMA store, bf16 copy, GroupNorm sums) in bytes of TMA
    // ingest, one constant per variant family.  Fitted with `tools/gpu_layer_profile.py --sweep` (every tile op of the 16->128 B=16,
    // 64->512 B=4 and unconditional 128 B=32 steps under every candidate, H100, DESIGN.md section 8) by minimising the summed time of the
    // tiles the model picks, with the plain 3x3 convs of the 16->128 step at B = 16 held to their measured-and-tested schedules (128x64
    // ping-pong at 128x128 and 64x64, cooperative at 32x32).  The 256x128 cooperative tile and the 128-register ping-pong forms (256x64,
    // 128x128) spill through their epilogue (section 8, ptxas table), the 128x64 ping-pong form barely does, so they cannot share one
    // constant; the tall and generic 128x64 ping-pong tiles fitted apart.
    constexpr double EPI_COOP = 200000.0, EPI_COOP_256x128 = 2000000.0, EPI_PP_128REG = 600000.0;
    const double EPI_PP_64REG = tall_ok ? 200000.0 : 10000.0;
    // cost in bytes of the slowest CTA; `split` returns the factor the cost was computed for.  pp: the ping-pong schedule (never split):
    // a warpgroup's epilogue (all MH x NCH items of the tile on its 4 warps) runs under the other warpgroup's MMAs, so only the last one is
    // exposed, unless the epilogue is longer than the MMA phase it hides behind.  The cooperative cost includes its epilogue, shared by the
    // consumer warps and never overlapped with MMAs.
    auto items_of = [](int rows, int bn) { return (double)(rows / 128) * (bn >= 32 ? bn / 32 : 1); };   // 32x32 items per warp quadrant
    auto model = [&](long long tiles, int nstage, long long stage_bytes, int rows, int bn, int& split, bool pp = false) -> double {
        if (pp) {
            split = 1;
            const long long t = (tiles + sms - 1) / sms;               // tiles of the busiest CTA
            const double mma = (double)nstage * stage_bytes, epi = items_of(rows, bn) * (rows == 128 && bn == 64 ? EPI_PP_64REG : EPI_PP_128REG);
            const double serial = (double)t * mma + epi, paired = (double)((t + 1) / 2) * (mma + epi);
            return serial > paired ? serial : paired;
        }
        int smax = 1;
        if (bn >= 32 && cout % 32 == 0) {
            smax = (int)(sms / tiles);
            const int units = (rows / 128) * (bn / 32) * 4;
            if (smax > units) smax = units;
            if (smax > nstage / 2) smax = nstage / 2;
            if (smax > 16) smax = 16;
            if (smax < 1) smax = 1;
            smax = fit_split(smax, tiles);
        }
        split = smax;
        const long long waves = (tiles * smax + sms - 1) / sms;
        double c = (double)waves * ((nstage + smax - 1) / smax) * (double)stage_bytes;
        // the 8 consumer warps (4: single-warpgroup tile) share the items of the tile's 1/split share
        const double warps = gemm_single_wg(bn, rows / 128) ? 4.0 : 8.0;
        c += (double)waves * items_of(rows, bn) * 4.0 / (warps * smax) * (rows == 256 && bn == 128 ? EPI_COOP_256x128 : EPI_COOP);
        // a split tile: partial tile out (registers -> L2) and back, weighted 2x against streamed TMA bytes, plus the grid-level
        // handshake (fitted with the epilogue constants); a residual is then read with plain loads instead of TMA
        if (smax > 1) c += 4.0 * rows * bn * 4 + 2000000.0 + (has_resid ? 2.0 * rows * bn * 4 : 0.0);
        return c;
    };
    d.ksplit_max = 1;
    if (tall_ok) {
        d.tall = 1; d.w_box = 8;
        struct Cand { int mh, bn; };
        const Cand cands[4] = {{2, 128}, {2, 64}, {1, 64}, {1, 32}};
        auto geom = [&](int mh, int& h_box, int& b_box) {
            if (mh == 2 && OH >= 32) { h_box = 32; b_box = 1; }
            else if (mh == 2) { h_box = 16; b_box = 2; }
            else { h_box = 16; b_box = 1; }
        };
        // stages per tile: one per (source, 64-channel chunk, dw) group of vertical taps
        int nstage = 0;
        for (size_t i = 0; i < d.slabs.size(); ++i) {
            bool first = true;
            for (size_t j = 0; j < i; ++j)
                if (d.slabs[j].a_sel == d.slabs[i].a_sel && d.slabs[j].a_chan == d.slabs[i].a_chan && d.slabs[j].dw == d.slabs[i].dw) { first = false; break; }
            if (first) ++nstage;
        }
        int mh = 2, bn = 16, split = 1, pp = 0;       // Cout = 3 (final conv) keeps the 16-wide tile
        if (cout % 32 == 0) {
            double best = 1e300, best_pp = 1e300;
            int pp_mh = 0, pp_bn = 0;
            for (int i = 0; i < 4; ++i) {
                const Cand& c = cands[i];
                if (cout % c.bn != 0) continue;
                int hb, bb; geom(c.mh, hb, bb);
                const long long tiles = (long long)(OW / 8) * (OH / hb) * ((Bt + bb - 1) / bb) * (cout / c.bn) * nz;
                const long long stage_bytes = (c.mh == 2 ? 36864 : 18432) + 3ll * c.bn * 128;
                int sp = 1;
                const double cost = model(tiles, nstage * npass, stage_bytes, c.mh * 128, c.bn, sp);
                if (gemm_pingpong_ok(c.bn, c.mh)) {
                    int sp1 = 1;
                    const double cpp = model(tiles, nstage * npass, stage_bytes, c.mh * 128, c.bn, sp1, true);
                    if (cpp < best_pp) { best_pp = cpp; pp_mh = c.mh; pp_bn = c.bn; }
                }
                // the residual is staged through smem (8 warps x 8 KB) unless the tile is split: a 256x128 tile would be left with one stage
                if (c.bn == 128 && has_resid && sp <= 1) continue;
                if (cost < best) { best = cost; mh = c.mh; bn = c.bn; split = sp; }
            }
            if (!shape_forced && pp_bn && (pp_force || (pp_auto && best_pp < best))) { mh = pp_mh; bn = pp_bn; split = 1; pp = 1; }
        }
        if (const char* e = getenv("SR3_TALL_BN")) { int v = atoi(e); if ((v == 32 || v == 64 || v == 128) && cout % v == 0) { bn = v; split = 16; } }
        if (const char* e = getenv("SR3_TALL_MH")) { int v = atoi(e); if (v == 1 || v == 2) { mh = v; split = 16; } }
        if (mh == 2 && bn == 32) bn = 64;
        if (shape_forced) pp = (pp_force && gemm_pingpong_ok(bn, mh)) ? 1 : 0;
        if (pp) split = 1;
        d.mh = mh; d.block_n = bn; d.ksplit_max = split; d.pingpong = pp;
        geom(mh, d.h_box, d.b_box);
        d.a_box_w = 8; d.a_box_b = d.b_box;
        if (mh == 2 && d.b_box == 1) { d.a_box_h = 34; d.a_half_off = 16 * 1024; }
        else if (mh == 2) { d.a_box_h = 18; d.a_half_off = 18 * 1024; }
        else { d.a_box_h = 18; d.a_half_off = 0; }
    } else {
        d.tall = 0; d.mh = 1;
        pick_image_box(OW, OH, d.w_box, d.h_box, d.b_box);
        d.block_n = pick_block_n(cout);
        const long long mt = (long long)(OW / d.w_box) * ((OH + d.h_box - 1) / d.h_box) * ((Bt + d.b_box - 1) / d.b_box) * nz;
        if (getenv("SR3_BLOCK_N") == nullptr && cout % 32 == 0) {
            // generic stages group up to three K slabs (one A box + one B box each)
            const int nstage = (((int)d.slabs.size() + 2) / 3) * npass;
            double best = 1e300, best_pp = 1e300;
            int pp_bn = 0;
            for (int bn = 128; bn >= 32; bn >>= 1) {
                if (cout % bn != 0) continue;
                int sp = 1;
                const long long tiles = mt * (cout / bn);
                const double cost = model(tiles, nstage, 3ll * (16384 + bn * 128), 128, bn, sp);
                // ping-pong needs two stages in flight: one warpgroup holds a stage while the other waits for the next
                if (gemm_pingpong_ok(bn, 1) && gemm_smem_bytes(bn, 3 * 16384, 3, 2, has_resid, nstage / npass) <= SMEM_LIMIT) {
                    int sp1 = 1;
                    const double cpp = model(tiles, nstage, 3ll * (16384 + bn * 128), 128, bn, sp1, true);
                    if (cpp < best_pp) { best_pp = cpp; pp_bn = bn; }
                }
                if (bn == 128 && sp > 1) continue;      // 96 KB stages leave a 2-deep pipeline: measured slower than 64-wide split tiles
                if (cost < best) { best = cost; d.block_n = bn; d.ksplit_max = sp; }
            }
            if (pp_bn && (pp_force || (pp_auto && best_pp < best))) { d.block_n = pp_bn; d.ksplit_max = 1; d.pingpong = 1; }
        } else if (pp_force && gemm_pingpong_ok(d.block_n, 1)) {
            d.pingpong = 1;
        }
    }
    if (d.pingpong) d.ksplit_max = 1;
    if (const char* e = getenv("SR3_KSPLIT")) d.ksplit_max = atoi(e);
    d.tiles_w = OW / d.w_box; d.tiles_h = (OH + d.h_box - 1) / d.h_box; d.tiles_b = (Bt + d.b_box - 1) / d.b_box;
}

// An image of fewer than 32 pixels (4x4) gets a patch padded to 32 rows (4 x 8: rows 4..7 lie outside the image, TMA loads them as zeros
// and the epilogue masks them), so that a warp's 32 rows still hold one image: its FiLM bias, GroupNorm run and TMA boxes stay per image.
void pick_image_box(int W, int H, int& w_box, int& h_box, int& b_box) {
    w_box = W < 16 ? W : 16;
    h_box = 128 / w_box;
    if (h_box > H) h_box = H;
    if (w_box * h_box < 32) h_box = 32 / w_box;
    b_box = 128 / (w_box * h_box);
}

int pick_block_n(int cout) {
    if (const char* e = getenv("SR3_BLOCK_N")) { int v = atoi(e); if (v == 32 || v == 64 || v == 128 || v == 256) if (cout % v == 0) return v; }
    if (cout % 128 == 0) return 128;
    if (cout % 64 == 0) return 64;
    return 16;
}

// `row` = channels per pixel of the source tensor (2 * cin in precise mode: [hi | lo]); only the stride-2 view needs it
void add_conv_slabs(std::vector<KSlab>& slabs, int a_sel, int cin, int ksize, int stride, int b_col0, int row = 0) {
    if (row == 0) row = cin;
    if (ksize == 1) {
        for (int c = 0; c < cin; c += 64) slabs.push_back({a_sel, c, 0, 0, 0, b_col0 + c});
        return;
    }
    for (int r = 0; r < 3; ++r)
        for (int s = 0; s < 3; ++s)
            for (int c = 0; c < cin; c += 64) {
                KSlab k; k.a_sel = a_sel; k.b_col = b_col0 + (r * 3 + s) * cin + c;
                if (stride == 1) { k.dh = r - 1; k.dw = s - 1; k.p = 0; k.a_chan = c; }
                else {   // input row 2*oh + r - 1, column 2*ow + s - 1 in the (2C, W/2, 2, H/2, B) view
                    k.dh = (r == 0) ? -1 : 0; k.p = (r == 1) ? 0 : 1;
                    k.dw = (s == 0) ? -1 : 0; k.a_chan = ((s == 1) ? 0 : row) + c;
                }
                slabs.push_back(k);
            }
}

// ------------------------------------------------------------------------------------------------ engine
struct Act {
    float* p = nullptr; double* stats = nullptr;
    int C = 0, H = 0, W = 0;
    // training plan only: gradient of the loss with respect to this tensor (fp32 NHWC), its bf16 copy (operand of the data / weight gradient
    // GEMMs) and its per-(image, channel) sums (bias gradients), all complete when the producing layer's backward runs
    float* g = nullptr; bf16* gb = nullptr; float* gsum = nullptr;
};

struct ParamEntry {
    std::string name;
    std::vector<int64_t> shape;
    int64_t numel = 0;
    bool loaded = false;
};

struct LayerSpec { std::string name; int kind; int cin, cout; bool attn; int res; };   // kind: 0 conv, 1 res, 2 down, 3 up

// precise mode: three passes over the stage table; the low halves of A source i start c_i channels after its high halves, those of the
// weights ktot columns after theirs
void set_precise_fields(GemmDesc& d, int c0, int c1, int ktot) {
    d.passes = 3; d.lo_a_chan[0] = c0; d.lo_a_chan[1] = c1; d.lo_b_col = ktot;
}

// generic image conv: A sources already bf16; out fp32 NHWC (+stats)
struct ConvArgs {
    ASrc a[2]; int n_a = 1;
    std::vector<KSlab> slabs;
    const bf16* w = nullptr; int ktot = 0; int cout = 0;
    int OH = 0, OW = 0;
    const float* bias = nullptr; const float* bias2 = nullptr; int bias2_stride = 0;
    const float* resid = nullptr;
    Act out;
    bf16* raw_out = nullptr;          // also store bf16(out) (input of a following Down / Upsample conv): no separate cast pass
    bool custom_os = false; OutSpec os{};   // output addressing other than plain NHWC (phase of a folded upsample conv)
    int nz = 1, b_zrows = 0, z_phase = 0; long long z_off_hi = 0, z_off_lo = 0;   // the four phases of a folded upsample conv in ONE launch
    int c0 = 0, c1 = 0;               // channels of the A sources (precise mode: where their low halves start)
};

// Tile-kernel descriptor of an image conv over B images whose tiles cover Bt >= B images (conv_geometry); PW = 2 in precise mode
// ([hi | lo] operand pairs).  The engine's layer builders and the stand-alone test hook both go through here.
GemmDesc conv_desc(const ConvArgs& c, int B, int Bt, int PW) {
    GemmDesc d;
    d.n_a = c.n_a; d.a[0] = c.a[0]; d.a[1] = c.a[1];
    d.slabs = c.slabs;
    REQUIRE(PW == 1 || c.c0 > 0, "precise mode: conv without source channel counts");
    // the bf16 store addresses plain NHWC rows: it has no phase offsets (z_off_*) and no custom output map
    REQUIRE(!(c.raw_out && c.custom_os), "a bf16 copy of a phase-addressed (folded upsample) output is not supported");
    if (PW == 2) set_precise_fields(d, c.c0, c.c1, c.ktot);
    conv_geometry(d, c.OW, c.OH, Bt, c.cout, c.resid != nullptr, c.nz);
    d.b_ptr = c.w; d.b_K = PW * c.ktot; d.b_rows = (long long)c.nz * (((c.cout + 127) / 128) * 128);      // weights are padded to 128 rows (new_weight)
    d.b_is_param = true;
    d.n_tiles = (c.cout + d.block_n - 1) / d.block_n; d.nz = c.nz; d.a_zstep = 0; d.b_zrows = c.b_zrows;
    d.z_phase = c.z_phase; d.z_off_hi = c.z_off_hi; d.z_off_lo = c.z_off_lo;
    d.OW = c.OW; d.OH = c.OH; d.OB = B; d.n_valid = c.cout;
    d.bias = c.bias; d.bias2 = c.bias2; d.bias2_stride = c.bias2_stride;
    d.resid = c.resid; d.rs = nhwc_out(c.OH, c.OW, c.cout);
    d.out_f32 = c.out.p; d.os = c.custom_os ? c.os : nhwc_out(c.OH, c.OW, c.cout);
    if (c.raw_out) { d.out_bf16 = c.raw_out; d.hs = nhwc_out(c.OH, c.OW, PW * c.cout); d.lo_out_off = PW == 2 ? c.cout : 0; }
    d.stats = c.out.stats; d.stats_C = c.cout; d.stats_coff = 0;
    return d;
}

// Upsample folded (nearest 2x -> conv3x3 on a Hl x Wl x C input, bf16 NHWC rows of PW * C at `raw`): output pixel (2i+py, 2j+px) only sees
// a 2x2 neighbourhood of the low-res input, with the 3x3 taps that alias onto the same low-res pixel summed into one weight
// (pack_entry type 5: exact in real arithmetic, 2.25x fewer MACs, no 4x-sized intermediate).  Fills the A source, K slabs and
// output addressing of one op that runs all four phases (gemm-batch z = 2 py + px = phase, weights of phase z start at row z * rows_pad),
// each phase writing its quarter of the NHWC output.  The slabs are those of phase 0; the kernel shifts them by (py, px) for the others.
// The caller sets weights, bias and output.
void fold_up_conv(ConvArgs& c, const bf16* raw, int Bp, int Hl, int Wl, int C, int PW) {
    c.n_a = 1; c.a[0] = nhwc_src(raw, Bp, Hl, Wl, C * PW); c.c0 = C;
    for (int a = 0; a < 2; ++a)
        for (int bb = 0; bb < 2; ++bb)
            for (int ch = 0; ch < C; ch += 64) {
                KSlab k; k.a_sel = 0; k.a_chan = ch; k.dh = a - 1; k.dw = bb - 1; k.p = 0; k.b_col = (a * 2 + bb) * C + ch;
                c.slabs.push_back(k);
            }
    c.ktot = 4 * C; c.cout = C; c.OH = Hl; c.OW = Wl;
    c.custom_os = true;
    c.os.sZ = 0; c.os.sB = 4LL * Hl * Wl * C; c.os.sH = 4LL * Wl * C; c.os.sW = 2LL * C; c.os.off = 0;
    c.nz = 4; c.b_zrows = ((C + 127) / 128) * 128; c.z_phase = 1; c.z_off_hi = 2LL * Wl * C; c.z_off_lo = C;
}

// ---- weight gradient (wgrad_kernel + wgrad_reduce_kernel), shared by the training plan and the stand-alone test hook
std::vector<WgradTap> taps_3x3() {
    std::vector<WgradTap> t;
    for (int r = 0; r < 3; ++r) for (int s = 0; s < 3; ++s) t.push_back({0, s - 1, 0, r - 1});
    return t;
}
std::vector<WgradTap> taps_1x1() { return {{0, 0, 0, 0}}; }
// stride-2 conv: input pixel (2 oh + r - 1, 2 ow + s - 1) in the (2C, W/2, 2, H/2, B) parity view (see add_conv_slabs)
std::vector<WgradTap> taps_3x3_stride2(int C) {
    std::vector<WgradTap> t;
    for (int r = 0; r < 3; ++r) for (int s = 0; s < 3; ++s) t.push_back({(s == 1) ? 0 : C, (s == 0) ? -1 : 0, (r == 1) ? 0 : 1, (r == 0) ? -1 : 0});
    return t;
}

// WgradOut: instead of a parameter gradient, every one of `nb` batches (one slice each, no reduction) writes its own [CY][Cin] result at
// ptr + batch * slice_stride + row * row_stride + col: the attention backward's dV = P^T dO and dK = dS^T Q (contractions over the query index)
struct WgradOut { float* ptr = nullptr; long long slice_stride = 0, row_stride = 0; int nb = 0; };

// Grid of the weight gradient of one conv: x = (co_pad / 128) * (Cin / 64) output tiles, y = groups of <= 3 taps, z = slices of the
// nbatch * (OH/8) * (OW/8) pixel patches.  slices = 0: the default (one wave of CTAs); raw: one slice per batch.
// A 4x4 image is one patch: its other 48 pixels lie outside dY and load as zeros, so they add nothing.
struct WgradShape { int co_pad = 0, tpc = 0, nx = 0, ny = 0, patches = 0, slices = 0; };
int wgrad_grid(int extent) { return extent == 4 ? 8 : extent; }      // pixels of the patch grid along one side
WgradShape wgrad_shape(int CY, int OHh, int OWw, int nbatch, int Cin, int ntaps, int slices, const WgradOut* raw) {
    OHh = wgrad_grid(OHh); OWw = wgrad_grid(OWw);
    REQUIRE(OHh % 8 == 0 && OWw % 8 == 0 && Cin % 64 == 0 && CY % 64 == 0, "wgrad geometry %dx%d Cin=%d CY=%d", OHh, OWw, Cin, CY);
    REQUIRE(ntaps >= 1 && ntaps <= WGRAD_MAX_TAPS, "too many taps");
    WgradShape s;
    s.co_pad = ((CY + 127) / 128) * 128;
    s.tpc = ntaps < 3 ? ntaps : 3;
    s.ny = (ntaps + s.tpc - 1) / s.tpc;
    s.nx = (s.co_pad / 128) * (Cin / 64);
    s.patches = nbatch * (OHh / 8) * (OWw / 8);
    if (raw) {
        s.slices = raw->nb;
    } else if (slices > 0) {
        REQUIRE(slices <= s.patches, "%d slices of %d patches", slices, s.patches);
        s.slices = slices;
    } else {
        // one wave of CTAs: a CTA's fixed cost (pipeline fill, 96 KB partial tile out) is as long as ~10 K steps of its main loop,
        // and every extra slice is another partial tile for the reduction kernel to read
        const int nxy = s.nx * s.ny;
        s.slices = (num_sms() + nxy / 2) / nxy;
        if (s.slices > s.patches / 2) s.slices = s.patches / 2;
        if (s.slices < 1) s.slices = 1;
    }
    return s;
}
// dW[co][tap][ci] = sum_p dY[p][co] X[p + tap][ci] as partial tiles ws[slice][co][tap][ci].  dy: bf16 [nmap][OH][OW][CY] (nmap >= the
// batches the patches cover); xs: the X view the taps index (nhwc_src / nhwc_stride2_src)
WgradParams wgrad_params(const WgradShape& s, const bf16* dy, int CY, int OHh, int OWw, int nmap, int nbatch, const ASrc& xs, int Cin,
                         const std::vector<WgradTap>& taps, int cout_valid, float* ws, const WgradOut* raw) {
    WgradParams p; memset(&p, 0, sizeof(p));
    const int ntaps = (int)taps.size();
    {
        const uint64_t dims[5] = {(uint64_t)CY, (uint64_t)OWw, 1ull, (uint64_t)OHh, (uint64_t)nmap};
        const uint64_t str[4] = {2ull * CY, 2ull * OWw * CY, 2ull * OWw * CY, 2ull * OHh * OWw * CY};
        const uint32_t box[5] = {64u, 8u, 1u, 8u, 1u};
        p.dy_map = encode_map(5, dy, dims, str, box);
    }
    {
        const uint64_t dims[5] = {(uint64_t)xs.C, (uint64_t)xs.W, (uint64_t)xs.P, (uint64_t)xs.H, (uint64_t)xs.Bn};
        const uint64_t str[4] = {(uint64_t)xs.sW, (uint64_t)xs.sP, (uint64_t)xs.sH, (uint64_t)xs.sB};
        const uint32_t box[5] = {64u, 8u, 1u, 8u, 1u};
        p.x_map = encode_map(5, xs.ptr, dims, str, box);
    }
    p.ws = ws; p.Cin = Cin; p.co_pad = s.co_pad; p.cout_valid = cout_valid;
    p.ws_slice_stride = raw ? raw->slice_stride : (long long)s.co_pad * ntaps * Cin; p.ws_row_stride = raw ? raw->row_stride : (long long)ntaps * Cin;
    p.OH = wgrad_grid(OHh); p.OW = wgrad_grid(OWw); p.B = nbatch; p.ntaps = ntaps; p.taps_per_cta = s.tpc; p.patches = s.patches; p.slices = s.slices;
    for (int i = 0; i < ntaps; ++i) p.taps[i] = taps[i];
    return p;
}
// slice reduction into the OIHW gradient [cout_valid][cin_valid][taps] (block range and destination are set where the launch is batched)
WgradReduceDesc wgrad_reduce_desc(const WgradShape& s, const float* ws, int ntaps, int Cin, int cout_valid, int cin_valid) {
    const int sw = s.slices >= 8 ? 8 : (s.slices >= 4 ? 4 : (s.slices >= 2 ? 2 : 1));
    const int ci_per_block = 32 * (8 / sw);
    WgradReduceDesc rd{}; rd.ws = ws; rd.grad = nullptr; rd.slices = s.slices; rd.co_pad = s.co_pad; rd.ntaps = ntaps; rd.Cin = Cin; rd.cout_valid = cout_valid;
    rd.cin_valid = cin_valid; rd.sw = sw; rd.blocks_x = (cin_valid + ci_per_block - 1) / ci_per_block;
    return rd;
}
// one packed copy (pack_entry) as its own launch: loading a single parameter, sr3_test_conv_ex
void pack_one(const PackDesc& d, cudaStream_t st) {
    pack_one_kernel<<<pack_entry_blocks(d), 256, 0, st>>>(d);
    CK(cudaGetLastError());
}
void init_wgrad_attrs() {
    static std::vector<int> seen;
    if (first_use_on_device(seen)) CK(cudaFuncSetAttribute(wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WGRAD_SMEM_BYTES));
}

// ---- GroupNorm / elementwise launches of the plan, shared by the layer builders and the stand-alone test hooks.  Every thread owns one
// 4-channel column and walks the pixels of its block kpix at a time; grid = (blocks per image, images).
struct RowLaunch { int threads = 0, ppb = 0, smem = 0; dim3 grid; };
// the GroupNorm op a = act(GN(cat(src0, src1))) as prep_kernel and gn_bwd_kernel both see it (no outputs, launch shape or dropout yet)
PrepParams gn_op(const float* src0, const double* st0, int C0, const float* src1, const double* st1, int C1, const float* gamma, const float* beta,
                 int groups, int HW, bool silu) {
    PrepParams p{};
    p.src0 = src0; p.st0 = st0; p.C0 = C0;
    p.src1 = src1; p.st1 = st1; p.C1 = C1;
    p.gamma = gamma; p.beta = beta; p.groups = groups; p.HW = HW; p.silu = silu ? 1 : 0; p.eps = 1e-5f;
    const int C = C0 + C1;
    REQUIRE(C % groups == 0 && C % 4 == 0 && C0 % 4 == 0, "bad GroupNorm geometry C=%d groups=%d", C, groups);
    REQUIRE(C / 4 <= 512, "GroupNorm over %d channels is not supported", C);
    return p;
}
// prep_kernel: ONE wave of blocks.  The kernel uses 64 registers per thread, i.e. 4 resident 256-thread blocks (2 of 512) per SM; a grid
// sized for 8 per SM (round 1, 32-register version) runs as two waves and pays the statistics set-up twice (24 vs 15 us on the 128x128 level).
RowLaunch prep_launch(int C, int groups, int HW, int B) {
    const int vpp = C / 4;
    const int kpix = vpp >= 256 ? 1 : 256 / vpp;
    RowLaunch L; L.threads = vpp * kpix;                         // <= 512, every thread owns one 4-channel column
    const int per_sm = L.threads > 256 ? 2 : 4;
    int bpi = per_sm * num_sms() / B; if (bpi < 1) bpi = 1;    // blocks per image
    const int q = kpix * 4;                                    // 4 loads in flight per thread
    int ppb = (HW + bpi - 1) / bpi;
    ppb = ((ppb + q - 1) / q) * q;
    if (ppb < q) ppb = q;
    if (ppb > HW) ppb = HW;
    L.ppb = ppb; L.grid = dim3((HW + ppb - 1) / ppb, B); L.smem = (2 * C + 2 * groups) * sizeof(float);
    return L;
}
void launch_prep(const PrepParams& p, const RowLaunch& L, cudaStream_t st) {
    if (p.drop) launch_k(prep_kernel<true>, L.grid, dim3(L.threads), (size_t)L.smem, st, p);
    else launch_k(prep_kernel<false>, L.grid, dim3(L.threads), (size_t)L.smem, st, p);
}
// gn_bwd_kernel, measured (8 images, 16->128): 64 pixel rows per thread column and ~4 blocks per SM beat 32 / 8 (2.67 -> 2.53 ms) and
// 128 / 2 (3.06 ms)
RowLaunch gn_bwd_launch(int C, int groups, int HW, int B) {
    const int vpp = C / 4;
    const int kpix = vpp >= 256 ? 1 : 256 / vpp;
    RowLaunch L; L.threads = vpp * kpix;
    int ppb = kpix * 64;
    { const int cap = (int)(((long long)HW * B) / 592); if (ppb > cap) ppb = cap; }
    if (ppb < kpix * 4) ppb = kpix * 4;
    if (ppb > HW) ppb = HW;
    L.ppb = ppb; L.grid = dim3((HW + ppb - 1) / ppb, B); L.smem = gn_bwd_smem_bytes(C, groups);
    return L;
}
// both passes; p.sums must be zero
void launch_gn_bwd(const GnBwdParams& p, const RowLaunch& L, cudaStream_t st) {
    launch_k(gn_bwd_kernel<false>, L.grid, dim3(L.threads), (size_t)L.smem, st, p);
    launch_k(gn_bwd_kernel<true>, L.grid, dim3(L.threads), (size_t)L.smem, st, p);
}
RowLaunch combine_launch(int C, int HW, int B) {
    const int vpp = C / 4;
    REQUIRE(C % 4 == 0 && vpp <= 256, "combine over %d channels", C);
    const int kpix = 256 / vpp;
    RowLaunch L; L.threads = vpp * kpix;
    int ppb = kpix * 32;
    { const int cap = (int)(((long long)HW * B) / 1184); if (ppb > cap) ppb = cap; }
    if (ppb < kpix) ppb = kpix;
    if (ppb > HW) ppb = HW;
    L.ppb = ppb; L.grid = dim3((HW + ppb - 1) / ppb, B); L.smem = C * 4;
    return L;
}
void launch_combine(const RowLaunch& L, const float* a, const float* b2, float* dst, int acc, bf16* dst_b, float* gsum, int B, int HW, int C, cudaStream_t st) {
    launch_k(grad_combine_kernel, L.grid, dim3(L.threads), (size_t)L.smem, st, a, b2, dst, acc, dst_b, gsum, B, HW, C, L.ppb);
}
void launch_bias_grad(const float* gsum, int ld, float* d0, float* d1, int B, int C, float gscale, cudaStream_t st) {
    bias_grad_kernel<<<(C + 255) / 256, 256, 0, st>>>(gsum, ld, d0, d1, B, C, gscale);
    CK(cudaGetLastError());
}
void launch_loss_grad(const float* noise, const float* eps, int B, int C, int H, int W, int l2, double* loss, bf16* deps, int ld, float* bias_sum,
                      cudaStream_t st) {
    loss_grad_kernel<<<296, 256, 0, st>>>(noise, eps, B, C, H, W, l2, loss, deps, ld, bias_sum);
    CK(cudaGetLastError());
}
// the upstream gradient of UNet.forward in place of the loss gradient (same operand, same launch shape); bias_sum must be zero
void launch_grad_load(const float* g, int B, int C, int H, int W, bf16* deps, int ld, float* bias_sum, cudaStream_t st) {
    grad_load_kernel<<<296, 256, 0, st>>>(g, B, C, H, W, deps, ld, bias_sum);
    CK(cudaGetLastError());
}
// dx NCHW [B][C][H][W] from the first conv's fp32 NHWC data gradient (ld channels per pixel)
void launch_input_grad_store(const float* src, int B, int C, int H, int W, int ld, float* dst, cudaStream_t st) {
    const long long total = 1LL * B * C * H * W;
    input_grad_store_kernel<<<(int)std::min<long long>((total + 255) / 256, num_sms() * 8LL), 256, 0, st>>>(src, B, C, H, W, ld, dst);
    CK(cudaGetLastError());
}

// ---- noise-level embedding + FiLM projections forward (the plan's first two launches; sr3_test_film_embed_fwd)
constexpr int FILM_SMEM_BYTES = 48 * 1024;      // film_kernel stays within the default dynamic shared-memory limit (no opt-in)
// images of tau film_kernel stages at once next to its 64 weight rows; larger batches are walked in chunks of this many
int film_tau_chunk(int inner, int B) {
    const int cap = (FILM_SMEM_BYTES / 4 - 64 * (inner + 1)) / inner;
    REQUIRE(cap >= 1, "FiLM projections: inner_channel %d does not fit film_kernel's %d KB of shared memory", inner, FILM_SMEM_BYTES / 1024);
    return std::min(B, cap);
}
void launch_embed(const EmbedParams& ep, int B, cudaStream_t st) {
    launch_k(embed_kernel, dim3(B), dim3(256), (size_t)(5 * ep.inner * 4), st, ep);
}
void launch_film(const float* wf, const float* bf, const float* cb, const float* tau, float* film, int F, int inner, int B, cudaStream_t st) {
    const int chunk = film_tau_chunk(inner, B);
    launch_k(film_kernel, dim3((F + 63) / 64), dim3(256), (size_t)((64 * (inner + 1) + chunk * inner) * 4), st, wf, bf, cb, tau, film, F, inner, B,
             chunk);
}

// ---- FiLM projections + noise-level MLP backward: one block's shared memory holds every image's embedding (and the MLP's hidden layer)
constexpr int FILM_BWD_SMEM_MAX = 200 * 1024;
int film_bwd_smem(int B, int inner) { return 2 * B * inner * 4; }
int embed_bwd_smem(int B, int inner) { return (2 * B * inner + 2 * B * 4 * inner) * 4; }
// dtau must be zero
void launch_film_bwd(const float* wf, const float* tau, const float* dfilm, float* dwf, float* dbf, float* dcb, float* dtau, int F, int inner, int B,
                     float gscale, cudaStream_t st) {
    const int smem = film_bwd_smem(B, inner);
    static std::vector<int> seen;
    if (first_use_on_device(seen)) CK(cudaFuncSetAttribute(film_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FILM_BWD_SMEM_MAX));
    REQUIRE(smem <= FILM_BWD_SMEM_MAX, "FiLM backward: batch %d too large for one block's shared memory", B);
    film_bwd_kernel<<<(F + 63) / 64, 256, smem, st>>>(wf, tau, dfilm, dwf, dbf, dcb, dtau, F, inner, B, gscale);
    CK(cudaGetLastError());
}
void launch_embed_bwd(const float* nl, const float* w1, const float* b1, const float* w2, const float* dtau, float* dw1, float* db1, float* dw2, float* db2,
                      int inner, int B, float gscale, cudaStream_t st) {
    const int esm = embed_bwd_smem(B, inner);
    static std::vector<int> seen;
    if (first_use_on_device(seen)) CK(cudaFuncSetAttribute(embed_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FILM_BWD_SMEM_MAX));
    REQUIRE(esm <= FILM_BWD_SMEM_MAX, "noise-level MLP backward: batch %d too large for one block", B);
    embed_bwd_kernel<<<1, 256, esm, st>>>(nl, w1, b1, w2, dtau, dw1, db1, dw2, db2, inner, B, gscale);
    CK(cudaGetLastError());
}
void launch_noise_level_bwd(const float* nl, const float* w1, const float* b1, const float* w2, const float* dtau, float* dnl, int inner, int B,
                            cudaStream_t st) {
    const int esm = embed_bwd_smem(B, inner);
    static std::vector<int> seen;
    if (first_use_on_device(seen)) CK(cudaFuncSetAttribute(noise_level_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FILM_BWD_SMEM_MAX));
    REQUIRE(esm <= FILM_BWD_SMEM_MAX, "noise-level backward: batch %d too large for one block", B);
    noise_level_bwd_kernel<<<1, 256, esm, st>>>(nl, w1, b1, w2, dtau, dnl, inner, B);
    CK(cudaGetLastError());
}

// ---- data gradients on the forward tile kernel
// the packed weight of a data gradient (pack_entry types 2, 3, 4; the source parameter is filled in when it is packed):
//   2: stride-1 conv, Cout -> Cin, k x k: rows Cin, k*k*cout_pad columns (mirrored taps, cout_pad = Cout rounded up to 64)
//   3: Downsample, C -> C: four phase matrices of rows_pad rows x 4C columns
//   4: Upsample, C -> C: rows C, 16C columns (the 4x4 kernel)
PackDesc dgrad_pack_desc(int type, void* dst, int Cout, int Cin, int k) {
    PackDesc d{}; d.type = type; d.dst = dst; d.Cout = Cout; d.Cin = Cin;
    if (type == 2) {
        const int cout_pad = ((Cout + 63) / 64) * 64;
        d.k = k; d.ld = k * k * cout_pad; d.tap_stride = cout_pad;
    } else if (type == 3) {
        d.rows_pad = ((Cin + 127) / 128) * 128;
    }
    return d;
}
// bf16 elements of the packed weight of dgrad_pack_desc (rows padded to 128)
size_t dgrad_weight_elems(int type, int Cout, int Cin, int k) {
    const size_t rows_pad = ((Cin + 127) / 128) * 128;
    if (type == 2) return rows_pad * k * k * (((Cout + 63) / 64) * 64);
    if (type == 3) return 4 * rows_pad * 4 * Cin;
    return rows_pad * 16 * Cin;
}
// dX = conv_k(dY, W') of a stride-1 conv: A bf16 [Bp][H][W][CA] (CA: dY channels, >= Cout: the final conv reads 3 of 64); out fp32 [Bp][H][W][N]
ConvArgs dgrad_conv(const bf16* A, int Bp, int CA, int Hh, int Ww, int k, const bf16* w, int N, float* out, bf16* out_b) {
    ConvArgs c; c.n_a = 1; c.a[0] = nhwc_src(A, Bp, Hh, Ww, CA); c.c0 = CA;
    add_conv_slabs(c.slabs, 0, CA, k, 1, 0);
    c.w = w; c.ktot = k * k * CA; c.cout = N; c.OH = Hh; c.OW = Ww;
    Act o; o.p = out; o.C = N; o.H = Hh; o.W = Ww; c.out = o;
    c.raw_out = out_b;
    return c;
}
// the data gradient of the first conv (unet.py:193, in_channel -> inner, 3x3): dy = its output gradient, bf16 [Bp][H][W][inner], w = the
// type-2 packed weight (rows = in_channel, zero up to 128) -> out fp32 [Bp][H][W][64].  The output channels are padded to the 64 of the
// input buffer, as the final conv's 3 channels are in its 64-channel gradient operand; channels >= in_channel come out zero.
constexpr int INPUT_GRAD_LD = 64;
ConvArgs input_dgrad_conv(const bf16* dy, int Bp, int Hh, int Ww, int inner, const bf16* w, float* out) {
    return dgrad_conv(dy, Bp, inner, Hh, Ww, 3, w, INPUT_GRAD_LD, out, nullptr);
}
// Downsample (conv3x3 stride 2): four input-parity phases on the low-resolution dY grid (bf16 [Bp][yH][yW][C]) -> out fp32 [Bp][2yH][2yW][C]
ConvArgs downsample_dgrad_conv(const bf16* dy, int Bp, int yH, int yW, int C, const bf16* w, float* out) {
    ConvArgs c; c.n_a = 1; c.a[0] = nhwc_src(dy, Bp, yH, yW, C); c.c0 = C;
    for (int a = 0; a < 2; ++a)
        for (int bb = 0; bb < 2; ++bb)
            for (int ch = 0; ch < C; ch += 64) { KSlab k; k.a_sel = 0; k.a_chan = ch; k.dh = -1 + a; k.dw = -1 + bb; k.p = 0; k.b_col = (a * 2 + bb) * C + ch; c.slabs.push_back(k); }
    c.w = w; c.ktot = 4 * C; c.cout = C; c.OH = yH; c.OW = yW;
    Act o; o.p = out; o.C = C; o.H = yH; o.W = yW; c.out = o;
    c.custom_os = true;
    c.os.sZ = 0; c.os.sB = 4LL * yH * yW * C; c.os.sH = 4LL * yW * C; c.os.sW = 2LL * C; c.os.off = 0;
    c.nz = 4; c.b_zrows = ((C + 127) / 128) * 128; c.z_phase = 1; c.z_off_hi = 2LL * yW * C; c.z_off_lo = C;
    return c;
}
// Upsample (nearest 2x -> conv3x3): dX[i][j] = sum_{u,v} K[u][v] dY[2i-1+u][2j-1+v], a 4x4 stride-2 conv over dY (bf16 [Bp][yH][yW][C]) in
// the parity view -> out fp32 [Bp][yH/2][yW/2][C]
ConvArgs upsample_dgrad_conv(const bf16* dy, int Bp, int yH, int yW, int C, const bf16* w, float* out) {
    ConvArgs c; c.n_a = 1; c.a[0] = nhwc_stride2_src(dy, Bp, yH, yW, C); c.c0 = C;
    for (int u = 0; u < 4; ++u)
        for (int v = 0; v < 4; ++v)
            for (int ch = 0; ch < C; ch += 64) {
                KSlab k; k.a_sel = 0; k.b_col = (u * 4 + v) * C + ch;
                k.dh = (u == 0) ? -1 : (u == 3 ? 1 : 0); k.p = (u == 0 || u == 2) ? 1 : 0;
                k.dw = (v == 0) ? -1 : (v == 3 ? 1 : 0); k.a_chan = ((v == 0 || v == 2) ? C : 0) + ch;
                c.slabs.push_back(k);
            }
    c.w = w; c.ktot = 16 * C; c.cout = C; c.OH = yH / 2; c.OW = yW / 2;
    Act o; o.p = out; o.C = C; o.H = yH / 2; o.W = yW / 2; c.out = o;
    return c;
}

// ---- unfused attention forward (precise mode, training): nz batches of Lt tokens, HW
// tokens per image, head dim C; PW = 2 in precise mode (every bf16 row is [hi | lo])
// S[z] = q k^T / sqrt(C): qk bf16 [nz][Lt][2C PW] (rows [q_hi | k_hi | q_lo | k_lo]) -> S fp32 [nz][Lt][Lt]
GemmDesc attn_s_desc(const bf16* qk, float* S, int nz, int Lt, int C, int PW) {
    GemmDesc d; d.n_a = 1; d.a[0] = matrix_src(qk, nz, Lt, 2 * C * PW, 2 * C * PW, (long long)Lt * 2 * C * PW);
    for (int c = 0; c < C; c += 64) d.slabs.push_back({0, c, 0, 0, 0, C + c});
    if (PW == 2) set_precise_fields(d, 2 * C, 0, 2 * C);
    d.block_n = 128; d.b_ptr = qk; d.b_K = 2 * C * PW; d.b_rows = (long long)nz * Lt;
    d.w_box = 128; d.h_box = 1; d.b_box = 1; d.tiles_w = Lt / 128; d.tiles_h = 1; d.tiles_b = 1;
    d.n_tiles = Lt / 128; d.nz = nz; d.a_zstep = 1; d.b_zrows = Lt;
    d.OW = Lt; d.OH = 1; d.OB = nz; d.n_valid = Lt; d.scale = 1.0f / sqrtf((float)C);
    d.out_f32 = S; d.os = OutSpec{0, (long long)Lt * Lt, 0, Lt, 0};
    return d;
}
// P = softmax of each S row over the keys of its own image (segments of HW keys), bf16 [nz][Lt][Lt PW]
SoftmaxParams attn_softmax_params(const float* S, bf16* P, int nz, int Lt, int HW, int PW) {
    SoftmaxParams sp{}; sp.S = S; sp.P = P; sp.rows = (long long)nz * Lt; sp.L = Lt; sp.seg = HW; sp.precise = PW == 2 ? 1 : 0;
    return sp;
}
void launch_softmax(const SoftmaxParams& sp, cudaStream_t st) {
    launch_k(softmax_kernel, dim3((int)((sp.rows + 7) / 8)), dim3(256), 0, st, sp.S, sp.P, sp.rows, sp.L, sp.seg, sp.precise);
}
// O[z] = P v: rows = queries, N = head dim, K = keys.  vT bf16 [nz][C][Lt PW] -> O bf16 [nz][Lt][C PW]
GemmDesc attn_pv_desc(const bf16* P, const bf16* vT, bf16* O, int nz, int Lt, int C, int PW) {
    GemmDesc d; d.n_a = 1; d.a[0] = matrix_src(P, nz, Lt, Lt * PW, Lt * PW, (long long)Lt * Lt * PW);
    for (int c = 0; c < Lt; c += 64) d.slabs.push_back({0, c, 0, 0, 0, c});
    if (PW == 2) set_precise_fields(d, Lt, 0, Lt);
    d.block_n = 128; d.b_ptr = vT; d.b_K = Lt * PW; d.b_rows = (long long)nz * C;
    d.w_box = 128; d.h_box = 1; d.b_box = 1; d.tiles_w = Lt / 128; d.tiles_h = 1; d.tiles_b = 1;
    d.n_tiles = C / 128; d.nz = nz; d.a_zstep = 1; d.b_zrows = C;
    d.OW = Lt; d.OH = 1; d.OB = nz; d.n_valid = C;
    d.out_bf16 = O; d.hs = OutSpec{0, (long long)Lt * C * PW, 0, (long long)C * PW, 0}; d.lo_out_off = PW == 2 ? C : 0;
    return d;
}

// ---- attention backward: the four matrix products of nz attention batches of Lt tokens, head dim C
// dP[z] = dO V^T: rows = queries, N = keys, K = head dim.  dOb bf16 [nz][Lt][C], V bf16 [nz][Lt][C] -> dS fp32 [nz][Lt][Lt]
GemmDesc attn_bwd_dp_desc(const bf16* dOb, const bf16* v, float* dS, int nz, int Lt, int C) {
    GemmDesc d; d.n_a = 1; d.a[0] = matrix_src(dOb, nz, Lt, C, C, (long long)Lt * C);
    for (int ch = 0; ch < C; ch += 64) d.slabs.push_back({0, ch, 0, 0, 0, ch});
    d.block_n = 128; d.b_ptr = v; d.b_K = C; d.b_rows = (long long)nz * Lt;
    d.w_box = 128; d.h_box = 1; d.b_box = 1; d.tiles_w = Lt / 128; d.tiles_h = 1; d.tiles_b = 1;
    d.n_tiles = Lt / 128; d.nz = nz; d.a_zstep = 1; d.b_zrows = Lt;
    d.OW = Lt; d.OH = 1; d.OB = nz; d.n_valid = Lt;
    d.out_f32 = dS; d.os = OutSpec{0, (long long)Lt * Lt, 0, Lt, 0};
    return d;
}
// dQ[z] = dS K: rows = queries, N = head dim, K = keys.  dSb bf16 [nz][Lt][Lt], K^T bf16 [nz][C][Lt] -> dqkv[:, 0:C] (rows of 3C floats)
GemmDesc attn_bwd_dq_desc(const bf16* dSb, const bf16* kT, float* dqkv, int nz, int Lt, int C) {
    GemmDesc d; d.n_a = 1; d.a[0] = matrix_src(dSb, nz, Lt, Lt, Lt, (long long)Lt * Lt);
    for (int ch = 0; ch < Lt; ch += 64) d.slabs.push_back({0, ch, 0, 0, 0, ch});
    d.block_n = 128; d.b_ptr = kT; d.b_K = Lt; d.b_rows = (long long)nz * C;
    d.w_box = 128; d.h_box = 1; d.b_box = 1; d.tiles_w = Lt / 128; d.tiles_h = 1; d.tiles_b = 1;
    d.n_tiles = C / 128; d.nz = nz; d.a_zstep = 1; d.b_zrows = C;
    d.OW = Lt; d.OH = 1; d.OB = nz; d.n_valid = C;
    d.out_f32 = dqkv; d.os = OutSpec{0, (long long)Lt * 3 * C, 0, (long long)3 * C, 0};
    return d;
}
// dK = dS^T Q and dV = P^T dO contract over the QUERY index: the weight-gradient kernel's batched form with the tokens of an attention batch
// as a 16-wide "image" of 8x8 patches and the keys as its "output channels".  Q is read inside the q|k rows (2C wide) of qk.
ASrc attn_bwd_q_view(const bf16* qk, int nz, int Lt, int C) {
    ASrc q; q.ptr = qk; q.C = C; q.W = 16; q.P = 1; q.H = Lt / 16; q.Bn = nz;
    q.sW = 2LL * 2 * C; q.sP = 2LL * 16 * 2 * C; q.sH = 2LL * 16 * 2 * C; q.sB = 2LL * Lt * 2 * C;
    return q;
}
void launch_transpose_bf16(const bf16* src, bf16* dst, int R, int Cc, long long src_ld, long long src_z, long long dst_z, int nzb, cudaStream_t st) {
    launch_k(transpose_bf16_kernel, dim3((Cc + 31) / 32, (R + 31) / 32, nzb), dim3(256), 0, st, src, dst, R, Cc, src_ld, src_z, dst_z);
}
// vT[z][d][key] (the forward's) -> V[z][key][d]
void launch_v_from_vT(const bf16* vT, bf16* v, int nz, int Lt, int C, cudaStream_t st) {
    launch_transpose_bf16(vT, v, C, Lt, Lt, (long long)C * Lt, (long long)Lt * C, nz, st);
}
// K[z][key][d] inside the q|k rows -> K^T[z][d][key]
void launch_kT_from_qk(const bf16* qk, bf16* kT, int nz, int Lt, int C, cudaStream_t st) {
    launch_transpose_bf16(qk + C, kT, Lt, C, 2 * C, (long long)Lt * 2 * C, (long long)C * Lt, nz, st);
}
// dS = P * (dP - rowsum(P dP)) / sqrt(C) in place on dP = dS fp32 [nz][Lt][Lt], over the seg-token segments of each row; dSb = bf16(dS)
void launch_softmax_bwd(const bf16* P, float* dS, bf16* dSb, int nz, int Lt, int seg, int C, cudaStream_t st) {
    const long long rows = (long long)nz * Lt;
    launch_k(softmax_bwd_kernel, dim3((int)((rows + 7) / 8)), dim3(256), 0, st, P, dS, dSb, rows, Lt, seg, 1.0f / sqrtf((float)C));
}
void launch_cast_bf16(const float* src, bf16* dst, long long n4, cudaStream_t st) {
    launch_k(cast_bf16_kernel, dim3((int)std::min<long long>((n4 + 255) / 256, 2368)), dim3(256), 0, st, src, dst, n4);
}
// where such a product lands: columns [col, col + C) of the 3C-wide d(qkv) rows, one slice per attention batch
WgradOut attn_bwd_qkv_out(float* dqkv, int col, int nz, int Lt, int C) {
    WgradOut o; o.ptr = dqkv ? dqkv + col : nullptr; o.slice_stride = (long long)Lt * 3 * C; o.row_stride = 3LL * C; o.nb = nz;
    return o;
}

// Image sizes an inference plan runs on: at every UNet level (the image halved n_mults - 1 times) both sides are powers of two and at
// least 8, except that the lowest level may be exactly 4x4.  Returns the lowest level's side, or throws naming the size and the rule.
int check_image_size(int n_mults, int height, int width) {
    auto pow2 = [](int v) { return v > 0 && (v & (v - 1)) == 0; };
    const int lh = height >> (n_mults - 1), lw = width >> (n_mults - 1);
    REQUIRE(height > 0 && width > 0, "image size %dx%d: sides must be positive", height, width);
    REQUIRE(lh >= 4 && lw >= 4, "image size %dx%d: lowest UNet resolution %dx%d < 4 is not supported (%d levels)", height, width, lh, lw, n_mults);
    REQUIRE(pow2(height) && pow2(width), "image size %dx%d: both sides must be powers of two", height, width);
    REQUIRE((lh >= 8 && lw >= 8) || (lh == 4 && lw == 4),
            "image size %dx%d: lowest UNet level %dx%d is not supported (every level must be at least 8x8, or the lowest exactly 4x4)", height, width,
            lh, lw);
    return lh < lw ? lh : lw;
}

}  // namespace

struct sr3_engine {
    sr3_unet_config cfg{};
    // Bp: images allocated per activation.  Bt: images the tile-kernel launches cover (Bp, or B when Bp was padded to 8 for a 4x4 level:
    // the high-resolution layers then do not compute the padded images).
    int B = 0, Bp = 0, Bt = 0, dev = 0;
    int H = 0, W = 0, inner = 0, cond_c = 0, in_C = 64;
    bool precise = false; int PW = 1;       // precise mode: every bf16 operand tensor is PW = 2 times as wide ([hi | lo] per pixel / row)
    DevAllocs mem;
    std::vector<ParamEntry> params;
    std::map<std::string, int> pindex;
    std::vector<Op> ops;
    std::vector<GemmHandle> gemms;          // tile-kernel launches of the step, in order (for next-layer weight prefetch)
    // kind: 0 gemm, 1 groupnorm-apply, 2 cast/upsample, 3 softmax, 4 other, 5 fused attention core.  Tile ops also keep the variant they launch (sr3_tile_schedule):
    // geometry, schedule (0 cooperative, 1 ping-pong; -1 not a tile op) and output rows x columns x channels.
    struct OpInfo { int kind; double flops; double bytes; sr3_gemm_geometry geo; int schedule; int out_hwc[3]; };
    std::vector<OpInfo> op_info;
    std::map<std::string, Act> taps;
    std::map<std::string, size_t> role_max;
    std::map<std::string, void*> role_ptr;
    bool dry = true;
    size_t plan_bytes = 0;                  // sizing pass: the bytes the real pass allocates outside the shared scratch (role_max) and arenas
    // ---- training plan (sr3_engine_create_train): every scratch tensor of the forward is kept for the backward, which is recorded layer by
    // layer while the forward plan is built and replayed in reverse order
    bool train = false; float drop_p = 0.f;
    std::vector<Op>* bwd_sink = nullptr;                   // where push() records while a layer's backward is being described
    std::vector<int>* kind_sink = nullptr;                 // ... and the kinds of those ops
    std::vector<std::vector<Op>> bwd_blocks;               // one op list per forward layer, executed last to first
    std::vector<std::vector<int>> bwd_kinds;               // op kinds (profiling): 0 data-gradient tile kernel, 1 GroupNorm / elementwise, 4 other, 6 weight gradient, 7 attention GEMMs
    // the input gradient (data gradient of the first conv, then its NCHW store into dx_out): recorded with the backward, outside the blocks,
    // and run only when sr3_train_unet_backward is asked for dx
    std::vector<Op> dx_ops; std::vector<int> dx_kinds; float* dx_out = nullptr;
    // every packed copy of a parameter: one PackDesc, its source = parameter `pack_src[i]` (second source of a fused bias: `pack_src2[i]`).
    // sr3_engine_load_all_params binds the sources to the caller's tensors and packs the whole table in one launch (device table rebuilt
    // only when the parameter pointers change); sr3_engine_load_param packs the entries of one parameter, and sr3_engine_finalize_params
    // the fused biases, from the engine's own fp32 copies of their two parameters (the src / src2 registered with them).
    std::vector<PackDesc> pack_descs; std::vector<int> pack_src, pack_src2;
    PackDesc* pack_dev = nullptr; int* pack_ends_dev = nullptr; int pack_blocks = 0; std::vector<const float*> pack_last_ptrs;
    void add_pack(const std::string& pname, PackDesc d, const std::string& pname2 = "") {
        if (dry) return;
        pack_descs.push_back(d); pack_src.push_back(pindex.at(pname)); pack_src2.push_back(pname2.empty() ? -1 : pindex.at(pname2));
    }
    std::vector<float*> grad_dst;                          // per parameter (state_dict order): where the running backward writes its gradient
    float gscale = 1.f;                                    // d(total) / d(summed loss) of the running backward (1 / (b c h w), model.py:50-53)
    float* zero_arena = nullptr; size_t zero_cap = 0, zero_used = 0;    // everything the backward accumulates into (cleared at its start)
    DropSpec* drop_dev = nullptr; std::vector<DropSpec> drop_host; std::vector<std::string> drop_names;
    bf16* last_xraw = nullptr;
    bf16* deps_b = nullptr; float* fin_bias_sum = nullptr; float* dfilm = nullptr; float* dtau = nullptr;
    float *dwf_all = nullptr, *dbf_all = nullptr, *dcb_all = nullptr;
    float *hr_buf = nullptr;
    int loss_type_cur = 1;

    StepCtl* ctl_dev = nullptr;
    StepCtl ctl{};
    double* stats_arena = nullptr; size_t stats_cap = 0, stats_used = 0;
    bf16* in_buf = nullptr;
    float *x_state = nullptr, *eps_buf = nullptr, *mean_buf = nullptr, *noise_buf = nullptr, *nl_buf = nullptr, *io_a = nullptr, *io_b = nullptr;
    float *nl_table = nullptr, *post_tab = nullptr;
    int T = 0, T_cap = 0;
    std::vector<float> logvar_host;
    double* loss_dev = nullptr;
    float *tau = nullptr, *film = nullptr, *film_w = nullptr, *film_b = nullptr, *film_cb = nullptr;
    float *mlp_w1 = nullptr, *mlp_b1 = nullptr, *mlp_w2 = nullptr, *mlp_b2 = nullptr;
    int F = 0;
    cudaGraphExec_t graph = nullptr;
    cudaStream_t cap_stream = nullptr;
    cudaStream_t side_stream = nullptr;            // graph capture only: the noise-level embedding + FiLM projections run beside the first conv
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    int side_begin = -1, side_end = -1, side_join = -1;   // ops [side_begin, side_end) on the side branch, joined before op side_join
    uint64_t seed = 0, first_index = 0;
    bool have_cond = false;

    ~sr3_engine() {
        if (graph) cudaGraphExecDestroy(graph);
        if (cap_stream) cudaStreamDestroy(cap_stream);
        if (side_stream) cudaStreamDestroy(side_stream);
        if (ev_fork) cudaEventDestroy(ev_fork);
        if (ev_join) cudaEventDestroy(ev_join);
    }

    // ---- buffers shared between layers of the same role (stream order makes reuse safe)
    void* role(const std::string& r, size_t bytes) {
        // training plan: forward scratch is read again by the backward -> one allocation per use ("g_*" = backward scratch stays shared)
        if (train && r.compare(0, 2, "g_") != 0) {
            if (dry) { plan_bytes += bytes; return reinterpret_cast<void*>(0x1000); }
            return mem.alloc(bytes);
        }
        if (dry) { size_t& m = role_max[r]; if (bytes > m) m = bytes; return reinterpret_cast<void*>(0x1000); }
        REQUIRE(role_ptr.count(r) && role_max[r] >= bytes, "role buffer %s too small", r.c_str());
        return role_ptr[r];
    }
    double* new_stats(int C) {
        const size_t n = (size_t)Bp * C * 2;
        if (dry) { stats_used += n; return nullptr; }
        REQUIRE(stats_used + n <= stats_cap, "stats arena overflow");
        double* p = stats_arena + stats_used;
        stats_used += n;
        return p;
    }
    Act new_act(int C, int Hh, int Ww, const std::string& tap_name = "") {
        Act a; a.C = C; a.H = Hh; a.W = Ww;
        a.stats = new_stats(C);
        if (train) a.gsum = new_zero((size_t)Bp * C);
        if (dry) plan_bytes += (size_t)Bp * Hh * Ww * C * (train ? 10 : 4);      // fp32 value (+ fp32 and bf16 gradient)
        if (!dry) {
            a.p = static_cast<float*>(mem.alloc((size_t)Bp * Hh * Ww * C * sizeof(float)));
            if (train) {
                a.g = static_cast<float*>(mem.alloc((size_t)Bp * Hh * Ww * C * sizeof(float)));
                a.gb = static_cast<bf16*>(mem.alloc((size_t)Bp * Hh * Ww * C * sizeof(bf16)));
            }
            if (!tap_name.empty()) taps[tap_name] = a;
        }
        return a;
    }
    // floats from the arena the backward clears before it starts (sums it accumulates into with atomics)
    float* new_zero(size_t n) {
        n = (n + 3) & ~size_t(3);
        if (dry) { zero_used += n; return nullptr; }
        REQUIRE(zero_used + n <= zero_cap, "zero arena overflow");
        float* p = zero_arena + zero_used;
        zero_used += n;
        return p;
    }
    void add_param(const std::string& name, std::vector<int64_t> shape) {
        if (dry) return;
        ParamEntry e; e.name = name; e.shape = shape; e.numel = 1;
        for (auto s : shape) e.numel *= s;
        pindex[name] = (int)params.size();
        params.push_back(std::move(e));
    }
    float* f32_param(const std::string& name, std::vector<int64_t> shape) {
        int64_t n = 1; for (auto s : shape) n *= s;
        if (dry) { plan_bytes += n * sizeof(float); return nullptr; }
        float* dst = static_cast<float*>(mem.alloc(n * sizeof(float)));
        f32_param_into(name, shape, dst);
        return dst;
    }
    // f32 parameter stored into a slice of a bigger array
    void f32_param_into(const std::string& name, std::vector<int64_t> shape, float* dst) {
        if (dry) return;
        add_param(name, shape);
        PackDesc d{}; d.type = 0; d.dst = dst; d.n = params.back().numel; add_pack(name, d);
    }
    // conv weight packed into rows [0,Cout) of a [rows_pad][ktot] bf16 matrix at column k_off
    void conv_weight_param(const std::string& name, bf16* dst, int Cout, int Cin, int k, int ktot, int k_off, int cin_pad) {
        if (dry) return;
        add_param(name, {Cout, Cin, k, k});
        PackDesc d{}; d.type = 1; d.dst = dst; d.Cout = Cout; d.Cin = Cin; d.k = k; d.ld = PW * ktot; d.k_off = k_off; d.tap_stride = cin_pad;
        d.lo_off = precise ? ktot : 0;
        add_pack(name, d);
    }
    bf16* new_weight(int rows, int ktot) {      // [rows_pad][PW * ktot]: precise mode appends the low halves of every row
        const int rows_pad = ((rows + 127) / 128) * 128;
        const size_t bytes = (size_t)rows_pad * PW * ktot * sizeof(bf16);
        if (dry) { plan_bytes += bytes; return nullptr; }
        return static_cast<bf16*>(mem.alloc(bytes));
    }
    // precise-mode fields of an image conv whose A sources have c0 (c1) channels and whose weight rows hold ktot (high) columns
    void set_precise(GemmDesc& d, int c0, int c1, int ktot) {
        if (precise) set_precise_fields(d, c0, c1, ktot);
    }
    void push(Op op, int kind = 4, double flops = 0, double bytes = 0) {
        if (dry) return;
        if (bwd_sink) { bwd_sink->push_back(std::move(op)); kind_sink->push_back(kind); return; }
        ops.push_back(std::move(op));
        op_info.push_back({kind, flops, bytes, sr3_gemm_geometry{}, -1, {0, 0, 0}});
    }
    // executed work of a gemm op: 2*M*N*K flops; bytes = A read once per tap set + B once + outputs
    void push_gemm(const GemmDesc& d) {
        const double M = (double)d.OW * d.OH * d.OB * (d.nz > 1 && d.a_zstep == 0 ? d.nz : 1);
        const double K = 64.0 * d.slabs.size() * (d.passes > 1 ? d.passes : 1);      // executed MACs (precise mode: three passes)
        const double N = d.n_valid;
        double bytes = N * K * 2;
        if (d.out_f32) bytes += M * N * 4;
        if (d.out_bf16) bytes += M * N * 2;
        if (d.resid) bytes += M * N * 4;
        double a_elems = 0;
        for (int i = 0; i < d.n_a; ++i) a_elems += (double)d.a[i].C * d.a[i].W * d.a[i].P * d.a[i].H * d.a[i].Bn;
        bytes += a_elems * 2;
        sr3_gemm_geometry geo{};
        int schedule = 0;
        push(make_gemm_op(d, mem, &geo, &schedule), 0, 2.0 * M * N * K, bytes);
        if (!dry && !bwd_sink) {
            OpInfo& info = op_info.back();
            info.geo = geo; info.schedule = schedule;
            // output rows x columns (a folded upsample's four phases land at twice the resolution) x channels
            info.out_hwc[0] = d.OH * (d.z_phase ? 2 : 1); info.out_hwc[1] = d.OW * (d.z_phase ? 2 : 1); info.out_hwc[2] = d.n_valid;
        }
    }

    // ---- layer builders -------------------------------------------------------------------------
    float* last_mr = nullptr;              // training plan: (mean, rstd) buffer written by the most recent add_prep, read by its backward
    void add_prep(const Act& s0, const Act* s1, const float* gamma, const float* beta, int groups, bool silu, bf16* out_a, bf16* out_raw, const DropSpec* drop = nullptr) {
        if (dry) return;
        PrepParams p = gn_op(s0.p, s0.stats, s0.C, s1 ? s1->p : nullptr, s1 ? s1->stats : nullptr, s1 ? s1->C : 0, gamma, beta, groups, s0.H * s0.W, silu);
        p.drop = drop;
        if (train) { last_mr = static_cast<float*>(mem.alloc((size_t)Bp * groups * 2 * sizeof(float))); p.save_mr = last_mr; }
        p.out_a = out_a; p.out_raw = out_raw; p.precise = precise ? 1 : 0;
        const int C = p.C0 + p.C1;
        const RowLaunch L = prep_launch(C, groups, p.HW, B);
        p.pix_per_block = L.ppb;
        push([p, L](cudaStream_t st) { launch_prep(p, L, st); }, 1, 0, (double)B * p.HW * C * (4.0 + 2.0 + (out_raw ? 2.0 : 0.0)));
    }
    void add_cast(const Act& s, bf16* dst, int up) {
        if (dry) return;
        const long long total = 1LL * B * s.H * up * s.W * up * (s.C / 4);
        const int blocks = (int)std::min<long long>((total + 255) / 256, num_sms() * 16LL);
        const float* src = s.p; const int Bn = B, Hh = s.H, Ww = s.W, C = s.C;
        push([=](cudaStream_t st) { launch_k(cast_kernel, dim3(blocks), dim3(256), 0, st, src, dst, Bn, Hh, Ww, C, up); }, 2, 0, (double)Bn * Hh * Ww * C * (4.0 + 2.0 * up * up));
    }

    void add_conv(const ConvArgs& c) {
        if (dry) return;
        push_gemm(conv_desc(c, B, Bt, PW));
    }

    // ResnetBlock (+ optional SelfAttention): reference unet.py:94-158
    Act add_res_block(const LayerSpec& L, const Act& x, const Act* skip, int& film_off, bf16* raw_out = nullptr, bool x_has_skip = false) {
        const int cin = x.C + (skip ? skip->C : 0), cout = L.cout, Hh = x.H, Ww = x.W, G = cfg.norm_groups;
        REQUIRE(cin == L.cin, "%s: cin mismatch %d vs %d", L.name.c_str(), cin, L.cin);
        const std::string p = L.name + ".res_block";
        const bool has_res = cin != cout;
        // parameters in the reference's registration order
        const int foff = film_off; film_off += cout;
        f32_param_into(p + ".noise_func.noise_func.0.weight", {cout, inner}, dry ? nullptr : film_w + (size_t)foff * inner);
        f32_param_into(p + ".noise_func.noise_func.0.bias", {cout}, dry ? nullptr : film_b + foff);
        float* g1 = f32_param(p + ".block1.block.0.weight", {cin});
        float* b1 = f32_param(p + ".block1.block.0.bias", {cin});
        bf16* w1 = new_weight(cout, 9 * cin);
        conv_weight_param(p + ".block1.block.3.weight", w1, cout, cin, 3, 9 * cin, 0, cin);
        f32_param_into(p + ".block1.block.3.bias", {cout}, dry ? nullptr : film_cb + foff);
        float* g2 = f32_param(p + ".block2.block.0.weight", {cout});
        float* b2 = f32_param(p + ".block2.block.0.bias", {cout});
        const int k2 = 9 * cout + (has_res ? cin : 0);
        bf16* w2 = new_weight(cout, k2);
        conv_weight_param(p + ".block2.block.3.weight", w2, cout, cout, 3, k2, 0, cout);
        float* cb2 = f32_param(p + ".block2.block.3.bias", {cout});
        float* bias_total = cb2;
        if (has_res) {
            conv_weight_param(p + ".res_conv.weight", w2, cout, cin, 1, k2, 9 * cout, cin);
            float* cbr = f32_param(p + ".res_conv.bias", {cout});
            if (!dry) {
                bias_total = static_cast<float*>(mem.alloc(cout * sizeof(float)));
                PackDesc d{}; d.type = 6; d.dst = bias_total; d.src = cb2; d.src2 = cbr; d.n = cout;
                add_pack(p + ".block2.block.3.bias", d, p + ".res_conv.bias");
            }
        }
        // scratch
        bf16* a1 = static_cast<bf16*>(role("a1", (size_t)Bp * Hh * Ww * cin * 2 * PW));
        bf16* raw = has_res ? static_cast<bf16*>(role("raw", (size_t)Bp * Hh * Ww * cin * 2 * PW)) : nullptr;
        bf16* a2 = static_cast<bf16*>(role("a2", (size_t)Bp * Hh * Ww * cout * 2 * PW));
        Act h; h.C = cout; h.H = Hh; h.W = Ww; h.stats = new_stats(cout);
        h.p = static_cast<float*>(role("h", (size_t)Bp * Hh * Ww * cout * 4));
        Act y = new_act(cout, Hh, Ww, L.attn ? "" : L.name);

        add_prep(x, skip, g1, b1, G, true, a1, raw);
        float* mr1 = last_mr;
        {
            ConvArgs c; c.n_a = 1; c.a[0] = nhwc_src(a1, Bp, Hh, Ww, cin * PW); c.c0 = cin;
            add_conv_slabs(c.slabs, 0, cin, 3, 1, 0);
            c.w = w1; c.ktot = 9 * cin; c.cout = cout; c.OH = Hh; c.OW = Ww;
            c.bias2 = dry ? nullptr : film + foff; c.bias2_stride = F;
            c.out = h;
            add_conv(c);
        }
        const DropSpec* drop = nullptr;
        if (train && drop_p > 0.f) {          // Dropout sits in block2 only (unet.py:100-101)
            if (!dry) {
                REQUIRE(drop_host.size() < 256, "too many dropout layers");
                DropSpec ds{}; ds.mask = nullptr; ds.p = drop_p; ds.layer = (unsigned)drop_host.size(); ds.seed = 0;
                drop = drop_dev + drop_host.size();
                drop_host.push_back(ds); drop_names.push_back(p + ".block2");
            }
        }
        add_prep(h, nullptr, g2, b2, G, true, a2, nullptr, drop);
        float* mr2 = last_mr;
        {
            ConvArgs c; c.n_a = has_res ? 2 : 1; c.a[0] = nhwc_src(a2, Bp, Hh, Ww, cout * PW); c.c0 = cout;
            add_conv_slabs(c.slabs, 0, cout, 3, 1, 0);
            if (has_res) { c.a[1] = nhwc_src(raw, Bp, Hh, Ww, cin * PW); c.c1 = cin; add_conv_slabs(c.slabs, 1, cin, 1, 1, 9 * cout); }
            c.w = w2; c.ktot = k2; c.cout = cout; c.OH = Hh; c.OW = Ww;
            c.bias = bias_total; c.resid = has_res ? nullptr : x.p;
            c.out = y;
            if (!L.attn) c.raw_out = raw_out;
            add_conv(c);
        }
        if (train) {
            if (!dry) film_slices.push_back({foff, cout, pid(p + ".noise_func.noise_func.0.weight"), pid(p + ".noise_func.noise_func.0.bias"), pid(p + ".block1.block.3.bias")});
            ResBwdCtx c; c.p = p; c.x = x; c.skip = skip; c.h = h; c.y = y; c.cin = cin; c.cout = cout; c.Hh = Hh; c.Ww = Ww; c.foff = foff;
            c.has_res = has_res; c.x_acc = x_has_skip; c.a1 = a1; c.raw = raw; c.a2 = a2; c.g1 = g1; c.b1 = b1; c.g2 = g2; c.b2 = b2; c.drop = drop; c.mr1 = mr1; c.mr2 = mr2;
            bwd_res_block(c);
        }
        return L.attn ? add_attention(L, y, raw_out) : y;      // (its backward is recorded after the block's: it runs first)
    }

    // SelfAttention (reference unet.py:113-142): GN -> qkv 1x1 (no bias) -> softmax(q k^T / sqrt(C)) v -> out 1x1 + bias + x
    Act add_attention(const LayerSpec& L, const Act& x, bf16* raw_out = nullptr) {
        const int C = x.C, Hh = x.H, Ww = x.W, HW = Hh * Ww, G = cfg.norm_groups;
        const std::string p = L.name + ".attn";
        const int Lt = HW >= 128 ? HW : 128;            // tokens per attention batch (two 8x8 or eight 4x4 images share one)
        const int per = Lt / HW;                         // images per attention batch
        REQUIRE(Lt % 128 == 0 && (Bp % per) == 0, "attention geometry HW=%d", HW);
        REQUIRE(C % 128 == 0, "%s: self-attention over %d channels is not supported (the q/k/v and P.v tiles are 128 columns wide; C must be a multiple of 128)", L.name.c_str(), C);
        const int nz = (Bt + per - 1) / per;
        float* gn_w = f32_param(p + ".norm.weight", {C});
        float* gn_b = f32_param(p + ".norm.bias", {C});
        bf16* wqkv = new_weight(3 * C, C);
        conv_weight_param(p + ".qkv.weight", wqkv, 3 * C, C, 1, C, 0, C);
        bf16* wout = new_weight(C, C);
        conv_weight_param(p + ".out.weight", wout, C, C, 1, C, 0, C);
        float* bout = f32_param(p + ".out.bias", {C});
        bf16* n = static_cast<bf16*>(role("a1", (size_t)Bp * HW * C * 2 * PW));
        bf16* qk = static_cast<bf16*>(role("qk", (size_t)Bp * HW * 2 * C * 2 * PW));
        bf16* vT = static_cast<bf16*>(role("vT", (size_t)nz * C * Lt * 2 * PW));
        const bool fused = attn_fusable(Lt, C) && !precise && !train;      // one launch; S and P then never exist in device memory
        float* S = fused ? nullptr : static_cast<float*>(role("S", (size_t)nz * Lt * Lt * 4));
        bf16* P = fused ? nullptr : static_cast<bf16*>(role("P", (size_t)nz * Lt * Lt * 2 * PW));
        bf16* O = static_cast<bf16*>(role("O", (size_t)Bp * HW * C * 2 * PW));
        Act y = new_act(C, Hh, Ww, L.name);
        add_prep(x, nullptr, gn_w, gn_b, G, false, n, nullptr);
        float* mr_attn = last_mr;
        if (dry) {
            if (train) { AttnBwdCtx c; c.p = p; c.x = x; c.y = y; c.C = C; c.Hh = Hh; c.Ww = Ww; c.Lt = Lt; c.per = per; c.nz = nz; c.n = n; c.qk = qk; c.vT = vT; c.P = P; c.O = O; c.gn_w = gn_w; c.gn_b = gn_b; c.mr = mr_attn; bwd_attention(c); }
            return y;
        }
        {   // q,k,v = Wqkv n : [Bp*HW tokens] x [3C]; the v columns (whole 128-column tiles: C % 128 == 0) are stored transposed as vT[z][d][token]
            GemmDesc d; d.n_a = 1; d.a[0] = nhwc_src(n, Bp, Hh, Ww, C * PW);
            add_conv_slabs(d.slabs, 0, C, 1, 1, 0);
            set_precise(d, C, 0, C);
            const int ncol = 3 * C;
            d.block_n = 128; d.b_ptr = wqkv; d.b_K = C * PW; d.b_rows = ncol; d.b_is_param = true;
            pick_image_box(Ww, Hh, d.w_box, d.h_box, d.b_box);
            d.tiles_w = Ww / d.w_box; d.tiles_h = (Hh + d.h_box - 1) / d.h_box; d.tiles_b = (Bt + d.b_box - 1) / d.b_box; d.n_tiles = ncol / 128;
            d.OW = Ww; d.OH = Hh; d.OB = Bp; d.n_valid = ncol;
            d.out_bf16 = qk; d.hs = nhwc_out(Hh, Ww, 2 * C * PW); d.lo_out_off = precise ? 2 * C : 0;      // rows [q_hi | k_hi | q_lo | k_lo]
            d.out_t = vT; d.t_col0 = 2 * C; d.t_rows = C; d.t_ld = Lt * PW; d.t_per = per; d.lo_t_off = precise ? Lt : 0;
            d.pingpong = pingpong_knob() == 1 ? 1 : 0;         // (fixed 128x128 shape: the byte model is not consulted)
            push_gemm(d);
        }
        if (fused) {
            // S = q k^T / sqrt(C), softmax over the keys of the same image, O = P v: one launch (attn_wgmma.cuh, attn_long_wgmma.cuh)
            const double fl = 4.0 * nz * (double)Lt * Lt * C;
            push(make_attn_op(qk, vT, O, nz, Lt, HW, C), 5, fl, (double)nz * Lt * C * 2 * 4);
        } else {
            push_gemm(attn_s_desc(qk, S, nz, Lt, C, PW));
            const SoftmaxParams sp = attn_softmax_params(S, P, nz, Lt, HW, PW);
            push([=](cudaStream_t st) { launch_softmax(sp, st); }, 3, 0, (double)sp.rows * Lt * 6.0);
            push_gemm(attn_pv_desc(P, vT, O, nz, Lt, C, PW));
        }
        {   // out projection + bias + residual (un-normalised input)
            ConvArgs c; c.n_a = 1; c.a[0] = nhwc_src(O, Bp, Hh, Ww, C * PW); c.c0 = C;
            add_conv_slabs(c.slabs, 0, C, 1, 1, 0);
            c.w = wout; c.ktot = C; c.cout = C; c.OH = Hh; c.OW = Ww; c.bias = bout; c.resid = x.p; c.out = y; c.raw_out = raw_out;
            add_conv(c);
        }
        if (train) {
            AttnBwdCtx c; c.p = p; c.x = x; c.y = y; c.C = C; c.Hh = Hh; c.Ww = Ww; c.Lt = Lt; c.per = per; c.nz = nz; c.n = n; c.qk = qk; c.vT = vT; c.P = P; c.O = O;
            c.gn_w = gn_w; c.gn_b = gn_b; c.mr = mr_attn;
            bwd_attention(c);
        }
        return y;
    }

#include "train_plan.inc"

    void build_plan() {
        // topology: reference unet.py:186-231
        std::vector<LayerSpec> downs, mid, ups;
        std::vector<int> feat;
        int pre = inner, res = cfg.image_size;
        feat.push_back(pre);
        downs.push_back({"downs.0", 0, cfg.in_channel, inner, false, res});
        for (int ind = 0; ind < cfg.n_mults; ++ind) {
            const bool last = ind == cfg.n_mults - 1;
            bool use_attn = false;
            for (int i = 0; i < cfg.n_attn_res; ++i) use_attn |= (cfg.attn_res[i] == res);
            const int ch = inner * cfg.channel_mults[ind];
            for (int r = 0; r < cfg.res_blocks; ++r) {
                downs.push_back({"downs." + std::to_string(downs.size()), 1, pre, ch, use_attn, res});
                feat.push_back(ch); pre = ch;
            }
            if (!last) { downs.push_back({"downs." + std::to_string(downs.size()), 2, pre, pre, false, res}); feat.push_back(pre); res /= 2; }
        }
        mid.push_back({"mid.0", 1, pre, pre, true, res});
        mid.push_back({"mid.1", 1, pre, pre, false, res});
        for (int ind = cfg.n_mults - 1; ind >= 0; --ind) {
            const bool last = ind < 1;
            bool use_attn = false;
            for (int i = 0; i < cfg.n_attn_res; ++i) use_attn |= (cfg.attn_res[i] == res);
            const int ch = inner * cfg.channel_mults[ind];
            for (int r = 0; r < cfg.res_blocks + 1; ++r) {
                ups.push_back({"ups." + std::to_string(ups.size()), 1, pre + feat.back(), ch, use_attn, res});
                feat.pop_back(); pre = ch;
            }
            if (!last) { ups.push_back({"ups." + std::to_string(ups.size()), 3, pre, pre, false, res}); res *= 2; }
        }
        int F_total = 0;
        for (auto* v : {&downs, &mid, &ups}) for (auto& L : *v) if (L.kind == 1) F_total += L.cout;
        F = F_total;
        if (train) {
            fin_bias_sum = new_zero(4); dfilm = new_zero((size_t)Bp * F); dtau = new_zero((size_t)Bp * inner);
            if (dry) plan_bytes += (size_t)Bp * H * W * 64 * sizeof(bf16) + (size_t)F * (inner + 2) * 4;
            if (!dry) {
                deps_b = static_cast<bf16*>(mem.alloc((size_t)Bp * H * W * 64 * sizeof(bf16)));
                dwf_all = static_cast<float*>(mem.alloc((size_t)F * inner * 4)); dbf_all = static_cast<float*>(mem.alloc((size_t)F * 4));
                dcb_all = static_cast<float*>(mem.alloc((size_t)F * 4));
                drop_dev = static_cast<DropSpec*>(mem.alloc(256 * sizeof(DropSpec)));
            }
        }

        if (!dry) {
            mlp_w1 = f32_param("noise_level_mlp.1.weight", {4 * inner, inner});
            mlp_b1 = f32_param("noise_level_mlp.1.bias", {4 * inner});
            mlp_w2 = f32_param("noise_level_mlp.3.weight", {inner, 4 * inner});
            mlp_b2 = f32_param("noise_level_mlp.3.bias", {inner});
            film_w = static_cast<float*>(mem.alloc((size_t)F * inner * 4));
            film_b = static_cast<float*>(mem.alloc((size_t)F * 4));
            film_cb = static_cast<float*>(mem.alloc((size_t)F * 4));
            film = static_cast<float*>(mem.alloc((size_t)Bp * F * 4));
            tau = static_cast<float*>(mem.alloc((size_t)Bp * inner * 4));
            // step prologue
            float4* sa = reinterpret_cast<float4*>(stats_arena);
            const long long n4 = (long long)(stats_cap * sizeof(double) / 16);
            StepCtl* c = ctl_dev;
            push([=](cudaStream_t st) { launch_k(step_begin_kernel, dim3((int)std::min<long long>((n4 + 255) / 256, 592)), dim3(256), 0, st, sa, n4, c); });
            EmbedParams ep{}; ep.ctl = ctl_dev; ep.nl_table = nl_table; ep.nl_buf = nl_buf; ep.w1 = mlp_w1; ep.b1 = mlp_b1; ep.w2 = mlp_w2; ep.b2 = mlp_b2;
            ep.tau = tau; ep.inner = inner;
            const int Bn = B;
            film_tau_chunk(inner, B);                   // (refuses an inner_channel film_kernel cannot stage before anything is launched)
            side_begin = (int)ops.size();
            push([=](cudaStream_t st) { launch_embed(ep, Bn, st); });
            float *fw = film_w, *fb = film_b, *fc = film_cb, *ta = tau, *fi = film; const int Fn = F, inn = inner;
            push([=](cudaStream_t st) { launch_film(fw, fb, fc, ta, fi, Fn, inn, Bn, st); });
            side_end = (int)ops.size();
        }

        int film_off = 0;
        std::vector<Act> feats;
        Act x;
        // the res block in front of a Down / Upsample also emits the bf16 copy ("xraw") that conv reads
        for (size_t li = 0; li < downs.size(); ++li) {
            auto& L = downs[li];
            const bool next_is_down = li + 1 < downs.size() && downs[li + 1].kind == 2;
            if (L.kind == 0) {          // first conv on the (zero-padded to 64 ch) input buffer
                bf16* w = new_weight(inner, 9 * in_C);
                conv_weight_param(L.name + ".weight", w, inner, cfg.in_channel, 3, 9 * in_C, 0, in_C);
                float* b = f32_param(L.name + ".bias", {inner});
                x = new_act(inner, H, W, L.name);
                ConvArgs c; c.n_a = 1; c.a[0] = nhwc_src(in_buf, Bp, H, W, in_C * PW); c.c0 = in_C;
                add_conv_slabs(c.slabs, 0, in_C, 3, 1, 0);
                c.w = w; c.ktot = 9 * in_C; c.cout = inner; c.OH = H; c.OW = W; c.bias = b; c.out = x;
                add_conv(c);
                if (train) bwd_first_conv(L.name, x);
                if (!dry) side_join = (int)ops.size();      // the FiLM biases are first read by the next block's conv1 epilogue
            } else if (L.kind == 1) {
                bf16* xr = next_is_down ? static_cast<bf16*>(role("xraw", (size_t)Bp * x.H * x.W * L.cout * 2 * PW)) : nullptr;
                last_xraw = xr;
                x = add_res_block(L, x, nullptr, film_off, xr, /*x_has_skip=*/true);
            } else {                    // Downsample: conv3x3 stride 2 on the raw stream (unet.py:68-74)
                const int C = x.C;
                bf16* w = new_weight(C, 9 * C);
                conv_weight_param(L.name + ".conv.weight", w, C, C, 3, 9 * C, 0, C);
                float* b = f32_param(L.name + ".conv.bias", {C});
                bf16* raw = train ? last_xraw : static_cast<bf16*>(role("xraw", (size_t)Bp * x.H * x.W * C * 2 * PW));
                Act y = new_act(C, x.H / 2, x.W / 2, L.name);
                ConvArgs c; c.n_a = 1; c.a[0] = nhwc_stride2_src(raw, Bp, x.H, x.W, C * PW); c.c0 = C;
                add_conv_slabs(c.slabs, 0, C, 3, 2, 0, C * PW);
                c.w = w; c.ktot = 9 * C; c.cout = C; c.OH = y.H; c.OW = y.W; c.bias = b; c.out = y;
                add_conv(c);
                if (train) bwd_downsample(L.name, x, y, raw);
                x = y;
            }
            feats.push_back(x);
        }
        for (size_t mi = 0; mi < mid.size(); ++mi) x = add_res_block(mid[mi], x, nullptr, film_off, nullptr, /*x_has_skip=*/mi == 0);
        for (size_t li = 0; li < ups.size(); ++li) {
            auto& L = ups[li];
            const bool next_is_up = li + 1 < ups.size() && ups[li + 1].kind == 3;
            if (L.kind == 1) {
                Act skip = feats.back(); feats.pop_back();
                bf16* xr = next_is_up ? static_cast<bf16*>(role("xraw", (size_t)Bp * x.H * x.W * L.cout * 2 * PW)) : nullptr;
                last_xraw = xr;
                x = add_res_block(L, x, &skip, film_off, xr);
            } else {
                // Upsample (nearest 2x then conv3x3, unet.py:58-65) folded onto the low-res input (fold_up_conv)
                const int C = x.C, Hl = x.H, Wl = x.W;
                const int rows_pad = ((C + 127) / 128) * 128;
                bf16* wall = nullptr;     // [phase][rows_pad][PW * 4C]
                const size_t wall_bytes = (size_t)4 * rows_pad * 4 * C * PW * sizeof(bf16);
                if (dry) plan_bytes += wall_bytes;
                if (!dry) {
                    wall = static_cast<bf16*>(mem.alloc(wall_bytes));
                    add_param(L.name + ".conv.weight", {C, C, 3, 3});
                    PackDesc d{}; d.type = 5; d.dst = wall; d.Cout = C; d.Cin = C; d.ld = 4 * C * PW; d.lo_off = precise ? 4 * C : 0;
                    d.n = (long long)rows_pad * 4 * C * PW;
                    add_pack(L.name + ".conv.weight", d);
                }
                float* b = f32_param(L.name + ".conv.bias", {C});
                bf16* raw = train ? last_xraw : static_cast<bf16*>(role("xraw", (size_t)Bp * Hl * Wl * C * 2 * PW));
                bf16* upb = nullptr;
                if (train) {      // the weight gradient contracts dY with the nearest-2x upsampled input: keep a bf16 copy of it
                    upb = static_cast<bf16*>(role("up_x", (size_t)Bp * Hl * 2 * Wl * 2 * C * 2));
                    add_cast(x, upb, 2);
                }
                Act y = new_act(C, Hl * 2, Wl * 2, L.name);
                ConvArgs c;
                fold_up_conv(c, raw, Bp, Hl, Wl, C, PW);
                c.w = wall; c.bias = b; c.out = y;
                add_conv(c);
                if (train) bwd_upsample(L.name, x, y, upb);
                x = y;
            }
        }
        REQUIRE(film_off == F, "film bookkeeping");
        {   // final Block (GN -> SiLU -> conv 64 -> out_channel) with the eps / posterior epilogue
            const int C = x.C, co = cfg.out_channel;
            REQUIRE(co <= 4 && co == cfg.channels, "out_channel must equal diffusion channels (<=4)");
            float* g = f32_param("final_conv.block.0.weight", {C});
            float* be = f32_param("final_conv.block.0.bias", {C});
            bf16* w = new_weight(co, 9 * C);
            conv_weight_param("final_conv.block.3.weight", w, co, C, 3, 9 * C, 0, C);
            float* b = f32_param("final_conv.block.3.bias", {co});
            bf16* a = static_cast<bf16*>(role("a1", (size_t)Bp * H * W * C * 2 * PW));
            add_prep(x, nullptr, g, be, cfg.norm_groups, true, a, nullptr);
            if (train) bwd_final(x, a, g, be, last_mr);
            if (!dry) {
                GemmDesc d; d.n_a = 1; d.a[0] = nhwc_src(a, Bp, H, W, C * PW);
                add_conv_slabs(d.slabs, 0, C, 3, 1, 0);
                set_precise(d, C, 0, 9 * C);
                conv_geometry(d, W, H, Bt, 16);
                d.block_n = 16; d.b_ptr = w; d.b_K = 9 * C * PW; d.b_rows = 128; d.n_tiles = 1; d.b_is_param = true;
                d.mode = 1; d.OW = W; d.OH = H; d.OB = B; d.n_valid = co; d.bias = b; d.ctl = ctl_dev;
                d.post.tab = post_tab; d.post.T = T_cap; d.post.H = H; d.post.W = W; d.post.C = co;
                d.post.x_state = x_state; d.post.eps_out = eps_buf; d.post.mean_out = mean_buf; d.post.noise_buf = noise_buf;
                d.post.in_buf = in_buf; d.post.in_C = in_C * PW; d.post.in_coff = cond_c; d.post.in_lo_off = precise ? in_C : 0;
                push_gemm(d);
            }
        }
    }

    // height x width: the size of the images the plan runs on (image_size x image_size unless sr3_engine_create_sized says otherwise).
    // cfg.image_size only places the attention layers (build_plan); every activation takes its size from height and width.
    void init(const sr3_unet_config& c, int batch, int height, int width, int device) {
        cfg = c; B = batch; dev = device;
        REQUIRE(B >= 1, "batch must be >= 1");
        REQUIRE(cfg.n_mults >= 1 && cfg.n_mults <= SR3_MAX_LEVELS, "bad n_mults");
        // checked before anything touches the device
        const int min_h = check_image_size(cfg.n_mults, height, width);
        CK(cudaSetDevice(dev));
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, dev));
        REQUIRE(prop.major == 9 && prop.minor == 0, "sr3_b200 needs an sm_90 GPU (found sm_%d%d); there is no fallback path", prop.major, prop.minor);
        REQUIRE(cfg.inner_channel % 64 == 0, "inner_channel must be a multiple of 64 (got %d)", cfg.inner_channel);
        // the FiLM / noise-level MLP backward holds every image's embedding in one block's shared memory: refuse a training batch it
        // cannot hold now, not at the end of the first backward
        REQUIRE(!train || (film_bwd_smem(B, cfg.inner_channel) <= FILM_BWD_SMEM_MAX && embed_bwd_smem(B, cfg.inner_channel) <= FILM_BWD_SMEM_MAX),
                "FiLM / noise-level MLP backward: batch %d too large for one block's shared memory", B);
        REQUIRE(cfg.in_channel <= 64, "in_channel must be <= 64");
        for (int i = 0; i < cfg.n_mults; ++i) REQUIRE((cfg.inner_channel * cfg.channel_mults[i]) % (2 * cfg.norm_groups) == 0 || (cfg.inner_channel * cfg.channel_mults[i]) % cfg.norm_groups == 0, "norm_groups must divide the channel counts");
        inner = cfg.inner_channel; H = height; W = width;
        REQUIRE(cfg.precision == 0 || cfg.precision == 1, "precision must be 0 (bf16) or 1 (precise)");
        precise = cfg.precision == 1; PW = precise ? 2 : 1;
        cond_c = cfg.conditional ? cfg.in_channel - cfg.channels : 0;
        // 8x8 levels tile two images per CTA.  A 4x4 level tiles four, and its attention batches hold eight 16-token images, which
        // read (P = 0 makes them inert, but they must be finite) every image slot of their batch: Bp is a multiple of 8, and the
        // slots no layer writes hold the zeros of the allocation (or, in shared scratch, another layer's finite values).  What counts
        // is the lowest level of the images actually run, not the one image_size would give.
        const int min_res = min_h;
        Bp = min_res == 4 ? (B + 7) & ~7 : (B + 1) & ~1;
        Bt = min_res == 4 ? B : Bp;
        T_cap = 4096;
        REQUIRE(!(train && precise), "the training plan supports the bf16 precision only");
        // pass 1: sizes
        dry = true; stats_used = 0; zero_used = 0; plan_bytes = 0;
        build_plan();
        bwd_blocks.clear(); bwd_kinds.clear(); bwd_block_params.clear(); film_slices.clear(); drop_host.clear(); drop_names.clear();
        if (train) {
            // a training plan keeps every intermediate, and its attention scratch grows as (tokens per image)^2: refuse one that cannot fit
            // now, rather than let an allocation fail halfway through the plan
            size_t need = plan_bytes + ((stats_used + 3) & ~size_t(3)) * sizeof(double) + (zero_used + 4) * sizeof(float);
            for (auto& kv : role_max) need += kv.second;
            need += (size_t)Bp * H * W * in_C * 2 + (size_t)6 * Bp * cfg.channels * H * W * 4;     // in_buf and the six image buffers
            size_t free_b = 0, total_b = 0;
            CK(cudaMemGetInfo(&free_b, &total_b));
            REQUIRE(need <= free_b, "training plan at %dx%d, batch %d: needs %zu bytes (%.2f GiB) of device memory, %zu bytes (%.2f GiB) are free",
                    H, W, B, need, need / 1073741824.0, free_b, free_b / 1073741824.0);
        }
        if (train) {
            zero_cap = zero_used + 4;
            zero_arena = static_cast<float*>(mem.alloc(zero_cap * sizeof(float)));
            loss_dev = static_cast<double*>(mem.alloc(sizeof(double)));
        }
        // allocate
        stats_cap = (stats_used + 3) & ~size_t(3);
        stats_arena = static_cast<double*>(mem.alloc(stats_cap * sizeof(double)));
        for (auto& kv : role_max) role_ptr[kv.first] = mem.alloc(kv.second);
        ctl_dev = static_cast<StepCtl*>(mem.alloc(sizeof(StepCtl)));
        in_buf = static_cast<bf16*>(mem.alloc((size_t)Bp * H * W * in_C * 2 * PW));
        const size_t img = (size_t)Bp * cfg.channels * H * W * 4;
        x_state = static_cast<float*>(mem.alloc(img)); eps_buf = static_cast<float*>(mem.alloc(img));
        mean_buf = static_cast<float*>(mem.alloc(img)); noise_buf = static_cast<float*>(mem.alloc(img));
        io_a = static_cast<float*>(mem.alloc(img)); io_b = static_cast<float*>(mem.alloc(img));
        nl_buf = static_cast<float*>(mem.alloc(Bp * 4));
        nl_table = static_cast<float*>(mem.alloc((T_cap + 1) * 4));
        post_tab = static_cast<float*>(mem.alloc((size_t)5 * T_cap * 4));
        // pass 2: real plan
        dry = false; stats_used = 0; zero_used = 0;
        g_gemm_registry = &gemms;
        try { build_plan(); } catch (...) { g_gemm_registry = nullptr; throw; }
        g_gemm_registry = nullptr;
        if (!train) {
            // every tile kernel pulls the weights of the next one into L2 (the last one those of the next step's first)
            for (size_t i = 0; i < gemms.size(); ++i) {
                const GemmHandle& nx = gemms[(i + 1) % gemms.size()];
                // attention "weights" (B operands that are activations produced by an earlier kernel of this step) are skipped
                bool is_param = false;
                is_param = nx.w_is_param;
                if (is_param) { gemms[i].p->pf_ptr = nx.w_ptr; gemms[i].p->pf_bytes = nx.w_bytes & ~15ll; }
            }
        }
        CK(cudaStreamCreateWithFlags(&cap_stream, cudaStreamNonBlocking));
        CK(cudaDeviceSynchronize());
    }

    // Records the ops of one step into the capture running on `main` (the noise-level embedding + FiLM projections on a forked branch).
    void record_step(cudaStream_t main) {
        const bool fork = side_begin > 0 && side_end > side_begin && side_join >= side_end;
        if (fork && !side_stream) {
            CK(cudaStreamCreateWithFlags(&side_stream, cudaStreamNonBlocking));
            CK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
        }
        for (int i = 0; i < (int)ops.size(); ++i) {
            if (fork && i == side_begin) {              // branch: embed + film depend on the step prologue only
                CK(cudaEventRecord(ev_fork, main));
                CK(cudaStreamWaitEvent(side_stream, ev_fork, 0));
            }
            if (fork && i == side_join) {
                CK(cudaEventRecord(ev_join, side_stream));
                CK(cudaStreamWaitEvent(main, ev_join, 0));
            }
            ops[i](fork && i >= side_begin && i < side_end ? side_stream : main);
        }
    }
    void run_step(cudaStream_t st) {
        if (!graph) {
            cudaGraph_t g;
            CK(cudaStreamBeginCapture(cap_stream, cudaStreamCaptureModeThreadLocal));
            record_step(cap_stream);
            CK(cudaStreamEndCapture(cap_stream, &g));
            CK(cudaGraphInstantiate(&graph, g, 0));
            CK(cudaGraphDestroy(g));
        }
        CK(cudaGraphLaunch(graph, st));
    }
    void push_ctl(cudaStream_t st) { CK(cudaMemcpyAsync(ctl_dev, &ctl, sizeof(StepCtl), cudaMemcpyHostToDevice, st)); }
    void load_nchw(const float* src, int C, int coff, float* copy, cudaStream_t st) {
        const long long total = 1LL * B * C * H * W;
        const int blocks = (int)std::min<long long>((total + 255) / 256, num_sms() * 8LL);
        load_nchw_kernel<<<blocks, 256, 0, st>>>(src, B, C, H, W, in_buf, in_C * PW, coff, copy, precise ? in_C : 0);
        CK(cudaGetLastError());
    }
    size_t img_bytes() const { return (size_t)B * cfg.channels * H * W * 4; }
    void check_params() {
        for (auto& p : params) REQUIRE(p.loaded, "parameter %s was never loaded", p.name.c_str());
    }
    void load_inputs(const float* x, const float* cond, cudaStream_t st) {
        if (cfg.conditional) { REQUIRE(cond != nullptr, "condition_x is required by a conditional model"); load_nchw(cond, cond_c, 0, nullptr, st); }
        else REQUIRE(cond == nullptr, "condition_x given to an unconditional model");
        load_nchw(x, cfg.channels, cond_c, x_state, st);
    }
};

// ------------------------------------------------------------------------------------------------ windowed sampling
// Window origins along one axis of length L: one window when L == side, else n = ceil((L - overlap) / (side - overlap)) windows at
// round-half-up(i (L - side) / (n - 1)) -- the first starts at 0, the last ends at L, neighbours overlap by at least `overlap`.
static std::vector<int> window_origins(int L, int side, int overlap) {
    std::vector<int> o(1, 0);
    if (L == side) return o;
    const int n = (L - overlap + (side - overlap) - 1) / (side - overlap);
    o.resize(n);
    for (int i = 0; i < n; ++i) o[i] = (int)((2LL * i * (L - side) + (n - 1)) / (2LL * (n - 1)));
    return o;
}
// Blend weights [n][side] of the n windows of one axis: min(i + 1, side - i, ramp) / ramp with ramp = max(overlap, 1); the ramp towards a
// border of the canvas (no neighbour there) is dropped, so a single window weighs 1 everywhere.
static std::vector<float> window_weights(int n, int side, int overlap) {
    const int ramp = std::max(overlap, 1);
    std::vector<float> w((size_t)n * side);
    for (int k = 0; k < n; ++k)
        for (int i = 0; i < side; ++i) {
            int m = ramp;
            if (k > 0) m = std::min(m, i + 1);
            if (k < n - 1) m = std::min(m, side - i);
            w[(size_t)k * side + i] = (float)m / (float)ramp;
        }
    return w;
}

struct sr3_windowed {
    sr3_engine* e = nullptr;               // borrowed: runs Bw = e->B windows of e->H x e->W per pass
    int B = 0, H = 0, W = 0, N = 0;        // canvas batch and size; windows of all images
    std::vector<int> oy, ox;
    std::vector<float> wy, wx;
    DevAllocs mem;
    WindowGeom g{};
    float *x = nullptr, *cond = nullptr, *noise = nullptr, *means = nullptr;
    WindowCtl* ctl_dev = nullptr;
    WindowCtl ctl{};
    uint64_t seed = 0, first_index = 0;
    float* snapshots = nullptr; int snapshot_cap = 0;
    cudaGraphExec_t graph = nullptr;
    cudaStream_t cap_stream = nullptr;

    ~sr3_windowed() {
        if (graph) cudaGraphExecDestroy(graph);
        if (cap_stream) cudaStreamDestroy(cap_stream);
    }
    size_t canvas_elems() const { return (size_t)B * e->cfg.channels * H * W; }

    void init(sr3_engine* eng, int batch, int height, int width, int overlap_h, int overlap_w) {
        e = eng; B = batch; H = height; W = width;
        const int wh = e->H, ww = e->W, C = e->cfg.channels;
        // checked before anything is allocated
        REQUIRE(B >= 1, "batch must be >= 1");
        REQUIRE(H >= wh && W >= ww, "canvas %dx%d is smaller than the window %dx%d (canvases are not padded)", H, W, wh, ww);
        REQUIRE(overlap_h >= 0 && overlap_h < wh && overlap_w >= 0 && overlap_w < ww, "overlap %dx%d must be at least 0 and below the window %dx%d",
                overlap_h, overlap_w, wh, ww);
        REQUIRE((long long)B * H * W < (1LL << 31) && (long long)H * W < (1LL << 31), "canvas too large");
        oy = window_origins(H, wh, overlap_h); ox = window_origins(W, ww, overlap_w);
        wy = window_weights((int)oy.size(), wh, overlap_h); wx = window_weights((int)ox.size(), ww, overlap_w);
        N = B * (int)(oy.size() * ox.size());
        CK(cudaSetDevice(e->dev));
        const size_t cb = canvas_elems() * sizeof(float);
        x = static_cast<float*>(mem.alloc(cb)); noise = static_cast<float*>(mem.alloc(cb));
        if (e->cond_c) cond = static_cast<float*>(mem.alloc((size_t)B * e->cond_c * H * W * sizeof(float)));
        means = static_cast<float*>(mem.alloc((size_t)N * C * wh * ww * sizeof(float)));
        ctl_dev = static_cast<WindowCtl*>(mem.alloc(sizeof(WindowCtl)));
        int* oyd = static_cast<int*>(mem.alloc(oy.size() * sizeof(int))); int* oxd = static_cast<int*>(mem.alloc(ox.size() * sizeof(int)));
        float* wyd = static_cast<float*>(mem.alloc(wy.size() * sizeof(float))); float* wxd = static_cast<float*>(mem.alloc(wx.size() * sizeof(float)));
        CK(cudaMemcpy(oyd, oy.data(), oy.size() * sizeof(int), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(oxd, ox.data(), ox.size() * sizeof(int), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(wyd, wy.data(), wy.size() * sizeof(float), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(wxd, wx.data(), wx.size() * sizeof(float), cudaMemcpyHostToDevice));
        g.B = B; g.C = C; g.H = H; g.W = W; g.wh = wh; g.ww = ww; g.ny = (int)oy.size(); g.nx = (int)ox.size();
        g.oy = oyd; g.ox = oxd; g.wy = wyd; g.wx = wxd;
        CK(cudaStreamCreateWithFlags(&cap_stream, cudaStreamNonBlocking));
    }

    // One canvas step: advance the canvas timestep, then per pass of Bw windows gather -> the engine's step (mean-only form) -> store of
    // the pass's means; then the merge.  Slots of the last pass beyond the window list repeat the last window (finite, never stored).
    void begin_step(cudaStream_t st) { launch_k(step_begin_kernel, dim3(1), dim3(32), 0, st, static_cast<float4*>(nullptr), 0LL, &ctl_dev->step); }
    void gather(int first, cudaStream_t st) {
        WindowGather p{};
        p.g = g; p.cond = cond; p.x = x; p.first = first; p.n_total = N; p.Bw = e->B;
        p.in_buf = e->in_buf; p.in_ld = e->in_C * e->PW; p.cond_c = e->cond_c; p.lo_off = e->precise ? e->in_C : 0;
        p.x_state = e->x_state; p.wctl = ctl_dev; p.ectl = e->ctl_dev;
        const long long total = 1LL * e->B * g.wh * (g.ww / 4);
        launch_k(window_gather_kernel, dim3((int)std::min<long long>((total + 255) / 256, num_sms() * 8LL)), dim3(256), 0, st, p);
    }
    void store_means(int first, cudaStream_t st) {
        const size_t win = (size_t)g.C * g.wh * g.ww;
        CK(cudaMemcpyAsync(means + first * win, e->mean_buf, std::min(e->B, N - first) * win * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    void merge(cudaStream_t st) {
        WindowMerge m{};
        m.g = g; m.means = means; m.x = x; m.noise = noise; m.tab = e->post_tab; m.tab_T = e->T_cap; m.ctl = ctl_dev;
        const long long total = 1LL * B * H * W;
        launch_k(window_merge_kernel, dim3((int)std::min<long long>((total + 255) / 256, num_sms() * 8LL)), dim3(256), 0, st, m);
    }
    void record_step(cudaStream_t st) {
        begin_step(st);
        for (int first = 0; first < N; first += e->B) {
            gather(first, st);
            e->record_step(st);
            store_means(first, st);
        }
        merge(st);
    }
    void run_step(cudaStream_t st) {
        if (!graph) {
            cudaGraph_t gr;
            CK(cudaStreamBeginCapture(cap_stream, cudaStreamCaptureModeThreadLocal));
            record_step(cap_stream);
            CK(cudaStreamEndCapture(cap_stream, &gr));
            CK(cudaGraphInstantiate(&graph, gr, 0));
            CK(cudaGraphDestroy(gr));
        }
        CK(cudaGraphLaunch(graph, st));
    }
    // Control blocks of a run of steps starting at timestep t: the engine computes clipped posterior means only (its own noise add is
    // discarded: update_state = 0, z read from its zeroed noise buffer); the canvas block carries the timestep, the noise source and the key.
    void push_ctl(int t, bool injected, cudaStream_t st) {
        StepCtl& c = e->ctl; memset(&c, 0, sizeof(c));
        c.nl_from_table = 1; c.out_mode = 1; c.write_mean = 1; c.update_state = 0; c.use_noise_buf = 1; c.clip = 1; c.t_next = t;
        CK(cudaMemsetAsync(e->noise_buf, 0, e->img_bytes(), st));
        e->push_ctl(st);
        memset(&ctl, 0, sizeof(ctl));
        ctl.step.t_next = t; ctl.step.use_noise_buf = injected ? 1 : 0; ctl.step.seed = seed; ctl.step.sample_offset = first_index;
        ctl.snapshots = snapshots; ctl.snapshot_cap = snapshot_cap; ctl.T = e->T;
        CK(cudaMemcpyAsync(ctl_dev, &ctl, sizeof(WindowCtl), cudaMemcpyHostToDevice, st));
    }
};

// ------------------------------------------------------------------------------------------------ C ABI
#define API_BEGIN try {
#define API_END                      \
    }                                \
    catch (const std::exception& e) { \
        g_err = e.what();            \
        return 1;                    \
    }                                \
    return 0;

extern "C" {

const char* sr3_last_error(void) { return g_err.c_str(); }
int sr3_abi_version(void) { return 4; }

int sr3_engine_create_sized(const sr3_unet_config* cfg, int batch, int height, int width, int device, sr3_engine** out) {
    API_BEGIN
    REQUIRE(cfg && out, "null argument");
    std::unique_ptr<sr3_engine> e(new sr3_engine());
    e->init(*cfg, batch, height, width, device);
    *out = e.release();
    API_END
}
int sr3_engine_create(const sr3_unet_config* cfg, int batch, int device, sr3_engine** out) {
    if (!cfg) { g_err = "null argument"; return 1; }
    return sr3_engine_create_sized(cfg, batch, cfg->image_size, cfg->image_size, device, out);
}
int sr3_engine_create_train_sized(const sr3_unet_config* cfg, int batch, int height, int width, int device, float dropout, sr3_engine** out) {
    API_BEGIN
    REQUIRE(cfg && out, "null argument");
    REQUIRE(dropout >= 0.f && dropout < 1.f, "dropout %f out of range", dropout);
    std::unique_ptr<sr3_engine> e(new sr3_engine());
    e->train = true; e->drop_p = dropout;
    e->init(*cfg, batch, height, width, device);
    *out = e.release();
    API_END
}
int sr3_engine_create_train(const sr3_unet_config* cfg, int batch, int device, float dropout, sr3_engine** out) {
    if (!cfg) { g_err = "null argument"; return 1; }
    return sr3_engine_create_train_sized(cfg, batch, cfg->image_size, cfg->image_size, device, dropout, out);
}
void sr3_engine_destroy(sr3_engine* e) { delete e; }

int sr3_train_forward(sr3_engine* e, const float* hr, const float* sr, const float* gamma, const float* noise, int loss_type, uint64_t dropout_seed,
                      double* loss_host, void* stream) {
    API_BEGIN
    REQUIRE(e && hr && gamma && noise, "null argument");
    REQUIRE(loss_type == 1 || loss_type == 2, "loss_type must be 1 (l1) or 2 (l2)");
    CK(cudaSetDevice(e->dev));
    e->check_params();
    e->train_forward(hr, sr, gamma, noise, loss_type, dropout_seed, loss_host, static_cast<cudaStream_t>(stream));
    API_END
}
int sr3_train_backward(sr3_engine* e, float grad_scale, float* const* grads, int n_grads, void* stream) {
    API_BEGIN
    REQUIRE(e && grads, "null argument");
    REQUIRE(n_grads == (int)e->params.size(), "expected %d gradient pointers, got %d", (int)e->params.size(), n_grads);
    CK(cudaSetDevice(e->dev));
    e->train_backward(grad_scale, grads, static_cast<cudaStream_t>(stream));
    API_END
}
int sr3_train_unet_forward(sr3_engine* e, const float* x, const float* noise_level, uint64_t dropout_seed, float* eps, void* stream) {
    API_BEGIN
    REQUIRE(e && x && noise_level && eps, "null argument");
    CK(cudaSetDevice(e->dev));
    e->check_params();
    e->train_unet_forward(x, noise_level, dropout_seed, eps, static_cast<cudaStream_t>(stream));
    API_END
}
int sr3_train_unet_backward(sr3_engine* e, const float* deps, float* const* grads, int n_grads, float* dx, float* dnoise_level, void* stream) {
    API_BEGIN
    REQUIRE(e && deps && grads, "null argument");
    REQUIRE(n_grads == (int)e->params.size(), "expected %d gradient pointers, got %d", (int)e->params.size(), n_grads);
    CK(cudaSetDevice(e->dev));
    e->train_unet_backward(deps, grads, dx, dnoise_level, static_cast<cudaStream_t>(stream));
    API_END
}
/* the same backward, layer by layer (last layer first), so that a caller can overlap the gradient all-reduce of finished layers */
int sr3_train_num_backward_blocks(const sr3_engine* e) { return e ? (int)e->bwd_blocks.size() : 0; }
int sr3_train_backward_begin(sr3_engine* e, float grad_scale, float* const* grads, int n_grads) {
    API_BEGIN
    REQUIRE(e && grads && n_grads == (int)e->params.size(), "bad argument");
    e->train_backward_begin(grad_scale, grads);
    API_END
}
int sr3_train_backward_block(sr3_engine* e, int block, void* stream) {
    API_BEGIN
    REQUIRE(e, "null engine");
    CK(cudaSetDevice(e->dev));
    e->train_backward_block(block, static_cast<cudaStream_t>(stream));
    API_END
}
/* Reduce the weight-gradient partial tiles of the layers run since the last flush (one launch): call it before handing a finished bucket of
 * gradients to the all-reduce.  sr3_train_backward / _finish flush what is left themselves. */
int sr3_train_backward_flush(sr3_engine* e, void* stream) {
    API_BEGIN
    REQUIRE(e && !e->grad_dst.empty(), "sr3_train_backward_begin has not been called");
    CK(cudaSetDevice(e->dev));
    e->reduce_flush(static_cast<cudaStream_t>(stream));
    API_END
}
int sr3_train_backward_finish(sr3_engine* e, void* stream) {
    API_BEGIN
    REQUIRE(e && !e->grad_dst.empty(), "sr3_train_backward_begin has not been called");
    CK(cudaSetDevice(e->dev));
    e->bwd_film_and_embed(static_cast<cudaStream_t>(stream));
    API_END
}
int sr3_train_block_params(const sr3_engine* e, int block, int* indices, int cap, int* n) {
    API_BEGIN
    REQUIRE(e && block >= 0 && block < (int)e->bwd_block_params.size() && n, "bad argument");
    const std::vector<int>& v = e->bwd_block_params[block];
    *n = (int)v.size();
    for (int i = 0; i < (int)v.size() && i < cap; ++i) indices[i] = v[i];
    API_END
}
/* Profiling: the backward of the forward that just ran, with CUDA events around every op; ms_by_kind[8] receives the summed device time per
 * op kind (0 data-gradient tile kernel, 1 GroupNorm / elementwise, 4 other, 6 weight gradient + slice reduction, 7 attention GEMMs). */
int sr3_train_backward_profile(sr3_engine* e, float grad_scale, float* const* grads, int n_grads, float* ms_by_kind, void* stream) {
    API_BEGIN
    REQUIRE(e && grads && ms_by_kind && n_grads == (int)e->params.size(), "bad argument");
    CK(cudaSetDevice(e->dev));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    e->train_backward_begin(grad_scale, grads);
    e->reduce_prepare(st); e->reduce_begun = true;
    std::vector<cudaEvent_t> evs;
    std::vector<int> kinds;
    auto mark = [&]() { cudaEvent_t ev; CK(cudaEventCreate(&ev)); CK(cudaEventRecord(ev, st)); evs.push_back(ev); };
    mark();
    int blocks_since_flush = 0;
    for (size_t i = e->bwd_blocks.size(); i-- > 0;) {
        for (size_t j = 0; j < e->bwd_blocks[i].size(); ++j) { e->bwd_blocks[i][j](st); kinds.push_back(e->bwd_kinds[i][j]); mark(); }
        if (++blocks_since_flush == 6) { e->reduce_flush(st); kinds.push_back(5); mark(); blocks_since_flush = 0; }     // about one flush per gradient bucket
    }
    e->reduce_flush(st); kinds.push_back(5); mark();
    e->bwd_film_and_embed(st); kinds.push_back(4); mark();
    CK(cudaStreamSynchronize(st));
    for (int k = 0; k < 8; ++k) ms_by_kind[k] = 0.f;
    for (size_t i = 0; i < kinds.size(); ++i) {
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, evs[i], evs[i + 1]));
        ms_by_kind[kinds[i] & 7] += ms;
    }
    for (auto ev : evs) cudaEventDestroy(ev);
    API_END
}
int sr3_train_set_dropout_mask(sr3_engine* e, const char* block_name, const unsigned char* mask_nchw) {
    API_BEGIN
    REQUIRE(e && block_name, "null argument");
    REQUIRE(e->train, "engine was not created with sr3_engine_create_train");
    bool found = false;
    for (size_t i = 0; i < e->drop_names.size(); ++i)
        if (e->drop_names[i] == block_name) { e->drop_host[i].mask = mask_nchw; found = true; }
    REQUIRE(found, "no dropout layer named %s", block_name);
    API_END
}
int sr3_test_train_film_state(const sr3_engine* e, float* tau, float* dfilm, float* dtau, int* rows, int* F, void* stream) {
    API_BEGIN
    REQUIRE(e && rows && F, "null argument");
    REQUIRE(e->train, "engine was not created with sr3_engine_create_train");
    *rows = e->Bp; *F = e->F;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(e->dev));
    if (tau) CK(cudaMemcpyAsync(tau, e->tau, (size_t)e->Bp * e->inner * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (dfilm) CK(cudaMemcpyAsync(dfilm, e->dfilm, (size_t)e->Bp * e->F * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (dtau) CK(cudaMemcpyAsync(dtau, e->dtau, (size_t)e->Bp * e->inner * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CK(cudaStreamSynchronize(st));
    API_END
}
int sr3_train_num_dropout_layers(const sr3_engine* e) { return e ? (int)e->drop_names.size() : 0; }
int sr3_train_dropout_layer_name(const sr3_engine* e, int index, char* name, int name_cap) {
    API_BEGIN
    REQUIRE(e && index >= 0 && index < (int)e->drop_names.size() && name && name_cap > 0, "bad argument");
    strncpy(name, e->drop_names[index].c_str(), name_cap - 1); name[name_cap - 1] = 0;
    API_END
}
int sr3_adam_step(const void* table_dev, int n_tensors, float lr, float beta1, float beta2, float eps, int step, float grad_scale, void* stream) {
    API_BEGIN
    REQUIRE(table_dev && n_tensors > 0 && step >= 1, "bad argument");
    const float bc1 = 1.0f - powf(beta1, (float)step), bc2 = 1.0f - powf(beta2, (float)step);
    const int ny = n_tensors < 65535 ? n_tensors : 65535;
    adam_kernel<<<dim3(64, ny), 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const AdamTensor*>(table_dev), n_tensors, lr, beta1, beta2, eps, bc1, sqrtf(bc2), grad_scale);
    CK(cudaGetLastError());
    API_END
}

int sr3_engine_num_params(const sr3_engine* e) { return e ? (int)e->params.size() : 0; }
int sr3_engine_param_info(const sr3_engine* e, int index, char* name, int name_cap, int64_t shape[4], int* ndim) {
    API_BEGIN
    REQUIRE(e && index >= 0 && index < (int)e->params.size(), "bad param index");
    const ParamEntry& p = e->params[index];
    if (name && name_cap > 0) { strncpy(name, p.name.c_str(), name_cap - 1); name[name_cap - 1] = 0; }
    for (int i = 0; i < 4; ++i) shape[i] = i < (int)p.shape.size() ? p.shape[i] : 1;
    if (ndim) *ndim = (int)p.shape.size();
    API_END
}
int sr3_engine_load_param(sr3_engine* e, const char* name, const float* src, int64_t numel, void* stream) {
    API_BEGIN
    REQUIRE(e && name && src, "null argument");
    auto it = e->pindex.find(name);
    REQUIRE(it != e->pindex.end(), "unexpected key in state_dict: %s", name);
    ParamEntry& p = e->params[it->second];
    REQUIRE(p.numel == numel, "size mismatch for %s: expected %lld elements, got %lld", name, (long long)p.numel, (long long)numel);
    CK(cudaSetDevice(e->dev));
    for (size_t i = 0; i < e->pack_descs.size(); ++i) {      // every packed copy of this parameter; the fused biases wait for finalize
        if (e->pack_src[i] != it->second || e->pack_descs[i].type == 6) continue;
        PackDesc d = e->pack_descs[i]; d.src = src;
        pack_one(d, static_cast<cudaStream_t>(stream));
    }
    p.loaded = true;
    API_END
}
/* load_state_dict in one call: srcs[i] = DEVICE fp32 pointer of parameter i (sr3_engine_param_info order); re-packs everything and runs the
 * finalisation.  Asynchronous on `stream` (the training loop calls it after every optimizer step). */
int sr3_engine_load_all_params(sr3_engine* e, const float* const* srcs, int n, void* stream) {
    API_BEGIN
    REQUIRE(e && srcs && n == (int)e->params.size(), "expected %d parameter pointers", e ? (int)e->params.size() : 0);
    CK(cudaSetDevice(e->dev));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int i = 0; i < n; ++i) REQUIRE(srcs[i] != nullptr, "null pointer for %s", e->params[i].name.c_str());
    // one launch over the descriptor table (rebuilt only when a parameter moved)
    const size_t nd = e->pack_descs.size();
    if (e->pack_last_ptrs.size() != (size_t)n || memcmp(e->pack_last_ptrs.data(), srcs, n * sizeof(float*)) != 0 || !e->pack_dev) {
        std::vector<PackDesc> tab = e->pack_descs;
        for (size_t i = 0; i < nd; ++i) { tab[i].src = srcs[e->pack_src[i]]; tab[i].src2 = e->pack_src2[i] >= 0 ? srcs[e->pack_src2[i]] : nullptr; }
        if (!e->pack_dev) {
            e->pack_dev = static_cast<PackDesc*>(e->mem.alloc(nd * sizeof(PackDesc)));
            e->pack_ends_dev = static_cast<int*>(e->mem.alloc(nd * sizeof(int)));
            std::vector<int> ends(nd);
            int acc = 0;
            for (size_t i = 0; i < nd; ++i) { acc += pack_entry_blocks(tab[i]); ends[i] = acc; }
            e->pack_blocks = acc;
            CK(cudaMemcpy(e->pack_ends_dev, ends.data(), nd * sizeof(int), cudaMemcpyHostToDevice));
        }
        CK(cudaMemcpyAsync(e->pack_dev, tab.data(), nd * sizeof(PackDesc), cudaMemcpyHostToDevice, st));
        CK(cudaStreamSynchronize(st));                 // `tab` is pageable host memory
        e->pack_last_ptrs.assign(srcs, srcs + n);
    }
    pack_all_kernel<<<dim3((unsigned)e->pack_blocks), 256, 0, st>>>(e->pack_dev, e->pack_ends_dev, (int)nd);
    CK(cudaGetLastError());
    for (auto& p : e->params) p.loaded = true;
    API_END
}
int sr3_engine_finalize_params(sr3_engine* e, void* stream) {
    API_BEGIN
    REQUIRE(e, "null engine");
    e->check_params();
    for (const PackDesc& d : e->pack_descs)
        if (d.type == 6) pack_one(d, static_cast<cudaStream_t>(stream));     // src / src2: the engine's copies of the two biases
    API_END
}

int sr3_engine_set_schedule(sr3_engine* e, int T, const float* a, const float* b, const float* c1, const float* c2, const float* lv,
                            const double* sqrt_ac_prev, void* stream) {
    API_BEGIN
    REQUIRE(e && a && b && c1 && c2 && lv && sqrt_ac_prev, "null argument");
    REQUIRE(T >= 1 && T <= e->T_cap, "n_timestep %d out of range (max %d)", T, e->T_cap);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(e->dev));
    e->T = T;
    std::vector<float> tab((size_t)5 * e->T_cap, 0.f), nl(T + 1);
    const float* srcs[5] = {a, b, c1, c2, lv};
    for (int k = 0; k < 5; ++k) memcpy(tab.data() + (size_t)k * e->T_cap, srcs[k], T * sizeof(float));
    for (int i = 0; i <= T; ++i) nl[i] = static_cast<float>(sqrt_ac_prev[i]);     // FloatTensor([f64]) rounding, diffusion.py:153
    e->logvar_host.assign(lv, lv + T);
    CK(cudaMemcpyAsync(e->post_tab, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(e->nl_table, nl.data(), nl.size() * 4, cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_unet_forward(sr3_engine* e, const float* x, const float* noise_level, float* eps, void* stream) {
    API_BEGIN
    REQUIRE(e && x && noise_level && eps, "null argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(e->dev));
    e->load_nchw(x, e->cfg.in_channel, 0, nullptr, st);
    CK(cudaMemcpyAsync(e->nl_buf, noise_level, e->B * 4, cudaMemcpyDeviceToDevice, st));
    StepCtl& c = e->ctl; memset(&c, 0, sizeof(c));
    c.nl_from_table = 0; c.out_mode = 0; c.t_next = 0;
    e->push_ctl(st);
    e->run_step(st);
    CK(cudaMemcpyAsync(eps, e->eps_buf, e->img_bytes(), cudaMemcpyDeviceToDevice, st));
    API_END
}

int sr3_p_mean_variance(sr3_engine* e, const float* x, const float* cond, int t, int clip, float* mean, float* log_variance, void* stream) {
    API_BEGIN
    REQUIRE(e && x && mean, "null argument");
    REQUIRE(e->T > 0, "set_new_noise_schedule has not been called");
    REQUIRE(t >= 0 && t < e->T, "t=%d out of range [0,%d)", t, e->T);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(e->dev));
    e->load_inputs(x, cond, st);
    StepCtl& c = e->ctl; memset(&c, 0, sizeof(c));
    c.nl_from_table = 1; c.out_mode = 1; c.write_mean = 1; c.update_state = 0; c.use_noise_buf = 1; c.clip = clip; c.t_next = t;
    CK(cudaMemsetAsync(e->noise_buf, 0, e->img_bytes(), st));
    e->push_ctl(st);
    e->run_step(st);
    CK(cudaMemcpyAsync(mean, e->mean_buf, e->img_bytes(), cudaMemcpyDeviceToDevice, st));
    if (log_variance) *log_variance = e->logvar_host[t];
    API_END
}

int sr3_p_sample(sr3_engine* e, const float* x, const float* cond, int t, const float* noise, uint64_t seed, uint64_t first_index,
                 float* x_prev, void* stream) {
    API_BEGIN
    REQUIRE(e && x && x_prev, "null argument");
    REQUIRE(e->T > 0, "set_new_noise_schedule has not been called");
    REQUIRE(t >= 0 && t < e->T, "t=%d out of range [0,%d)", t, e->T);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(e->dev));
    e->load_inputs(x, cond, st);
    StepCtl& c = e->ctl; memset(&c, 0, sizeof(c));
    c.nl_from_table = 1; c.out_mode = 1; c.update_state = 1; c.clip = 1; c.t_next = t; c.seed = seed; c.sample_offset = first_index;
    if (noise) { c.use_noise_buf = 1; CK(cudaMemcpyAsync(e->noise_buf, noise, e->img_bytes(), cudaMemcpyDeviceToDevice, st)); }
    e->push_ctl(st);
    e->run_step(st);
    CK(cudaMemcpyAsync(x_prev, e->x_state, e->img_bytes(), cudaMemcpyDeviceToDevice, st));
    API_END
}

int sr3_p_losses(sr3_engine* e, const float* hr, const float* sr, const float* gamma, const float* noise, int loss_type, double* loss_host,
                 void* stream) {
    API_BEGIN
    REQUIRE(e && hr && gamma && noise && loss_host, "null argument");
    REQUIRE(loss_type == 1 || loss_type == 2, "loss_type must be 1 (l1) or 2 (l2)");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(e->dev));
    if (e->cfg.conditional) { REQUIRE(sr != nullptr, "x_in['SR'] is required by a conditional model"); e->load_nchw(sr, e->cond_c, 0, nullptr, st); }
    const long long total = 1LL * e->B * e->cfg.channels * e->H * e->W;
    const int blocks = (int)std::min<long long>((total + 255) / 256, num_sms() * 8LL);
    q_sample_load_kernel<<<blocks, 256, 0, st>>>(hr, noise, gamma, e->B, e->cfg.channels, e->H, e->W, e->in_buf, e->in_C * e->PW, e->cond_c,
                                                 e->precise ? e->in_C : 0);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(e->nl_buf, gamma, e->B * 4, cudaMemcpyDeviceToDevice, st));
    StepCtl& c = e->ctl; memset(&c, 0, sizeof(c));
    c.nl_from_table = 0; c.out_mode = 0; c.t_next = 0;
    e->push_ctl(st);
    e->run_step(st);
    if (!e->loss_dev) e->loss_dev = static_cast<double*>(e->mem.alloc(sizeof(double)));
    CK(cudaMemsetAsync(e->loss_dev, 0, sizeof(double), st));
    loss_sum_kernel<<<blocks, 256, 0, st>>>(noise, e->eps_buf, total, loss_type == 2 ? 1 : 0, e->loss_dev);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(loss_host, e->loss_dev, sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_p_sample_loop_begin(sr3_engine* e, const float* cond, const float* x_T, uint64_t seed, uint64_t first_index, void* stream) {
    API_BEGIN
    REQUIRE(e && x_T, "null argument");
    REQUIRE(e->T > 0, "set_new_noise_schedule has not been called");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(e->dev));
    e->load_inputs(x_T, cond, st);
    e->seed = seed; e->first_index = first_index;
    API_END
}
int sr3_p_sample_steps(sr3_engine* e, int t_start, int steps, void* stream) {
    API_BEGIN
    REQUIRE(e, "null engine");
    REQUIRE(t_start < e->T && steps >= 0 && t_start - steps + 1 >= 0, "bad step range t_start=%d steps=%d T=%d", t_start, steps, e->T);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(e->dev));
    StepCtl& c = e->ctl; memset(&c, 0, sizeof(c));
    c.nl_from_table = 1; c.out_mode = 1; c.update_state = 1; c.clip = 1; c.t_next = t_start; c.seed = e->seed; c.sample_offset = e->first_index;
    e->push_ctl(st);
    for (int i = 0; i < steps; ++i) e->run_step(st);
    API_END
}
int sr3_read_state(sr3_engine* e, float* x_out, void* stream) {
    API_BEGIN
    REQUIRE(e && x_out, "null argument");
    CK(cudaMemcpyAsync(x_out, e->x_state, e->img_bytes(), cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
    API_END
}

int sr3_p_sample_loop(sr3_engine* e, const float* cond, const float* x_T, const float* noises, uint64_t seed, uint64_t first_index,
                      float* final, float* snapshots, int snapshot_cap, int* n_snapshots, void* stream) {
    API_BEGIN
    REQUIRE(e && x_T, "null argument");
    REQUIRE(e->T > 0, "set_new_noise_schedule has not been called");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(e->dev));
    e->load_inputs(x_T, cond, st);
    const int T = e->T;
    StepCtl& c = e->ctl; memset(&c, 0, sizeof(c));
    c.nl_from_table = 1; c.out_mode = 1; c.update_state = 1; c.clip = 1; c.t_next = T - 1; c.seed = seed; c.sample_offset = first_index;
    c.use_noise_buf = noises ? 1 : 0;
    e->push_ctl(st);
    const int inter = 1 | (T / 10);                     // diffusion.py:179
    const size_t ib = e->img_bytes();
    int ns = 0;
    for (int i = T - 1; i >= 0; --i) {
        if (noises) CK(cudaMemcpyAsync(e->noise_buf, noises + (size_t)i * (ib / 4), ib, cudaMemcpyDeviceToDevice, st));
        e->run_step(st);
        if (i % inter == 0) {
            if (snapshots) {
                REQUIRE(ns < snapshot_cap, "snapshot buffer too small (%d)", snapshot_cap);
                CK(cudaMemcpyAsync(snapshots + (size_t)ns * (ib / 4), e->x_state, ib, cudaMemcpyDeviceToDevice, st));
            }
            ++ns;
        }
    }
    if (final) CK(cudaMemcpyAsync(final, e->x_state, ib, cudaMemcpyDeviceToDevice, st));
    if (n_snapshots) *n_snapshots = ns;
    API_END
}

int sr3_super_resolution_host(sr3_engine* e, const float* cond_host, const float* x_T_host, uint64_t seed, uint64_t first_index,
                              float* final_host, void* stream) {
    API_BEGIN
    REQUIRE(e && x_T_host && final_host, "null argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(e->dev));
    const size_t ib = e->img_bytes();
    if (cond_host) CK(cudaMemcpyAsync(e->io_a, cond_host, ib, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(e->io_b, x_T_host, ib, cudaMemcpyHostToDevice, st));
    int ns = 0;
    int rc = sr3_p_sample_loop(e, cond_host ? e->io_a : nullptr, e->io_b, nullptr, seed, first_index, nullptr, nullptr, 0, &ns, stream);
    if (rc) return rc;
    CK(cudaMemcpyAsync(final_host, e->x_state, ib, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_windowed_create(sr3_engine* e, int batch, int height, int width, int overlap_h, int overlap_w, sr3_windowed** out) {
    API_BEGIN
    REQUIRE(e && out, "null argument");
    std::unique_ptr<sr3_windowed> w(new sr3_windowed());
    w->init(e, batch, height, width, overlap_h, overlap_w);
    *out = w.release();
    API_END
}
void sr3_windowed_destroy(sr3_windowed* w) { delete w; }
int sr3_windowed_begin(sr3_windowed* w, const float* cond, const float* x_T, uint64_t seed, uint64_t first_index, void* stream) {
    API_BEGIN
    REQUIRE(w && x_T, "null argument");
    REQUIRE(w->e->T > 0, "set_new_noise_schedule has not been called");
    if (w->e->cfg.conditional) REQUIRE(cond != nullptr, "condition_x is required by a conditional model");
    else REQUIRE(cond == nullptr, "condition_x given to an unconditional model");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(w->e->dev));
    if (cond) CK(cudaMemcpyAsync(w->cond, cond, (size_t)w->B * w->e->cond_c * w->H * w->W * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(w->x, x_T, w->canvas_elems() * sizeof(float), cudaMemcpyDeviceToDevice, st));
    w->seed = seed; w->first_index = first_index;
    API_END
}
int sr3_windowed_set_snapshots(sr3_windowed* w, float* snapshots, int snapshot_cap) {
    API_BEGIN
    REQUIRE(w && snapshot_cap >= 0 && (snapshots || snapshot_cap == 0), "bad snapshot buffer");
    w->snapshots = snapshots; w->snapshot_cap = snapshot_cap;
    API_END
}
int sr3_windowed_steps(sr3_windowed* w, int t_start, int steps, const float* noises, void* stream) {
    API_BEGIN
    REQUIRE(w, "null argument");
    sr3_engine* e = w->e;
    REQUIRE(t_start < e->T && steps >= 0 && t_start - steps + 1 >= 0, "bad step range t_start=%d steps=%d T=%d", t_start, steps, e->T);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(e->dev));
    e->check_params();
    w->push_ctl(t_start, noises != nullptr, st);
    const size_t n = w->canvas_elems();
    for (int i = 0; i < steps; ++i) {
        if (noises) CK(cudaMemcpyAsync(w->noise, noises + (size_t)(t_start - i) * n, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
        w->run_step(st);
    }
    API_END
}
int sr3_windowed_read_state(sr3_windowed* w, float* x_out, void* stream) {
    API_BEGIN
    REQUIRE(w && x_out, "null argument");
    CK(cudaMemcpyAsync(x_out, w->x, w->canvas_elems() * sizeof(float), cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
    API_END
}
int sr3_windowed_grid(const sr3_windowed* w, int* ny, int* nx, int* origins_y, int* origins_x, float* weights_y, float* weights_x) {
    API_BEGIN
    REQUIRE(w && ny && nx, "null argument");
    *ny = (int)w->oy.size(); *nx = (int)w->ox.size();
    if (origins_y) memcpy(origins_y, w->oy.data(), w->oy.size() * sizeof(int));
    if (origins_x) memcpy(origins_x, w->ox.data(), w->ox.size() * sizeof(int));
    if (weights_y) memcpy(weights_y, w->wy.data(), w->wy.size() * sizeof(float));
    if (weights_x) memcpy(weights_x, w->wx.data(), w->wx.size() * sizeof(float));
    API_END
}
// Eager (non-graph) canvas steps at timestep t with CUDA events around the gathers, the engine passes and the merge: ms[3] = their device
// time per step, averaged over `reps` steps after one warm-up.  Overwrites the canvas state with the steps' results.
int sr3_windowed_profile_step(sr3_windowed* w, int t, int reps, float* ms, void* stream) {
    API_BEGIN
    REQUIRE(w && ms && reps >= 1, "bad argument");
    sr3_engine* e = w->e;
    REQUIRE(e->T > 0 && t >= 0 && t < e->T, "bad t");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(e->dev));
    const int Bw = e->B, passes = (w->N + Bw - 1) / Bw;
    std::vector<cudaEvent_t> ev(3 * passes + 2);
    for (auto& x : ev) CK(cudaEventCreate(&x));
    double acc[3] = {0, 0, 0};
    for (int r = 0; r < reps + 1; ++r) {
        w->push_ctl(t, false, st);
        w->begin_step(st);
        for (int pi = 0; pi < passes; ++pi) {
            CK(cudaEventRecord(ev[3 * pi], st));
            w->gather(pi * Bw, st);
            CK(cudaEventRecord(ev[3 * pi + 1], st));
            for (auto& op : e->ops) op(st);
            CK(cudaEventRecord(ev[3 * pi + 2], st));
            w->store_means(pi * Bw, st);
        }
        CK(cudaEventRecord(ev[3 * passes], st));
        w->merge(st);
        CK(cudaEventRecord(ev[3 * passes + 1], st));
        CK(cudaStreamSynchronize(st));
        if (r == 0) continue;
        float v = 0;
        for (int pi = 0; pi < passes; ++pi) {
            CK(cudaEventElapsedTime(&v, ev[3 * pi], ev[3 * pi + 1])); acc[0] += v;
            CK(cudaEventElapsedTime(&v, ev[3 * pi + 1], ev[3 * pi + 2])); acc[1] += v;
        }
        CK(cudaEventElapsedTime(&v, ev[3 * passes], ev[3 * passes + 1])); acc[2] += v;
    }
    for (int k = 0; k < 3; ++k) ms[k] = (float)(acc[k] / reps);
    for (auto& x : ev) cudaEventDestroy(x);
    API_END
}

int sr3_engine_profile_step(sr3_engine* e, int t, int reps, int cap, int* kinds, float* ms, double* flops, double* bytes, int* n_ops, void* stream) {
    API_BEGIN
    REQUIRE(e && kinds && ms && flops && bytes && n_ops, "null argument");
    REQUIRE(e->T > 0 && t >= 0 && t < e->T, "bad t");
    const int n = (int)e->ops.size();
    REQUIRE(cap >= n, "profile buffers too small (%d ops)", n);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(e->dev));
    std::vector<cudaEvent_t> ev(n + 1);
    for (auto& x : ev) CK(cudaEventCreate(&x));
    std::vector<double> acc(n, 0.0);
    for (int r = 0; r < reps + 1; ++r) {          // first repetition is a warm-up
        StepCtl& c = e->ctl; memset(&c, 0, sizeof(c));
        c.nl_from_table = 1; c.out_mode = 1; c.update_state = 0; c.clip = 1; c.t_next = t; c.seed = 1;
        e->push_ctl(st);
        for (int i = 0; i < n; ++i) { CK(cudaEventRecord(ev[i], st)); e->ops[i](st); }
        CK(cudaEventRecord(ev[n], st));
        CK(cudaStreamSynchronize(st));
        if (r == 0) continue;
        for (int i = 0; i < n; ++i) { float m = 0; CK(cudaEventElapsedTime(&m, ev[i], ev[i + 1])); acc[i] += m; }
    }
    for (int i = 0; i < n; ++i) {
        kinds[i] = e->op_info[i].kind; ms[i] = (float)(acc[i] / (reps > 0 ? reps : 1));
        flops[i] = e->op_info[i].flops; bytes[i] = e->op_info[i].bytes;
    }
    *n_ops = n;
    for (auto& x : ev) cudaEventDestroy(x);
    API_END
}

int sr3_engine_num_launches_per_step(const sr3_engine* e) { return e ? (int)e->ops.size() : 0; }
int sr3_engine_num_ops_per_step(const sr3_engine* e) { return e ? (int)e->ops.size() : 0; }
int64_t sr3_engine_workspace_bytes(const sr3_engine* e) { return e ? e->mem.bytes : 0; }

int sr3_engine_read_activation(sr3_engine* e, const char* name, float* dst, int64_t cap, int64_t* numel, int shape_bhwc[4], void* stream) {
    API_BEGIN
    REQUIRE(e && name, "null argument");
    auto it = e->taps.find(name);
    REQUIRE(it != e->taps.end(), "no activation tap named %s", name);
    const Act& a = it->second;
    const int64_t n = (int64_t)e->B * a.H * a.W * a.C;
    if (numel) *numel = n;
    if (shape_bhwc) { shape_bhwc[0] = e->B; shape_bhwc[1] = a.H; shape_bhwc[2] = a.W; shape_bhwc[3] = a.C; }
    if (dst) {
        REQUIRE(cap >= n, "destination too small");
        CK(cudaMemcpyAsync(dst, a.p, n * 4, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
    }
    API_END
}

int sr3_test_gemm(const void* a, const void* b, float* dptr, int M, int N, int K, int block_n, void* stream) {
    API_BEGIN
    REQUIRE(M % 128 == 0 && K % 64 == 0 && N % block_n == 0, "bad test gemm shape");
    DevAllocs mem;
    GemmDesc d; d.n_a = 1; d.a[0] = matrix_src(a, 1, M, K, K, 0);
    for (int c = 0; c < K; c += 64) d.slabs.push_back({0, c, 0, 0, 0, c});
    d.block_n = block_n; d.b_ptr = b; d.b_K = K; d.b_rows = N;
    d.w_box = 128; d.h_box = 1; d.b_box = 1; d.tiles_w = M / 128; d.tiles_h = 1; d.tiles_b = 1; d.n_tiles = N / block_n; d.nz = 1;
    d.OW = M; d.OH = 1; d.OB = 1; d.n_valid = N;
    d.out_f32 = dptr; d.os = OutSpec{0, 0, 0, N, 0};
    Op op = make_gemm_op(d, mem);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    op(st);
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_test_attention(const void* qk, const void* vT, void* out, int nz, int Lt, int HW, int C, void* stream) {
    API_BEGIN
    Op op = make_attn_op(static_cast<const bf16*>(qk), static_cast<const bf16*>(vT), static_cast<bf16*>(out), nz, Lt, HW, C);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    op(st);
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_test_attention_unfused(const void* qk, const void* vT, float* S, void* P, void* O, int nz, int Lt, int HW, int C, int precise,
                               void* stream) {
    API_BEGIN
    REQUIRE(qk && vT && S && P && O, "null argument");
    REQUIRE(nz >= 1 && Lt % 128 == 0 && C % 128 == 0 && HW >= 1 && Lt % HW == 0, "unfused attention geometry Lt=%d HW=%d C=%d", Lt, HW, C);
    const int PW = precise ? 2 : 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    make_gemm_op(attn_s_desc(static_cast<const bf16*>(qk), S, nz, Lt, C, PW), mem)(st);
    launch_softmax(attn_softmax_params(S, static_cast<bf16*>(P), nz, Lt, HW, PW), st);
    make_gemm_op(attn_pv_desc(static_cast<const bf16*>(P), static_cast<const bf16*>(vT), static_cast<bf16*>(O), nz, Lt, C, PW), mem)(st);
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_bench_conv(int B, int H, int W, int Cin, int Cout, int ksize, int stride, int with_resid, int with_stats, int reps, float* ms_out) {
    API_BEGIN
    REQUIRE(ms_out && reps > 0, "bad arguments");
    DevAllocs mem;
    const int ktot = ksize * ksize * Cin;
    const int OH = H / stride, OW = W / stride;
    bf16* x = static_cast<bf16*>(mem.alloc((size_t)B * H * W * Cin * 2));
    bf16* wp = static_cast<bf16*>(mem.alloc((size_t)Cout * ktot * 2));
    float* y = static_cast<float*>(mem.alloc((size_t)B * OH * OW * Cout * 4));
    float* r = with_resid ? static_cast<float*>(mem.alloc((size_t)B * OH * OW * Cout * 4)) : nullptr;
    double* st = with_stats ? static_cast<double*>(mem.alloc((size_t)B * Cout * 2 * 8)) : nullptr;
    float* bias = static_cast<float*>(mem.alloc((size_t)Cout * 4));
    GemmDesc d; d.n_a = 1;
    d.a[0] = stride == 1 ? nhwc_src(x, B, H, W, Cin) : nhwc_stride2_src(x, B, H, W, Cin);
    add_conv_slabs(d.slabs, 0, Cin, ksize, stride, 0);
    conv_geometry(d, OW, OH, B, Cout, with_resid != 0);
    d.b_ptr = wp; d.b_K = ktot; d.b_rows = Cout;
    REQUIRE(B % d.b_box == 0, "batch must be a multiple of %d at this resolution", d.b_box);
    REQUIRE(Cout >= d.block_n, "Cout smaller than the tile");
    d.n_tiles = Cout / d.block_n;
    d.OW = OW; d.OH = OH; d.OB = B; d.n_valid = Cout; d.bias = bias;
    d.out_f32 = y; d.os = nhwc_out(OH, OW, Cout);
    d.resid = r; d.rs = nhwc_out(OH, OW, Cout);
    d.stats = st; d.stats_C = Cout;
    Op op = make_gemm_op(d, mem);
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    // timed as ONE captured graph of `reps` launches: no CPU launch overhead in the number (as inside the step graph)
    cudaStream_t cs;
    CK(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
    for (int i = 0; i < 3; ++i) op(cs);
    CK(cudaStreamSynchronize(cs));
    cudaGraph_t g; cudaGraphExec_t ge;
    CK(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
    for (int i = 0; i < reps; ++i) op(cs);
    CK(cudaStreamEndCapture(cs, &g));
    CK(cudaGraphInstantiate(&ge, g, 0));
    CK(cudaGraphLaunch(ge, cs));
    CK(cudaStreamSynchronize(cs));
    CK(cudaEventRecord(e0, cs));
    CK(cudaGraphLaunch(ge, cs));
    CK(cudaEventRecord(e1, cs));
    CK(cudaEventSynchronize(e1));
    float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
    cudaGraphExecDestroy(ge); cudaGraphDestroy(g); cudaStreamDestroy(cs);
    *ms_out = ms / reps;
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    API_END
}

int sr3_test_conv_ex(const sr3_test_conv_args* a, sr3_gemm_geometry* geometry, void* stream) {
    API_BEGIN
    REQUIRE(a && a->x && a->w && a->y, "null argument");
    const int B = a->B, H = a->H, W = a->W, Cin = a->Cin, Cout = a->Cout, k = a->ksize, s = a->stride;
    const int PW = a->precise ? 2 : 1;
    REQUIRE(B >= 1 && (k == 1 || k == 3) && (s == 1 || s == 2) && Cin % 64 == 0 && Cout % 64 == 0, "bad test conv shape");
    REQUIRE(!a->fold_up || (k == 3 && s == 1 && Cin == Cout && !a->x2), "folded upsample: 3x3 stride 1 with Cin == Cout and one source");
    REQUIRE(!a->x2 || (a->w2 && a->Cin2 > 0 && a->Cin2 % 64 == 0 && s == 1), "second source: 1x1 weights over Cin2 (multiple of 64) channels, stride 1");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    const int rows_pad = ((Cout + 127) / 128) * 128;
    ConvArgs c;
    // the weights are packed by the engine's descriptors (conv_weight_param, the Upsample fold of the layer builder)
    PackDesc pd{}; pd.Cout = Cout; pd.Cin = Cin; pd.src = a->w;
    if (a->fold_up) {
        fold_up_conv(c, static_cast<const bf16*>(a->x), B, H, W, Cin, PW);
        pd.type = 5; pd.ld = PW * c.ktot; pd.n = (long long)rows_pad * pd.ld; pd.lo_off = PW == 2 ? c.ktot : 0;
        bf16* wall = static_cast<bf16*>(mem.alloc((size_t)4 * pd.n * sizeof(bf16)));     // [phase][rows_pad][PW * 4C]
        pd.dst = wall; c.w = wall;
        pack_one(pd, st);
    } else {
        const int ktot = k * k * Cin + (a->x2 ? a->Cin2 : 0);
        pd.type = 1; pd.k = k; pd.ld = PW * ktot; pd.k_off = 0; pd.tap_stride = Cin; pd.lo_off = PW == 2 ? ktot : 0;
        bf16* wp = static_cast<bf16*>(mem.alloc((size_t)rows_pad * pd.ld * sizeof(bf16)));
        pd.dst = wp; c.w = wp;
        pack_one(pd, st);
        c.a[0] = s == 1 ? nhwc_src(a->x, B, H, W, Cin * PW) : nhwc_stride2_src(a->x, B, H, W, Cin * PW); c.c0 = Cin;
        add_conv_slabs(c.slabs, 0, Cin, k, s, 0, Cin * PW);
        if (a->x2) {      // ResnetBlock block2 + res_conv (add_res_block): the 1x1 shortcut is K columns [k*k*Cin, ktot) of the same GEMM
            pd.src = a->w2; pd.Cin = a->Cin2; pd.k = 1; pd.k_off = k * k * Cin; pd.tap_stride = a->Cin2;
            pack_one(pd, st);
            c.n_a = 2; c.a[1] = nhwc_src(a->x2, B, H, W, a->Cin2 * PW); c.c1 = a->Cin2;
            add_conv_slabs(c.slabs, 1, a->Cin2, 1, 1, k * k * Cin);
        }
        c.ktot = ktot; c.cout = Cout; c.OH = H / s; c.OW = W / s;
    }
    c.bias = a->bias; c.bias2 = a->bias2; c.bias2_stride = Cout; c.resid = a->resid;
    c.out.p = a->y; c.out.stats = a->stats;
    c.raw_out = static_cast<bf16*>(a->y_bf16);
    GemmDesc d = conv_desc(c, B, B, PW);
    d.out_imgs = B;          // the last tile may cover images past B: they load as zeros and are not stored
    g_last_test_conv = LastTestConv{};
    Op op = make_gemm_op(d, mem, &g_last_test_conv.geo, &g_last_test_conv.schedule);
    g_last_test_conv.out_hwc[0] = d.OH * (d.z_phase ? 2 : 1); g_last_test_conv.out_hwc[1] = d.OW * (d.z_phase ? 2 : 1); g_last_test_conv.out_hwc[2] = d.n_valid;
    if (geometry) *geometry = g_last_test_conv.geo;
    op(st);
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_tile_schedule(const sr3_engine* e, int op, sr3_gemm_geometry* geometry, int* schedule, int* out_hwc) {
    API_BEGIN
    REQUIRE(schedule, "null argument");
    sr3_gemm_geometry geo{};
    int sch = -1, hwc[3] = {0, 0, 0};
    if (e == nullptr) {
        REQUIRE(g_last_test_conv.schedule >= 0, "no sr3_test_conv_ex call on this thread yet");
        geo = g_last_test_conv.geo; sch = g_last_test_conv.schedule;
        for (int i = 0; i < 3; ++i) hwc[i] = g_last_test_conv.out_hwc[i];
    } else {
        REQUIRE(op >= 0 && op < (int)e->op_info.size(), "op %d out of range (%d ops per step)", op, (int)e->op_info.size());
        const sr3_engine::OpInfo& info = e->op_info[op];
        geo = info.geo; sch = info.schedule;
        for (int i = 0; i < 3; ++i) hwc[i] = info.out_hwc[i];
    }
    if (geometry) *geometry = geo;
    *schedule = sch;
    if (out_hwc) for (int i = 0; i < 3; ++i) out_hwc[i] = hwc[i];
    API_END
}

int sr3_test_conv(const void* x, const float* w_oihw, const float* bias, float* y, double* stats, int B, int H, int W, int Cin, int Cout,
                  int ksize, int stride, void* stream) {
    sr3_test_conv_args a;
    memset(&a, 0, sizeof(a));
    a.x = x; a.w = w_oihw; a.bias = bias; a.y = y; a.stats = stats;
    a.B = B; a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.ksize = ksize; a.stride = stride;
    return sr3_test_conv_ex(&a, nullptr, stream);
}

int sr3_test_wgrad(const void* dy, const void* x, float* grad, int B, int OH, int OW, int CY, int Cin, int ksize, int stride, int cout_valid,
                   int cin_valid, int slices, float gscale, int raw, int* slices_used, void* stream) {
    API_BEGIN
    REQUIRE(dy && x && grad, "null argument");
    REQUIRE(B >= 1 && ((ksize == 1 && stride == 1) || (ksize == 3 && (stride == 1 || stride == 2))), "bad wgrad shape");
    REQUIRE(cout_valid >= 1 && cout_valid <= CY && cin_valid >= 1 && cin_valid <= Cin, "valid channels %d / %d of %d / %d", cout_valid, cin_valid, CY, Cin);
    REQUIRE(!raw || (ksize == 1 && slices == 0 && cout_valid == CY && cin_valid == Cin), "batched form: 1x1, one slice per batch, every channel");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    const std::vector<WgradTap> taps = ksize == 1 ? taps_1x1() : (stride == 2 ? taps_3x3_stride2(Cin) : taps_3x3());
    const int ntaps = (int)taps.size();
    const ASrc xs = stride == 2 ? nhwc_stride2_src(x, B, 2 * OH, 2 * OW, Cin) : nhwc_src(x, B, OH, OW, Cin);
    WgradOut ro;
    if (raw) { ro.ptr = grad; ro.slice_stride = (long long)CY * Cin; ro.row_stride = Cin; ro.nb = B; }
    const WgradShape s = wgrad_shape(CY, OH, OW, B, Cin, ntaps, slices, raw ? &ro : nullptr);
    float* ws = raw ? grad : static_cast<float*>(mem.alloc((size_t)s.slices * s.co_pad * ntaps * Cin * sizeof(float), false));
    const WgradParams p = wgrad_params(s, static_cast<const bf16*>(dy), CY, OH, OW, B, B, xs, Cin, taps, cout_valid, ws, raw ? &ro : nullptr);
    init_wgrad_attrs();
    launch_k(wgrad_kernel, dim3(s.nx, s.ny, s.slices), dim3(WGRAD_THREADS), (size_t)WGRAD_SMEM_BYTES, st, p);
    if (!raw) {
        WgradReduceDesc rd = wgrad_reduce_desc(s, ws, ntaps, Cin, cout_valid, cin_valid);
        rd.grad = grad; rd.block_begin = 0; rd.block_end = rd.blocks_x * cout_valid;
        WgradReduceDesc* tab = static_cast<WgradReduceDesc*>(mem.alloc(sizeof(WgradReduceDesc), false));
        int* ends = static_cast<int*>(mem.alloc(sizeof(int), false));
        CK(cudaMemcpyAsync(tab, &rd, sizeof(rd), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(ends, &rd.block_end, sizeof(int), cudaMemcpyHostToDevice, st));
        launch_k(wgrad_reduce_kernel, dim3(rd.block_end), dim3(256), 0, st, (const WgradReduceDesc*)tab, (const int*)ends, 0, 1, 0, gscale);
    }
    CK(cudaStreamSynchronize(st));           // the partial tiles and the table die with this call
    if (slices_used) *slices_used = s.slices;
    API_END
}

// core/metrics.py:8-34 tensor2img on the device (see tensor2img_kernel).  src fp32 [n][C][H][W] DEVICE, dst uint8 DEVICE [GH][GW][C] with
// n == 1: GH = H, GW = W;  n > 1: make_grid geometry, nrow images per row: GH = rows * (H + 2) + 2, GW = ncol * (W + 2) + 2.
int sr3_tensor2img(const float* src, unsigned char* dst, int n, int C, int H, int W, int nrow, float min_v, float max_v, void* stream) {
    API_BEGIN
    REQUIRE(src && dst && n >= 1 && C >= 1 && H >= 1 && W >= 1 && max_v > min_v, "bad tensor2img arguments");
    int ncol = 1, GH = H, GW = W;
    if (n > 1) {
        REQUIRE(nrow >= 1, "nrow must be >= 1");
        ncol = nrow < n ? nrow : n;                       // make_grid: xmaps = min(nrow, nmaps), ymaps = ceil(nmaps / xmaps)
        const int rows = (n + ncol - 1) / ncol;
        GH = rows * (H + 2) + 2; GW = ncol * (W + 2) + 2;
    }
    const long long total = 1LL * GH * GW * C;
    const int blocks = (int)std::min<long long>((total + 255) / 256, num_sms() * 8LL);
    tensor2img_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(src, dst, n, C, H, W, ncol, GH, GW, min_v, max_v);
    CK(cudaGetLastError());
    API_END
}

}  // extern "C"

namespace {
// Pillow's Resample.c: precompute_coeffs (bicubic filter, a = -0.5, support 2) + normalize_coeffs_8bpc (PRECISION_BITS = 22), whole input range
double pil_bicubic_filter(double x) {
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
    return 0.0;
}
void pil_bicubic_tables(int in_size, int out_size, std::vector<int>& bounds, std::vector<int>& coef, int& ksize) {
    const double scale = (double)in_size / out_size;
    double filterscale = scale;
    if (filterscale < 1.0) filterscale = 1.0;
    const double support = 2.0 * filterscale;
    ksize = (int)ceil(support) * 2 + 1;
    bounds.assign((size_t)out_size * 2, 0);
    coef.assign((size_t)out_size * ksize, 0);
    const double ss = 1.0 / filterscale;
    std::vector<double> w((size_t)ksize);
    for (int xx = 0; xx < out_size; ++xx) {
        const double center = 0.0 + (xx + 0.5) * scale;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        double ww = 0.0;
        for (int x = 0; x < xmax; ++x) { w[x] = pil_bicubic_filter((x + xmin - center + 0.5) * ss); ww += w[x]; }
        for (int x = 0; x < xmax; ++x) {
            const double v = (ww != 0.0) ? w[x] / ww : w[x];
            coef[(size_t)xx * ksize + x] = v < 0 ? (int)(-0.5 + v * (1 << 22)) : (int)(0.5 + v * (1 << 22));
        }
        bounds[2 * xx] = xmin; bounds[2 * xx + 1] = xmax;
    }
}

// cv2.getGaussianKernel(11, 1.5) (core/metrics.py:58): g_i = exp(-(i-5)^2 / (2 * 1.5^2)), normalised to sum 1
SsimWindow ssim_window() {
    SsimWindow w;
    double s = 0.0;
    for (int i = 0; i < SSIM_TAPS; ++i) {
        const double x = i - (SSIM_TAPS - 1) / 2;
        w.g[i] = std::exp(-0.5 / (1.5 * 1.5) * x * x);
        s += w.g[i];
    }
    const double inv = 1.0 / s;
    for (int i = 0; i < SSIM_TAPS; ++i) w.g[i] *= inv;
    return w;
}

// SSIM of n pairs of HWC images (dtype 0 uint8, 1 float64) into out[n] (DEVICE), asynchronously on st.  An image smaller than the window
// in either direction has an empty valid region: its value is NaN (the reference's mean of an empty crop), written here without a kernel.
void launch_ssim(const void* a, const void* b, int dtype, int n, int H, int W, int C, double* out, DevAllocs& mem, cudaStream_t st) {
    const int Hv = H - (SSIM_TAPS - 1), Wv = W - (SSIM_TAPS - 1);
    if (Hv < 1 || Wv < 1) {
        const std::vector<double> nan((size_t)n, std::numeric_limits<double>::quiet_NaN());
        CK(cudaMemcpyAsync(out, nan.data(), (size_t)n * sizeof(double), cudaMemcpyHostToDevice, st));
        CK(cudaStreamSynchronize(st));           // `nan` is pageable host memory that dies with this call
        return;
    }
    const dim3 grid((Wv + SSIM_TW - 1) / SSIM_TW, (Hv + SSIM_TH - 1) / SSIM_TH, n);
    const int tiles = (int)(grid.x * grid.y);
    double* partial = static_cast<double*>(mem.alloc((size_t)n * tiles * sizeof(double), false));
    const SsimWindow win = ssim_window();
    if (dtype == 0)
        ssim_kernel<unsigned char><<<grid, SSIM_THREADS, 0, st>>>(static_cast<const unsigned char*>(a), static_cast<const unsigned char*>(b), H, W, C,
                                                                   win, partial);
    else
        ssim_kernel<double><<<grid, SSIM_THREADS, 0, st>>>(static_cast<const double*>(a), static_cast<const double*>(b), H, W, C, win, partial);
    CK(cudaGetLastError());
    ssim_finish_kernel<<<(n + 127) / 128, 128, 0, st>>>(partial, tiles, (double)Hv * Wv * C, n, out);
    CK(cudaGetLastError());
}
}  // namespace

extern "C" {

// Host-only: the integer coefficient tables of one resampling pass (needs no GPU; checked against Pillow's by the CPU test-suite).
int sr3_pil_bicubic_tables(int in_size, int out_size, int* bounds, int* coef, int coef_cap, int* ksize) {
    API_BEGIN
    REQUIRE(in_size >= 1 && out_size >= 1 && bounds && coef && ksize, "bad arguments");
    std::vector<int> b, c;
    int ks = 0;
    pil_bicubic_tables(in_size, out_size, b, c, ks);
    REQUIRE((int)c.size() <= coef_cap, "coefficient buffer too small (%d needed)", (int)c.size());
    memcpy(bounds, b.data(), b.size() * sizeof(int));
    memcpy(coef, c.data(), c.size() * sizeof(int));
    *ksize = ks;
    API_END
}

// data/prepare_data.py:17-40 (`trans_fn.resize(img, size, Image.BICUBIC)`: Pillow's two-pass fixed-point bicubic resampler) and
// data/util.py:74-83 (ToTensor, optional horizontal flip, range mapping) on the device.  src uint8 DEVICE [B][h][w][C] (HWC, as PIL hands
// it over); dst_u8 (optional) uint8 DEVICE [B][H][W][C]; dst_f32 (optional) fp32 DEVICE [B][C][H][W] = (resized / 255) * (max - min) + min,
// mirrored along W when flip != 0.  Integer-exact against Pillow.
int sr3_resize_bicubic_u8(const unsigned char* src, unsigned char* dst_u8, float* dst_f32, int B, int h, int w, int C, int H, int W, int flip,
                          float min_v, float max_v, void* stream) {
    API_BEGIN
    REQUIRE(src && (dst_u8 || dst_f32) && B >= 1 && h >= 1 && w >= 1 && C >= 1 && C <= 4 && H >= 1 && W >= 1, "bad resize arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    std::vector<int> bh, ch, bv, cv;
    int ksh = 0, ksv = 0;
    pil_bicubic_tables(w, W, bh, ch, ksh);
    pil_bicubic_tables(h, H, bv, cv, ksv);
    auto up = [&](const std::vector<int>& v) {
        int* d = static_cast<int*>(mem.alloc(v.size() * sizeof(int), false));
        CK(cudaMemcpyAsync(d, v.data(), v.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        return d;
    };
    int *dbh = up(bh), *dch = up(ch), *dbv = up(bv), *dcv = up(cv);
    // horizontal pass first (Pillow's order): [B][h][w][C] -> tmp [B][h][W][C]; then vertical: -> [B][H][W][C] (+ float planes)
    unsigned char* tmp = static_cast<unsigned char*>(mem.alloc((size_t)B * h * W * C, false));
    {
        const long long total = 1LL * B * h * W * C;
        resample_u8_kernel<<<(int)std::min<long long>((total + 255) / 256, num_sms() * 16LL), 256, 0, st>>>(
            src, tmp, nullptr, B, /*lines*/ h, /*out*/ W, C, /*in axis*/ C, /*in line*/ 1LL * w * C, /*in img*/ 1LL * h * w * C,
            /*out axis*/ C, /*out line*/ 1LL * W * C, /*out img*/ 1LL * h * W * C, dbh, dch, ksh, 0, 0.f, 1.f);
        CK(cudaGetLastError());
    }
    {
        const long long total = 1LL * B * W * H * C;
        resample_u8_kernel<<<(int)std::min<long long>((total + 255) / 256, num_sms() * 16LL), 256, 0, st>>>(
            tmp, dst_u8, dst_f32, B, /*lines = x*/ W, /*out = y*/ H, C, /*in axis (y)*/ 1LL * W * C, /*in line (x)*/ C, /*in img*/ 1LL * h * W * C,
            /*out axis*/ 1LL * W * C, /*out line*/ C, /*out img*/ 1LL * H * W * C, dbv, dcv, ksv, flip, min_v, max_v);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(st));             // the tables / intermediate die with this call
    API_END
}

// calculate_psnr (core/metrics.py:42-50): returns the exact integer sum of squared differences of two uint8 DEVICE images through *ssd_host.
int sr3_ssd_u8(const unsigned char* a, const unsigned char* b, int64_t n, unsigned long long* ssd_host, void* stream) {
    API_BEGIN
    REQUIRE(a && b && ssd_host && n >= 1, "bad arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    unsigned long long* d = static_cast<unsigned long long*>(mem.alloc(sizeof(unsigned long long)));
    ssd_u8_kernel<<<(int)std::min<long long>((n + 255) / 256, num_sms() * 8LL), 256, 0, st>>>(a, b, (long long)n, d);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(ssd_host, d, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    API_END
}

// ssim (core/metrics.py:52-72) of n pairs of DEVICE images [n][H][W][C] (dtype 0 uint8, 1 float64) -> ssim_host[n] (see ssim_kernel).
int sr3_ssim(const void* a, const void* b, int dtype, int n, int H, int W, int C, double* ssim_host, void* stream) {
    API_BEGIN
    REQUIRE(a && b && ssim_host && (dtype == 0 || dtype == 1) && n >= 1 && n <= 65535 && H >= 1 && W >= 1 && C >= 1, "bad ssim arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    double* d = static_cast<double*>(mem.alloc((size_t)n * sizeof(double), false));
    launch_ssim(a, b, dtype, n, H, W, C, d, mem, st);
    CK(cudaMemcpyAsync(ssim_host, d, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    API_END
}

// The evaluation of a sampled batch (sr.py:216-217 for every image): tensor2img of sr[i] and hr[i] (fp32 DEVICE [n][C][H][W]) into uint8 HWC
// images (sr_u8 / hr_u8: DEVICE [n][H][W][C], or NULL for scratch), then per pair the exact integer SSD (calculate_psnr) and the SSIM of
// ssim_kernel.  Both results come back in one device-to-host copy.
int sr3_image_metrics(const float* sr, const float* hr, int n, int C, int H, int W, float min_v, float max_v, unsigned char* sr_u8, unsigned char* hr_u8,
                      unsigned long long* ssd_host, double* ssim_host, void* stream) {
    API_BEGIN
    REQUIRE(sr && hr && ssd_host && ssim_host && n >= 1 && n <= 65535 && C >= 1 && H >= 1 && W >= 1 && max_v > min_v, "bad image_metrics arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    const long long per = 1LL * H * W * C;
    if (!sr_u8) sr_u8 = static_cast<unsigned char*>(mem.alloc((size_t)(n * per), false));
    if (!hr_u8) hr_u8 = static_cast<unsigned char*>(mem.alloc((size_t)(n * per), false));
    // results: n SSDs then n SSIMs (both 8 bytes), one copy back
    unsigned long long* res = static_cast<unsigned long long*>(mem.alloc((size_t)n * 16, false));
    CK(cudaMemsetAsync(res, 0, (size_t)n * sizeof(unsigned long long), st));
    const dim3 grid((unsigned)std::min<long long>((per + 255) / 256, num_sms() * 8LL), n);
    tensor2img_kernel<<<grid, 256, 0, st>>>(sr, sr_u8, 1, C, H, W, 1, H, W, min_v, max_v);
    CK(cudaGetLastError());
    tensor2img_kernel<<<grid, 256, 0, st>>>(hr, hr_u8, 1, C, H, W, 1, H, W, min_v, max_v);
    CK(cudaGetLastError());
    ssd_u8_kernel<<<grid, 256, 0, st>>>(sr_u8, hr_u8, per, res);
    CK(cudaGetLastError());
    launch_ssim(sr_u8, hr_u8, 0, n, H, W, C, reinterpret_cast<double*>(res + n), mem, st);
    std::vector<unsigned long long> host((size_t)n * 2);
    CK(cudaMemcpyAsync(host.data(), res, (size_t)n * 16, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    memcpy(ssd_host, host.data(), (size_t)n * sizeof(unsigned long long));
    memcpy(ssim_host, host.data() + n, (size_t)n * sizeof(double));
    API_END
}

// Test hook: conv (tile kernel, statistics in its epilogue) followed by the GroupNorm(+SiLU) apply pass, i.e. one Block of the
// reference (GN -> Swish -> conv, unet.py:80-91) seen from the GN's side: y = conv(x) + bias, a = [silu](GN(y; gamma, beta)).
int sr3_test_conv_groupnorm(const void* x, const float* w_oihw, const float* bias, const float* gamma, const float* beta, int groups, int silu,
                            float* y, void* a_bf16, int B, int H, int W, int Cin, int Cout, int ksize, void* stream) {
    API_BEGIN
    REQUIRE((ksize == 1 || ksize == 3) && Cin % 64 == 0 && Cout % 64 == 0 && Cout % groups == 0, "bad test shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    double* stats = static_cast<double*>(mem.alloc((size_t)B * Cout * 2 * sizeof(double)));
    int rc = sr3_test_conv(x, w_oihw, bias, y, stats, B, H, W, Cin, Cout, ksize, 1, stream);
    if (rc) return rc;
    PrepParams p = gn_op(y, stats, Cout, nullptr, nullptr, 0, gamma, beta, groups, H * W, silu != 0);
    p.out_a = static_cast<bf16*>(a_bf16);
    const RowLaunch L = prep_launch(Cout, groups, p.HW, B);      // the geometry of the engine's add_prep
    p.pix_per_block = L.ppb;
    launch_prep(p, L, st);
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_test_groupnorm_layer(const sr3_test_groupnorm_args* a, void* stream) {
    API_BEGIN
    REQUIRE(a && a->x0 && a->st0 && a->gamma && a->beta && a->dA && a->a_bf16 && a->mr && a->dst0 && a->dgamma && a->dbeta, "null argument");
    REQUIRE(a->C1 == 0 || (a->x1 && a->st1 && a->dst1), "second source without its statistics or gradient");
    REQUIRE(a->drop >= 0 && a->drop <= 2 && (a->drop != 2 || a->drop_mask), "bad dropout source");
    REQUIRE(a->B >= 1 && a->HW >= 1 && (!a->add || a->add_ld >= a->C0 + a->C1), "bad shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    const int C = a->C0 + a->C1;
    DropSpec* drop = nullptr;
    if (a->drop) {
        DropSpec ds{}; ds.mask = a->drop == 2 ? a->drop_mask : nullptr; ds.p = a->drop_p; ds.layer = a->drop_layer; ds.seed = a->drop_seed;
        drop = static_cast<DropSpec*>(mem.alloc(sizeof(DropSpec), false));
        CK(cudaMemcpyAsync(drop, &ds, sizeof(ds), cudaMemcpyHostToDevice, st));
    }
    // forward apply, as add_prep launches it in a training plan
    PrepParams f = gn_op(a->x0, a->st0, a->C0, a->x1, a->st1, a->C1, a->gamma, a->beta, a->groups, a->HW, a->silu != 0);
    PrepParams fp = f;
    fp.drop = drop; fp.save_mr = a->mr; fp.out_a = static_cast<bf16*>(a->a_bf16);
    const RowLaunch Lf = prep_launch(C, a->groups, a->HW, a->B);
    fp.pix_per_block = Lf.ppb;
    launch_prep(fp, Lf, st);
    // backward, as bwd_groupnorm launches it
    GnBwdParams p; memset(&p, 0, sizeof(p));
    p.f = f; p.f.B = a->B;
    p.dA = a->dA; p.drop = drop; p.sums = static_cast<float*>(mem.alloc((size_t)a->B * C * 2 * sizeof(float))); p.add = a->add; p.add_ld = a->add_ld;
    p.mr = a->mr;
    p.dst0 = a->dst0; p.acc0 = a->acc0; p.dst0_b = static_cast<bf16*>(a->dst0_b); p.gsum0 = a->gsum0; p.gsum_ld0 = a->C0;
    p.dst1 = a->dst1;
    p.dgamma = a->dgamma; p.dbeta = a->dbeta; p.gscale = a->gscale;
    const RowLaunch Lb = gn_bwd_launch(C, a->groups, a->HW, a->B);
    p.f.pix_per_block = Lb.ppb;
    launch_gn_bwd(p, Lb, st);
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_test_grad_combine(const float* a, const float* b, float* dst, int acc, void* dst_b, float* gsum, float* bias0, float* bias1, float gscale,
                          int B, int HW, int C, void* stream) {
    API_BEGIN
    REQUIRE(a && B >= 1 && HW >= 1 && (!bias0 || gsum) && (!acc || dst), "bad arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    launch_combine(combine_launch(C, HW, B), a, b, dst, acc, static_cast<bf16*>(dst_b), gsum, B, HW, C, st);
    if (bias0) launch_bias_grad(gsum, C, bias0, bias1, B, C, gscale, st);
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_test_dgrad(const void* dy_bf16, const float* w_oihw, float* dx, int form, int B, int H, int W, int CY, int Cin, int Cout, int ksize,
                   void* stream) {
    API_BEGIN
    REQUIRE(dy_bf16 && w_oihw && dx && B >= 1, "null argument");
    REQUIRE((form == 0 && (ksize == 1 || ksize == 3) && CY == ((Cout + 63) / 64) * 64 && Cin % 64 == 0) ||
            ((form == 1 || form == 2) && ksize == 3 && Cin == Cout && CY == Cin && Cin % 64 == 0), "bad data-gradient shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    const int type = form == 0 ? 2 : (form == 1 ? 3 : 4);
    bf16* w = static_cast<bf16*>(mem.alloc(dgrad_weight_elems(type, Cout, Cin, ksize) * sizeof(bf16)));     // zero padding, as new_weight
    PackDesc pd = dgrad_pack_desc(type, w, Cout, Cin, ksize);
    pd.src = w_oihw;
    pack_one(pd, st);
    const bf16* dy = static_cast<const bf16*>(dy_bf16);
    const ConvArgs c = form == 0 ? dgrad_conv(dy, B, CY, H, W, ksize, w, Cin, dx, nullptr)
                     : form == 1 ? downsample_dgrad_conv(dy, B, H / 2, W / 2, Cin, w, dx)
                                 : upsample_dgrad_conv(dy, B, 2 * H, 2 * W, Cin, w, dx);
    GemmDesc d = conv_desc(c, B, B, 1);
    d.out_imgs = B;
    Op op = make_gemm_op(d, mem);
    op(st);
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_test_attention_bwd(const void* qk_bf16, const void* vT_bf16, const void* P_bf16, const void* dO_bf16, float* dS, void* dS_bf16, float* dqkv,
                           void* dqkv_bf16, int nz, int Lt, int HW, int C, void* stream) {
    API_BEGIN
    REQUIRE(qk_bf16 && vT_bf16 && P_bf16 && dO_bf16 && dS && dS_bf16 && dqkv && dqkv_bf16, "null argument");
    REQUIRE(nz >= 1 && Lt % 128 == 0 && C % 128 == 0 && HW >= 1 && Lt % HW == 0, "attention backward geometry Lt=%d HW=%d C=%d", Lt, HW, C);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    const bf16* qk = static_cast<const bf16*>(qk_bf16);
    const bf16* P = static_cast<const bf16*>(P_bf16);
    const bf16* dO = static_cast<const bf16*>(dO_bf16);
    bf16* dSb = static_cast<bf16*>(dS_bf16);
    bf16* v = static_cast<bf16*>(mem.alloc((size_t)nz * Lt * C * 2, false));
    bf16* kT = static_cast<bf16*>(mem.alloc((size_t)nz * C * Lt * 2, false));
    // the sequence of bwd_attention, from the transposes to the bf16 copy of d(qkv)
    launch_v_from_vT(static_cast<const bf16*>(vT_bf16), v, nz, Lt, C, st);
    launch_kT_from_qk(qk, kT, nz, Lt, C, st);
    make_gemm_op(attn_bwd_dp_desc(dO, v, dS, nz, Lt, C), mem)(st);
    launch_softmax_bwd(P, dS, dSb, nz, Lt, HW, C, st);
    make_gemm_op(attn_bwd_dq_desc(dSb, kT, dqkv, nz, Lt, C), mem)(st);
    init_wgrad_attrs();
    const WgradOut ok = attn_bwd_qkv_out(dqkv, C, nz, Lt, C), ov = attn_bwd_qkv_out(dqkv, 2 * C, nz, Lt, C);
    const std::vector<WgradTap> taps = taps_1x1();
    {   // dK = dS^T Q
        const WgradShape s = wgrad_shape(Lt, Lt / 16, 16, nz, C, 1, 0, &ok);
        const WgradParams p = wgrad_params(s, dSb, Lt, Lt / 16, 16, nz, nz, attn_bwd_q_view(qk, nz, Lt, C), C, taps, Lt, ok.ptr, &ok);
        launch_k(wgrad_kernel, dim3(s.nx, s.ny, s.slices), dim3(WGRAD_THREADS), (size_t)WGRAD_SMEM_BYTES, st, p);
    }
    {   // dV = P^T dO
        const WgradShape s = wgrad_shape(Lt, Lt / 16, 16, nz, C, 1, 0, &ov);
        const WgradParams p = wgrad_params(s, P, Lt, Lt / 16, 16, nz, nz, nhwc_src(dO, nz, Lt / 16, 16, C), C, taps, Lt, ov.ptr, &ov);
        launch_k(wgrad_kernel, dim3(s.nx, s.ny, s.slices), dim3(WGRAD_THREADS), (size_t)WGRAD_SMEM_BYTES, st, p);
    }
    launch_cast_bf16(dqkv, static_cast<bf16*>(dqkv_bf16), (long long)nz * Lt * 3 * C / 4, st);
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_test_film_embed_bwd(const sr3_test_film_args* a, void* stream) {
    API_BEGIN
    REQUIRE(a && a->wf && a->tau && a->dfilm && a->nl && a->w1 && a->b1 && a->w2 && a->dwf && a->dbf && a->dcb && a->dtau && a->dw1 && a->db1 &&
            a->dw2 && a->db2, "null argument");
    REQUIRE(a->F >= 1 && a->inner >= 2 && a->inner % 2 == 0 && a->B >= 1, "bad shape");
    // both kernels' shared-memory limits before anything is launched
    REQUIRE(film_bwd_smem(a->B, a->inner) <= FILM_BWD_SMEM_MAX && embed_bwd_smem(a->B, a->inner) <= FILM_BWD_SMEM_MAX,
            "FiLM / noise-level MLP backward: batch %d too large for one block's shared memory", a->B);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaMemsetAsync(a->dtau, 0, (size_t)a->B * a->inner * sizeof(float), st));
    launch_film_bwd(a->wf, a->tau, a->dfilm, a->dwf, a->dbf, a->dcb, a->dtau, a->F, a->inner, a->B, a->gscale, st);
    launch_embed_bwd(a->nl, a->w1, a->b1, a->w2, a->dtau, a->dw1, a->db1, a->dw2, a->db2, a->inner, a->B, a->gscale, st);
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_test_film_embed_fwd(const float* nl, const float* w1, const float* b1, const float* w2, const float* b2, const float* wf, const float* bf,
                            const float* cb, float* tau, float* film, int F, int inner, int B, void* stream) {
    API_BEGIN
    REQUIRE(nl && w1 && b1 && w2 && b2 && wf && bf && cb && tau && film, "null argument");
    REQUIRE(F >= 1 && inner >= 2 && inner % 2 == 0 && B >= 1, "bad shape");
    film_tau_chunk(inner, B);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    StepCtl* ctl = static_cast<StepCtl*>(mem.alloc(sizeof(StepCtl), false));
    CK(cudaMemsetAsync(ctl, 0, sizeof(StepCtl), st));           // nl_from_table = 0: image b's noise level is nl[b]
    EmbedParams ep{}; ep.ctl = ctl; ep.nl_buf = nl; ep.w1 = w1; ep.b1 = b1; ep.w2 = w2; ep.b2 = b2; ep.tau = tau; ep.inner = inner;
    launch_embed(ep, B, st);
    launch_film(wf, bf, cb, tau, film, F, inner, B, st);
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_test_loss_grad(const float* noise, const float* eps, int B, int C, int H, int W, int l2, double* loss_host, void* deps_bf16, int ld,
                       float* bias_sum, void* stream) {
    API_BEGIN
    REQUIRE(noise && eps && loss_host && deps_bf16 && bias_sum, "null argument");
    REQUIRE(B >= 1 && C >= 1 && C <= ld && H >= 1 && W >= 1, "bad loss shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    double* loss = static_cast<double*>(mem.alloc(sizeof(double)));
    launch_loss_grad(noise, eps, B, C, H, W, l2 ? 1 : 0, loss, static_cast<bf16*>(deps_bf16), ld, bias_sum, st);
    CK(cudaMemcpyAsync(loss_host, loss, sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_test_grad_load(const float* g, int B, int C, int H, int W, void* deps_bf16, int ld, float* bias_sum, void* stream) {
    API_BEGIN
    REQUIRE(g && deps_bf16 && bias_sum, "null argument");
    REQUIRE(B >= 1 && C >= 1 && C <= ld && H >= 1 && W >= 1, "bad gradient shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    launch_grad_load(g, B, C, H, W, static_cast<bf16*>(deps_bf16), ld, bias_sum, st);
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_test_noise_level_bwd(const float* nl, const float* w1, const float* b1, const float* w2, const float* dtau, float* dnl, int inner, int B,
                             void* stream) {
    API_BEGIN
    REQUIRE(nl && w1 && b1 && w2 && dtau && dnl, "null argument");
    REQUIRE(inner >= 2 && inner % 2 == 0 && B >= 1, "bad shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    launch_noise_level_bwd(nl, w1, b1, w2, dtau, dnl, inner, B, st);
    CK(cudaStreamSynchronize(st));
    API_END
}

int sr3_test_input_grad(const void* dy_bf16, const float* w_oihw, float* dx, int B, int H, int W, int inner, int in_channel, void* stream) {
    API_BEGIN
    REQUIRE(dy_bf16 && w_oihw && dx, "null argument");
    REQUIRE(B >= 1 && H >= 1 && W >= 1 && inner % 64 == 0 && in_channel >= 1 && in_channel <= INPUT_GRAD_LD, "bad input-gradient shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevAllocs mem;
    bf16* w = static_cast<bf16*>(mem.alloc(dgrad_weight_elems(2, inner, in_channel, 3) * sizeof(bf16)));     // zero padding, as new_weight
    PackDesc pd = dgrad_pack_desc(2, w, inner, in_channel, 3);
    pd.src = w_oihw;
    pack_one(pd, st);
    float* gx = static_cast<float*>(mem.alloc((size_t)B * H * W * INPUT_GRAD_LD * sizeof(float), false));
    GemmDesc d = conv_desc(input_dgrad_conv(static_cast<const bf16*>(dy_bf16), B, H, W, inner, w, gx), B, B, 1);
    d.out_imgs = B;
    make_gemm_op(d, mem)(st);
    launch_input_grad_store(gx, B, in_channel, H, W, INPUT_GRAD_LD, dx, st);
    CK(cudaStreamSynchronize(st));
    API_END
}

}  // extern "C"
