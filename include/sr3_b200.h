/* sr3_b200 -- C ABI of the H100-native SR3 hot path (libsr3_b200.so).
 *
 * The reference (Janspiry/Image-Super-Resolution-via-Iterative-Refinement) is pure Python/PyTorch and has no
 * FFI; its boundary for this path is the Python factory model/networks.py:83-116 `define_G(opt)` and the methods of
 * the module it returns.  Each entry point below replaces the reference function cited next to it, with the same
 * argument meaning, on plain device pointers (fp32, NCHW contiguous, exactly the tensors the reference passes).
 * No torch types appear here; `stream` is a cudaStream_t passed as void*.  All functions return 0 on success and a
 * non-zero code otherwise, with a message available from sr3_last_error().  There is no CPU fallback.
 *
 * Binding shown in INTEGRATION.md (ctypes, what a maintainer of the reference would add to model/networks.py).
 */
#ifndef SR3_B200_H
#define SR3_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SR3_MAX_LEVELS 8

/* opt['model']['unet'] + opt['model']['diffusion'] as consumed by define_G (model/networks.py:83-109) */
typedef struct sr3_unet_config {
    int in_channel;                    /* 6 conditional, 3 unconditional */
    int out_channel;                   /* 3 */
    int inner_channel;                 /* 64 (must be a multiple of 64) */
    int norm_groups;                   /* 32 (define_G default, networks.py:89-90) or 16 */
    int n_mults;
    int channel_mults[SR3_MAX_LEVELS]; /* channel_multiplier */
    int n_attn_res;
    int attn_res[SR3_MAX_LEVELS];
    int res_blocks;
    int image_size;
    int channels;                      /* diffusion.channels (3) */
    int conditional;                   /* diffusion.conditional */
    int precision;                     /* 0: bf16 operands, fp32 accumulate / stream (north_star tolerance 1e-2 rel);
                                          1: "precise" -- every tensor-core operand is a (hi, lo) bf16 pair and each product is
                                             hi*hi + hi*lo + lo*hi (fp32-level accuracy, north_star tolerance 1e-3 rel; ~3x the MMA work).
                                          The reference arithmetic is fp32 nn.Conv2d / nn.Linear (unet.py:87). */
} sr3_unet_config;

typedef struct sr3_engine sr3_engine;

/* Message of the last failure on the calling thread ("" if none). */
const char* sr3_last_error(void);
/* ABI version of this header. */
int sr3_abi_version(void);

/* UNet.__init__ (model/sr3_modules/unet.py:161-233) + GaussianDiffusion.__init__ (diffusion.py:64-82):
 * builds the layer plan, allocates activations / packed weights on `device` for a fixed batch size.
 * Runs image_size x image_size images (sr3_engine_create_sized: other sizes).
 * The lowest UNet level (image_size / 2^(n_mults - 1)) must be at least 4x4; a net with a 4x4 level allocates its activations for the batch
 * rounded up to 8 images, but launches the work of the real images only.
 * Threading: calls on one engine must be serialised by the caller.  Kernels whose CTAs wait for partners are safe next to other work on the
 * device: the split-K partners of a tile are one thread-block cluster (gang-scheduled by the hardware) -- engines driven concurrently from
 * different streams of one device cannot deadlock each other. */
int sr3_engine_create(const sr3_unet_config* cfg, int batch, int device, sr3_engine** out);
/* The same inference plan for images of height x width instead of image_size x image_size: the reference UNet is fully convolutional and
 * runs whatever size it is given (unet.py:235-259; p_sample_loop takes its shape from x_in, diffusion.py:188-200).  cfg->image_size still
 * decides which levels get self-attention (unet.py:186-231: `now_res in attn_res` at construction); the attention itself runs over the
 * h * w tokens of the level it sits on.  Supported sizes: at every level (height and width halved n_mults - 1 times) both sides are powers
 * of two and at least 8, or the lowest level is exactly 4x4; anything else fails before any allocation.  The batch of a plan whose lowest
 * level is 4x4 is padded to 8 as above.  sr3_engine_create(cfg, ...) is sr3_engine_create_sized(cfg, ..., image_size, image_size, ...).
 * Every entry point below then reads and writes [B,C,height,width] images.  Training plans take the same sizes through
 * sr3_engine_create_train_sized. */
int sr3_engine_create_sized(const sr3_unet_config* cfg, int batch, int height, int width, int device, sr3_engine** out);
void sr3_engine_destroy(sr3_engine* e);

/* Parameter table in the reference's state_dict order and naming ("downs.1.res_block.block1.block.3.weight", ...;
 * keys are relative to denoise_fn).  shape has up to 4 entries (OIHW for convs). */
int sr3_engine_num_params(const sr3_engine* e);
int sr3_engine_param_info(const sr3_engine* e, int index, char* name, int name_cap, int64_t shape[4], int* ndim);
/* load_state_dict for one tensor (model/model.py:146-160): `src` is a DEVICE fp32 pointer in the reference layout.
 * Weights are re-packed (OIHW -> K-major bf16) by a kernel on `stream`. */
int sr3_engine_load_param(sr3_engine* e, const char* name, const float* src, int64_t numel, void* stream);
/* The whole state_dict in one call (srcs[i] = DEVICE fp32 pointer of parameter i in sr3_engine_param_info order) including the finalisation;
 * asynchronous on `stream`.  What the training loop calls after every optimizer step (model/model.py:58). */
int sr3_engine_load_all_params(sr3_engine* e, const float* const* srcs, int n, void* stream);
/* Must be called after the last load_param of a batch of updates (fuses bias vectors). */
int sr3_engine_finalize_params(sr3_engine* e, void* stream);

/* set_new_noise_schedule (model/sr3_modules/diffusion.py:92-139): HOST pointers to the fp32 buffers
 * sqrt_recip_alphas_cumprod, sqrt_recipm1_alphas_cumprod, posterior_mean_coef1, posterior_mean_coef2,
 * posterior_log_variance_clipped (each [T]) and the float64 sqrt_alphas_cumprod_prev ([T+1]). */
int sr3_engine_set_schedule(sr3_engine* e, int T, const float* sqrt_recip_ac, const float* sqrt_recipm1_ac, const float* post_coef1,
                            const float* post_coef2, const float* post_logvar, const double* sqrt_ac_prev, void* stream);

/* UNet.forward (model/sr3_modules/unet.py:235-259): x [B,in_channel,H,W], noise_level [B] (the reference's [B,1]) -> eps
 * [B,out_channel,H,W].  All DEVICE fp32. */
int sr3_unet_forward(sr3_engine* e, const float* x, const float* noise_level, float* eps, void* stream);

/* p_mean_variance (diffusion.py:151-167): x [B,3,H,W], condition_x [B,3,H,W] or NULL, integer t -> posterior mean
 * [B,3,H,W] (DEVICE) and the clipped log-variance (HOST scalar, may be NULL). */
int sr3_p_mean_variance(sr3_engine* e, const float* x, const float* condition_x, int t, int clip_denoised, float* mean, float* log_variance,
                        void* stream);

/* p_sample (diffusion.py:169-174): x_{t-1} = mean + exp(0.5 logvar) * z for t > 0.  `noise` (DEVICE [B,3,H,W]) replaces
 * torch.randn_like when non-NULL; otherwise z comes from Philox4x32-10 keyed by (seed, first_sample_index + b, pixel, t). */
int sr3_p_sample(sr3_engine* e, const float* x, const float* condition_x, int t, const float* noise, uint64_t seed,
                 uint64_t first_sample_index, float* x_prev, void* stream);

/* p_losses forward (diffusion.py:221-246) with the random draws injected: hr = x_in['HR'] [B,3,H,W], sr = x_in['SR'] (NULL when
 * unconditional), gamma [B] = continuous_sqrt_alpha_cumprod, noise [B,3,H,W] (all DEVICE fp32).  q_sample (diffusion.py:212-219),
 * the UNet and the summed L1 (loss_type 1) / L2 (2) loss (diffusion.py:84-90) run natively; *loss_host receives the scalar.
 * Forward value only: gradients come from the training entry points below. */
int sr3_p_losses(sr3_engine* e, const float* hr, const float* sr, const float* gamma, const float* noise, int loss_type, double* loss_host,
                 void* stream);

/* ---- training step: DDPM.optimize_parameters (model/model.py:48-58) = zero_grad -> GaussianDiffusion.forward / p_losses
 * (diffusion.py:221-249) in train() mode -> l_pix.sum() / (b c h w) -> backward -> Adam step (model.py:39-40).
 *
 * sr3_engine_create_train: as sr3_engine_create, for a fixed batch, with a plan that keeps every intermediate of the forward and has the
 * backward recorded next to it.  `dropout` = opt['model']['unet']['dropout'] (nn.Dropout in block2 of every ResnetBlock, unet.py:86,100-101);
 * bf16 precision only.  Inference entry points keep working on such an engine (eval-mode semantics are NOT applied: use a plain engine). */
int sr3_engine_create_train(const sr3_unet_config* cfg, int batch, int device, float dropout, sr3_engine** out);
/* The same training plan for images of height x width (p_losses takes its size from x_in['HR'], diffusion.py:221-246): the sizes, the
 * attention placement and the batch padding of sr3_engine_create_sized; an unsupported size fails before any device work.  The training
 * plan keeps every intermediate, and its attention scratch grows as (tokens per image)^2, so the plan's device bytes are counted before
 * anything is allocated: a plan larger than the device's free memory fails here, with a message naming the size, the batch and the bytes,
 * never in a step.  sr3_engine_create_train(cfg, ...) is sr3_engine_create_train_sized(cfg, ..., image_size, image_size, ...). */
int sr3_engine_create_train_sized(const sr3_unet_config* cfg, int batch, int height, int width, int device, float dropout, sr3_engine** out);
/* p_losses forward in training mode with the random draws injected (as sr3_p_losses): q_sample, UNet with Dropout (Philox keyed by
 * dropout_seed, or the masks given to sr3_train_set_dropout_mask), summed L1 / L2 loss -> *loss_host (may be NULL: no synchronisation). */
int sr3_train_forward(sr3_engine* e, const float* hr, const float* sr, const float* gamma, const float* noise, int loss_type, uint64_t dropout_seed,
                      double* loss_host, void* stream);
/* loss.backward() for the forward that just ran: grads[i] (DEVICE fp32, reference layout, one pointer per parameter in
 * sr3_engine_param_info order, n_grads == sr3_engine_num_params) is OVERWRITTEN with grad_scale * d(summed loss)/d(parameter i)
 * (grad_scale = 1 / (b c h w) reproduces model.py:50-53).  One backward per forward. */
int sr3_train_backward(sr3_engine* e, float grad_scale, float* const* grads, int n_grads, void* stream);
/* UNet.forward (model/sr3_modules/unet.py:235-259) in training form, on a training engine: x [B,in_channel,H,W] (for a conditional net the
 * already concatenated cat(cond, x_t)), noise_level [B] -> eps [B,out_channel,H,W], all DEVICE fp32 NCHW.  Every intermediate is kept for
 * sr3_train_unet_backward; Dropout as in sr3_train_forward (the plan's p, Philox keyed by dropout_seed, or the masks given to
 * sr3_train_set_dropout_mask).  Like sr3_train_forward it replaces whatever forward the engine ran before. */
int sr3_train_unet_forward(sr3_engine* e, const float* x, const float* noise_level, uint64_t dropout_seed, float* eps, void* stream);
/* The backward of the sr3_train_unet_forward that just ran, for an upstream gradient deps = d(anything)/d eps (DEVICE fp32 NCHW, eps's
 * shape; any scale is carried in deps).  grads as in sr3_train_backward (OVERWRITTEN, sr3_engine_param_info order).  dx [B,in_channel,H,W]
 * and dnoise_level [B] (DEVICE fp32) receive the gradients of the input and of the noise level; either may be NULL, and is then not
 * computed at all.  One backward per forward. */
int sr3_train_unet_backward(sr3_engine* e, const float* deps, float* const* grads, int n_grads, float* dx, float* dnoise_level, void* stream);
/* The same backward layer by layer, so that the caller can overlap the gradient all-reduce (SURVEY 8e, training row) with the layers still to
 * come: begin -> block n-1, n-2, ..., 0 -> finish (FiLM projections + noise-level MLP).  sr3_train_block_params lists the parameters whose
 * gradient is final once `block` has run AND sr3_train_backward_flush has been called (conv weight gradients leave the tensor-core kernel as
 * per-slice partial tiles; one table-driven launch per flush sums them) -- the rest (noise_func / block1 conv bias / noise_level_mlp) are
 * final after finish. */
int sr3_train_num_backward_blocks(const sr3_engine* e);
int sr3_train_backward_begin(sr3_engine* e, float grad_scale, float* const* grads, int n_grads);
int sr3_train_backward_block(sr3_engine* e, int block, void* stream);
int sr3_train_backward_flush(sr3_engine* e, void* stream);    /* reduce the weight-gradient partial tiles produced since the last flush (one launch) */
int sr3_train_backward_finish(sr3_engine* e, void* stream);
int sr3_train_block_params(const sr3_engine* e, int block, int* indices, int cap, int* n);
/* Profiling: the whole backward with CUDA events around every op; ms_by_kind[8]: device time per op kind (0 data-gradient tile kernel,
 * 1 GroupNorm / elementwise, 4 other, 6 weight gradient + slice reduction, 7 attention GEMMs). */
int sr3_train_backward_profile(sr3_engine* e, float grad_scale, float* const* grads, int n_grads, float* ms_by_kind, void* stream);
/* Tests: replace the Philox dropout mask of ResnetBlock `block_name` ("downs.1.res_block.block2", the module that owns the nn.Dropout) by a
 * keep-mask, uint8 DEVICE [B][C][H][W] (1 = keep), e.g. the one the reference drew; NULL restores Philox. */
int sr3_train_set_dropout_mask(sr3_engine* e, const char* block_name, const unsigned char* mask_nchw);
/* Tests, read-only: the FiLM state of a training engine's latest forward and backward, copied into DEVICE fp32 buffers of *rows images
 * (*rows = the batch the plan allocates: the batch, padded to even or, for a 4x4 lowest level, to a multiple of 8): tau [rows][inner] (the
 * noise-level embedding), dfilm [rows][F] (the per-image channel sums of the gradient of every ResnetBlock's FiLM output, the blocks'
 * slices in downs / mid / ups order, F their summed output channels) and dtau [rows][inner] (its gradient).  Any of the three may be NULL;
 * *rows and *F are always written. */
int sr3_test_train_film_state(const sr3_engine* e, float* tau, float* dfilm, float* dtau, int* rows, int* F, void* stream);
int sr3_train_num_dropout_layers(const sr3_engine* e);
int sr3_train_dropout_layer_name(const sr3_engine* e, int index, char* name, int name_cap);
/* torch.optim.Adam(lr, betas, eps, weight_decay 0) step `step` (1-based) over a DEVICE table of n_tensors records
 * {float* param; const float* grad; float* exp_avg; float* exp_avg_sq; int64 numel} (40 bytes each) in ONE launch; gradients are multiplied by
 * grad_scale first (1 / world_size after a summing all-reduce). */
int sr3_adam_step(const void* table_dev, int n_tensors, float lr, float beta1, float beta2, float eps, int step, float grad_scale, void* stream);

/* p_sample_loop / super_resolution / sample (diffusion.py:176-210): runs t = T-1 .. 0 as T launches of one captured CUDA
 * graph.  x_T: DEVICE [B,3,H,W] initial noise (the reference's torch.randn(shape)).  noises: optional DEVICE
 * [T][B,3,H,W], noises[i] used at step i.  Every (i % (1|T/10) == 0) the image is appended to `snapshots`
 * (DEVICE [n][B,3,H,W], capacity snapshot_cap images-batches; may be NULL) -- the `continous=True` return value without
 * its first B rows.  final: DEVICE [B,3,H,W] = x_0.  *n_snapshots receives the count. */
int sr3_p_sample_loop(sr3_engine* e, const float* condition_x, const float* x_T, const float* noises, uint64_t seed,
                      uint64_t first_sample_index, float* final, float* snapshots, int snapshot_cap, int* n_snapshots, void* stream);

/* Same loop on HOST buffers (H2D of condition_x / x_T, D2H of final inside): the end-to-end entry point. */
int sr3_super_resolution_host(sr3_engine* e, const float* condition_x_host, const float* x_T_host, uint64_t seed,
                              uint64_t first_sample_index, float* final_host, void* stream);

/* Run `steps` reverse steps starting at timestep t_start on the engine's resident state (benchmark / profiling hook:
 * no copies, no snapshots).  State must have been initialised by sr3_p_sample_loop_begin. */
int sr3_p_sample_loop_begin(sr3_engine* e, const float* condition_x, const float* x_T, uint64_t seed, uint64_t first_sample_index, void* stream);
int sr3_p_sample_steps(sr3_engine* e, int t_start, int steps, void* stream);
int sr3_read_state(sr3_engine* e, float* x_out, void* stream);

/* ---- windowed sampling: super-resolve a canvas of ANY size H >= window height, W >= window width with an engine of a supported window
 * size.  Each image of the canvas [B,3,H,W] is covered by overlapping windows (per axis: one window when the side equals the window's, else
 * n = ceil((L - overlap) / (side - overlap)) windows at origins round-half-up(i (L - side) / (n - 1))); the windows of all images form one list,
 * walked in passes of the engine's batch.  Every reverse step t merges the windows on the canvas:
 *   mean(p)    = sum_n w_n(p) mean_n(p) / sum_n w_n(p)   over the windows covering p in ascending index, fp32, mean_n = the clipped posterior
 *                mean of p_mean_variance on the window's crops of x_t and the condition;
 *   x_{t-1}(p) = mean(p) + exp(0.5 logvar_t) z(p)  (t > 0),  z from Philox keyed by (seed, first_sample_index + b, pixel index IN THE CANVAS, t)
 *                or from `noises`.
 * w_n(p) = wy(y) wx(x), w(i) = min(i + 1, side - i, ramp) / ramp with ramp = max(overlap, 1), the ramp towards a canvas border dropped.
 * A canvas of the window's size has one window of weight 1 and reproduces sr3_p_sample_loop bit for bit.  The result does not depend on the
 * engine's batch, and repeat runs are bit identical.  A whole canvas step is one CUDA graph (captured at the first step).
 * The canvas object owns the canvas state, a copy of the condition, the window means, the tables and the graph; it BORROWS the engine, which
 * must outlive it and must not run anything else between sr3_windowed_steps calls that belong together. */
typedef struct sr3_windowed sr3_windowed;
/* Fails before any allocation when the canvas is smaller than the engine's image size or an overlap is not in [0, side). */
int sr3_windowed_create(sr3_engine* e, int batch, int height, int width, int overlap_h, int overlap_w, sr3_windowed** out);
void sr3_windowed_destroy(sr3_windowed* w);
/* condition_x, x_T: DEVICE [B,3,H,W] (copied); as sr3_p_sample_loop_begin. */
int sr3_windowed_begin(sr3_windowed* w, const float* condition_x, const float* x_T, uint64_t seed, uint64_t first_sample_index, void* stream);
/* Where the following steps keep x_{t-1} of every t with t % (1 | T/10) == 0 (the `continous=True` images): DEVICE [snapshot_cap][B,3,H,W]
 * owned by the caller, first kept image first; NULL / 0: none. */
int sr3_windowed_set_snapshots(sr3_windowed* w, float* snapshots, int snapshot_cap);
/* `steps` canvas steps from timestep t_start down, graph launches only.  noises: optional DEVICE [T][B,3,H,W], noises[t] used at step t. */
int sr3_windowed_steps(sr3_windowed* w, int t_start, int steps, const float* noises, void* stream);
int sr3_windowed_read_state(sr3_windowed* w, float* x_out, void* stream);
/* The window grid: *ny, *nx windows per axis; optional HOST outputs origins_y [ny], origins_x [nx], weights_y [ny][window height],
 * weights_x [nx][window width]. */
int sr3_windowed_grid(const sr3_windowed* w, int* ny, int* nx, int* origins_y, int* origins_x, float* weights_y, float* weights_x);
/* Profiling: eager canvas steps at timestep t (Philox noise), CUDA events around the launches; ms[3] = device time per step of the gathers,
 * of the engine passes and of the merge, averaged over `reps` steps after one warm-up.  Advances the canvas state. */
int sr3_windowed_profile_step(sr3_windowed* w, int t, int reps, float* ms, void* stream);
/* DPM-Solver++(2M) on the canvas (added in ABI 5).  coefs: HOST [3][steps] (copied), rows A, B, C per step index k; steps = 0 (coefs may
 * be NULL) returns to the posterior-sample merge.  While set, the merge of the step at k blends the window means like the posterior-sample
 * merge, takes the blend as x0 (the engine's schedule must then have pc1 = 1, pc2 = 0 and `steps` entries) and writes
 *   x_{k-1} = (A_k x_k + B_k x0) + C_k x0_prev,   x0_prev = x0,
 * separately rounded in that order, with no noise; sr3_windowed_begin zeroes x0_prev.  sr3_windowed_steps refuses to run when `steps` is not
 * the engine's schedule length.  Refused for a ranged canvas. */
int sr3_windowed_set_solver(sr3_windowed* w, int steps, const float* coefs);

/* ---- windowed sampling sharded by window (one canvas on several GPUs).  A ranged canvas runs only windows [first_window, end_window) of
 * the list and stores their means into `means`, a DEVICE arena [N][3][window height][window width] of all N windows owned by the caller;
 * the caller fills the slots of the other windows it needs (the ones covering its band) between the two phases of every step.  `bands`:
 * optional HOST [batch][2] rows [y0, y1) per image the merge computes (copied; NULL: every row); the merge reads the means of every window
 * that covers a pixel of the band and nothing else, and the gathers read only the rows of the range's windows, so rows outside the band
 * may hold anything.  A step of a ranged canvas equals the same rows of a whole canvas's step bit for bit when the arena holds the same
 * means.  sr3_windowed_steps refuses a ranged canvas; sr3_windowed_profile_step profiles its range.  Ranged canvases may share one engine
 * when their phases are issued in order on one stream: every pass rewrites the engine's input and state. */
int sr3_windowed_create_range(sr3_engine* e, int batch, int height, int width, int overlap_h, int overlap_w, int first_window, int end_window,
                              float* means, const int* bands, sr3_windowed** out);
/* Starts a run of steps from timestep t_start down (Philox noise); then per step: phase_means (timestep advance, passes over the range,
 * means into the arena), the caller's exchange into the arena on or behind `stream`, phase_merge (merge of the band -> x_{t-1}).  Each phase
 * is one CUDA graph (captured at its first call); neither synchronises the host.  Calls out of this order are refused. */
int sr3_windowed_phase_begin(sr3_windowed* w, int t_start, void* stream);
int sr3_windowed_phase_means(sr3_windowed* w, void* stream);
int sr3_windowed_phase_merge(sr3_windowed* w, void* stream);

/* ---- continuous batching: serve a stream of requests of ANY size (each at least the engine's H x W, the window) on one inference
 * engine, every request at its own timestep.  A request is a canvas whose ny x nx overlapping windows (the grid and fp32 blend weights of
 * sr3_windowed_*, with the stream's overlap) take ny * nx of the engine's B slots, one window each; all windows of a request run at the
 * request's own timestep, windows of different requests at different timesteps share the batch.  Every request samples on its own noise
 * schedule: the engine's (sr3_engine_set_schedule), or one registered with sr3_wstream_add_schedule; requests on different schedules
 * share the batch.  A request on a schedule of T steps takes exactly T steps, one per sr3_wstream_step, and then waits for
 * sr3_wstream_retire.  A step is: a gather of every slot's window crop of its canvas (idle slots get zeros), the engine's step graph in its
 * UNet.forward form (noise level of slot s = sqrt_alphas_cumprod_prev[t + 1] of its request's schedule), the clipped posterior mean of
 * every running slot at its request's t, and a merge that blends the means on each canvas and adds sigma_t z with z from Philox keyed by
 * (seed, the request's sample_index, the pixel's index in its canvas, t), writing x_{t-1} into the canvas.
 * Bit-exactness: a request's x_0 equals what sr3_windowed_* computes for that canvas alone as image 0 with first_sample_index =
 * sample_index on an engine of the same shape, after sr3_engine_set_schedule of the request's schedule, with its windows in the same slots,
 * bit for bit, whatever the other slots hold and whenever it was admitted (every UNet op is per image; the means and the merge are the
 * windowed sampler's arithmetic operation for operation, and both calls build the schedule's tables with the same host routine).
 * A window-sized request (one window, weight 1) in slot b equals what sr3_p_sample_loop computes for the same condition, x_T and
 * first_sample_index + b = sample_index at image b, bit for bit.  Whether the slots matter depends on the plan: on a 4x4-lowest-level
 * plan a window moved to another slot changes within rounding.
 * No step synchronises the host, copies to it or allocates: the host mirrors the request table, since every request takes exactly the
 * T steps of its schedule.
 * The stream BORROWS the engine (which must outlive it; nothing else may run on it while requests are in flight, and all calls of one
 * stream go to one CUDA stream) and every admitted canvas until its request is retired.  Creating a stream zeroes the engine's state
 * and input.  Refused at creation: a training engine, an overlap outside [0, window side). */
typedef struct sr3_wstream sr3_wstream;
int sr3_wstream_create(sr3_engine* e, uint64_t seed, int overlap_h, int overlap_w, sr3_wstream** out);
void sr3_wstream_destroy(sr3_wstream* s);
/* Register a noise schedule of T steps for this stream's requests: the arrays, their meaning and the T range of sr3_engine_set_schedule
 * (HOST, fp32 [T] each, sqrt_ac_prev fp64 [T + 1]).  *schedule = its id (0, 1, ... in registration order).  The device tables are allocated
 * here, never in a step, and freed by sr3_wstream_destroy; the call synchronises `stream`.  Allowed while requests are in flight; a
 * request on a registered schedule is unaffected by sr3_engine_set_schedule.  Refused, with nothing registered: a null table, T outside
 * [1, the engine's maximum]. */
int sr3_wstream_add_schedule(sr3_wstream* s, int T, const float* sqrt_recip_ac, const float* sqrt_recipm1_ac, const float* post_coef1,
                             const float* post_coef2, const float* post_logvar, const double* sqrt_ac_prev, int* schedule, void* stream);
/* Admit one request into the n_slots free slots `slots` (HOST, window k of the grid, row-major, into slots[k]).  condition_x: DEVICE fp32
 * [cond_c][height][width] (NULL for an unconditional model), x: DEVICE fp32 [3][height][width] holding x_T, overwritten with x_{t-1} by
 * every step and holding x_0 once the request has finished; both are BORROWED until sr3_wstream_retire, nothing is copied but the window geometry.  *request = the request's
 * id; it samples on the engine's schedule and its first step runs at t = T - 1.  Refused, with no slot or request changed: a slot out of
 * range, busy or listed twice, n_slots other than the canvas's window count, a canvas smaller than the window, a null x, a condition
 * missing for a conditional model or given to an unconditional one, an engine with no schedule, the engine's schedule changed since the
 * requests in flight on it were admitted.  sr3_wstream_admit_scheduled with schedule -1. */
int sr3_wstream_admit(sr3_wstream* s, const int* slots, int n_slots, const float* condition_x, float* x, int height, int width,
                      uint64_t sample_index, int* request, void* stream);
/* sr3_wstream_admit of a request that samples on registered schedule `schedule` of T_S steps (-1: the engine's schedule): its first step
 * runs at t = T_S - 1 and it finishes T_S steps later.  Also refused: an unknown schedule id. */
int sr3_wstream_admit_scheduled(sr3_wstream* s, const int* slots, int n_slots, const float* condition_x, float* x, int height, int width,
                                uint64_t sample_index, int schedule, int* request, void* stream);
/* One reverse step of every running request.  Refused when the engine has no schedule or sr3_engine_set_schedule was called while
 * requests on the engine's schedule are in flight (they would finish on a mixed schedule); requests on registered schedules do not count. */
int sr3_wstream_step(sr3_wstream* s, void* stream);
/* Free the slots of a finished request and end the borrow of its canvases (x holds x_0).  Refuses a running request or an id not held. */
int sr3_wstream_retire(sr3_wstream* s, int request, void* stream);
/* HOST request[B], t[B], state[B] per slot: the request it runs (-1: free), the request's t (timestep of its next step; -1 once finished)
 * and state 0 free, 1 running, 2 finished and not yet retired. */
int sr3_wstream_slot_state(const sr3_wstream* s, int* request, int* t, int* state);

/* core/metrics.py:8-34 `tensor2img` on the device: src fp32 DEVICE [n][C][H][W] -> clamp to [min_v, max_v] -> [0, 1] -> * 255, round half
 * to even -> uint8 DEVICE, HWC.  n == 1: dst [H][W][C].  n > 1: the images are tiled like torchvision.utils.make_grid(nrow, padding 2,
 * pad_value 0), which is what the reference does for 4-D input: dst [rows*(H+2)+2][cols*(W+2)+2][C], cols = min(nrow, n).
 * Saves the D2H of fp32 snapshots (model.py:98-110 get_current_visuals + sr.py): a quarter of the bytes cross PCIe. */
int sr3_tensor2img(const float* src, unsigned char* dst_u8, int n, int C, int H, int W, int nrow, float min_v, float max_v, void* stream);
/* core/metrics.py:42-50 `calculate_psnr`: exact integer sum of squared differences of two uint8 DEVICE images (n elements) -> *ssd_host;
 * PSNR = 20 log10(255 / sqrt(ssd / n)) is formed by the caller in float64 as the reference does. */
int sr3_ssd_u8(const unsigned char* a_u8, const unsigned char* b_u8, int64_t n, unsigned long long* ssd_host, void* stream);
/* core/metrics.py:52-72 `ssim` of n image pairs: a, b DEVICE [n][H][W][C] (HWC; dtype 0 uint8, 1 float64) -> ssim_host[n] (HOST).  fp64
 * throughout: the 11x11 Gaussian window (sigma 1.5) as two separable passes over x, y, x^2, y^2, xy, valid pixels only, each channel on its
 * own, mean over every kept pixel of every channel; NaN when H or W is below 11.  The work split depends on (H, W, C) only: a pair scores
 * bit-identically alone or inside any batch.  calculate_ssim (:75-93) is formed by the caller. */
int sr3_ssim(const void* a, const void* b, int dtype, int n, int H, int W, int C, double* ssim_host, void* stream);
/* The evaluation of a sampled batch (sr.py:216-217 for every image): tensor2img (as sr3_tensor2img with n == 1) of each of the n images of
 * sr_f32 and hr_f32 (DEVICE fp32 [n][C][H][W]) into uint8 [n][H][W][C] (sr_u8 / hr_u8 DEVICE, or NULL: internal scratch), then per pair
 * the sr3_ssd_u8 sum (ssd_host[n]) and the sr3_ssim value (ssim_host[n]), in one call with one device-to-host copy. */
int sr3_image_metrics(const float* sr_f32, const float* hr_f32, int n, int C, int H, int W, float min_v, float max_v, unsigned char* sr_u8,
                      unsigned char* hr_u8, unsigned long long* ssd_host, double* ssim_host, void* stream);

/* Entrance of the path: the conditioning image.  data/prepare_data.py:17-40 `trans_fn.resize(img, size, Image.BICUBIC)` (Pillow's two-pass
 * fixed-point bicubic resampler on uint8) + data/util.py:74-83 `transform_augment` (ToTensor, optional horizontal flip, range mapping).
 * src uint8 DEVICE [B][h][w][C] (HWC); dst_u8 (optional) uint8 DEVICE [B][H][W][C]; dst_f32 (optional) fp32 DEVICE [B][C][H][W] =
 * (resized / 255) * (max_v - min_v) + min_v, mirrored along W when flip != 0.  Integer-exact against Pillow 12. */
/* Host-only helper: Pillow's integer coefficient tables of one bicubic pass in_size -> out_size (bounds [out][2] = first tap, tap count;
 * coef [out][ksize], 22 fractional bits). */
int sr3_pil_bicubic_tables(int in_size, int out_size, int* bounds, int* coef, int coef_cap, int* ksize);
int sr3_resize_bicubic_u8(const unsigned char* src_u8, unsigned char* dst_u8, float* dst_f32, int B, int h, int w, int C, int H, int W, int flip,
                          float min_v, float max_v, void* stream);

/* Introspection for tests / bench. */
int sr3_engine_num_launches_per_step(const sr3_engine* e);   /* kernel launches per reverse step (the nodes of the captured step graph) */
int sr3_engine_num_ops_per_step(const sr3_engine* e);        /* ops of the step plan, one launch each (what sr3_engine_profile_step times) */
int64_t sr3_engine_workspace_bytes(const sr3_engine* e);
/* Per-kernel timing of one eager (non-graph) reverse step at timestep t, averaged over `reps` repetitions after one warm-up,
 * CUDA events on `stream` around every launch.  kinds: 0 tensor-core tile kernel, 1 GroupNorm apply, 2 cast/upsample,
 * 3 softmax, 4 other, 5 fused attention core (flops: the algorithmic 4 nz Lt^2 C, not the recomputed S); flops / bytes are otherwise the
 * executed work of each launch.  Does not modify the sampler state. */
int sr3_engine_profile_step(sr3_engine* e, int t, int reps, int cap, int* kinds, float* ms, double* flops, double* bytes, int* n_ops,
                            void* stream);
/* Debug tap: copy the fp32 NHWC output of top-level layer `name` ("downs.3", "mid.0", ...) of the last forward to dst
 * (DEVICE, [B,H,W,C]); returns C*H*W*B through *numel.  The tap of a layer with self-attention is the attention's output; the output of
 * its ResnetBlock, the attention's input, is the tap "<layer>.res_block" ("mid.0.res_block"). */
int sr3_engine_read_activation(sr3_engine* e, const char* name, float* dst, int64_t cap, int64_t* numel, int shape_bhwc[4], void* stream);
/* Tests, read-only: the gradient a training engine's latest backward left for the tensor of tap `name` (the names of
 * sr3_engine_read_activation), the first B images, into DEVICE fp32 dst.  form 0: g, the fp32 gradient, NHWC [B,H,W,C]; form 1: gb, its
 * bf16 copy (the operand of the producing layer's data and weight gradients), widened to fp32, [B,H,W,C]; form 2: gsum, its per-image
 * channel sums (the bias gradients), [B,C] (shape_bhwc {B, 1, 1, C}).  *numel and shape_bhwc are written whether or not dst is given.
 * Refused on an engine not created for training, which keeps no gradients.  Synchronises `stream`. */
int sr3_test_read_gradient(sr3_engine* e, const char* name, int form, float* dst, int64_t cap, int64_t* numel, int shape_bhwc[4], void* stream);

/* Stand-alone tile GEMM for unit tests: D[M,N] = A[M,K] * B[N,K]^T (bf16 row-major DEVICE inputs, fp32 output), M%128==0,
 * K%64==0, N%block_n==0. */
int sr3_test_gemm(const void* a_bf16, const void* b_bf16, float* d, int M, int N, int K, int block_n, void* stream);
/* Test hook for the fused attention core (S = q k^T / sqrt(C), softmax per image, O = P v; unet.py:129-139): qk bf16 [nz*Lt][2C]
 * (q | k), vT bf16 [nz*C][Lt], out bf16 [nz*Lt][C]; Lt keys per attention batch (a multiple of 128), HW tokens per image (Lt % HW == 0; above 256 keys
 * HW == Lt and the streaming-softmax kernel runs). */
int sr3_test_attention(const void* qk_bf16, const void* vT_bf16, void* out_bf16, int nz, int Lt, int HW, int C, void* stream);
/* sr3_test_attention with attn_kernel's channel slice forced: dn = 64, 128 or 256 output channels per CTA (Lt <= 256, C % dn == 0), or
 * 0 for the one make_attn_op picks.  Any dn computes the same bits. */
int sr3_test_attention_dn(const void* qk_bf16, const void* vT_bf16, void* out_bf16, int nz, int Lt, int HW, int C, int dn, void* stream);
/* The channel slice the fused attention core runs at for nz attention batches of Lt keys and C channels on a GPU of `sms` SMs
 * (sms <= 0: the current device's): the fewest waves of one CTA per SM, then the narrowest slice. */
int sr3_attention_dn(int nz, int Lt, int C, int sms, int* dn);
/* Test hook for the unfused attention path (precise mode, training), the plan's three launches:
 * S = q k^T / sqrt(C) on the tile kernel, softmax_kernel over the keys of each image, O = P v on the tile kernel.  qk bf16 [nz*Lt][2C PW]
 * (rows [q | k], precise = 1: [q_hi | k_hi | q_lo | k_lo]), vT bf16 [nz*C][Lt PW] -> S fp32 [nz*Lt][Lt], P bf16 [nz*Lt][Lt PW],
 * O bf16 [nz*Lt][C PW]; PW = 2 in precise mode (rows [hi | lo]), else 1.  Lt % 128 == 0, C % 128 == 0, HW tokens per image (Lt % HW == 0). */
int sr3_test_attention_unfused(const void* qk_bf16, const void* vT_bf16, float* S, void* P_bf16, void* O_bf16, int nz, int Lt, int HW, int C,
                               int precise, void* stream);
/* Stand-alone NHWC conv for unit tests: x bf16 [B,H,W,Cin], w fp32 OIHW [Cout,Cin,k,k] (k in {1,3}), stride in {1,2},
 * y fp32 [B,OH,OW,Cout]; stats (optional) fp64 [B,Cout,2] (sum, sum of squares per image and channel: the GroupNorm statistics of
 * unet.py:84, accumulated with order-independent fp64 atomics) must be zeroed by the caller. */
int sr3_test_conv(const void* x_bf16, const float* w_oihw, const float* bias, float* y, double* stats, int B, int H, int W, int Cin,
                  int Cout, int ksize, int stride, void* stream);

/* The tile-kernel variant and launch shape one conv actually ran with (after every SR3_* override and host-side cap): tall-halo form,
 * 128-row halves per tile, BLOCK_N, the tile's pixel box (h_box rows x b_box images), split-K factor, pipeline stages, grid CTAs, output
 * tiles (times the z phases), and whether the residual was staged through shared memory by TMA (0: plain loads). */
typedef struct sr3_gemm_geometry {
    int tall, mh, block_n, h_box, b_box, ksplit, stages, ctas, tiles, res_smem;
} sr3_gemm_geometry;
/* One image conv exactly as a UNet layer builds it, every operand on the DEVICE:
 *   y = conv(x, w) [+ conv1x1(x2, w2)] + bias + bias2[image] + resid,   y fp32 NHWC [B][OH][OW][Cout]
 * x bf16 NHWC [B][H][W][Cin]; w fp32 OIHW [Cout][Cin][k][k]; optional: bias [Cout], bias2 [B][Cout] (per-image FiLM bias), resid fp32 NHWC
 * like y, a second A source x2 bf16 NHWC [B][H][W][Cin2] whose 1x1 conv w2 [Cout][Cin2][1][1] is appended as extra K columns (ResnetBlock
 * block2 + res_conv), y_bf16 = bf16(y) NHWC, stats fp64 [B][Cout][2] zeroed by the caller.
 * fold_up = 1: the Upsample conv, nearest 2x then conv3x3 (Cin == Cout, stride 1), run as the merged four-phase op on the folded weights;
 * y is then [B][2H][2W][Cout].  precise = 1: x / x2 rows are [hi | lo] (2 Cin channels: hi = bf16(v), lo = bf16(v - hi)), three tensor-core
 * passes, y_bf16 rows [hi | lo] of 2 Cout.  geometry (optional) receives the variant that ran. */
typedef struct sr3_test_conv_args {
    const void* x; const float* w; const float* bias; const float* bias2; const float* resid;
    const void* x2; const float* w2;
    float* y; void* y_bf16; double* stats;
    int B, H, W, Cin, Cout, Cin2, ksize, stride;
    int fold_up, precise;
} sr3_test_conv_args;
int sr3_test_conv_ex(const sr3_test_conv_args* args, sr3_gemm_geometry* geometry, void* stream);
/* Schedule of a tile-kernel launch: *schedule = 0 cooperative (both consumer warpgroups share every tile), 1 ping-pong (each warpgroup owns
 * whole tiles and its epilogue overlaps the other one's MMAs), -1 op `op` is not a tile-kernel launch.  e = NULL: the most recent
 * sr3_test_conv_ex call of the calling thread (`op` ignored); otherwise op `op` of e's eager step, indexed as sr3_engine_profile_step
 * reports them.  geometry and out_hwc (output rows, columns, channels; optional) receive the rest of the launch. */
int sr3_tile_schedule(const sr3_engine* e, int op, sr3_gemm_geometry* geometry, int* schedule, int* out_hwc);
/* Weight gradient of one conv through wgrad_kernel + wgrad_reduce_kernel (the training plan's path): dy bf16 NHWC [B][OH][OW][CY], x bf16
 * NHWC [B][OH*stride][OW*stride][Cin]; k = 1 (stride 1) or 3 (stride 1 or 2, padding 1).  grad fp32 OIHW [cout_valid][cin_valid][k][k] =
 * gscale * dW over the first cout_valid / cin_valid channels.  slices = 0: the training plan's slice count; *slices_used (optional) reports it.
 * raw = 1: the batched form of the attention backward (k = 1, every channel): grad [B][CY][Cin], image b alone contracted into slice b, no
 * reduction and no gscale. */
int sr3_test_wgrad(const void* dy_bf16, const void* x_bf16, float* grad, int B, int OH, int OW, int CY, int Cin, int ksize, int stride,
                   int cout_valid, int cin_valid, int slices, float gscale, int raw, int* slices_used, void* stream);

/* Test hook for the GroupNorm path of a Block (unet.py:80-91): y = conv(x) + bias with the statistics taken in the conv epilogue, then
 * a = [silu](GroupNorm(y; groups, gamma, beta, eps 1e-5)) as bf16 NHWC.  Shapes as sr3_test_conv (stride 1). */
int sr3_test_conv_groupnorm(const void* x_bf16, const float* w_oihw, const float* bias, const float* gamma, const float* beta, int groups,
                            int silu, float* y, void* a_bf16, int B, int H, int W, int Cin, int Cout, int ksize, void* stream);

/* ---- kernel-level hooks of the training backward: each builds its launches with the training plan's own helpers (csrc/train_plan.inc).
 * Every pointer is DEVICE memory; tensors are NHWC with HW = H * W pixels per image. */

/* One GroupNorm (+SiLU, +Dropout) layer of a ResnetBlock / attention / final Block as the plan pairs its forward and backward:
 * prep_kernel (a = drop(silu(GN(cat(x0, x1)))) as bf16, saving (mean, rstd)), then both passes of gn_bwd_kernel given dA.
 *   x0 fp32 [B][HW][C0], x1 (optional) fp32 [B][HW][C1]; st0 / st1 fp64 [B][C][2] (channel sum, sum of squares);
 *   drop: 0 none, 1 Philox keyed by (drop_seed; vector index, drop_layer), 2 the uint8 keep-mask drop_mask [B][C0+C1][HW] (NCHW);
 *   dA fp32 [B][HW][C0+C1]; add (optional) fp32 [B][HW][add_ld] (its first C0 + C1 channels are added to the input gradient);
 *   outputs: a_bf16 [B][HW][C0+C1], mr [B][groups][2], dst0 fp32 [B][HW][C0] (acc0: added to what it holds), dst0_b (optional) bf16(dst0),
 *   gsum0 (optional, zeroed by the caller) [B][C0] += per-image channel sums of dst0, dst1 (optional) fp32 [B][HW][C1] (stored),
 *   dgamma / dbeta [C0+C1] = gscale * the parameter gradients. */
typedef struct sr3_test_groupnorm_args {
    const float* x0; const float* x1; const double* st0; const double* st1; const float* gamma; const float* beta;
    const unsigned char* drop_mask; const float* dA; const float* add;
    void* a_bf16; float* mr; float* dst0; void* dst0_b; float* gsum0; float* dst1; float* dgamma; float* dbeta;
    uint64_t drop_seed;
    int B, HW, C0, C1, groups, silu, drop, add_ld, acc0;
    unsigned int drop_layer;
    float drop_p, gscale;
} sr3_test_groupnorm_args;
int sr3_test_groupnorm_layer(const sr3_test_groupnorm_args* args, void* stream);
/* grad_combine_kernel: out = a (+ b) fp32 [B][HW][C]; dst (optional) = out, or += out when acc; dst_b (optional) = bf16 of it; gsum (optional,
 * zeroed by the caller) [B][C] += its per-image channel sums.  Then, when bias0 is given, bias_grad_kernel: bias0 (and bias1) [C] =
 * gscale * sum over images of gsum. */
int sr3_test_grad_combine(const float* a, const float* b, float* dst, int acc, void* dst_b, float* gsum, float* bias0, float* bias1, float gscale,
                          int B, int HW, int C, void* stream);
/* Data gradient of a conv on the tile kernel, its weight packed on the device from w (fp32 OIHW) as the plan packs it.  dx fp32
 * [B][H][W][Cin] (H, W: the conv's input size).  form 0: stride-1 k x k conv Cin -> Cout, dy bf16 [B][H][W][CY] (CY = Cout rounded up to a multiple
 * of 64: the final conv's 3 channels sit in a 64-channel buffer); form 1: Downsample (3x3 stride 2, C -> C), dy bf16 [B][H/2][W/2][C];
 * form 2: Upsample (nearest 2x then 3x3, C -> C), dy bf16 [B][2H][2W][C]. */
int sr3_test_dgrad(const void* dy_bf16, const float* w_oihw, float* dx, int form, int B, int H, int W, int CY, int Cin, int Cout, int ksize,
                   void* stream);
/* Attention backward from the transposes to the bf16 copy of d(qkv), nz batches of Lt tokens (HW per image), head dim C:
 * qk bf16 [nz*Lt][2C] (q | k), vT bf16 [nz*C][Lt], P bf16 [nz*Lt][Lt] (the forward's softmax), dO bf16 [nz*Lt][C] ->
 * dS fp32 [nz*Lt][Lt], dS_b bf16 [nz*Lt][Lt], dqkv fp32 [nz*Lt][3C] (dQ | dK | dV), dqkv_b bf16 of it. */
int sr3_test_attention_bwd(const void* qk_bf16, const void* vT_bf16, const void* P_bf16, const void* dO_bf16, float* dS, void* dS_bf16, float* dqkv,
                           void* dqkv_bf16, int nz, int Lt, int HW, int C, void* stream);
/* FiLM projections + noise-level MLP backward (film_bwd_kernel into a zeroed dtau, then embed_bwd_kernel): film = W_f tau(nl) + b_f + cb,
 * tau(nl) = W2 swish(W1 PE(nl) + b1) + b2, inner = tau's width, hidden 4 inner.  wf [F][inner], tau [B][inner], dfilm [B][F], nl [B],
 * w1 [4 inner][inner], b1 [4 inner], w2 [inner][4 inner] -> dwf, dbf, dcb, dtau [B][inner], dw1, db1, dw2, db2 (all but dtau times gscale). */
typedef struct sr3_test_film_args {
    const float* wf; const float* tau; const float* dfilm; const float* nl; const float* w1; const float* b1; const float* w2;
    float* dwf; float* dbf; float* dcb; float* dtau; float* dw1; float* db1; float* dw2; float* db2;
    int F, inner, B;
    float gscale;
} sr3_test_film_args;
int sr3_test_film_embed_bwd(const sr3_test_film_args* args, void* stream);
/* The forward of the same two layers as the plan launches them (embed_kernel, then film_kernel): nl [B] (one noise level per image),
 * w1 [4 inner][inner], b1 [4 inner], w2 [inner][4 inner], b2 [inner], wf [F][inner], bf [F], cb [F] (block1 conv biases) ->
 * tau [B][inner], film [B][F] = wf tau + bf + cb.  Any batch that fits in device memory. */
int sr3_test_film_embed_fwd(const float* nl, const float* w1, const float* b1, const float* w2, const float* b2, const float* wf, const float* bf,
                            const float* cb, float* tau, float* film, int F, int inner, int B, void* stream);
/* loss_grad_kernel: noise, eps fp32 NCHW [B][C][H][W] (H * W a multiple of 32) -> *loss_host = sum |eps - noise| (l2 = 0) or
 * sum (eps - noise)^2 (l2 = 1); deps bf16 [B][H][W][ld] channels 0..C-1 = sign(d) or 2 d (the rest untouched); bias_sum [C] += its sums. */
int sr3_test_loss_grad(const float* noise, const float* eps, int B, int C, int H, int W, int l2, double* loss_host, void* deps_bf16, int ld,
                       float* bias_sum, void* stream);
/* grad_load_kernel, the start of sr3_train_unet_backward: g fp32 NCHW [B][C][H][W] -> deps bf16 [B][H][W][ld] channels 0..C-1 = bf16(g) (the
 * rest untouched); bias_sum [C] += the fp32 sums of g. */
int sr3_test_grad_load(const float* g, int B, int C, int H, int W, void* deps_bf16, int ld, float* bias_sum, void* stream);
/* noise_level_bwd_kernel: the gradient of the noise level through the positional encoding and the noise-level MLP, given dtau [B][inner]
 * (the gradient of its output): nl [B], w1 [4 inner][inner], b1 [4 inner], w2 [inner][4 inner] -> dnl [B]. */
int sr3_test_noise_level_bwd(const float* nl, const float* w1, const float* b1, const float* w2, const float* dtau, float* dnl, int inner, int B,
                             void* stream);
/* The input gradient of sr3_train_unet_backward: the data gradient of the first conv (in_channel -> inner, 3x3, padding 1; w fp32 OIHW
 * [inner][in_channel][3][3], packed on the device as the plan packs it) on the tile kernel, then the store of its first in_channel channels:
 * dy bf16 NHWC [B][H][W][inner] -> dx fp32 NCHW [B][in_channel][H][W]. */
int sr3_test_input_grad(const void* dy_bf16, const float* w_oihw, float* dx, int B, int H, int W, int inner, int in_channel, void* stream);

/* Timing harness for one conv shape on zero-filled buffers (kernel-tuning experiments): average ms over `reps` launches. */
int sr3_bench_conv(int B, int H, int W, int Cin, int Cout, int ksize, int stride, int with_resid, int with_stats, int reps, float* ms_out);
/* Timing harness for the fused attention core (operands as sr3_test_attention, dn as sr3_test_attention_dn): average ms over `reps`
 * launches captured in one graph; out holds the result. */
int sr3_bench_attention(const void* qk_bf16, const void* vT_bf16, void* out_bf16, int nz, int Lt, int HW, int C, int dn, int reps, float* ms_out);

#ifdef __cplusplus
}
#endif
#endif /* SR3_B200_H */
