"""ctypes binding of libsr3_b200.so (include/sr3_b200.h).  torch is used only for device memory and streams."""
import contextlib
import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int64, c_uint64, c_void_p

import torch

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "lib", "libsr3_b200.so")
SR3_MAX_LEVELS = 8
_lib = None


class NativeLibraryError(RuntimeError):
    pass


class UNetConfigC(ctypes.Structure):
    _fields_ = [("in_channel", c_int), ("out_channel", c_int), ("inner_channel", c_int), ("norm_groups", c_int),
                ("n_mults", c_int), ("channel_mults", c_int * SR3_MAX_LEVELS), ("n_attn_res", c_int),
                ("attn_res", c_int * SR3_MAX_LEVELS), ("res_blocks", c_int), ("image_size", c_int), ("channels", c_int),
                ("conditional", c_int), ("precision", c_int)]


PRECISIONS = {"bf16": 0, "fp32": 1}          # "fp32" = precise mode: (hi, lo) bf16 operand pairs, three tensor-core passes


class GemmGeometryC(ctypes.Structure):
    _fields_ = [(n, c_int) for n in ("tall", "mh", "block_n", "h_box", "b_box", "ksplit", "stages", "ctas", "tiles", "res_smem")]


class TestConvArgsC(ctypes.Structure):
    _fields_ = [("x", c_void_p), ("w", c_void_p), ("bias", c_void_p), ("bias2", c_void_p), ("resid", c_void_p),
                ("x2", c_void_p), ("w2", c_void_p),
                ("y", c_void_p), ("y_bf16", c_void_p), ("stats", c_void_p)] + \
               [(n, c_int) for n in ("B", "H", "W", "Cin", "Cout", "Cin2", "ksize", "stride", "fold_up", "precise")]


class TestGroupNormArgsC(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in ("x0", "x1", "st0", "st1", "gamma", "beta", "drop_mask", "dA", "add", "a_bf16", "mr", "dst0", "dst0_b",
                                         "gsum0", "dst1", "dgamma", "dbeta")] + \
               [("drop_seed", c_uint64)] + [(n, c_int) for n in ("B", "HW", "C0", "C1", "groups", "silu", "drop", "add_ld", "acc0")] + \
               [("drop_layer", ctypes.c_uint), ("drop_p", c_float), ("gscale", c_float)]


class TestFilmArgsC(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in ("wf", "tau", "dfilm", "nl", "w1", "b1", "w2", "dwf", "dbf", "dcb", "dtau", "dw1", "db1", "dw2", "db2")] + \
               [(n, c_int) for n in ("F", "inner", "B")] + [("gscale", c_float)]


_SIGS = {
    "sr3_last_error": (c_char_p, []),
    "sr3_abi_version": (c_int, []),
    "sr3_engine_create": (c_int, [POINTER(UNetConfigC), c_int, c_int, POINTER(c_void_p)]),
    "sr3_engine_create_sized": (c_int, [POINTER(UNetConfigC), c_int, c_int, c_int, c_int, POINTER(c_void_p)]),
    "sr3_engine_create_train": (c_int, [POINTER(UNetConfigC), c_int, c_int, c_float, POINTER(c_void_p)]),
    "sr3_engine_create_train_sized": (c_int, [POINTER(UNetConfigC), c_int, c_int, c_int, c_int, c_float, POINTER(c_void_p)]),
    "sr3_train_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_uint64, POINTER(c_double), c_void_p]),
    "sr3_train_backward": (c_int, [c_void_p, c_float, POINTER(c_void_p), c_int, c_void_p]),
    "sr3_train_unet_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_uint64, c_void_p, c_void_p]),
    "sr3_train_unet_backward": (c_int, [c_void_p, c_void_p, POINTER(c_void_p), c_int, c_void_p, c_void_p, c_void_p]),
    "sr3_train_num_backward_blocks": (c_int, [c_void_p]),
    "sr3_train_backward_begin": (c_int, [c_void_p, c_float, POINTER(c_void_p), c_int]),
    "sr3_train_backward_block": (c_int, [c_void_p, c_int, c_void_p]),
    "sr3_train_backward_flush": (c_int, [c_void_p, c_void_p]),
    "sr3_train_backward_finish": (c_int, [c_void_p, c_void_p]),
    "sr3_train_block_params": (c_int, [c_void_p, c_int, POINTER(c_int), c_int, POINTER(c_int)]),
    "sr3_train_backward_profile": (c_int, [c_void_p, c_float, POINTER(c_void_p), c_int, POINTER(c_float), c_void_p]),
    "sr3_train_set_dropout_mask": (c_int, [c_void_p, c_char_p, c_void_p]),
    "sr3_test_train_film_state": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int), POINTER(c_int), c_void_p]),
    "sr3_train_num_dropout_layers": (c_int, [c_void_p]),
    "sr3_train_dropout_layer_name": (c_int, [c_void_p, c_int, c_char_p, c_int]),
    "sr3_adam_step": (c_int, [c_void_p, c_int, c_float, c_float, c_float, c_float, c_int, c_float, c_void_p]),
    "sr3_engine_destroy": (None, [c_void_p]),
    "sr3_engine_num_params": (c_int, [c_void_p]),
    "sr3_engine_param_info": (c_int, [c_void_p, c_int, c_char_p, c_int, POINTER(c_int64), POINTER(c_int)]),
    "sr3_engine_load_param": (c_int, [c_void_p, c_char_p, c_void_p, c_int64, c_void_p]),
    "sr3_engine_load_all_params": (c_int, [c_void_p, POINTER(c_void_p), c_int, c_void_p]),
    "sr3_engine_finalize_params": (c_int, [c_void_p, c_void_p]),
    "sr3_engine_set_schedule": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "sr3_unet_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "sr3_p_mean_variance": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, POINTER(c_float), c_void_p]),
    "sr3_p_sample": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_uint64, c_uint64, c_void_p, c_void_p]),
    "sr3_p_losses": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, POINTER(c_double), c_void_p]),
    "sr3_p_sample_loop": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint64, c_uint64, c_void_p, c_void_p, c_int,
                                  POINTER(c_int), c_void_p]),
    "sr3_super_resolution_host": (c_int, [c_void_p, c_void_p, c_void_p, c_uint64, c_uint64, c_void_p, c_void_p]),
    "sr3_p_sample_loop_begin": (c_int, [c_void_p, c_void_p, c_void_p, c_uint64, c_uint64, c_void_p]),
    "sr3_p_sample_steps": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "sr3_read_state": (c_int, [c_void_p, c_void_p, c_void_p]),
    "sr3_windowed_create": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, POINTER(c_void_p)]),
    "sr3_windowed_destroy": (None, [c_void_p]),
    "sr3_windowed_begin": (c_int, [c_void_p, c_void_p, c_void_p, c_uint64, c_uint64, c_void_p]),
    "sr3_windowed_set_snapshots": (c_int, [c_void_p, c_void_p, c_int]),
    "sr3_windowed_steps": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "sr3_windowed_read_state": (c_int, [c_void_p, c_void_p, c_void_p]),
    "sr3_windowed_grid": (c_int, [c_void_p, POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_float), POINTER(c_float)]),
    "sr3_windowed_profile_step": (c_int, [c_void_p, c_int, c_int, POINTER(c_float), c_void_p]),
    "sr3_windowed_set_solver": (c_int, [c_void_p, c_int, c_void_p]),
    "sr3_windowed_create_range": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, POINTER(c_int), POINTER(c_void_p)]),
    "sr3_windowed_phase_begin": (c_int, [c_void_p, c_int, c_void_p]),
    "sr3_windowed_phase_means": (c_int, [c_void_p, c_void_p]),
    "sr3_windowed_phase_merge": (c_int, [c_void_p, c_void_p]),
    "sr3_wstream_create": (c_int, [c_void_p, c_uint64, c_int, c_int, POINTER(c_void_p)]),
    "sr3_wstream_destroy": (None, [c_void_p]),
    "sr3_wstream_admit": (c_int, [c_void_p, POINTER(c_int), c_int, c_void_p, c_void_p, c_int, c_int, c_uint64, POINTER(c_int), c_void_p]),
    "sr3_wstream_add_schedule": (c_int, [c_void_p, c_int] + [c_void_p] * 6 + [POINTER(c_int), c_void_p]),
    "sr3_wstream_admit_scheduled": (c_int, [c_void_p, POINTER(c_int), c_int, c_void_p, c_void_p, c_int, c_int, c_uint64, c_int, POINTER(c_int),
                                            c_void_p]),
    "sr3_wstream_step": (c_int, [c_void_p, c_void_p]),
    "sr3_wstream_retire": (c_int, [c_void_p, c_int, c_void_p]),
    "sr3_wstream_slot_state": (c_int, [c_void_p, POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "sr3_engine_profile_step": (c_int, [c_void_p, c_int, c_int, c_int, POINTER(c_int), POINTER(c_float), POINTER(c_double), POINTER(c_double),
                                        POINTER(c_int), c_void_p]),
    "sr3_pil_bicubic_tables": (c_int, [c_int, c_int, POINTER(c_int), POINTER(c_int), c_int, POINTER(c_int)]),
    "sr3_resize_bicubic_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_void_p]),
    "sr3_tensor2img": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_void_p]),
    "sr3_ssd_u8": (c_int, [c_void_p, c_void_p, c_int64, POINTER(c_uint64), c_void_p]),
    "sr3_ssim": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, POINTER(c_double), c_void_p]),
    "sr3_image_metrics": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_float, c_void_p, c_void_p, POINTER(c_uint64),
                                  POINTER(c_double), c_void_p]),
    "sr3_engine_num_launches_per_step": (c_int, [c_void_p]),
    "sr3_engine_num_ops_per_step": (c_int, [c_void_p]),
    "sr3_engine_workspace_bytes": (c_int64, [c_void_p]),
    "sr3_engine_read_activation": (c_int, [c_void_p, c_char_p, c_void_p, c_int64, POINTER(c_int64), POINTER(c_int), c_void_p]),
    "sr3_test_read_gradient": (c_int, [c_void_p, c_char_p, c_int, c_void_p, c_int64, POINTER(c_int64), POINTER(c_int), c_void_p]),
    "sr3_bench_conv": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_float)]),
    "sr3_test_gemm": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "sr3_test_attention": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "sr3_test_attention_dn": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "sr3_attention_dn": (c_int, [c_int, c_int, c_int, c_int, POINTER(c_int)]),
    "sr3_bench_attention": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_float)]),
    "sr3_test_conv_groupnorm": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                        c_int, c_void_p]),
    "sr3_test_conv": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                              c_void_p]),
    "sr3_test_conv_ex": (c_int, [POINTER(TestConvArgsC), POINTER(GemmGeometryC), c_void_p]),
    "sr3_tile_schedule": (c_int, [c_void_p, c_int, POINTER(GemmGeometryC), POINTER(c_int), POINTER(c_int)]),
    "sr3_test_wgrad": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float,
                               c_int, POINTER(c_int), c_void_p]),
    "sr3_test_groupnorm_layer": (c_int, [POINTER(TestGroupNormArgsC), c_void_p]),
    "sr3_test_grad_combine": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_int,
                                      c_void_p]),
    "sr3_test_dgrad": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "sr3_test_attention_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                       c_void_p]),
    "sr3_test_film_embed_bwd": (c_int, [POINTER(TestFilmArgsC), c_void_p]),
    "sr3_test_film_embed_fwd": (c_int, [c_void_p] * 10 + [c_int, c_int, c_int, c_void_p]),
    "sr3_test_attention_unfused": (c_int, [c_void_p] * 5 + [c_int] * 5 + [c_void_p]),
    "sr3_test_loss_grad": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, POINTER(c_double), c_void_p, c_int, c_void_p, c_void_p]),
    "sr3_test_grad_load": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "sr3_test_noise_level_bwd": (c_int, [c_void_p] * 6 + [c_int, c_int, c_void_p]),
    "sr3_test_input_grad": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
}
EXPORTED_SYMBOLS = tuple(_SIGS.keys())


def lib():
    """Load (never build silently on a GPU box) the native library; raise loudly if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError(
            f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (nvcc, sm_90a). "
            "sr3_b200 has no CPU or eager-PyTorch fallback.")
    try:
        l = ctypes.CDLL(LIB_PATH)
    except OSError as e:
        raise NativeLibraryError(f"cannot load {LIB_PATH}: {e}") from e
    for name, (res, args) in _SIGS.items():
        try:
            fn = getattr(l, name)
        except AttributeError as e:
            raise NativeLibraryError(f"{LIB_PATH} does not export {name}") from e
        fn.restype = res
        fn.argtypes = args
    _lib = l
    return l


def _check(rc):
    if rc != 0:
        raise RuntimeError("sr3_b200: " + lib().sr3_last_error().decode())


def _stream():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return c_void_p(0) if t is None else c_void_p(t.data_ptr())


def _f32c(t, device):
    return t.detach().to(device=device, dtype=torch.float32).contiguous()


class UnsupportedSizeError(ValueError, RuntimeError):
    """An image size the native plan cannot run (check_image_size)."""


def check_image_size(n_levels, height, width):
    """The image sizes an inference plan runs on (sr3_engine_create_sized): at every UNet level -- the image halved n_levels - 1 times --
    both sides are powers of two and at least 8, except that the lowest level may be exactly 4x4.  Returns the lowest level (h, w);
    raises UnsupportedSizeError naming the size and the rule otherwise."""
    height, width = int(height), int(width)
    lh, lw = height >> (n_levels - 1), width >> (n_levels - 1)
    if height <= 0 or width <= 0:
        raise UnsupportedSizeError("image size %dx%d: sides must be positive" % (height, width))
    if lh < 4 or lw < 4:
        raise UnsupportedSizeError("image size %dx%d: lowest UNet resolution %dx%d < 4 is not supported (%d levels)" % (height, width, lh, lw, n_levels))
    if height & (height - 1) or width & (width - 1):
        raise UnsupportedSizeError("image size %dx%d: both sides must be powers of two" % (height, width))
    if not ((lh >= 8 and lw >= 8) or (lh == 4 and lw == 4)):
        raise UnsupportedSizeError("image size %dx%d: lowest UNet level %dx%d is not supported (every level must be at least 8x8, or the lowest "
                                   "exactly 4x4)" % (height, width, lh, lw))
    return lh, lw


class Engine:
    """One (config, batch, height, width, device) instance of the native plan: packed weights + activations + captured step graph."""

    def __init__(self, cfg: dict, batch: int, device: torch.device, train_dropout=None, height=None, width=None):
        """train_dropout: None = inference plan; a float = TRAINING plan (forward keeps every intermediate, backward recorded) with that
        Dropout probability (sr3_engine_create_train_sized).  height / width: the image size the plan runs on (default image_size; any size
        check_image_size accepts, for both kinds of plan)."""
        if device.type != "cuda":
            raise NativeLibraryError("sr3_b200 runs on a CUDA (sm_90a) device only; got device=%s" % device)
        self.device = device
        self.batch = batch
        self.channels = cfg["channels"]
        self.in_channel = cfg["in_channel"]
        self.out_channel = cfg["out_channel"]
        self.inner_channel = cfg["inner_channel"]
        self.image_size = cfg["image_size"]
        self.height = int(cfg["image_size"] if height is None else height)
        self.width = int(cfg["image_size"] if width is None else width)
        check_image_size(len(cfg["channel_mults"]), self.height, self.width)
        self.conditional = bool(cfg["conditional"])
        c = UNetConfigC()
        c.in_channel, c.out_channel, c.inner_channel = cfg["in_channel"], cfg["out_channel"], cfg["inner_channel"]
        c.norm_groups = cfg["norm_groups"]
        mults, attn = list(cfg["channel_mults"]), list(cfg["attn_res"])
        c.n_mults, c.n_attn_res = len(mults), len(attn)
        for i, m in enumerate(mults):
            c.channel_mults[i] = m
        for i, a in enumerate(attn):
            c.attn_res[i] = a
        c.res_blocks, c.image_size, c.channels, c.conditional = cfg["res_blocks"], cfg["image_size"], cfg["channels"], int(cfg["conditional"])
        self.precision = cfg.get("precision", "bf16")
        if self.precision not in PRECISIONS:
            raise ValueError("precision must be one of %s, got %r" % (sorted(PRECISIONS), self.precision))
        c.precision = PRECISIONS[self.precision]
        self._h = c_void_p()
        idx = device.index if device.index is not None else torch.cuda.current_device()
        self.train_dropout = train_dropout
        if train_dropout is None:
            _check(lib().sr3_engine_create_sized(ctypes.byref(c), batch, self.height, self.width, idx, ctypes.byref(self._h)))
        else:
            _check(lib().sr3_engine_create_train_sized(ctypes.byref(c), batch, self.height, self.width, idx, float(train_dropout),
                                                       ctypes.byref(self._h)))
        self.T = 0
        self._keep = []
        # training forwards run on this engine (train_forward and train_unet_forward alike): each replaces the intermediates the previous
        # one kept, so a UNet backward checks that its forward is still the latest one and has not been backpropagated yet
        self.forward_count = 0
        self._last_forward = None
        self._unet_backward_done = 0

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().sr3_engine_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ---- parameters
    def param_table(self):
        out = []
        n = lib().sr3_engine_num_params(self._h)
        buf = ctypes.create_string_buffer(256)
        shape = (c_int64 * 4)()
        nd = c_int()
        for i in range(n):
            _check(lib().sr3_engine_param_info(self._h, i, buf, 256, shape, ctypes.byref(nd)))
            out.append((buf.value.decode(), tuple(shape[j] for j in range(nd.value))))
        return out

    def load_params_fast(self, tensors):
        """One native call for the whole parameter set (fp32 contiguous CUDA tensors in param_table() order), no synchronisation: the
        training loop's re-pack after every optimizer step."""
        arr = (c_void_p * len(tensors))()
        for i, t in enumerate(tensors):
            if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
                raise RuntimeError("load_params_fast needs contiguous fp32 CUDA tensors")
            arr[i] = t.data_ptr()
        with torch.cuda.device(self.device):
            _check(lib().sr3_engine_load_all_params(self._h, arr, len(tensors), _stream()))

    def load_state_dict(self, sd: dict):
        keep = []
        with torch.cuda.device(self.device):
            for name, _shape in self.param_table():
                if name not in sd:
                    raise KeyError("missing key in state_dict: " + name)
                t = _f32c(sd[name], self.device)
                keep.append(t)
                _check(lib().sr3_engine_load_param(self._h, name.encode(), _ptr(t), t.numel(), _stream()))
            _check(lib().sr3_engine_finalize_params(self._h, _stream()))
            torch.cuda.current_stream().synchronize()

    def set_schedule(self, bufs: dict, sqrt_alphas_cumprod_prev):
        T, host, sp = _schedule_host(bufs, sqrt_alphas_cumprod_prev)
        with torch.cuda.device(self.device):
            _check(lib().sr3_engine_set_schedule(self._h, T, *[c_void_p(h.data_ptr()) for h in host], c_void_p(sp.ctypes.data), _stream()))
        self.T = T
        self._schedule = (bufs, sqrt_alphas_cumprod_prev)

    @contextlib.contextmanager
    def sampling_on(self, sampler):
        """Runs the body on a few-step sampler's tables: `sampler` = (buffers, sqrt_alphas_cumprod_prev, solver) of
        model.sr3_modules.samplers.sampler_schedule (None: the engine's schedule, unchanged).  The engine's schedule is set back when the
        body ends, however it ends, so a later call without a sampler reads exactly the tables it read before."""
        if sampler is None:
            yield
            return
        saved = getattr(self, "_schedule", None)
        if saved is None:
            raise RuntimeError("set_new_noise_schedule has not been called")
        self.set_schedule(sampler[0], sampler[1])
        try:
            yield
        finally:
            self.set_schedule(*saved)

    # ---- compute
    def _img(self):
        return torch.empty(self.batch, self.channels, self.height, self.width, device=self.device, dtype=torch.float32)

    def _check_img(self, t, channels, what):
        if t is not None and tuple(t.shape) != (self.batch, channels, self.height, self.width):
            raise ValueError("%s has shape %s; this engine runs [%d, %d, %d, %d]" % (what, tuple(t.shape), self.batch, channels, self.height,
                                                                                     self.width))

    def _check_inputs(self, x, cond):
        self._check_img(x, self.channels, "x")
        self._check_img(cond, self.in_channel - self.channels, "condition_x")

    def unet_forward(self, x, noise_level):
        x = _f32c(x, self.device)
        nl = _f32c(noise_level, self.device).reshape(-1)
        assert x.shape == (self.batch, self.in_channel, self.height, self.width), x.shape
        assert nl.numel() == self.batch
        eps = torch.empty(self.batch, self.out_channel, self.height, self.width, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _check(lib().sr3_unet_forward(self._h, _ptr(x), _ptr(nl), _ptr(eps), _stream()))
        return eps

    def p_mean_variance(self, x, t, clip_denoised=True, condition_x=None):
        x = _f32c(x, self.device)
        c = None if condition_x is None else _f32c(condition_x, self.device)
        self._check_inputs(x, c)
        mean = self._img()
        lv = c_float()
        with torch.cuda.device(self.device):
            _check(lib().sr3_p_mean_variance(self._h, _ptr(x), _ptr(c), int(t), int(bool(clip_denoised)), _ptr(mean), ctypes.byref(lv), _stream()))
        return mean, lv.value

    def p_sample(self, x, t, condition_x=None, noise=None, seed=0, first_index=0):
        x = _f32c(x, self.device)
        c = None if condition_x is None else _f32c(condition_x, self.device)
        n = None if noise is None else _f32c(noise, self.device)
        self._check_inputs(x, c)
        self._check_img(n, self.channels, "noise")
        out = self._img()
        with torch.cuda.device(self.device):
            _check(lib().sr3_p_sample(self._h, _ptr(x), _ptr(c), int(t), _ptr(n), int(seed), int(first_index), _ptr(out), _stream()))
        return out

    def p_losses(self, hr, sr, gamma, noise, loss_type="l1"):
        hr, noise = _f32c(hr, self.device), _f32c(noise, self.device)
        s = None if sr is None else _f32c(sr, self.device)
        g = _f32c(gamma, self.device).reshape(-1)
        self._check_inputs(hr, s)
        self._check_img(noise, self.channels, "noise")
        out = c_double()
        with torch.cuda.device(self.device):
            _check(lib().sr3_p_losses(self._h, _ptr(hr), _ptr(s), _ptr(g), _ptr(noise), 1 if loss_type == "l1" else 2, ctypes.byref(out), _stream()))
        return out.value

    # ---- training step (model/model.py:48-58): forward with the draws injected, backward into caller-owned gradient tensors
    def train_forward(self, hr, sr, gamma, noise, loss_type="l1", dropout_seed=0, want_loss=True):
        hr, noise = _f32c(hr, self.device), _f32c(noise, self.device)
        s = None if sr is None else _f32c(sr, self.device)
        g = _f32c(gamma, self.device).reshape(-1)
        self._check_inputs(hr, s)
        self._check_img(noise, self.channels, "noise")
        self._keep = [hr, noise, s, g]
        self.forward_count += 1
        self._last_forward = "p_losses"
        out = c_double()
        with torch.cuda.device(self.device):
            _check(lib().sr3_train_forward(self._h, _ptr(hr), _ptr(s), _ptr(g), _ptr(noise), 1 if loss_type == "l1" else 2, int(dropout_seed),
                                           ctypes.byref(out) if want_loss else None, _stream()))
        return out.value if want_loss else None

    def _grad_ptrs(self, grads):
        arr = (c_void_p * len(grads))()
        for i, gten in enumerate(grads):
            assert gten.is_cuda and gten.dtype == torch.float32 and gten.is_contiguous()
            arr[i] = gten.data_ptr()
        return arr

    def train_backward(self, grad_scale, grads):
        """grads: one contiguous fp32 CUDA tensor per parameter, in param_table() order; overwritten."""
        arr = self._grad_ptrs(grads)
        with torch.cuda.device(self.device):
            _check(lib().sr3_train_backward(self._h, float(grad_scale), arr, len(grads), _stream()))

    # ---- UNet.forward alone in training form, and its backward from any upstream gradient (the differentiable denoise_fn)
    def train_unet_forward(self, x, noise_level, dropout_seed=0):
        """x [B,in_channel,H,W] (cat(cond, x_t) for a conditional net), noise_level [B] or [B,1] -> (eps [B,out_channel,H,W], the index of
        this forward on the engine, which train_unet_backward takes).  sr3_train_unet_forward."""
        x = _f32c(x, self.device)
        nl = _f32c(noise_level, self.device).reshape(-1)
        self._check_img(x, self.in_channel, "x")
        if nl.numel() != self.batch:
            raise ValueError("noise_level has %d elements; this engine runs a batch of %d" % (nl.numel(), self.batch))
        eps = torch.empty(self.batch, self.out_channel, self.height, self.width, device=self.device, dtype=torch.float32)
        self._keep = [x, nl]
        self.forward_count += 1
        self._last_forward = None
        with torch.cuda.device(self.device):
            _check(lib().sr3_train_unet_forward(self._h, _ptr(x), _ptr(nl), int(dropout_seed), _ptr(eps), _stream()))
        self._last_forward = "unet"
        return eps, self.forward_count

    def train_unet_backward(self, deps, grads, want_dx=False, want_dnl=False, forward=None):
        """Backward of the UNet forward with index `forward` (default: the latest) for the upstream gradient deps [B,out_channel,H,W].  grads:
        one contiguous fp32 CUDA tensor per parameter, in param_table() order; overwritten.  Returns (dx [B,in_channel,H,W] or None,
        d noise_level [B] or None).  Raises RuntimeError when a later forward on this engine has replaced that forward's intermediates, or
        when it has already been backpropagated: either would give silently wrong gradients."""
        fwd = self.forward_count if forward is None else int(forward)
        if fwd != self.forward_count:
            raise RuntimeError("sr3_b200: cannot backpropagate UNet forward #%d: a later forward (#%d, %s) on the same engine has replaced the "
                               "intermediates it kept; run the backward before the next forward" %
                               (fwd, self.forward_count, "p_losses" if self._last_forward == "p_losses" else "UNet"))
        if self._last_forward != "unet":
            raise RuntimeError("sr3_b200: the latest forward on this engine is not a UNet forward (train_unet_forward)")
        if self._unet_backward_done == fwd:
            raise RuntimeError("sr3_b200: UNet forward #%d has already been backpropagated; the native backward runs once per forward "
                               "(retain_graph is not supported)" % fwd)
        deps = _f32c(deps, self.device)
        self._check_img(deps, self.out_channel, "the gradient of eps")
        arr = self._grad_ptrs(grads)
        dx = torch.empty(self.batch, self.in_channel, self.height, self.width, device=self.device, dtype=torch.float32) if want_dx else None
        dnl = torch.empty(self.batch, device=self.device, dtype=torch.float32) if want_dnl else None
        self._unet_backward_done = fwd
        with torch.cuda.device(self.device):
            _check(lib().sr3_train_unet_backward(self._h, _ptr(deps), arr, len(grads), _ptr(dx), _ptr(dnl), _stream()))
        return dx, dnl

    def film_state(self):
        """Tests: copies of the FiLM state of this training engine's latest forward and backward, one row per image the plan allocates
        (the batch, padded): {"tau": [rows, inner], "dfilm": [rows, F], "dtau": [rows, inner]}.  sr3_test_train_film_state."""
        rows, F = c_int(), c_int()
        with torch.cuda.device(self.device):
            _check(lib().sr3_test_train_film_state(self._h, None, None, None, ctypes.byref(rows), ctypes.byref(F), _stream()))
            inner = self.inner_channel
            out = {"tau": torch.empty(rows.value, inner, device=self.device), "dfilm": torch.empty(rows.value, F.value, device=self.device),
                   "dtau": torch.empty(rows.value, inner, device=self.device)}
            _check(lib().sr3_test_train_film_state(self._h, _ptr(out["tau"]), _ptr(out["dfilm"]), _ptr(out["dtau"]), ctypes.byref(rows),
                                                   ctypes.byref(F), _stream()))
        return out

    def train_backward_profile(self, grad_scale, grads):
        """{kind: ms} of one backward, CUDA events around every op."""
        arr = self._grad_ptrs(grads)
        ms = (c_float * 8)()
        with torch.cuda.device(self.device):
            _check(lib().sr3_train_backward_profile(self._h, float(grad_scale), arr, len(grads), ms, _stream()))
        names = {0: "dgrad_tile_kernel", 1: "groupnorm_elementwise", 3: "bookkeeping", 4: "other", 5: "wgrad_slice_reduce", 6: "wgrad", 7: "attention_backward"}
        return {names.get(k, str(k)): ms[k] for k in range(8) if ms[k] > 0}

    def num_backward_blocks(self):
        return lib().sr3_train_num_backward_blocks(self._h)

    def backward_begin(self, grad_scale, grads):
        self._grad_arr = self._grad_ptrs(grads)
        _check(lib().sr3_train_backward_begin(self._h, float(grad_scale), self._grad_arr, len(grads)))

    def backward_block(self, i):
        with torch.cuda.device(self.device):
            _check(lib().sr3_train_backward_block(self._h, int(i), _stream()))

    def backward_flush(self):
        """Sum the weight-gradient partial tiles of the layers run since the last flush (one launch); call before all-reducing a bucket."""
        with torch.cuda.device(self.device):
            _check(lib().sr3_train_backward_flush(self._h, _stream()))

    def backward_finish(self):
        with torch.cuda.device(self.device):
            _check(lib().sr3_train_backward_finish(self._h, _stream()))

    def block_params(self, i):
        cap = 64
        idx = (c_int * cap)()
        n = c_int()
        _check(lib().sr3_train_block_params(self._h, int(i), idx, cap, ctypes.byref(n)))
        return [idx[k] for k in range(min(n.value, cap))]

    def dropout_layers(self):
        out = []
        buf = ctypes.create_string_buffer(256)
        for i in range(lib().sr3_train_num_dropout_layers(self._h)):
            _check(lib().sr3_train_dropout_layer_name(self._h, i, buf, 256))
            out.append(buf.value.decode())
        return out

    def set_dropout_mask(self, block_name, mask_nchw_u8):
        """Tests: inject the keep-mask (uint8 CUDA [B,C,H,W], 1 = keep) of the nn.Dropout of `block_name` ("downs.1.res_block.block2")."""
        if mask_nchw_u8 is not None:
            assert mask_nchw_u8.is_cuda and mask_nchw_u8.dtype == torch.uint8 and mask_nchw_u8.is_contiguous()
            self._keep_masks = getattr(self, "_keep_masks", {})
            self._keep_masks[block_name] = mask_nchw_u8
        _check(lib().sr3_train_set_dropout_mask(self._h, block_name.encode(), _ptr(mask_nchw_u8)))

    def p_sample_loop(self, condition_x, x_T, noises=None, seed=0, first_index=0, want_snapshots=True, sampler=None):
        """The whole reverse loop; `sampler`: the tables of a DDIM spec (Engine.sampling_on), whose K steps then run instead of the
        schedule's (noises [K, ...], K snapshots' worth of steps).  DPM-Solver++(2M) runs on a canvas (WindowedSampler.sample_loop)."""
        if sampler is not None:
            if sampler[2] is not None:
                raise ValueError("DPM-Solver++(2M) keeps the previous step's x0 on a canvas: use WindowedSampler.sample_loop")
            with self.sampling_on(sampler):
                return self.p_sample_loop(condition_x, x_T, noises, seed, first_index, want_snapshots)
        c = None if condition_x is None else _f32c(condition_x, self.device)
        x_T = _f32c(x_T, self.device)
        n = None if noises is None else _f32c(noises, self.device)
        self._check_inputs(x_T, c)
        if n is not None and tuple(n.shape[1:]) != (self.batch, self.channels, self.height, self.width):
            raise ValueError("noises has shape %s; this engine needs [T, %d, %d, %d, %d]" % (tuple(n.shape), self.batch, self.channels,
                                                                                           self.height, self.width))
        T = self.T
        inter = 1 | (T // 10)
        cap = len([i for i in range(T) if i % inter == 0])
        final = self._img()
        snaps = torch.empty(cap, *final.shape, device=self.device, dtype=torch.float32) if want_snapshots else None
        ns = c_int()
        with torch.cuda.device(self.device):
            _check(lib().sr3_p_sample_loop(self._h, _ptr(c), _ptr(x_T), _ptr(n), int(seed), int(first_index), _ptr(final), _ptr(snaps), cap,
                                           ctypes.byref(ns), _stream()))
        return final, snaps

    def super_resolution_host(self, cond_host, x_T_host, seed=0, first_index=0):
        """Host (pinned) buffers in, host buffer out; H2D + T steps + D2H inside one native call."""
        self._check_inputs(x_T_host, cond_host)
        out = torch.empty(self.batch, self.channels, self.height, self.width, dtype=torch.float32).pin_memory()
        with torch.cuda.device(self.device):
            _check(lib().sr3_super_resolution_host(self._h, _ptr(cond_host), _ptr(x_T_host), int(seed), int(first_index), _ptr(out), _stream()))
        return out

    def loop_begin(self, condition_x, x_T, seed=0, first_index=0):
        c = None if condition_x is None else _f32c(condition_x, self.device)
        x_T = _f32c(x_T, self.device)
        self._check_inputs(x_T, c)
        with torch.cuda.device(self.device):
            _check(lib().sr3_p_sample_loop_begin(self._h, _ptr(c), _ptr(x_T), int(seed), int(first_index), _stream()))

    def steps(self, t_start, n):
        with torch.cuda.device(self.device):
            _check(lib().sr3_p_sample_steps(self._h, int(t_start), int(n), _stream()))

    def read_state(self):
        out = self._img()
        with torch.cuda.device(self.device):
            _check(lib().sr3_read_state(self._h, _ptr(out), _stream()))
        return out

    def profile_step(self, t, reps=3):
        """[(kind, ms, flops, bytes)] per launch of one eager step (kinds: 0 gemm tile, 1 GN apply, 2 cast, 3 softmax, 4 other,
        5 fused attention core: attn_kernel up to 256 tokens per attention batch, attn_long_kernel above)."""
        cap = lib().sr3_engine_num_ops_per_step(self._h)
        kinds, ms = (c_int * cap)(), (c_float * cap)()
        fl, by = (c_double * cap)(), (c_double * cap)()
        n = c_int()
        with torch.cuda.device(self.device):
            _check(lib().sr3_engine_profile_step(self._h, int(t), int(reps), cap, kinds, ms, fl, by, ctypes.byref(n), _stream()))
        return [(kinds[i], ms[i], fl[i], by[i]) for i in range(n.value)]

    def tile_schedules(self):
        """Per op of the eager step (the order of profile_step): None for an op that is not a tile-kernel launch, else its geometry dict
        plus "schedule" ("cooperative" / "pingpong") and "out_hwc" (output rows, columns, channels)."""
        return [_tile_schedule(self._h, i) for i in range(lib().sr3_engine_num_ops_per_step(self._h))]

    def launches_per_step(self):
        return lib().sr3_engine_num_launches_per_step(self._h)

    def ops_per_step(self):
        return lib().sr3_engine_num_ops_per_step(self._h)

    def uses_step_kernel(self):
        # Every reverse step runs as the graph of per-layer launches.  Kept for bench.py, which asks before it reads a per-op
        # step-kernel profile.
        return False

    def workspace_bytes(self):
        return lib().sr3_engine_workspace_bytes(self._h)

    def read_activation(self, name):
        """fp32 output of a top-level UNet layer of the last forward, returned NCHW like a reference forward hook.  For a layer with
        self-attention that is the attention's output; "<layer>.res_block" ("mid.0.res_block") is its ResnetBlock's output."""
        numel = c_int64()
        shape = (c_int * 4)()
        _check(lib().sr3_engine_read_activation(self._h, name.encode(), c_void_p(0), 0, ctypes.byref(numel), shape, _stream()))
        t = torch.empty(tuple(shape), device=self.device, dtype=torch.float32)
        _check(lib().sr3_engine_read_activation(self._h, name.encode(), _ptr(t), t.numel(), ctypes.byref(numel), shape, _stream()))
        return t.permute(0, 3, 1, 2).contiguous()

    def read_gradient(self, name, form="g"):
        """Tests: the gradient the latest backward of this training engine left for the tensor of tap `name` (read_activation's names).
        form "g": fp32 NCHW [B,C,H,W]; "gb": its bf16 copy, widened to fp32, NCHW; "gsum": its per-image channel sums [B,C].
        sr3_test_read_gradient."""
        f = {"g": 0, "gb": 1, "gsum": 2}[form]
        numel = c_int64()
        shape = (c_int * 4)()
        with torch.cuda.device(self.device):
            _check(lib().sr3_test_read_gradient(self._h, name.encode(), f, c_void_p(0), 0, ctypes.byref(numel), shape, _stream()))
            t = torch.empty(tuple(shape), device=self.device, dtype=torch.float32)
            _check(lib().sr3_test_read_gradient(self._h, name.encode(), f, _ptr(t), t.numel(), ctypes.byref(numel), shape, _stream()))
        return t.view(shape[0], shape[3]) if f == 2 else t.permute(0, 3, 1, 2).contiguous()


def window_grid(length, side, overlap):
    """Window origins along one axis of `length` pixels for windows of `side` pixels that overlap their neighbours by at least `overlap`:
    one window when length == side, else n = ceil((length - overlap) / (side - overlap)) windows at round-half-up(i (length - side) / (n - 1)),
    so the first starts at 0, the last ends at `length` and nothing lies outside.  Pure host arithmetic, the same as the native side's."""
    length, side, overlap = int(length), int(side), int(overlap)
    if length < side:
        raise ValueError("canvas side %d is smaller than the window side %d (canvases are not padded)" % (length, side))
    if not 0 <= overlap < side:
        raise ValueError("overlap %d must be at least 0 and below the window side %d" % (overlap, side))
    if length == side:
        return [0]
    n = -(-(length - overlap) // (side - overlap))
    return [(2 * i * (length - side) + (n - 1)) // (2 * (n - 1)) for i in range(n)]


def window_weights(n, side, overlap):
    """Blend weights [n][side] (fp32) of the n windows of one axis: min(i + 1, side - i, ramp) / ramp with ramp = max(overlap, 1); the ramp
    towards a border of the canvas, where no neighbour exists, is replaced by 1."""
    ramp = max(int(overlap), 1)
    i = torch.arange(side)
    rows = []
    for k in range(n):
        m = torch.full((side,), ramp)
        if k > 0:
            m = torch.minimum(m, i + 1)
        if k < n - 1:
            m = torch.minimum(m, side - i)
        rows.append(m.to(torch.float32) / float(ramp))
    return torch.stack(rows)


class WindowedSampler:
    """A canvas [batch, C, height, width] sampled by overlapping windows of `engine`'s image size, merged inside every reverse step
    (sr3_windowed_*).  Borrows the engine (engine.batch windows run per pass) and keeps it alive.

    With `window_range` = (n0, n1) the sampler runs only windows [n0, n1) of the list (sr3_windowed_create_range): their means go to
    `self.means`, an arena [N, C, wh, ww] of all N windows, NaN until written, into whose slots the means of other windows are copied or
    received between phase_means() and phase_merge(); `bands` ([(y0, y1)] per image) limits the merge to those rows."""

    def __init__(self, engine, batch, height, width, overlap_h, overlap_w, window_range=None, bands=None):
        self.engine = engine
        self.device = engine.device
        self.shape = (int(batch), engine.channels, int(height), int(width))
        self.overlap = (int(overlap_h), int(overlap_w))
        self.window_range = None if window_range is None else (int(window_range[0]), int(window_range[1]))
        self.means = None
        self._h = c_void_p()
        with torch.cuda.device(self.device):
            if self.window_range is None:
                _check(lib().sr3_windowed_create(engine._h, *self.shape[:1], *self.shape[2:], *self.overlap, ctypes.byref(self._h)))
            else:
                n = self.shape[0] * len(window_grid(height, engine.height, overlap_h)) * len(window_grid(width, engine.width, overlap_w))
                if not 0 <= self.window_range[0] < self.window_range[1] <= n:
                    raise ValueError("window range %s is not a non-empty part of the %d windows" % (self.window_range, n))
                bt = None
                if bands is not None:
                    if len(bands) != self.shape[0]:
                        raise ValueError("bands has %d entries for %d images" % (len(bands), self.shape[0]))
                    bt = (c_int * (2 * self.shape[0]))(*[int(v) for yb in bands for v in yb])
                self.means = torch.full((n, engine.channels, engine.height, engine.width), float("nan"), device=self.device)
                _check(lib().sr3_windowed_create_range(engine._h, *self.shape[:1], *self.shape[2:], *self.overlap, *self.window_range,
                                                       _ptr(self.means), bt, ctypes.byref(self._h)))
        self._keep = None

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().sr3_windowed_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def grid(self):
        """(origins_y, origins_x, weights_y [ny, wh], weights_x [nx, ww]) as the native side built them."""
        ny, nx = c_int(), c_int()
        _check(lib().sr3_windowed_grid(self._h, ctypes.byref(ny), ctypes.byref(nx), None, None, None, None))
        wh, ww = self.engine.height, self.engine.width
        oy, ox = (c_int * ny.value)(), (c_int * nx.value)()
        wy, wx = (c_float * (ny.value * wh))(), (c_float * (nx.value * ww))()
        _check(lib().sr3_windowed_grid(self._h, ctypes.byref(ny), ctypes.byref(nx), oy, ox, wy, wx))
        return list(oy), list(ox), torch.tensor(list(wy)).view(ny.value, wh), torch.tensor(list(wx)).view(nx.value, ww)

    def _canvas(self, t, channels, what):
        t = _f32c(t, self.device)
        want = (self.shape[0], channels, self.shape[2], self.shape[3])
        if tuple(t.shape) != want:
            raise ValueError("%s has shape %s; this canvas is %s" % (what, tuple(t.shape), want))
        return t

    def begin(self, condition_x, x_T, seed=0, first_index=0):
        c = None if condition_x is None else self._canvas(condition_x, self.engine.in_channel - self.engine.channels, "condition_x")
        x_T = self._canvas(x_T, self.shape[1], "x_T")
        with torch.cuda.device(self.device):
            _check(lib().sr3_windowed_begin(self._h, _ptr(c), _ptr(x_T), int(seed), int(first_index), _stream()))

    def steps(self, t_start, n, noises=None, snapshots=None):
        """n canvas steps from timestep t_start down.  noises: [T, *canvas shape], noises[t] used at step t; snapshots: a CUDA fp32 tensor
        [cap, *canvas shape] that receives x_{t-1} of every t with t % (1 | T // 10) == 0."""
        if noises is not None:
            noises = _f32c(noises, self.device)
            if tuple(noises.shape) != (self.engine.T,) + self.shape:
                raise ValueError("noises has shape %s; this canvas needs %s" % (tuple(noises.shape), (self.engine.T,) + self.shape))
        self._keep = (noises, snapshots)
        with torch.cuda.device(self.device):
            _check(lib().sr3_windowed_set_snapshots(self._h, _ptr(snapshots), 0 if snapshots is None else snapshots.shape[0]))
            _check(lib().sr3_windowed_steps(self._h, int(t_start), int(n), _ptr(noises), _stream()))

    def read_state(self):
        out = torch.empty(self.shape, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _check(lib().sr3_windowed_read_state(self._h, _ptr(out), _stream()))
        return out

    def set_solver(self, coefs):
        """DPM-Solver++(2M) merges from the next step on: coefs [3, K] (A, B, C per step index; samplers.sampler_schedule), or None for
        the posterior-sample merge (sr3_windowed_set_solver)."""
        host = None if coefs is None else coefs.detach().to("cpu", torch.float32).contiguous()
        if host is not None and (host.dim() != 2 or host.shape[0] != 3):
            raise ValueError("solver coefficients must be [3, K], got %s" % (tuple(host.shape),))
        with torch.cuda.device(self.device):
            _check(lib().sr3_windowed_set_solver(self._h, 0 if host is None else host.shape[1], _ptr(host)))

    def sample_loop(self, condition_x, x_T, noises=None, seed=0, first_index=0, want_snapshots=True, sampler=None):
        """The whole reverse loop; returns (x_0, snapshots or None) like Engine.p_sample_loop.  `sampler`: the tables of a few-step
        sampler (Engine.sampling_on), run instead of the engine's schedule; DPM-Solver++(2M) draws no noise and ignores `noises`."""
        if sampler is not None:
            with self.engine.sampling_on(sampler):
                if sampler[2] is not None:
                    self.set_solver(sampler[2])
                try:
                    return self.sample_loop(condition_x, x_T, noises, seed, first_index, want_snapshots)
                finally:
                    if sampler[2] is not None:
                        self.set_solver(None)
        T = self.engine.T
        inter = 1 | (T // 10)
        cap = len([i for i in range(T) if i % inter == 0])
        snaps = torch.empty((cap,) + self.shape, device=self.device, dtype=torch.float32) if want_snapshots else None
        self.begin(condition_x, x_T, seed, first_index)
        self.steps(T - 1, T, noises, snaps)
        return self.read_state(), snaps

    def phase_begin(self, t_start):
        """Start a run of split steps from timestep t_start down (Philox noise keyed by begin()'s seed and first_index)."""
        with torch.cuda.device(self.device):
            _check(lib().sr3_windowed_phase_begin(self._h, int(t_start), _stream()))

    def phase_means(self):
        """Phase (a) of a step: advance the timestep, run this canvas's windows, store their means into the arena."""
        with torch.cuda.device(self.device):
            _check(lib().sr3_windowed_phase_means(self._h, _stream()))

    def phase_merge(self):
        """Phase (b) of the step: merge the arena's means (over the band) into x_{t-1}."""
        with torch.cuda.device(self.device):
            _check(lib().sr3_windowed_phase_merge(self._h, _stream()))

    def profile_step(self, t, reps=3):
        """{"gather", "engine", "merge"}: device ms per eager canvas step (CUDA events)."""
        ms = (c_float * 3)()
        with torch.cuda.device(self.device):
            _check(lib().sr3_windowed_profile_step(self._h, int(t), int(reps), ms, _stream()))
        return {"gather": ms[0], "engine": ms[1], "merge": ms[2]}


MAX_TIMESTEPS = 4096     # the largest n_timestep an engine's schedule tables hold (sr3_engine T_cap)


def _schedule_host(bufs: dict, sqrt_alphas_cumprod_prev):
    """(T, the five fp32 host tables, fp64 sqrt_alphas_cumprod_prev) of a schedule's buffers, the arguments of sr3_engine_set_schedule and
    sr3_wstream_add_schedule."""
    import numpy as np
    T = int(bufs["betas"].shape[0])
    host = [bufs[k].detach().to("cpu", torch.float32).contiguous() for k in
            ("sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_mean_coef1", "posterior_mean_coef2",
             "posterior_log_variance_clipped")]
    sp = np.ascontiguousarray(np.asarray(sqrt_alphas_cumprod_prev, dtype=np.float64))
    assert sp.shape[0] == T + 1
    return T, host, sp


def stream_plan(arrival_steps, slots, T):
    """The slot plan of continuous batching: for request n arriving before step arrival_steps[n] (non-decreasing; any iterable, read
    lazily, one value per request planned), yields (slot, admit_step, finish_step).  Requests are admitted first come first served, each
    at the first step at which it has arrived, every earlier request has been admitted and a slot is free, into the lowest free slot; it
    runs steps admit_step .. admit_step + T - 1 and its image is ready after step finish_step - 1 = admit_step + T - 1, so the slot is free
    again from step finish_step on.  Pure host arithmetic: GaussianDiffusion.super_resolution_stream follows it step for step.
    windowed_stream_plan with one window per request."""
    for slot_list, k, finish in windowed_stream_plan(((a, 1) for a in arrival_steps), slots, T):
        yield slot_list[0], k, finish


def windowed_stream_plan(requests, slots, T):
    """The slot plan of continuous batching when a request takes several slots: for request n = (arrival_step, n_windows) or
    (arrival_step, n_windows, steps) (arrival steps non-decreasing; any iterable, read lazily, one value per request planned), yields
    (slot_list, admit_step, finish_step).  First come first served with head-of-line blocking: a request is admitted at the first step at
    which it has arrived, every earlier request has been admitted and n_windows slots are free -- a later, smaller request never overtakes
    it -- into the n_windows lowest free slots; it runs `steps` steps (default T: a request on a schedule of its own runs that schedule's
    n_timestep) and its slots are free again from finish_step = admit_step + steps on.  Pure host arithmetic:
    GaussianDiffusion.super_resolution_windowed_stream follows it step for step."""
    slots, T = int(slots), int(T)
    if slots < 1 or T < 1:
        raise ValueError("stream plans need slots >= 1 and T >= 1, got slots=%d T=%d" % (slots, T))
    free_at = [0] * slots                   # the step from which each slot is free
    last_arrival, last_admit = 0, 0
    for req in requests:
        a, n, steps = (tuple(int(v) for v in req) + (T,))[:3]
        if a < last_arrival:
            raise ValueError("arrival steps must be non-decreasing: %d after %d" % (a, last_arrival))
        if not 1 <= n <= slots:
            raise ValueError("a request of %d windows cannot run on %d slots" % (n, slots))
        if steps < 1:
            raise ValueError("a request of %d steps cannot run: steps must be >= 1" % steps)
        last_arrival = a
        k = max(a, last_admit, sorted(free_at)[n - 1])     # the first step at which n slots are free
        taken = [s for s in range(slots) if free_at[s] <= k][:n]
        for s in taken:
            free_at[s] = k + steps
        last_admit = k
        yield taken, k, k + steps


class WindowedStreamSampler:
    """Continuous batching of canvases of any size on `engine` (sr3_wstream_*): every request is a canvas of ny x nx windows of the engine's
    size (overlap_h x overlap_w, the windowed sampler's grid) that takes as many of the engine.batch slots and runs at its own timestep.
    The online interface: a server calls admit() with free slots, step() once per reverse step and retire() for every request finished()
    lists.  This object owns each request's canvas (x_t, and a copy of the condition) until retire(), which returns x_0; the native side
    borrows them, so admission allocates nothing on the device.  Borrows the engine (and keeps it alive); nothing else may run on it while
    requests are in flight.  A request samples on the engine's noise schedule, or on one registered with add_schedule (requests on
    different schedules share the batch)."""

    def __init__(self, engine, seed, overlap_h, overlap_w):
        self.engine = engine
        self.device = engine.device
        self.slots = engine.batch
        self.seed = int(seed)
        self.overlap = (int(overlap_h), int(overlap_w))
        self._canvases = {}                    # request id -> (x, condition)
        self._h = c_void_p()
        with torch.cuda.device(self.device):
            _check(lib().sr3_wstream_create(engine._h, self.seed, *self.overlap, ctypes.byref(self._h)))

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().sr3_wstream_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def windows(self, height, width):
        """The number of windows (= slots) of a height x width canvas."""
        return len(window_grid(height, self.engine.height, self.overlap[0])) * len(window_grid(width, self.engine.width, self.overlap[1]))

    def add_schedule(self, bufs: dict, sqrt_alphas_cumprod_prev):
        """Register a noise schedule (Engine.set_schedule's arguments: GaussianDiffusion's buffers, see
        diffusion.noise_schedule_buffers) for requests of this stream; returns its id for admit(schedule=...).  Allowed while requests run."""
        T, host, sp = _schedule_host(bufs, sqrt_alphas_cumprod_prev)
        sid = c_int()
        with torch.cuda.device(self.device):
            _check(lib().sr3_wstream_add_schedule(self._h, T, *[c_void_p(h.data_ptr()) for h in host], c_void_p(sp.ctypes.data),
                                                  ctypes.byref(sid), _stream()))
        return sid.value

    def admit(self, slots, condition_x, x_T, sample_index, schedule=None):
        """Admit a request ([C_cond, H, W] condition, None for an unconditional model, and [C, H, W] x_T) into the free `slots`, one per
        window of its grid (row-major); its Philox draws are keyed by the global `sample_index`.  `schedule`: an id from add_schedule, or
        None for the engine's schedule; the request starts at t = n_timestep - 1 of it.  Returns the request's id."""
        cond_c = self.engine.in_channel - self.engine.channels
        if condition_x is not None and (condition_x.dim() != 3 or condition_x.shape[0] != cond_c):
            raise ValueError("condition_x must be [%d, H, W], got %s" % (cond_c, tuple(condition_x.shape)))
        hw = tuple((x_T if condition_x is None else condition_x).shape[-2:])     # without a condition the size is x_T's
        if tuple(x_T.shape) != (self.engine.channels,) + hw:
            raise ValueError("x_T has shape %s; this request needs %s" % (tuple(x_T.shape), (self.engine.channels,) + hw))
        cond = None if condition_x is None else torch.empty(condition_x.shape, device=self.device, dtype=torch.float32).copy_(condition_x)
        x = torch.empty(x_T.shape, device=self.device, dtype=torch.float32).copy_(x_T)
        sl = [int(s) for s in slots]
        rid = c_int()
        with torch.cuda.device(self.device):
            _check(lib().sr3_wstream_admit_scheduled(self._h, (c_int * max(len(sl), 1))(*sl), len(sl), _ptr(cond), _ptr(x), hw[0], hw[1],
                                                     int(sample_index), -1 if schedule is None else int(schedule), ctypes.byref(rid),
                                                     _stream()))
        self._canvases[rid.value] = (x, cond)
        return rid.value

    def step(self, n=1):
        with torch.cuda.device(self.device):
            for _ in range(int(n)):
                _check(lib().sr3_wstream_step(self._h, _stream()))

    def slot_state(self):
        """(request, t, state) per slot: the request id (-1 free), its t (timestep of its next step, -1 once finished) and state 0 free,
        1 running, 2 finished, waiting for retire()."""
        r, t, st = (c_int * self.slots)(), (c_int * self.slots)(), (c_int * self.slots)()
        _check(lib().sr3_wstream_slot_state(self._h, r, t, st))
        return list(r), list(t), list(st)

    def finished(self):
        """The ids of the requests whose image is ready."""
        r, _, st = self.slot_state()
        return sorted({q for q, v in zip(r, st) if v == 2})

    def retire(self, request):
        """x_0 [C, H, W] of finished `request`; frees its slots."""
        with torch.cuda.device(self.device):
            _check(lib().sr3_wstream_retire(self._h, int(request), _stream()))
        return self._canvases.pop(int(request))[0]


def bench_conv(B, H, W, Cin, Cout, k=3, stride=1, resid=False, stats=True, reps=20):
    ms = c_float()
    _check(lib().sr3_bench_conv(B, H, W, Cin, Cout, k, stride, int(resid), int(stats), reps, ctypes.byref(ms)))
    return ms.value


def test_attention(qk_bf16, vT_bf16, nz, Lt, HW, C):
    """Fused attention core: qk [nz*Lt, 2C] bf16, vT [nz*C, Lt] bf16 -> O [nz*Lt, C] bf16."""
    out = torch.empty(nz * Lt, C, device=qk_bf16.device, dtype=torch.bfloat16)
    _check(lib().sr3_test_attention(_ptr(qk_bf16), _ptr(vT_bf16), _ptr(out), nz, Lt, HW, C, _stream()))
    return out


def test_attention_dn(qk_bf16, vT_bf16, nz, Lt, HW, C, dn):
    """test_attention with attn_kernel's channel slice forced to dn (64, 128 or 256; 0 = the one the library picks)."""
    out = torch.empty(nz * Lt, C, device=qk_bf16.device, dtype=torch.bfloat16)
    _check(lib().sr3_test_attention_dn(_ptr(qk_bf16), _ptr(vT_bf16), _ptr(out), nz, Lt, HW, C, dn, _stream()))
    return out


def attention_dn(nz, Lt, C, sms=0):
    """Output channels per CTA the fused attention core runs at for this shape on a GPU of `sms` SMs (0: the current device's)."""
    dn = c_int()
    _check(lib().sr3_attention_dn(nz, Lt, C, sms, ctypes.byref(dn)))
    return dn.value


def bench_attention(qk_bf16, vT_bf16, nz, Lt, HW, C, dn=0, reps=50):
    """Average ms of one fused attention launch (one captured graph of `reps` launches) and its output."""
    out = torch.empty(nz * Lt, C, device=qk_bf16.device, dtype=torch.bfloat16)
    ms = c_float()
    torch.cuda.synchronize()
    _check(lib().sr3_bench_attention(_ptr(qk_bf16), _ptr(vT_bf16), _ptr(out), nz, Lt, HW, C, dn, reps, ctypes.byref(ms)))
    return ms.value, out


def test_gemm(a_bf16, b_bf16, block_n):
    M, K = a_bf16.shape
    N = b_bf16.shape[0]
    d = torch.empty(M, N, device=a_bf16.device, dtype=torch.float32)
    _check(lib().sr3_test_gemm(_ptr(a_bf16), _ptr(b_bf16), _ptr(d), M, N, K, block_n, _stream()))
    return d


def test_conv(x_nhwc_bf16, w_oihw, bias, ksize, stride, want_stats=False):
    B, H, W, Cin = x_nhwc_bf16.shape
    Cout = w_oihw.shape[0]
    y = torch.empty(B, H // stride, W // stride, Cout, device=x_nhwc_bf16.device, dtype=torch.float32)
    stats = torch.zeros(B, Cout, 2, device=y.device, dtype=torch.float64) if want_stats else None
    _check(lib().sr3_test_conv(_ptr(x_nhwc_bf16), _ptr(w_oihw), _ptr(bias), _ptr(y), _ptr(stats), B, H, W, Cin, Cout, ksize, stride, _stream()))
    return y, stats


def test_conv_ex(x, w, ksize=3, stride=1, bias=None, bias2=None, resid=None, x2=None, w2=None, want_bf16=False, want_stats=False,
                 fold_up=False, precise=False):
    """One image conv as a UNet layer builds it (sr3_test_conv_ex); CUDA operands.  x bf16 NHWC [B,H,W,Cin] ([B,H,W,2Cin] = [hi | lo] when
    precise), w fp32 OIHW.  Returns (y fp32 NHWC, y_bf16 or None, stats fp64 [B,Cout,2] or None, geometry dict)."""
    B, H, W, CX = x.shape
    Cin = CX // 2 if precise else CX
    Cout = w.shape[0]
    OH, OW = (2 * H, 2 * W) if fold_up else (H // stride, W // stride)
    y = torch.empty(B, OH, OW, Cout, device=x.device, dtype=torch.float32)
    yb = torch.empty(B, OH, OW, Cout * (2 if precise else 1), device=x.device, dtype=torch.bfloat16) if want_bf16 else None
    stats = torch.zeros(B, Cout, 2, device=x.device, dtype=torch.float64) if want_stats else None
    keep = [_f32c(t, x.device) if t is not None else None for t in (w, bias, bias2, resid, w2)]
    a = TestConvArgsC()
    a.x, a.w, a.bias, a.bias2, a.resid = x.data_ptr(), *[(t.data_ptr() if t is not None else None) for t in keep[:4]]
    a.x2 = x2.data_ptr() if x2 is not None else None
    a.w2 = keep[4].data_ptr() if keep[4] is not None else None
    a.y, a.y_bf16, a.stats = y.data_ptr(), (yb.data_ptr() if yb is not None else None), (stats.data_ptr() if stats is not None else None)
    a.B, a.H, a.W, a.Cin, a.Cout = B, H, W, Cin, Cout
    a.Cin2 = (x2.shape[3] // (2 if precise else 1)) if x2 is not None else 0
    a.ksize, a.stride, a.fold_up, a.precise = ksize, stride, int(bool(fold_up)), int(bool(precise))
    geo = GemmGeometryC()
    _check(lib().sr3_test_conv_ex(ctypes.byref(a), ctypes.byref(geo), _stream()))
    return y, yb, stats, {n: getattr(geo, n) for n, _ in GemmGeometryC._fields_}


SCHEDULES = {0: "cooperative", 1: "pingpong"}


def _tile_schedule(handle, op):
    geo, sch, hwc = GemmGeometryC(), c_int(), (c_int * 3)()
    _check(lib().sr3_tile_schedule(handle, int(op), ctypes.byref(geo), ctypes.byref(sch), hwc))
    if sch.value < 0:
        return None
    d = {n: getattr(geo, n) for n, _ in GemmGeometryC._fields_}
    d["schedule"] = SCHEDULES[sch.value]
    d["out_hwc"] = tuple(hwc)
    return d


def last_test_conv_schedule():
    """Geometry dict + "schedule" + "out_hwc" of the most recent test_conv_ex call on this thread."""
    return _tile_schedule(None, 0)


def test_wgrad(dy, x, ksize, stride=1, cout_valid=None, cin_valid=None, slices=0, gscale=1.0, raw=False):
    """Weight gradient through wgrad_kernel + wgrad_reduce_kernel (sr3_test_wgrad).  dy bf16 NHWC [B,OH,OW,CY], x bf16 NHWC [B,H,W,Cin].
    Returns (grad fp32 OIHW [cout_valid, cin_valid, k, k], or [B, CY, Cin] when raw; slices used)."""
    B, OH, OW, CY = dy.shape
    Cin = x.shape[3]
    cv = CY if cout_valid is None else cout_valid
    civ = Cin if cin_valid is None else cin_valid
    shape = (B, CY, Cin) if raw else (cv, civ, ksize, ksize)
    g = torch.empty(shape, device=dy.device, dtype=torch.float32)
    used = c_int()
    _check(lib().sr3_test_wgrad(_ptr(dy), _ptr(x), _ptr(g), B, OH, OW, CY, Cin, ksize, stride, cv, civ, int(slices), float(gscale), int(bool(raw)),
                                ctypes.byref(used), _stream()))
    return g, used.value


def test_conv_groupnorm(x_nhwc_bf16, w_oihw, bias, gamma, beta, groups, silu, ksize):
    """conv (+ statistics in the epilogue) -> GroupNorm(+SiLU) apply: returns (y fp32 NHWC, a bf16 NHWC)."""
    B, H, W, Cin = x_nhwc_bf16.shape
    Cout = w_oihw.shape[0]
    y = torch.empty(B, H, W, Cout, device=x_nhwc_bf16.device, dtype=torch.float32)
    a = torch.empty(B, H, W, Cout, device=x_nhwc_bf16.device, dtype=torch.bfloat16)
    _check(lib().sr3_test_conv_groupnorm(_ptr(x_nhwc_bf16), _ptr(w_oihw), _ptr(bias), _ptr(gamma), _ptr(beta), groups, int(silu), _ptr(y), _ptr(a),
                                         B, H, W, Cin, Cout, ksize, _stream()))
    return y, a


def adam_step(table_dev, n_tensors, lr, beta1, beta2, eps, step, grad_scale=1.0):
    """torch.optim.Adam step over a device table of {param, grad, exp_avg, exp_avg_sq, numel} records (int64 [n, 5]) in one launch."""
    _check(lib().sr3_adam_step(_ptr(table_dev), int(n_tensors), float(lr), float(beta1), float(beta2), float(eps), int(step), float(grad_scale), _stream()))


# ---- kernel-level hooks of the training backward (CUDA tensors in, CUDA tensors out; see include/sr3_b200.h)
def test_groupnorm_layer(x0, st0, gamma, beta, groups, silu, dA, x1=None, st1=None, add=None, dst0=None, acc0=False, drop=None, gscale=1.0):
    """GroupNorm(+SiLU, +Dropout) forward apply then backward, as the training plan pairs them.  x0 / x1 fp32 [B,HW,C0|C1], st fp64 [B,C,2],
    dA fp32 [B,HW,C], add fp32 [B,HW,>=C], dst0 (initial, accumulated into when acc0) fp32 [B,HW,C0].  drop: None, ("philox", p, seed,
    layer) or ("mask", p, uint8 [B,C,HW]).  Returns a dict: a (bf16), mr, dst0, dst0_b, gsum0, dst1, dgamma, dbeta."""
    B, HW, C0 = x0.shape
    C1 = 0 if x1 is None else x1.shape[2]
    C = C0 + C1
    dev = x0.device
    out = {"a": torch.empty(B, HW, C, device=dev, dtype=torch.bfloat16), "mr": torch.empty(B, groups, 2, device=dev),
           "dst0": dst0.clone() if dst0 is not None else torch.zeros(B, HW, C0, device=dev),
           "dst0_b": torch.empty(B, HW, C0, device=dev, dtype=torch.bfloat16), "gsum0": torch.zeros(B, C0, device=dev),
           "dst1": torch.empty(B, HW, C1, device=dev) if C1 else None, "dgamma": torch.empty(C, device=dev), "dbeta": torch.empty(C, device=dev)}
    a = TestGroupNormArgsC()
    for n, t in (("x0", x0), ("x1", x1), ("st0", st0), ("st1", st1), ("gamma", gamma), ("beta", beta), ("dA", dA), ("add", add)):
        setattr(a, n, t.data_ptr() if t is not None else None)
    for n in ("a_bf16", "mr", "dst0", "dst0_b", "gsum0", "dst1", "dgamma", "dbeta"):
        k = "a" if n == "a_bf16" else n
        setattr(a, n, out[k].data_ptr() if out[k] is not None else None)
    a.B, a.HW, a.C0, a.C1, a.groups, a.silu = B, HW, C0, C1, groups, int(bool(silu))
    a.add_ld = add.shape[2] if add is not None else 0
    a.acc0, a.gscale = int(bool(acc0)), float(gscale)
    if drop is not None:
        if drop[0] == "philox":
            a.drop, a.drop_p, a.drop_seed, a.drop_layer = 1, float(drop[1]), int(drop[2]), int(drop[3])
        else:
            a.drop, a.drop_p, a.drop_mask = 2, float(drop[1]), drop[2].data_ptr()
    _check(lib().sr3_test_groupnorm_layer(ctypes.byref(a), _stream()))
    return out


def test_grad_combine(a, b=None, dst=None, acc=False, want_bf16=True, want_gsum=True, bias_outputs=0, gscale=1.0):
    """grad_combine_kernel (+ bias_grad_kernel into bias_outputs = 0, 1 or 2 destinations).  a, b, dst fp32 [B,HW,C] (dst is updated in
    place).  Returns (dst_b, gsum, [bias gradients])."""
    B, HW, C = a.shape
    dev = a.device
    db = torch.empty(B, HW, C, device=dev, dtype=torch.bfloat16) if want_bf16 else None
    gs = torch.zeros(B, C, device=dev) if want_gsum else None
    bias = [torch.empty(C, device=dev) for _ in range(bias_outputs)]
    _check(lib().sr3_test_grad_combine(_ptr(a), _ptr(b), _ptr(dst), int(bool(acc)), _ptr(db), _ptr(gs), _ptr(bias[0] if bias else None),
                                       _ptr(bias[1] if len(bias) > 1 else None), float(gscale), B, HW, C, _stream()))
    return db, gs, bias


DGRAD_FORMS = {"conv": 0, "down": 1, "up": 2}


def test_dgrad(dy, w_oihw, form, H, W):
    """Data gradient on the tile kernel with the weight packed on the device (sr3_test_dgrad).  dy bf16 NHWC; w fp32 OIHW [Cout,Cin,k,k];
    H, W: the conv's input size.  Returns dx fp32 [B,H,W,Cin]."""
    B, CY = dy.shape[0], dy.shape[3]
    Cout, Cin, k = w_oihw.shape[0], w_oihw.shape[1], w_oihw.shape[2]
    dx = torch.empty(B, H, W, Cin, device=dy.device)
    w = _f32c(w_oihw, dy.device)
    _check(lib().sr3_test_dgrad(_ptr(dy), _ptr(w), _ptr(dx), DGRAD_FORMS[form], B, H, W, CY, Cin, Cout, k, _stream()))
    return dx


def test_attention_bwd(qk, vT, P, dO, nz, Lt, HW, C):
    """Attention backward from the transposes to the bf16 copy of d(qkv).  Returns (dS fp32 [nz*Lt,Lt], dS bf16, dqkv fp32 [nz*Lt,3C],
    dqkv bf16)."""
    dev = qk.device
    dS = torch.empty(nz * Lt, Lt, device=dev)
    dSb = torch.empty(nz * Lt, Lt, device=dev, dtype=torch.bfloat16)
    dqkv = torch.empty(nz * Lt, 3 * C, device=dev)
    dqkvb = torch.empty(nz * Lt, 3 * C, device=dev, dtype=torch.bfloat16)
    _check(lib().sr3_test_attention_bwd(_ptr(qk), _ptr(vT), _ptr(P), _ptr(dO), _ptr(dS), _ptr(dSb), _ptr(dqkv), _ptr(dqkvb), nz, Lt, HW, C, _stream()))
    return dS, dSb, dqkv, dqkvb


def test_film_embed_bwd(wf, tau, dfilm, nl, w1, b1, w2, gscale=1.0):
    """film_bwd_kernel + embed_bwd_kernel.  Returns a dict: dwf, dbf, dcb, dtau, dw1, db1, dw2, db2."""
    F, inner = wf.shape
    B = tau.shape[0]
    dev = wf.device
    out = {"dwf": torch.empty(F, inner, device=dev), "dbf": torch.empty(F, device=dev), "dcb": torch.empty(F, device=dev),
           "dtau": torch.empty(B, inner, device=dev), "dw1": torch.empty(4 * inner, inner, device=dev), "db1": torch.empty(4 * inner, device=dev),
           "dw2": torch.empty(inner, 4 * inner, device=dev), "db2": torch.empty(inner, device=dev)}
    a = TestFilmArgsC()
    for n, t in (("wf", wf), ("tau", tau), ("dfilm", dfilm), ("nl", nl), ("w1", w1), ("b1", b1), ("w2", w2)):
        setattr(a, n, t.data_ptr())
    for n, t in out.items():
        setattr(a, n, t.data_ptr())
    a.F, a.inner, a.B, a.gscale = F, inner, B, float(gscale)
    _check(lib().sr3_test_film_embed_bwd(ctypes.byref(a), _stream()))
    return out


def test_film_embed_fwd(nl, w1, b1, w2, b2, wf, bf, cb):
    """embed_kernel + film_kernel as the plan launches them; CUDA fp32 operands, nl [B].  Returns (tau [B, inner], film [B, F])."""
    F, inner = wf.shape
    B = nl.numel()
    tau = torch.empty(B, inner, device=wf.device)
    film = torch.empty(B, F, device=wf.device)
    _check(lib().sr3_test_film_embed_fwd(*[_ptr(t) for t in (nl, w1, b1, w2, b2, wf, bf, cb, tau, film)], F, inner, B, _stream()))
    return tau, film


def test_attention_unfused(qk, vT, nz, Lt, HW, C, precise=False):
    """The unfused attention launches: qk bf16 [nz*Lt, 2C PW], vT bf16 [nz*C, Lt PW] (PW = 2 in precise mode) -> (S fp32 [nz*Lt, Lt],
    P bf16 [nz*Lt, Lt PW], O bf16 [nz*Lt, C PW])."""
    pw = 2 if precise else 1
    dev = qk.device
    S = torch.empty(nz * Lt, Lt, device=dev)
    P = torch.empty(nz * Lt, Lt * pw, device=dev, dtype=torch.bfloat16)
    O = torch.empty(nz * Lt, C * pw, device=dev, dtype=torch.bfloat16)
    _check(lib().sr3_test_attention_unfused(_ptr(qk), _ptr(vT), _ptr(S), _ptr(P), _ptr(O), nz, Lt, HW, C, int(bool(precise)), _stream()))
    return S, P, O


def test_loss_grad(noise, eps, l2, deps=None, ld=64):
    """loss_grad_kernel.  noise, eps fp32 NCHW.  deps: bf16 [B,H,W,ld] updated in place (fresh zeros by default).  Returns (loss, deps,
    bias_sum [C])."""
    B, C, H, W = noise.shape
    if deps is None:
        deps = torch.zeros(B, H, W, ld, device=noise.device, dtype=torch.bfloat16)
    bias = torch.zeros(C, device=noise.device)
    loss = c_double()
    _check(lib().sr3_test_loss_grad(_ptr(noise), _ptr(eps), B, C, H, W, int(bool(l2)), ctypes.byref(loss), _ptr(deps), deps.shape[3], _ptr(bias),
                                    _stream()))
    return loss.value, deps, bias


def test_grad_load(g, deps=None, ld=64):
    """grad_load_kernel.  g fp32 NCHW.  deps: bf16 [B,H,W,ld] updated in place (fresh zeros by default).  Returns (deps, bias_sum [C])."""
    B, C, H, W = g.shape
    if deps is None:
        deps = torch.zeros(B, H, W, ld, device=g.device, dtype=torch.bfloat16)
    bias = torch.zeros(C, device=g.device)
    _check(lib().sr3_test_grad_load(_ptr(g), B, C, H, W, _ptr(deps), deps.shape[3], _ptr(bias), _stream()))
    return deps, bias


def test_noise_level_bwd(nl, w1, b1, w2, dtau):
    """noise_level_bwd_kernel: nl [B], w1 [4 inner, inner], b1, w2 [inner, 4 inner], dtau [B, inner] (CUDA fp32) -> dnl [B]."""
    B, inner = dtau.shape
    dnl = torch.empty(B, device=nl.device)
    _check(lib().sr3_test_noise_level_bwd(*[_ptr(t) for t in (nl, w1, b1, w2, dtau, dnl)], inner, B, _stream()))
    return dnl


def test_input_grad(dy, w_oihw):
    """The input gradient of the UNet backward: dy bf16 NHWC [B,H,W,inner] (the first conv's output gradient), w fp32 OIHW
    [inner,in_channel,3,3] -> dx fp32 NCHW [B,in_channel,H,W]."""
    B, H, W, inner = dy.shape
    cin = w_oihw.shape[1]
    dx = torch.empty(B, cin, H, W, device=dy.device)
    w = _f32c(w_oihw, dy.device)
    _check(lib().sr3_test_input_grad(_ptr(dy), _ptr(w), _ptr(dx), B, H, W, inner, cin, _stream()))
    return dx
