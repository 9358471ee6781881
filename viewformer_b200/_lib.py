"""ctypes binding of libvf_b200.so (include/vf_b200.h) + thin tensor-level helpers.

torch is used here only as the device-memory / stream plumbing.  ``PROTOTYPES`` declares every entry point's parameter types, so a
call site passes tensors, plain Python numbers and the current CUDA stream handle, and ctypes converts them as the header says.
There is no CPU or PyTorch fallback: if the shared library is missing or the device is not sm_90, calls raise.
"""
import ctypes as C
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("VF_B200_LIB") or os.path.join(HERE, "libvf_b200.so")

F32, BF16, F16X2 = 0, 1, 2     # F16X2: an fp32 value as two fp16 (hi | lo*2^11) along the channel axis — torch.float16 tensors with 2C channels
ACT_NONE, ACT_GELU = 0, 1
BIAS_NONE, BIAS_N, BIAS_M = 0, 1, 2


class LibraryError(RuntimeError):
    pass


class DevPtr(C.c_void_p):
    """Argument type of a device pointer: a CUDA tensor passes its data_ptr(), an int its own value, None NULL; an explicit c_void_p is
    taken as it is.  A CPU tensor raises here instead of faulting on the device.  The address goes through c_void_p's own conversion,
    which keeps the full pointer width (a bare int returned from here would be passed as a C int) and costs less than a c_void_p object."""

    @classmethod
    def from_param(cls, obj):
        if isinstance(obj, torch.Tensor):
            if not obj.is_cuda:
                raise LibraryError(f"a device pointer argument got a {obj.device} tensor")
            obj = obj.data_ptr()
        return C.c_void_p.from_param(obj)            # an int, None or a c_void_p; anything else is a TypeError


_p = DevPtr.from_param      # explicit conversion for raw callers that still wrap their pointers themselves


# Host-side mirrors of the parameter structs of include/vf_b200.h (tests/test_abi.py compares them field by field).
class SimtGemm(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("a_dtype", C.c_int), ("conv", C.c_int),
        ("N", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cin", C.c_int),
        ("OH", C.c_int), ("OW", C.c_int), ("KH", C.c_int), ("KW", C.c_int), ("stride", C.c_int),
        ("pad_t", C.c_int), ("pad_l", C.c_int), ("upsample2x", C.c_int),
        ("a_sm", C.c_int64), ("a_sk", C.c_int64),
        ("B", C.c_void_p), ("b_dtype", C.c_int), ("b_sk", C.c_int64), ("b_sn", C.c_int64),
        ("M", C.c_int), ("Ncols", C.c_int), ("K", C.c_int), ("batch1", C.c_int), ("batch2", C.c_int),
        ("a_sb1", C.c_int64), ("a_sb2", C.c_int64), ("b_sb1", C.c_int64), ("b_sb2", C.c_int64),
        ("c_sb1", C.c_int64), ("c_sb2", C.c_int64),
        ("alpha", C.c_float), ("bias", C.c_void_p), ("bias_mode", C.c_int), ("act", C.c_int),
        ("residual", C.c_void_p), ("C_f32", C.c_void_p), ("C_bf16", C.c_void_p), ("ldc", C.c_int64),
    ]


class TcGemm(C.Structure):
    _fields_ = [
        ("conv", C.c_int), ("ab_dtype", C.c_int), ("A", C.c_void_p), ("B", C.c_void_p),
        ("M", C.c_int), ("Ncols", C.c_int), ("K", C.c_int), ("batch1", C.c_int), ("batch2", C.c_int),
        ("lda", C.c_int64), ("ldb", C.c_int64),
        ("a_sb1", C.c_int64), ("a_sb2", C.c_int64), ("b_sb1", C.c_int64), ("b_sb2", C.c_int64),
        ("N", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Ctot", C.c_int), ("Cin", C.c_int),
        ("OH", C.c_int), ("OW", C.c_int), ("ntaps", C.c_int),
        ("tap_dy", C.c_int * 9), ("tap_dx", C.c_int * 9), ("tap_coff", C.c_int * 9),
        ("causal_block", C.c_int), ("causal_skip_n", C.c_int),
        ("alpha", C.c_float), ("bias", C.c_void_p), ("bias_mode", C.c_int), ("act", C.c_int),
        ("residual", C.c_void_p), ("C_f32", C.c_void_p), ("C_bf16", C.c_void_p),
        ("ldc", C.c_int64), ("c_sb1", C.c_int64), ("c_sb2", C.c_int64),
        ("gn_sums", C.c_void_p), ("gn_groups", C.c_int), ("gn_rows_per_img", C.c_int),
        ("norm_mean_rstd", C.c_void_p), ("norm_gamma", C.c_void_p), ("norm_beta", C.c_void_p),
        ("norm_groups", C.c_int), ("norm_swish", C.c_int),
        ("exact_lo_a", C.c_int64), ("exact_lo_b", C.c_int64),
    ]


class ConvWeightsBf16(C.Structure):            # a row of vf_conv_weights_bf16's device table
    _fields_ = [("w_kn", C.c_void_p), ("fw_bf16", C.c_void_p), ("bw_bf16", C.c_void_p), ("cin", C.c_int64), ("cout", C.c_int64)]


class DenseWeightsBf16(C.Structure):           # a row of vf_dense_weights_bf16's device table
    _fields_ = [("w_kn", C.c_void_p), ("fw_bf16", C.c_void_p), ("bw_bf16", C.c_void_p), ("k", C.c_int64), ("n", C.c_int64)]


def _prototypes():
    """The parameter types of every function include/vf_b200.h declares, in order (tests/test_abi.py holds this table to the header).
    p: a device pointer, the two weight tables included; s: vf_stream_t.  The parameter blocks and the plan array are host memory."""
    i, i64, u64, f32, f64, p, s = C.c_int, C.c_int64, C.c_uint64, C.c_float, C.c_double, DevPtr, C.c_void_p
    return {
        "vf_last_error": [], "vf_version": [], "vf_sizeof_simt_gemm": [], "vf_sizeof_tc_gemm": [], "vf_device_check": [],
        "vf_u8_to_unit_f32": [p, p, i64, i64, i64, s], "vf_f01_to_unit_f32": [p, p, i64, i64, i64, s], "vf_unit_f32_to_u8": [p, p, i64, s],
        "vf_nchw_to_nhwc_f32": [p, p, i, i, i, i, s], "vf_nhwc_to_nchw_f32": [p, p, i, i, i, i, s], "vf_split_f16x2": [p, i64, i, p, s],
        "vf_groupnorm_stats": [p, i, i, i, i, f32, p, p, s], "vf_groupnorm_finalize": [p, i, f64, f32, p, s],
        "vf_groupnorm_apply": [p, i, p, p, p, i, i, i, i, i, f32, i, i, i, p, i, s], "vf_conv3x3_small_cin": [p, p, p, i, i, i, i, i, p, p, s],
        "vf_conv3x3_small_cout": [p, i, p, p, i, i, i, i, i, p, s], "vf_layernorm": [p, p, p, i64, i, f32, p, i, s],
        "vf_simt_gemm": [C.POINTER(SimtGemm), s], "vf_tc_gemm": [C.POINTER(TcGemm), s], "vf_tc_gemm_plan": [C.POINTER(TcGemm), C.POINTER(C.c_int)],
        "vf_attn_block_causal_decode": [p, p, i, i, i, i, i, i, i, p, s], "vf_attn_block_multiend": [p, p, i, i, i, i, i, i, i, p, s],
        "vf_attn_multiend_train": [p, p, i, i, i, i, i, i, i, f32, u64, p, p, p, s],
        "vf_attn_multiend_bwd": [p, p, p, p, p, i, i, i, i, i, i, f32, u64, p, s],
        "vf_conv_wgrad": [p, p, i, i, i, i, i, i, i, i, i, i, i, i, i, i64, i64, p, s], "vf_col_sums": [p, i64, i, p, s],
        "vf_groupnorm_bwd": [p, p, p, p, p, i, i, i, i, i, p, p, p, p, p, p, s], "vf_softmax_bwd_rows": [p, p, i64, i, p, s],
        "vf_l1_grad": [p, p, i64, f32, p, p, s], "vf_lincomb3": [f32, p, f32, p, f32, p, i64, p, s],
        "vf_pad_transpose_split": [p, i, i, i, i, i, i, i64, i64, p, s], "vf_sum_splits": [p, i, i, i64, i, p, s],
        "vf_pad_transpose_bf16": [p, i, i, i, i, i, i, i, i64, i64, p, p, p, i, i, p, s], "vf_conv_weights_bf16": [p, i, s],
        "vf_sumpool2x2": [p, i, i, i, i, p, s], "vf_adam": [p, p, p, p, i64, f32, f32, f32, f32, i, f32, s],
        "vf_layernorm_bwd": [p, p, p, p, i64, i, f32, p, p, p, s], "vf_gelu_fwd": [p, i64, p, s], "vf_gelu_bwd": [p, p, i64, p, s],
        "vf_migt_embed_bwd": [p, p, i, i64, i, i, p, p, p, s], "vf_cross_entropy_grad": [p, p, p, i64, i, f32, p, s],
        "vf_pose_loss_grad": [p, p, p, i64, i, f32, f32, f32, p, s], "vf_adamw_keras": [p, p, p, p, i64, f32, f32, f32, f32, f32, i, f32, f32, s],
        "vf_sumsq": [p, i64, p, s], "vf_dropout": [p, i64, f32, u64, p, s], "vf_to_bf16": [p, i64, f32, u64, p, p, s],
        "vf_dense_weights_bf16": [p, i, s], "vf_resize_u8": [p, i, i, i, i, i, i, i, p, s], "vf_resize_f32": [p, i, i, i, i, i, i, i, p, s],
        "vf_image_pair_sums": [p, p, i, i64, p, s], "vf_ssim_u8": [p, p, i, i, i, i, p, s], "vf_ssim_u8_k": [p, p, i, i, i, i, f64, f64, p, s],
        "vf_vq_lookup": [p, p, p, i64, i, i, p, p, p, s], "vf_vq_prepare_codebook_f16": [p, i, i, p, s],
        "vf_vq_lookup_fused": [p, p, p, p, p, i64, i, i, f32, p, p, p, p, p, s], "vf_gather_rows": [p, p, i64, i, i64, p, s],
        "vf_vq_ema_stats": [p, p, i64, i, i, p, p, s], "vf_vq_commit_grad": [p, p, p, i, i, f32, i, p, s],
        "vf_vq_ema_update": [p, p, i, i, f32, f32, f32, p, p, p, p, p, s], "vf_vq_prepare_codebook": [p, i, i, p, p, s],
        "vf_migt_embed": [p, i, p, p, p, i64, i, i, p, s], "vf_softmax_rows": [p, i64, i, i, i64, i, i, i, p, i, i64, s],
        "vf_argmax_rows": [p, i64, i, i64, p, s], "vf_pose_postprocess": [p, i64, f32, p, s], "vf_cameras_prepare": [p, i, i, i, p, p, s],
        "vf_cameras_from_relative": [p, p, i, i, p, s], "vf_camera_knn": [p, i64, i64, p, i, i, i, p, p, s],
        "vf_cross_entropy_rows": [p, p, i64, i, f32, p, s], "vf_pose_loss_rows": [p, p, i64, i, f32, p, p, s], "vf_row_mean": [p, i64, i, i, p, s],
    }


PROTOTYPES = _prototypes()          # every entry point returns int, except vf_last_error (const char*)
EXPORTS = tuple(PROTOTYPES)

_lib = None
_device_ok = []


def load(require_device=False):
    """dlopen the in-tree library and declare every entry point's types.  Fails loudly — there is no fallback path."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LibraryError(f"{LIB_PATH} not found — run `python -m viewformer_b200.build` (no CPU/PyTorch fallback exists)")
        lib = C.CDLL(LIB_PATH)
        for name, argtypes in PROTOTYPES.items():
            if not hasattr(lib, name):
                raise LibraryError(f"{LIB_PATH} does not export {name}")
            fn = getattr(lib, name)
            fn.argtypes = argtypes
            fn.restype = C.c_char_p if name == "vf_last_error" else C.c_int
        if lib.vf_sizeof_simt_gemm() != C.sizeof(SimtGemm) or lib.vf_sizeof_tc_gemm() != C.sizeof(TcGemm):
            raise LibraryError("parameter struct layout mismatch between _lib.py and include/vf_b200.h")
        _lib = lib
    if require_device and not _device_ok:
        if not torch.cuda.is_available():
            raise LibraryError("viewformer_b200 needs a CUDA device (sm_90a); no CPU fallback exists")
        rc = _lib.vf_device_check()
        if rc != 0:
            raise LibraryError(_lib.vf_last_error().decode())
        _device_ok.append(True)          # checked once per process (cudaGetDeviceProperties is slow)
    return _lib


_launches = 0


def reset_launch_count():
    global _launches
    _launches = 0


def launch_count():
    """Number of libvf_b200 kernel-launching C-ABI calls since the last reset (bench.py's gpu_launches)."""
    return _launches


def _check(rc):
    global _launches
    _launches += 1
    if rc != 0:
        raise LibraryError(f"libvf_b200 error {rc}: {_lib.vf_last_error().decode()}")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _seed64(seed):                  # a dropout seed as the uint64 the kernels hash: negative and wide seeds wrap here, explicitly
    return int(seed) & ((1 << 64) - 1)


def on_model_device(fn):
    """Method decorator for the model classes: run with the model's device as the CURRENT CUDA device.  Every wrapper below launches on
    ``torch.cuda.current_stream()`` of the current device and the library caches per-device attributes, so a model built with
    ``device='cuda:1'`` must not run while device 0 is current."""
    import functools

    @functools.wraps(fn)
    def wrap(self, *a, **k):
        dev = getattr(self, "device", None)
        if dev is None or dev.type != "cuda" or dev.index is None or dev.index == torch.cuda.current_device():
            return fn(self, *a, **k)
        with torch.cuda.device(dev):
            return fn(self, *a, **k)
    return wrap


def _dt(t):
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.bfloat16:
        return BF16
    if t.dtype == torch.float16:
        return F16X2
    raise TypeError(f"unsupported dtype {t.dtype}")


def _dev(t, dtype=None):
    assert t.is_cuda and t.is_contiguous(), "device-contiguous tensor expected"
    if t.device.index != torch.cuda.current_device():
        raise LibraryError(f"tensor on cuda:{t.device.index} but the current device is cuda:{torch.cuda.current_device()}: kernels launch on the "
                           "current device's stream (the model classes switch devices themselves; raw _lib callers must use torch.cuda.device)")
    if dtype is not None:
        assert t.dtype == dtype, f"expected {dtype}, got {t.dtype}"
    return t


# ----------------------------------------------------------------------------------------------- pixels / layout
def u8_to_unit(x_u8, first_views=None):
    """uint8 -> f32 x*(1/255)*2-1.  ``first_views=n`` on a [B,T,H,W,3] tensor converts views 0..n-1 of every scene
    into a contiguous [B*n,H,W,3] tensor (strided read, no gather copy)."""
    lib = load(True)
    _dev(x_u8, torch.uint8)
    if first_views is None:
        out = torch.empty(x_u8.shape, dtype=torch.float32, device=x_u8.device)
        _check(lib.vf_u8_to_unit_f32(x_u8, out, 1, x_u8.numel(), 0, _stream()))
        return out
    b, t = x_u8.shape[:2]
    per_view = x_u8[0, 0].numel()
    out = torch.empty((b * first_views,) + tuple(x_u8.shape[2:]), dtype=torch.float32, device=x_u8.device)
    _check(lib.vf_u8_to_unit_f32(x_u8, out, b, first_views * per_view, t * per_view, _stream()))
    return out


def unit_to_u8(x):
    lib = load(True)
    _dev(x, torch.float32)
    out = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    _check(lib.vf_unit_f32_to_u8(x, out, x.numel(), _stream()))
    return out


def nchw_to_nhwc(x):
    lib = load(True)
    _dev(x, torch.float32)
    n, c, h, w = x.shape
    out = torch.empty((n, h, w, c), dtype=torch.float32, device=x.device)
    _check(lib.vf_nchw_to_nhwc_f32(x, out, n, c, h, w, _stream()))
    return out


def nhwc_to_nchw(x):
    lib = load(True)
    _dev(x, torch.float32)
    n, h, w, c = x.shape
    out = torch.empty((n, c, h, w), dtype=torch.float32, device=x.device)
    _check(lib.vf_nhwc_to_nchw_f32(x, out, n, c, h, w, _stream()))
    return out


def resize_u8(x_u8, size, method=None):
    """data/_common.py:19-62 (resize, then resize_th) for uint8 NHWC images [N,H,W,C] -> [N,size,size,C]: bilinear (align_corners=False)
    when the height shrinks, nearest when it grows (or the explicit ``method``).  The input comes back unchanged when W == size (resize()
    tests shape[-2] of NHWC) or H == size (resize_th() tests shape[-2] of NCHW), so a non-square frame with one side already at ``size``
    stays non-square, as in the reference."""
    lib = load(True)
    _dev(x_u8, torch.uint8)
    n, h, w, c = x_u8.shape
    if w == size or h == size:
        return x_u8
    if method is None:
        method = "nearest" if size > h else "bilinear"
    assert method in ("nearest", "bilinear")
    out = torch.empty((n, size, size, c), dtype=torch.uint8, device=x_u8.device)
    _check(lib.vf_resize_u8(x_u8, n, h, w, c, size, size, int(method == "bilinear"), out, _stream()))
    return out


def image_pair_sums(a_u8, b_u8):
    """uint8 images [N,...] x2 -> int64 [N,2] = (sum |a-b|, sum (a-b)^2) per image (exact)."""
    lib = load(True)
    _dev(a_u8, torch.uint8)
    _dev(b_u8, torch.uint8)
    assert a_u8.shape == b_u8.shape
    n = a_u8.shape[0]
    out = torch.empty((n, 2), dtype=torch.int64, device=a_u8.device)
    _check(lib.vf_image_pair_sums(a_u8, b_u8, n, a_u8[0].numel() if n else 1, out, _stream()))
    return out


def ssim_u8(a_u8, b_u8, k1=None, k2=None):
    """utils/metrics.py:17-73 on uint8 NHWC images -> float64 [N] mean SSIM per image.  ``k1`` / ``k2``: the K1 / K2 of ``ssim()``
    (defaults 0.01 / 0.03); the reference's SSIMMetric passes K1 = 1 (metrics.py:183)."""
    lib = load(True)
    if a_u8.dim() != 4 or a_u8.shape != b_u8.shape:
        raise ValueError(f"ssim_u8: a and b must be uint8 [N,H,W,C] images of one shape, got {tuple(a_u8.shape)} and {tuple(b_u8.shape)}")
    _dev(a_u8, torch.uint8)
    _dev(b_u8, torch.uint8)
    n, h, w, c = a_u8.shape
    out = torch.empty((n,), dtype=torch.float64, device=a_u8.device)
    if k1 is None and k2 is None:
        _check(lib.vf_ssim_u8(a_u8, b_u8, n, h, w, c, out, _stream()))
    else:
        _check(lib.vf_ssim_u8_k(a_u8, b_u8, n, h, w, c, 0.01 if k1 is None else float(k1), 0.03 if k2 is None else float(k2), out, _stream()))
    return out


# ----------------------------------------------------------------------------------------------- norms
def groupnorm(x, gamma, beta, *, swish, out_dtype, eps=1e-6, groups=32, upsample=False, normalize=True, s2d=False, stats=None):
    """x f32|bf16 [N,H,W,C] -> GroupNorm(32) [+swish] [+nearest x2] as out_dtype (vqgan_th.py:11-17,29-30).  The statistics are ``stats``
    (mean, rstd) [N, groups, 2] when given, else gn_mean_rstd(x): a bf16 x must then carry the statistics its producing conv accumulated
    (from the fp32 accumulators) in ``_gn_sums``."""
    lib = load(True)
    _dev(x)
    n, h, w, c = x.shape
    if normalize and stats is None:
        stats = gn_mean_rstd(x, groups, eps)
    oshape = (n, 2 * h, 2 * w, c) if upsample else ((n, h // 2, w // 2, 4 * c) if s2d else (n, h, w, c))
    if out_dtype == torch.float16:          # split-fp16 pair [hi | lo] (exact tensor-core operand): twice the channels
        oshape = oshape[:3] + (2 * oshape[3],)
    y = torch.empty(oshape, dtype=out_dtype, device=x.device)
    _check(lib.vf_groupnorm_apply(x, _dt(x), stats, gamma, beta, n, h, w, c, groups, eps,
                                  int(normalize), int(swish), 1 if upsample else (2 if s2d else 0), y, _dt(y), _stream()))
    return y


def layernorm(x, gamma, beta, out_dtype, eps=1e-5):
    lib = load(True)
    _dev(x, torch.float32)
    d = x.shape[-1]
    rows = x.numel() // d
    y = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    _check(lib.vf_layernorm(x, gamma, beta, rows, d, eps, y, _dt(y), _stream()))
    return y


# ----------------------------------------------------------------------------------------------- GEMM / conv
def _epilogue(p, out, ldc, *, c_bs=(0, 0), out2=None, alpha=1.0, bias=None, bias_mode=BIAS_N, act=ACT_NONE, residual=None, c_off=0):
    """The epilogue fields vf_simt_gemm_t and vf_tc_gemm_t share: C = act(alpha*acc + bias) + residual, written to ``out`` and ``out2``
    (one f32, one bf16) from element ``c_off`` on, with row stride ``ldc`` and batch strides ``c_bs``; the residual is f32 and indexed as C."""
    p.alpha, p.act, p.ldc = alpha, act, ldc
    p.c_sb1, p.c_sb2 = c_bs
    p.bias, p.bias_mode = (bias.data_ptr(), bias_mode) if bias is not None else (None, BIAS_NONE)
    p.residual = residual.data_ptr() + c_off * 4 if residual is not None else None
    for o in (o for o in (out, out2) if o is not None):
        if o.dtype == torch.float32:
            p.C_f32 = o.data_ptr() + c_off * 4
        elif o.dtype == torch.bfloat16:
            p.C_bf16 = o.data_ptr() + c_off * 2
        else:
            raise TypeError(f"GEMM output must be float32 or bfloat16, got {o.dtype}")


def simt_conv(x, w_kn, bias, *, kh, stride=1, pad=(1, 1), upsample=False, residual=None, out_dtype=torch.float32, out=None):
    """fp32 CUDA-core convolution.  x [N,H,W,Cin] f32|bf16, w_kn [kh*kh*Cin, Cout] f32."""
    lib = load(True)
    _dev(x)
    n, h, w, cin = x.shape
    cout = w_kn.shape[1]
    vh, vw = (2 * h, 2 * w) if upsample else (h, w)
    if stride == 1:
        oh, ow = vh, vw
    else:
        oh, ow = vh // 2, vw // 2
    if out is None:
        out = torch.empty((n, oh, ow, cout), dtype=out_dtype, device=x.device)
    p = SimtGemm(A=x.data_ptr(), a_dtype=_dt(x), conv=1, N=n, H=h, W=w, Cin=cin, OH=oh, OW=ow, KH=kh, KW=kh, stride=stride,
                 pad_t=pad[0], pad_l=pad[1], upsample2x=int(upsample), B=w_kn.data_ptr(), b_dtype=_dt(w_kn), b_sk=cout, b_sn=1,
                 M=n * oh * ow, Ncols=cout, K=kh * kh * cin, batch1=1, batch2=1)
    _epilogue(p, out, cout, bias=bias, residual=residual)
    _check(lib.vf_simt_gemm(p, _stream()))
    return out


def simt_gemm(A, B, out, *, M, N, K, a_strides, b_strides, ldc, batch=(1, 1), a_bs=(0, 0), b_bs=(0, 0), c_bs=(0, 0),
              alpha=1.0, bias=None, bias_mode=BIAS_NONE, act=ACT_NONE, residual=None, a_off=0, b_off=0, c_off=0):
    """Dense strided fp32 GEMM: C[m,n] = act(alpha*sum_k A(m,k) B(k,n) + bias) + residual.
    a_strides = (stride_m, stride_k), b_strides = (stride_k, stride_n) in elements; *_off element offsets."""
    lib = load(True)
    p = SimtGemm(A=A.data_ptr() + a_off * A.element_size(), a_dtype=_dt(A), conv=0, B=B.data_ptr() + b_off * B.element_size(), b_dtype=_dt(B),
                 M=M, Ncols=N, K=K, batch1=batch[0], batch2=batch[1])
    p.a_sm, p.a_sk = a_strides
    p.b_sk, p.b_sn = b_strides
    p.a_sb1, p.a_sb2 = a_bs
    p.b_sb1, p.b_sb2 = b_bs
    _epilogue(p, out, ldc, c_bs=c_bs, alpha=alpha, bias=bias, bias_mode=bias_mode, act=act, residual=residual, c_off=c_off)
    _check(lib.vf_simt_gemm(p, _stream()))
    return out


_PLAN_KEYS = ("block_n", "TW", "TH", "TN", "halo", "exact", "tiles", "ctas")


def _plan(p):
    """vf_tc_gemm_plan: the tiling vf_tc_gemm would launch for parameter block p, as a dict of _PLAN_KEYS (nothing is launched)."""
    plan = (C.c_int * len(_PLAN_KEYS))()
    rc = load(True).vf_tc_gemm_plan(p, plan)
    if rc != 0:
        raise LibraryError(f"libvf_b200 error {rc}: {_lib.vf_last_error().decode()}")
    return dict(zip(_PLAN_KEYS, plan))


def _fuse_gn_sums(p, out, images, groups, rows_per_img=0):
    """Point p's epilogue (vf_tc_gemm_t.gn_sums) at fresh fp64 GroupNorm sums [images, groups, 2] of ``out``, kept as ``out._gn_sums``."""
    sums = torch.empty((images, groups, 2), dtype=torch.float64, device=out.device)
    p.gn_sums, p.gn_groups, p.gn_rows_per_img = sums.data_ptr(), groups, rows_per_img
    out._gn_sums = (sums, groups)


def tc_gemm(A, B, out, *, M, N, K, lda, ldb, ldc, batch=(1, 1), a_bs=(0, 0), b_bs=(0, 0), c_bs=(0, 0), alpha=1.0,
            bias=None, bias_mode=BIAS_NONE, act=ACT_NONE, residual=None, a_off=0, b_off=0, c_off=0, causal_block=0,
            causal_skip_n=False, out2=None, gn_rows_per_img=0, gn_groups=32, lo_a=None, lo_b=None, k_offsets=None, plan=False):
    """Tensor-core (wgmma) GEMM: C[m,n] = act(alpha*sum_k A[m,k] B[n,k] + bias) + residual; A,B K-major bf16 (or f32 -> TF32).
    ``out2`` optionally receives a second copy in the other dtype (f32 + bf16 from one epilogue).
    float16 operands = split-fp16 pairs (exact mode): a row holds hi(K) at column 0 and lo(K) at column ``lo_a`` / ``lo_b``.
    ``plan=True`` launches nothing and returns the tiling this call would take (see _plan)."""
    lib = load(True)
    assert A.dtype == B.dtype
    p = TcGemm(conv=0, ab_dtype=_dt(A), A=A.data_ptr() + a_off * A.element_size(), B=B.data_ptr() + b_off * B.element_size(),
               M=M, Ncols=N, K=K, batch1=batch[0], batch2=batch[1], lda=lda, ldb=ldb)
    if A.dtype == torch.float16:
        p.exact_lo_a, p.exact_lo_b = (K if lo_a is None else lo_a), (K if lo_b is None else lo_b)
    p.a_sb1, p.a_sb2 = a_bs
    p.b_sb1, p.b_sb2 = b_bs
    p.causal_block, p.causal_skip_n = causal_block, int(causal_skip_n)
    if k_offsets is not None:            # batch1 index b reads A shifted by k_offsets[b] elements along K (vf_tc_gemm_t.ntaps in gemm mode)
        assert len(k_offsets) == batch[0] <= 9
        p.ntaps = len(k_offsets)
        for i, o in enumerate(k_offsets):
            p.tap_coff[i] = int(o)
    _epilogue(p, out, ldc, c_bs=c_bs, out2=out2, alpha=alpha, bias=bias, bias_mode=bias_mode, act=act, residual=residual, c_off=c_off)
    if plan:
        return _plan(p)
    if gn_rows_per_img and batch == (1, 1) and gn_fusable(N, gn_groups, M, gn_rows_per_img, ldc):
        _fuse_gn_sums(p, out, M // gn_rows_per_img, gn_groups, gn_rows_per_img)
    _check(lib.vf_tc_gemm(p, _stream()))
    return out


def gn_fusable(channels, groups, rows, rows_per_img, ldc):
    """Shapes for which the tensor-core epilogue can accumulate GroupNorm statistics (see vf_tc_gemm_t.gn_sums)."""
    if channels % groups:
        return False
    cpg = channels // groups
    return (cpg % 4 == 0 and cpg <= 32 and 32 % cpg == 0 and channels % 128 == 0 and rows_per_img >= 32 and rows_per_img % 32 == 0
            and rows % rows_per_img == 0 and ldc % 4 == 0)


TAPS_3x3 = [(dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
# stride-2 conv over a space-to-depth operand: filter tap (dy,dx) in 0..2 reads phase (dy%2, dx%2) at offset (dy//2, dx//2)
TAPS_S2D = [(dy // 2, dx // 2) for dy in (0, 1, 2) for dx in (0, 1, 2)]


def s2d_coffs(c):
    return [((dy % 2) * 2 + (dx % 2)) * c for dy in (0, 1, 2) for dx in (0, 1, 2)]


def conv3x3_small_cin(x, w_kn, bias, gn_groups=0):
    """exact fp32 conv_in (Cin = 3 or 4): x f32 [N,H,W,Cin], w_kn [9 Cin, Cout].  ``gn_groups=32`` (Cout = 128) also accumulates the
    GroupNorm statistics of the output and attaches them as ``_gn_sums`` (consumed by ``groupnorm``)."""
    lib = load(True)
    _dev(x, torch.float32)
    n, h, w, cin = x.shape
    cout = w_kn.shape[1]
    y = torch.empty((n, h, w, cout), dtype=torch.float32, device=x.device)
    sums = None
    if gn_groups == 32 and cout == 128:
        sums = torch.empty((n, 32, 2), dtype=torch.float64, device=x.device)
    _check(lib.vf_conv3x3_small_cin(x, w_kn, bias, n, h, w, cin, cout, y, sums, _stream()))
    if sums is not None:
        y._gn_sums = (sums, 32)
    return y


def conv3x3_small_cout(x, w_kn, bias):
    """exact fp32-accumulate conv_out (128 -> Cout, Cout = 3 or 4): x f32|bf16 [N,H,W,128], w_kn [1152, Cout]."""
    lib = load(True)
    _dev(x)
    n, h, w, cin = x.shape
    cout = w_kn.shape[1]
    y = torch.empty((n, h, w, cout), dtype=torch.float32, device=x.device)
    _check(lib.vf_conv3x3_small_cout(x, _dt(x), w_kn, bias, n, h, w, cin, cout, y, _stream()))
    return y


def conv_norm_fusable(x, cout):
    """Shapes for which vf_tc_gemm can apply GroupNorm+swish to the conv INPUT on the fly (vf_tc_gemm_t.norm_*): the halo-tile
    path of 3x3 bf16 convs on maps >= 32 rows."""
    n, h, w, c = x.shape
    return x.dtype == torch.bfloat16 and c % 64 == 0 and cout % 128 == 0 and h >= 32 and w >= 8 and n * h * w * cout < 2 ** 31


def gn_mean_rstd(x, groups=32, eps=1e-6):
    """(mean, rstd) float [N, groups, 2] of x [N,H,W,C] — from the statistics its producer fused, else one statistics pass."""
    lib = load(True)
    n, h, w, c = x.shape
    stats = torch.empty((n, groups, 2), dtype=torch.float32, device=x.device)
    fused = getattr(x, "_gn_sums", None)
    if fused is not None and fused[1] == groups:
        _check(lib.vf_groupnorm_finalize(fused[0], n * groups, float(h * w * (c // groups)), eps, stats, _stream()))
    else:
        if x.dtype != torch.float32:
            raise LibraryError("gn_mean_rstd: a bf16 input needs fused statistics from its producer")
        sums = torch.empty((n, groups, 2), dtype=torch.float64, device=x.device)
        _check(lib.vf_groupnorm_stats(x, n, h * w, c, groups, eps, sums, stats, _stream()))
    return stats


def tc_conv(x, w_nk, bias, *, taps=TAPS_3x3, coffs=None, cin=None, out_hw=None, residual=None, out=None,
            out_dtype=torch.float32, out2=None, gn_groups=0, norm=None, plan=False):
    """Tensor-core (wgmma) implicit-GEMM conv.  x [N,H,W,Ctot] bf16|f32 NHWC; w_nk [Cout, ntaps*Cin] (K-major, same dtype).
    ``norm=(mean_rstd, gamma, beta, groups, swish)``: x is the RAW activation and GroupNorm(+swish) is applied to it inside the
    kernel (only for ``conv_norm_fusable`` shapes).  ``plan=True`` launches nothing and returns the tiling this call would take
    (see _plan)."""
    lib = load(True)
    _dev(x)
    n, h, w, ctot = x.shape
    split = 2 if x.dtype == torch.float16 else 1            # exact mode: x = [hi | lo] halves, weights [Cout][tap][hi(Cin) | lo(Cin)]
    cin = ctot // split if cin is None else cin
    cout = w_nk.shape[0]
    oh, ow = (h, w) if out_hw is None else out_hw
    if out is None:
        out = torch.empty((n, oh, ow, cout), dtype=out_dtype, device=x.device)
    assert w_nk.dtype == x.dtype and w_nk.shape[1] == len(taps) * cin * split
    p = TcGemm(conv=1, ab_dtype=_dt(x), A=x.data_ptr(), B=w_nk.data_ptr(), Ncols=cout, N=n, H=h, W=w, Ctot=ctot, Cin=cin, OH=oh, OW=ow,
               ntaps=len(taps))
    for i, (dy, dx) in enumerate(taps):
        p.tap_dy[i], p.tap_dx[i] = dy, dx
        p.tap_coff[i] = 0 if coffs is None else coffs[i]
    _epilogue(p, out, cout, out2=out2, bias=bias, residual=residual)
    if plan:
        return _plan(p)
    if gn_groups and gn_fusable(cout, gn_groups, n * oh * ow, oh * ow, cout):
        _fuse_gn_sums(p, out, n, gn_groups)
    if norm is not None:
        mr, gamma, beta, ngroups, swish = norm
        _dev(mr, torch.float32); _dev(gamma, torch.float32); _dev(beta, torch.float32)
        p.norm_mean_rstd, p.norm_gamma, p.norm_beta = mr.data_ptr(), gamma.data_ptr(), beta.data_ptr()
        p.norm_groups, p.norm_swish = ngroups, int(swish)      # 0 none, 1 = ex2/rcp fp32 (as vf_groupnorm_apply), 2 = packed bf16 tanh
    _check(lib.vf_tc_gemm(p, _stream()))
    return out


# ----------------------------------------------------------------------------------------------- codebook
def vq_prepare_codebook(emb_dk):
    lib = load(True)
    _dev(emb_dk, torch.float32)
    d, k = emb_dk.shape
    et = torch.empty((k, d), dtype=torch.float32, device=emb_dk.device)
    esq = torch.empty((k,), dtype=torch.float32, device=emb_dk.device)
    _check(lib.vf_vq_prepare_codebook(emb_dk, d, k, et, esq, _stream()))
    return et, esq


def vq_lookup(z_rows, et, esq, want_quant=True, want_diff=True):
    """z_rows f32 [M,D] -> (idx int64 [M], quant f32 [M,D] | None, diff_sum f64[1] | None)."""
    lib = load(True)
    _dev(z_rows, torch.float32)
    m, d = z_rows.shape
    k = et.shape[0]
    idx = torch.empty((m,), dtype=torch.int64, device=z_rows.device)
    quant = torch.empty((m, d), dtype=torch.float32, device=z_rows.device) if want_quant else None
    dsum = torch.zeros((1,), dtype=torch.float64, device=z_rows.device) if want_diff else None
    _check(lib.vf_vq_lookup(z_rows, et, esq, m, d, k, idx, quant, dsum, _stream()))
    return idx, quant, dsum


def split_f16x2(x_rows):
    """f32 [rows, C] -> f16 [rows, 2C] = [hi | lo], hi = fp16(v), lo = fp16((v - hi) * 2^11) (weights of the exact convolution)."""
    lib = load(True)
    _dev(x_rows, torch.float32)
    rows, c = x_rows.shape
    out = torch.empty((rows, 2 * c), dtype=torch.float16, device=x_rows.device)
    _check(lib.vf_split_f16x2(x_rows, rows, c, out, _stream()))
    return out


def vq_prepare_codebook_f16(et):
    """Et f32 [K,D] -> fp16(-2 e) [K,D], the B operand of the fused lookup."""
    lib = load(True)
    _dev(et, torch.float32)
    k, d = et.shape
    eh = torch.empty((k, d), dtype=torch.float16, device=et.device)
    _check(lib.vf_vq_prepare_codebook_f16(et, k, d, eh, _stream()))
    return eh


def vq_fused_ok(d, k):
    return d % 64 == 0 and d <= 256 and k % 256 == 0 and k <= 1024


def vq_lookup_fused(z_rows, et, esq, eh, emb_dk=None, want_quant=True, want_diff=True, tol_factor=1.0, return_counts=False):
    """Fused wgmma lookup (vf_vq_fused.cu): z read once, top-2 from the accumulator registers, exact fp64 settlement of near-ties.  Same outputs as
    vq_lookup; ``return_counts`` adds the int32[2] tensor (rows settled between two candidates, rows settled over all codes).  ``tol_factor``
    scales the fp16 rounding bound that sends a row to the exact pass: 1.0 is the proven worst case, smaller values can misrank rows whose
    roundings align."""
    lib = load(True)
    _dev(z_rows, torch.float32)
    m, d = z_rows.shape
    k = et.shape[0]
    if emb_dk is None:
        emb_dk = et.t().contiguous()                         # callers that hold the reference's [D,K] layout pass it instead
    idx = torch.empty((m,), dtype=torch.int64, device=z_rows.device)
    work = torch.empty((max(m, 1), 4), dtype=torch.int32, device=z_rows.device)
    counter = torch.empty((2,), dtype=torch.int32, device=z_rows.device)
    quant = torch.empty((m, d), dtype=torch.float32, device=z_rows.device) if want_quant else None
    dsum = torch.zeros((1,), dtype=torch.float64, device=z_rows.device) if want_diff else None
    _check(lib.vf_vq_lookup_fused(z_rows, eh, et, emb_dk, esq, m, d, k, tol_factor, idx, work, counter, quant, dsum, _stream()))
    return (idx, quant, dsum, counter) if return_counts else (idx, quant, dsum)


def gather_rows(table, idx):
    lib = load(True)
    _dev(table, torch.float32)
    _dev(idx, torch.int64)
    m = idx.numel()
    d = table.shape[1]
    out = torch.empty((m, d), dtype=torch.float32, device=table.device)
    _check(lib.vf_gather_rows(table, idx, m, d, table.shape[0], out, _stream()))
    return out


def vq_ema_stats(z_rows, idx, k):
    lib = load(True)
    m, d = z_rows.shape
    counts = torch.zeros((k,), dtype=torch.float32, device=z_rows.device)
    esum = torch.zeros((d, k), dtype=torch.float32, device=z_rows.device)
    _check(lib.vf_vq_ema_stats(z_rows, idx, m, d, k, counts, esum, _stream()))
    return counts, esum


def vq_commit_grad(emb_dk, counts, esum, coef, grad_dk, accumulate=False):
    """grad_dk = coef (count_k e_k - esum) (``accumulate``: grad_dk += that)."""
    lib = load(True)
    d, k = emb_dk.shape
    _check(lib.vf_vq_commit_grad(emb_dk, counts, esum, d, k, coef, int(bool(accumulate)), grad_dk, _stream()))
    return grad_dk


def vq_ema_update(counts, esum, alpha, corr, eps, cs_hidden, dw_hidden, emb_dk, et, esq):
    lib = load(True)
    d, k = emb_dk.shape
    _check(lib.vf_vq_ema_update(counts, esum, d, k, alpha, corr, eps, cs_hidden, dw_hidden, emb_dk, et, esq, _stream()))


# ----------------------------------------------------------------------------------------------- transformer glue
def migt_embed(ids_i32, fixed_token, wte, wpe, pose_rows, BT, L):
    lib = load(True)
    d = wte.shape[1]
    out = torch.empty((BT * L, d), dtype=torch.float32, device=wte.device)
    _check(lib.vf_migt_embed(ids_i32, int(fixed_token), wte, wpe, pose_rows, BT, L, d, out, _stream()))
    return out


def attn_block_causal(qk, vt, B, S, H, d, block, first_query=0, out=None, skip_view=-1):
    """Fused wgmma block-causal attention: qk bf16 [B,S,2d] (q|k), vt bf16 [B,d,S] -> bf16 [B*S, d].
    ``first_query`` > 0 computes only the query rows from that row's 128-row tile on (KV-cache decode); ``skip_view`` >= 0 leaves the
    keys of that view out (an unused slot of the cache)."""
    lib = load(True)
    _dev(qk, torch.bfloat16)
    _dev(vt, torch.bfloat16)
    if out is None:
        out = torch.empty((B * S, d), dtype=torch.bfloat16, device=qk.device)
    _check(lib.vf_attn_block_causal_decode(qk, vt, B, S, H, d, block, int(first_query), int(skip_view), out, _stream()))
    return out


def attn_block_multiend(qk, vt, B, S, n_streams, stream, H, d, block, out=None):
    """Fused branching attention of stream ``stream`` (0 = block-causal over stream 0; s >= 1 = stream-0 keys of earlier views + own
    view of stream s): qk bf16 [B, n_streams*S, 2d], vt bf16 [B, d, n_streams*S] -> bf16 [B*S, d]."""
    lib = load(True)
    _dev(qk, torch.bfloat16)
    _dev(vt, torch.bfloat16)
    if out is None:
        out = torch.empty((B * S, d), dtype=torch.bfloat16, device=qk.device)
    _check(lib.vf_attn_block_multiend(qk, vt, B, S, n_streams, stream, H, d, block, out, _stream()))
    return out


def attn_multiend_train(qk, vt, B, S, n_streams, stream, H, d, block, *, rate=0.0, seed=0, lse=None, out_f32=None, out=None):
    """Training forward of stream ``stream`` of the multi-end attention: attn_block_multiend plus the per-row log-sum-exp ``lse`` f32 [B,H,S]
    and an fp32 copy ``out_f32`` [B*S, d] (both optional, written in place) and hash dropout of the probabilities (vf_dropout's mask of the
    stream's [B,H,S,cols] tensor) -> bf16 [B*S, d]."""
    lib = load(True)
    _dev(qk, torch.bfloat16)
    _dev(vt, torch.bfloat16)
    if out is None:
        out = torch.empty((B * S, d), dtype=torch.bfloat16, device=qk.device)
    for t in (lse, out_f32):
        if t is not None:
            _dev(t, torch.float32)
    _check(lib.vf_attn_multiend_train(qk, vt, B, S, n_streams, stream, H, d, block, rate, _seed64(seed), lse, out_f32, out, _stream()))
    return out


def attn_multiend_bwd(qk, vt, dout, out_f32, lse, B, S, n_streams, H, d, block, *, rate=0.0, seed=0, dvqk=None):
    """Fused backward of all streams: dout bf16 [ns, B*S, d], out_f32 [ns, B*S, d], lse [ns, B, H, S] -> dvqk f32 [ns, B*S, 3d] (v | q | k).
    Stream s's dropout seed is seed + s (the sites of the fp32 trainer)."""
    lib = load(True)
    for t, dt in ((qk, torch.bfloat16), (vt, torch.bfloat16), (dout, torch.bfloat16), (out_f32, torch.float32), (lse, torch.float32)):
        _dev(t, dt)
    if dvqk is None:
        dvqk = torch.zeros((n_streams, B * S, 3 * d), dtype=torch.float32, device=qk.device)
    _check(lib.vf_attn_multiend_bwd(qk, vt, dout, out_f32, lse, B, S, n_streams, H, d, block, rate, _seed64(seed), dvqk, _stream()))
    return dvqk


def to_bf16(x, rate=0.0, seed=0, out_f32=False):
    """bf16(dropout(x)) with vf_dropout's mask (rate 0: the plain rounding); ``out_f32=True`` returns (fp32 dropout(x), bf16) from one pass."""
    lib = load(True)
    _dev(x, torch.float32)
    y16 = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    y = torch.empty_like(x) if out_f32 else None
    _check(lib.vf_to_bf16(x, x.numel(), rate, _seed64(seed), y, y16, _stream()))
    return (y, y16) if out_f32 else y16


def _device_table(struct, rows, device):
    """Host struct rows -> the bytes of the device array a one-launch kernel walks, as int64 [n, sizeof(struct) / 8]."""
    words = memoryview(bytearray((struct * len(rows))(*rows))).cast("q").tolist()
    return torch.tensor(words, dtype=torch.int64).reshape(-1, C.sizeof(struct) // 8).to(device)


def dense_weights_bf16_table(entries, device):
    """entries: (w_kn f32 [k, n], fw bf16 [n, k] or None, bw bf16 [k, n] or None) -> the device table of vf_dense_weights_bf16
    (int64 [n, 5] = vf_dense_weights_bf16_t).  The tensors must outlive the table."""
    rows = []
    for w_kn, fw, bw in entries:
        assert w_kn.is_cuda and w_kn.dtype == torch.float32 and w_kn.is_contiguous()
        k, n = w_kn.shape
        assert fw is None or (fw.dtype == torch.bfloat16 and fw.is_contiguous() and tuple(fw.shape) == (n, k))
        assert bw is None or (bw.dtype == torch.bfloat16 and bw.is_contiguous() and tuple(bw.shape) == (k, n))
        rows.append(DenseWeightsBf16(w_kn.data_ptr(), fw.data_ptr() if fw is not None else None, bw.data_ptr() if bw is not None else None, k, n))
    return _device_table(DenseWeightsBf16, rows, device)


def dense_weights_bf16(table):
    """Rewrite every dense layer's bf16 operand copies listed in ``table`` (dense_weights_bf16_table) from its fp32 master weights: one launch."""
    lib = load(True)
    _check(lib.vf_dense_weights_bf16(table, table.shape[0], _stream()))


def softmax_rows(scores, P, *, rows_total, rows_per_batch, cols, ld_in, ld_out, mask_mode=0, block=0, row0=0):
    lib = load(True)
    _check(lib.vf_softmax_rows(scores, rows_total, rows_per_batch, cols, ld_in, mask_mode, block, row0, P, _dt(P), ld_out, _stream()))
    return P


def argmax_rows(x_rows):
    lib = load(True)
    _dev(x_rows, torch.float32)
    rows, cols = x_rows.shape
    out = torch.empty((rows,), dtype=torch.int64, device=x_rows.device)
    _check(lib.vf_argmax_rows(x_rows, rows, cols, cols, out, _stream()))
    return out


def pose_postprocess(raw_rows, mult):
    lib = load(True)
    _dev(raw_rows, torch.float32)
    out = torch.empty_like(raw_rows)
    _check(lib.vf_pose_postprocess(raw_rows, raw_rows.shape[0], mult, out, _stream()))
    return out


def cameras_prepare(cams, relative):
    """cams f32 [B,T,7] (device) -> (relative+normalised cams [B,T,7], transform [B,7]) in one launch."""
    lib = load(True)
    _dev(cams, torch.float32)
    b, t, _ = cams.shape
    out = torch.empty_like(cams)
    tr = torch.empty((b, 7), dtype=torch.float32, device=cams.device)
    _check(lib.vf_cameras_prepare(cams, b, t, int(relative), out, tr, _stream()))
    return out, tr


def cameras_from_relative(cams, transform):
    lib = load(True)
    _dev(cams, torch.float32)
    b, n, _ = cams.shape
    out = torch.empty_like(cams)
    _check(lib.vf_cameras_from_relative(cams, transform, b, n, out, _stream()))
    return out


def cross_entropy_rows(logits_rows, labels_i32, smoothing=0.0):
    lib = load(True)
    _dev(logits_rows, torch.float32)
    _dev(labels_i32, torch.int32)
    rows, cols = logits_rows.shape
    out = torch.empty((rows,), dtype=torch.float32, device=logits_rows.device)
    _check(lib.vf_cross_entropy_rows(logits_rows, labels_i32, rows, cols, smoothing, out, _stream()))
    return out


def pose_loss_rows(raw_rows, poses_bt7, tokens_per_view, mult):
    lib = load(True)
    rows = raw_rows.shape[0]
    pos = torch.empty((rows,), dtype=torch.float32, device=raw_rows.device)
    ori = torch.empty((rows,), dtype=torch.float32, device=raw_rows.device)
    _check(lib.vf_pose_loss_rows(raw_rows, poses_bt7, rows, tokens_per_view, mult, pos, ori, _stream()))
    return pos, ori


def row_mean(x_rows, start=0):
    """x [rows, n] -> [rows] mean over columns start..n-1."""
    lib = load(True)
    _dev(x_rows, torch.float32)
    rows, n = x_rows.shape
    out = torch.empty((rows,), dtype=torch.float32, device=x_rows.device)
    _check(lib.vf_row_mean(x_rows, rows, n, start, out, _stream()))
    return out


# ----------------------------------------------------------------------------------------------- backward pass (training step)
def simt_conv_dgrad_s2(dy, w_dgrad_kn, in_hw):
    """Data gradient of the stride-2 Downsample conv: dy f32 [N,OH,OW,Cout], w_dgrad_kn [9*Cout, Cin] (tap-major, NOT flipped)
    -> dx f32 [N,H,W,Cin]."""
    lib = load(True)
    _dev(dy, torch.float32)
    n, oh, ow, cout = dy.shape
    h, w = in_hw
    cin = w_dgrad_kn.shape[1]
    out = torch.empty((n, h, w, cin), dtype=torch.float32, device=dy.device)
    p = SimtGemm(A=dy.data_ptr(), a_dtype=F32, conv=2, N=n, H=oh, W=ow, Cin=cout, OH=h, OW=w, KH=3, KW=3, stride=1,
                 B=w_dgrad_kn.data_ptr(), b_dtype=F32, b_sk=cin, b_sn=1, M=n * h * w, Ncols=cin, K=9 * cout, batch1=1, batch2=1)
    _epilogue(p, out, cin)
    _check(lib.vf_simt_gemm(p, _stream()))
    return out


def conv_wgrad(x, dy, dw, *, kh, stride=1, pad=(1, 1), upsample=False, so=None):
    """dw (zeroed by the caller, accumulated here) [kh*kh*Cin, Cout] (or any layout via ``so`` = (stride of k, stride of co))."""
    lib = load(True)
    _dev(x, torch.float32); _dev(dy, torch.float32); _dev(dw, torch.float32)
    n, h, w, cin = x.shape
    _, oh, ow, cout = dy.shape
    so_k, so_n = (cout, 1) if so is None else so
    _check(lib.vf_conv_wgrad(x, dy, n, h, w, cin, oh, ow, cout, kh, kh, stride, pad[0], pad[1], int(upsample), so_k, so_n, dw, _stream()))
    return dw


_wgrad_bufs = {}


def conv_wgrad_tc_ok(x, dy, kh, stride, upsample):
    n, h, w, cin = x.shape
    return kh == 3 and stride == 1 and not upsample and cin % 128 == 0 and dy.shape[-1] % 128 == 0 and dy.shape[1:3] == x.shape[1:3]


def conv_wgrad_bf16_ok(x, dy, kh, stride, upsample):
    """Shapes conv_wgrad_bf16 takes: those of conv_wgrad_tc_ok, and the upsample convs (x [N,H,W,Cin], dy [N,2H,2W,Cout])."""
    n, h, w, cin = x.shape
    up = 2 if upsample else 1
    return kh == 3 and stride == 1 and cin % 128 == 0 and dy.shape[-1] % 128 == 0 and tuple(dy.shape[1:3]) == (up * h, up * w)


def conv_wgrad_tc(x, dy, dw, *, accumulate=True):
    """Weight gradient of a 3x3 stride-1 pad-1 convolution on the exact split-fp16 tensor-core GEMM.  x [N,H,W,Cin], dy [N,H,W,Cout] fp32;
    dw [9*Cin, Cout] (k = (ky*3 + kx)*Cin + c).  dW[ky,kx][c, co] = sum_q xpad[c, q + (ky-1) pitch + (kx-1)] * dypad[co, q] over the
    zero-padded pixel grid: both operands are transposed to K-major split form, the horizontal shifts are three row blocks of the activation
    operand (M = 3 Cin), the vertical ones are K offsets of whole (8-aligned) rows, the pixel axis is split over the SMs and the partial
    products are folded by vf_sum_splits."""
    return _wgrad_tc(x, dy, dw, bf16=False, conv=True, accumulate=accumulate)


def conv_wgrad_bf16(x, dy, dw, *, norm=None, upsample=False, accumulate=True):
    """conv_wgrad_tc on the single-pass bf16 tensor-core GEMM (bf16 operands, fp32 accumulation).  x f32 [N,H,W,Cin] is the conv's input
    before ``norm`` (see pad_transpose_bf16) and before the nearest x2 upsample when ``upsample``; dy f32 [N,OH,OW,Cout]; dw f32 [9*Cin, Cout]."""
    return _wgrad_tc(x, dy, dw, bf16=True, conv=True, norm=norm, upsample=upsample, accumulate=accumulate)


def dense_wgrad_tc(x_rows, dy_rows, dw_kn, *, accumulate=True):
    """dW[k, n] (+)= sum_m x[m, k] dy[m, n] on the exact split-fp16 tensor-core GEMM (K = rows): both operands are transposed to K-major
    split form, the row axis is split over the SMs, vf_sum_splits folds the partial products."""
    return _wgrad_tc(x_rows, dy_rows, dw_kn, bf16=False, conv=False, accumulate=accumulate)


def dense_wgrad_bf16(x_rows, dy_rows, dw_kn, *, accumulate=True):
    """dense_wgrad_tc on the single-pass bf16 tensor-core GEMM: both fp32 operands rounded once to bf16 by the K-major transposer."""
    return _wgrad_tc(x_rows, dy_rows, dw_kn, bf16=True, conv=False, accumulate=accumulate)


def _wgrad_tc(x, dy, dw, *, bf16, conv, norm=None, upsample=False, accumulate=True):
    """The split-K weight-gradient GEMM behind conv_wgrad_tc / conv_wgrad_bf16 (``conv``) and dense_wgrad_tc / dense_wgrad_bf16: one plan,
    the same launches for both operand formats (``bf16``: single-pass bf16, else exact split-fp16)."""
    lib = load(True)
    _dev(x, torch.float32); _dev(dy, torch.float32); _dev(dw, torch.float32)
    cin, cout = x.shape[-1], dy.shape[-1]
    key = (bf16, conv, x.device, tuple(dy.shape[:-1]), cin, cout)
    if conv:                                                   # K = pixels of the zero-padded logical (upsampled) image
        n, h, w = dy.shape[:3]
        pitch = (w + 2 + 7) // 8 * 8
        klen, blocks, max_splits, margin = n * (h + 2) * pitch, 3, 64, pitch + 8        # margin: a multiple of 8, >= pitch + 1
    else:                                                      # K = rows: one plain row of pixels
        x, dy = x.reshape(1, 1, -1, cin), dy.reshape(1, 1, -1, cout)
        pitch, klen, blocks, max_splits, margin = 0, x.shape[2], 1, 32, 0
    M = blocks * cin
    tiles = (M // 128) * (cout // 128)
    splits = max(1, min(max_splits, (132 + blocks * tiles - 1) // (blocks * tiles)))
    kc = ((klen + splits - 1) // splits + 63) // 64 * 64       # the tensor-core GEMM walks K in blocks of 64
    kpad = kc * splits
    la, lb = kpad + 2 * margin, kpad
    # operand buffers are cached per shape: the transposer rewrites every interior position on each call and never touches the zero
    # borders / pitch padding / margins / columns past K, so they are cleared once
    bufs = _wgrad_bufs.get(key)
    if bufs is None:
        if len(_wgrad_bufs) >= 32:
            _wgrad_bufs.clear()
        dt = torch.bfloat16 if bf16 else torch.float16

        def operand(rows, length):                             # a split-fp16 row holds its hi and lo halves
            return torch.zeros((rows, length) if bf16 else (rows, 2, length), dtype=dt, device=x.device)

        bufs = (operand(M, la), operand(cout, lb), torch.empty(((blocks,) if conv else ()) + (splits, M, cout), dtype=torch.float32, device=x.device))
        _wgrad_bufs[key] = bufs
    at, bt, partial = bufs
    transpose = pad_transpose_bf16 if bf16 else pad_transpose_split
    transpose(x, at, pitch=pitch, copies=blocks, margin=margin, norm=norm, upsample=upsample)
    transpose(dy, bt, pitch=pitch, copies=1, margin=0)
    ld = 1 if bf16 else 2
    tc_gemm(at, bt, partial, M=M, N=cout, K=kc, lda=ld * la, ldb=ld * lb, ldc=cout, batch=(blocks, splits), a_bs=(0, kc), b_bs=(0, kc),
            c_bs=(splits * M * cout if conv else 0, M * cout), lo_a=la, lo_b=lb, k_offsets=[margin - pitch, margin, margin + pitch] if conv else None)
    _check(lib.vf_sum_splits(partial, blocks, splits, M * cout, int(accumulate), dw, _stream()))
    return dw


def pad_transpose_split(x, out, *, pitch, copies, margin, norm=None, upsample=False):
    """x f32 NHWC -> out split-fp16 [copies*C, 2, L] (zeroed by the caller): the K-major operand of the exact weight-gradient GEMM, the column
    map of pad_transpose_bf16 with a lo half after the hi one.  The split transposer applies neither GroupNorm nor the x2 upsample."""
    if norm is not None or upsample:
        raise ValueError("pad_transpose_split: no GroupNorm or x2 upsample on the split-fp16 operand")
    lib = load(True)
    _dev(x, torch.float32); _dev(out, torch.float16)
    n, h, w, c = x.shape
    _check(lib.vf_pad_transpose_split(x, n, h, w, c, pitch, copies, margin, out.shape[-1], out, _stream()))
    return out


def pad_transpose_bf16(x, out, *, pitch, copies, margin, norm=None, upsample=False):
    """x f32 NHWC -> out bf16 [copies*C, L] (zeroed by the caller): the K-major operand of the bf16 weight-gradient GEMM over the zero-padded
    pixel grid of the logical image (x, or its nearest x2 upsample), column margin + ((n (H+2) + y + 1) pitch + x + 1) - (k - copies/2) of copy k.
    ``norm=(mean_rstd, gamma, beta, swish)`` applies GroupNorm(32) [+ swish] first, as vf_groupnorm_apply does for a bf16 output."""
    lib = load(True)
    _dev(x, torch.float32); _dev(out, torch.bfloat16)
    n, h, w, c = x.shape
    mr, gamma, beta, swish = norm if norm is not None else (None, None, None, False)
    groups = mr.shape[1] if mr is not None else 0
    _check(lib.vf_pad_transpose_bf16(x, n, h, w, c, int(upsample), pitch, copies, margin, out.shape[-1], mr, gamma,
                                     beta, groups, int(swish), out, _stream()))
    return out


def conv_weights_bf16_table(entries, device):
    """entries: (w_kn f32 [9*Cin, Cout], fw bf16 [Cout, 9*Cin], bw bf16 [Cin, 9*Cout] or None) -> the device table of vf_conv_weights_bf16
    (int64 [n, 5] = vf_conv_weights_bf16_t).  The tensors must outlive the table."""
    rows = []
    for w_kn, fw, bw in entries:
        _dev(w_kn, torch.float32); _dev(fw, torch.bfloat16)
        k, cout = w_kn.shape
        assert k % 9 == 0 and fw.shape == (cout, k) and (bw is None or (bw.dtype == torch.bfloat16 and bw.shape == (k // 9, 9 * cout)))
        rows.append(ConvWeightsBf16(w_kn.data_ptr(), fw.data_ptr(), bw.data_ptr() if bw is not None else None, k // 9, cout))
    return _device_table(ConvWeightsBf16, rows, device)


def conv_weights_bf16(table):
    """Rewrite every conv's bf16 operand copies listed in ``table`` (conv_weights_bf16_table) from its fp32 master weights: one launch."""
    lib = load(True)
    _check(lib.vf_conv_weights_bf16(table, table.shape[0], _stream()))


def col_sums(x_rows, out):
    lib = load(True)
    _dev(x_rows, torch.float32)
    _check(lib.vf_col_sums(x_rows, x_rows.numel() // x_rows.shape[-1], x_rows.shape[-1], out, _stream()))
    return out


def groupnorm_bwd(x, dout, mean_rstd, gamma, beta, dgamma, dbeta, *, swish, groups=32, add=None, out_bf16=False):
    """dx f32; ``out_bf16`` also writes dx rounded to bf16 from the same pass and attaches it as ``dx._bf16``."""
    lib = load(True)
    _dev(x, torch.float32); _dev(dout, torch.float32)
    n, h, w, c = x.shape
    dx = torch.empty_like(x)
    dx16 = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device) if out_bf16 else None
    gs = torch.empty((n, groups, 2), dtype=torch.float64, device=x.device)
    _check(lib.vf_groupnorm_bwd(x, dout, mean_rstd, gamma, beta, n, h * w, c, groups, int(swish), add, gs, dgamma, dbeta, dx, dx16, _stream()))
    if dx16 is not None:
        dx._bf16 = dx16
    return dx


def softmax_bwd_rows(P, dP):
    lib = load(True)
    dS = torch.empty_like(P)
    _check(lib.vf_softmax_bwd_rows(P, dP, P.numel() // P.shape[-1], P.shape[-1], dS, _stream()))
    return dS


def l1_grad(x, y, scale):
    """(dy = scale * sign(y - x), loss_sum f64[1] = sum |y - x|)"""
    lib = load(True)
    dy = torch.empty_like(y)
    ls = torch.zeros((1,), dtype=torch.float64, device=y.device)
    _check(lib.vf_l1_grad(x, y, y.numel(), scale, dy, ls, _stream()))
    return dy, ls


def lincomb3(a, x, b=0.0, y=None, c=0.0, z=None, out=None):
    lib = load(True)
    if out is None:
        out = torch.empty_like(x)
    _check(lib.vf_lincomb3(a, x, b, y, c, z, x.numel(), out, _stream()))
    return out


def sumpool2x2(x):
    lib = load(True)
    n, h2, w2, c = x.shape
    y = torch.empty((n, h2 // 2, w2 // 2, c), dtype=torch.float32, device=x.device)
    _check(lib.vf_sumpool2x2(x, n, h2 // 2, w2 // 2, c, y, _stream()))
    return y


def adam(p, g, m, v, *, lr, beta1, beta2, eps, step, grad_scale=1.0):
    lib = load(True)
    _check(lib.vf_adam(p, g, m, v, p.numel(), lr, beta1, beta2, eps, int(step), grad_scale, _stream()))


def layernorm_bwd(x, dy, gamma, dgamma, dbeta, eps=1e-5, add=None):
    lib = load(True)
    d = x.shape[-1]
    dx = torch.empty_like(x)
    _check(lib.vf_layernorm_bwd(x, dy, gamma, add, x.numel() // d, d, eps, dgamma, dbeta, dx, _stream()))
    return dx


def gelu(x):
    lib = load(True)
    y = torch.empty_like(x)
    _check(lib.vf_gelu_fwd(x, x.numel(), y, _stream()))
    return y


def gelu_bwd(pre, dy):
    lib = load(True)
    out = torch.empty_like(pre)
    _check(lib.vf_gelu_bwd(pre, dy, pre.numel(), out, _stream()))
    return out


def migt_embed_bwd(dh, ids_i32, fixed_token, BT, L, dwte, dwpe, dpose):
    lib = load(True)
    _check(lib.vf_migt_embed_bwd(dh, ids_i32, int(fixed_token), BT, L, dh.shape[-1], dwte, dwpe, dpose, _stream()))


def cross_entropy_grad(logits_rows, labels_i32, row_weight, smoothing=0.0):
    lib = load(True)
    rows, cols = logits_rows.shape
    out = torch.empty_like(logits_rows)
    _check(lib.vf_cross_entropy_grad(logits_rows, labels_i32, row_weight, rows, cols, smoothing, out, _stream()))
    return out


def pose_loss_grad(raw_rows, poses_bt7, row_weight, tokens_per_view, mult, pos_scale=1.0, ori_scale=1.0):
    lib = load(True)
    out = torch.empty_like(raw_rows)
    _check(lib.vf_pose_loss_grad(raw_rows, poses_bt7, row_weight, raw_rows.shape[0], tokens_per_view, mult, pos_scale, ori_scale, out, _stream()))
    return out


def adamw_keras(p, g, m, v, *, lr, beta1, beta2, eps, weight_decay, step, grad_scale=1.0, clip_scale=1.0):
    lib = load(True)
    _check(lib.vf_adamw_keras(p, g, m, v, p.numel(), lr, beta1, beta2, eps, weight_decay, int(step), grad_scale, clip_scale, _stream()))


def sumsq(x):
    lib = load(True)
    out = torch.zeros((1,), dtype=torch.float64, device=x.device)
    _check(lib.vf_sumsq(x, x.numel(), out, _stream()))
    return out


def dropout(x, rate, seed):
    lib = load(True)
    y = torch.empty_like(x)
    _check(lib.vf_dropout(x, x.numel(), rate, _seed64(seed), y, _stream()))
    return y
