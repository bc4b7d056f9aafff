"""ctypes binding of the in-tree CUDA library `libb200sht.so` (C ABI: include/b200sht.h).

The product path has no CPU or PyTorch fallback: if the library cannot be loaded, or a call fails, a
`B200ShtError` is raised.  The library is built in-tree by `makani_b200/build.py` (nvcc, sm_90a).
"""
import ctypes
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200SHT_LIBRARY: another build of the same library (e.g. the wait-profile build of scripts/dft_waitprof.py); default: the in-tree one
LIB_PATH = os.environ.get("B200SHT_LIBRARY") or os.path.join(_HERE, "libb200sht.so")
HEADER_PATH = os.path.join(_HERE, "..", "include", "b200sht.h")

F32, BF16 = 0, 1
PREC_FP32, PREC_TF32, PREC_FP32X3 = 0, 1, 2
PLAN_FFT_ONLY, PLAN_VECTOR = 1, 2
OP_DHCONV, OP_DIAGONAL, OP_SEP_DHCONV, OP_SEP_DIAGONAL, OP_SHARED, OP_LDEP = range(6)
DENSE_FLAG = 0x100


class B200ShtError(RuntimeError):
    pass


_lib = None

c_int, c_void_p, c_int64, c_float = ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_float
_P = c_void_p

# name -> (restype, argtypes)
_SIGNATURES = {
    "b200sht_last_error": (ctypes.c_char_p, []),
    "b200sht_version": (c_int, []),
    "b200sht_plan_create": (c_int, [ctypes.POINTER(_P), c_int, c_int, c_int, c_int, _P, _P, c_int, _P]),
    "b200sht_plan_create_ex": (c_int, [ctypes.POINTER(_P), c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, c_int, _P]),
    "b200sht_plan_destroy": (c_int, [_P]),
    "b200sht_plan_query": (c_int64, [_P, c_int]),
    "b200sht_plan_table": (_P, [_P]),
    "b200sht_plan_copy_table": (c_int, [_P, _P, _P]),
    "b200sht_latspec_elems": (c_int64, [_P, c_int, c_int]),
    "b200sht_spec_elems": (c_int64, [_P, c_int, c_int]),
    "b200sht_spec_elems_lm": (c_int64, [c_int, c_int, c_int, c_int]),
    "b200sht_fft_analysis": (c_int, [_P, _P, c_int, c_int, c_int, _P, c_int, _P]),
    "b200sht_fft_synthesis": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P, c_int, _P]),
    "b200sht_legendre_analysis": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "b200sht_legendre_synthesis": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "b200sht_legendre_synthesis_tiled": (c_int, [_P, _P, _P, c_int, c_int, _P]),
    "b200sht_spec_unpack": (c_int, [c_int, c_int, _P, _P, c_int, c_int, _P]),
    "b200sht_spec_pack": (c_int, [c_int, c_int, _P, _P, c_int, c_int, _P]),
    "b200sht_spec_unpack_ex": (c_int, [c_int, c_int, c_int, c_int, _P, _P, c_int, c_int, _P]),
    "b200sht_spec_pack_ex": (c_int, [c_int, c_int, c_int, c_int, _P, _P, c_int, c_int, _P]),
    "b200sht_latspec_unpack": (c_int, [_P, _P, _P, c_int, c_int, _P]),
    "b200sht_latspec_pack": (c_int, [_P, _P, _P, c_int, c_int, _P]),
    "b200sht_sht_workspace_bytes": (c_int64, [_P, c_int, c_int]),
    "b200sht_sht_forward": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P, c_int, _P]),
    "b200sht_sht_inverse": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P, c_int, _P]),
    "b200sht_sht_forward_adjoint": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P, c_int, _P]),
    "b200sht_sht_inverse_adjoint": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P, c_int, _P]),
    "b200sht_mix_weight_elems": (c_int64, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "b200sht_mix_weight_pack": (c_int, [c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200sht_mix_weight_unpack": (c_int, [c_int, _P, _P, c_int, c_int, c_int, c_int, _P]),
    "b200sht_mix_uses_tensor_cores": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "b200sht_mix_forward": (c_int, [c_int, c_int, c_int, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200sht_mix_backward": (c_int, [c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200sht_complex_relu_forward": (c_int, [c_int, c_int, c_int, _P, _P, c_float, _P, c_int, c_int, _P]),
    "b200sht_complex_relu_backward": (c_int, [c_int, c_int, c_int, _P, _P, c_float, _P, _P, _P, c_int, c_int, _P]),
    # vector SHT
    "b200sht_vector_legendre_analysis": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "b200sht_vector_legendre_synthesis": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "b200sht_vector_legendre_synthesis_tiled": (c_int, [_P, _P, _P, c_int, c_int, _P]),
    "b200sht_vector_spec_unpack": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "b200sht_vector_spec_pack": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "b200sht_vsht_workspace_bytes": (c_int64, [_P, c_int, c_int]),
    "b200sht_vsht_forward": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P, c_int, _P]),
    "b200sht_vsht_inverse": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P, c_int, _P]),
    "b200sht_vsht_forward_adjoint": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P, c_int, _P]),
    "b200sht_vsht_inverse_adjoint": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P, c_int, _P]),
    "b200sht_spectral_conv_workspace_bytes": (c_int64, [_P, _P, _P]),
    "b200sht_spectral_conv_forward": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "b200sht_spectral_conv_backward": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "b200sht_spectral_conv_backward_ex": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "b200sht_bias_grad": (c_int, [_P, _P, _P, c_int, c_int, _P]),
    "b200sht_spectral_conv_forward_host": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P]),
    # pointwise tail of the SFNO block (row N2)
    "b200sht_pointwise_workspace_floats": (c_int64, [c_int, c_int, c_int64]),
    "b200sht_instance_norm_forward": (c_int, [_P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int64, c_float, c_int, _P]),
    "b200sht_instance_norm_backward": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int64, c_int, _P]),
    "b200sht_bias_gelu_forward": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int64, _P]),
    "b200sht_bias_gelu_backward": (c_int, [_P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int64, _P]),
    # quadrature-weighted instance norm on the sphere
    "b200sht_geometric_norm_workspace_floats": (c_int64, [c_int, c_int, c_int64]),
    "b200sht_geometric_norm_partials": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200sht_geometric_norm_finalize": (c_int, [_P, c_int, c_int, ctypes.c_double, c_float, _P, _P]),
    "b200sht_geometric_norm_apply": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200sht_geometric_norm_backward_sums": (c_int, [_P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200sht_geometric_norm_backward_apply": (c_int, [_P, _P, _P, _P, _P, _P, _P, c_int, _P, ctypes.c_double, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "b200sht_geometric_norm_param_grads": (c_int, [_P, _P, _P, c_int, c_int, _P]),
    # channel layer norm
    "b200sht_layer_norm_workspace_floats": (c_int64, [c_int, c_int, c_int64]),
    "b200sht_layer_norm_forward": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int64, c_float, c_int, _P]),
    "b200sht_layer_norm_backward": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int64, c_int, _P]),
    # DISCO convolution (row N1)
    "b200sht_disco_plan_create": (c_int, [ctypes.POINTER(_P), c_int, c_int, c_int, c_int, c_int, c_int64, _P, _P, _P, _P, _P]),
    "b200sht_disco_plan_destroy": (c_int, [_P]),
    "b200sht_disco_plan_query": (c_int64, [_P, c_int]),
    "b200sht_disco_forward": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P]),
    "b200sht_disco_adjoint": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    # neighbourhood attention on the sphere (on a K = 1 DISCO plan)
    "b200sht_attention_forward": (c_int, [_P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_float, _P]),
    "b200sht_attention_backward": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_float, _P]),
    # global attention on the sphere
    "b200sht_attention_global_workspace_floats": (c_int64, [c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    "b200sht_attention_global_forward": (c_int, [_P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float, c_int, _P, _P]),
    "b200sht_attention_global_backward": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float, c_int, _P,
                                                  _P]),
    "b200sht_attention_global_rowdot": (c_int, [_P, _P, _P, c_int64, c_int, _P]),
    "b200sht_attention_global_backward_kv": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float, c_int, _P,
                                                     _P]),
    "b200sht_attention_global_backward_q": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float, c_int, _P, _P]),
    # bilinear resampling on the sphere
    "b200sht_resample_plan_create": (c_int, [ctypes.POINTER(_P), c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P]),
    "b200sht_resample_plan_destroy": (c_int, [_P]),
    "b200sht_resample_plan_query": (c_int64, [_P, c_int]),
    "b200sht_resample_forward": (c_int, [_P, _P, _P, c_int, _P]),
    "b200sht_resample_adjoint": (c_int, [_P, _P, _P, c_int, _P]),
    # debug / CPU-testable entry points (same device code compiled for the host)
    "b200sht_debug_fft_host": (c_int, [c_int, c_int, c_int, _P, _P, _P, _P]),
    "b200sht_debug_dft_host": (c_int, [c_int, c_int, c_int, c_int, c_float, _P, _P]),
    "b200sht_debug_dft_profile": (c_int, [_P]),
    "b200sht_debug_umma_profile": (c_int, [_P]),
    "b200sht_debug_set_pdl": (c_int, [c_int]),
    "b200sht_debug_fft_plan": (c_int, [c_int, _P, c_int]),
    "b200sht_debug_table_host": (c_int, [c_int, c_int, c_int, _P, c_int, _P]),
    "b200sht_debug_vector_table_host": (c_int, [c_int, c_int, c_int, _P, c_int, _P, _P]),
}


class ConvDesc(ctypes.Structure):
    _fields_ = [("B", c_int), ("Cin", c_int), ("Cout", c_int), ("G", c_int), ("op", c_int), ("dtype", c_int), ("precision", c_int)]


def declared_symbols():
    """Every function name declared in include/b200sht.h (used by the symbol-export test)."""
    with open(HEADER_PATH) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200sht_[a-z0-9_]+)\s*\(", text)))


def load():
    """Load the CUDA library; raises B200ShtError when it is missing (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200ShtError(
            f"{LIB_PATH} not found: build it with `python -m makani_b200.build` (nvcc, sm_90a). "
            "makani_b200 has no CPU / PyTorch fallback for the spherical-harmonic path."
        )
    try:
        lib = ctypes.CDLL(LIB_PATH)
    except OSError as e:  # pragma: no cover
        raise B200ShtError(f"cannot load {LIB_PATH}: {e}") from e
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().b200sht_last_error().decode("utf-8", "replace")
        raise B200ShtError(f"{what} failed (status {rc}): {msg}")


def ptr(t):
    """the `void*` argument of a tensor (None -> NULL)"""
    return c_void_p(t.data_ptr()) if t is not None else c_void_p(0)


def dtype_code(dtype):
    """the activation dtype code of the C ABI (B200SHT_F32 / B200SHT_BF16)"""
    if dtype == torch.float32:
        return F32
    if dtype == torch.bfloat16:
        return BF16
    raise B200ShtError(f"unsupported activation dtype {dtype} (float32 and bfloat16 are supported)")


class LaunchStream(c_void_p):
    """A `void* stream` argument that also names the CUDA device the stream belongs to (`.device`, an index)."""


def launch_stream(device):
    """The stream argument of a library call: torch's current stream of `device`, carrying the device index for `call`."""
    dev = torch.device(device)
    stream = LaunchStream(torch.cuda.current_stream(dev).cuda_stream)
    stream.device = dev.index if dev.index is not None else torch.cuda.current_device()
    return stream


def call(name, *args):
    """Run entry point `name`; a non-zero status raises B200ShtError.  Every entry point that takes a stream takes it last: when that is a
    `launch_stream` handle whose device is not the current one, the device is made current around the call, because the library keeps its
    per-device state (scratch buffers, SM count, tensor-core setup) by the current device.  A plain c_void_p stream is passed as it is."""
    lib = load()
    stream = args[-1] if args else None
    if isinstance(stream, LaunchStream) and stream.device != torch.cuda.current_device():
        with torch.cuda.device(stream.device):
            rc = getattr(lib, name)(*args)
    else:
        rc = getattr(lib, name)(*args)
    check(rc, name)
