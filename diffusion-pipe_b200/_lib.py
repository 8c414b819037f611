"""ctypes binding of libdpipe_b200.so (C ABI declared in include/dpipe.h).

There is deliberately no fallback: if the shared library is missing or a call fails, the error is
raised.  The product path never routes through oracle/ or a PyTorch re-implementation.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libdpipe_b200.so')

c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_int64 = ctypes.c_int64
c_float = ctypes.c_float

# epilogue enums (include/dpipe.h)
EPI_STORE = 0
EPI_BIAS_GELU = 1
EPI_GATE_RES = 2
EPI_QKV_ROPE = 3
EPI_MUL_GELU_GRAD = 4


class QkvEpilogue(ctypes.Structure):
    _fields_ = [
        ('q', c_void_p), ('k', c_void_p), ('v', c_void_p),
        ('qhat', c_void_p), ('khat', c_void_p),
        ('q_rstd', c_void_p), ('k_rstd', c_void_p),
        ('q_norm_w', c_void_p), ('k_norm_w', c_void_p),
        ('rope_cos', c_void_p), ('rope_sin', c_void_p),
        ('heads', c_int), ('seq_total', c_int), ('seq_offset', c_int), ('n_qkv', c_int),
        ('eps', c_float),
    ]


class GemmArgs(ctypes.Structure):
    _fields_ = [
        ('A', c_void_p), ('lda', c_int64), ('a_mn', c_int),
        ('B', c_void_p), ('ldb', c_int64), ('b_mn', c_int),
        ('M', c_int), ('N', c_int), ('K', c_int),
        ('epilogue', c_int),
        ('out', c_void_p), ('ldo', c_int64),
        ('out2', c_void_p), ('ldo2', c_int64),
        ('bias', c_void_p),
        ('aux', c_void_p), ('ldaux', c_int64),
        ('gate', c_void_p), ('gate_stride', c_int64),
        ('rows_per_batch', c_int),
        ('accumulate', c_int),
        ('cta_group', c_int),
        ('qkv', ctypes.POINTER(QkvEpilogue)),
    ]


class DpipeError(RuntimeError):
    pass


_lib = None


def lib():
    """Loads libdpipe_b200.so once.  Raises (never falls back) when it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise DpipeError(
                f'{LIB_PATH} is missing: build it with `python tools/build_native.py` '
                '(or __graft_entry__.build()).  There is no CPU/PyTorch fallback for the sm_90a kernels.')
        l = ctypes.CDLL(LIB_PATH)
        l.dpipe_last_error.restype = ctypes.c_char_p
        l.dpipe_abi_version.restype = c_int
        l.dpipe_check_device.argtypes = [c_int]
        l.dpipe_gemm_bf16.argtypes = [ctypes.POINTER(GemmArgs), c_void_p]
        _declare_optional(l)
        _lib = l
    return _lib


def _declare_optional(l):
    """argtypes for entry points added after ABI v1 (declared when present so that an old .so fails at
    call time with a clear AttributeError rather than a segfault)."""
    from . import _abi  # noqa: F401  (populates signatures)
    _abi.declare(l)


def check(rc, what):
    if rc != 0:
        msg = lib().dpipe_last_error().decode('utf-8', 'replace')
        raise DpipeError(f'{what} failed (rc={rc}): {msg}')


def exported_symbols():
    """Names declared in include/dpipe.h (parsed), used by the CPU-side ABI test."""
    import re
    hdr = os.path.join(os.path.dirname(_HERE), 'include', 'dpipe.h')
    with open(hdr) as f:
        text = f.read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    return sorted(set(re.findall(r'\b(dpipe_[a-z0-9_]+)\s*\(', text)))
