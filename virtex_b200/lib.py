"""ctypes binding of libvirtex_b200.so (the C ABI declared in include/virtex_b200.h).

The library is the product's only compute path: there is no CPU or eager-PyTorch fallback.  Importing this module
without the built library, or calling any op without a CUDA device, raises.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvirtex_b200.so")

c_int = ctypes.c_int
c_i32 = ctypes.c_int32
c_i64 = ctypes.c_int64
c_f32 = ctypes.c_float
c_void_p = ctypes.c_void_p


class VtxError(RuntimeError):
    pass


class VtxGemm(ctypes.Structure):
    _fields_ = [
        ("A", c_void_p), ("B", c_void_p), ("D", c_void_p),
        ("bias", c_void_p), ("residual", c_void_p), ("stats", c_void_p),
        ("lda", c_i64), ("ldb", c_i64), ("ldd", c_i64), ("ldr", c_i64),
        ("M", c_i32), ("N", c_i32), ("K", c_i32),
        ("a_mn", c_i32), ("b_mn", c_i32),
        ("out_f32", c_i32), ("atomic", c_i32), ("act", c_i32), ("split_k", c_i32), ("tile_n", c_i32),
        ("alpha", c_f32),
        ("conv_n", c_i32), ("conv_h", c_i32), ("conv_w", c_i32), ("conv_c", c_i32), ("conv_mode", c_i32),
        ("conv_stride", c_i32), ("conv_taps", c_i32),
        ("conv_taps_h", c_i32), ("conv_taps_w", c_i32), ("conv_pad", c_i32),
        ("conv_out_h", c_i32), ("conv_out_w", c_i32),
        ("ldd_w", c_i64), ("ldd_h", c_i64), ("ldd_n", c_i64),
        ("residual_mask", c_void_p),
        ("bnr_y", c_void_p), ("bnr_bnp", c_void_p), ("bnr_sums", c_void_p), ("bnr_mask", c_void_p), ("bnr_ldy", c_i64),
        ("col_scale", c_void_p), ("col_shift", c_void_p),
    ]


_lib = None


def load():
    """Load (once) and return the shared library; raises VtxError if it has not been built."""
    global _lib
    if _lib is None:
        path = LIB_PATH
        if not os.path.exists(path):
            raise VtxError(
                f"{path} is missing: run `python -m virtex_b200.build` (there is no fallback path)")
        lib = ctypes.CDLL(path)
        lib.vtx_last_error.restype = ctypes.c_char_p
        if lib.vtx_sizeof_gemm() != ctypes.sizeof(VtxGemm):
            raise VtxError(f"{path} was built from another include/virtex_b200.h (VtxGemm is {lib.vtx_sizeof_gemm()} bytes "
                           f"there, {ctypes.sizeof(VtxGemm)} here): run `python -m virtex_b200.build`")
        _lib = lib
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = load().vtx_last_error().decode("utf-8", "replace")
        raise VtxError(f"{what} failed ({rc}): {msg}")


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else t.data_ptr()
