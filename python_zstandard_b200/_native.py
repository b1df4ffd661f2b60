"""ctypes binding of libzb200.so (the C ABI in include/zb200.h).

There is no CPU fallback: if the CUDA library is missing or no device is
present, the product path raises -- it never routes through oracle/.
"""
import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get("ZB200_LIB") or os.path.join(_HERE, "libzb200.so")     # ZB200_LIB: a tuning build (phase timers)

K_COUNT = 16
SRC_DEVICE = 1
DST_DEVICE = 2
SEGS_HOST = 8


class Segment(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("length", C.c_uint64)]


class FrameInfo(C.Structure):
    _fields_ = [("content_size", C.c_uint64), ("window_size", C.c_uint64), ("dict_id", C.c_uint32),
                ("header_size", C.c_uint32), ("has_checksum", C.c_uint32), ("status", C.c_uint32)]


class DParams(C.Structure):
    """zb200_dparams (include/zb200.h): what ZstdDecompressor(max_window_size=...) configures."""
    _fields_ = [("max_window_size", C.c_uint64), ("reserved", C.c_uint32 * 2)]


class TrainParams(C.Structure):
    """zb200_train_params (include/zb200.h)."""
    _fields_ = [("k", C.c_uint32), ("d", C.c_uint32), ("f", C.c_uint32), ("steps", C.c_uint32), ("accel", C.c_uint32),
                ("level", C.c_int32), ("dict_id", C.c_uint32), ("reserved", C.c_uint32), ("split_point", C.c_double)]


class NativeError(RuntimeError):
    pass


_lib = None
_lock = threading.Lock()


def lib():
    """Load libzb200.so (building it first if the sources are newer and nvcc is present)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(_LIB_PATH):
            raise NativeError(
                "libzb200.so is not built (run `python -c 'import __graft_entry__ as g; g.build()'`); "
                "python_zstandard_b200 has no CPU fallback")
        L = C.CDLL(_LIB_PATH)
        vp, sz, u64, u32, i = C.c_void_p, C.c_size_t, C.c_uint64, C.c_uint32, C.c_int
        sigs = {
            "zb200_device_count": (i, []),
            "zb200_ctx_create": (i, [i, C.POINTER(vp)]),
            "zb200_ctx_destroy": (None, [vp]),
            "zb200_ctx_last_error": (C.c_char_p, [vp]),
            "zb200_error_string": (C.c_char_p, [i]),
            "zb200_ctx_synchronize": (i, [vp]),
            "zb200_ctx_stream": (vp, [vp]),
            "zb200_host_alloc": (vp, [vp, sz]),
            "zb200_host_free": (None, [vp, vp]),
            "zb200_device_alloc": (vp, [vp, sz]),
            "zb200_device_free": (None, [vp, vp]),
            "zb200_memcpy_h2d": (i, [vp, vp, vp, sz]),
            "zb200_memcpy_d2h": (i, [vp, vp, vp, sz]),
            "zb200_host_copy": (None, [vp, vp, sz]),
            "zb200_pointer_device": (i, [vp]),
            "zb200_ddict_create": (i, [vp, vp, sz, C.POINTER(vp)]),
            "zb200_ddict_free": (None, [vp]),
            "zb200_ddict_id": (u32, [vp]),
            "zb200_decompress_batch": (i, [vp, vp, vp, sz, vp, vp, u32, C.POINTER(vp)]),
            "zb200_decompress_batch_ptrs": (i, [vp, vp, vp, sz, vp, vp, u32, C.POINTER(vp)]),
            "zb200_decompress_batch_ex": (i, [vp, vp, vp, sz, vp, vp, vp, u32, C.POINTER(vp)]),
            "zb200_decompress_batch_ptrs_ex": (i, [vp, vp, vp, sz, vp, vp, vp, u32, C.POINTER(vp)]),
            "zb200_decompress_chain": (i, [vp, vp, vp, sz, vp, vp, C.POINTER(vp)]),
            "zb200_compress_batch": (i, [vp, vp, vp, sz, vp, vp, u32, C.POINTER(vp)]),
            "zb200_compress_batch_ptrs": (i, [vp, vp, vp, sz, vp, vp, u32, C.POINTER(vp)]),
            "zb200_compress_chain": (i, [vp, vp, vp, sz, vp, vp, C.POINTER(vp)]),
            "zb200_compress_bound": (u64, [u64]),
            "zb200_result_data": (vp, [vp]),
            "zb200_result_size": (u64, [vp]),
            "zb200_result_count": (sz, [vp]),
            "zb200_result_segments": (vp, [vp]),
            "zb200_result_first_error": (i, [vp, C.POINTER(sz), C.POINTER(i), C.POINTER(u64), C.POINTER(u64)]),
            "zb200_result_free": (None, [vp]),
            "zb200_frame_info": (i, [vp, sz, C.POINTER(FrameInfo)]),
            "zb200_profile_enable": (None, [vp, i]),
            "zb200_profile_reset": (None, [vp]),
            "zb200_profile_read": (i, [vp, C.POINTER(C.c_float), C.POINTER(u32)]),
            "zb200_kernel_name": (C.c_char_p, [i]),
            "zb200_last_scratch_bytes": (u64, [vp]),
            "zb200_last_chase_rounds": (i, [vp]),
            "zb200_decompress_batch_multi": (i, [vp, i, vp, vp, sz, vp, vp, sz, vp, u32, vp, vp]),
            "zb200_compress_batch_multi": (i, [vp, i, vp, vp, sz, vp, vp, sz, u32, vp, vp]),
            "zb200_multi_last_error": (C.c_char_p, []),
            "zb200_last_compress_kernel": (C.c_char_p, [vp]),
            "zb200_train_dictionary": (i, [vp, vp, vp, sz, vp, vp, sz, C.POINTER(sz), C.POINTER(u32), C.POINTER(u32)]),
        }
        for name, (res, args) in sigs.items():
            f = getattr(L, name, None)
            if f is None:
                continue          # entry points added by later milestones
            f.restype = res
            f.argtypes = args
        _lib = L
        return L


class Context:
    """One codec context per device (stream + scratch arenas + pinned pool)."""

    _by_device = {}
    _guard = threading.Lock()

    def __init__(self, device=0):
        L = lib()
        if L.zb200_device_count() <= 0:
            raise NativeError("no CUDA device visible: python_zstandard_b200 has no CPU fallback")
        h = C.c_void_p()
        rc = L.zb200_ctx_create(device, C.byref(h))
        if rc != 0:
            raise NativeError("zb200_ctx_create(device=%d) failed with %d" % (device, rc))
        self.L = L
        self.h = h
        self.device = device
        self.lock = threading.Lock()

    @classmethod
    def get(cls, device=0, slot=0):
        """Context `slot` of `device`.  Slot 0 is the default; slots 1.. are extra contexts (own stream,
        scratch and pinned pool) used to keep several sub-batches in flight so that host->device copies,
        kernels and device->host copies of different sub-batches overlap."""
        with cls._guard:
            c = cls._by_device.get((device, slot))
            if c is None:
                c = cls(device)
                cls._by_device[(device, slot)] = c
            return c

    def last_error(self):
        return self.L.zb200_ctx_last_error(self.h).decode()

    def check(self, rc, what):
        if rc != 0:
            raise NativeError("%s failed (%d): %s" % (what, rc, self.last_error()))

    # profiling ---------------------------------------------------------
    def profile(self, on=True):
        self.L.zb200_profile_enable(self.h, int(on))
        self.L.zb200_profile_reset(self.h)

    def profile_read(self):
        ms = (C.c_float * K_COUNT)()
        n = (C.c_uint32 * K_COUNT)()
        self.L.zb200_profile_read(self.h, ms, n)
        out = {}
        for k in range(K_COUNT):
            name = self.L.zb200_kernel_name(k).decode()
            if name and n[k]:
                out[name] = (float(ms[k]), int(n[k]))
        return out


_bytes_new = C.pythonapi.PyBytes_FromStringAndSize
_bytes_new.restype = C.py_object
_bytes_new.argtypes = [C.c_void_p, C.c_ssize_t]
_bytes_data = C.pythonapi.PyBytes_AsString
_bytes_data.restype = C.c_void_p
_bytes_data.argtypes = [C.py_object]


def bytes_from_address(addr, n):
    """bytes(n) filled from host memory at addr; large results are copied on several threads (zb200_host_copy)."""
    if n < (2 << 20):
        return C.string_at(addr, n) if n else b""
    b = _bytes_new(None, n)
    lib().zb200_host_copy(_bytes_data(b), addr, n)
    return b


def device_count():
    return lib().zb200_device_count()


_default_device = 0


def set_device(index):
    """Device that single-device calls use (one process per GPU: set it to LOCAL_RANK)."""
    global _default_device
    if index < 0 or index >= device_count():
        raise ValueError("invalid device index %d" % index)
    _default_device = index


def default_device():
    return _default_device
