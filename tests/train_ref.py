"""The reference's fastCover trainer through ctypes (oracle/_ref/libzstd_ref.so), with zstandard.train_dictionary's
argument defaulting (c-ext/compressiondict.c:52-61).  TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import ctypes as C
import os

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libzstd_ref.so")


class FastCoverParams(C.Structure):
    """ZDICT_fastCover_params_t with its ZDICT_params_t (zstd/zstd.c:48221-48233)."""
    _fields_ = [("k", C.c_uint), ("d", C.c_uint), ("f", C.c_uint), ("steps", C.c_uint), ("nbThreads", C.c_uint),
                ("splitPoint", C.c_double), ("accel", C.c_uint), ("shrinkDict", C.c_uint),
                ("shrinkDictMaxRegression", C.c_uint),
                ("compressionLevel", C.c_int), ("notificationLevel", C.c_uint), ("dictID", C.c_uint)]


class TrainError(Exception):
    pass


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(REF, mode=C.RTLD_GLOBAL)
        L.ZDICT_optimizeTrainFromBuffer_fastCover.restype = C.c_size_t
        L.ZDICT_optimizeTrainFromBuffer_fastCover.argtypes = [C.c_void_p, C.c_size_t, C.c_char_p, C.POINTER(C.c_size_t),
                                                              C.c_uint, C.POINTER(FastCoverParams)]
        L.ZDICT_isError.restype = C.c_uint
        L.ZDICT_isError.argtypes = [C.c_size_t]
        L.ZDICT_getErrorName.restype = C.c_char_p
        L.ZDICT_getErrorName.argtypes = [C.c_size_t]
        L.ZDICT_getDictID.restype = C.c_uint
        L.ZDICT_getDictID.argtypes = [C.c_char_p, C.c_size_t]
        _lib = L
    return _lib


def train_fastcover(dict_size, samples, k=0, d=0, f=0, split_point=0.0, accel=0, dict_id=0, level=0, steps=0, threads=0, nb_threads=1):
    """(dictionary bytes, k, d) as zstandard.train_dictionary would return them; TrainError(ZDICT_getErrorName) on failure.
    The call runs on nb_threads threads (1: candidates finish in ZDICT's loop order, which decides ties)."""
    if threads < 0:
        threads = os.cpu_count() or 1
    if not steps and not threads:
        d = d or 8
        steps = steps or 4
        level = level or 3
    L = lib()
    p = FastCoverParams(k=k, d=d, f=f, steps=steps, nbThreads=nb_threads, splitPoint=split_point, accel=accel,
                        compressionLevel=level, dictID=dict_id)
    blob = b"".join(samples)
    sizes = (C.c_size_t * max(len(samples), 1))(*[len(s) for s in samples])
    out = C.create_string_buffer(max(dict_size, 1))
    n = L.ZDICT_optimizeTrainFromBuffer_fastCover(out, dict_size, blob, sizes, len(samples), C.byref(p))
    if L.ZDICT_isError(n):
        raise TrainError(L.ZDICT_getErrorName(n).decode())
    return out.raw[:n], p.k, p.d


def dict_id(data):
    return lib().ZDICT_getDictID(bytes(data), len(data))
