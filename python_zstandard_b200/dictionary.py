"""ZstdCompressionDict -- the dictionary object handed to (de)compressors -- and train_dictionary.

ZstdCompressionDict mirrors c-ext/compressiondict.c:164-348 for the *use* of a dictionary (bytes,
dict_id(), as_bytes(), len()).  train_dictionary mirrors c-ext/compressiondict.c:13-146: the fastCover
trainer (ZDICT_optimizeTrainFromBuffer_fastCover) runs on the device through zb200_train_dictionary,
candidates side by side, each scored with this package's own compressor.
"""
import struct
import threading

from . import _native
from .errors import ZstdError

DICT_TYPE_AUTO = 0
DICT_TYPE_RAWCONTENT = 1
DICT_TYPE_FULLDICT = 2
_DICT_MAGIC = 0xEC30A437


class ZstdCompressionDict:
    def __init__(self, data, dict_type=DICT_TYPE_AUTO, k=0, d=0):
        if dict_type not in (DICT_TYPE_AUTO, DICT_TYPE_RAWCONTENT, DICT_TYPE_FULLDICT):
            raise ValueError("invalid dictionary load mode: %d; must use DICT_TYPE_* constants" % dict_type)
        self._data = bytes(memoryview(data))
        self._dict_type = dict_type
        self.k = k
        self.d = d
        self._ddicts = {}       # device index -> native handle
        self._lock = threading.Lock()
        is_full = len(self._data) >= 8 and struct.unpack_from("<I", self._data)[0] == _DICT_MAGIC
        if dict_type == DICT_TYPE_FULLDICT and not is_full:
            raise ZstdError("dictionary is not a full zstd dictionary")
        self._raw = dict_type == DICT_TYPE_RAWCONTENT or not is_full

    def __len__(self):
        return len(self._data)

    def dict_id(self):
        if self._raw:
            return 0
        return struct.unpack_from("<I", self._data, 4)[0]

    def as_bytes(self):
        return self._data

    def precompute_compress(self, level=0, compression_params=None):
        if level and compression_params:
            raise ValueError("must only specify one of level or compression_params")
        if not level and not compression_params:
            raise ValueError("must specify one of level or compression_params")
        # digests are built lazily per device on first use

    # -- device digest (ensure_ddict, c-ext/compressiondict.c:148-162)
    def _ddict(self, ctx):
        """The device digest of this dictionary on ctx's device: one per device, created under the dictionary's lock and
        the context's lock (several pipeline workers may ask at once), freed when the dictionary object goes away."""
        h = self._ddicts.get(ctx.device)
        if h is not None:
            return h
        with self._lock:
            h = self._ddicts.get(ctx.device)
            if h is None:
                import ctypes as C
                import weakref
                h = C.c_void_p()
                data = self._data
                if self._raw and len(data) >= 8 and struct.unpack_from("<I", data)[0] == _DICT_MAGIC:
                    raise ZstdError("raw-content dictionaries starting with the dictionary magic are not supported")
                with ctx.lock:
                    rc = ctx.L.zb200_ddict_create(ctx.h, data, len(data), C.byref(h))
                if rc != 0:
                    raise ZstdError("unable to load dictionary: %s" % ctx.last_error())
                self._ddicts[ctx.device] = h
                weakref.finalize(self, ctx.L.zb200_ddict_free, h)
        return h


def train_dictionary(dict_size, samples, k=0, d=0, f=0, split_point=0.0, accel=0, notifications=0, dict_id=0, level=0,
                     steps=0, threads=0):
    """zstandard.train_dictionary (c-ext/compressiondict.c:13-146): a full dictionary of at most dict_size bytes trained
    from `samples` (a list of bytes) with fastCover, on the device.  `threads` only matters for the defaulting rule below
    and `notifications` not at all: the candidates of the search always run side by side on the GPU."""
    import ctypes as C
    if not isinstance(samples, list):
        raise TypeError("train_dictionary() argument 2 must be list, not %s" % type(samples).__name__)
    for s in samples:
        if not isinstance(s, bytes):
            raise ValueError("samples must be bytes")
    if threads < 0:
        import os
        threads = os.cpu_count() or 1
    if not steps and not threads:          # the defaults of ZDICT_trainFromBuffer, as the reference applies them
        d = d or 8
        steps = steps or 4
        level = level or 3
    p = _native.TrainParams(k=k, d=d, f=f, steps=steps, accel=accel, level=level, dict_id=dict_id, reserved=0,
                            split_point=split_point)
    blob = b"".join(samples)
    sizes = (C.c_size_t * max(len(samples), 1))(*[len(s) for s in samples])
    out = C.create_string_buffer(max(dict_size, 1))
    n = C.c_size_t(0)
    ck, cd = C.c_uint32(0), C.c_uint32(0)
    ctx = _native.Context.get(_native.default_device())
    with ctx.lock:
        rc = ctx.L.zb200_train_dictionary(ctx.h, blob, sizes, len(samples), C.byref(p), out, dict_size, C.byref(n),
                                          C.byref(ck), C.byref(cd))
    if rc > 0:
        raise ZstdError("cannot train dict: %s" % ctx.last_error())
    ctx.check(rc, "zb200_train_dictionary")
    return ZstdCompressionDict(out.raw[:n.value], DICT_TYPE_FULLDICT, k=ck.value, d=cd.value)
