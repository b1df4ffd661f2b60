"""python_zstandard_b200 -- H100-native backend for python-zstandard's batch path.

Exposes the reference's names for that path (zstandard/__init__.pyi:312-320, 423-438 and the
buffer types) so a caller can ``import python_zstandard_b200 as zstandard``:

    ZstdCompressor(...).multi_compress_to_buffer / .compress
    ZstdDecompressor(...).multi_decompress_to_buffer / .decompress
    BufferWithSegments, BufferSegments, BufferSegment, BufferWithSegmentsCollection
    ZstdCompressionDict, train_dictionary (fastCover on the device), ZstdError, frame helpers and constants
    DeviceBufferWithSegments (not in the reference): the same batch calls on device-resident data, device-resident results

All codec work runs as CUDA kernels in ``libzb200.so`` (C ABI: include/zb200.h).
"""
from .errors import ZstdError  # noqa: F401
from .buffers import (BufferSegment, BufferSegments, BufferWithSegments,  # noqa: F401
                      BufferWithSegmentsCollection, DeviceBufferWithSegments, DeviceBufferSegment)
from .dictionary import (ZstdCompressionDict, DICT_TYPE_AUTO, DICT_TYPE_RAWCONTENT,  # noqa: F401
                         DICT_TYPE_FULLDICT, train_dictionary)
from .decompressor import ZstdDecompressor, FORMAT_ZSTD1, FORMAT_ZSTD1_MAGICLESS  # noqa: F401
from .compressor import ZstdCompressor, ZstdCompressionParameters  # noqa: F401
from ._native import set_device, default_device  # noqa: F401
from .streams import (COMPRESSOBJ_FLUSH_FINISH, COMPRESSOBJ_FLUSH_BLOCK, DECOMPRESSION_RECOMMENDED_INPUT_SIZE,  # noqa: F401
                      DECOMPRESSION_RECOMMENDED_OUTPUT_SIZE, COMPRESSION_RECOMMENDED_INPUT_SIZE,
                      COMPRESSION_RECOMMENDED_OUTPUT_SIZE)

__version__ = "0.25.0+b200"
backend = "b200"
backend_features = {"buffer_types", "multi_compress_to_buffer", "multi_decompress_to_buffer", "device_buffers"}

ZSTD_VERSION = (1, 5, 7)
FRAME_HEADER = b"\x28\xb5\x2f\xfd"
MAGIC_NUMBER = 0xFD2FB528
BLOCKSIZE_MAX = 131072
BLOCKSIZE_LOG_MAX = 17
CONTENTSIZE_UNKNOWN = (1 << 64) - 1
CONTENTSIZE_ERROR = (1 << 64) - 2
MAX_COMPRESSION_LEVEL = 22
WINDOWLOG_MIN = 10
WINDOWLOG_MAX = 31


def frame_content_size(data):
    """zstandard.frame_content_size (c-ext/backend_c.c:43-72)."""
    import ctypes as C
    from . import _native
    b = bytes(memoryview(data))
    info = _native.FrameInfo()
    _native.lib().zb200_frame_info(b, len(b), C.byref(info))
    if info.status:
        raise ZstdError("error when determining content size")
    if info.content_size == CONTENTSIZE_UNKNOWN:
        return -1
    return info.content_size


def frame_header_size(data):
    """zstandard.frame_header_size (c-ext/backend_c.c:74-102)."""
    import ctypes as C
    from . import _native
    b = bytes(memoryview(data))
    info = _native.FrameInfo()
    _native.lib().zb200_frame_info(b, len(b), C.byref(info))
    # ZSTD_frameHeaderSize (zstd/zstd.c:43637) looks at no magic number: anything shorter than 5 bytes is srcSize_wrong
    status = 72 if len(b) < 5 else info.status
    if status:
        raise ZstdError("could not determine frame header size: %s"
                        % _native.lib().zb200_error_string(status).decode())
    return info.header_size


class PinnedBuffer:
    """Page-locked host memory from the codec context's pool.  Data placed here (e.g. the `data`
    of a BufferWithSegments) is DMA-copied to the device at full PCIe rate instead of being staged."""

    def __init__(self, nbytes, device=None):
        import ctypes as C
        from . import _native
        self._ctx = _native.Context.get(_native.default_device() if device is None else device)
        self._ptr = self._ctx.L.zb200_host_alloc(self._ctx.h, nbytes)
        if not self._ptr:
            raise MemoryError("pinned allocation of %d bytes failed" % nbytes)
        self.nbytes = nbytes
        self._arr = (C.c_ubyte * nbytes).from_address(self._ptr)
        import weakref
        self._fin = weakref.finalize(self, self._ctx.L.zb200_host_free, self._ctx.h, self._ptr)

    def __buffer__(self, flags):
        return memoryview(self._arr).cast("B")

    def __release_buffer__(self, view):
        pass

    def __len__(self):
        return self.nbytes
