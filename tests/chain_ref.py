"""ZstdDecompressor.decompress_content_dict_chain of the reference (c-ext/decompressor.c:620-890) restated over ctypes on
oracle/_ref/libzstd_ref.so, and a writer of revision chains: each revision compressed with the previous one as a raw-content
prefix (ZSTD_CCtx_refPrefix).  TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import ctypes as C
import os

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libzstd_ref.so")
CONTENTSIZE_UNKNOWN = (1 << 64) - 1
DCT_RAW_CONTENT = 1
C_COMPRESSION_LEVEL, C_CONTENT_SIZE_FLAG, C_CHECKSUM_FLAG = 100, 200, 201
E_END = 2                     # ZSTD_e_end


class FrameHeader(C.Structure):
    """ZSTD_FrameHeader (zstd/zstd.h)."""
    _fields_ = [("frameContentSize", C.c_ulonglong), ("windowSize", C.c_ulonglong), ("blockSizeMax", C.c_uint),
                ("frameType", C.c_int), ("headerSize", C.c_uint), ("dictID", C.c_uint), ("checksumFlag", C.c_uint),
                ("_reserved1", C.c_uint), ("_reserved2", C.c_uint)]


class InBuffer(C.Structure):
    _fields_ = [("src", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


class OutBuffer(C.Structure):
    _fields_ = [("dst", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


class ChainError(Exception):
    """What the reference raises as ZstdError."""


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(REF, mode=C.RTLD_GLOBAL)
        sz, vp = C.c_size_t, C.c_void_p
        for name, res, args in [
                ("ZSTD_getFrameHeader", sz, [C.POINTER(FrameHeader), vp, sz]),
                ("ZSTD_createDCtx", vp, []), ("ZSTD_freeDCtx", sz, [vp]),
                ("ZSTD_DCtx_setMaxWindowSize", sz, [vp, sz]),
                ("ZSTD_DCtx_refPrefix_advanced", sz, [vp, vp, sz, C.c_int]),
                ("ZSTD_DCtx_loadDictionary", sz, [vp, vp, sz]),
                ("ZSTD_decompressStream", sz, [vp, C.POINTER(OutBuffer), C.POINTER(InBuffer)]),
                ("ZSTD_isError", C.c_uint, [sz]), ("ZSTD_getErrorName", C.c_char_p, [sz]),
                ("ZSTD_createCCtx", vp, []), ("ZSTD_freeCCtx", sz, [vp]),
                ("ZSTD_CCtx_setParameter", sz, [vp, C.c_int, C.c_int]),
                ("ZSTD_CCtx_refPrefix", sz, [vp, vp, sz]),
                ("ZSTD_compressBound", sz, [sz]),
                ("ZSTD_compress2", sz, [vp, vp, sz, vp, sz])]:
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _lib = L
    return _lib


def _err(L, z):
    return L.ZSTD_getErrorName(z).decode()


def decompress_chain(frames, dict_data=None, max_window_size=0):
    """The reference function on a decompressor built with `dict_data` (raw dictionary bytes, referenced by the constructor,
    so chunk 0 decodes with it) and `max_window_size`.  Same exception types and texts; ZstdError is ChainError here."""
    if not isinstance(frames, list):
        raise TypeError("decompress_content_dict_chain() argument 1 must be list")
    if not frames:
        raise ValueError("empty input chain")
    L = lib()
    dctx = L.ZSTD_createDCtx()
    try:
        if max_window_size:
            L.ZSTD_DCtx_setMaxWindowSize(dctx, max_window_size)
        if dict_data:
            d = bytes(dict_data)
            L.ZSTD_DCtx_loadDictionary(dctx, d, len(d))
        prev = None
        for k, chunk in enumerate(frames):
            if not isinstance(chunk, bytes):
                raise ValueError("chunk %d must be bytes" % k)
            fh = FrameHeader()
            z = L.ZSTD_getFrameHeader(C.byref(fh), chunk, len(chunk))
            if L.ZSTD_isError(z):
                raise ValueError("chunk %d is not a valid zstd frame" % k)
            if z:
                raise ValueError("chunk %d is too small to contain a zstd frame" % k)
            if fh.frameContentSize == CONTENTSIZE_UNKNOWN:
                raise ValueError("chunk %d missing content size in frame" % k)
            size = fh.frameContentSize
            if k == 0:
                caps = [size, size]            # the reference's two buffers: grown, never shrunk
                cap = size
            else:
                caps[k % 2] = cap = max(caps[k % 2], size)
                z = L.ZSTD_DCtx_refPrefix_advanced(dctx, prev, len(prev), DCT_RAW_CONTENT)
                if L.ZSTD_isError(z):
                    raise ChainError("failed to load prefix dictionary at chunk %d" % k)
            out = C.create_string_buffer(max(cap, 1))
            ob = OutBuffer(C.cast(out, C.c_void_p), cap, 0)
            ib = InBuffer(C.cast(C.c_char_p(chunk), C.c_void_p), len(chunk), 0)
            z = L.ZSTD_decompressStream(dctx, C.byref(ob), C.byref(ib))
            if L.ZSTD_isError(z):
                raise ChainError("could not decompress chunk %d: %s" % (k, _err(L, z)))
            if z:
                raise ChainError("chunk %d did not decompress full frame" % k)
            if len(frames) == 1:
                return out.raw[:size]          # (the reference returns the header's size; beyond ob.pos its bytes are uninitialised)
            prev = out.raw[:ob.pos]
        return prev
    finally:
        L.ZSTD_freeDCtx(dctx)


def compress_chain(revisions, level=3, checksum=False):
    """Frame k: revisions[k] compressed with revisions[k - 1] as a raw-content prefix (frame 0: no prefix); content size set."""
    L = lib()
    cctx = L.ZSTD_createCCtx()
    out = []
    try:
        prev = None
        for rev in revisions:
            rev = bytes(rev)
            L.ZSTD_CCtx_setParameter(cctx, C_COMPRESSION_LEVEL, level)
            L.ZSTD_CCtx_setParameter(cctx, C_CONTENT_SIZE_FLAG, 1)
            L.ZSTD_CCtx_setParameter(cctx, C_CHECKSUM_FLAG, 1 if checksum else 0)
            if prev is not None:
                L.ZSTD_CCtx_refPrefix(cctx, prev, len(prev))
            cap = L.ZSTD_compressBound(len(rev))
            buf = C.create_string_buffer(cap)
            z = L.ZSTD_compress2(cctx, buf, cap, rev, len(rev))
            if L.ZSTD_isError(z):
                raise ChainError(_err(L, z))
            out.append(buf.raw[:z])
            prev = rev
        return out
    finally:
        L.ZSTD_freeCCtx(cctx)


def revisions(base, n, seed=0, edits=3, lo=10, hi=200):
    """n revisions of `base`: each changes the previous one by `edits` seeded replacements / insertions / deletions of
    lo..hi bytes."""
    import random
    rng = random.Random(seed)
    cur = bytearray(base)
    out = [bytes(cur)]
    for _ in range(n - 1):
        for _ in range(edits):
            ln = rng.randint(lo, hi)
            at = rng.randrange(max(1, len(cur) - ln))
            kind = rng.randrange(3)
            blob = bytes(rng.randrange(32, 127) for _ in range(ln))
            if kind == 0:
                cur[at:at + ln] = blob
            elif kind == 1:
                cur[at:at] = blob
            else:
                del cur[at:at + ln]
        out.append(bytes(cur))
    return out
