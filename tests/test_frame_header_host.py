"""The host's frame-header parse against the reference, without a GPU: zb200_frame_info (libzb200.so, the parser the frame
scans run on the device) against ZSTD_getFrameHeader, and frame_header_size against ZSTD_frameHeaderSize, both from
oracle/_ref/libzstd_ref.so over ctypes.  Skippable frames of 5 bytes or more are not compared: zb200_frame_info reports
them as prefix_unknown."""
import ctypes as C
import itertools
import os
import random
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import __graft_entry__ as entry  # noqa: E402
import chain_ref as R          # noqa: E402
import helpers                 # noqa: E402

pytestmark = pytest.mark.skipif(not os.path.exists(R.REF), reason="oracle/_ref/libzstd_ref.so not built")

MAGIC = bytes.fromhex("28b52ffd")
# the bytes of the zstd and skippable magic numbers (0x184D2A50..5F), and a few others
ALPHABET = bytes([0x28, 0xB5, 0x2F, 0xFD, 0x50, 0x5A, 0x2A, 0x4D, 0x18, 0x00, 0x51, 0xFF])


@pytest.fixture(scope="module")
def libs():
    entry.build()
    from python_zstandard_b200 import _native
    ref = C.CDLL(R.REF)
    ref.ZSTD_getFrameHeader.restype = C.c_size_t
    ref.ZSTD_getFrameHeader.argtypes = [C.POINTER(R.FrameHeader), C.c_char_p, C.c_size_t]
    ref.ZSTD_frameHeaderSize.restype = C.c_size_t
    ref.ZSTD_frameHeaderSize.argtypes = [C.c_char_p, C.c_size_t]
    ref.ZSTD_isError.restype = C.c_uint
    ref.ZSTD_isError.argtypes = [C.c_size_t]
    ref.ZSTD_getErrorName.restype = C.c_char_p
    ref.ZSTD_getErrorName.argtypes = [C.c_size_t]
    return _native, ref


def _ours(native, b):
    info = native.FrameInfo()
    native.lib().zb200_frame_info(b, len(b), C.byref(info))
    if info.status:
        return (info.status,)
    return (0, info.header_size, info.content_size, info.window_size, info.dict_id, info.has_checksum)


def _reference(ref, b):
    """ZSTD_getFrameHeader's result as a zb200_frame_info status (an error: its code; more bytes wanted: srcSize_wrong)."""
    fh = R.FrameHeader()
    r = ref.ZSTD_getFrameHeader(C.byref(fh), b, len(b))
    if ref.ZSTD_isError(r):
        return ((1 << 64) - r,)
    if r > 0:
        return (72,)
    return (0, fh.headerSize, fh.frameContentSize, fh.windowSize, fh.dictID, fh.checksumFlag)


def _inputs():
    for _name, frame, _raw, _dct in helpers.golden_vectors():
        for n in range(min(len(frame), 18) + 1):
            yield frame[:n]
    for n in range(1, 5):
        for t in itertools.product(ALPHABET, repeat=n):
            yield bytes(t)
    rng = random.Random(8878)
    for _ in range(4000):
        yield MAGIC + bytes(rng.randrange(256) for _ in range(rng.randrange(1, 15)))


def test_frame_info_equals_the_reference(libs):
    native, ref = libs
    seen = set()
    for b in _inputs():
        if b in seen:
            continue
        seen.add(b)
        assert _ours(native, b) == _reference(ref, b), b.hex()
    assert len(seen) > 20000


def test_frame_header_size_of_short_input_equals_the_reference(libs):
    import python_zstandard_b200 as zstd
    ref = libs[1]
    for n in range(5):
        for t in itertools.product(ALPHABET, repeat=n):
            b = bytes(t)
            z = ref.ZSTD_frameHeaderSize(b, n)
            assert ref.ZSTD_isError(z), b.hex()
            want = "could not determine frame header size: %s" % ref.ZSTD_getErrorName(z).decode()
            with pytest.raises(zstd.ZstdError) as e:
                zstd.frame_header_size(b)
            assert str(e.value) == want, b.hex()
