"""The lazy mode (an explicit greedy / lazy / lazy2 strategy) through the public API, on the device.

Every frame must regenerate through the reference decoder and pass tests/frame_check.py, which holds every offset to the
window the frame header declares.  The device frames of the pinned lazy2 batch must equal the CPU build's
(tests/test_compress_lazy_host.py), and the launcher must report zb_compress_lazy exactly when a strategy is set."""
import hashlib
import os
import struct

import numpy as np
import pytest
import torch

import corpus
import python_zstandard_b200 as zstd
from python_zstandard_b200 import _native
from oracle import Oracle, RefZstd, have_ref
from tests.frame_check import check_frame
from tests.test_compress_lazy_host import COMBOS, PINNED_LAZY2, SILESIA, TEXT, pinned_batch

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_ref(), reason="oracle/_ref is built from /root/reference")]

HERE = os.path.dirname(os.path.abspath(__file__))
DICT = open(os.path.join(HERE, "golden", "dict.bin"), "rb").read()
DICT_ID = struct.unpack_from("<I", DICT, 4)[0]


@pytest.fixture(scope="module")
def ref():
    return RefZstd()


@pytest.fixture(scope="module")
def orc():
    return Oracle()


def _kernel():
    ctx = _native.Context.get(_native.default_device())
    return ctx.L.zb200_last_compress_kernel(ctx.h).decode()


def _compressor(strategy, search_log, min_match, window_log=0, checksum=True, content_size=True, dct=None):
    p = zstd.ZstdCompressionParameters(strategy=strategy, search_log=search_log, min_match=min_match, window_log=window_log,
                                       write_checksum=int(checksum), write_content_size=int(content_size), write_dict_id=1)
    return zstd.ZstdCompressor(compression_params=p, dict_data=zstd.ZstdCompressionDict(dct) if dct else None)


def _check(ref, orc, segs, frames, checksum=True, content_size=True, dct=b"", dict_id=0):
    for i, (s, f) in enumerate(zip(segs, frames)):
        assert ref.decompress(f, len(s), dct) == s, i
        check_frame(f, s, dct, checksum=checksum, content_size=content_size, dict_id=dict_id, oracle=orc)


def _table(segs):
    lens = [len(s) for s in segs]
    off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
    return np.stack([off, np.array(lens, dtype=np.uint64)], axis=1).astype(np.uint64).tobytes()


@pytest.mark.parametrize("strategy,search_log,min_match", COMBOS)
def test_round_trips(ref, orc, strategy, search_log, min_match):
    """The CPU suite's inputs through multi_compress_to_buffer (list, BufferWithSegments, DeviceBufferWithSegments),
    compress(), compressobj and frame 0 of compress_content_dict_chain."""
    rng = np.random.default_rng(search_log * 10 + min_match)
    segs = [TEXT[:65536], SILESIA[:65536], SILESIA[65536:], bytes(70000), rng.integers(0, 256, 5000).astype(np.uint8).tobytes(),
            b"x", b"", TEXT[3:3 + 300000]]
    c = _compressor(strategy, search_log, min_match)
    res = c.multi_compress_to_buffer(segs)
    assert _kernel() == "zb_compress_lazy"
    frames = [res[i].tobytes() for i in range(len(segs))]
    _check(ref, orc, segs, frames)
    blob, table = b"".join(segs), _table(segs)
    host = c.multi_compress_to_buffer(zstd.BufferWithSegments(blob, table))
    assert [host[i].tobytes() for i in range(len(segs))] == frames
    dev = c.multi_compress_to_buffer(zstd.DeviceBufferWithSegments(torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda(), table))
    assert [dev[i].tobytes() for i in range(len(segs))] == frames
    assert c.compress(segs[-1]) == frames[-1]
    o = c.compressobj()
    assert o.compress(segs[0]) + o.flush() == frames[0]
    chain = c.compress_content_dict_chain([segs[0], segs[0][:60000] + b"edit" + segs[0][60000:]])
    _check(ref, orc, segs[:1], chain[:1])
    for k, W in enumerate((10, 12, 14, 15, 16, 17)):
        B = 1 << W
        segs = [TEXT[W * 1000:W * 1000 + B - 1], TEXT[W * 2000:W * 2000 + B + 1], TEXT[W * 3000:W * 3000 + 3 * min(B, 1 << 17) + 5]]
        checksum, content_size = k % 2 == 0, k % 3 != 2
        res = _compressor(strategy, search_log, min_match, W, checksum, content_size).multi_compress_to_buffer(segs)
        _check(ref, orc, segs, [res[i].tobytes() for i in range(len(segs))], checksum, content_size)
    recs = [r[:1024] for r in corpus.json_records(24)]
    res = _compressor(strategy, search_log, min_match, dct=DICT).multi_compress_to_buffer(recs)
    assert _kernel() == "zb_compress_lazy"
    _check(ref, orc, recs, [res[i].tobytes() for i in range(len(recs))], dct=DICT, dict_id=DICT_ID)


def test_several_devices(ref, orc):
    """threads= over the visible devices: each range through the lazy mode, the same frames as one device writes."""
    segs = [TEXT[i * 50000:i * 50000 + 70000] for i in range(12)]
    c = _compressor(zstd.STRATEGY_LAZY, 4, 5)
    one = c.multi_compress_to_buffer(segs)
    many = c.multi_compress_to_buffer(segs, threads=-1)
    assert [many[i].tobytes() for i in range(len(segs))] == [one[i].tobytes() for i in range(len(segs))]
    _check(ref, orc, segs, [one[i].tobytes() for i in range(len(segs))])


def test_pinned_frames_equal_the_cpu_build(ref, orc):
    segs = pinned_batch()
    res = _compressor(zstd.STRATEGY_LAZY2, 4, 5).multi_compress_to_buffer(segs)
    frames = [res[i].tobytes() for i in range(len(segs))]
    _check(ref, orc, segs, frames)
    assert hashlib.sha256(b"".join(frames)).hexdigest() == PINNED_LAZY2


def test_kernel_choice(ref, orc):
    """A strategy takes the lazy mode at every edge of the level paths' kernel choice (8191 / 8192-byte blocks, level 4,
    records of up to 2 KiB with a dictionary); without one the names are today's."""
    small = [TEXT[i * 9000:i * 9000 + 8191] for i in range(4)]
    big = small + [TEXT[50000:50000 + 8192]]
    recs = corpus.json_records(60)
    recs2k = [(r * 40)[:2048] for r in recs]
    for segs, level, dct, plain in ((small, 3, None, "zb_compress_blocks"), (big, 3, None, "zb_compress_smem"),
                                    (big, 4, None, "zb_compress_blocks"), (recs2k, 3, DICT, "zb_compress_recs"),
                                    (recs2k, 4, DICT, "zb_compress_blocks")):
        d = zstd.ZstdCompressionDict(dct) if dct else None
        p = zstd.ZstdCompressionParameters(compression_level=level, write_checksum=1, write_dict_id=1)
        zstd.ZstdCompressor(compression_params=p, dict_data=d).multi_compress_to_buffer(segs)
        assert _kernel() == plain, (level, plain)
        zstd.ZstdCompressor(compression_params=zstd.ZstdCompressionParameters.from_level(level, write_checksum=1, write_dict_id=1),
                            dict_data=d).multi_compress_to_buffer(segs)
        assert _kernel() == plain, (level, plain)
        for strategy in (zstd.STRATEGY_GREEDY, zstd.STRATEGY_LAZY, zstd.STRATEGY_LAZY2):
            p = zstd.ZstdCompressionParameters(compression_level=level, strategy=strategy, write_checksum=1, write_dict_id=1)
            res = zstd.ZstdCompressor(compression_params=p, dict_data=d).multi_compress_to_buffer(segs)
            assert _kernel() == "zb_compress_lazy", (level, strategy)
            _check(ref, orc, segs, [res[i].tobytes() for i in range(len(segs))], dct=dct or b"", dict_id=DICT_ID if dct else 0)
