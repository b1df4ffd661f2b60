"""The compressor through the public API across levels, window logs and dictionaries, on the device.

Every frame must regenerate through the reference decoder and through ours, and pass tests/frame_check.py, which also
holds every match to the window the frame header declares (a streaming decoder keeps only that much history).  The
launcher's kernel choices are pinned at their edges: zb_compress_smem from a largest block of 8 KiB at levels below 4,
zb_compress_recs for records of up to 2 KiB with a trained dictionary, zb_compress_blocks for the rest."""
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

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_ref(), reason="oracle/_ref is built from /root/reference")]

HERE = os.path.dirname(os.path.abspath(__file__))
TEXT = corpus.text_corpus(1 << 20).tobytes()
LEVELS = [-5, 1, 2, 3, 4, 5, 9, 19, 22]
WINDOW_LOGS = [0, 10, 12, 14, 15, 16, 17]


@pytest.fixture(scope="module")
def ref():
    return RefZstd()


@pytest.fixture(scope="module")
def orc():
    return Oracle()


def _block(window_log):
    return 1 << window_log if window_log and window_log < 17 else 128 << 10


def _segments(window_log):
    B = _block(window_log)
    rng = np.random.default_rng(window_log + 1)
    two = TEXT[1000:1000 + 2 * B]
    return [two, two, TEXT[500000:500000 + 3 * B + 5], TEXT[200000:200000 + B - 1], TEXT[300000:300000 + B + 1],
            bytes(B + 1), rng.integers(0, 256, B + 1).astype(np.uint8).tobytes(), b"", b"x"]


def _kernel():
    ctx = _native.Context.get(_native.default_device())
    return ctx.L.zb200_last_compress_kernel(ctx.h).decode()


def _check_all(ref, orc, segs, frames, checksum=True, content_size=True, dct=b"", dict_id=0):
    for i, (s, f) in enumerate(zip(segs, frames)):
        assert ref.decompress(f, len(s), dct) == s, i
        check_frame(f, s, dct, checksum=checksum, content_size=content_size, dict_id=dict_id, oracle=orc)
    d = zstd.ZstdDecompressor(dict_data=zstd.ZstdCompressionDict(dct) if dct else None)
    out = d.multi_decompress_to_buffer(frames, decompressed_sizes=struct.pack("=%dQ" % len(segs), *map(len, segs)))
    assert [out[i].tobytes() for i in range(len(segs))] == list(segs)


@pytest.mark.parametrize("level", LEVELS)
def test_levels_and_window_logs(ref, orc, level):
    """multi_compress_to_buffer with ZstdCompressionParameters(compression_level=L, window_log=W): a batch that repeats
    its first segment (history that leaks across a frame's border finds matches there), segments around the block size
    2^W, zeros and random bytes."""
    for W in WINDOW_LOGS:
        segs = _segments(W)
        p = zstd.ZstdCompressionParameters(compression_level=level, window_log=W, write_checksum=1)
        frames = zstd.ZstdCompressor(compression_params=p).multi_compress_to_buffer(segs)
        frames = [frames[i].tobytes() for i in range(len(segs))]
        _check_all(ref, orc, segs, frames)
        B = _block(W)
        assert all(max(check_frame(f, s, checksum=True, content_size=True, oracle=orc)["blocks"]) <= B for s, f in zip(segs, frames))


@pytest.mark.parametrize("level", [3, 4, 19])
def test_one_shot_and_header_variants(ref, orc, level):
    """compress() with content size and checksum off and on, at the window logs that cut blocks below 32 KiB."""
    for W in (0, 10, 14, 15, 16):
        B = _block(W)
        data = TEXT[7:7 + 3 * B + 5]
        for ck, cs in ((False, True), (True, False), (False, False)):
            p = zstd.ZstdCompressionParameters(compression_level=level, window_log=W, write_checksum=int(ck), write_content_size=int(cs))
            f = zstd.ZstdCompressor(compression_params=p).compress(data)
            assert ref.decompress(f, len(data)) == data
            check_frame(f, data, checksum=ck, content_size=cs, oracle=orc)


@pytest.mark.parametrize("level", [1, 3, 4, 9, 19])
def test_from_level_windows(ref, orc, level):
    """ZstdCompressionParameters.from_level(L, source_size=S) fills in the reference's window log for the size (14 at
    16 KB and below, 17 at 128 KB and below, ...); the frames follow it."""
    for S in (5000, 16384, 40000, 131072, 300000):
        p = zstd.ZstdCompressionParameters.from_level(level, source_size=S, write_checksum=1)
        segs = [TEXT[:S], TEXT[:S], TEXT[400000:400000 + S]]
        frames = zstd.ZstdCompressor(compression_params=p).multi_compress_to_buffer(segs)
        frames = [frames[i].tobytes() for i in range(3)]
        _check_all(ref, orc, segs, frames)
        f = zstd.ZstdCompressor(compression_params=p).compress(segs[2])
        assert ref.decompress(f, S) == segs[2]
        check_frame(f, segs[2], checksum=True, content_size=True, oracle=orc)


@pytest.mark.parametrize("level,window_log", [(3, 0), (4, 14), (5, 10), (19, 15)])
def test_device_buffers(ref, orc, level, window_log):
    """DeviceBufferWithSegments in, device frames out: the same frames as the host path, checked the same way."""
    segs = _segments(window_log)
    blob = b"".join(segs)
    lens = [len(s) for s in segs]
    off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
    table = np.stack([off, np.array(lens, dtype=np.uint64)], axis=1).astype(np.uint64).tobytes()
    p = zstd.ZstdCompressionParameters(compression_level=level, window_log=window_log, write_checksum=1)
    c = zstd.ZstdCompressor(compression_params=p)
    dbuf = zstd.DeviceBufferWithSegments(torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda(), table)
    dev = c.multi_compress_to_buffer(dbuf)
    frames = [dev[i].tobytes() for i in range(len(segs))]
    _check_all(ref, orc, segs, frames)
    host = c.multi_compress_to_buffer(zstd.BufferWithSegments(blob, table))
    assert [host[i].tobytes() for i in range(len(segs))] == frames


def test_kernel_choice_edges(ref, orc):
    """The launcher's edges, each side checked: largest block 8191 / 8192 bytes at level 3 (zb_compress_smem from 8 KiB),
    level 3 / 4 (the level >= 4 mode stays on zb_compress_blocks), records of 2048 / 2049 bytes with a trained dictionary
    (zb_compress_recs up to 2 KiB), and a dictionary at level >= 4 with blocks of 1 to 32 KiB."""
    def run(segs, kernel, level=3, window_log=0, dct=None, dict_id=0):
        p = zstd.ZstdCompressionParameters(compression_level=level, window_log=window_log, write_checksum=1, write_dict_id=1)
        c = zstd.ZstdCompressor(compression_params=p, dict_data=zstd.ZstdCompressionDict(dct) if dct else None)
        res = c.multi_compress_to_buffer(segs)
        assert _kernel() == kernel, (kernel, level, window_log, max(map(len, segs)))
        _check_all(ref, orc, segs, [res[i].tobytes() for i in range(len(segs))], dct=dct or b"", dict_id=dict_id)

    small = [TEXT[i * 9000:i * 9000 + 8191] for i in range(4)] + [TEXT[100:4000]]
    run(small, "zb_compress_blocks")
    run(small + [TEXT[50000:50000 + 8192]], "zb_compress_smem")
    run(small + [TEXT[50000:50000 + 8192]], "zb_compress_blocks", level=4)
    run([TEXT[:40000]] * 2, "zb_compress_smem", window_log=13)            # 8 KiB blocks
    run([TEXT[:40000]] * 2, "zb_compress_blocks", window_log=12)          # 4 KiB blocks
    dct = open(os.path.join(HERE, "golden", "dict.bin"), "rb").read()
    did = struct.unpack_from("<I", dct, 4)[0]
    recs = corpus.json_records(200)
    recs2k = [(r * 40)[:2048] for r in recs[:30]] + [r[:2048] for r in recs[30:60]]
    run(recs2k, "zb_compress_recs", dct=dct, dict_id=did)
    run(recs2k + [(recs[70] * 40)[:2049]], "zb_compress_blocks", dct=dct, dict_id=did)
    for W in (10, 12, 14, 15):
        long = b"".join(recs)[:3 * _block(W) + 5]
        run([long, long, recs[5], recs[6] * 3], "zb_compress_blocks", level=5, window_log=W, dct=dct, dict_id=did)
