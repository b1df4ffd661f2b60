"""The hand-built frames of tests/crafted_frames.py on the device, through the public API, on all four launcher modes:
a lane per frame, a lane per block with the tile executor, a lane per block with pointer jumping, and the automatic
choice.  What the writer's executor predicts (and the CPU suite checks against the reference) must come back byte for
byte; every frame it calls malformed must raise."""
import numpy as np
import pytest
import torch

import python_zstandard_b200 as zstd
from oracle import have_ref
from tests import crafted_frames

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_ref(), reason="oracle/_ref is built from /root/reference")]

CASES = crafted_frames.catalogue() + crafted_frames.stream_cases(np.random.default_rng(106))
DICT_REPS = crafted_frames.dict_rep_cases(np.random.default_rng(107))
MODES = {"lane-per-frame": ("0", None), "blocks+tiles": ("1", "0"), "blocks+pointer-jumping": ("1", "1"), "auto": (None, None)}


@pytest.fixture(params=list(MODES))
def mode(request, monkeypatch):
    for k, v in zip(("ZB200_BLOCK_PATH", "ZB200_CHASE"), MODES[request.param]):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, v)
    return request.param


def _decompressor(dct):
    return zstd.ZstdDecompressor(dict_data=zstd.ZstdCompressionDict(dct) if dct else None)


def _table(lens):
    off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
    return np.stack([off, np.asarray(lens, dtype=np.uint64)], axis=1).astype(np.uint64)


def _groups(cases):
    out = {}
    for c in cases:
        out.setdefault(c.dict, []).append(c)
    return out.items()


def test_valid_frames_in_batches(mode):
    """Valid frames of one dictionary in one call: host buffers, then device-resident buffers."""
    for dct, cases in _groups([c for c in CASES if c.expected is not None]):
        d = _decompressor(dct)
        sizes = np.array([len(c.expected) for c in cases], dtype=np.uint64)
        out = d.multi_decompress_to_buffer([c.frame for c in cases], decompressed_sizes=sizes.tobytes())
        for i, c in enumerate(cases):
            assert out[i].tobytes() == c.expected, (mode, c.name)
        blob = bytearray(b"".join(c.frame for c in cases))
        dev = zstd.DeviceBufferWithSegments(torch.frombuffer(blob, dtype=torch.uint8).cuda(), _table([len(c.frame) for c in cases]).tobytes())
        dout = d.multi_decompress_to_buffer(dev, decompressed_sizes=sizes.tobytes())
        for i, c in enumerate(cases):
            assert dout[i].tobytes() == c.expected, (mode, c.name)


def test_every_frame_alone(mode):
    """ZstdDecompressor.decompress of each frame; malformed ones raise, also from a batch of one on the device.  (decompress()
    sizes its output from the first frame header it sees, so the frame behind a skippable frame is left to the batch
    test above.)"""
    for dct, cases in _groups(CASES):
        d = _decompressor(dct)
        for c in cases:
            if c.name == "skippable_frame_in_front":
                continue
            cap = c.size
            if c.expected is not None:
                assert d.decompress(c.frame, max_output_size=cap) == c.expected, (mode, c.name)
                continue
            with pytest.raises(zstd.ZstdError):
                d.decompress(c.frame, max_output_size=cap)
            dev = zstd.DeviceBufferWithSegments(torch.frombuffer(bytearray(c.frame), dtype=torch.uint8).cuda(), _table([len(c.frame)]).tobytes())
            with pytest.raises(zstd.ZstdError):
                d.multi_decompress_to_buffer(dev, decompressed_sizes=np.array([cap], dtype=np.uint64).tobytes())


def test_dictionary_repcodes_at_the_content_size(mode):
    for c in DICT_REPS:
        if c.expected is not None:
            assert _decompressor(c.dict).decompress(c.frame) == c.expected, c.name
        else:
            with pytest.raises(zstd.ZstdError):
                _decompressor(c.dict).decompress(c.frame)


def test_offset_above_2_31_in_a_frame_over_2_gib(mode):
    """A legal offset of 2^31 + 512 KiB - 7: 512 KiB of raw blocks, 2 GiB of RLE blocks, then a match that copies from the
    raw blocks.  The window (2.25 GiB) keeps the batch off the block path, whose history tags symbolic repcodes with bit
    31, whatever ZB200_BLOCK_PATH says.  The compressed frame is above 512 KiB, so zb_scan_frames_big scans it."""
    from tests import frame_writer as fw
    raw = ((torch.arange(4 * 131072, dtype=torch.int64) * 2654435761) >> 13).to(torch.uint8)
    raw_b = raw.numpy().tobytes()
    n_rle = 16384
    start = len(raw_b) + n_rle * 131072 + 3                                   # where the match starts
    off = start - 10
    assert off >= 1 << 31
    blocks = [fw.Raw(raw_b[k * 131072:(k + 1) * 131072]) for k in range(4)] + [fw.Rle(k & 0xFF, 131072) for k in range(n_rle)]
    blocks.append(fw.Comp(fw.Lits(b"XYZ"), [(3, 64, off + 3)], ll=fw.RLE_T(3), of=fw.RLE_T(31), ml=fw.RLE_T(39)))
    total = start + 64
    frame = fw.frame_bytes(fw.Frame(blocks, window_log=31, window_mantissa=1, fcs_bytes=8), total)
    assert len(frame) > 512 << 10
    dev = zstd.DeviceBufferWithSegments(torch.frombuffer(bytearray(frame), dtype=torch.uint8).cuda(), _table([len(frame)]).tobytes())
    out = zstd.ZstdDecompressor().multi_decompress_to_buffer(dev)
    assert out.size == total
    t = torch.as_tensor(out, device="cuda")
    assert torch.equal(t[:len(raw_b)], raw.cuda())
    rle = t[len(raw_b):len(raw_b) + n_rle * 131072].view(n_rle, 131072)
    assert bool((rle == (torch.arange(n_rle, device="cuda") & 0xFF).to(torch.uint8)[:, None]).all())
    del rle
    assert t[start - 3:].cpu().numpy().tobytes() == b"XYZ" + raw_b[10:74]
