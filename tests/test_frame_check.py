"""Self-test of the RFC 8878 frame checker (tests/frame_check.py): frames from tests/frame_writer.py that keep every
rule pass, and a frame that breaks one rule fails -- one case per rule, so a checker that accepts everything is caught."""
import struct

import numpy as np
import pytest

from tests import frame_writer as fw
from tests.frame_check import FrameCheckError, check_frame, dict_content, parse_header
from tests.frame_writer import FSE, Comp, Dictionary, Frame, Lits, Raw, Rle


@pytest.fixture(scope="module")
def orc():
    from oracle import Oracle
    return Oracle()


def _text(n, seed=1):
    rng = np.random.default_rng(seed)
    return bytes(rng.choice(np.frombuffer(b"abcdefgh ", np.uint8), n))


def written(F, dictionary=None):
    data, expected, _ = fw.write(F, dictionary)
    assert expected is not None
    return data, expected


def ok(orc, frame, data, dct=b"", **kw):
    kw.setdefault("checksum", False)
    kw.setdefault("content_size", True)
    return check_frame(frame, data, dct, oracle=orc, **kw)


def bad(orc, frame, data, match, dct=b"", **kw):
    with pytest.raises(FrameCheckError, match=match):
        ok(orc, frame, data, dct, **kw)


def test_valid_frames_pass(orc):
    t = _text(5000)
    f, d = written(Frame([Raw(t[:1024]), Comp(Lits(t[1024:1100]), [(10, 50, 3 + 900), (0, 20, 1)]), Rle(7, 1000)], window_log=10))
    h = ok(orc, f, d)
    assert h["window_size"] == 1024 and h["blocks"] == [1024, h["blocks"][1], 1000] and h["max_offset"] == 900
    f, d = written(Frame([Raw(t[:300])], single_segment=True, checksum=True))
    assert ok(orc, f, d, checksum=True)["window_size"] == 300
    f, d = written(Frame([Raw(t[:300])], window_log=12, content_size=False))
    assert ok(orc, f, d, content_size=False)["content_size"] is None


def test_window_size_follows_the_descriptor(orc):
    """Window_Size = 2^(10 + exponent) + mantissa eighths: a 1920-byte block fits window_log 10 with mantissa 7, one more
    byte does not, and neither does a block above 128 KiB under a larger window."""
    t = _text(140000)
    f, d = written(Frame([Raw(t[:1920])], window_log=10, window_mantissa=7))
    assert ok(orc, f, d)["window_size"] == 1920
    f, d = fw.write(Frame([Raw(t[:1921])], window_log=10, window_mantissa=7))[:2]
    bad(orc, f, t[:1921], "Block_Maximum_Size")
    f = fw.frame_bytes(Frame([Raw(t[:(128 << 10) + 1])], window_log=18), (128 << 10) + 1)
    bad(orc, f, t[:(128 << 10) + 1], "Block_Maximum_Size")
    # a compressed block that is small but regenerates more than the window (the oracle refuses it too)
    f = fw.write(Frame([Comp(Lits(t[:100]), [(50, 1500, 3 + 40)])], window_log=10))[0]
    bad(orc, f, t[:50] + (t[10:50] * 40)[:1500] + t[50:100], "regenerates|rejects")


def test_offsets_beyond_the_window(orc):
    """An offset that stays inside the frame but reaches past Window_Size is caught (the oracle itself decodes it)."""
    t = _text(3000)
    F = Frame([Raw(t[:1024]), Raw(t[1024:2048]), Comp(Lits(t[2048:2050]), [(2, 16, 3 + 2000)])], window_log=10)
    f, d = fw.write(F)[:2]
    assert d is not None and orc.decompress(f, len(d)) == d
    bad(orc, f, d, "beyond Window_Size")
    F.window_log = 11
    f, d = written(F)
    assert ok(orc, f, d)["max_offset"] == 2000


def test_offsets_into_the_dictionary(orc):
    """Offsets may reach the dictionary content whatever the window; with a zstd-format dictionary its content starts after
    the entropy tables, which dict_content finds."""
    content = _text(4000, seed=2)
    wts = [0] * 32 + [1, 1] + [0] * 63 + [4, 3, 3, 2, 2, 2, 2, 2, 1, 1, 1, 1]
    for D in (Dictionary(content, raw=True),
              Dictionary(content, dict_id=9, weights=wts, of=FSE(fw.OF_DEFAULT[0], 5), ml=FSE(fw.ML_DEFAULT[0], 6), ll=FSE(fw.LL_DEFAULT[0], 6)),
              Dictionary(content, dict_id=11, weights=wts, weights_fse=([12, 8, 6, 4, 2], 5),
                         of=FSE(fw.OF_DEFAULT[0], 5), ml=FSE(fw.ML_DEFAULT[0], 6), ll=FSE(fw.LL_DEFAULT[0], 6))):
        assert dict_content(D.data) == content
        did = D.dict_id if not D.raw else 0
        f, d = written(Frame([Comp(Lits(b"abc"), [(3, 40, 3 + 3500)])], single_segment=True, dict_id=did), D)
        assert ok(orc, f, d, D.data, dict_id=did)["max_offset"] == 3500           # 3500 > the 43-byte window: fine
        # the same frame checked against a dictionary with less content reaches in front of it
        short = Dictionary(content[:3000], raw=True)
        bad(orc, f, d, "in front of the frame|rejects", short.data, dict_id=did)


def test_header_rules(orc):
    t = _text(600)
    f, d = written(Frame([Raw(t)], single_segment=True))
    g = bytearray(f); g[0] ^= 1
    bad(orc, bytes(g), d, "magic")
    g = bytearray(f); g[4] |= 1 << 3
    bad(orc, bytes(g), d, "reserved")
    # the 2-byte content size stores size - 256
    assert parse_header(f)["content_size"] == 600 and f[5:7] == struct.pack("<H", 600 - 256)
    g = bytearray(f); g[5:7] = struct.pack("<H", 600)
    bad(orc, bytes(g), d, "content size 856")
    # a window descriptor in front of a single-segment frame's fields shifts everything behind it
    g = bytes(f[:5]) + bytes([0]) + bytes(f[5:])
    bad(orc, g, d, "content size|block|frame")
    f2, _ = written(Frame([Raw(t)], content_size=False, window_log=10))
    bad(orc, f2, d, "not written")
    bad(orc, f, d, "not requested", content_size=False)
    bad(orc, fw.write(Frame([Raw(t)], single_segment=True, content_size=601))[0], d, "content size 601")


def test_dictionary_id_rules(orc):
    t = _text(100)
    D = Dictionary(b"", raw=True)
    f, d = written(Frame([Raw(t)], single_segment=True, dict_id=7))
    assert ok(orc, f, d, dict_id=7)["dict_id"] == 7
    bad(orc, f, d, "not requested")
    bad(orc, f, d, "dictionary ID 7, expected 8", dict_id=8)
    f, d = written(Frame([Raw(t)], single_segment=True), D)
    bad(orc, f, d, "dictionary ID None", dict_id=7)


def test_last_block_flag(orc):
    t = _text(2000)
    f, d = written(Frame([Raw(t[:1000]), Raw(t[1000:])], window_log=10))
    h = parse_header(f)["header_size"]
    g = bytearray(f); g[h] |= 1                                   # the first block claims to be the last
    bad(orc, bytes(g), d, "after the last block")
    g = bytearray(f); g[h + 3 + 1000] &= ~1                       # no block is the last
    bad(orc, bytes(g), d, "no last block|runs past")


def test_checksum_rules(orc):
    t = _text(700)
    f, d = written(Frame([Raw(t)], single_segment=True, checksum=True))
    assert ok(orc, f, d, checksum=True)
    bad(orc, f, d, "checksum flag", checksum=False)
    g = bytearray(f); g[-1] ^= 0x40
    bad(orc, bytes(g), d, "checksum does not match", checksum=True)
    f, d = written(Frame([Raw(t)], single_segment=True))
    bad(orc, f, d, "checksum flag", checksum=True)
