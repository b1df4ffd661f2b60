"""Hand-built frames (tests/crafted_frames.py, written by tests/frame_writer.py from RFC 8878) through every decode path
of the kernels' own source on the CPU.

First the writer is checked against the reference: for every case the reference regenerates what the writer's executor
predicts, the plain-C oracle traces the predicted (ll, ml, offset) list and per-block sequence counts, and every case the
executor calls malformed is rejected.  Then each case goes through the lane-per-frame kernel one frame at a time
(t_decode_frame), and through the whole batch pipeline on its three paths -- lane per frame, lane per block, lane per
block with pointer jumping -- with 7 or 8 warps, 3 or 32 frames per warp, crafted frames mixed with reference frames.
The rule: what the reference rejects every path rejects; what it accepts every path regenerates byte for byte with
status 0.  The cases with a `note` are invalid by RFC 8878 but accepted by the reference; every path rejects them."""
import ctypes as C
import os

import numpy as np
import pytest

import corpus
from tests import crafted_frames, host_encoder

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libzstd_ref.so")
pytestmark = pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref is built from /root/reference (see oracle/Makefile)")
PAD = 64

CASES = crafted_frames.catalogue()
BY_NAME = {c.name: c for c in CASES}
STREAMS = crafted_frames.stream_cases(np.random.default_rng(106))
DICT_REPS = crafted_frames.dict_rep_cases(np.random.default_rng(107))


@pytest.fixture(scope="module")
def ref():
    from oracle import RefZstd
    return RefZstd()


@pytest.fixture(scope="module")
def orc():
    from oracle import Oracle
    return Oracle()


@pytest.fixture(scope="module")
def dsim():
    L = host_encoder.build_sim()
    yield L
    L.t_set_block_path(0)


def _cap(c):
    return c.size


def test_catalogue_size():
    assert len(CASES) + len(STREAMS) + len(DICT_REPS) >= 150
    assert sum(c.expected is None for c in CASES) >= 40 and sum(c.expected is not None for c in CASES) >= 80


@pytest.mark.parametrize("name", [c.name for c in CASES + STREAMS + DICT_REPS])
def test_writer_agrees_with_the_reference(ref, orc, name):
    c = BY_NAME.get(name) or next(x for x in STREAMS + DICT_REPS if x.name == name)
    try:
        got = ref.decompress(c.frame, _cap(c) + (1 << 18), c.dict)
    except ref.Error:
        got = None
    if c.note:
        assert c.expected is None and got is not None, c.note
        return
    assert got == c.expected
    if c.expected is not None and not name.startswith("skippable"):
        _, _, seqs, counts = orc.trace(c.frame, len(c.expected) + 16, c.dict)
        assert (seqs, counts) == c.trace


def test_writer_checksum_is_xxh64(orc):
    from tests import frame_writer
    data = corpus.text_corpus(1 << 16).tobytes()
    for n in (0, 1, 3, 4, 7, 8, 31, 32, 33, 63, 64, 65, 1000, 65536):
        assert frame_writer.xxh64(data[:n]) == orc.xxh64(data[:n]), n


def _single(kern, c):
    src = (C.c_ubyte * (len(c.frame) + 2 * PAD))()
    C.memmove(C.addressof(src) + PAD, c.frame, len(c.frame))
    dbuf = (C.c_ubyte * (len(c.dict) + 2 * PAD))()
    if c.dict:
        C.memmove(C.addressof(dbuf) + PAD, c.dict, len(c.dict))
    cap = _cap(c)
    out = (C.c_ubyte * (cap + 2 * PAD))()
    out_n, nb, ns = C.c_uint64(0), C.c_uint32(0), C.c_uint32(0)
    rc = kern.t_decode_frame(C.addressof(src) + PAD, len(c.frame), (C.addressof(dbuf) + PAD) if c.dict else None, len(c.dict),
                             C.addressof(out) + PAD, cap, C.byref(out_n), C.byref(nb), C.byref(ns))
    assert bytes(out[:PAD]) == bytes(PAD) and bytes(out[PAD + cap:]) == bytes(PAD)
    return rc, bytes(out[PAD:PAD + out_n.value])


def test_one_lane(dsim):
    """The lane-per-frame kernel through its launcher, one frame per call: one busy lane in a warp.  (The content
    checksum is compared by zb_verify_checksums, which only the batch pipeline runs: the wrong checksum is checked on
    every path below.)"""
    for c in CASES + DICT_REPS:
        if c.name == "wrong_checksum":
            continue
        rc, got = _single(dsim, c)
        if c.expected is None:
            assert rc != 0, c.name
        else:
            assert rc == 0 and got == c.expected, c.name


def _batch(sim, frames, sizes, dct, gaps, warps, take, n_ctas=2):
    """(outputs, statuses) of one batch call; frame k starts gaps[k] bytes after the previous one ends."""
    parts, off, pos = [bytes(PAD)], [], PAD
    for f, g in zip(frames, gaps):
        parts.append(bytes(g))
        pos += g
        off.append(pos)
        parts.append(f)
        pos += len(f)
    parts.append(bytes(PAD))
    blob = b"".join(parts)
    off = np.array(off, dtype=np.uint64)
    ln = np.array([len(f) for f in frames], dtype=np.uint64)
    src = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
    dbuf = (C.c_ubyte * (len(dct) + 2 * PAD)).from_buffer_copy(bytes(PAD) + dct + bytes(PAD))
    cap = sum(sizes) + 64
    out = (C.c_ubyte * cap)()
    n = len(frames)
    oo = (C.c_uint64 * n)(); ol = (C.c_uint64 * n)(); st = (C.c_uint32 * n)()
    want = (C.c_uint64 * n)(*sizes)
    tot = sim.t_decompress_batch(C.addressof(src), off.ctypes.data, ln.ctypes.data, n, (C.addressof(dbuf) + PAD) if dct else None, len(dct),
                                 n_ctas, warps, take, C.addressof(out), cap, C.addressof(oo), C.addressof(ol), C.addressof(st), C.addressof(want), 0, None)
    if tot < 0:
        return None, None
    return [bytes(out[oo[i]:oo[i] + ol[i]]) for i in range(n)], list(st)


def _check(cases, outs, st, tag):
    for c, got, s in zip(cases, outs, st):
        if c.expected is None:
            assert s != 0, (tag, c.name)
        else:
            assert s == 0 and got == c.expected, (tag, c.name, s)


def _ref_frames(ref, k):
    text = corpus.text_corpus(1 << 20)
    segs = [bytes(text[i * 7919:i * 7919 + 300 + 611 * i]) for i in range(k)]
    return [crafted_frames.Case("ref%d" % i, ref.compress(s, level=1 + i % 5, checksum=bool(i & 1)), s, None) for i, s in enumerate(segs)]


PATHS = {"lane-per-frame": 0, "lane-per-block": 1, "lane-per-block+pointer-jumping": 2}


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("warps,take", [(8, 32), (7, 3)])
def test_every_path(dsim, ref, path, warps, take):
    """All cases in a batch per dictionary, crafted and reference frames interleaved so that they share warps."""
    dsim.t_set_block_path(PATHS[path])
    rng = np.random.default_rng(7 + take)
    groups = {}
    for c in CASES:
        groups.setdefault(c.dict, []).append(c)
    for dct, cases in groups.items():
        batch = list(cases)
        if not dct:
            refs = _ref_frames(ref, 12)
            for i, r in enumerate(refs):
                batch.insert((i * 7) % len(batch), r)
        gaps = [int(g) for g in rng.integers(0, 16, len(batch))]
        outs, st = _batch(dsim, [c.frame for c in batch], [_cap(c) for c in batch], dct, gaps, warps, take)
        _check(batch, outs, st, path)
    dsim.t_set_block_path(0)


@pytest.mark.parametrize("path", list(PATHS))
def test_short_streams_at_every_phase(dsim, path):
    """Sequence streams of 1, 2, 15, 16, 17 and 63 bytes at every 16-byte phase of the batch blob (the ring bit reader's
    aligned cover), 96 frames, 32 per warp, so that every lane of a warp holds one."""
    dsim.t_set_block_path(PATHS[path])
    for shift in (0, 5, 11):
        gaps = [(shift + 3 * i) % 16 for i in range(len(STREAMS))]
        outs, st = _batch(dsim, [c.frame for c in STREAMS], [_cap(c) for c in STREAMS], b"", gaps, 8, 32, n_ctas=1)
        _check(STREAMS, outs, st, (path, shift))
    dsim.t_set_block_path(0)


@pytest.mark.parametrize("path", list(PATHS))
def test_dictionary_repcodes_at_the_content_size(dsim, path):
    """Repcodes equal to the dictionary content size load and reach its first byte; one more is refused at load."""
    dsim.t_set_block_path(PATHS[path])
    for c in DICT_REPS:
        outs, st = _batch(dsim, [c.frame], [_cap(c)], c.dict, [0], 8, 32, n_ctas=1)
        if c.expected is None:
            assert st is None or st[0] != 0, c.name
        else:
            assert st == [0] and outs[0] == c.expected, c.name
    dsim.t_set_block_path(0)


@pytest.mark.parametrize("path", list(PATHS))
def test_offsets_from_2_31_are_never_repcodes(dsim, path):
    """On the block path bit 31 of a history entry marks a symbolic repcode.  OF code 31 with extra bits >= 3 decodes to a
    concrete offset >= 2^31: it must be rejected, not resolved as 'entry repcode k minus d'."""
    dsim.t_set_block_path(PATHS[path])
    cases = [c for c in CASES if c.name.startswith(("of29", "of30", "of31", "rep0_minus1_is_zero"))]
    assert len(cases) == 31
    for c in cases:
        outs, st = _batch(dsim, [c.frame], [_cap(c)], b"", [0], 7, 3, n_ctas=1)
        assert st[0] != 0, (path, c.name)
    dsim.t_set_block_path(0)


def test_sequences_fill_the_window_exactly_at_every_alignment():
    """The decoder reads a sequence's offset, ML + LL and state bits without refilling when they fit its bit window
    (`slow` in zb_seq_block).  At every 16-byte alignment of the stream, some valid case has a sequence whose bits equal
    the window exactly and one that needs exactly one bit more (frame_writer.window_margins restates the window)."""
    from tests import frame_writer
    for skew in range(16):
        margins = [m for c in CASES if c.expected is not None for plan in c.bitplans for m in frame_writer.window_margins(plan, skew)]
        assert 0 in margins and 1 in margins, skew


def _scan_totals(dsim, frames):
    blob = bytes(PAD) + b"".join(frames) + bytes(PAD)
    off = (np.cumsum([0] + [len(f) for f in frames[:-1]]) + PAD).astype(np.uint64)
    ln = np.array([len(f) for f in frames], dtype=np.uint64)
    src = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
    tot = (C.c_uint64 * 6)()
    dsim.t_scan_totals(C.addressof(src), off.ctypes.data, ln.ctypes.data, len(frames), C.addressof(tot))
    return list(tot)


def test_far_windows_are_flagged_by_both_frame_scans(dsim):
    """totals[5] keeps a batch off the block path (zb_api.cu) when one of its frames has a window of 2 GiB - 128 MiB or
    more.  Frames above ZB_SCAN_BIG (24 KB in this build) are scanned by zb_scan_frames_big, the others by zb_scan_frames;
    both must set the flag, from a window descriptor or from a single-segment content size."""
    from tests import frame_writer as fw
    raw = bytes(range(256)) * 40                                           # 10240 bytes a block
    small, big = [fw.Raw(raw)], [fw.Raw(raw)] * 3                          # big: more than 24 KB compressed

    def frame(blocks, **kw):
        return fw.write(fw.Frame(blocks, **kw))[0]
    near = frame(small, window_log=30, window_mantissa=6)                  # 1.75 GiB: below the limit
    for blocks in (small, big):
        for kw in ({"window_log": 30, "window_mantissa": 7}, {"window_log": 31, "window_mantissa": 3},
                   {"single_segment": True, "content_size": (1 << 31) - (1 << 27), "fcs_bytes": 4}):
            far = frame(blocks, **kw)
            assert _scan_totals(dsim, [far])[5] == 1, (len(blocks), kw)
            assert _scan_totals(dsim, [frame(small), near, far, frame(big)])[5] == 1, (len(blocks), kw)
    assert _scan_totals(dsim, [frame(small), near, frame(big, window_log=27), frame(big, window_log=30, window_mantissa=6)])[5] == 0
