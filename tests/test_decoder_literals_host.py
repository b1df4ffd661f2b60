"""CPU tests of the decoder's literal path on the CPU build of the kernel source (tests/host_encoder.build_sim), whose
wrappers call the helpers by name: bit reader (zb_common.cuh), NCount reader (zb_decode.cu), Huffman weights, split
decode table and the 1- and 4-stream decoders (zb_entropy.cuh) -- against payloads written by the reference's
HUF_compress1X/4X (zstd/zstd.c:18193, :18207) and against FSE_readNCount (:3433).  The GPU parity tests cover the same
code inside the kernel; these run everywhere and fuzz harder."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import host_encoder

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libzstd_ref.so")
pytestmark = pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref is built from /root/reference (see oracle/Makefile)")
PAD = 64


@pytest.fixture(scope="module")
def libs():
    ours = host_encoder.build_sim()
    ref = C.CDLL(REF)
    for name in ("HUF_compress1X_repeat", "HUF_compress4X_repeat", "FSE_normalizeCount", "FSE_writeNCount", "FSE_readNCount"):
        getattr(ref, name).restype = C.c_size_t
    ref.FSE_isError.restype = C.c_uint
    return ours, ref


def _ref_huf(ref, data, four):
    """Literals payload (weights header + streams) as the reference writes it, or None when it declines."""
    n = len(data)
    dst = (C.c_ubyte * (n + 1024))()
    wk = (C.c_uint64 * 2048)()
    table = (C.c_size_t * 260)()
    repeat = C.c_int(0)
    fn = ref.HUF_compress4X_repeat if four else ref.HUF_compress1X_repeat
    r = fn(dst, n + 1024, data, n, 255, 11, wk, 8 * 2048, table, C.byref(repeat), 0)
    if ref.FSE_isError(C.c_size_t(r)) or r <= 1 or r >= n:
        return None
    return bytes(dst[:r])


def _decode(ours, payload, regen, single):
    buf = (C.c_ubyte * (len(payload) + 2 * PAD))()                 # the bit reader loads aligned words around the stream
    C.memmove(C.addressof(buf) + PAD, payload, len(payload))
    out = (C.c_ubyte * (regen + 2 * PAD))()
    used, tb = C.c_uint32(), C.c_uint32()
    ok = ours.t_literals_decode(C.cast(C.addressof(out) + PAD, C.POINTER(C.c_ubyte)), regen,
                                C.cast(C.addressof(buf) + PAD, C.POINTER(C.c_ubyte)), len(payload), int(single),
                                C.byref(used), C.byref(tb))
    guard_ok = bytes(out[:PAD]) == bytes(PAD) and bytes(out[PAD + regen:]) == bytes(PAD)      # nothing written outside dst
    return ok, bytes(out[PAD:PAD + regen]), tb.value, guard_ok


def _samples():
    rng = np.random.default_rng(21)
    text = open(__file__, "rb").read() * 8
    out = []
    for size in (12, 63, 255, 256, 257, 1000, 4096, 20000, 70000, 131072):
        out.append(text[:size])
        out.append(np.clip(rng.geometric(0.04, size), 0, 255).astype(np.uint8).tobytes())
        out.append(np.clip(rng.normal(120, 2.5, size), 0, 255).astype(np.uint8).tobytes())
        out.append((rng.integers(0, 4, size) * 60).astype(np.uint8).tobytes())
        out.append(np.where(rng.random(size) < 0.97, 32, rng.integers(0, 256, size)).astype(np.uint8).tobytes())
    return out


def test_reference_written_literals_decode_bit_exact(libs):
    ours, ref = libs
    done = {False: 0, True: 0}
    small_tables = 0
    for data in _samples():
        for four in (False, True):
            if four and len(data) < 256 or not four and len(data) > 70000:
                continue
            payload = _ref_huf(ref, data, four)
            if payload is None:
                continue
            ok, got, tb, guard_ok = _decode(ours, payload, len(data), single=not four)
            assert ok and got == data and guard_ok, (len(data), four)
            small_tables += tb < 2048
            done[four] += 1
    assert done[False] >= 15 and done[True] >= 20 and small_tables >= 10


def test_corrupt_literals_never_crash_or_overrun(libs):
    """Every single-byte corruption of a payload is either rejected or decoded inside the destination bounds."""
    ours, ref = libs
    rng = np.random.default_rng(22)
    rejected = accepted = 0
    for data in _samples()[5:25]:
        four = len(data) >= 256
        payload = _ref_huf(ref, data, four)
        if payload is None:
            continue
        for _ in range(40):
            bad = bytearray(payload)
            k = int(rng.integers(0, len(bad)))
            bad[k] ^= 1 << int(rng.integers(0, 8))
            ok, got, _, guard_ok = _decode(ours, bytes(bad), len(data), single=not four)
            assert guard_ok
            rejected += not ok
            accepted += bool(ok)
        # truncations
        for cut in (1, 2, len(payload) // 2):
            ok, _, _, guard_ok = _decode(ours, payload[:len(payload) - cut], len(data), single=not four)
            assert guard_ok
    assert rejected > 100        # most corruptions break the exact-consumption check of some stream


def test_ncount_reader_equals_the_reference(libs):
    """zb_read_ncount == FSE_readNCount on valid headers (norm, max symbol, log, bytes used) and on corrupted ones
    (same accept / reject decision; same result when accepted)."""
    ours, ref = libs
    rng = np.random.default_rng(23)
    valid = agree = 0
    for n_sym, total in ((36, 300), (53, 9000), (32, 2000), (29, 100), (16, 200)):
        for k in range(40):
            p = rng.geometric(0.3, total) - 1 if k % 2 else rng.integers(0, n_sym, total)
            count = np.bincount(np.clip(p, 0, n_sym - 1), minlength=n_sym).astype(np.uint32)
            max_sym = int(np.nonzero(count)[0].max())
            if np.count_nonzero(count) < 2:
                continue
            for log in (5, 6, 7, 9):
                if (1 << log) < np.count_nonzero(count):
                    continue
                norm = (C.c_short * 64)()
                r = ref.FSE_normalizeCount(norm, log, (C.c_uint * 64)(*count.tolist()), int(count.sum()), max_sym, 1)
                if ref.FSE_isError(C.c_size_t(r)):
                    continue
                buf = (C.c_ubyte * 512)()
                n = ref.FSE_writeNCount(buf, 512, norm, max_sym, log)
                # ample room after the header: at the very end of its input the reference's reader wraps its bit counter
                # (bitCount &= 31, zstd/zstd.c:3304) and may accept a header that runs past the end, which ours rejects
                hdr = bytes(buf[:n]) + bytes(64)
                for trial in range(4):
                    b = bytearray(hdr)
                    if trial:
                        b[int(rng.integers(0, n))] ^= 1 << int(rng.integers(0, 8))
                    src = (C.c_ubyte * len(b))(*b)
                    mine = (C.c_short * 256)(); ms = C.c_uint32(n_sym - 1); lg = C.c_uint32()
                    used = ours.t_read_ncount(mine, C.byref(ms), C.byref(lg), src, len(b))
                    theirs = (C.c_short * 256)(); rms = C.c_uint(n_sym - 1); rlg = C.c_uint()
                    rused = ref.FSE_readNCount(theirs, C.byref(rms), C.byref(rlg), src, len(b))
                    rerr = bool(ref.FSE_isError(C.c_size_t(rused)))
                    if not trial:
                        assert used == n and not rerr and rused == n
                        valid += 1
                    assert (used == 0) == rerr, (n_sym, log, trial, used, rused)
                    if used:
                        assert used == rused and ms.value == rms.value and lg.value == rlg.value
                        assert list(mine[:ms.value + 1]) == list(theirs[:rms.value + 1])
                        agree += 1
    assert valid > 200 and agree > valid


LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
LL_DEF = [4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1]
OF_DEF = [1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1]
ML_DEF = [1, 4, 3, 2, 2, 2, 2, 2, 2] + [1] * 37 + [-1] * 7


def test_sequence_decode_tables_equal_the_reference(libs):
    """zb_build_fse (our 4-byte cells: next state | bits | extra bits | symbol) holds the same state machine as the
    reference's ZSTD_buildFSETable (zstd/zstd.c:46118) for the predefined distributions and for random ones."""
    ours, ref = libs
    rng = np.random.default_rng(24)
    cases = [(0, LL_DEF, 6), (1, OF_DEF, 5), (2, ML_DEF, 6)]
    for kind, n_sym, maxlog in ((0, 36, 9), (1, 32, 8), (2, 53, 9)):
        for k in range(25):
            total = int(rng.integers(40, 20000))
            p = rng.geometric(0.2, total) - 1 if k % 2 else rng.integers(0, n_sym, total)
            count = np.bincount(np.clip(p, 0, n_sym - 1), minlength=n_sym).astype(np.uint32)
            max_sym = int(np.nonzero(count)[0].max())
            if np.count_nonzero(count) < 2:
                continue
            log = int(rng.integers(5, maxlog + 1))
            if (1 << log) < np.count_nonzero(count):
                continue
            norm = (C.c_short * 64)()
            r = ref.FSE_normalizeCount(norm, log, (C.c_uint * 64)(*count.tolist()), total, max_sym, 1)
            if not ref.FSE_isError(C.c_size_t(r)):
                cases.append((kind, list(norm[:max_sym + 1]), log))
    assert len(cases) > 40
    ident = (C.c_uint32 * 64)(*range(64))                      # baseValue := the symbol itself, so the reference cell names its symbol
    for kind, norm_l, log in cases:
        bits_l = LL_BITS if kind == 0 else (list(range(32)) if kind == 1 else ML_BITS)
        bits = (C.c_ubyte * 64)(*bits_l)
        size = 1 << log
        dt = (C.c_uint64 * (size + 1))()                       # ZSTD_seqSymbol is 8 bytes; dt[0] is the header
        wk = (C.c_uint32 * 512)()
        ref.ZSTD_buildFSETable(dt, (C.c_short * 64)(*norm_l), len(norm_l) - 1, ident, bits, log, wk, 2048, 0)
        raw = np.frombuffer(dt, dtype=np.uint8)[8:].reshape(size, 8)
        next_state = raw[:, 0:2].copy().view(np.uint16)[:, 0]
        add_bits, nb_bits = raw[:, 2], raw[:, 3]
        sym = raw[:, 4:8].copy().view(np.uint32)[:, 0]
        cells = (C.c_uint32 * size)()
        ours.t_build_fse(cells, (C.c_short * 64)(*norm_l), len(norm_l) - 1, log, kind)
        c = np.frombuffer(cells, dtype=np.uint32)
        assert ((c & 1023) == next_state).all() and (((c >> 10) & 15) == nb_bits).all()
        assert (((c >> 14) & 31) == add_bits).all() and ((c >> 19) == sym).all(), (kind, log)


def test_frame_header_parser_equals_the_reference(libs):
    """The device header parser (zb_parse_header) against ZSTD_getFrameHeader (zstd/zstd.c:43668) on headers the
    reference wrote, on headers our encoder writes, and on thousands of random mutations: same accept / need-more / reject
    decision, same fields when accepted."""
    ours, ref = libs
    ref.ZSTD_getFrameHeader.restype = C.c_size_t
    ref.ZSTD_isError.restype = C.c_uint
    from oracle import RefZstd
    rz = RefZstd()
    rng = np.random.default_rng(25)
    seeds = []
    for size in (0, 1, 255, 256, 65791, 65792, 200000, 3 << 20):
        data = bytes(size)
        for ck in (False, True):
            seeds.append((rz.compress(data, level=3, checksum=ck) + bytes(18))[:18])
            seeds.append((rz.compress(data, level=3, checksum=ck, content_size=False) + bytes(18))[:18])
    for did in (0, 9, 40000, 1123828263):
        for cs in (0, 1):
            out = (C.c_ubyte * 32)()
            n = ours.t_frame_header(out, 70000, 1, cs, did)
            seeds.append(bytes(out[:n]) + bytes(18 - n))
    accepted = rejected = short = 0
    for seed in seeds:
        for trial in range(120):
            b = bytearray(seed)
            if trial:
                for _ in range(int(rng.integers(1, 3))):
                    b[int(rng.integers(4 if trial % 4 else 0, 14))] = int(rng.integers(0, 256))
            n = len(b) if trial % 5 else int(rng.integers(0, len(b) + 1))
            src = (C.c_ubyte * 32)(*b)
            zfh = (C.c_uint64 * 8)()
            r = ref.ZSTD_getFrameHeader(zfh, src, n)
            out = (C.c_uint64 * 6)()
            ours.t_parse_header(src, n, out)
            status = out[5]
            if ref.ZSTD_isError(C.c_size_t(r)):
                assert status != 0, (bytes(b[:n]).hex(), r)
                rejected += 1
            elif r > 0:                                   # more input needed
                assert status == 72, (bytes(b[:n]).hex(), r, status)
                short += 1
            else:
                raw = np.frombuffer(zfh, dtype=np.uint8)
                fcs, wsize = int(raw[0:8].view(np.uint64)[0]), int(raw[8:16].view(np.uint64)[0])
                ftype, hsize, dict_id, cksum = (int(x) for x in raw[20:36].view(np.uint32))
                if ftype != 0:                             # skippable frame: handled by zb_skip_skippable, not by this parser
                    continue
                assert status == 0, (bytes(b[:n]).hex(), status)
                assert (out[0], out[2], out[3], out[4]) == (fcs, dict_id, hsize, cksum), bytes(b[:n]).hex()
                assert out[1] == wsize or (fcs == 0 and out[1] == 0), bytes(b[:n]).hex()
                accepted += 1
    assert accepted > 1500 and rejected > 50 and short > 100
