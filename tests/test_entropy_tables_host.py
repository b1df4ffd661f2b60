"""The entropy decoder's table builders against cells kept in a fixture: every FSE and Huffman-weights table of the crafted
catalogue, the golden frames and the golden dictionary, plus random FSE tables of logs 5-9 with and without -1 symbols.

tests/golden/entropy_tables.npz holds each table's input (normalized counts, or a Huffman tree description) and the cells
the builders wrote when the fixture was made: the 16-bit cells of the entropy kernels and the 32-bit cells of the
predefined and dictionary tables for FSE; for Huffman, the lane workspace (nibble weights and the weight stream's 64-cell
FSE table), the weights' counts, log and symbol count, and the split decode table.  The builders run here on the CPU build
of zb_decode.cu (tests/simt_tables.cpp), so the cells they must reproduce bit for bit are the ones the device reads.

`python -m tests.test_entropy_tables_host --write` remakes the fixture from the current builders.
"""
import ctypes as C
import glob
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from tests import host_encoder  # noqa: E402

FIXTURE = os.path.join(HERE, "golden", "entropy_tables.npz")
SRC = os.path.join(HERE, "simt_tables.cpp")
LIB = os.path.join(HERE, "_build", "libztables.so")
KINDS = ((0, 35, 9), (1, 31, 8), (2, 52, 9))                 # LL, OF, ML: kind, largest symbol, largest log


def _lib():
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    cmd = (["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-I" + host_encoder.CSRC, "-I" + HERE]
           + host_encoder.SIM_FLAGS + [SRC])
    h = hashlib.sha256(" ".join(cmd).encode())
    for f in sorted(glob.glob(os.path.join(host_encoder.CSRC, "*.cu*"))) + [SRC, os.path.join(HERE, "simt.h")]:
        h.update(open(f, "rb").read())
    stamp = LIB + ".sha256"
    if not (os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == h.hexdigest()):
        tmp = "%s.%d.tmp" % (LIB, os.getpid())
        subprocess.check_call(cmd + ["-o", tmp])
        os.replace(tmp, LIB)
        open(stamp, "w").write(h.hexdigest())
    return C.CDLL(LIB)


# ---- the builders
def _fse(L, norm, log, kind):
    nn = (C.c_short * 64)(*norm)
    c16 = np.zeros(1 << log, dtype=np.uint16)
    c32 = np.zeros(1 << log, dtype=np.uint32)
    L.tt_build_fse(nn, C.c_uint32(len(norm) - 1), C.c_uint32(log), C.c_int(kind), c16.ctypes.data_as(C.c_void_p), c32.ctypes.data_as(C.c_void_p))
    return c16, c32


def _huf(L, desc):
    """(used, ws[256], rank[13], log, nsym, split table); the table only when the description is valid."""
    buf = (C.c_ubyte * (len(desc) + 64)).from_buffer_copy(bytes(desc) + bytes(64))
    ws = (C.c_ubyte * 256)(); rank = (C.c_uint32 * 13)(); log = C.c_uint32(); nsym = C.c_uint32()
    L.tt_huf_weights.restype = C.c_uint32
    used = L.tt_huf_weights(buf, C.c_uint32(len(desc)), ws, rank, C.byref(log), C.byref(nsym))
    cells = np.zeros(4096 + 8, dtype=np.uint16)
    if used:
        L.tt_huf_fill.restype = C.c_uint32
        cells = cells[:L.tt_huf_fill(ws, log, nsym, rank, cells.ctypes.data_as(C.c_void_p)) // 2]
    return (used, np.frombuffer(bytes(ws), dtype=np.uint8), np.array(rank[:], dtype=np.uint32) if used else np.zeros(13, np.uint32),
            log.value if used else 0, nsym.value if used else 0, cells)


# ---- the tables of the catalogue, the golden frames and the dictionary (used only to write the fixture)
def _ncount(L, buf, pos, max_sym):
    norm = (C.c_short * 64)(); ms = C.c_uint32(max_sym); log = C.c_uint32()
    b = (C.c_ubyte * (len(buf) - pos + 64)).from_buffer_copy(bytes(buf[pos:]) + bytes(64))
    L.tt_read_ncount.restype = C.c_uint32
    used = L.tt_read_ncount(norm, C.byref(ms), C.byref(log), b, C.c_uint32(len(buf) - pos))
    return used, list(norm[:ms.value + 1]), log.value


def _huf_desc(buf, pos):
    hb = buf[pos]
    return bytes(buf[pos:pos + 1 + (hb if hb < 128 else (hb - 127 + 1) // 2)])


def _walk_frame(L, f, fse, huf):
    """Collect the tables one frame defines; stops quietly where the frame is malformed."""
    from tests import frame_check
    try:
        p = frame_check.parse_header(f)["header_size"]
    except Exception:
        return
    while p + 3 <= len(f):
        bh = int.from_bytes(f[p:p + 3], "little"); p += 3
        last, kind, size = bh & 1, (bh >> 1) & 3, bh >> 3
        body = f[p:p + (1 if kind == 1 else size)]
        p += 1 if kind == 1 else size
        if kind == 2 and len(body) == size and size >= 1:
            b0 = body[0]; lt, form = b0 & 3, (b0 >> 2) & 3
            if lt < 2:
                hdr = (1, 2, 1, 3)[form]
                regen = frame_check._literals_regen(body)
                q = hdr + (regen if lt == 0 else 1)
            else:
                hdr, width = {0: (3, 10), 1: (3, 10), 2: (4, 14), 3: (5, 18)}[form]
                csize = (int.from_bytes(body[:hdr], "little") >> (4 + width)) & ((1 << width) - 1)
                if lt == 2 and hdr < len(body):
                    huf.append(_huf_desc(body, hdr))
                q = hdr + csize
            if q < len(body):
                nseq = body[q]; q += 1
                if nseq >= 0xFF:
                    q += 2
                elif nseq >= 0x80:
                    q += 1
                if nseq and q < len(body):
                    modes = body[q]; q += 1
                    for (k, ms, lmax), m in zip(KINDS, (modes >> 6, (modes >> 4) & 3, (modes >> 2) & 3)):
                        if m == 1:
                            q += 1
                        elif m == 2:
                            used, norm, log = _ncount(L, body, q, ms)
                            if not used or log > lmax:
                                break
                            fse.append((k, log, norm)); q += used
        if last or kind == 3:
            break


def _walk_dict(L, d, fse, huf):
    if len(d) < 8 or int.from_bytes(d[:4], "little") != 0xEC30A437:
        return
    p = 8
    desc = _huf_desc(d, p); huf.append(desc); p += len(desc)
    for k in (1, 2, 0):                                           # offsets, match lengths, literal lengths
        used, norm, log = _ncount(L, d, p, KINDS[k][1])
        if not used:
            return
        fse.append((k, log, norm)); p += used


def _random_norm(rng, nsym, log, minus1):
    """Normalized counts over nsym symbols summing to 2^log, `minus1` of them -1."""
    norm = [0] * nsym
    syms = rng.permutation(nsym)
    for s in syms[:minus1]:
        norm[int(s)] = -1
    room = min(nsym, 1 << log) - minus1                            # symbols that can take a cell of their own
    live = [int(s) for s in syms[minus1:minus1 + int(rng.integers(1, room + 1))]]
    for s in live:
        norm[s] = 1
    for _ in range((1 << log) - minus1 - len(live)):
        norm[live[int(rng.integers(0, len(live)))]] += 1
    assert sum(abs(c) for c in norm) == 1 << log
    while norm[-1] == 0:
        norm.pop()
    return norm


def _collect(L, W):
    from tests import crafted_frames, helpers
    fse, huf = [], []
    for c in crafted_frames.catalogue():
        _walk_frame(L, bytes(c.frame), fse, huf)
        _walk_dict(L, bytes(c.dict), fse, huf)
    for name, frame, raw, dct in helpers.golden_vectors():
        p = 0
        while p + 8 <= len(frame):
            magic = int.from_bytes(frame[p:p + 4], "little")
            if magic & 0xFFFFFFF0 == 0x184D2A50:
                p += 8 + int.from_bytes(frame[p + 4:p + 8], "little")
                continue
            _walk_frame(L, frame[p:], fse, huf)
            break
    _walk_dict(L, open(os.path.join(HERE, "golden", "dict.bin"), "rb").read(), fse, huf)
    rng = np.random.default_rng(20261017)
    for k, ms, _ in KINDS:
        for log in range(5, 10):
            for minus1 in (0, 1, 5):
                for _ in range(2):
                    fse.append((k, log, _random_norm(rng, ms + 1, log, minus1)))
    seen, out = set(), []
    for t in fse:
        key = (t[0], t[1], tuple(t[2]))
        if key not in seen:
            seen.add(key); out.append(t)
    hs = list(dict.fromkeys(huf + _weight_headers_at_symbol_15(W)))
    return out, hs


def _weight_headers_at_symbol_15(W):
    """FSE-coded weight descriptions whose normalized counts reach past symbol 15 (a count on 16, a -1 on 16, a run of
    zeros across 15: every decoder must reject them) or end exactly at 15.  W: the CPU build's NCount writer."""
    out = []
    for log, norm in ((5, [8, 8, 8, 4] + [0] * 12 + [4]), (5, [10, 10, 6] + [0] * 17 + [6]),
                      (5, [16, 8, 7] + [0] * 13 + [-1]), (6, [4] * 16), (6, [39, 8, 4, 4, 4, 2, 1, -1] + [0] * 7 + [1])):
        buf = (C.c_ubyte * 64)()
        n = W.t_write_ncount(buf, (C.c_short * 64)(*norm), C.c_uint32(len(norm) - 1), C.c_uint32(log))
        body = bytes(buf[:n]) + bytes([0x5A, 0xC3, 0x81])
        out.append(bytes([len(body)]) + body)
    return out


def write_fixture(W=None):
    L = _lib()
    fse, huf = _collect(L, W or host_encoder.build_sim())
    arrays = {"fse_kind": np.array([t[0] for t in fse], np.int32), "fse_log": np.array([t[1] for t in fse], np.int32),
              "fse_norm": np.array([t[2] + [0] * (64 - len(t[2])) for t in fse], np.int16),
              "fse_nsym": np.array([len(t[2]) for t in fse], np.int32)}
    c16, c32 = zip(*(_fse(L, t[2], t[1], t[0]) for t in fse))
    arrays["fse_cells16"] = np.concatenate(c16); arrays["fse_cells32"] = np.concatenate(c32)
    arrays["huf_desc"] = np.frombuffer(b"".join(huf), np.uint8)
    arrays["huf_len"] = np.array([len(h) for h in huf], np.int32)
    res = [_huf(L, h) for h in huf]
    arrays["huf_used"] = np.array([r[0] for r in res], np.uint32)
    arrays["huf_ws"] = np.stack([r[1] for r in res]); arrays["huf_rank"] = np.stack([r[2] for r in res])
    arrays["huf_log"] = np.array([r[3] for r in res], np.uint32); arrays["huf_nsym"] = np.array([r[4] for r in res], np.uint32)
    arrays["huf_cells"] = np.concatenate([r[5] for r in res if r[0]])
    np.savez_compressed(FIXTURE, **arrays)
    return len(fse), len(huf)


@pytest.fixture(scope="module")
def tables():
    return _lib(), np.load(FIXTURE)


def test_fixture_covers_logs_and_low_probability_symbols(tables):
    _, F = tables
    logs, nsym = F["fse_log"], F["fse_nsym"]
    minus1 = np.array([(F["fse_norm"][i][:nsym[i]] == -1).any() for i in range(len(logs))])
    for log in range(5, 10):
        assert (minus1 & (logs == log)).any() and (~minus1 & (logs == log)).any(), log
    assert (F["huf_used"] > 0).sum() >= 10 and (F["huf_used"] == 0).sum() >= 3          # valid, and rejected past symbol 15
    assert any(F["huf_desc"][o] < 128 for o in np.cumsum(np.concatenate([[0], F["huf_len"][:-1]])))     # FSE-coded weights


def test_fse_cells_match_fixture(tables):
    L, F = tables
    o = 0
    for i in range(len(F["fse_log"])):
        log, n = int(F["fse_log"][i]), int(F["fse_nsym"][i])
        c16, c32 = _fse(L, [int(v) for v in F["fse_norm"][i][:n]], log, int(F["fse_kind"][i]))
        assert np.array_equal(c16, F["fse_cells16"][o:o + (1 << log)]), ("16-bit cells", i, log)
        assert np.array_equal(c32, F["fse_cells32"][o:o + (1 << log)]), ("32-bit cells", i, log)
        o += 1 << log
    assert o == len(F["fse_cells16"])


def test_huffman_weights_and_cells_match_fixture(tables):
    L, F = tables
    o = oc = 0
    for i, n in enumerate(F["huf_len"]):
        used, ws, rank, log, nsym, cells = _huf(L, F["huf_desc"][o:o + n].tobytes())
        o += n
        assert used == F["huf_used"][i], i
        if not used:
            continue
        assert np.array_equal(ws, F["huf_ws"][i]), ("workspace", i)
        assert np.array_equal(rank, F["huf_rank"][i]) and log == F["huf_log"][i] and nsym == F["huf_nsym"][i], i
        assert np.array_equal(cells, F["huf_cells"][oc:oc + len(cells)]), ("decode table", i)
        oc += len(cells)
    assert oc == len(F["huf_cells"])


if __name__ == "__main__":
    if "--write" in sys.argv:
        print("fixture: %d FSE tables, %d Huffman descriptions" % write_fixture())
