"""CPU known-answer tests of the encoder's entropy-table code against the reference's own functions.

tests/host_encoder.build_sim() compiles python_zstandard_b200/csrc/zb_encode.cu whole for the host, and its wrappers
call the kernel's serial helpers (NCount writer, CTable builder, normalisation, table choice, Huffman code + weight
header) by name; oracle/_ref/libzstd_ref.so is the unmodified reference (zstd/zstd.c) and exports FSE_normalizeCount
(:16402), FSE_writeNCount (:16267), FSE_readNCount (:3433), FSE_buildCTable_wksp (:16005), HUF_buildCTable_wksp
(:17513) and HUF_readStats (:3448).  Bit-exact where the format leaves no freedom (NCount bytes, CTable cells,
weight headers that decode to our code lengths); within a stated cost margin where it does (normalisation,
length-limited Huffman)."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from tests import host_encoder

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libzstd_ref.so")
pytestmark = pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref is built from /root/reference (see oracle/Makefile)")

LL_DEF = [4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1]


@pytest.fixture(scope="module")
def libs():
    ours = host_encoder.build_sim()
    ref = C.CDLL(REF)
    for name in ("FSE_normalizeCount", "FSE_writeNCount", "FSE_readNCount", "FSE_buildCTable_wksp", "HUF_buildCTable_wksp",
                 "HUF_readStats"):
        getattr(ref, name).restype = C.c_size_t
    ref.FSE_isError.restype = C.c_uint
    ref.FSE_optimalTableLog.restype = C.c_uint
    ref.HUF_getNbBitsFromCTable.restype = C.c_uint32
    return ours, ref


def _histograms(rng, n_sym, total, kinds=40):
    """Sequence-code-like histograms: geometric, flat, one dominant symbol, sparse."""
    out = []
    for k in range(kinds):
        shape = k % 4
        if shape == 0:
            p = rng.geometric(0.25, total) - 1
        elif shape == 1:
            p = rng.integers(0, n_sym, total)
        elif shape == 2:
            p = np.where(rng.random(total) < 0.9, 3, rng.integers(0, n_sym, total))
        else:
            p = rng.choice(rng.choice(n_sym, 5, replace=False), total)
        p = np.clip(p, 0, n_sym - 1)
        out.append(np.bincount(p, minlength=n_sym).astype(np.uint32))
    return out


def _cost_bits(count, norm, log):
    bits = 0.0
    for c, n in zip(count, norm):
        if c:
            assert n != 0
            bits += c * (log - math.log2(1 if n == -1 else n))
    return bits


def test_ncount_writer_is_byte_exact(libs):
    """ze_write_ncount == FSE_writeNCount on the reference's own normalisations, and the bytes read back to the norm."""
    ours, ref = libs
    rng = np.random.default_rng(5)
    checked = 0
    for n_sym, total in ((36, 300), (32, 300), (53, 9000), (36, 40000), (29, 64)):
        for count in _histograms(rng, n_sym, total):
            max_sym = int(np.nonzero(count)[0].max())
            if np.count_nonzero(count) < 2:
                continue
            for log in (5, 6, 8, 9):
                if (1 << log) < np.count_nonzero(count):
                    continue
                norm = (C.c_short * 64)()
                cnt = (C.c_uint * 64)(*count.tolist())
                r = ref.FSE_normalizeCount(norm, log, cnt, int(count.sum()), max_sym, 1)
                if ref.FSE_isError(C.c_size_t(r)):
                    continue
                buf_ref = (C.c_ubyte * 512)()
                n_ref = ref.FSE_writeNCount(buf_ref, 512, norm, max_sym, log)
                assert not ref.FSE_isError(C.c_size_t(n_ref))
                buf = (C.c_ubyte * 512)()
                n = ours.t_write_ncount(buf, norm, max_sym, log)
                assert n == n_ref and bytes(buf[:n]) == bytes(buf_ref[:n_ref]), (n_sym, total, log)
                back = (C.c_short * 64)(); ms = C.c_uint(63); lg = C.c_uint(0)
                used = ref.FSE_readNCount(back, C.byref(ms), C.byref(lg), buf, n)
                assert used == n and lg.value == log and ms.value == max_sym and list(back[:max_sym + 1]) == list(norm[:max_sym + 1])
                checked += 1
    assert checked > 300


def test_ctable_cells_equal_the_reference(libs):
    """ze_build_ctable fills the same state table and per-symbol transforms as FSE_buildCTable_wksp (incl. -1 counts)."""
    ours, ref = libs
    rng = np.random.default_rng(6)
    cases = [(list(LL_DEF), 35, 6)]
    for n_sym, total in ((36, 500), (53, 5000), (32, 200)):
        for count in _histograms(rng, n_sym, total, kinds=12):
            max_sym = int(np.nonzero(count)[0].max())
            if np.count_nonzero(count) < 2:
                continue
            for log in (5, 7, 9):
                norm = (C.c_short * 64)()
                r = ref.FSE_normalizeCount(norm, log, (C.c_uint * 64)(*count.tolist()), int(count.sum()), max_sym, 1)
                if not ref.FSE_isError(C.c_size_t(r)):
                    cases.append((list(norm[:max_sym + 1]), max_sym, log))
    for norm_l, max_sym, log in cases:
        norm = (C.c_short * 64)(*norm_l)
        size = 1 << log
        ct = (C.c_uint32 * (1 + size // 2 + 2 * 64 + 8))()
        wk = (C.c_uint32 * 1024)()
        assert not ref.FSE_isError(C.c_size_t(ref.FSE_buildCTable_wksp(ct, norm, max_sym, log, wk, 4096)))
        raw = np.frombuffer(ct, dtype=np.uint8)
        ref_state = raw[4:4 + 2 * size].view(np.uint16)
        tt = raw[4 + 2 * size:4 + 2 * size + 8 * (max_sym + 1)].view(np.int32).reshape(-1, 2)      # {deltaFindState, deltaNbBits}
        state = (C.c_uint16 * 512)(); dnb = (C.c_int * 64)(); dfs = (C.c_int * 64)()
        ours.t_build_ctable(norm, max_sym, log, state, dnb, dfs)
        assert list(state[:size]) == ref_state.tolist()
        for s in range(max_sym + 1):
            if norm_l[s] != 0:          # absent symbols are never encoded; the reference leaves a debug value there
                assert (dfs[s], dnb[s]) == (int(tt[s, 0]), int(tt[s, 1])), (s, norm_l[s], log)


def test_normalisation_is_valid_and_close_to_the_reference(libs):
    """Our rounding rule differs from FSE_normalizeCount's; the result must be a valid distribution and cost at most
    1 % more bits than the reference's on sequence-like histograms."""
    ours, ref = libs
    rng = np.random.default_rng(7)
    worst = 0.0
    for n_sym, total in ((36, 300), (53, 9000), (32, 2000), (36, 60000)):
        for count in _histograms(rng, n_sym, total):
            max_sym = int(np.nonzero(count)[0].max())
            present = int(np.count_nonzero(count))
            if present < 2:
                continue
            # at the table log the encoder uses for this histogram (FSE_optimalTableLog, zstd/zstd.c:16308, restated in
            # ze_make_table); far smaller logs, where rare symbols fill the table, cost us up to 17 % and are never chosen
            for log in sorted({int(ref.FSE_optimalTableLog(9, int(count.sum()), max_sym)), 9}):
                if (1 << log) < 2 * present:
                    continue
                cnt = (C.c_uint * 64)(*count.tolist())
                mine = (C.c_short * 64)()
                if not ours.t_normalize(mine, cnt, max_sym, int(count.sum()), log):
                    continue
                m = list(mine[:max_sym + 1])
                assert sum(m) == 1 << log and all((v >= 1) == (c > 0) for v, c in zip(m, count[:max_sym + 1]))
                theirs = (C.c_short * 64)()
                r = ref.FSE_normalizeCount(theirs, log, cnt, int(count.sum()), max_sym, 0)
                if ref.FSE_isError(C.c_size_t(r)):
                    continue
                a, b = _cost_bits(count, m, log), _cost_bits(count, list(theirs[:max_sym + 1]), log)
                worst = max(worst, a / b - 1.0)
                # the kernel's own cost estimate agrees with the exact entropy sum
                assert abs(ours.t_cost(cnt, mine, max_sym, log) - a) <= 2 + a * 1e-3
    assert worst <= 0.01, worst


def test_table_choice_modes(libs):
    """ze_make_table: one symbol -> RLE; few sequences -> predefined; enough skewed sequences -> compressed with a header
    that the reference reads back."""
    ours, ref = libs
    mode, log, hb = C.c_uint32(), C.c_uint32(), C.c_uint32()
    hdr = (C.c_ubyte * 64)()
    defn = (C.c_short * 36)(*LL_DEF)
    count = (C.c_uint * 64)(); count[7] = 50
    ours.t_make_table(count, 35, 50, 9, 6, defn, 35, C.byref(mode), C.byref(log), C.byref(hb), hdr)
    assert (mode.value, hb.value, hdr[0]) == (1, 1, 7)
    count = (C.c_uint * 64)(); count[0] = 5; count[3] = 4; count[9] = 3
    ours.t_make_table(count, 35, 12, 9, 6, defn, 35, C.byref(mode), C.byref(log), C.byref(hb), hdr)
    assert (mode.value, hb.value, log.value) == (0, 0, 6)
    rng = np.random.default_rng(8)
    c = np.bincount(np.clip(rng.geometric(0.5, 4000) - 1, 0, 35), minlength=36).astype(np.uint32)
    count = (C.c_uint * 64)(*c.tolist())
    ours.t_make_table(count, 35, 4000, 9, 6, defn, 35, C.byref(mode), C.byref(log), C.byref(hb), hdr)
    assert mode.value == 2 and 5 <= log.value <= 9 and hb.value > 0
    back = (C.c_short * 64)(); ms = C.c_uint(35); lg = C.c_uint(0)
    used = ref.FSE_readNCount(back, C.byref(ms), C.byref(lg), hdr, hb.value)
    assert used == hb.value and lg.value == log.value and sum(abs(v) for v in back[:ms.value + 1]) == 1 << log.value


def test_huffman_code_and_weight_header(libs):
    """ze_huf_build: complete prefix code, <= 11 bits, canonical values; cost within 1 % of HUF_buildCTable_wksp's;
    ze_huf_write_table decodes through HUF_readStats to exactly our code lengths."""
    ours, ref = libs
    rng = np.random.default_rng(9)
    text = open(__file__, "rb").read()
    samples = [np.frombuffer(text, dtype=np.uint8), np.frombuffer(text[:700], dtype=np.uint8),
               rng.integers(0, 256, 20000).astype(np.uint8), np.clip(rng.geometric(0.08, 30000), 0, 255).astype(np.uint8),
               np.clip(rng.normal(100, 3, 5000), 0, 255).astype(np.uint8),
               np.concatenate([np.full(60000, 65, np.uint8), np.arange(256, dtype=np.uint8)])]      # forces the depth limit
    worst = 0.0
    for data in samples:
        count = np.bincount(data, minlength=256).astype(np.uint32)
        cnt = (C.c_uint * 256)(*count.tolist())
        nb = (C.c_ubyte * 256)(); code = (C.c_uint16 * 256)(); ms = C.c_uint32(); lg = C.c_uint32()
        assert ours.t_huf_build(cnt, nb, code, C.byref(ms), C.byref(lg))
        lens = np.array(nb[:], dtype=np.int64)
        assert lg.value <= 11 and lens.max() == lg.value and ((lens > 0) == (count > 0)).all()
        assert sum(2.0 ** -int(l) for l in lens if l) == 1.0                      # complete (Kraft equality)
        codes = {}
        for s in range(256):
            if lens[s]:
                assert code[s] < (1 << lens[s])
                codes[(int(lens[s]), code[s])] = s
        assert len(codes) == int((lens > 0).sum())                                 # distinct values per length
        # cost against the reference's length-limited code
        tree = (C.c_size_t * 260)(); wk = (C.c_uint32 * 2048)()
        r = ref.HUF_buildCTable_wksp(tree, cnt, int(ms.value), 11, wk, 4 * 2048)
        assert not ref.FSE_isError(C.c_size_t(r))
        ref_bits = sum(int(count[s]) * ref.HUF_getNbBitsFromCTable(tree, s) for s in range(256))
        mine_bits = int((count.astype(np.int64) * lens).sum())
        worst = max(worst, mine_bits / ref_bits - 1.0)
        # the weight header reads back to our lengths
        out = (C.c_ubyte * 512)()
        tb = ours.t_huf_write_table(cnt, out)
        if tb:
            w = (C.c_ubyte * 256)(); rank = (C.c_uint32 * 16)(); nsym = C.c_uint32(); tlog = C.c_uint32()
            used = ref.HUF_readStats(w, 256, rank, C.byref(nsym), C.byref(tlog), out, tb)
            assert used == tb and tlog.value == lg.value and nsym.value == ms.value + 1
            got = [tlog.value + 1 - w[s] if w[s] else 0 for s in range(nsym.value)]
            assert got == lens[:nsym.value].tolist()
    assert worst <= 0.01, worst


def test_split_huffman_decode_table_equals_the_full_table(libs):
    """The decoder keeps full-resolution cells only for codes longer than 8 bits (zb_entropy.cuh).  For every code our
    encoder can emit, every index of the reference-shaped full table must read the same cell through the split table."""
    ours, ref = libs
    rng = np.random.default_rng(10)
    text = open(__file__, "rb").read()
    samples = [np.frombuffer(text, dtype=np.uint8), np.frombuffer(text[:900], dtype=np.uint8),
               np.clip(rng.geometric(0.05, 50000), 0, 255).astype(np.uint8), rng.integers(0, 256, 70000).astype(np.uint8),
               np.concatenate([np.full(60000, 65, np.uint8), np.arange(256, dtype=np.uint8)]),
               np.concatenate([np.full(3000, 7, np.uint8), np.full(40, 9, np.uint8), np.arange(20, dtype=np.uint8)])]
    saw_split = False
    for data in samples:
        count = np.bincount(data, minlength=256).astype(np.uint32)
        nb = (C.c_ubyte * 256)(); code = (C.c_uint16 * 256)(); ms = C.c_uint32(); lg = C.c_uint32()
        assert ours.t_huf_build((C.c_uint * 256)(*count.tolist()), nb, code, C.byref(ms), C.byref(lg))
        log, nsym = lg.value, ms.value + 1
        ws = (C.c_ubyte * 128)(); rank = (C.c_uint32 * 13)()
        for s in range(nsym):
            w = log + 1 - nb[s] if nb[s] else 0
            ws[s >> 1] |= w << ((s & 1) * 4)
            rank[w] += 1 if w else 0
        full = (C.c_uint16 * 4096)(); split = (C.c_uint16 * 4096)()
        ours.t_huf_full(ws, log, nsym, rank, full)
        shift, T, base, nbytes = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
        ours.t_huf_split(ws, log, nsym, rank, split, C.byref(shift), C.byref(T), C.byref(base), C.byref(nbytes))
        assert nbytes.value <= 2 << log and (shift.value == 0) == (log <= 8)
        saw_split |= shift.value > 0 and nbytes.value < (2 << log)
        for v in range(1 << log):
            assert ours.t_huf_cell(split, log, shift.value, T.value, base.value, v) == full[v], (log, v)
        # and the full table is the canonical one: index -> (symbol, length) of the code that prefixes it
        for s in range(nsym):
            if nb[s]:
                lo = code[s] << (log - nb[s])
                assert full[lo] == (s | (nb[s] << 8)) and full[lo + (1 << (log - nb[s])) - 1] == (s | (nb[s] << 8))
    assert saw_split


def test_frame_header_bytes_equal_the_reference():
    """ze_frame_header writes the header the reference writes (ZSTD_writeFrameHeader, zstd/zstd.c:27649) for every size
    class of the content-size field, with and without checksum, and for 1-, 2- and 4-byte dictionary ids; and a header the
    reference parses back when the content size is left out."""
    from oracle import RefZstd
    ref = RefZstd()
    H = host_encoder.build_sim()
    rng = np.random.default_rng(11)
    for size in (0, 1, 255, 256, 257, 4096, 65791, 65792, 131072, 300000, 1 << 20, 2 << 20, (2 << 20) + 1, 3 << 20, 9 << 20):
        data = rng.integers(0, 256, size).astype(np.uint8).tobytes() if size <= (1 << 20) else bytes(size)
        for checksum in (0, 1):
            frame = ref.compress(data, level=3, checksum=bool(checksum))
            out = (C.c_ubyte * 32)()
            n = H.t_frame_header(out, size, checksum, 1, 0)
            assert bytes(out[:n]) == frame[:n], (size, checksum)
    # dictionary ids: the header field the reference's parser reads back
    for did in (7, 300, 70000, 1123828263):
        for cs in (0, 1):
            out = (C.c_ubyte * 32)()
            n = H.t_frame_header(out, 5000, 1, cs, did)
            hdr = bytes(out[:n])
            fhd = hdr[4]
            assert fhd & 3 == (1 if did < 256 else 2 if did < 65536 else 3) and (fhd >> 2) & 1 == 1
            pos = 5 + (0 if cs else 1)
            k = [0, 1, 2, 4][fhd & 3]
            assert int.from_bytes(hdr[pos:pos + k], "little") == did
            if cs:
                assert (fhd >> 5) & 1 == 1 and int.from_bytes(hdr[pos + k:n], "little") + 256 == 5000
            else:
                assert (fhd >> 5) & 1 == 0 and (1 << (10 + (hdr[5] >> 3))) >= 5000
