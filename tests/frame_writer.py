"""A test-only zstd frame writer, written from RFC 8878 alone.

It shares nothing with the product encoder (python_zstandard_b200/csrc/zb_encode.cu): a frame is described explicitly --
header fields, block types and sizes, literal modes, Huffman weights, the (literal length, match length, Offset_Value)
of every sequence, each FSE table's mode, normalized counts and accuracy log -- and `write()` turns the description into
bytes.  The expected output comes from `execute()`, a plain Python executor of the same description, so it never comes
from any decoder.  With it the tests reach parts of the format the reference encoder never writes: tables where one
symbol holds every state, logs at the decoder's limits, repeat and treeless modes in any order, hand-placed repcodes,
and offsets far beyond the window.
"""
import struct

import numpy as np

# --- RFC 8878 section 3.1.1.3.2.1: codes, baselines and extra bits ---------------------------------------------------
LL_BASE = list(range(16)) + [16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536]
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BASE = list(range(3, 35)) + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
# predefined distributions (section 3.1.1.3.2.2)
LL_DEFAULT = ([4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1], 6)
ML_DEFAULT = ([1, 4, 3, 2, 2, 2, 2, 2, 2] + [1] * 37 + [-1] * 7, 6)
OF_DEFAULT = ([1, 1, 1, 1, 1, 1, 2, 2, 2] + [1] * 15 + [-1] * 5, 5)
MAX_SYM = {"ll": 35, "of": 31, "ml": 52}
MAX_LOG = {"ll": 9, "of": 8, "ml": 9}
BLOCK_MAX = 128 << 10


class FrameError(Exception):
    """The description is not a valid frame: the executor found what a conforming decoder must reject."""


def ll_code(v):
    c = max(i for i in range(36) if LL_BASE[i] <= v)
    if v - LL_BASE[c] >= 1 << LL_BITS[c]:
        raise ValueError("literal length %d out of range" % v)
    return c, v - LL_BASE[c], LL_BITS[c]


def ml_code(v):
    if v < 3:
        raise ValueError("match length %d below 3" % v)
    c = max(i for i in range(53) if ML_BASE[i] <= v)
    if v - ML_BASE[c] >= 1 << ML_BITS[c]:
        raise ValueError("match length %d out of range" % v)
    return c, v - ML_BASE[c], ML_BITS[c]


def of_code(ov):
    if not 1 <= ov < 1 << 32:
        raise ValueError("Offset_Value %d out of range" % ov)
    c = ov.bit_length() - 1
    return c, ov - (1 << c), c


# --- descriptions ----------------------------------------------------------------------------------------------------
class Table:
    """One sequence table: kind 'pre' (predefined), 'rle' (sym), 'fse' (norm, log) or 'rep' (repeat the previous one;
    `fallback` is the table to encode with when there is no previous one, for frames that must be rejected)."""

    def __init__(self, kind, sym=0, norm=None, log=0, fallback=None):
        self.kind, self.sym, self.norm, self.log, self.fallback = kind, sym, norm, log, fallback

    def __repr__(self):
        return {"pre": "PRE", "rep": "REP"}.get(self.kind) or ("RLE(%d)" % self.sym if self.kind == "rle" else "FSE(log %d)" % self.log)


PRE = Table("pre")
REP = Table("rep")


def RLE_T(sym):
    return Table("rle", sym=sym)


def FSE(norm, log):
    return Table("fse", norm=list(norm), log=log)


class Lits:
    """A literals section.  mode: 'raw', 'rle', 'huf' (Huffman with a tree description) or 'treeless' (reuse the previous
    tree; `weights` is used to encode only when there is none, for frames that must be rejected).  hdr: the header size in
    bytes (raw / RLE: 1, 2 or 3; Huffman: 3, 4 or 5), chosen from the size when None.  streams: 1 or 4.  weights: the
    Huffman weight of every symbol up to the last one with a nonzero weight; written directly, or FSE-compressed when
    weights_fse = (normalized counts, log) is given."""

    def __init__(self, data, mode="raw", hdr=None, streams=None, weights=None, weights_fse=None, regen=None):
        self.data, self.mode, self.hdr, self.streams = bytes(data), mode, hdr, streams
        self.weights, self.weights_fse = weights, weights_fse
        self.regen = len(self.data) if regen is None else regen          # RLE: the regenerated size


class Raw:
    def __init__(self, data, size=None):
        self.data = bytes(data)
        self.size = len(self.data) if size is None else size              # a wrong size makes a truncated frame


class Rle:
    def __init__(self, byte, size):
        self.byte, self.size = byte, size


class Comp:
    """A compressed block: a literals section, then `seqs` = [(literal length, match length, Offset_Value)] coded with the
    LL / OF / ML tables.  nseq_bytes forces the 1-, 2- or 3-byte form of the sequence count; `trailing` is appended to
    the block (a malformed block when it is not empty); `final` picks which of its symbol's states each table ends in
    after the last sequence (an index into that symbol's states)."""

    def __init__(self, lits, seqs=(), ll=PRE, of=PRE, ml=PRE, nseq_bytes=None, trailing=b"", final=0):
        self.lits, self.seqs, self.ll, self.of, self.ml = lits, list(seqs), ll, of, ml
        self.nseq_bytes, self.trailing, self.final = nseq_bytes, trailing, final


class Frame:
    """fcs_bytes: 0/1/2/4/8 (None: the smallest that holds the size); window_log (+ mantissa) makes a window descriptor
    unless single_segment; dict_id with dict_id_bytes 0/1/2/4; checksum; skippable: payload of a skippable frame in front;
    content_size: what the header declares (None: the executed size; False: none)."""

    def __init__(self, blocks, single_segment=False, fcs_bytes=None, window_log=17, window_mantissa=0, dict_id=0,
                 dict_id_bytes=None, checksum=False, skippable=None, content_size=None, bad_checksum=False):
        self.blocks, self.single_segment, self.fcs_bytes = blocks, single_segment, fcs_bytes
        self.window_log, self.window_mantissa, self.dict_id, self.dict_id_bytes = window_log, window_mantissa, dict_id, dict_id_bytes
        self.checksum, self.skippable, self.content_size, self.bad_checksum = checksum, skippable, content_size, bad_checksum


class Dictionary:
    """A zstd dictionary: magic, ID, Huffman weights (direct, or FSE-compressed with weights_fse), the OF, ML and LL
    tables (FSE tables only), three repcodes and the content.  raw=True: content only."""

    def __init__(self, content, dict_id=0, weights=None, weights_fse=None, of=None, ml=None, ll=None, reps=(1, 4, 8), raw=False):
        self.content, self.dict_id, self.weights, self.weights_fse = bytes(content), dict_id, weights, weights_fse
        self.of, self.ml, self.ll, self.reps, self.raw = of, ml, ll, tuple(reps), raw

    @property
    def data(self):
        if self.raw:
            return self.content
        out = bytearray(struct.pack("<II", 0xEC30A437, self.dict_id))
        out += huf_description(self.weights, self.weights_fse)
        for t in (self.of, self.ml, self.ll):
            out += write_ncount(t.norm, t.log)
        out += struct.pack("<III", *self.reps)
        return bytes(out + self.content)


# --- bit streams -----------------------------------------------------------------------------------------------------
class _Bits:
    def __init__(self):
        self.acc, self.n, self.out = 0, 0, bytearray()

    def add(self, v, nb):
        assert 0 <= v < (1 << nb) or nb == 0 and v == 0, (v, nb)
        self.acc |= v << self.n
        self.n += nb
        while self.n >= 8:
            self.out.append(self.acc & 0xFF)
            self.acc >>= 8
            self.n -= 8

    def flush(self):
        if self.n:
            self.out.append(self.acc & 0xFF)
            self.acc, self.n = 0, 0
        return bytes(self.out)


def backward_stream(fields):
    """A backward bit stream (section 4.1): `fields` [(value, bits)] in the order the DECODER reads them.  They are
    written last-read first, then the 1-bit end marker, then zero padding to a byte."""
    w = _Bits()
    for v, nb in reversed(fields):
        w.add(v, nb)
    w.add(1, 1)
    return w.flush()


# --- FSE (section 4.1.1) ---------------------------------------------------------------------------------------------
def write_ncount(norm, log):
    """The FSE table description of normalized counts (-1: 'less than 1')."""
    assert 5 <= log <= 9, log
    assert sum(1 if c == -1 else c for c in norm) == 1 << log, "normalized counts must sum to 2^log"
    w = _Bits()
    w.add(log - 5, 4)
    remaining, threshold, nbits = (1 << log) + 1, 1 << log, log + 1
    s, prev0, n = 0, False, len(norm)
    while s < n and remaining > 1:
        if prev0:
            start = s
            while s < n and norm[s] == 0:
                s += 1
            while s >= start + 3:
                start += 3
                w.add(3, 2)
            w.add(s - start, 2)
        c = norm[s]
        s += 1
        mx = (2 * threshold - 1) - remaining
        remaining -= -c if c < 0 else c
        v = c + 1
        if v >= threshold:
            v += mx
        if v < mx:
            w.add(v, nbits - 1)
        else:
            w.add(v, nbits)
        prev0 = c == 0
        assert remaining >= 1
        while remaining < threshold:
            nbits -= 1
            threshold >>= 1
    assert remaining == 1
    return w.flush()


class FseTable:
    """The decoding table of section 4.1.1, and for the writer the inverse: which state of a symbol leads to a given
    next state."""

    def __init__(self, norm, log):
        size = 1 << log
        self.log, self.size = log, size
        sym = [0] * size
        high = size - 1
        for s, c in enumerate(norm):
            if c == -1:
                sym[high] = s
                high -= 1
        step, pos = (size >> 1) + (size >> 3) + 3, 0
        for s, c in enumerate(norm):
            for _ in range(max(c, 0)):
                sym[pos] = s
                pos = (pos + step) & (size - 1)
                while pos > high:
                    pos = (pos + step) & (size - 1)
        assert pos == 0
        nxt = [1 if c == -1 else c for c in norm]
        self.sym, self.nb, self.base = sym, [0] * size, [0] * size
        for u in range(size):
            x = nxt[sym[u]]
            nxt[sym[u]] += 1
            self.nb[u] = log - (x.bit_length() - 1)
            self.base[u] = (x << self.nb[u]) - size
        self._cover = {}

    @staticmethod
    def rle(sym):
        t = FseTable.__new__(FseTable)
        t.log, t.size, t.sym, t.nb, t.base, t._cover = 0, 1, [sym], [0], [0], {}
        return t

    def states(self, s):
        return [u for u in range(self.size) if self.sym[u] == s]

    def cover(self, s):
        if s not in self._cover:
            arr = [-1] * self.size
            for u in self.states(s):
                for t in range(self.base[u], self.base[u] + (1 << self.nb[u])):
                    arr[t] = u
            if not self.states(s):
                raise ValueError("symbol %d has no state in this table" % s)
            assert -1 not in arr
            self._cover[s] = arr
        return self._cover[s]

    def encode(self, syms, final=0):
        """States for decoding `syms` in order: (first state, [(update bits, nb) after symbol i, i < n - 1])."""
        n = len(syms)
        st = [0] * n
        cand = self.states(syms[-1])
        if not cand:
            raise ValueError("symbol %d has no state in this table" % syms[-1])
        st[-1] = cand[final % len(cand)]
        upd = [None] * (n - 1)
        for i in range(n - 2, -1, -1):
            u = self.cover(syms[i])[st[i + 1]]
            upd[i] = (st[i + 1] - self.base[u], self.nb[u])
            st[i] = u
        return st[0], upd


def table_of(t):
    return FseTable.rle(t.sym) if t.kind == "rle" else FseTable(t.norm, t.log)


# --- Huffman (section 4.2) -------------------------------------------------------------------------------------------
def huf_codes(weights):
    """{symbol: (code, bits)} of the prefix code given by the weights of every symbol (the last one included)."""
    total = sum(1 << (w - 1) for w in weights if w)
    log = total.bit_length() - 1
    assert total == 1 << log, "weights must sum to a power of two"
    codes, p = {}, 0
    for w in range(1, max(weights) + 1):
        for s, ws in enumerate(weights):
            if ws == w:
                codes[s] = (p >> (w - 1), log + 1 - w)
                p += 1 << (w - 1)
    return codes


def _fse_weights(ws, norm, log):
    """Huffman weights coded with FSE, two interleaved states (section 4.2.1.2)."""
    t = FseTable(norm, log)
    n = len(ws)
    assert n >= 2
    # state A decodes the even-indexed weights, B the odd ones; the update after weight n - 2 runs past the stream's
    # start, which tells the decoder that weight n - 1 (from the other state) is the last
    a_syms, b_syms = ws[0::2], ws[1::2]
    # the state that decodes weight n - 2 must read at least one bit when it updates
    pen = a_syms if (n - 2) % 2 == 0 else b_syms
    cands = t.states(pen[-1])
    k = next(i for i, u in enumerate(cands) if t.nb[u] > 0)
    fa = k if pen is a_syms else 0
    fb = k if pen is b_syms else 0
    # the update after weight n - 2 is not written: its state is the one that decodes that weight, free to choose
    a0, aupd = t.encode(a_syms, fa)
    b0, bupd = t.encode(b_syms, fb)
    fields = [(a0, log), (b0, log)]
    for i in range(n - 2):
        fields.append(aupd[i // 2] if i % 2 == 0 else bupd[i // 2])
    return write_ncount(norm, log) + backward_stream(fields)


def huf_description(weights, weights_fse=None):
    """The Huffman tree description: the weights of all symbols but the last."""
    ws = list(weights[:-1])
    if weights_fse is None:
        assert len(ws) <= 128
        body = bytes(((ws[i] << 4) | (ws[i + 1] if i + 1 < len(ws) else 0)) for i in range(0, len(ws), 2))
        return bytes([127 + len(ws)]) + body
    body = _fse_weights(ws, *weights_fse)
    assert len(body) < 128
    return bytes([len(body)]) + body


def huf_stream(data, codes):
    return backward_stream([codes[b] for b in data])


def huf_streams(data, codes, streams):
    if streams == 1:
        return huf_stream(data, codes)
    seg = (len(data) + 3) // 4
    parts = [huf_stream(data[k * seg:(k + 1) * seg] if k < 3 else data[3 * seg:], codes) for k in range(4)]
    return struct.pack("<HHH", len(parts[0]), len(parts[1]), len(parts[2])) + b"".join(parts)


# --- the writer ------------------------------------------------------------------------------------------------------
def _lit_header(kind, regen, csize, hdr, streams):
    if kind in (0, 1):
        if hdr is None:
            hdr = 1 if regen < 32 else (2 if regen < 4096 else 3)
        if hdr == 1:
            return bytes([kind | (regen << 3)])
        if hdr == 2:
            return struct.pack("<H", kind | (1 << 2) | (regen << 4))
        return struct.pack("<I", kind | (3 << 2) | (regen << 4))[:3]
    if hdr is None:
        hdr = 3 if max(regen, csize) < 1024 else (4 if max(regen, csize) < 16384 else 5)
    if hdr == 3:
        sf = 0 if streams == 1 else 1
        return struct.pack("<I", kind | (sf << 2) | (regen << 4) | (csize << 14))[:3]
    assert streams == 4
    if hdr == 4:
        return struct.pack("<I", kind | (2 << 2) | (regen << 4) | (csize << 18))
    v = kind | (3 << 2) | (regen << 4) | (csize << 22)
    return struct.pack("<Q", v)[:5]


class _State:
    """What later blocks inherit: the Huffman weights and the three sequence tables."""

    def __init__(self, dictionary):
        self.huf = None
        self.tabs = {"ll": None, "of": None, "ml": None}
        if dictionary is not None and not dictionary.raw:
            self.huf = dictionary.weights
            self.tabs = {"ll": dictionary.ll, "of": dictionary.of, "ml": dictionary.ml}


def _literals(L, st):
    if L.mode == "raw":
        return _lit_header(0, len(L.data), 0, L.hdr, 1) + L.data
    if L.mode == "rle":
        return _lit_header(1, L.regen, 0, L.hdr, 1) + L.data[:1]
    streams = L.streams or (1 if len(L.data) < 256 else 4)
    if L.mode == "huf":
        tree = huf_description(L.weights, L.weights_fse)
        weights = L.weights
        st.huf = L.weights
    else:
        tree = b""
        weights = st.huf if st.huf is not None else L.weights
    payload = tree + huf_streams(L.data, huf_codes(weights), streams)
    return _lit_header(2 if L.mode == "huf" else 3, len(L.data), len(payload), L.hdr, streams) + payload


def _nseq_bytes(n, form):
    if form is None:
        form = 1 if n < 128 else (2 if n < 0x7F00 else 3)
    if form == 1:
        assert n < 128
        return bytes([n])
    if form == 2:
        assert n < 0x7F00
        return bytes([0x80 + (n >> 8), n & 0xFF])
    return bytes([0xFF]) + struct.pack("<H", n - 0x7F00)


def _sequences(B, st):
    out = bytearray(_nseq_bytes(len(B.seqs), B.nseq_bytes))
    if not B.seqs:
        return bytes(out + B.trailing)
    descs = {"ll": B.ll, "of": B.of, "ml": B.ml}
    modes = {"pre": 0, "rle": 1, "fse": 2, "rep": 3}
    out.append((modes[B.ll.kind] << 6) | (modes[B.of.kind] << 4) | (modes[B.ml.kind] << 2))
    tabs = {}
    for k in ("ll", "of", "ml"):
        d = descs[k]
        pre = FSE(*{"ll": LL_DEFAULT, "of": OF_DEFAULT, "ml": ML_DEFAULT}[k])
        if d.kind == "pre":
            eff = pre
        elif d.kind == "rep":
            eff = st.tabs[k] or d.fallback or pre
        else:
            eff = d
        if d.kind == "rle":
            out.append(d.sym)
        elif d.kind == "fse":
            out += write_ncount(d.norm, d.log)
        st.tabs[k] = eff
        tabs[k] = table_of(eff)
    codes = [(ll_code(ll), ml_code(ml), of_code(ov)) for ll, ml, ov in B.seqs]
    s_ll, u_ll = tabs["ll"].encode([c[0][0] for c in codes], B.final)
    s_of, u_of = tabs["of"].encode([c[2][0] for c in codes], B.final)
    s_ml, u_ml = tabs["ml"].encode([c[1][0] for c in codes], B.final)
    fields = [(s_ll, tabs["ll"].log), (s_of, tabs["of"].log), (s_ml, tabs["ml"].log)]
    n = len(codes)
    per_seq = []
    for i, (lc, mc, oc) in enumerate(codes):
        fields += [(oc[1], oc[2]), (mc[1], mc[2]), (lc[1], lc[2])]
        if i + 1 < n:
            fields += [u_ll[i], u_ml[i], u_of[i]]
        per_seq.append((oc[2], mc[2] + lc[2], u_ll[i][1] + u_ml[i][1] + u_of[i][1] if i + 1 < n else 0))
    B.bitplan = ((tabs["ll"].log, tabs["of"].log, tabs["ml"].log), per_seq, sum(nb for _, nb in fields))
    return bytes(out + backward_stream(fields) + B.trailing)


def window_margins(plan, skew):
    """For a sequence stream whose first byte lies `skew` bytes past a 16-byte boundary: per sequence, its offset + ML/LL
    extra + state bits minus the bits the decoder's window holds when the sequence starts (ZbBitR of zb_common.cuh: the
    window is refilled by 32 bits whenever it holds 32 or fewer and words are left).  0: the bits fill the window exactly;
    1: one bit more than the window, so the decoder must refill between the reads."""
    logs, seqs, total = plan
    p = 8 * skew + total                      # bits from the aligned base up to the end mark
    wi = (p - 1) >> 5
    st = [p - 32 * wi, wi - 1]                # bits in the window, index of the next word to load

    def refill():
        if st[0] <= 32 and st[1] >= 0:
            st[0] += 32
            st[1] -= 1
    refill()
    st[0] -= logs[0] + logs[1]
    refill()
    st[0] -= logs[2]
    out = []
    for ofc, ab, sb in seqs:
        refill()
        out.append(ofc + ab + sb - st[0])
        slow = ofc + ab + sb > st[0]
        st[0] -= ofc
        if slow:
            refill()
        st[0] -= ab
        if slow:
            refill()
        st[0] -= sb
    return out


def _block(B, last, st):
    if isinstance(B, Raw):
        body, btype, size = B.data, 0, B.size
    elif isinstance(B, Rle):
        body, btype, size = bytes([B.byte]), 1, B.size
    else:
        body = _literals(B.lits, st) + _sequences(B, st)
        btype, size = 2, len(body)
    return struct.pack("<I", int(last) | (btype << 1) | (size << 3))[:3] + body


def frame_header(F, content_size):
    fcs = F.content_size if F.content_size is not None else content_size
    if fcs is False:
        fb = 0
        assert not F.single_segment
    elif F.fcs_bytes is not None:
        fb = F.fcs_bytes
    else:
        fb = (1 if F.single_segment else 4) if fcs < 256 else (2 if fcs < 65536 + 256 else (4 if fcs < 1 << 32 else 8))
    if not F.single_segment and fb == 1:
        raise ValueError("a 1-byte content size needs a single-segment frame")
    dib = F.dict_id_bytes if F.dict_id_bytes is not None else (0 if not F.dict_id else (1 if F.dict_id < 256 else (2 if F.dict_id < 65536 else 4)))
    fcs_flag = {0: 0, 1: 0, 2: 1, 4: 2, 8: 3}[fb]
    fhd = (fcs_flag << 6) | (int(F.single_segment) << 5) | (int(F.checksum) << 2) | {0: 0, 1: 1, 2: 2, 4: 3}[dib]
    out = bytearray(struct.pack("<I", 0xFD2FB528)) + bytes([fhd])
    if not F.single_segment:
        out.append(((F.window_log - 10) << 3) | F.window_mantissa)
    if dib:
        out += struct.pack("<I", F.dict_id)[:dib]
    if fb == 1:
        out.append(fcs)
    elif fb == 2:
        out += struct.pack("<H", fcs - 256)
    elif fb == 4:
        out += struct.pack("<I", fcs)
    elif fb == 8:
        out += struct.pack("<Q", fcs)
    return bytes(out)


def window_size(F, content_size):
    if F.single_segment:
        return F.content_size if F.content_size is not None else content_size
    wl = 1 << F.window_log
    return wl + (wl >> 3) * F.window_mantissa


def execute(F, dictionary=None):
    """Regenerate the frame's content from its description (section 3.1.1.4-5).  Returns (bytes, [(ll, ml, offset)],
    [sequences per compressed block], [regenerated size per block]); raises FrameError where a decoder must reject the
    frame."""
    hist = b""
    rep = [1, 4, 8]
    if dictionary is not None:
        hist = dictionary.content
        if not dictionary.raw:
            rep = list(dictionary.reps)
            if any(r == 0 or r > len(hist) for r in rep):
                raise FrameError("dictionary repcode outside the dictionary content")
            if F.dict_id and dictionary.dict_id and F.dict_id != dictionary.dict_id:
                raise FrameError("frame made for another dictionary")
    out = bytearray(hist)
    base = len(hist)
    trace, counts, sizes = [], [], []
    have_huf = dictionary is not None and not dictionary.raw
    have = {k: have_huf for k in ("ll", "of", "ml")}
    for B in F.blocks:
        if isinstance(B, Raw):
            out += B.data
            sizes.append(len(B.data))
            if B.size != len(B.data):
                raise FrameError("truncated raw block")
            continue
        if isinstance(B, Rle):
            out += bytes([B.byte]) * B.size
            sizes.append(B.size)
            continue
        L, start = B.lits, len(out)
        if L.mode == "treeless" and not have_huf:
            raise FrameError("treeless literals without a previous Huffman table")
        if L.mode in ("huf", "treeless"):
            have_huf = True
            if (L.streams or (1 if len(L.data) < 256 else 4)) == 4 and len(L.data) < 6:
                raise FrameError("4 streams need at least 6 literals")
        lits = L.data if L.mode != "rle" else L.data[:1] * L.regen
        if B.trailing and not B.seqs:
            raise FrameError("bytes after a sequence count of 0")
        for k, t in (("ll", B.ll), ("of", B.of), ("ml", B.ml)):
            if B.seqs and t.kind == "rep" and not have[k]:
                raise FrameError("repeat mode with no previous table")
            if B.seqs:
                have[k] = True
        lp = 0
        counts.append(len(B.seqs))
        for ll, ml, ov in B.seqs:
            if ov > 3:
                off = ov - 3
                rep = [off, rep[0], rep[1]]
            else:
                idx = ov - 1 + (ll == 0)
                if idx == 0:
                    off = rep[0]
                elif idx == 1:
                    off = rep[1]
                    rep = [off, rep[0], rep[2]]
                else:
                    off = rep[2] if idx == 2 else rep[0] - 1
                    rep = [off, rep[0], rep[1]]
            trace.append((ll, ml, off if off else 0xFFFFFFFF))
            if ll > len(lits) - lp:
                raise FrameError("literal length beyond the literals")
            out += lits[lp:lp + ll]
            lp += ll
            if off == 0 or off > len(out):
                raise FrameError("offset %d beyond the history" % off)
            for _ in range(ml):
                out.append(out[-off])
        out += lits[lp:]
        sizes.append(max(len(out) - start, len(lits)))
    return bytes(out[base:]), trace, counts, sizes


def write(F, dictionary=None):
    """(frame bytes, expected content or None when the frame must be rejected, trace or None)."""
    try:
        expected, trace, counts, sizes = execute(F, dictionary)
    except FrameError:
        expected, trace, counts, sizes = None, None, None, []
    size = len(expected) if expected is not None else regen_size(F)
    st = _State(dictionary)
    out = bytearray()
    if F.skippable is not None:
        out += struct.pack("<II", 0x184D2A50, len(F.skippable)) + F.skippable
    out += frame_header(F, size)
    block_max = min(window_size(F, size), BLOCK_MAX)
    for i, B in enumerate(F.blocks):
        blk = _block(B, i == len(F.blocks) - 1, st)
        out += blk
        if isinstance(B, Comp) and len(blk) - 3 > block_max:          # a block's size is capped by the window too
            expected = None
    if any(n > block_max for n in sizes):
        expected = None
    if F.checksum:
        h = xxh64(expected if expected is not None else b"") & 0xFFFFFFFF
        out += struct.pack("<I", h ^ (1 if F.bad_checksum else 0))
    if expected is not None and (F.bad_checksum or F.content_size not in (None, False) and F.content_size != len(expected)):
        expected = None
    if expected is None:
        trace = counts = None
    return bytes(out), expected, (trace, counts) if trace is not None else None


def frame_bytes(F, content_size, dictionary=None):
    """The bytes of a frame whose content is too large to regenerate here: no executor, no content checksum."""
    assert not F.checksum
    st = _State(dictionary)
    return frame_header(F, content_size) + b"".join(_block(B, i == len(F.blocks) - 1, st) for i, B in enumerate(F.blocks))


def regen_size(F):
    """The bytes a frame's blocks regenerate, taken from the description alone (what its header declares)."""
    n = 0
    for B in F.blocks:
        if isinstance(B, Raw):
            n += len(B.data)
        elif isinstance(B, Rle):
            n += B.size
        else:
            n += B.lits.regen + sum(ml for _, ml, _ in B.seqs)
    return n


# --- XXH64 (for the content checksum) --------------------------------------------------------------------------------
_P1, _P2, _P3, _P4, _P5 = 0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63, 0x27D4EB2F165667C5
_M = (1 << 64) - 1


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & _M


def _round(acc, lane):
    return (_rotl((acc + lane * _P2) & _M, 31) * _P1) & _M


def xxh64(data, seed=0):
    data = bytes(data)
    n, p = len(data), 0
    if n >= 32:
        v = [(seed + _P1 + _P2) & _M, (seed + _P2) & _M, seed & _M, (seed - _P1) & _M]
        lanes = np.frombuffer(data[:n - n % 32], dtype="<u8").tolist()
        for i in range(0, len(lanes), 4):
            v = [_round(v[0], lanes[i]), _round(v[1], lanes[i + 1]), _round(v[2], lanes[i + 2]), _round(v[3], lanes[i + 3])]
        p = n - n % 32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & _M
        for x in v:
            h = ((h ^ _round(0, x)) * _P1 + _P4) & _M
    else:
        h = (seed + _P5) & _M
    h = (h + n) & _M
    while p + 8 <= n:
        h = (_rotl(h ^ _round(0, struct.unpack_from("<Q", data, p)[0]), 27) * _P1 + _P4) & _M
        p += 8
    if p + 4 <= n:
        h = (_rotl(h ^ ((struct.unpack_from("<I", data, p)[0] * _P1) & _M), 23) * _P2 + _P3) & _M
        p += 4
    while p < n:
        h = (_rotl(h ^ ((data[p] * _P5) & _M), 11) * _P1) & _M
        p += 1
    h ^= h >> 33
    h = (h * _P2) & _M
    h ^= h >> 29
    h = (h * _P3) & _M
    return h ^ (h >> 32)
