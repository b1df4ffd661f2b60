"""An RFC 8878 conformance checker for frames the compressor writes.  Test infrastructure only.

A decoder that keeps the whole output in memory -- the reference's single-pass decoder, and ours -- accepts any offset
that stays inside the bytes decoded so far.  A streaming decoder keeps only Window_Size bytes of history, so a frame whose
matches reach further back than its header declares decodes in one and fails in the other.  `check_frame` holds one
frame to the rules a streaming decoder relies on:

  header     magic, reserved bit, Frame_Content_Size width and value (the 2-byte form stores size - 256), no window
             descriptor in a single-segment frame, dictionary ID as requested, Window_Size as section 3.1.1.1.2 defines it
  blocks     the 3-byte headers walked here; every Block_Size and every block's regenerated size at most
             Block_Maximum_Size = min(Window_Size, 128 KiB); the last-block flag on the final block only
  sequences  the offsets the oracle resolves (Oracle.trace), placed at their output position p in the frame by the block
             walk: offset <= p + dictionary content, and offset <= Window_Size when the source lies inside the frame
  checksum   present exactly when requested, equal to the low 32 bits of XXH64(content)

It is written from the RFC alone and shares nothing with the encoder.
"""
import struct

MAGIC = 0xFD2FB528
DICT_MAGIC = 0xEC30A437
BLOCK_MAX = 128 << 10


class FrameCheckError(AssertionError):
    """The frame breaks a rule of RFC 8878 (or is not what the call asked for)."""


def _fail(msg, *args):
    raise FrameCheckError(msg % args if args else msg)


def _ncount_bytes(buf, pos):
    """Bytes taken by the FSE table description (section 4.1.1) that starts at buf[pos]."""
    bits = int.from_bytes(buf[pos:pos + 512], "little")
    at = 0

    def read(n):
        nonlocal at
        v = (bits >> at) & ((1 << n) - 1)
        at += n
        return v

    log = read(4) + 5
    remaining, threshold, nbits = (1 << log) + 1, 1 << log, log + 1
    prev0 = False
    while remaining > 1:
        if prev0:
            while read(2) == 3:
                pass
        mx = (2 * threshold - 1) - remaining
        low = (bits >> at) & (threshold - 1)
        if low < mx:
            v = low
            at += nbits - 1
        else:
            v = read(nbits)
            if v >= threshold:
                v -= mx
        count = v - 1
        remaining -= -count if count < 0 else count
        prev0 = count == 0
        while remaining < threshold:
            nbits -= 1
            threshold >>= 1
    if remaining != 1:
        _fail("dictionary: malformed FSE table description")
    return (at + 7) // 8


def dict_content(dictionary):
    """The content of a dictionary (section 5): all of it for a raw-content dictionary; after the magic, the ID, the
    Huffman tree description, the three FSE tables and the three repcodes for a zstd dictionary."""
    d = bytes(dictionary or b"")
    if len(d) < 8 or struct.unpack_from("<I", d)[0] != DICT_MAGIC:
        return d
    p = 8
    hb = d[p]
    p += 1 + (hb if hb < 128 else (hb - 127 + 1) // 2)          # FSE-compressed weights, or 4-bit weights in pairs
    for _ in range(3):                                            # offset, match length, literal length tables
        p += _ncount_bytes(d, p)
    return d[p + 12:]


def _literals_regen(body):
    """Regenerated_Size of a compressed block's literals section (section 3.1.1.3.1.1)."""
    b0 = body[0]
    kind, form = b0 & 3, (b0 >> 2) & 3
    if kind < 2:                                                  # raw or RLE
        if form in (0, 2):
            return b0 >> 3
        if form == 1:
            return (b0 >> 4) | (body[1] << 4)
        return (b0 >> 4) | (body[1] << 4) | (body[2] << 12)
    size, width = {0: (3, 10), 1: (3, 10), 2: (4, 14), 3: (5, 18)}[form]
    return (int.from_bytes(body[:size], "little") >> 4) & ((1 << width) - 1)


def parse_header(frame):
    """The frame header fields: dict with single, checksum, dict_id (None: no field), content_size (None: no field),
    window_size and header_size."""
    f = bytes(frame)
    if len(f) < 6:
        _fail("frame of %d bytes", len(f))
    if struct.unpack_from("<I", f)[0] != MAGIC:
        _fail("magic number %08x", struct.unpack_from("<I", f)[0])
    fhd = f[4]
    fcs_flag, single, reserved, ck, did_flag = fhd >> 6, (fhd >> 5) & 1, (fhd >> 3) & 1, (fhd >> 2) & 1, fhd & 3
    if reserved:
        _fail("reserved bit of the frame header descriptor set")
    p, window = 5, None
    if not single:                                                # Window_Descriptor (section 3.1.1.1.2)
        wd = f[p]
        p += 1
        base = 1 << (10 + (wd >> 3))
        window = base + (base >> 3) * (wd & 7)
    did_bytes = (0, 1, 2, 4)[did_flag]
    dict_id = int.from_bytes(f[p:p + did_bytes], "little") if did_bytes else None
    p += did_bytes
    fcs_bytes = (1 if single else 0, 2, 4, 8)[fcs_flag]
    content_size = None
    if fcs_bytes:
        content_size = int.from_bytes(f[p:p + fcs_bytes], "little") + (256 if fcs_bytes == 2 else 0)
        p += fcs_bytes
    if single:
        window = content_size
    if p > len(f):
        _fail("frame header runs past the frame")
    return {"single": bool(single), "checksum": bool(ck), "dict_id": dict_id, "content_size": content_size,
            "window_size": window, "header_size": p}


def check_frame(frame, data, dictionary=b"", *, checksum, content_size, dict_id=0, oracle=None):
    """Assert that `frame` is one RFC 8878 frame of `data` that a decoder keeping only Window_Size bytes of history (plus
    the dictionary content) regenerates.  checksum / content_size: whether the call asked for them; dict_id: the ID the
    header must carry (0: none).  Returns what it found: the header fields, the block sizes and the largest offset."""
    from oracle import Oracle
    f, data = bytes(frame), bytes(data)
    h = parse_header(f)
    if content_size:
        if h["content_size"] is None:
            _fail("content size requested but not written")
        if h["content_size"] != len(data):
            _fail("content size %d, input %d bytes", h["content_size"], len(data))
    elif h["content_size"] is not None:
        _fail("content size written though not requested")
    if dict_id:
        if h["dict_id"] != dict_id:
            _fail("dictionary ID %r, expected %d", h["dict_id"], dict_id)
    elif h["dict_id"] is not None:
        _fail("dictionary ID field present though not requested")
    if h["checksum"] != bool(checksum):
        _fail("checksum flag %d, requested %d", h["checksum"], bool(checksum))
    window = h["window_size"]
    block_max = min(window, BLOCK_MAX)

    # ---- blocks
    p = h["header_size"]
    blocks = []                                                   # (type, Block_Size, content start)
    while True:
        if p + 3 > len(f):
            _fail("frame ends inside block %d's header (no last block)", len(blocks))
        bh = int.from_bytes(f[p:p + 3], "little")
        last, btype, size = bh & 1, (bh >> 1) & 3, bh >> 3
        if btype == 3:
            _fail("block %d: reserved block type", len(blocks))
        if size > block_max:
            _fail("block %d: Block_Size %d above Block_Maximum_Size %d", len(blocks), size, block_max)
        csize = 1 if btype == 1 else size
        if p + 3 + csize > len(f):
            _fail("block %d runs past the frame", len(blocks))
        blocks.append((btype, size, p + 3))
        p += 3 + csize
        if last:
            break
    rest = len(f) - p
    if rest != (4 if checksum else 0):
        _fail("%d bytes after the last block (checksum %s)", rest, "requested" if checksum else "not requested")

    # ---- checksum
    oracle = oracle or Oracle()
    if checksum and struct.unpack_from("<I", f, len(f) - 4)[0] != oracle.xxh64(data) & 0xFFFFFFFF:
        _fail("content checksum does not match")

    # ---- sequences: every offset against the window and the dictionary
    D = len(dict_content(dictionary))
    try:
        out, _, seqs, block_nseq = oracle.trace(f, len(data), dictionary)
    except Oracle.Error as e:
        _fail("the oracle rejects the frame: %s", e)
    if out != data:
        _fail("the frame does not regenerate the input")
    ncomp = sum(1 for b in blocks if b[0] == 2)
    if len(block_nseq) != ncomp:
        _fail("%d compressed blocks walked, %d decoded", ncomp, len(block_nseq))
    pos, k, ci, max_off = 0, 0, 0, 0
    for i, (btype, size, at) in enumerate(blocks):
        if btype != 2:
            regen = size
        else:
            lits = _literals_regen(f[at:at + size])
            q, used = pos, 0
            for ll, ml, off in seqs[k:k + block_nseq[ci]]:
                q += ll
                used += ll
                if off > q + D:
                    _fail("block %d: offset %d at frame position %d reaches in front of the frame (dictionary content %d)", i, off, q, D)
                if off <= q and off > window:
                    _fail("block %d: offset %d at frame position %d beyond Window_Size %d", i, off, q, window)
                max_off = max(max_off, off)
                q += ml
            if used > lits:
                _fail("block %d: sequences take %d literals of %d", i, used, lits)
            k += block_nseq[ci]
            ci += 1
            regen = q - pos + lits - used
        if regen > block_max:
            _fail("block %d regenerates %d bytes, above Block_Maximum_Size %d", i, regen, block_max)
        pos += regen
    if pos != len(data) or k != len(seqs):
        _fail("block walk regenerates %d bytes / %d sequences, decoder %d / %d", pos, k, len(data), len(seqs))
    return dict(h, blocks=[b[1] for b in blocks], max_offset=max_off)
