"""Chain mode of the block-parallel decode on the CPU: the launchers of zb_decode.cu on tests/simt.h (t_decompress_chain_run
of host_encoder.build_sim), driven run by run as zb200_decompress_chain (zb_api.cu) drives them on the device.
TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import ctypes as C
import numpy as np

class ChainSimError(Exception):
    def __init__(self, chunk, code):
        super().__init__("chunk %d: code %d" % (chunk, code))
        self.chunk, self.code = chunk, code


FAR_WINDOW = (1 << 31) - (1 << 27)


def _header(chunk, prev_size):
    """zb200_decompress_chain's host checks: (error code or 0, content size, skippable)."""
    n = len(chunk)
    if n >= 4 and int.from_bytes(chunk[:4], "little") & 0xFFFFFFF0 == 0x184D2A50:
        ln = int.from_bytes(chunk[4:8], "little") if n >= 8 else 0
        return (72 if n < 8 + ln else 0), 0, True
    import chain_ref
    fh = chain_ref.FrameHeader()
    L = chain_ref.lib()
    z = L.ZSTD_getFrameHeader(C.byref(fh), chunk, n)
    if L.ZSTD_isError(z) or z:
        return 10, 0, False
    if fh.frameContentSize == chain_ref.CONTENTSIZE_UNKNOWN:
        return 200, 0, False
    size = fh.frameContentSize
    if size >= FAR_WINDOW or fh.windowSize >= FAR_WINDOW or prev_size + size >= FAR_WINDOW:
        return 16, 0, False
    if fh.dictID:                # (no dictionary for chunk 0 here)
        return 32, 0, False
    return 0, size, False


def decompress_chain(L, frames, run_cut):
    """The last fulltext of the chain, or ChainSimError(lowest failing chunk, zstd code).  run_cut(k, sizes) -> the end of the
    run that starts at chunk k (the launcher's memory budget, made explicit)."""
    sizes, skip, h, h_code = [], [], len(frames), 0
    for k, f in enumerate(frames):
        code, size, sk = _header(f, sizes[-1] if sizes else 0)
        if code:
            h, h_code = k, code
            break
        sizes.append(size)
        skip.append(sk)
    blob = b"".join(frames[:h])
    offs = np.cumsum([0] + [len(f) for f in frames[:h]]).astype(np.uint64)
    lens = np.array([len(f) for f in frames[:h]] + [0], dtype=np.uint64)
    src = np.frombuffer(blob + bytes(64), dtype=np.uint8)
    carry, k = b"", 0
    while k < h:
        if skip[k]:
            carry, k = b"", k + 1
            continue
        b = max(k + 1, min(run_cut(k, sizes), h))
        b = next((j for j in range(k + 1, b) if skip[j]), b)
        n = b - k
        cap = len(carry) + sum(sizes[k:b]) + 64
        out = np.zeros(cap, dtype=np.uint8)
        o_off, o_len, st = np.zeros(n, np.uint64), np.zeros(n, np.uint64), np.zeros(n, np.uint32)
        rounds = C.c_int()
        r = L.t_decompress_chain_run(src.ctypes.data, offs[k:].ctypes.data, lens[k:].ctypes.data, n, carry, len(carry),
                                     out.ctypes.data, cap, o_off.ctypes.data, o_len.ctypes.data, st.ctypes.data, C.byref(rounds))
        assert r >= 0, r
        bad = np.nonzero(st)[0]
        if len(bad):
            raise ChainSimError(k + int(bad[0]), int(st[bad[0]]))
        carry = out[int(o_off[-1]):int(o_off[-1] + o_len[-1])].tobytes()
        k = b
    if h < len(frames):
        raise ChainSimError(h, h_code)
    return carry
