"""Chain mode of the block-parallel decode on the CPU: the kernels of zb_decode.cu on tests/simt.h (the same host build
host_encoder.build_decode_sim makes), driven run by run as zb200_decompress_chain (zb_api.cu) drives them on the device.
TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

import host_encoder as H

LIB = os.path.join(H.BUILD, "libzd_chain_sim.so")
WRAPPERS = r"""
// One run in chain mode, kernel by kernel as run_decompress launches them with a ChainRun: scan, placement, the shift behind
// the carried prefix, the block path, pointer jumping, checksums, finish.  out: the run's arena, carry[0, carry_n) first.
extern "C" long long t_decompress_chain_run(const u8* src, const u64* seg_off, const u64* seg_len, u32 n, const u8* carry, u64 carry_n,
                                            u8* out, u64 out_cap, u64* out_off, u64* out_len, u32* status_out, int* rounds_out)
{
    static bool tables = false;
    if (!tables) { simt::launch(1, 32, [] { zb_build_default_tables(); }); tables = true; }
    ZbDictDev dict; memset(&dict, 0, sizeof dict);
    std::vector<ZbSegment> segs(n); for (u32 i = 0; i < n; i++) { segs[i].offset = seg_off[i]; segs[i].length = seg_len[i]; }
    std::vector<ZbFrameInfo> info(n); std::vector<ZbFramePlace> place(n + 1); std::vector<u32> status(n, 0), big(n + 1, 0);
    u64 totals[8] = {0}; u32 const pctas = (n + ZB_PLACE_CTA - 1) / ZB_PLACE_CTA; std::vector<u64> partial(pctas * 4 + 4);
    simt::launch((n + 127) / 128, 128, [&] { zb_scan_frames(src, segs.data(), n, info.data(), (1ull << 27) + 1, big.data()); });
    simt::launch(n < 128 ? (n + 3) / 4 : 32, 128, [&] { zb_scan_frames_big(src, segs.data(), big.data(), info.data()); });
    simt::launch(pctas, ZB_PLACE_CTA, [&] { zb_place_reduce(info.data(), nullptr, n, partial.data()); });
    simt::launch(pctas, ZB_PLACE_CTA, [&] { zb_place_scan(info.data(), nullptr, n, partial.data(), place.data(), totals, status.data()); });
    if (carry_n) simt::launch((n + 1 + 255) / 256, 256, [&] { zb_chain_shift(place.data(), n + 1, carry_n); });
    if (totals[5]) return -1001;
    u64 const total = totals[0] + carry_n;
    if (total > out_cap) return -1000;
    memcpy(out, carry, carry_n);
    u64 const nb = totals[1];
    std::vector<ZbBlock> blocks(nb + 1); std::vector<ZbSeq> seqs(totals[2] + 2); std::vector<u8> lits(totals[3] + 64);
    std::vector<u64> out_sizes(n, 0); std::vector<u32> ck(n, 0); u32 counter = 0;
    std::vector<ZbBlkDesc> bdesc(nb + 1); std::vector<ZbBlkExit> bexit(nb + 1); std::vector<u32> erep(3 * (nb + 1)); std::vector<u64> fend(n);
    simt::launch((n + 63) / 64, 64, [&] { zb_scan_blocks(src, segs.data(), n, place.data(), dict, status.data(), bdesc.data(), fend.data(), big.data()); });
    simt::launch(n < 128 ? (n + 3) / 4 : 32, 128, [&] { zb_scan_blocks_big(src, segs.data(), big.data(), place.data(), dict, status.data(), bdesc.data(), fend.data()); });
    simt::launch(3, 7 * 32, [&] { zb_entropy_blocks<7>(src, bdesc.data(), (u32)nb, blocks.data(), seqs.data(), lits.data(), &counter, dict, status.data(), bexit.data(), 3); });
    simt::launch((n + 63) / 64, 64, [&] { zb_resolve_blocks(src, segs.data(), n, place.data(), info.data(), nullptr, blocks.data(), bdesc.data(), bexit.data(), fend.data(), dict, status.data(), out_sizes.data(), ck.data(), erep.data()); });
    if (nb) simt::launch((unsigned)((nb + 7) / 8), 256, [&] { zb_patch_blocks(blocks.data(), bdesc.data(), nb, seqs.data(), erep.data(), dict, status.data(), place.data()); });
    std::vector<u32> ptr(total + 16, 0xFFFFFFFFu); u32 changed = 0; int rounds = 0;
    simt::launch(2, 256, [&] { zb_chase_prefix<u32>(place.data(), ptr.data()); });
    simt::launch(3, 256, [&] { zb_chase_init<u32>(src, place.data(), status.data(), blocks.data(), (const ZbBlkDesc*)bdesc.data(), seqs.data(), lits.data(), out, ptr.data(), 0, nb, dict, true); });
    do { changed = 0; simt::launch(4, 256, [&] { zb_chase_round<u32>(ptr.data(), 0, total, &changed); }); rounds++; } while (changed && rounds < 72);
    simt::launch(4, 256, [&] { zb_chase_gather<u32>(ptr.data(), out, 0, total, total); });
    *rounds_out = rounds;
    if (totals[4]) simt::launch((n + 127) / 128, 128, [&] { zb_verify_checksums(out, place.data(), out_sizes.data(), info.data(), ck.data(), 0, n, status.data()); });
    if (totals[4]) simt::launch(n < 8 ? n : 8, 256, [&] { zb_verify_checksums_big(out, place.data(), out_sizes.data(), info.data(), ck.data(), 0, n, status.data()); });
    std::vector<ZbSegment> out_segs(n); u32 first_error = 0xFFFFFFFFu;
    simt::launch((n + 255) / 256, 256, [&] { zb_finish(place.data(), out_sizes.data(), status.data(), n, out_segs.data(), &first_error); });
    for (u32 i = 0; i < n; i++) { out_off[i] = out_segs[i].offset; out_len[i] = out_segs[i].length; status_out[i] = status[i]; }
    return (long long)total;
}
"""


def build():
    """The kernels' text exactly as host_encoder.build_decode_sim cuts it out of zb_decode.cu, with the chain driver."""
    os.makedirs(H.BUILD, exist_ok=True)
    csrc = os.path.join(H.ROOT, "python_zstandard_b200", "csrc")
    dec = open(os.path.join(csrc, "zb_decode.cu")).read()
    a = dec.index('#include "zb_common.cuh"')
    a = dec.index("\n", a) + 1
    b = dec.index('extern "C" {')
    b = dec.rindex("// ====", 0, dec.rindex("// ====", 0, b))
    body = dec[a:b].replace('#include "zb_entropy.cuh"', open(H.DEC_SRC).read().replace("#pragma once", ""))
    body = re.sub(r"extern __shared__ __align__\(16\) u8 (\w+)\[\];", r"u8* const \1 = simt_dyn_smem;", body)
    text = (H.LIT_PRELUDE + "#include <cmath>\n#include <vector>\n" + '#include "%s"\n' % os.path.join(csrc, "zb_common.cuh")
            + '#include "%s"\n' % os.path.join(H.HERE, "simt.h") + "alignas(16) static u8 simt_dyn_smem[256 << 10];\n#define ZB_SCAN_BIG 24000u\n#define ZB_XXH_BIG 50000u\n" + body + WRAPPERS)
    cpp = os.path.join(H.BUILD, "zd_chain_sim.cpp")
    if not (os.path.exists(LIB) and os.path.exists(cpp) and open(cpp).read() == text
            and os.path.getmtime(LIB) >= os.path.getmtime(os.path.join(H.HERE, "simt.h"))):
        open(cpp, "w").write(text)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", LIB, cpp])
    L = C.CDLL(LIB)
    L.t_decompress_chain_run.restype = C.c_longlong
    L.t_decompress_chain_run.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_char_p, C.c_uint64,
                                         C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]
    return L


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
