"""Host build of the encoder's serial entropy-table helpers, for CPU known-answer tests.

The helpers (FSE normalisation, NCount writer, CTable builder, table choice, Huffman code construction and its
weight header) are plain single-thread code inside python_zstandard_b200/csrc/zb_encode.cu.  This module cuts that
very text out of the .cu file, swaps the CUDA qualifiers for host ones and compiles it with g++ into
tests/_build/libze_host.so, so the CPU suite checks the same source lines the kernel runs -- against the
reference's own FSE_* / HUF_* functions in oracle/_ref (tests/test_encoder_tables.py).  Test infrastructure only.
"""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(ROOT, "python_zstandard_b200", "csrc", "zb_encode.cu")
BUILD = os.path.join(HERE, "_build")
LIB = os.path.join(BUILD, "libze_host.so")

PRELUDE = r"""
#include <cstdint>
#include <cmath>
#include <cstring>
typedef uint8_t u8; typedef uint16_t u16; typedef uint32_t u32; typedef uint64_t u64;
struct uint4 { u32 x, y, z, w; };
static inline u32 ze_hibit(u32 v) { return 31u - (u32)__builtin_clz(v); }
#define __log2f log2f
"""

WRAPPERS = r"""
extern "C" {
int t_normalize(short* norm, const u32* count, u32 max_sym, u32 total, u32 log) { return ze_normalize(norm, count, max_sym, total, log) ? 1 : 0; }
u32 t_write_ncount(u8* out, const short* norm, u32 max_sym, u32 log) { return ze_write_ncount(out, norm, max_sym, log); }
u32 t_cost(const u32* count, const short* norm, u32 max_sym, u32 log) { return ze_cost(count, norm, max_sym, log); }
void t_build_ctable(const short* norm, u32 max_sym, u32 log, u16* state, int* dnb, int* dfs)
{
    static ZeCTable ct; static u8 tmp[512];
    ze_build_ctable(ct, norm, max_sym, log, tmp);
    memcpy(state, ct.state, sizeof(u16) << log); memcpy(dnb, ct.dnb, sizeof(int) * (max_sym + 1)); memcpy(dfs, ct.dfs, sizeof(int) * (max_sym + 1));
}
// mode, log, header bytes of the table the encoder would pick for this histogram (no dictionary)
void t_make_table(const u32* count, u32 max_sym_kind, u32 nseq, u32 max_log, u32 def_log, const short* defnorm, u32 def_max,
                  u32* mode, u32* log, u32* hdr_bytes, u8* hdr)
{
    static ZeCTable ct; static u8 tmp[512];
    ze_make_table(ct, count, max_sym_kind, nseq, max_log, def_log, defnorm, def_max, tmp);
    *mode = ct.mode; *log = ct.log; *hdr_bytes = ct.hdr_bytes; memcpy(hdr, ct.hdr, 64);
}
int t_huf_build(const u32* count, u8* nb, u16* code, u32* max_sym, u32* log)
{
    static ZeHuf H; static u32 wk[1600];
    if (!ze_huf_build(H, count, wk)) return 0;
    memcpy(nb, H.nb, 256); memcpy(code, H.code, 512); *max_sym = H.max_sym; *log = H.log;
    return 1;
}
u32 t_huf_write_table(const u32* count, u8* out)
{
    static ZeHuf H; static u32 wk[1600]; static ZeCTable ct; static u8 tmp[512];
    if (!ze_huf_build(H, count, wk)) return 0;
    return ze_huf_write_table(out, H, ct, tmp);
}
}
"""


def _extract():
    src = open(SRC).read()
    a = src.index("struct ZeCTable {")
    b = src.index("// the block kernel")
    b = src.rindex("// ----", 0, b)
    chunk = src[a:b]
    return chunk.replace("__device__ static", "static").replace("__device__ __forceinline__", "static inline")


DEC_SRC = os.path.join(ROOT, "python_zstandard_b200", "csrc", "zb_entropy.cuh")
DEC_LIB = os.path.join(BUILD, "libzd_host.so")
DEC_WRAPPERS = r"""
extern "C" {
// builds the split table for the given nibble weights and returns its shape; cells must hold 4096 entries
void t_huf_split(const u8* ws, u32 log, u32 nsym, const u32* rank, u16* cells, u32* shift, u32* T, u32* base, u32* bytes)
{
    zb_huf_shape(log, rank, *shift, *T, *base, *bytes);
    zb_huf_fill(cells, ws, log, nsym, rank, *shift, *base);
}
void t_huf_full(const u8* ws, u32 log, u32 nsym, const u32* rank, u16* cells) { zb_huf_fill(cells, ws, log, nsym, rank, 0, 0); }
u32 t_huf_cell(const u16* cells, u32 log, u32 shift, u32 T, u32 base, u32 v)
{
    ZbHufTab t; t.cells = cells; t.log = log; t.shift = shift; t.T = T; t.base = base;
    return ZB_HCELL(t, v);
}
}
"""


def build_decoder_helpers():
    """Host build of the split Huffman decode table code of zb_entropy.cuh (shape, fill, lookup)."""
    os.makedirs(BUILD, exist_ok=True)
    src = open(DEC_SRC).read()
    a = src.index("#define ZB_HUF_COARSE")
    b = src.index("// one Huffman stream")
    chunk = src[a:b].replace("__device__ static", "static").replace("__device__ __forceinline__", "static inline")
    text = PRELUDE + chunk + DEC_WRAPPERS
    cpp = os.path.join(BUILD, "zd_host.cpp")
    if not (os.path.exists(DEC_LIB) and os.path.exists(cpp) and open(cpp).read() == text):
        open(cpp, "w").write(text)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-o", DEC_LIB, cpp])
    L = C.CDLL(DEC_LIB)
    L.t_huf_cell.restype = C.c_uint32
    return L


HDR_LIB = os.path.join(BUILD, "libzh_host.so")


def build_frame_header():
    """Host build of ze_frame_header (zb_encode.cu): u32 t_frame_header(u8* out, u64 size, checksum, content_size, dict_id)."""
    os.makedirs(BUILD, exist_ok=True)
    src = open(SRC).read()
    a = src.index("__device__ __forceinline__ u32 ze_frame_header")
    b = src.index("\n}\n", a) + 3
    text = (PRELUDE + "struct ZeParams { u32 checksum; u32 content_size; u32 dict_id; u32 level; u32 window_log = 0; };\n"
            + src[a:b].replace("__device__ __forceinline__", "static inline")
            + 'extern "C" u32 t_frame_header(u8* o, u64 size, u32 checksum, u32 content_size, u32 dict_id)\n'
              "{ ZeParams P; P.checksum = checksum; P.content_size = content_size; P.dict_id = dict_id; P.level = 3; return ze_frame_header(o, size, P); }\n")
    cpp = os.path.join(BUILD, "zh_host.cpp")
    if not (os.path.exists(HDR_LIB) and os.path.exists(cpp) and open(cpp).read() == text):
        open(cpp, "w").write(text)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-o", HDR_LIB, cpp])
    L = C.CDLL(HDR_LIB)
    L.t_frame_header.restype = C.c_uint32
    L.t_frame_header.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32]
    return L


PARSE_LIB = os.path.join(BUILD, "libzp_host.so")


def build_header_parser():
    """Host build of the device frame-header parser (zb_parse_header, zb_decode.cu):
    t_parse_header(src, n, out[6] = {content_size, window, dict_id, hdr_size, checksum, status})."""
    os.makedirs(BUILD, exist_ok=True)
    csrc = os.path.join(ROOT, "python_zstandard_b200", "csrc")
    dec = open(os.path.join(csrc, "zb_decode.cu")).read()
    a = dec.index("struct ZbHdr {")
    b = dec.index("// skip leading skippable frames")
    text = (LIT_PRELUDE + '#include "%s"\n' % os.path.join(csrc, "zb_common.cuh") + dec[a:b]
            + 'extern "C" void t_parse_header(const u8* s, u64 n, u64* out)\n'
              "{ ZbHdr h; zb_parse_header(s, n, h); out[0] = h.content_size; out[1] = h.window; out[2] = h.dict_id; out[3] = h.hdr_size; out[4] = h.checksum; out[5] = h.status; }\n")
    cpp = os.path.join(BUILD, "zp_host.cpp")
    if not (os.path.exists(PARSE_LIB) and os.path.exists(cpp) and open(cpp).read() == text):
        open(cpp, "w").write(text)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", PARSE_LIB, cpp])
    L = C.CDLL(PARSE_LIB)
    L.t_parse_header.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
    return L


SIM_LIB = os.path.join(BUILD, "libzs_host.so")
SIM_WRAPPERS = r"""
extern "C" unsigned long long t_any_calls(int reset) { unsigned long long v = simt_any_calls; if (reset) simt_any_calls = 0; return v; }
// The whole compression path of the library on the CPU: block jobs cut as zb_api.cu cuts them (zb_cut_blocks, blocks of
// min(2^window_log, 128 KiB)), zb_compress_blocks on `n_ctas` CTAs of 128 threads -- the two-table instantiation from level 4
// on, as the launcher picks it -- or zb_compress_recs when `recs` is set, then the frame layout kernels with the level and
// window_log of the call.  Input resident.  Returns total bytes.
extern "C" long long t_compress_batch(const u8* src, const u64* seg_off, const u64* seg_len, u32 n_segs, u32 checksum, u32 content_size,
                                      u32 n_ctas, u8* out, u64 out_cap, u64* out_off, u64* out_len, u32 recs, const u8* dict_raw, u32 dict_n,
                                      int level, u32 window_log)
{
    std::vector<ZbSegment> segs(n_segs); std::vector<ZeBlockJob> jobs; std::vector<ZeSegInfo> info(n_segs);
    for (u32 i = 0; i < n_segs; i++) { segs[i].offset = seg_off[i]; segs[i].length = seg_len[i]; }
    u32 const max_block = zb_cut_blocks(segs.data(), n_segs, zb_block_max(window_log), jobs, info);
    bool const dual = level >= 4;
    u32 const nj = (u32)jobs.size();
    u64 const slot_bytes = ((u64)max_block + (max_block >> 7) + 64 + 15) & ~15ull;
    std::vector<u8> slots((size_t)(nj + 1) * slot_bytes); std::vector<ZeBlockOut> outs(nj + 1);
    if (n_ctas > nj) n_ctas = nj ? nj : 1;
    ZeScratch* scratch = (ZeScratch*)aligned_alloc(64, ((sizeof(ZeScratch) + 63) & ~(size_t)63) * n_ctas);
    u32 counter = 0;
    ZeDict dict; memset(&dict, 0, sizeof dict);
    static ZbDictDigest dg; static u16 dtable[1 << ZE_HLOG]; static ZeCTable cct[3];
    u32 dict_id = 0;
    if (dict_raw && dict_n) {          // what zb200_ddict_create does: digest, compression view (last <= 32 KiB), hash table, CTables
        simt::launch(1, 32, [&] { zb_digest_dict(dict_raw, dict_n, &dg); });
        if (dg.status != ZB_OK) return -2;
        const u8* content = dg.has_entropy ? dict_raw + dg.content_off : dict_raw;
        u32 const csize = dg.has_entropy ? dict_n - dg.content_off : dict_n;
        u32 const D = csize < 32768u ? csize : 32768u;
        if (D >= 8) {
            dict.tail = content + (csize - D); dict.D = D; dict.table = dtable; dict_id = dg.dict_id;
            simt::launch(1, 32, [&] { zb_dict_table(dict.tail, D, dtable); });
            if (dg.has_entropy) { dict.ent = &dg; dict.cct = cct; simt::launch(1, 96, [&] { zb_dict_ctables(&dg, cct); }); }
        }
    }
    ZeUpload up; up.progress = nullptr; up.total = 0; up.status = nullptr;
    ZeParams P; P.checksum = checksum; P.content_size = content_size; P.dict_id = dict_id; P.level = (u32)level; P.window_log = window_log;
    bool const small_blocks = max_block <= ZE_SMALL_MAX;             // as zb_api.cu picks the instantiation
    if (nj && recs) simt::launch((nj + Z3_WARPS - 1) / Z3_WARPS < n_ctas ? (nj + Z3_WARPS - 1) / Z3_WARPS : n_ctas, Z3_NT, [&] { zb_compress_recs(src, jobs.data(), nj, slots.data(), slot_bytes, outs.data(), &counter, dict, up); });
    else if (nj && dual && small_blocks) simt::launch(n_ctas, ZE_THREADS, [&] { zb_compress_blocks<true, ZE_UNIT_SMALL>(src, jobs.data(), nj, (ZeScratch*)scratch, slots.data(), slot_bytes, outs.data(), &counter, dict, up); });
    else if (nj && small_blocks) simt::launch(n_ctas, ZE_THREADS, [&] { zb_compress_blocks<false, ZE_UNIT_SMALL>(src, jobs.data(), nj, (ZeScratch*)scratch, slots.data(), slot_bytes, outs.data(), &counter, dict, up); });
    else if (nj && dual) simt::launch(n_ctas, ZE_THREADS, [&] { zb_compress_blocks<true, ZE_UNIT>(src, jobs.data(), nj, (ZeScratch*)scratch, slots.data(), slot_bytes, outs.data(), &counter, dict, up); });
    else if (nj) simt::launch(n_ctas, ZE_THREADS, [&] { zb_compress_blocks<false, ZE_UNIT>(src, jobs.data(), nj, (ZeScratch*)scratch, slots.data(), slot_bytes, outs.data(), &counter, dict, up); });
    std::vector<u64> sizes(n_segs); std::vector<ZbSegment> out_segs(n_segs); u64 total = 0;
    simt::launch((n_segs + 255) / 256, 256, [&] { zb_frame_sizes(segs.data(), info.data(), outs.data(), n_segs, P, sizes.data()); });
    simt::launch(1, 1024, [&] { zb_scan_sizes(sizes.data(), n_segs, out_segs.data(), &total); });
    free(scratch);
    if (total > out_cap) return -1;
    simt::launch((n_segs + 7) / 8, 256, [&] { zb_write_frames(src, segs.data(), info.data(), outs.data(), slots.data(), slot_bytes, n_segs, P, out_segs.data(), out); });
    for (u32 i = 0; i < n_segs; i++) { out_off[i] = out_segs[i].offset; out_len[i] = out_segs[i].length; }
    return (long long)total;
}

// The round-2 kernel (zb_compress_smem: one CTA of 1024 threads per block, block resident in "shared memory") on the CPU,
// with the jobs and frame headers of a call with this level and window_log.
extern "C" long long t_compress_batch2(const u8* src, const u64* seg_off, const u64* seg_len, u32 n_segs, u32 checksum, u32 content_size,
                                       u32 n_ctas, u8* out, u64 out_cap, u64* out_off, u64* out_len, int level, u32 window_log)
{
    std::vector<ZbSegment> segs(n_segs); std::vector<ZeBlockJob> jobs; std::vector<ZeSegInfo> info(n_segs);
    for (u32 i = 0; i < n_segs; i++) { segs[i].offset = seg_off[i]; segs[i].length = seg_len[i]; }
    u32 const max_block = zb_cut_blocks(segs.data(), n_segs, zb_block_max(window_log), jobs, info);
    u32 const nj = (u32)jobs.size();
    u64 const slot_bytes = ((u64)max_block + (max_block >> 7) + 64 + 15) & ~15ull;
    u8* slots = (u8*)aligned_alloc(64, (size_t)(nj + 1) * slot_bytes + 64); std::vector<ZeBlockOut> outs(nj + 1);
    if (n_ctas > nj) n_ctas = nj ? nj : 1;
    Z2Scratch* scratch = (Z2Scratch*)aligned_alloc(64, ((sizeof(Z2Scratch) + 63) & ~(size_t)63) * n_ctas);
    u32 counter = 0;
    ZeUpload up; up.progress = nullptr; up.total = 0; up.status = nullptr;
    ZeParams P; P.checksum = checksum; P.content_size = content_size; P.dict_id = 0; P.level = (u32)level; P.window_log = window_log;
    if (nj) simt::launch(n_ctas, Z2_NT, [&] { zb_compress_smem(src, jobs.data(), nj, scratch, slots, slot_bytes, outs.data(), &counter, up); });
    std::vector<u64> sizes(n_segs); std::vector<ZbSegment> out_segs(n_segs); u64 total = 0;
    simt::launch((n_segs + 255) / 256, 256, [&] { zb_frame_sizes(segs.data(), info.data(), outs.data(), n_segs, P, sizes.data()); });
    simt::launch(1, 1024, [&] { zb_scan_sizes(sizes.data(), n_segs, out_segs.data(), &total); });
    free(scratch);
    if (total > out_cap) { free(slots); return -1; }
    simt::launch((n_segs + 7) / 8, 256, [&] { zb_write_frames(src, segs.data(), info.data(), outs.data(), slots, slot_bytes, n_segs, P, out_segs.data(), out); });
    free(slots);
    for (u32 i = 0; i < n_segs; i++) { out_off[i] = out_segs[i].offset; out_len[i] = out_segs[i].length; }
    return (long long)total;
}
"""


def build_compress_sim():
    """Host build of the whole compression kernel source (zb_encode.cu up to its launchers) on the mini SIMT runtime of
    tests/simt.h: 128 fibers per CTA, warp collectives and barriers as rendezvous."""
    os.makedirs(BUILD, exist_ok=True)
    import re
    csrc = os.path.join(ROOT, "python_zstandard_b200", "csrc")
    enc = open(SRC).read()
    a = enc.index('#include "zb_common.cuh"')
    a = enc.index("\n", a) + 1
    b = enc.index('extern "C" {')
    b = enc.rindex("// ====", 0, enc.rindex("// ====", 0, b))
    body = enc[a:b].replace('#include "zb_encode2.cuh"', open(os.path.join(csrc, "zb_encode2.cuh")).read().replace("#pragma once", ""))
    body = body.replace('#include "zb_encode3.cuh"', open(os.path.join(csrc, "zb_encode3.cuh")).read().replace("#pragma once", ""))
    dec = open(os.path.join(csrc, "zb_decode.cu")).read()
    da = dec.index("\n", dec.index('#include "zb_common.cuh"')) + 1
    db = dec.index('extern "C" {')
    db = dec.rindex("// ====", 0, dec.rindex("// ====", 0, db))
    dbody = dec[da:db].replace('#include "zb_entropy.cuh"', open(DEC_SRC).read().replace("#pragma once", ""))
    body = dbody + body                                      # the dictionary digest lives with the decoder
    body = re.sub(r"extern __shared__ __align__\(16\) u8 (\w+)\[\];", r"u8* const \1 = simt_dyn_smem;", body)
    text = (LIT_PRELUDE + "#include <cmath>\n#include <vector>\n" + '#include "%s"\n' % os.path.join(csrc, "zb_common.cuh")
            + '#include "%s"\n' % os.path.join(HERE, "simt.h") + "alignas(16) static u8 simt_dyn_smem[256 << 10];\n#define ZB_SIMT_STEP() __syncwarp()\n#define ZB_SIMT_EMULATION 1\n" + body + SIM_WRAPPERS)
    cpp = os.path.join(BUILD, "zs_host.cpp")
    if not (os.path.exists(SIM_LIB) and os.path.exists(cpp) and open(cpp).read() == text
            and os.path.getmtime(SIM_LIB) >= os.path.getmtime(os.path.join(HERE, "simt.h"))):
        open(cpp, "w").write(text)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", SIM_LIB, cpp])
    L = C.CDLL(SIM_LIB)
    L.t_compress_batch.restype = C.c_longlong
    L.t_compress_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                   C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                   C.c_int, C.c_uint32]
    L.t_compress_batch2.restype = C.c_longlong
    L.t_compress_batch2.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                    C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_int, C.c_uint32]
    return L


DSIM_LIB = os.path.join(BUILD, "libzd_sim.so")
DSIM_WRAPPERS = r"""
// The whole decompression path on the CPU, kernel by kernel as zb_api.cu launches them: scan, placement (reduce + scan),
// the lane-per-frame entropy kernel on `n_ctas` CTAs of `warps` warps with `take` frames per warp, both execute kernels,
// checksum verification, finish.  Output: tightly packed bytes + per-frame {offset, length}, status[] per frame.
static int g_block_path = 0;
extern "C" void t_set_block_path(int on) { g_block_path = on; }
// The frame scans (small frames a thread each, big ones a warp each) and the placement, as zb_api.cu runs them before it
// chooses a path: totals_out[0..5] = output, blocks, sequences, literals, any checksum, any window >= ZB_FAR_WINDOW.
extern "C" void t_scan_totals(const u8* src, const u64* seg_off, const u64* seg_len, u32 n, u64* totals_out)
{
    std::vector<ZbSegment> segs(n); for (u32 i = 0; i < n; i++) { segs[i].offset = seg_off[i]; segs[i].length = seg_len[i]; }
    std::vector<ZbFrameInfo> info(n); std::vector<ZbFramePlace> place(n + 1); std::vector<u32> status(n, 0), big(n + 1, 0);
    u64 totals[8] = {0}; u32 const pctas = (n + ZB_PLACE_CTA - 1) / ZB_PLACE_CTA; std::vector<u64> partial(pctas * 4 + 4);
    simt::launch((n + 127) / 128, 128, [&] { zb_scan_frames(src, segs.data(), n, info.data(), (1ull << 27) + 1, big.data()); });
    simt::launch(n < 128 ? (n + 3) / 4 : 32, 128, [&] { zb_scan_frames_big(src, segs.data(), big.data(), info.data()); });
    simt::launch(pctas, ZB_PLACE_CTA, [&] { zb_place_reduce(info.data(), nullptr, n, partial.data()); });
    simt::launch(pctas, ZB_PLACE_CTA, [&] { zb_place_scan(info.data(), nullptr, n, partial.data(), place.data(), totals, status.data()); });
    for (int k = 0; k < 6; k++) totals_out[k] = totals[k];
}
// `chunk_bytes` 0: one chunk of all frames, the entropy kernel on `n_ctas` CTAs of `warps` warps with `take` frames per warp.
// Otherwise the call is cut as run_decompress cuts a call whose output is copied back (zb_chunk_count with this chunk size,
// zb_chunk_cut), and every chunk runs what the launcher runs for it: the lane-per-frame entropy kernel over frames
// [0, cut[k + 1]) from a counter of its own that starts at cut[k], shaped by zb_chunk_shape from the chunk's output bytes
// with `n_ctas` as the SM count (the block path keeps its one entropy launch for all blocks); then the chunk's execute stage
// -- zb_execute_tile + zb_execute over its frames, zb_execute_big over its blocks with a fresh wave, or the pointer-jumping
// rounds over its output bytes -- and its checksums.  The pointer-jumping stage regenerates every frame itself, small ones
// included: as in zb_launch_execute_chase, no tile executor runs in front of it.
// The copy of chunk k overlaps the kernels of chunk k + 1 on the device.  Here the chunk's output range is copied into `out`
// as soon as its kernels are done, and is then overwritten in the working buffer with bytes that differ from every output
// byte (the copy may read at any moment, and no kernel of a later chunk may read or write there).  `out` holds nothing but
// these copies.  The chunk's regenerated sizes are set aside the same way until zb_finish: a later chunk must not decode
// its frames again.  plan (nullable, 3 + 5 * 33 words): n_chunks, bytes of earlier chunks that later chunks wrote, frames
// of earlier chunks that later chunks decoded again; then per chunk {cut, warps, take, ctas, output bytes}, where warps, take
// and ctas are those of the chunk's lane-per-frame entropy launch (0 on the block path, whose one launch is not per chunk).
extern "C" long long t_decompress_batch(const u8* src, const u64* seg_off, const u64* seg_len, u32 n, const u8* dict_raw, u32 dict_n,
                                        u32 n_ctas, u32 warps, u32 take, u8* out, u64 out_cap, u64* out_off, u64* out_len, u32* status_out,
                                        const u64* dst_sizes /* nullable: the decompressed_sizes argument of the batch call */,
                                        u64 chunk_bytes, u64* plan)
{
    static bool tables = false;
    if (!tables) { simt::launch(1, 32, [] { zb_build_default_tables(); }); tables = true; }
    static ZbDictDigest dg; ZbDictDev dict; memset(&dict, 0, sizeof dict);
    if (dict_raw && dict_n) {
        simt::launch(1, 32, [&] { zb_digest_dict(dict_raw, dict_n, &dg); });
        if (dg.status != ZB_OK) return -(long long)dg.status;
        if (dg.has_entropy) {
            dict.content = dict_raw + dg.content_off; dict.content_size = dict_n - dg.content_off; dict.dict_id = dg.dict_id; dict.has_entropy = 1;
            dict.huf = dg.huf; dict.huf_log = dg.huf_log; dict.ll = dg.ll; dict.of = dg.of; dict.ml = dg.ml;
            dict.ll_log = dg.ll_log; dict.of_log = dg.of_log; dict.ml_log = dg.ml_log;
            dict.rep[0] = dg.rep[0]; dict.rep[1] = dg.rep[1]; dict.rep[2] = dg.rep[2];
        } else { dict.content = dict_raw; dict.content_size = dict_n; }
    }
    std::vector<ZbSegment> segs(n); for (u32 i = 0; i < n; i++) { segs[i].offset = seg_off[i]; segs[i].length = seg_len[i]; }
    std::vector<ZbFrameInfo> info(n); std::vector<ZbFramePlace> place(n + 1); std::vector<u32> status(n, 0);
    u64 totals[8] = {0}; u32 const pctas = (n + ZB_PLACE_CTA - 1) / ZB_PLACE_CTA; std::vector<u64> partial(pctas * 4 + 4);
    std::vector<u32> big(n + 1, 0);            // frames above ZB_SCAN_BIG (24 KB in this build) are scanned by a warp each
    simt::launch((n + 127) / 128, 128, [&] { zb_scan_frames(src, segs.data(), n, info.data(), (1ull << 27) + 1, big.data()); });
    simt::launch(n < 128 ? (n + 3) / 4 : 32, 128, [&] { zb_scan_frames_big(src, segs.data(), big.data(), info.data()); });
    simt::launch(pctas, ZB_PLACE_CTA, [&] { zb_place_reduce(info.data(), dst_sizes, n, partial.data()); });
    simt::launch(pctas, ZB_PLACE_CTA, [&] { zb_place_scan(info.data(), dst_sizes, n, partial.data(), place.data(), totals, status.data()); });
    if (totals[0] > out_cap) return -1000;
    std::vector<ZbBlock> blocks(totals[1] + 1); std::vector<ZbSeq> seqs(totals[2] + 2); std::vector<u8> lits(totals[3] + 64);
    std::vector<u64> out_sizes(n, 0); std::vector<u32> ck(n, 0);
    std::vector<u8> dev(totals[0] + 64, 0); u8* const d_out = dev.data();       // the device's output buffer
    std::vector<ZbBlkDesc> bdesc;
    u32 const n_chunks = chunk_bytes ? zb_chunk_count(totals[0], n, true, chunk_bytes) : 1;
    std::vector<u32> cut(n_chunks + 1); for (u32 k = 0; k <= n_chunks; k++) cut[k] = zb_chunk_cut(n, k, n_chunks);
    if (g_block_path) {          // a lane per BLOCK: zb_scan_blocks -> zb_entropy_blocks -> zb_resolve_blocks -> zb_patch_blocks
        u64 const nb = totals[1];
        u32 const btake = chunk_bytes ? 3 : (take > 3 ? 3 : take);
        u32 bctas = n_ctas; if (chunk_bytes) { u64 const need = (nb + 7 * btake - 1) / (7 * btake); if (bctas > need) bctas = (u32)need; if (bctas == 0) bctas = 1; }
        u32 counter = 0;
        bdesc.resize(nb + 1); std::vector<ZbBlkExit> bexit(nb + 1); std::vector<u32> erep(3 * (nb + 1)); std::vector<u64> fend(n);
        simt::launch((n + 63) / 64, 64, [&] { zb_scan_blocks(src, segs.data(), n, place.data(), dict, status.data(), bdesc.data(), fend.data(), big.data()); });
        simt::launch(n < 128 ? (n + 3) / 4 : 32, 128, [&] { zb_scan_blocks_big(src, segs.data(), big.data(), place.data(), dict, status.data(), bdesc.data(), fend.data()); });
        simt::launch(bctas, 7 * 32, [&] { zb_entropy_blocks<7>(src, bdesc.data(), (u32)nb, blocks.data(), seqs.data(), lits.data(), &counter, dict, status.data(), bexit.data(), btake); });
        simt::launch((n + 63) / 64, 64, [&] { zb_resolve_blocks(src, segs.data(), n, place.data(), info.data(), dst_sizes, blocks.data(), bdesc.data(), bexit.data(), fend.data(), dict, status.data(), out_sizes.data(), ck.data(), erep.data()); });
        if (nb) simt::launch((unsigned)((nb + 7) / 8), 256, [&] { zb_patch_blocks(blocks.data(), bdesc.data(), nb, seqs.data(), erep.data(), dict, status.data()); });
    }
    std::vector<u32> ptr(g_block_path == 2 ? totals[0] + 16 : 0);
    u64 changed_bytes = 0, redone = 0;
    std::vector<u64> sizes_aside(n);
    std::vector<u8> copy(totals[0] + 64, 0);           // what the copy stream took, chunk by chunk
    auto poison = [](u64 p) { return (u8)(1 + p % 251); };
    for (u32 k = 0; k < n_chunks; k++) {
        u32 const f0 = cut[k], f1 = cut[k + 1];
        u64 const lo = n_chunks > 1 ? place[f0].dst_off : 0, hi = n_chunks > 1 ? place[f1].dst_off : totals[0];
        u64 const blo = n_chunks > 1 ? place[f0].blk_off : 0, bhi = n_chunks > 1 ? place[f1].blk_off : totals[1];
        ZbChunkShape sh; sh.warps = warps; sh.take = take; sh.ctas = n_ctas;
        if (g_block_path) sh.warps = sh.take = sh.ctas = 0;
        else if (chunk_bytes) sh = zb_chunk_shape(hi - lo, f1 - f0, n_ctas);
        if (!g_block_path) {
            u32 counter = f0;
            if (sh.warps == 8) simt::launch(sh.ctas, 8 * 32, [&] { zb_entropy_decode<8>(src, segs.data(), f1, place.data(), dst_sizes, blocks.data(), seqs.data(), lits.data(), &counter, dict, status.data(), out_sizes.data(), ck.data(), sh.take); });
            else simt::launch(sh.ctas, 7 * 32, [&] { zb_entropy_decode<7>(src, segs.data(), f1, place.data(), dst_sizes, blocks.data(), seqs.data(), lits.data(), &counter, dict, status.data(), out_sizes.data(), ck.data(), sh.take); });
        }
        if (g_block_path == 2) {     // pointer-jumping execute stage (zb_chase_*): init, doubling rounds until nothing changes, gather
            if (hi > lo && bhi > blo) {
                std::fill(ptr.begin() + lo, ptr.begin() + hi, 0xFFFFFFFFu); u32 changed = 0; int rounds = 0;
                simt::launch(3, 256, [&] { zb_chase_init<u32>(src, place.data(), status.data(), blocks.data(), (const ZbBlkDesc*)bdesc.data(), seqs.data(), lits.data(), d_out, ptr.data(), blo, bhi, dict); });
                do { changed = 0; simt::launch(4, 256, [&] { zb_chase_round<u32>(ptr.data(), lo, hi, &changed); }); rounds++; } while (changed && rounds < 72);
                simt::launch(4, 256, [&] { zb_chase_gather<u32>(ptr.data(), d_out, lo, hi, totals[0]); });
            }
        }
        else {
            simt::launch((f1 - f0 + ZB_TILE_WARPS - 1) / ZB_TILE_WARPS, ZB_TILE_WARPS * 32, [&] { zb_execute_tile(src, place.data(), status.data(), blocks.data(), seqs.data(), lits.data(), d_out, f0, f1, dict); });
            if (g_block_path && bhi > blo) {
                std::vector<unsigned long long> w_done(n + 1, 0); std::vector<u32> w_pre(n + 1, 0), w_flag(totals[1] + 1, 0); u32 w_ticket = 0;
                ZbWave w; w.done_pos = w_done.data(); w.pre_blk = w_pre.data(); w.blk_flag = w_flag.data(); w.ticket = &w_ticket;
                simt::launch(3, ZB_BIG_NT, [&] { zb_execute_big(src, place.data(), status.data(), blocks.data(), (const ZbBlkDesc*)bdesc.data(), seqs.data(), lits.data(), d_out,
                                                               blo, bhi, dict, (u64)ZB_TILE_CAP + 1, w); });
            }
            else if (!g_block_path) simt::launch((f1 - f0 + 7) / 8, 256, [&] { zb_execute(src, place.data(), status.data(), blocks.data(), seqs.data(), lits.data(), d_out, f0, f1, dict, (u64)ZB_TILE_CAP + 1); });
        }
        if (totals[4]) simt::launch((f1 - f0 + 127) / 128, 128, [&] { zb_verify_checksums(d_out, place.data(), out_sizes.data(), info.data(), ck.data(), f0, f1, status.data()); });
        if (totals[4]) simt::launch(f1 - f0 < 8 ? f1 - f0 : 8, 256, [&] { zb_verify_checksums_big(d_out, place.data(), out_sizes.data(), info.data(), ck.data(), f0, f1, status.data()); });
        // the copy of the chunk; the working buffer's bytes there are not read again
        for (u64 p = lo; p < hi; p++) { copy[p] = d_out[p]; d_out[p] ^= poison(p); }
        for (u32 f = f0; f < f1; f++) { sizes_aside[f] = out_sizes[f]; out_sizes[f] = ~0ull; }
        if (plan && k < 33) { u64* c = plan + 3 + 5 * k; c[0] = f0; c[1] = sh.warps; c[2] = sh.take; c[3] = sh.ctas; c[4] = hi - lo; }
    }
    for (u64 p = 0; p < totals[0]; p++) changed_bytes += d_out[p] != (u8)(copy[p] ^ poison(p));
    for (u32 f = 0; f < n; f++) { redone += out_sizes[f] != ~0ull; out_sizes[f] = sizes_aside[f]; }
    memcpy(out, copy.data(), totals[0]);
    if (plan) { plan[0] = n_chunks; plan[1] = changed_bytes; plan[2] = redone; }
    std::vector<ZbSegment> out_segs(n); u32 first_error = 0xFFFFFFFFu;
    simt::launch((n + 255) / 256, 256, [&] { zb_finish(place.data(), out_sizes.data(), status.data(), n, out_segs.data(), &first_error); });
    for (u32 i = 0; i < n; i++) { out_off[i] = out_segs[i].offset; out_len[i] = out_segs[i].length; status_out[i] = status[i]; }
    return (long long)totals[0];
}
"""


def build_decode_sim():
    """Host build of ALL decompression kernels (zb_decode.cu + zb_entropy.cuh up to the launchers) on tests/simt.h."""
    import re
    os.makedirs(BUILD, exist_ok=True)
    csrc = os.path.join(ROOT, "python_zstandard_b200", "csrc")
    dec = open(os.path.join(csrc, "zb_decode.cu")).read()
    a = dec.index('#include "zb_common.cuh"')
    a = dec.index("\n", a) + 1
    b = dec.index('extern "C" {')
    b = dec.rindex("// ====", 0, dec.rindex("// ====", 0, b))
    body = dec[a:b].replace('#include "zb_entropy.cuh"', open(DEC_SRC).read().replace("#pragma once", ""))
    body = re.sub(r"extern __shared__ __align__\(16\) u8 (\w+)\[\];", r"u8* const \1 = simt_dyn_smem;", body)
    text = (LIT_PRELUDE + "#include <cmath>\n#include <vector>\n" + '#include "%s"\n' % os.path.join(csrc, "zb_common.cuh")
            + '#include "%s"\n' % os.path.join(HERE, "simt.h") + "alignas(16) static u8 simt_dyn_smem[256 << 10];\n#define ZB_SCAN_BIG 24000u\n#define ZB_XXH_BIG 50000u\n" + body + DSIM_WRAPPERS)
    cpp = os.path.join(BUILD, "zd_sim.cpp")
    if not (os.path.exists(DSIM_LIB) and os.path.exists(cpp) and open(cpp).read() == text
            and os.path.getmtime(DSIM_LIB) >= os.path.getmtime(os.path.join(HERE, "simt.h"))):
        open(cpp, "w").write(text)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", DSIM_LIB, cpp])
    L = C.CDLL(DSIM_LIB)
    L.t_decompress_batch.restype = C.c_longlong
    L.t_decompress_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32,
                                     C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_uint64, C.c_void_p]
    L.t_scan_totals.restype = None
    L.t_scan_totals.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    return L


KERNEL_LIB = os.path.join(BUILD, "libzk_host.so")
KERNEL_SHIMS = r"""
// one emulated thread (lane 0 of warp 0 of CTA 0): warp votes and shuffles see only that lane
struct ZbDim3 { unsigned x, y, z; };
static ZbDim3 zb_tid = {0, 0, 0}, zb_bid = {0, 0, 0}, zb_bdim = {256, 1, 1};
#define threadIdx zb_tid
#define blockIdx zb_bid
#define blockDim zb_bdim
static ZbDim3 zb_gdim = {1, 1, 1};
#define gridDim zb_gdim
template <class T, class U, class V> static inline T atomicCAS(T* p, U cmp, V v) { T o = *p; if (o == (T)cmp) *p = (T)v; return o; }
static inline int __any_sync(unsigned, int p) { return p; }
static inline unsigned __ballot_sync(unsigned, int p) { return p ? 1u : 0u; }
template <class T> static inline T __shfl_sync(unsigned, T v, int) { return v; }
template <class T> static inline T __shfl_up_sync(unsigned, T v, int) { return v; }
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int) { return T(0); }     // partner lanes contribute nothing
static inline void __syncwarp(unsigned = 0xFFFFFFFFu) {}
static inline void __syncthreads() {}
static inline long long clock64() { return 0; }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p += v; return o; }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; *p += v; return o; }
alignas(16) unsigned char zb_smem[232448 + 64];
#undef __launch_bounds__
#define __launch_bounds__(...)
"""
KERNEL_WRAPPERS = r"""
// Decode ONE frame with the entropy kernel's own code (one lane), then regenerate the bytes from its block / sequence /
// literal records exactly as the execute kernels read them.  returns the status code; *out_n = bytes produced.
extern "C" int t_decode_frame(const u8* src, u64 n, const u8* dict_raw, u32 dict_n, u8* out, u64 cap, u64* out_n, u32* n_blocks, u32* n_seq)
{
    static bool tables = false;
    if (!tables) { zb_build_default_tables(); tables = true; }
    // the CTA-wide baseline LUT is filled by threads 0..52; only thread 0 exists here
    { u32* const lutLL = (u32*)zb_smem; u32* const lutML = lutLL + 36; for (u32 i = 0; i < 36; i++) lutLL[i] = c_LL_base[i]; for (u32 i = 0; i < 53; i++) lutML[i] = c_ML_base[i]; }
    static ZbDictDigest dg; ZbDictDev dict; memset(&dict, 0, sizeof dict);
    if (dict_raw && dict_n) {
        zb_digest_dict(dict_raw, dict_n, &dg);
        if (dg.status != ZB_OK) return (int)dg.status;
        if (dg.has_entropy) {
            dict.content = dict_raw + dg.content_off; dict.content_size = dict_n - dg.content_off; dict.dict_id = dg.dict_id; dict.has_entropy = 1;
            dict.huf = dg.huf; dict.huf_log = dg.huf_log; dict.ll = dg.ll; dict.of = dg.of; dict.ml = dg.ml;
            dict.ll_log = dg.ll_log; dict.of_log = dg.of_log; dict.ml_log = dg.ml_log;
            dict.rep[0] = dg.rep[0]; dict.rep[1] = dg.rep[1]; dict.rep[2] = dg.rep[2];
        } else { dict.content = dict_raw; dict.content_size = dict_n; }
    }
    ZbSegment seg; seg.offset = 0; seg.length = n;
    ZbFrameInfo fi; zb_scan_frames(src, &seg, 1, &fi, (1ull << 27) + 1, nullptr);
    if (fi.status != ZB_OK) return (int)fi.status;
    u64 const want = fi.content_size != ZB_CONTENT_UNKNOWN ? fi.content_size : cap;
    if (want > cap) return (int)ZB_E_DSTSIZE_TOO_SMALL;
    ZbFramePlace place[2]; memset(place, 0, sizeof place);
    place[0].dst_cap = want; place[1].dst_off = want; place[1].blk_off = fi.n_blocks; place[1].seq_off = fi.n_seq_rec; place[1].lit_off = fi.n_lit;
    ZbBlock* blocks = new ZbBlock[fi.n_blocks + 1]; ZbSeq* seqs = new ZbSeq[fi.n_seq_rec + 2]; u8* lits = new u8[fi.n_lit + 64];
    u32 counter = 0, status = ZB_OK, ck = 0; u64 out_size = 0;
    u64 sizes = want;
    zb_entropy_decode<8>(src, &seg, 1, place, fi.content_size != ZB_CONTENT_UNKNOWN ? &sizes : nullptr, blocks, seqs, lits, &counter, dict, &status, &out_size, &ck, 1);
    *n_blocks = fi.n_blocks; *n_seq = 0;
    // zb_finish's job for one frame; the kernel records errors in status[]
    int rc = (int)status;
    if (rc == ZB_OK) {
        const u8* const dict_end = dict.content + dict.content_size;
        u64 total = 0;
        for (u32 bi = 0; bi < fi.n_blocks; bi++) {
            ZbBlock const& B = blocks[bi];
            u8* const bout = out + B.out_pos;
            if (B.out_pos + B.regen > cap) { rc = (int)ZB_E_DSTSIZE_TOO_SMALL; break; }
            if (B.kind == ZB_BLK_RAW) memcpy(bout, src + B.src_pos, B.regen);
            else if (B.kind == ZB_BLK_RLE) memset(bout, (int)B.lit_byte, B.regen);
            else {
                const u8* const lit = B.lit_kind == ZB_LIT_RAW ? src + B.src_pos : lits + B.src_pos;
                const ZbSeq* const sq = seqs + B.seq_pos;
                *n_seq += B.n_seq;
                for (u32 i = 0; i <= B.n_seq; i++) {
                    u32 const ll = i < B.n_seq ? sq[i + 1].x - sq[i].x : B.n_lit - sq[i].x;
                    for (u32 k = 0; k < ll; k++) bout[sq[i].y + k] = B.lit_kind == ZB_LIT_RLE ? (u8)B.lit_byte : lit[sq[i].x + k];
                    if (i == B.n_seq) break;
                    long long const m0 = (long long)B.out_pos + sq[i].y + ll;
                    for (u32 k = 0; k < sq[i].z; k++) { long long const sp = m0 + k - (long long)sq[i].w; out[m0 + k] = sp < 0 ? dict_end[sp] : out[sp]; }
                }
            }
            total = B.out_pos + B.regen;
        }
        *out_n = total;
    }
    delete[] blocks; delete[] seqs; delete[] lits;
    return rc;
}
"""


def build_entropy_kernel():
    """Host build of the decode kernels' own source (header scan, dictionary digest, the whole lane-per-frame entropy
    kernel) with a single emulated lane, plus a serial execute over the records the kernel writes."""
    os.makedirs(BUILD, exist_ok=True)
    csrc = os.path.join(ROOT, "python_zstandard_b200", "csrc")
    dec = open(os.path.join(csrc, "zb_decode.cu")).read()
    a = dec.index('#include "zb_common.cuh"')
    a = dec.index("\n", a) + 1
    b = dec.index("// K4: LZ copy-execute")
    b = dec.rindex("// ====", 0, b)
    body = dec[a:b].replace('#include "zb_entropy.cuh"', open(DEC_SRC).read().replace("#pragma once", ""))
    d0 = dec.index("__global__ void zb_digest_dict(")
    d1 = dec.index("// ====", d0)
    text = (LIT_PRELUDE + '#include "%s"\n' % os.path.join(csrc, "zb_common.cuh") + KERNEL_SHIMS + body + dec[d0:d1] + KERNEL_WRAPPERS)
    cpp = os.path.join(BUILD, "zk_host.cpp")
    if not (os.path.exists(KERNEL_LIB) and os.path.exists(cpp) and open(cpp).read() == text):
        open(cpp, "w").write(text)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", KERNEL_LIB, cpp])
    L = C.CDLL(KERNEL_LIB)
    L.t_decode_frame.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64,
                                 C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    return L


LIT_LIB = os.path.join(BUILD, "libzl_host.so")
LIT_PRELUDE = r"""
#include <cstdint>
#include <cstring>
// host stand-ins for the few device intrinsics the bit reader uses (PTX shf.{l,r}.{wrap,clamp})
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned s) { unsigned long long v = ((unsigned long long)hi << 32) | lo; return (unsigned)(v >> (s & 31)); }
static inline unsigned __funnelshift_rc(unsigned lo, unsigned hi, unsigned s) { unsigned long long v = ((unsigned long long)hi << 32) | lo; s = s > 32 ? 32 : s; return (unsigned)(s == 32 ? v >> 32 : v >> s); }
static inline unsigned __funnelshift_lc(unsigned lo, unsigned hi, unsigned s) { unsigned long long v = ((unsigned long long)hi << 32) | lo; s = s > 32 ? 32 : s; return (unsigned)((s == 32 ? (v << 31) << 1 : v << s) >> 32); }
static inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
template <class T> static inline T __ldcg(const T* p) { return *p; }
"""
LIT_WRAPPERS = r"""
extern "C" {
// a Huffman-coded literals payload (weights header + 1 or 4 streams, as HUF_compress{1,4}X writes it) -> regen bytes.
// returns 1 on success, 0 on a rejected payload; *hdr_used = bytes of the weights header
int t_literals_decode(u8* dst, u32 regen, const u8* payload, u32 n, int single, u32* hdr_used, u32* table_bytes)
{
    static u8 ws[256]; static u16 cells[4096 + 8]; u32 rank[13], log = 0, nsym = 0;
    u32 const used = zb_huf_weights(ws, payload, n, log, nsym, rank);
    *hdr_used = used;
    if (used == 0 || used >= n) return 0;
    u32 shift, T, base, bytes;
    zb_huf_shape(log, rank, shift, T, base, bytes);
    *table_bytes = bytes;
    zb_huf_fill(cells, ws, log, nsym, rank, shift, base);
    ZbHufTab t; t.cells = cells; t.log = log; t.shift = shift; t.T = T; t.base = base;
    return zb_huf_block(dst, regen, payload + used, n - used, single != 0, t) ? 1 : 0;
}
// the tANS decode table of one sequence stream (kind 0 LL, 1 OF, 2 ML): cells[1 << log], norm is consumed
void t_build_fse(u32* cells, short* norm, u32 max_sym, u32 log, int kind) { zb_build_fse((ZbFseCell*)cells, norm, max_sym, log, kind); }
u32 t_read_ncount(short* norm, u32* max_sym, u32* log, const u8* s, u32 n) { u32 ms = *max_sym, lg = 0; u32 r = zb_read_ncount(norm, ms, lg, s, n); *max_sym = ms; *log = lg; return r; }
}
"""


def build_literals_decoder():
    """Host build of the decoder's literal path: zb_common.cuh (bit reader) + the NCount reader of zb_decode.cu + the
    Huffman weights / split table / 1- and 4-stream decode of zb_entropy.cuh."""
    os.makedirs(BUILD, exist_ok=True)
    csrc = os.path.join(ROOT, "python_zstandard_b200", "csrc")
    dec = open(os.path.join(csrc, "zb_decode.cu")).read()
    a = dec.index("struct ZbFwdR {"); b = dec.index("__global__ void zb_build_default_tables()")
    k0 = dec.index("__constant__ u8 c_LL_bits[36]"); k1 = dec.index("enum { K_LL = 0")
    k1 = dec.index("\n", k1) + 1
    ent = open(DEC_SRC).read()
    c = ent.index("// --- Huffman weights (HUF_readStats_body)"); d = ent.index("// Resolve one sequence-table descriptor")
    text = (LIT_PRELUDE + '#include "%s"\n' % os.path.join(csrc, "zb_common.cuh") + dec[k0:k1] + dec[a:b] + ent[c:d] + LIT_WRAPPERS)
    cpp = os.path.join(BUILD, "zl_host.cpp")
    if not (os.path.exists(LIT_LIB) and os.path.exists(cpp) and open(cpp).read() == text):
        open(cpp, "w").write(text)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", LIT_LIB, cpp])
    L = C.CDLL(LIT_LIB)
    L.t_read_ncount.restype = C.c_uint32
    return L


def build():
    os.makedirs(BUILD, exist_ok=True)
    cpp = os.path.join(BUILD, "ze_host.cpp")
    text = PRELUDE + _extract() + WRAPPERS
    if not (os.path.exists(LIB) and os.path.exists(cpp) and open(cpp).read() == text):
        open(cpp, "w").write(text)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-o", LIB, cpp, "-lm"])
    L = C.CDLL(LIB)
    L.t_write_ncount.restype = C.c_uint32
    L.t_cost.restype = C.c_uint32
    L.t_huf_write_table.restype = C.c_uint32
    return L
