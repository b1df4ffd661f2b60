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
CSRC = os.path.join(ROOT, "python_zstandard_b200", "csrc")
SRC = os.path.join(CSRC, "zb_encode.cu")
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


SIM_SRC = os.path.join(HERE, "simt_kernels.cpp")
SIM_LIB = os.path.join(BUILD, "libzsim.so")
# The CPU build of the kernels: simt.h's runtime, the compressor's lock-step markers, and the decoder's big-frame thresholds
# lowered from 512 KiB / 256 KiB so that small test frames reach the warp-cooperative scans and checksums.
SIM_FLAGS = ["-DZB_SIMT_EMULATION", "-DZB_SIMT_STEP()=__syncwarp()", "-DZB_SCAN_BIG=24000u", "-DZB_XXH_BIG=50000u"]


def build_sim(lib=SIM_LIB, extra=()):
    """Host build of the whole kernel source -- zb_decode.cu and zb_encode.cu as they are, launchers included -- on the mini
    SIMT runtime of tests/simt.h, with the wrappers of tests/simt_kernels.cpp.  `extra`: more g++ flags (sanitizers)."""
    import glob
    import hashlib
    os.makedirs(os.path.dirname(lib), exist_ok=True)
    # -Bsymbolic: the library's calls bind to its own definitions -- simt.h's cudaMemsetAsync and the launchers -- even
    # when the process has loaded the CUDA runtime or libzb200.so, which export the same names
    cmd = (["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-Wl,-Bsymbolic", "-I/usr/local/cuda/include", "-I" + CSRC, "-I" + HERE]
           + SIM_FLAGS + list(extra) + [SIM_SRC])
    h = hashlib.sha256(" ".join(cmd).encode())
    for f in sorted(glob.glob(os.path.join(CSRC, "*.cu*"))) + [SIM_SRC, os.path.join(HERE, "simt.h")]:
        h.update(open(f, "rb").read())
    stamp = lib + ".sha256"
    if not (os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read() == h.hexdigest()):
        tmp = "%s.%d.tmp" % (lib, os.getpid())          # processes that build at once each replace the library whole
        subprocess.check_call(cmd + ["-o", tmp])
        os.replace(tmp, lib)
        open(stamp, "w").write(h.hexdigest())
    L = C.CDLL(lib)
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    L.t_any_calls.restype = C.c_ulonglong
    L.t_compress_batch.restype = C.c_longlong
    L.t_compress_batch.argtypes = [vp, vp, vp, u32, u32, u32, u32, vp, u64, vp, vp, u32, vp, u32, i32, u32]
    L.t_compress_batch2.restype = C.c_longlong
    L.t_compress_batch2.argtypes = [vp, vp, vp, u32, u32, u32, u32, vp, u64, vp, vp, i32, u32]
    L.t_compress_chain_run.restype = C.c_longlong
    L.t_compress_chain_run.argtypes = [vp, vp, vp, u32, u32, u32, vp, u64, vp, vp]
    L.t_decompress_batch.restype = C.c_longlong
    L.t_decompress_batch.argtypes = [vp, vp, vp, u32, vp, u32, u32, u32, u32, vp, u64, vp, vp, vp, vp, u64, vp]
    L.t_scan_totals.restype = None
    L.t_scan_totals.argtypes = [vp, vp, vp, u32, vp]
    L.t_decompress_chain_run.restype = C.c_longlong
    L.t_decompress_chain_run.argtypes = [vp, vp, vp, u32, C.c_char_p, u64, vp, u64, vp, vp, vp, C.POINTER(C.c_int)]
    L.t_freqs.argtypes = [vp, vp, u32, u32, u32, u32, vp]
    L.t_prev.argtypes = [vp, u32, u32, vp]
    L.t_select.argtypes = [vp, vp, u32, u32, u32, u32, u32, u32, vp, vp]
    L.t_finalize.argtypes = [vp, u32, u32, vp, u32, vp]
    L.t_finalize.restype = C.c_longlong
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
