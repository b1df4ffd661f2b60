// zb_encode.cu -- batch zstd compression for sm_90a (H100).
//
// Replaces the per-segment ZSTD_compressStream2(e_end) call of the reference batch path
// (c-ext/compressor.c:1035-1044 -> zstd/zstd.c:29401 -> ZSTD_compress_frameChunk :27545 ->
// ZSTD_compressBlock_internal :27337).  The output is RFC 8878 zstd; it is NOT byte-identical to
// the reference's (the parse is ours), it round-trips through the reference decoder and its size
// is measured against the reference's level 3.
//
// One CTA (4 warps) per <=128 KiB block, persistent over the batch:
//   A  hash links   warp 0 walks the block 32 positions per step; a 2^14-entry u16 hash table in
//                   shared memory gives every position its nearest earlier occurrence with the same
//                   4-byte hash (exact: same-step collisions resolved with match.any) -> dist[] (L2)
//   C  parse        128 lanes, one per 1 KiB unit: lazy-greedy walk over dist[] with repcode tracking
//                   (what ZSTD_compressBlock_doubleFast/_lazy do serially, zstd/zstd.c:31039,:32701)
//   D  compaction   units' sequences -> one list (warp prefix scan), literals gathered
//   E  entropy      symbol codes + histograms (ZSTD_seqToCodes :25647), table choice/normalisation/
//                   NCount header/CTable (ZSTD_buildSequencesStatistics :25717, FSE_normalizeCount :16402,
//                   FSE_writeNCount :16267, FSE_buildCTable_wksp :16005), three FSE state chains in
//                   three warps + prefix-scanned parallel bit packing (ZSTD_encodeSequences_body :21387),
//                   Huffman literals: histogram, length-limited code, weights header, 4 streams packed in
//                   parallel from prefix-scanned code lengths (HUF_compress4X_usingCTable_internal :17925)
//   F  assembly     literals + sequences sections, raw/RLE fallbacks (ZSTD_compressBlock_internal :27337)
// A second kernel lays the frames out tightly (frame header ZSTD_writeFrameHeader :27649).
#include "zb_common.cuh"

// A kernel's dynamic shared memory.  The CPU build of these sources (ZB_SIMT_EMULATION, tests/simt.h) runs one CTA at a time
// and points every kernel at simt.h's static buffer.  Defined with the kernels rather than in zb_common.cuh, and word for word
// the same in zb_decode.cu and zb_encode.cu: host builds of the kernel text that define ZB_SIMT_EMULATION after that header,
// or that rewrite this declaration line, get the CPU form too.
#ifdef ZB_SIMT_EMULATION
#define ZB_DYN_SMEM(name) u8* const name = simt_dyn_smem;
#else
#define ZB_DYN_SMEM(name) extern __shared__ __align__(16) u8 name[];
#endif

// Lock-step marker for the CPU emulation of tests/simt.h (fibers run ahead between warp collectives; the hardware does not).
// Expands to nothing in the device build.
#ifndef ZB_SIMT_STEP
#define ZB_SIMT_STEP()
#endif

#define ZE_THREADS   128
#define ZE_HLOG      14
#define ZE_UNIT      1024                // bytes per parse lane ...
// ... except in batches of small blocks: a 1 KiB record would be parsed by ONE lane (585 K of 745 K cycles per record on the
// config-4 workload).  When no block of a call exceeds ZE_SMALL_MAX bytes the launcher takes the UNIT = 256 instantiation,
// which puts four lanes on such a record; matches end at unit borders, which costs size (CPU build of the kernel, against
// the reference: dictionary records -0.8 % -> +0.5 %, 1-2 KiB text +0.4 % -> +1.0 %; 128-byte units: +2.2 % / +1.8 %).
#define ZE_UNIT_SMALL 256
#ifndef ZE_SMALL_MAX
#define ZE_SMALL_MAX  2048
#endif
#define ZE_UNIT_SEQ  257                 // max sequences of a unit (+1)
#define ZE_MAXSEQ    32768
#define ZE_BLOCK     (128u << 10)

__constant__ u8 e_LL_bits[36] = {0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,1,1,1,1,2,2,3,3,4,6,7,8,9,10,11,12,13,14,15,16};
__constant__ u8 e_ML_bits[53] = {0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,
                                 1,1,1,1,2,2,3,3,4,4,5,7,8,9,10,11,12,13,14,15,16};
__constant__ u32 e_LL_base[36] = {0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,16,18,20,22,24,28,32,40,48,64,
                                  0x80,0x100,0x200,0x400,0x800,0x1000,0x2000,0x4000,0x8000,0x10000};
__constant__ u32 e_ML_base[53] = {3,4,5,6,7,8,9,10,11,12,13,14,15,16,17,18,19,20,21,22,23,24,25,26,27,28,29,30,31,32,33,34,
                                  35,37,39,41,43,47,51,59,67,83,99,0x83,0x103,0x203,0x403,0x803,0x1003,0x2003,0x4003,0x8003,0x10003};
__constant__ short e_LL_defnorm[36] = {4,3,2,2,2,2,2,2,2,2,2,2,2,1,1,1,2,2,2,2,2,2,2,2,2,3,2,1,1,1,1,1,-1,-1,-1,-1};
__constant__ short e_ML_defnorm[53] = {1,4,3,2,2,2,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,
                                       1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1,-1,-1};
__constant__ short e_OF_defnorm[29] = {1,1,1,1,1,1,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1};

// ---------------------------------------------------------------------------
// work description
// ---------------------------------------------------------------------------
struct ZeBlockJob {        // one <=128 KiB block of one segment
    u64 src_pos;           // byte position of the block in src
    u32 size;              // block bytes
    u32 seg;               // owning segment
    u32 last;              // last block of its frame
    u32 first;             // first block of its frame
};
struct ZeBlockOut { u32 csize; u32 pad; };     // compressed block bytes (header included) in its slot

struct ZeParams { u32 checksum; u32 content_size; u32 dict_id; u32 level; u32 window_log = 0; };     // window_log: 0 = default (21)

// dictionary as the block compressor sees it: the last <= 32 KiB of the dictionary content act as history
// right before the first block of every frame (restates the "attach dictionary" mode, zstd/zstd.c:25263-25277)
struct ZeDict { const u8* tail; u32 D; u32 pad; const u16* table; const ZbDictDigest* ent; const void* cct; };   // ent: the dictionary's entropy tables (nullptr: none)
struct ZeUpload { const unsigned long long* progress; unsigned long long total; u32* status; };   // progress == nullptr: input already resident

// per-CTA scratch in global memory (L2 resident: reused for every block the CTA processes)
struct ZeScratch {
    u16 dist[ZE_BLOCK + 64];
    uint2 useq[128 * ZE_UNIT_SEQ];      // per-unit sequences {ll | ml << 16, offBase}
    uint2 seq[ZE_MAXSEQ + 8];           // compacted {ll, offBase | ml << 20}
    u8 lit[ZE_BLOCK + 64];
    u8 llc[ZE_MAXSEQ + 8], mlc[ZE_MAXSEQ + 8], ofc[ZE_MAXSEQ + 8];
    u16 sbits[3][ZE_MAXSEQ + 8];        // per sequence and stream: state bits value | count << 12
    u32 bitpos[ZE_MAXSEQ + 8];
    u32 tmp_lit[(ZE_BLOCK + 1024) / 4]; // literals section payload (Huffman streams)
    u32 tmp_seq[(ZE_BLOCK + 1024) / 4]; // sequence bitstream
    u16 distL[ZE_BLOCK + 64];           // dual-table mode: distance to the nearest earlier position with the same 8-byte hash
};
// Prefix mode (content-dictionary chains) needs 32-bit distances and match lengths beyond the 12 bits of the compacted
// record, and a sequence bitstream beyond tmp_seq (30-bit offsets on 4-byte matches); the other modes keep their scratch as
// it is.
#define ZE_PSEQ_BITS 88u                // most bits of one sequence: states 9 + 8 + 9, LL 16, ML 16, OF 30
struct ZePScratch : ZeScratch {
    u32 dist32[ZE_BLOCK + 64];          // distance of the verified index candidate of every position, 0 = none
    u32 seqml[ZE_MAXSEQ + 8];           // match length of compacted sequence i (seq[i] = {ll, offBase})
    u32 seqbits[(ZE_MAXSEQ * ZE_PSEQ_BITS + 32 * 4) / 32 + 4];   // the sequence bitstream (tmp_seq's job in the other modes)
};
static_assert(sizeof(ZePScratch::seqbits) * 8 >= (size_t)ZE_MAXSEQ * ZE_PSEQ_BITS + 26 + 1 + 2 * 32 + 64,
              "the prefix-mode bitstream must hold the worst block: every sequence at its widest, the final states, the zeroed tail");
// one chunk of a chain run as the prefix-mode kernel sees it: its bytes, its index, and those of the chunk in front of it
// (which lies directly in front of it in the run's buffer)
struct ZeChainSeg {
    u64 start;                          // byte position of the chunk in src
    const u32* tab;                     // its index: 2^log u32 slots, the earliest sampled position of every key (two per position)
    const u32* prev_tab;                // the previous chunk's index (nullptr: none)
    u32 len, prev_len, log, prev_log;
};
// The index samples every ZE_CHAIN_STEP-th position (zb_common.cuh).  A slot is keyed on the 8 bytes at a position AND on
// its 4 KiB bucket: in a revision the bytes of position p mostly sit near p in the previous revision, and a lookup probes the
// buckets around p.  Keyed on the bytes alone, the earliest occurrence of a common 8-byte string (indentation, a keyword)
// would answer for all of them.
#define ZE_CHAIN_BUCKET 12u
__device__ __forceinline__ u32 ze_chain_slot(u64 v, u32 pos, u32 log)
{
    return (u32)(((v ^ ((u64)(pos >> ZE_CHAIN_BUCKET) * 0xC2B2AE3D27D4EB4Full)) * 0x9E3779B185EBCA87ull) >> (64 - log));
}
// The same table also keys every sampled position on the 32 bytes at it, whatever the position: this key finds a source
// anywhere in the chunk (content moved, inserted or deleted by any amount).  32 bytes rather than 8, so that the earliest
// occurrence of the key is rarely a repeat of the bytes rather than their source.
#define ZE_CHAIN_FAR 32u

// ---------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ u32 ze_ld32(const u8* p)     // unaligned little-endian 32-bit load (reads the two aligned words)
{
    uintptr_t const a = (uintptr_t)p; const u32* w = (const u32*)(a & ~(uintptr_t)3);
    u32 const sh = (u32)(a & 3) * 8;
    u32 const lo = w[0];
    if (sh == 0) return lo;
    return __funnelshift_r(lo, w[1], sh);
}
// unaligned little-endian 64-bit load built from three aligned 32-bit loads (reads up to 11 bytes past p)
__device__ __forceinline__ u64 ze_ld64(const u8* p)
{
    uintptr_t const a = (uintptr_t)p; const u32* w = (const u32*)(a & ~(uintptr_t)3);
    u32 const sh = (u32)(a & 3) * 8;
    u32 const w0 = w[0], w1 = w[1], w2 = w[2];
    return (u64)__funnelshift_r(w0, w1, sh) | ((u64)__funnelshift_r(w1, w2, sh) << 32);
}
// number of equal leading (little-endian) bytes of two 64-bit words, 0..8
__device__ __forceinline__ u32 ze_common8(u64 a, u64 b)
{
    u64 const x = a ^ b; u32 const lo = (u32)x, hi = (u32)(x >> 32);
    if (lo) return ((u32)__ffs((int)lo) - 1) >> 3;
    if (hi) return 4 + (((u32)__ffs((int)hi) - 1) >> 3);
    return 8;
}
__device__ __forceinline__ u32 ze_hash4(u32 v) { return (v * 2654435761u) >> (32 - ZE_HLOG); }
// length of the common prefix of a[0..) and b[0..), at most `limit` bytes
__device__ __forceinline__ u32 ze_count(const u8* a, const u8* b, u32 limit)
{
    u32 m = 0;
    while (m + 4 <= limit) { u32 const x = ze_ld32(a + m) ^ ze_ld32(b + m); if (x) return m + ((u32)__ffs((int)x) - 1) / 8; m += 4; }
    while (m < limit && a[m] == b[m]) m++;
    return m;
}
__device__ __forceinline__ u32 ze_hibit(u32 v) { return 31 - __clz(v); }
// the chain index's position-free key (ZE_CHAIN_FAR bytes at p)
__device__ __forceinline__ u32 ze_chain_far_slot(const u8* p, u32 log)
{
    u64 const h = ((((ze_ld64(p) * 0x9E3779B185EBCA87ull) ^ ze_ld64(p + 8)) * 0xC2B2AE3D27D4EB4Full ^ ze_ld64(p + 16)) * 0x165667B19E3779F9ull
                   ^ ze_ld64(p + 24)) * 0x27D4EB2F165667C5ull;
    return (u32)(h >> (64 - log));
}

__device__ __forceinline__ u32 ze_ll_code(u32 ll)       // ZSTD_LLcode, zstd/zstd.c:19738
{
    if (ll < 16) return ll;
    if (ll > 63) return ze_hibit(ll) + 19;
    u32 c = 16; while (c < 35 && ll >= e_LL_base[c + 1]) c++; return c;
}
__device__ __forceinline__ u32 ze_ml_code(u32 mlb)      // ZSTD_MLcode (mlb = matchLength - 3), zstd/zstd.c:19755
{
    if (mlb < 32) return mlb;
    if (mlb > 127) return ze_hibit(mlb) + 36;
    u32 c = 32; while (c < 52 && mlb + 3 >= e_ML_base[c + 1]) c++; return c;
}

// block-wide exclusive scan of one u32 per thread (128 threads); returns exclusive prefix, total in `total`
__device__ __forceinline__ u32 ze_block_scan(u32 v, u32* s_warp, u32& total)
{
    u32 const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 x = v;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { u32 y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= (u32)d) x += y; }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    u32 base = 0;
    #pragma unroll
    for (u32 w = 0; w < ZE_THREADS / 32; w++) { u32 t = s_warp[w]; if (w < warp) base += t; }
    total = s_warp[0] + s_warp[1] + s_warp[2] + s_warp[3];
    __syncthreads();
    return base + x - v;
}

// LSB-first bit writer into a zeroed u32 array, shared by many threads (atomicOr on boundary words)
__device__ __forceinline__ void ze_put_bits(u32* words, u32 bitpos, u32 value, u32 nb)
{
    if (!nb) return;
    u32 const w = bitpos >> 5, sh = bitpos & 31;
    u64 const v = (u64)(value & (nb >= 32 ? 0xFFFFFFFFu : ((1u << nb) - 1))) << sh;
    atomicOr(&words[w], (u32)v);
    if (sh + nb > 32) atomicOr(&words[w + 1], (u32)(v >> 32));
}

// ---------------------------------------------------------------------------
// FSE compression tables in shared memory
// ---------------------------------------------------------------------------
struct ZeCTable {
    u16 state[512];          // next-state table, sorted by symbol (FSE_buildCTable_wksp "tableU16")
    int dnb[56];             // deltaNbBits per symbol
    int dfs[56];             // deltaFindState per symbol
    u32 log;
    u32 mode;                // 0 predefined, 1 RLE, 2 compressed
    u32 rle_sym;
    u32 hdr_bytes;           // NCount / RLE byte count
    u8 hdr[64];
};

// restates FSE_buildCTable_wksp (zstd/zstd.c:16005-16155); serial, one thread; tmp: 512 bytes
__device__ static void ze_build_ctable(ZeCTable& ct, const short* norm, u32 max_sym, u32 log, u8* tmp_sym)
{
    u32 const size = 1u << log, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
    u16 cumul[58]; u32 high = size - 1;
    cumul[0] = 0;
    for (u32 u = 1; u <= max_sym + 1; u++) {
        if (norm[u - 1] == -1) { cumul[u] = cumul[u - 1] + 1; tmp_sym[high--] = (u8)(u - 1); }
        else cumul[u] = cumul[u - 1] + (u16)norm[u - 1];
    }
    u32 pos = 0;
    for (u32 s = 0; s <= max_sym; s++) {
        int const c = norm[s];
        for (int i = 0; i < c; i++) { tmp_sym[pos] = (u8)s; do pos = (pos + step) & mask; while (pos > high); }
    }
    for (u32 u = 0; u < size; u++) { u32 const s = tmp_sym[u]; ct.state[cumul[s]++] = (u16)(size + u); }
    u32 total = 0;
    for (u32 s = 0; s <= max_sym; s++) {
        int const c = norm[s];
        if (c == 0) { ct.dnb[s] = (int)(((log + 1) << 16) - size); ct.dfs[s] = 0; }
        else if (c == -1 || c == 1) { ct.dnb[s] = (int)((log << 16) - size); ct.dfs[s] = (int)total - 1; total++; }
        else {
            u32 const maxBitsOut = log - ze_hibit((u32)c - 1), minStatePlus = (u32)c << maxBitsOut;
            ct.dnb[s] = (int)((maxBitsOut << 16) - minStatePlus); ct.dfs[s] = (int)total - c; total += (u32)c;
        }
    }
    ct.log = log;
}

// restates FSE_writeNCount_generic (zstd/zstd.c:16175-16262); returns bytes written
__device__ static u32 ze_write_ncount(u8* out, const short* norm, u32 max_sym, u32 log)
{
    u32 const alphabet = max_sym + 1; int const size = 1 << log;
    int remaining = size + 1, threshold = size, nbBits = (int)log + 1;
    u64 bits = 0; int bc = 0; u32 o = 0, symbol = 0; int prev0 = 0;
    bits |= (u64)(log - 5); bc = 4;
    while (symbol < alphabet && remaining > 1) {
        if (prev0) {
            u32 start = symbol;
            while (symbol < alphabet && !norm[symbol]) symbol++;
            if (symbol == alphabet) break;
            while (symbol >= start + 24) { start += 24; bits |= (u64)0xFFFF << bc; bc += 16; while (bc >= 16) { out[o++] = (u8)bits; out[o++] = (u8)(bits >> 8); bits >>= 16; bc -= 16; } }
            while (symbol >= start + 3) { start += 3; bits |= (u64)3 << bc; bc += 2; }
            bits |= (u64)(symbol - start) << bc; bc += 2;
            while (bc >= 16) { out[o++] = (u8)bits; out[o++] = (u8)(bits >> 8); bits >>= 16; bc -= 16; }
        }
        {
            int count = norm[symbol++];
            int const mx = (2 * threshold - 1) - remaining;
            remaining -= count < 0 ? -count : count;
            count++;
            if (count >= threshold) count += mx;
            bits |= (u64)(u32)count << bc; bc += nbBits; bc -= (count < mx);
            prev0 = (count == 1);
            while (remaining < threshold) { nbBits--; threshold >>= 1; }
        }
        while (bc >= 16) { out[o++] = (u8)bits; out[o++] = (u8)(bits >> 8); bits >>= 16; bc -= 16; }
    }
    out[o] = (u8)bits; out[o + 1] = (u8)(bits >> 8);
    o += (u32)(bc + 7) / 8;
    return o;
}

// normalise a histogram to sum 2^log with every present symbol >= 1.  Our own rounding rule
// (proportional, remainder to the most frequent symbol); FSE_normalizeCount (zstd/zstd.c:16402)
// solves the same constraint.  returns false if it cannot (then the caller uses another mode).
__device__ static bool ze_normalize(short* norm, const u32* count, u32 max_sym, u32 total, u32 log)
{
    u32 const size = 1u << log; int used = 0; u32 largest = 0, largest_c = 0;
    u64 const scale = ((u64)size << 20) / total;
    for (u32 s = 0; s <= max_sym; s++) {
        u32 const c = count[s];
        if (!c) { norm[s] = 0; continue; }
        u32 p = (u32)(((u64)c * scale + (1u << 19)) >> 20);
        if (p == 0) p = 1;
        norm[s] = (short)p; used += (int)p;
        if (c > largest_c) { largest_c = c; largest = s; }
    }
    int const diff = (int)size - used;
    if ((int)norm[largest] + diff < 1) {
        // too many rare symbols rounded up: take the excess from the biggest ones, one at a time
        int need = -diff;
        for (int guard = 0; guard < 4096 && need > 0; guard++) {
            u32 best = 0; int bestv = 0;
            for (u32 s = 0; s <= max_sym; s++) if (norm[s] > bestv) { bestv = norm[s]; best = s; }
            if (bestv <= 1) return false;
            norm[best]--; need--;
        }
        return need == 0;
    }
    norm[largest] = (short)(norm[largest] + diff);
    return true;
}

// approximate cost in bits (x256) of coding `count` with distribution norm at 2^log
__device__ static u32 ze_cost(const u32* count, const short* norm, u32 max_sym, u32 log)
{
    float bits = 0.f;
    for (u32 s = 0; s <= max_sym; s++) {
        if (!count[s]) continue;
        int n = norm[s]; if (n == -1) n = 1;
        if (n <= 0) return 0xFFFFFFFFu;
        bits += (float)count[s] * ((float)log - __log2f((float)n));
    }
    return (u32)(bits + 0.5f);
}

// choose mode + build everything for one symbol stream (LL, OF or ML).  One thread.
__device__ static void ze_make_table(ZeCTable& ct, const u32* count, u32 max_sym_kind, u32 nseq, u32 max_log, u32 def_log,
                                     const short* defnorm, u32 def_max, u8* tmp_sym,
                                     const short* dictnorm = nullptr, u32 dict_max = 0, u32 dict_log = 0, const ZeCTable* prebuilt = nullptr)
{
    u32 max_sym = 0, present = 0, most = 0;
    for (u32 s = 0; s <= max_sym_kind; s++) if (count[s]) { max_sym = s; present++; if (count[s] > most) most = count[s]; }
    short norm[56];
    ct.hdr_bytes = 0;
    if (most == nseq && nseq > 2) {                       // one symbol only: RLE (ZSTD_selectEncodingType, zstd/zstd.c:21262)
        ct.mode = 1; ct.rle_sym = max_sym; ct.hdr[0] = (u8)max_sym; ct.hdr_bytes = 1; ct.log = 0;
        for (u32 s = 0; s <= max_sym_kind; s++) { ct.dnb[s] = 0; ct.dfs[s] = 0; }
        ct.state[0] = 1;                                  // size + 0
        return;
    }
    // predefined table usable?  every present symbol must have a cell in it
    bool def_ok = max_sym <= def_max;
    if (def_ok) for (u32 s = 0; s <= max_sym; s++) if (count[s] && defnorm[s] == 0) def_ok = false;
    u32 cost_def = 0xFFFFFFFFu;
    if (def_ok) { short dn[56]; for (u32 s = 0; s <= def_max; s++) dn[s] = defnorm[s]; cost_def = ze_cost(count, dn, max_sym, def_log); }
    // compressed table: log as FSE_optimalTableLog (zstd/zstd.c:16308)
    u32 log = max_log;
    if (nseq > 1) {
        u32 const maxBitsSrc = ze_hibit(nseq - 1) >= 2 ? ze_hibit(nseq - 1) - 2 : 0;
        u32 minBits = ze_hibit(nseq) + 1; u32 const mb2 = ze_hibit(max_sym ? max_sym : 1) + 2; if (mb2 < minBits) minBits = mb2;
        if (maxBitsSrc < log) log = maxBitsSrc;
        if (log < minBits) log = minBits;
        if (log < 5) log = 5;
        if (log > max_log) log = max_log;
    }
    u32 cost_cmp = 0xFFFFFFFFu; u32 nc_bytes = 0;
    bool ok = nseq >= 32 && (1u << log) >= present && ze_normalize(norm, count, max_sym, nseq, log);
    if (ok) { nc_bytes = ze_write_ncount(ct.hdr, norm, max_sym, log); cost_cmp = ze_cost(count, norm, max_sym, log) + nc_bytes * 8; }
    // the dictionary's table ("repeat" mode in the first block of a frame, ZSTD_selectEncodingType's set_repeat, zstd/zstd.c:21283):
    // no header at all, so it wins on the short records dictionaries are made for
    if (dictnorm && max_sym <= dict_max) {
        short dn[56]; for (u32 s = 0; s < 56; s++) dn[s] = s <= dict_max ? dictnorm[s] : 0;
        u32 const cost_rep = ze_cost(count, dn, max_sym, dict_log);
        u32 sum = 0; for (u32 s = 0; s <= dict_max; s++) sum += dn[s] == -1 ? 1u : (dn[s] > 0 ? (u32)dn[s] : 0u);
        if (sum == (1u << dict_log) && dict_log <= max_log && cost_rep != 0xFFFFFFFFu && cost_rep <= cost_def && cost_rep <= (ok ? cost_cmp : 0xFFFFFFFFu)) {
            if (prebuilt && prebuilt->mode == 3) {              // built once per dictionary (zb_dict_ctables): a copy instead of a 512-cell spread per record
                const uint4* const src4 = (const uint4*)prebuilt; uint4* const dst4 = (uint4*)&ct;
                for (u32 i = 0; i < sizeof(ZeCTable) / 16; i++) dst4[i] = src4[i];
            } else {
                ze_build_ctable(ct, dn, dict_max, dict_log, tmp_sym);
                for (u32 s = dict_max + 1; s < 56; s++) { ct.dnb[s] = 0; ct.dfs[s] = 0; }
            }
            ct.mode = 3; ct.hdr_bytes = 0;
            return;
        }
    }
    if (ok && cost_cmp < cost_def) {
        ct.mode = 2; ct.hdr_bytes = nc_bytes; ze_build_ctable(ct, norm, max_sym, log, tmp_sym);
        for (u32 s = max_sym + 1; s < 56; s++) { ct.dnb[s] = 0; ct.dfs[s] = 0; }
        return;
    }
    if (!def_ok) {     // neither fits (tiny block with a symbol outside the predefined alphabet): flat table over present symbols
        u32 lg = 5; while ((1u << lg) < present) lg++;
        u32 k = 0, per = (1u << lg) / present, extra = (1u << lg) - per * present;
        for (u32 s = 0; s <= max_sym; s++) { norm[s] = count[s] ? (short)(per + (k < extra ? 1 : 0)) : 0; if (count[s]) k++; }
        ct.mode = 2; ct.hdr_bytes = ze_write_ncount(ct.hdr, norm, max_sym, lg); ze_build_ctable(ct, norm, max_sym, lg, tmp_sym);
        for (u32 s = max_sym + 1; s < 56; s++) { ct.dnb[s] = 0; ct.dfs[s] = 0; }
        return;
    }
    ct.mode = 0; { short dn[56]; for (u32 s = 0; s <= def_max; s++) dn[s] = defnorm[s]; ze_build_ctable(ct, dn, def_max, def_log, tmp_sym); }
    for (u32 s = def_max + 1; s < 56; s++) { ct.dnb[s] = 0; ct.dfs[s] = 0; }
}

// ---------------------------------------------------------------------------
// Huffman code construction (length-limited to 11 bits), one thread.
// Restates the job of HUF_buildCTable_wksp (zstd/zstd.c:17513): sort, build the tree with two
// queues, limit the depth (HUF_setMaxHeight :17133 -- here by the simple "demote the deepest, pay
// back with the shallowest" repair), assign canonical codes (HUF_buildCTableFromTree :17487).
// ---------------------------------------------------------------------------
struct ZeHuf { u16 code[256]; u8 nb[256]; u32 max_sym; u32 log; };

// canonical values from the code lengths in H.nb: longest codes get the smallest values, symbols ascending within a length
__device__ static void ze_huf_assign(ZeHuf& H, u32 max_sym, u32 maxnb)
{
    u32 per[13]; for (u32 b = 0; b <= 12; b++) per[b] = 0;
    for (u32 s = 0; s <= max_sym; s++) per[H.nb[s]]++;
    u32 val[13]; { u32 mn = 0; for (u32 b = maxnb; b >= 1; b--) { val[b] = mn; mn += per[b]; mn >>= 1; } }
    for (u32 s = 0; s <= max_sym; s++) { H.code[s] = 0; if (H.nb[s]) H.code[s] = (u16)val[H.nb[s]]++; }
    H.max_sym = max_sym; H.log = maxnb;
}

// tree construction from symbols already sorted by (count, symbol) ascending in wk[0..n): two-queue merge, depths,
// depth limit, canonical codes.  One thread.
__device__ static bool ze_huf_from_sorted(ZeHuf& H, const u32* count, u32* wk /* >= 1600 u32 */, u32 n, u32 max_sym)
{
    u32* const sym = wk;                 // [256] symbols sorted by count ascending
    u32* const w = wk + 256;             // [512] node weights
    u16* const parent = (u16*)(wk + 768);// [512]
    for (u32 i = 0; i < n; i++) w[i] = count[sym[i]];
    u32 lo = 0, q = n, qe = n;           // leaves [lo, n), internal nodes [q, qe)
    while ((n - lo) + (qe - q) > 1) {
        u32 a, b;
        if (lo < n && (q >= qe || w[lo] <= w[q])) a = lo++; else a = q++;
        if (lo < n && (q >= qe || w[lo] <= w[q])) b = lo++; else b = q++;
        w[qe] = w[a] + w[b]; parent[a] = (u16)qe; parent[b] = (u16)qe; qe++;
    }
    u32 const root = qe - 1;
    u8* const depth = (u8*)(wk + 1024);  // [512]
    depth[root] = 0;
    for (int i = (int)root - 1; i >= 0; i--) depth[i] = depth[parent[i]] + 1;
    u32 const MAXB = 11;
    // depth limit: clamp, then repair Kraft sum (in units of 2^-MAXB)
    u32 kraft = 0;
    for (u32 i = 0; i < n; i++) { if (depth[i] > MAXB) depth[i] = (u8)MAXB; kraft += 1u << (MAXB - depth[i]); }
    u32 const full = 1u << MAXB;
    while (kraft > full) {               // over-subscribed: lengthen the rarest symbol that is still < MAXB
        bool moved = false;
        for (u32 i = 0; i < n; i++) if (depth[i] < MAXB) { kraft -= 1u << (MAXB - depth[i] - 1); depth[i]++; moved = true; break; }
        if (!moved) return false;
    }
    while (kraft < full) {               // slack: shorten the most frequent symbol that fits
        bool moved = false;
        for (int i = (int)n - 1; i >= 0; i--) { u32 const gain = 1u << (MAXB - depth[i]); if (depth[i] > 1 && kraft + gain <= full) { kraft += gain; depth[i]--; moved = true; break; } }
        if (!moved) break;
    }
    if (kraft != full) return false;
    u32 maxnb = 0; for (u32 i = 0; i < n; i++) if (depth[i] > maxnb) maxnb = depth[i];
    for (u32 s = 0; s < 256; s++) { H.nb[s] = 0; H.code[s] = 0; }
    for (u32 i = 0; i < n; i++) H.nb[sym[i]] = depth[i];
    ze_huf_assign(H, max_sym, maxnb);
    return true;
}

__device__ static bool ze_huf_build(ZeHuf& H, const u32* count, u32* wk /* >= 1600 u32 */)
{
    u32* const sym = wk;
    u32 n = 0, max_sym = 0;
    for (u32 s = 0; s < 256; s++) if (count[s]) { sym[n++] = s; max_sym = s; }
    if (n < 2) return false;
    for (u32 i = 1; i < n; i++) {        // insertion sort by (count, symbol)
        u32 const s = sym[i]; u32 const c = count[s]; int j = (int)i - 1;
        while (j >= 0 && (count[sym[j]] > c)) { sym[j + 1] = sym[j]; j--; }
        sym[j + 1] = s;
    }
    return ze_huf_from_sorted(H, count, wk, n, max_sym);
}

// Huffman tree description: weights, FSE-compressed when that is smaller, else 4-bit (HUF_writeCTable_wksp :17005).
// returns bytes written, 0 if the table cannot be described
__device__ static u32 ze_huf_write_table(u8* out, const ZeHuf& H, ZeCTable& ct, u8* tmp_sym)
{
    u32 const n = H.max_sym;             // weights for symbols 0..max_sym-1, the last one is implied
    u8 wt[256];
    for (u32 s = 0; s < n; s++) wt[s] = H.nb[s] ? (u8)(H.log + 1 - H.nb[s]) : 0;
    // FSE-compress the weights (HUF_compressWeights, zstd/zstd.c:16880): two interleaved states
    u32 fse_bytes = 0;
    if (n > 1) {
        u32 cnt[16]; for (int i = 0; i < 16; i++) cnt[i] = 0;
        u32 mx = 0, most = 0; for (u32 s = 0; s < n; s++) { cnt[wt[s]]++; if (wt[s] > mx) mx = wt[s]; }
        for (u32 s = 0; s <= mx; s++) if (cnt[s] > most) most = cnt[s];
        if (most != n && most != 1) {
            u32 log = 6; { u32 c = ze_hibit(n - 1) >= 2 ? ze_hibit(n - 1) - 2 : 0; if (c < log) log = c; u32 minBits = ze_hibit(n) + 1; u32 const m2 = ze_hibit(mx ? mx : 1) + 2; if (m2 < minBits) minBits = m2; if (log < minBits) log = minBits; if (log < 5) log = 5; if (log > 6) log = 6; }
            short norm[16];
            if (ze_normalize(norm, cnt, mx, n, log)) {
                u32 o = 1 + ze_write_ncount(out + 1, norm, mx, log);
                ze_build_ctable(ct, norm, mx, log, tmp_sym);
                // encode backwards with two states (FSE_compress_usingCTable_generic, zstd/zstd.c:16467)
                u64 acc = 0; u32 nb = 0; u8* p = out + o;
                auto put = [&](u32 v, u32 k) { acc |= (u64)(v & ((1u << k) - 1)) << nb; nb += k; while (nb >= 8) { *p++ = (u8)acc; acc >>= 8; nb -= 8; } };
                auto init = [&](u32 s) { u32 const nbo = (u32)(ct.dnb[s] + (1 << 15)) >> 16; u32 const v = (nbo << 16) - (u32)ct.dnb[s]; return (u32)ct.state[(v >> nbo) + ct.dfs[s]]; };
                auto enc = [&](u32& st, u32 s) { u32 const nbo = (st + (u32)ct.dnb[s]) >> 16; put(st, nbo); st = ct.state[(st >> nbo) + ct.dfs[s]]; };
                u32 ip = n, s1, s2;
                if (n & 1) { s1 = init(wt[--ip]); s2 = init(wt[--ip]); enc(s1, wt[--ip]); }
                else { s2 = init(wt[--ip]); s1 = init(wt[--ip]); }
                while (ip > 0) { enc(s2, wt[--ip]); if (ip > 0) enc(s1, wt[--ip]); }
                put(s2, log); put(s1, log);
                put(1, 1); if (nb) { *p++ = (u8)acc; }
                u32 const total = (u32)(p - out);
                if (total - 1 < 128 && total - 1 < (n + 1) / 2) { out[0] = (u8)(total - 1); fse_bytes = total; }
            }
        }
    }
    if (fse_bytes) return fse_bytes;
    if (n > 128) return 0;
    out[0] = (u8)(128 + (n - 1));
    for (u32 s = 0; s < n; s += 2) out[1 + s / 2] = (u8)((wt[s] << 4) | (s + 1 < n ? wt[s + 1] : 0));
    return 1 + (n + 1) / 2;
}

// ---------------------------------------------------------------------------
// the block kernel
// ---------------------------------------------------------------------------
// per-phase cycle counters (thread 0 of every CTA) exist only in tuning builds (-DZB_PHASE_TIMERS)
#ifdef ZB_PHASE_TIMERS
__device__ unsigned long long g_ze_phase[16];
#define ZE_MARK(k) do { if (tid == 0) { long long const t_ = clock64(); atomicAdd(&g_ze_phase[k], (unsigned long long)(t_ - t_phase)); t_phase = t_; } } while (0)
#else
#define ZE_MARK(k) do { (void)t_phase; } while (0)
#endif
struct ZeShared {
    // The hash heads live only in phase A; the entropy-stage tables and staging are first touched in phase D/E, so
    // the two share storage (36 KB per CTA instead of 51 KB: 6 CTAs per SM instead of 4 -- the kernel is bound by
    // dependent-instruction latency, so resident warps are throughput).
    union {
        u16 head[1 << ZE_HLOG];       // A: hash heads
        struct {
            ZeCTable ct[4];           // LL, OF, ML, Huffman-weight table
            ZeHuf huf;
            u32 wk[1600];
            u8 tmp_sym[3][512];
            u8 lit_hdr_buf[8]; u8 seq_hdr_buf[256];
            u8 huf_tbl[160];
        };
    };
    u32 hist[256];
    u32 hLL[36], hOF[32], hML[56];
    u32 s_warp[8];
    __align__(16) u32 ring[256];      // A: 2 x 512 B input ring
    u16 ucnt[128]; u16 utail[128];
    u32 uoff[128]; u32 ucarry[128];
    u32 lit_treeless;                 // literals coded with the dictionary's Huffman table (no table in the block)
    u32 nseq, nlit, tail_lit, all_same, lit_mode, lit_hdr, lit_bytes, seq_bytes, stream_bits[4], huf_tbl_bytes, seq_hdr_bytes, use_raw, body;
};

__device__ __forceinline__ u32 ze_off_code(u32 off, u32 ll, u32& r0, u32& r1, u32& r2)
{
    // offBase for this match and the history update (ZSTD_updateRep, zstd/zstd.c:19971-19989); 0 = unknown slot
    u32 ob;
    if (ll) {
        if (off == r0) return 1;
        if (off == r1) { r1 = r0; r0 = off; return 2; }
        if (off == r2) { r2 = r1; r1 = r0; r0 = off; return 3; }
        ob = off + 3;
    } else {
        if (off == r1) { r1 = r0; r0 = off; return 1; }
        if (off == r2) { r2 = r1; r1 = r0; r0 = off; return 2; }
        if (r0 > 1 && off == r0 - 1) { r2 = r1; r1 = r0; r0 = off; return 3; }
        ob = off + 3;
    }
    r2 = r1; r1 = r0; r0 = off;
    return ob;
}

// what a unit record keeps of a match's offset: its offBase, or in prefix mode the raw offset (phase D codes it per block);
// the unit's repcode history is updated either way
template <bool PREFIX>
__device__ __forceinline__ u32 ze_rec_off(u32 off, u32 ll, u32& r0, u32& r1, u32& r2)
{
    u32 const ob = ze_off_code(off, ll, r0, r1, r2);
    return PREFIX ? off : ob;
}

// DUAL = the reference's double-fast idea (zstd/zstd.c:31039) in the same 32 KB of shared memory: 2^13 heads keyed on 4
// bytes plus 2^13 heads keyed on 8 bytes; a position takes its 8-byte candidate when that one verifies 8 bytes.  CPU
// model tools/enc_model3.c: 128 KiB text +3.2 % -> -1.6 % against level 3.  Used for level >= 4; the default
// instantiation compiles to the code it had before.
// STATS (dictionary training only): every block coded as a compressed block adds its literal bytes and its LL / ML / OF code
// histograms to stats[0..256), [256..292), [292..345), [345..377) -- the counts ZDICT_countEStats (zstd/zstd.c:53124) takes.
// The pointer is null and unused in the other instantiations.
// PREFIX (content-dictionary chains, DUAL false, UNIT 1 KiB): a block's history is contiguous in front of `in` -- its own chunk
// so far, then the whole previous chunk -- and dict.cct points to the run's ZeChainSeg table (job.seg indexes it).  Phase A
// is a lookup of every position's 8-byte hash in the two chunk indexes (zb_chain_index) instead of the hash links; the
// parse runs as in the other modes on 32-bit distances; the compaction merges matches that continue across unit borders
// and re-derives the repcodes of the whole block; scratch is a ZePScratch array.
template <bool DUAL, u32 UNIT, bool STATS = false, bool PREFIX = false>
__global__ void __launch_bounds__(ZE_THREADS)
zb_compress_blocks(const u8* __restrict__ src, const ZeBlockJob* __restrict__ jobs, u32 n_jobs,
                   ZeScratch* __restrict__ scratch, u8* __restrict__ slots, u64 slot_bytes,
                   ZeBlockOut* __restrict__ outs, u32* __restrict__ work_counter, ZeDict dict, ZeUpload up, u32* __restrict__ stats = nullptr)
{
    ZB_DYN_SMEM(ze_smem_raw);
    ZeShared& S = *(ZeShared*)ze_smem_raw;
    ZeScratch& G = PREFIX ? (ZeScratch&)((ZePScratch*)scratch)[blockIdx.x] : scratch[blockIdx.x];
    ZePScratch& GP = (ZePScratch&)G;            // (PREFIX only)
    u32 const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ u32 s_job;

    for (;;) {
        if (tid == 0) {
            u32 const jn = atomicAdd(work_counter, 1u);
            // Host input still in flight: the upload runs on the copy engine while this kernel is resident and publishes
            // how many bytes have landed.  Jobs are handed out in input order, so the first CTAs start after the first
            // chunk.  Wait for a margin past the block's end: the parse reads a few bytes beyond it, and a cache line
            // fetched before its bytes arrive would stay stale in this SM's L1 for the neighbouring block.
            if (up.progress && jn < n_jobs) {
                unsigned long long const want = jobs[jn].src_pos + jobs[jn].size + 256u;
                unsigned long long const need = want < up.total ? want : up.total;
                long long const t0 = clock64();
                while (*(volatile const unsigned long long*)up.progress < need) {
                    __nanosleep(400);
                    if (clock64() - t0 > 6000000000ll) { atomicExch(up.status, 1u); break; }      // ~3 s: the upload failed; the host reports it
                }
                __threadfence();
            }
            s_job = jn;
        }
        __syncthreads();
        u32 const j = s_job;
        if (j >= n_jobs) return;
        ZeBlockJob const job = jobs[j];
        long long t_phase = clock64();
        const u8* const in = src + job.src_pos;
        // bytes of history in front of the block: the dictionary tail for the first block of a frame; in the two-table mode the
        // last ZE_HIST bytes of the previous block for the others when that block holds at least 64 KiB; otherwise blocks are
        // compressed independently.  The previous job is the block in front of this one in the same frame (zb_cut_blocks), and
        // a block that is not its frame's last one is a full block_max = min(2^window_log, 128 KiB) bytes.  So the history sits
        // inside the frame, and the window is at least 64 KiB, which every offset here stays below (u16 distances).  Blocks
        // cut smaller by window_log < 16 get none: in front of a 1 .. 16 KiB block, 32 KiB would reach out of the frame, and
        // in front of a 32 KiB block the matches would reach up to 64 KiB back through a 32 KiB window.
        constexpr u32 ZE_HIST = 32768;
        bool const hist = DUAL && !job.first && jobs[j - 1].size >= 65536u;
        ZeChainSeg cs = {}; if constexpr (PREFIX) cs = ((const ZeChainSeg*)dict.cct)[job.seg];
        u32 const bpos = PREFIX ? (u32)(job.src_pos - cs.start) : 0u;             // (PREFIX) block position in its chunk
        // PREFIX: everything in front of the block back to the start of the previous chunk is history
        u32 const D = PREFIX ? bpos + cs.prev_len : (job.first ? dict.D : (hist ? ZE_HIST : 0u));
        const u8* const dict_end = (PREFIX || hist) ? in : dict.tail + dict.D;
        bool const dict_first = PREFIX ? false : (DUAL ? job.first != 0 : true);  // dictionary entropy tables / repcodes belong to first blocks only
        bool const skip0 = job.first && D == 0;                    // without a dictionary the reference never uses position 0 as a match source
        u32 const n = job.size;
        constexpr u32 unit = UNIT;                                 // bytes each parse lane owns
        u8* const out = slots + (u64)j * slot_bytes;       // block header (3 bytes) + payload
        __syncthreads();

        // ---------------- trivial blocks
        bool raw = n < 9;
        if (!raw) {   // RLE block? (all bytes equal)
            if (tid == 0) S.all_same = 1;
            __syncthreads();
            u8 const b0 = in[0]; bool same = true;
            for (u32 i = tid; i < n && same; i += ZE_THREADS) if (in[i] != b0) same = false;
            if (!same) S.all_same = 0;
            __syncthreads();
            if (S.all_same && !job.first) {
                if (tid == 0) { u32 const bh = job.last | (1u << 1) | (n << 3); out[0] = (u8)bh; out[1] = (u8)(bh >> 8); out[2] = (u8)(bh >> 16); out[3] = b0; outs[j].csize = 4; }
                __syncthreads();
                continue;
            }
        }
        if (raw) {
            for (u32 i = tid; i < n; i += ZE_THREADS) out[3 + i] = in[i];
            if (tid == 0) { u32 const bh = job.last | (n << 3); out[0] = (u8)bh; out[1] = (u8)(bh >> 8); out[2] = (u8)(bh >> 16); outs[j].csize = 3 + n; }
            __syncthreads();
            continue;
        }

        ZE_MARK(0);
        // ---------------- A: hash links (warp 0); the other warps clear the histograms meanwhile
        if constexpr (!PREFIX) {
        if (D && !hist) { const u32* t32 = (const u32*)dict.table; for (u32 i = tid; i < (1u << ZE_HLOG) / 2; i += ZE_THREADS) ((u32*)S.head)[i] = t32[i]; }
        else for (u32 i = tid; i < (1u << ZE_HLOG) / 2; i += ZE_THREADS) ((u32*)S.head)[i] = 0xFFFFFFFFu;
        }
        for (u32 i = tid; i < 256; i += ZE_THREADS) S.hist[i] = 0;
        if (tid < 36) S.hLL[tid] = 0; if (tid < 32) S.hOF[tid] = 0; if (tid < 56) S.hML[tid] = 0;
        __syncthreads();
        if constexpr (PREFIX) {
            // every position (a thread each) looks its 8 bytes up in the previous chunk's index (the buckets around its own
            // position) and in its own chunk's (its bucket and the one before, only candidates in front of it), and its 32
            // bytes in both indexes without a bucket, which finds sources anywhere in the two chunks; every
            // candidate is verified against the input (up to 32 bytes) and the best becomes the position's distance.  No
            // shared table, so no races: the result does not depend on timing.
            for (u32 p = tid; p < n; p += ZE_THREADS) {
                u32 d = 0, dl = 0;
                if (p + 8 <= n) {
                    u64 const v = ze_ld64(in + p);
                    u32 const cp = bpos + p, bk = cp >> ZE_CHAIN_BUCKET;
                    u32 best = 0, best_len = 7, best_gap = 0xFFFFFFFFu;
                    // candidate at chunk position q (dd bytes back): the longer verified match wins; on a tie the one nearer
                    // to where the position's bytes sat in the previous chunk (gap), then the nearer one
                    auto take = [&](u32 dd, u32 gap) {
                        u32 const m = ze_count(in + p, in + p - dd, 32);
                        if (m > best_len || (m == best_len && best && (gap < best_gap || (gap == best_gap && dd < best)))) { best = dd; best_len = m; best_gap = gap; }
                    };
                    if (cs.prev_tab) {
                        for (u32 b = bk ? bk - 1 : 0; b <= bk + 1; b++) {
                            u32 const q = cs.prev_tab[ze_chain_slot(v, b << ZE_CHAIN_BUCKET, cs.prev_log)];
                            if (q != 0xFFFFFFFFu && q < cs.prev_len && (q >> ZE_CHAIN_BUCKET) == b) take(cp + cs.prev_len - q, q > cp ? q - cp : cp - q);
                        }
                    }
                    for (u32 b = bk ? bk - 1 : 0; b <= bk; b++) {
                        u32 const q = cs.tab[ze_chain_slot(v, b << ZE_CHAIN_BUCKET, cs.log)];
                        if (q < cp && (q >> ZE_CHAIN_BUCKET) == b) take(cp - q, 0xFFFFFFFEu);
                    }
                    if (cp + ZE_CHAIN_FAR <= cs.len) {                 // anywhere in either chunk
                        if (cs.prev_tab) {
                            u32 const q = cs.prev_tab[ze_chain_far_slot(in + p, cs.prev_log)];
                            if (q < cs.prev_len) take(cp + cs.prev_len - q, q > cp ? q - cp : cp - q);
                        }
                        u32 const q = cs.tab[ze_chain_far_slot(in + p, cs.log)];
                        if (q < cp) take(cp - q, 0xFFFFFFFEu);
                    }
                    d = best; dl = best ? best_len : 0u;
                }
                GP.dist32[p] = d; G.distL[p] = (u16)dl;        // (distL: the verified length, for the units' hints below)
            }
            __syncthreads();
        }
        if (!PREFIX && warp == 0) {
            u32 const lt = (1u << lane) - 1;
            volatile u16* const vhead = S.head;      // one warp, converged every step: table accesses stay in program order
            bool const exact = n < 2048;
            // The block is streamed through a 2 x 512-byte shared-memory ring, filled with coalesced 128-bit
            // loads that are issued a whole chunk (16 steps) before their data is needed.
            u32 const Hh = hist ? ZE_HIST : 0u;                          // the link phase walks the history in front of the block too
            const u8* const in0 = in - Hh;
            const u8* const in_al = (const u8*)((uintptr_t)in0 & ~(uintptr_t)15);
            u32 const skew = (u32)(in0 - in_al);
            u32 const span = skew + Hh + n;                              // bytes of the aligned stream that belong to history + block
            auto chunk_ld = [&](u32 c) { u32 const o = c * 512 + lane * 16; return o < span ? *(const uint4*)(in_al + o) : make_uint4(0, 0, 0, 0); };   // aligned 16-byte loads never leave the allocation
            uint4* const ring = (uint4*)S.ring;
            ring[lane] = chunk_ld(0);
            uint4 pend = chunk_ld(1);
            u32 const nchunks = (span + 511) / 512;
            bool const use_dual = DUAL && (D == 0 || hist);              // (the dictionary's precomputed table is a single 2^14 table)
            if constexpr (DUAL) { if (use_dual) {
                // two tables of 2^13 heads: short (4-byte hash) in the lower half, long (8-byte hash) in the upper half.
                // Same branch-free stepping as below, one step at a time.
                volatile u16* const vS = S.head; volatile u16* const vL = S.head + (1u << (ZE_HLOG - 1));
                for (u32 c = 0; c < nchunks; c++) {
                    ring[((c + 1) & 1) * 32 + lane] = pend;
                    pend = chunk_ld(c + 2);
                    __syncwarp();
                    #pragma unroll 2
                    for (u32 k = 0; k < 16; k++) {
                        u32 const q = c * 512 + k * 32 + lane;
                        int const pp = (int)q - (int)skew - (int)Hh;              // block-relative; negative = history
                        u32 const bo = q & 1023;
                        u32 const w0 = S.ring[bo >> 2], w1 = S.ring[((bo >> 2) + 1) & 255], w2 = S.ring[((bo >> 2) + 2) & 255];
                        u32 const v0 = __funnelshift_r(w0, w1, (bo & 3) * 8), v1 = __funnelshift_r(w1, w2, (bo & 3) * 8);
                        bool const vaS = pp >= -(int)Hh && pp + 4 <= (int)n, vaL = pp >= -(int)Hh && pp + 8 <= (int)n;
                        u32 const pv = (u32)(pp + (int)Hh);                       // position in (history + block) space
                        bool const ins = (pv & 0xFFFFu) != 0xFFFFu && !(skip0 && pp == 0);
                        u32 const hS = vaS ? (v0 * 2654435761u) >> (32 - (ZE_HLOG - 1)) : 0;
                        u32 const hL = vaL ? (u32)((((u64)v1 << 32 | v0) * 0xCF1BBCDCB7A56463ull) >> (64 - (ZE_HLOG - 1))) : 0;
                        u32 const oS = vaS ? vS[hS] : 0xFFFFu, oL = vaL ? vL[hL] : 0xFFFFu;
                        ZB_SIMT_STEP();
                        if (vaS && ins) vS[hS] = (u16)pv;
                        if (vaL && ins) vL[hL] = (u16)pv;
                        ZB_SIMT_STEP();
                        if (pp >= 0 && (u32)pp < n) {
                            G.dist[pp] = (u16)(oS != 0xFFFFu ? ((pv - oS) & 0xFFFFu) : 0u);
                            G.distL[pp] = (u16)(oL != 0xFFFFu ? ((pv - oL) & 0xFFFFu) : 0u);
                        }
                    }
                }
            } }
            if (use_dual) { /* done above */ } else
            if (!exact) {
                // Big blocks: a branch-free step (no votes, no same-step resolution: the 32 positions of a step do not
                // see each other, +0.8 % size in the CPU model tools/enc_model2.c), four steps in flight so that the
                // shared-memory round trips of one step hide behind the arithmetic of its neighbours.  dist[] is only
                // a hint (the parse verifies every candidate against the input), so table races cost ratio, not correctness.
                for (u32 c = 0; c < nchunks; c++) {
                    ring[((c + 1) & 1) * 32 + lane] = pend;              // chunk c+1 (requested a chunk ago)
                    pend = chunk_ld(c + 2);
                    __syncwarp();
                    #pragma unroll 1
                    for (u32 k4 = 0; k4 < 16; k4 += 4) {
                        u32 hh[4], pvv[4]; bool va[4], in_[4];
                        #pragma unroll
                        for (u32 u = 0; u < 4; u++) {
                            u32 const q = c * 512 + (k4 + u) * 32 + lane;
                            int const pp = (int)q - (int)skew;
                            u32 const bo = q & 1023;
                            u32 const w0 = S.ring[bo >> 2], w1 = S.ring[((bo >> 2) + 1) & 255];
                            u32 const vcur = __funnelshift_r(w0, w1, (bo & 3) * 8);
                            va[u] = pp >= 0 && (u32)pp + 4 <= n;
                            pvv[u] = (u32)pp + D;
                            in_[u] = va[u] && (pvv[u] & 0xFFFFu) != 0xFFFFu && !(skip0 && pp == 0);
                            hh[u] = va[u] ? ze_hash4(vcur) : 0;
                        }
                        u32 oldv[4];
                        #pragma unroll
                        for (u32 u = 0; u < 4; u++) {
                            oldv[u] = va[u] ? vhead[hh[u]] : 0xFFFFu;
                            ZB_SIMT_STEP();                              // (CPU emulation only: all lanes load before any lane stores, as the hardware does)
                            if (in_[u]) vhead[hh[u]] = (u16)pvv[u];
                            ZB_SIMT_STEP();
                        }
                        #pragma unroll
                        for (u32 u = 0; u < 4; u++) {
                            int const pp = (int)(c * 512 + (k4 + u) * 32 + lane) - (int)skew;
                            u32 const d = oldv[u] != 0xFFFFu ? ((pvv[u] - oldv[u]) & 0xFFFFu) : 0u;      // nearest earlier slot owner, mod 2^16
                            if (pp >= 0 && (u32)pp < n) G.dist[pp] = (u16)d;
                        }
                    }
                }
            } else
            for (u32 c = 0; c < nchunks; c++) {
                ring[((c + 1) & 1) * 32 + lane] = pend;                  // chunk c+1 (requested a chunk ago)
                pend = chunk_ld(c + 2);
                __syncwarp();
                #pragma unroll 4
                for (u32 k = 0; k < 16; k++) {
                    int const pp = (int)(c * 512 + k * 32 + lane) - (int)skew;   // block position of this lane
                    if (__all_sync(0xFFFFFFFFu, pp < 0 || pp >= (int)n)) continue;
                    u32 const p = (u32)pp;
                    bool const valid = pp >= 0 && p + 4 <= n;
                    u32 const bo = (c * 512 + k * 32 + lane) & 1023;     // byte offset in the ring
                    u32 const w0 = S.ring[bo >> 2], w1 = S.ring[((bo >> 2) + 1) & 255];
                    u32 const vcur = __funnelshift_r(w0, w1, (bo & 3) * 8);
                    u32 const h = valid ? ze_hash4(vcur) : 0;
                    u32 const old = valid ? vhead[h] : 0xFFFFu;
                    // Two lanes of this step with the same hash are the exception; match.any costs one round per
                    // distinct value, so it only runs when the table itself shows a collision (a lane reads back
                    // somebody else's position from the slot it just wrote).
                    u32 const pv = p + D;                                        // position in (dictionary tail + block) space
                    bool const ins = valid && (pv & 0xFFFFu) != 0xFFFFu && !(skip0 && p == 0);
                    if (ins) vhead[h] = (u16)pv;
                    // exact same-step resolution (match.any: one round per distinct hash value, ~1.5 M cycles per 128 KiB
                    // block) only for small blocks, where a step is a large share of the input; big blocks accept that the
                    // 32 positions of a step do not see each other (+0.8 % size, CPU model tools/enc_model2.c)
                    bool const lost = exact && ins && vhead[h] != (u16)pv;
                    int cand = -1;                                                // candidate, in the same space
                    if (__any_sync(0xFFFFFFFFu, lost)) {
                        u32 const m = __match_any_sync(0xFFFFFFFFu, valid ? h : (0x10000u + lane));
                        u32 const lower = m & lt;
                        if (lower) { int const lsrc = 31 - __clz(lower); cand = (int)pv - ((int)lane - lsrc); if (skip0 && cand == 0) cand = -1; }
                        else if (old != 0xFFFFu) { cand = (int)((pv & ~0xFFFFu) | old); if (cand >= (int)pv) cand -= 0x10000; }
                        if (ins && (m >> lane) == 1u) vhead[h] = (u16)pv;         // the highest lane of a group owns the slot
                    } else if (old != 0xFFFFu) { cand = (int)((pv & ~0xFFFFu) | old); if (cand >= (int)pv) cand -= 0x10000; }
                    u32 d = 0;
                    if (valid && cand >= 0 && pv - (u32)cand <= 65535u) d = pv - (u32)cand;
                    if (pp >= 0 && p < n) G.dist[p] = (u16)d;
                }
            }
        }
        __syncthreads();
        if constexpr (DUAL) { if (D == 0 || hist) {
            // every position takes its 8-byte-hash candidate when that one really matches 8 bytes (all threads, independent
            // per position); the parse below then sees one candidate per position, as before
            const u32* const Wd = (const u32*)((uintptr_t)in & ~(uintptr_t)3);
            const u32* const Wend = Wd + ((((u32)((uintptr_t)in & 3)) + n + 3) >> 2);
            for (u32 p = tid; p + 8 <= n; p += ZE_THREADS) {
                u32 const dL = G.distL[p];
                if (dL == 0 || dL > p + D) continue;
                const u8* const qa = in + p; const u8* const qb = qa - dL;
                const u32* const wa = (const u32*)((uintptr_t)qa & ~(uintptr_t)3); const u32* const wb = (const u32*)((uintptr_t)qb & ~(uintptr_t)3);
                u32 const sa = (u32)((uintptr_t)qa & 3) * 8, sb = (u32)((uintptr_t)qb & 3) * 8;
                u32 const a0 = wa[0], a1 = wa[1], a2 = wa + 2 < Wend ? wa[2] : 0u, b0 = wb[0], b1 = wb[1], b2 = wb + 2 < Wend ? wb[2] : 0u;
                bool const same = __funnelshift_r(a0, a1, sa) == __funnelshift_r(b0, b1, sb) && __funnelshift_r(a1, a2, sa) == __funnelshift_r(b1, b2, sb);
                if (same) G.dist[p] = (u16)dL;
            }
            __syncthreads();
        } }
        ZE_MARK(1);
        // ---------------- C: parse, one lane per 1 KiB unit.
        // A uniform state machine: every iteration issues ALL of a lane's loads together (current bytes,
        // candidate bytes at ip and ip+1, both repcode candidates, the backward bytes, the next dist
        // entry) and then decides, so a step costs one memory round trip for the whole warp instead of
        // one per divergent path.  Long matches continue in EXTEND iterations, 8 bytes per step.
        {
            auto dist_at = [&](u32 i) -> u32 { if constexpr (PREFIX) return GP.dist32[i]; else return G.dist[i]; };
            u32 const u0 = tid * unit;
            u32 cnt = 0, tail = 0;
            bool alive = u0 < n;
            u32 const end = alive ? min(u0 + unit, n) : 0;
            u32 const ilimit = n >= 8 ? n - 8 : 0;
            u32 ip = u0, anchor = u0, r0 = 0, r1 = 0, r2 = 0;
            if (alive && ip == 0 && skip0) ip = 1;                 // the reference starts its search at position 1 (zstd/zstd.c:31075)
            if (tid == 0 && dict_first && D && dict.ent) { r0 = dict.ent->rep[0]; r1 = dict.ent->rep[1]; r2 = dict.ent->rep[2]; }   // a frame with a dictionary starts from its repcodes (ZSTD_loadCEntropy)
            if constexpr (PREFIX) {
                // A unit starts with a guess of the offset the match that ran to the end of the unit before it had, as both
                // repcodes: in a revision that match usually runs on, the repcode check at the unit's first byte picks it up,
                // and D merges the two halves.  The guess: of the distance to the unit's own place in the previous chunk and
                // the last 16 distinct candidates (verified >= 16 bytes) in front of the unit, the one whose match reaches
                // furthest back from the unit's first byte (on a tie, further ahead).  Records keep raw offsets and D codes
                // them against the true history, so these seeds never reach the output.
                if (alive && u0 + D > 0) {
                    u32 back = 0, guess = 0;
                    auto try_guess = [&](u32 d) {
                        u32 const lim = min(256u, u0 + D - d);
                        const u8* const a = in + u0;
                        u32 k = 0; while (k < lim && a[-1 - (int)k] == a[-1 - (int)k - (int)d]) k++;
                        if (k == lim) k += ze_count(a, a - d, min(256u, n - u0));      // (a tie behind the unit: the longer run ahead)
                        if (k > back) { back = k; guess = d; }
                    };
                    if (cs.prev_len) try_guess(cs.prev_len);                    // the unit's own place in the previous chunk
                    u32 const lo = u0 > 256 ? u0 - 256 : 0; u32 seen = 0;
                    for (u32 p = u0; p-- > lo && seen < 16;) {
                        u32 const d = G.distL[p] >= 16 ? dist_at(p) : 0u;
                        if (!d || d == guess || d > u0 + D) continue;
                        seen++; try_guess(d);
                    }
                    if (guess) r0 = r1 = guess;
                }
            }
            uint2* const rec = G.useq + tid * ZE_UNIT_SEQ;
            u32 mode = 0, m_start = 0, m_off = 0, m_len = 0;
            u32 d0 = 0, d1 = 0;
            if (alive) { d0 = dist_at(ip); d1 = ip + 1 < n ? dist_at(ip + 1) : 0; }
            for (;;) {
                if (alive && mode == 1 && m_start + m_len + 8 > n) {        // the last bytes of a block: finish the match bytewise (no wide reads past the input)
                    while (m_start + m_len < end) {
                        int const q = (int)(m_start + m_len) - (int)m_off;          // source position (negative: dictionary)
                        u8 const b = q >= 0 ? in[q] : dict_end[q];
                        if (in[m_start + m_len] != b) break;
                        m_len++;
                    }
                    u32 const ll = m_start - anchor;
                    rec[cnt++] = make_uint2(ll | (m_len << 16), ze_rec_off<PREFIX>(m_off, ll, r0, r1, r2));
                    ip = m_start + m_len; anchor = ip; mode = 0;
                    d0 = ip < n ? dist_at(ip) : 0; d1 = ip + 1 < n ? dist_at(ip + 1) : 0;
                }
                bool const searching = alive && mode == 0 && ip + 4 <= end && ip < ilimit;   // ... and stops one short of ilimit (:31100-31180)
                bool const extending = alive && mode == 1;
                if (!__any_sync(0xFFFFFFFFu, searching || extending)) break;
                if (alive && !searching && !extending) alive = false;
                // dist[] is a hint: a distance that would reach in front of the history (only a corrupted table could hold one)
                // is dropped here, so that the parse never forms an address outside the block and the dictionary tail
                if (searching) { if (d0 > ip + D) d0 = 0; if (d1 > ip + 1 + D) d1 = 0; }
                // all loads of the step, unconditional (invalid ones alias the current position) and issued
                // back to back as raw aligned words; the funnel shifts that consume them come afterwards
                u64 A = 0, B = 0, C1 = 0, RP = 0, RQ = 0; u32 bka = 0, bkb = 1, d2 = 0, bk_max = 0;
                u32 capB = 64, capC = 64, capP = 64, capQ = 64;
                bool has_c1 = false, has_rp = false, has_rq = false, has_bk = false, ext1 = false, ext2 = false; u64 X2 = 0;
                {
                    u32 const pa = extending ? m_start + m_len : ip;
                    // candidate positions are block-relative and may be negative: -k means k bytes before the
                    // dictionary end.  cap* = bytes that may be compared before that region ends.
                    int const pbi = extending ? (int)pa - (int)m_off : (d0 ? (int)ip - (int)d0 : (int)ip);
                    has_c1 = searching && d1 != 0 && ip + 5 <= end;
                    has_rp = searching && r0 != 0 && (int)ip + 1 - (int)r0 >= -(int)D && ip + 5 <= end;
                    has_rq = searching && anchor == ip && r1 != 0 && (int)ip - (int)r1 >= -(int)D;
                    // EXTEND has no use for the candidate slots, so they fetch the next 16 bytes of both sides (24 bytes per step).
                    // A further window counts only if it lies wholly inside the block and wholly on one side of the dictionary end.
                    // (PREFIX: the history is contiguous with the block, so no window has to stay on one side of its start)
                    ext1 = extending && pa + 16 <= n && (PREFIX || pbi >= 0 || pbi + 16 <= 0);
                    ext2 = ext1 && pa + 24 <= n && (PREFIX || pbi >= 0 || pbi + 24 <= 0);
                    int const pci = has_c1 ? (int)ip + 1 - (int)d1 : (ext1 ? (int)pa + 8 : (int)pa);
                    int const ppi = has_rp ? (int)ip + 1 - (int)r0 : (ext1 ? pbi + 8 : (int)pa);
                    int const pqi = has_rq ? (int)ip - (int)r1 : (ext2 ? (int)pa + 16 : (int)pa);
                    int const pxi = ext2 ? pbi + 16 : (int)pa;
                    capB = !PREFIX && pbi < 0 ? (u32)(-pbi) : 64u; capC = !PREFIX && pci < 0 ? (u32)(-pci) : 64u;
                    capP = !PREFIX && ppi < 0 ? (u32)(-ppi) : 64u; capQ = !PREFIX && pqi < 0 ? (u32)(-pqi) : 64u;
                    u32 const back_room = pbi >= 0 ? (u32)pbi : D - (u32)(-pbi);          // bytes available before the candidate
                    u32 const em = (searching && d0) ? min(4u, min(ip - anchor, back_room)) : 0u;   // bytes that may extend the match backwards
                    has_bk = em != 0; bk_max = em;
                    bool const act = searching || extending;
                    #define ZE_P(x) ((x) >= 0 ? in + (x) : dict_end + (x))
                    const u8* const qa = in + (act ? pa : 0); const u8* const qb = act ? ZE_P(pbi) : in; const u8* const qc = act ? ZE_P(pci) : in;
                    const u8* const qp = act ? ZE_P(ppi) : in; const u8* const qq = act ? ZE_P(pqi) : in; const u8* const qx = act ? ZE_P(pxi) : in;
                    #define ZE_W(q) ((const u32*)((uintptr_t)(q) & ~(uintptr_t)3))
                    #define ZE_S(q) ((u32)((uintptr_t)(q) & 3) * 8)
                    // predicated (not branched) loads: a lane only spends load bandwidth on what it will look at.
                    // A candidate that coincides with the main candidate (same distance) reuses its bytes.
                    // Every lane works in its own unit, so each load instruction costs 32 cache-sector lookups whatever its
                    // width, and this phase is bound by exactly those lookups: an 8-byte window is fetched as the two
                    // aligned 8-byte words that contain it (2 loads instead of 3) and the four bytes in front of a window
                    // come from the one word before it.
                    bool const ldb = extending || (searching && d0 != 0);
                    bool const c_same = has_c1 && d0 != 0 && d1 == d0, p_same = has_rp && d0 != 0 && r0 == d0;
                    bool const ldc = (has_c1 && !c_same) || ext1, ldp = (has_rp && !p_same) || ext1, ldq = has_rq || ext2;
                    uintptr_t const in_lo = (uintptr_t)in & ~(uintptr_t)7, in_hi = (uintptr_t)(in + n);    // block bytes: [in, in + n)
                    // x0..x2 = the three aligned 32-bit words that hold the 8 bytes at q (dictionary pointers have 16 bytes of slack)
                    #define ZE_LD3(q, on, blockptr, x0, x1, x2) \
                        u32 x0, x1, x2; { \
                            const uint2* const w_ = (const uint2*)((uintptr_t)(q) & ~(uintptr_t)7); \
                            bool const on1_ = (on) && (!(blockptr) || (uintptr_t)(w_ + 1) < in_hi); \
                            uint2 const lo_ = (on) ? w_[0] : make_uint2(0u, 0u), hi_ = on1_ ? w_[1] : make_uint2(0u, 0u); \
                            bool const up_ = ((uintptr_t)(q) & 4) != 0; \
                            x0 = up_ ? lo_.y : lo_.x; x1 = up_ ? hi_.x : lo_.y; x2 = up_ ? hi_.y : hi_.x; }
                    ZE_LD3(qa, act, true, a0, a1, a2)
                    ZE_LD3(qb, ldb, pbi >= 0, b0, b1, b2)
                    ZE_LD3(qc, ldc, pci >= 0, c0, c1, c2)
                    ZE_LD3(qp, ldp, ppi >= 0, p0, p1, p2)
                    ZE_LD3(qq, ldq, pqi >= 0, q0, q1, q2)
                    ZE_LD3(qx, ext2, pxi >= 0, x0, x1, x2)
                    // the word in front of the A and B windows (backward extension); never below the block's first word
                    const u32* const wka = ZE_W(qa) - 1; const u32* const wkb = ZE_W(qb) - 1;
                    u32 const ka = (has_bk && (uintptr_t)wka >= in_lo) ? *wka : 0u;
                    u32 const kb = (has_bk && (pbi < 0 || (uintptr_t)wkb >= in_lo)) ? *wkb : 0u;
                    u32 const dn = (searching && ip + 2 < n) ? dist_at(ip + 2) : 0;
                    #define ZE_J(x0, x1, x2, q) ((u64)__funnelshift_r(x0, x1, ZE_S(q)) | ((u64)__funnelshift_r(x1, x2, ZE_S(q)) << 32))
                    A = ZE_J(a0, a1, a2, qa); B = ZE_J(b0, b1, b2, qb); C1 = ZE_J(c0, c1, c2, qc); RP = ZE_J(p0, p1, p2, qp); RQ = ZE_J(q0, q1, q2, qq);
                    X2 = ZE_J(x0, x1, x2, qx);
                    if (c_same) { C1 = B >> 8; capC = capB > 0 ? capB - 1 : 0; }
                    if (p_same) { RP = B >> 8; capP = capB > 0 ? capB - 1 : 0; }
                    bka = __funnelshift_r(ka, a0, ZE_S(qa)); bkb = __funnelshift_r(kb, b0, ZE_S(qb));      // the 4 bytes before ip / before the candidate, nearest on top
                    d2 = dn;
                    if (searching && !d0) B = ~A;
                }
                bool fin = false; u32 f_start = 0, f_off = 0, f_len = 0;
                if (searching) {
                    u32 const room = end - ip;
                    bool found = false, sat = false; u32 start = 0, off = 0, len = 0;
                    if (has_rq && capQ >= 4 && (u32)A == (u32)RQ) {          // immediate repcode match (ll == 0)
                        u32 const c = min(ze_common8(A, RQ), capQ); start = ip; off = r1; len = min(c, room); sat = c == 8 && capQ > 8; found = true;
                    } else if (has_rp && capP >= 4 && (u32)(A >> 8) == (u32)RP) {   // repcode match at ip + 1
                        u32 const c = min(min(ze_common8(A >> 8, RP & 0x00FFFFFFFFFFFFFFull), 7u), capP);
                        start = ip + 1; off = r0; len = min(c, room - 1); sat = c == 7 && capP > 7; found = true;
                    } else if (d0 && capB >= 4 && (u32)A == (u32)B) {
                        u32 const m0 = min(ze_common8(A, B), capB);
                        bool skip = false;
                        if (m0 < 8 && has_c1 && capC >= 4 && (u32)(A >> 8) == (u32)C1) {  // one-step lazy: clearly longer one byte later?
                            u32 const m1 = min(min(ze_common8(A >> 8, C1 & 0x00FFFFFFFFFFFFFFull), 7u), capC);
                            skip = m1 > m0 + 1;
                        }
                        if (!skip) {
                            start = ip; off = d0; len = min(m0, room); sat = m0 == 8 && capB > 8; found = true;
                            if (has_bk) {                                    // backward extension, up to 4 bytes
                                u32 const x = bka ^ bkb; u32 e = x ? ((u32)__clz((int)x) >> 3) : 4u;
                                e = min(e, bk_max);
                                start -= e; len += e;
                            }
                        }
                    }
                    if (found) {
                        if (sat && start + len < end) { mode = 1; m_start = start; m_off = off; m_len = len; }
                        else { fin = true; f_start = start; f_off = off; f_len = len; }
                    } else {
                        u32 const step = 1 + ((ip - anchor) >> 8);
                        ip += step;
                        if (step == 1) { d0 = d1; d1 = d2; }
                        else { d0 = ip < n ? dist_at(ip) : 0; d1 = ip + 1 < n ? dist_at(ip + 1) : 0; }
                    }
                } else if (extending) {
                    u32 const room = end - (m_start + m_len);
                    u32 total = ze_common8(A, B), compared = 8;                      // in EXTEND: C1/RP = bytes 8..15, RQ/X2 = bytes 16..23 of the two sides
                    if (total == 8 && ext1) { total += ze_common8(C1, RP); compared = 16; if (total == 16 && ext2) { total += ze_common8(RQ, X2); compared = 24; } }
                    u32 const c = min(total, capB); u32 const k = min(c, room);
                    m_len += k;
                    if (!(total == compared && capB > total && m_start + m_len < end)) { fin = true; f_start = m_start; f_off = m_off; f_len = m_len; }
                }
                if (fin) {
                    u32 const ll = f_start - anchor;
                    rec[cnt++] = make_uint2(ll | (f_len << 16), ze_rec_off<PREFIX>(f_off, ll, r0, r1, r2));
                    ip = f_start + f_len; anchor = ip; mode = 0;
                    d0 = ip < n ? dist_at(ip) : 0; d1 = ip + 1 < n ? dist_at(ip + 1) : 0;
                }
            }
            if (u0 < n) tail = end - anchor;
            S.ucnt[tid] = (u16)cnt; S.utail[tid] = (u16)tail;
        }
        __syncthreads();

        ZE_MARK(2);
        // ---------------- D: compaction of the units' sequences + literal gather
        u32 nseq;
        if constexpr (PREFIX) {
            // One serial pass: a unit's leading match that continues the previous unit's trailing match (same offset, no
            // literals between) is merged into it -- a revision that is one long match stays one sequence, not one per
            // 1 KiB unit -- and every offset is coded against the block's own repcode history.  Repcodes start as zeros,
            // which match no offset, so every repcode this emits names a slot the decoder holds the same value in.
            if (tid == 0) {
                u32 o = 0, carry = 0, last_off = 0, r0 = 0, r1 = 0, r2 = 0; u32 const units = (n + unit - 1) / unit;
                for (u32 u = 0; u < units; u++) {
                    const uint2* const rec = G.useq + u * ZE_UNIT_SEQ;
                    u32 const c = S.ucnt[u];
                    for (u32 k = 0; k < c; k++) {
                        uint2 const r = rec[k];
                        u32 const ll = (r.x & 0xFFFFu) + (k == 0 ? carry : 0u), ml = r.x >> 16, off = r.y;
                        if (o && ll == 0 && off == last_off) { GP.seqml[o - 1] += ml; continue; }
                        G.seq[o] = make_uint2(ll, off); GP.seqml[o] = ml; o++; last_off = off;
                    }
                    if (c) carry = S.utail[u]; else carry += S.utail[u];
                }
                for (u32 i = 0; i < o; i++) G.seq[i].y = ze_off_code(G.seq[i].y, G.seq[i].x, r0, r1, r2);
                S.nseq = o; S.tail_lit = carry;
            }
            __syncthreads();
            nseq = S.nseq;
        } else {
        if (tid == 0) {
            u32 off = 0, carry = 0; u32 const units = (n + unit - 1) / unit;
            for (u32 u = 0; u < 128; u++) {
                S.uoff[u] = off; S.ucarry[u] = carry;
                if (u < units) { if (S.ucnt[u]) carry = S.utail[u]; else carry += S.utail[u]; off += S.ucnt[u]; }
            }
            S.nseq = off; S.tail_lit = carry;
        }
        __syncthreads();
        nseq = S.nseq;
        {
            u32 const c = S.ucnt[tid], o = S.uoff[tid];
            const uint2* const rec = G.useq + tid * ZE_UNIT_SEQ;
            for (u32 k = 0; k < c; k++) {
                uint2 const r = rec[k];
                u32 ll = r.x & 0xFFFFu; u32 const ml = r.x >> 16;
                if (k == 0) ll += S.ucarry[tid];
                G.seq[o + k] = make_uint2(ll, r.y | (ml << 20));
            }
        }
        __syncthreads();
        }
        // codes, histograms, literal positions; gather literals
        {
            u32 lit_run = 0, src_run = 0;      // running prefix over chunks of 128 sequences
            for (u32 base = 0; base < nseq; base += ZE_THREADS) {
                u32 const i = base + tid; bool const v = i < nseq;
                uint2 const r = v ? G.seq[i] : make_uint2(0, 0);
                u32 const ll = r.x, ml = PREFIX ? (v ? GP.seqml[i] : 0u) : r.y >> 20, ob = PREFIX ? r.y : r.y & 0xFFFFFu;
                u32 tot_l, tot_s;
                u32 const lpos = ze_block_scan(ll, S.s_warp, tot_l) + lit_run;
                u32 const spos = ze_block_scan(ll + ml, S.s_warp, tot_s) + src_run;
                if (v) {
                    u32 const lc = ze_ll_code(ll), mc = ze_ml_code(ml - 3), oc = ze_hibit(ob);
                    G.llc[i] = (u8)lc; G.mlc[i] = (u8)mc; G.ofc[i] = (u8)oc;
                    atomicAdd(&S.hLL[lc], 1u); atomicAdd(&S.hML[mc], 1u); atomicAdd(&S.hOF[oc], 1u);
                    const u8* sp = in + spos; u8* dp = G.lit + lpos;
                    for (u32 k = 0; k < ll; k++) { u8 const b = sp[k]; dp[k] = b; atomicAdd(&S.hist[b], 1u); }
                }
                lit_run += tot_l; src_run += tot_s;
            }
            // last literals of the block
            u32 const tl = n - src_run;
            for (u32 k = tid; k < tl; k += ZE_THREADS) { u8 const b = in[src_run + k]; G.lit[lit_run + k] = b; atomicAdd(&S.hist[b], 1u); }
            if (tid == 0) S.nlit = lit_run + tl;
        }
        __syncthreads();
        u32 const nlit = S.nlit;

        ZE_MARK(3);
        // ---------------- E: entropy tables.  thread 0: LL, 32: OF, 64: ML (own scratch each), 96: literals mode + Huffman code
        if (nseq) {
            const ZbDictDigest* const de = (dict_first && D && dict.ent) ? dict.ent : nullptr;      // first block of a frame that has a full dictionary
            if (tid == 0)  ze_make_table(S.ct[0], S.hLL, 35, nseq, 9, 6, e_LL_defnorm, 35, S.tmp_sym[0], de ? de->c_norm_ll : nullptr, de ? de->c_max_ll : 0, de ? de->ll_log : 0, de && dict.cct ? (const ZeCTable*)dict.cct + 0 : nullptr);
            if (tid == 32) ze_make_table(S.ct[1], S.hOF, 31, nseq, 8, 5, e_OF_defnorm, 28, S.tmp_sym[1], de ? de->c_norm_of : nullptr, de ? de->c_max_of : 0, de ? de->of_log : 0, de && dict.cct ? (const ZeCTable*)dict.cct + 1 : nullptr);
            if (tid == 64) ze_make_table(S.ct[2], S.hML, 52, nseq, 9, 6, e_ML_defnorm, 52, S.tmp_sym[2], de ? de->c_norm_ml : nullptr, de ? de->c_max_ml : 0, de ? de->ml_log : 0, de && dict.cct ? (const ZeCTable*)dict.cct + 2 : nullptr);
        }
        if (tid == 96) {
            S.lit_mode = 0; S.huf_tbl_bytes = 0; S.lit_treeless = 0;
            u32 most = 0; for (u32 s = 0; s < 256; s++) if (S.hist[s] > most) most = S.hist[s];
            const ZbDictDigest* const de = (dict_first && D && dict.ent) ? dict.ent : nullptr;
            if (nlit >= 8 && most == nlit) S.lit_mode = 1;                // RLE literals
            else {
                u32 cost_new = 0xFFFFFFFFu;                              // bytes with a table of this block's own
                if (nlit >= 64) {                                        // ZSTD_minLiteralsToCompress (dfast: 64), zstd/zstd.c:20918
                    if (ze_huf_build(S.huf, S.hist, S.wk)) {
                        u32 const tb = ze_huf_write_table(S.huf_tbl, S.huf, S.ct[3], (u8*)(S.wk + 1200));
                        if (tb) { S.huf_tbl_bytes = tb; S.lit_mode = 2; u32 bits = 0; for (u32 s = 0; s < 256; s++) bits += S.hist[s] * S.huf.nb[s]; cost_new = (bits + 7) / 8 + tb; }
                    }
                }
                // the dictionary's Huffman table ("treeless" literals; with a valid previous table the reference compresses
                // from 7 literals on, ZSTD_minLiteralsToCompress zstd/zstd.c:20918-20930)
                if (de && nlit > 6) {
                    bool ok = true; u32 bits = 0;
                    for (u32 s = 0; s < 256; s++) if (S.hist[s]) { u32 const nb = de->c_huf_nb[s]; if (!nb) ok = false; bits += S.hist[s] * nb; }
                    if (ok && (bits + 7) / 8 <= cost_new) {
                        for (u32 s = 0; s < 256; s++) S.huf.nb[s] = de->c_huf_nb[s];
                        ze_huf_assign(S.huf, de->c_huf_max, de->huf_log);
                        S.huf_tbl_bytes = 0; S.lit_mode = 2; S.lit_treeless = 1;
                    }
                }
            }
        }
        __syncthreads();

        ZE_MARK(4);
        // ---------------- E: literals section payload into tmp_lit
        u32 lit_payload = 0;        // bytes in tmp_lit (Huffman: table + jump table + streams)
        bool const four = nlit >= 256;
        if (S.lit_mode == 2) {
            // estimate first: sum of code lengths
            u32 bits_local = 0;
            for (u32 s = tid; s < 256; s += ZE_THREADS) bits_local += S.hist[s] * S.huf.nb[s];
            u32 tot; ze_block_scan(bits_local, S.s_warp, tot);
            u32 const est = (tot + 7) / 8 + S.huf_tbl_bytes + (four ? 6 + 4 : 1);
            if (est + (nlit >> 6) + 2 >= nlit) { if (tid == 0) S.lit_mode = 0; }   // ZSTD_minGain, zstd/zstd.c:19831
            __syncthreads();
        }
        if (S.lit_mode == 2) {
            u32 const tb = S.huf_tbl_bytes;
            u8* const pl = (u8*)G.tmp_lit;
            u32 const nstreams = four ? 4 : 1;
            u32 const seg = four ? (nlit + 3) / 4 : nlit;
            // zero the staging area that the streams may touch
            u32 const zero_words = (tb + 6 + nlit * 11 / 8 + 64) / 4 + 1;
            for (u32 i = tid; i < zero_words && i < (ZE_BLOCK + 1024) / 4; i += ZE_THREADS) G.tmp_lit[i] = 0;
            __syncthreads();
            for (u32 i = tid; i < tb; i += ZE_THREADS) pl[i] = S.huf_tbl[i];
            // pass 1: stream bit totals
            for (u32 st = 0; st < nstreams; st++) {
                u32 const a = st * seg, b = st == nstreams - 1 ? nlit : a + seg;
                u32 loc = 0; for (u32 i = a + tid; i < b; i += ZE_THREADS) loc += S.huf.nb[G.lit[i]];
                u32 tot; ze_block_scan(loc, S.s_warp, tot);
                if (tid == 0) S.stream_bits[st] = tot;
            }
            __syncthreads();
            // stream byte offsets
            u32 sbyte[4], sbytes[4]; { u32 o = tb + (four ? 6 : 0); for (u32 st = 0; st < nstreams; st++) { sbytes[st] = (S.stream_bits[st] + 1 + 7) / 8; sbyte[st] = o; o += sbytes[st]; } lit_payload = o; }
            if (four && tid == 0) { for (int k = 0; k < 3; k++) { pl[tb + 2 * k] = (u8)sbytes[k]; pl[tb + 2 * k + 1] = (u8)(sbytes[k] >> 8); } }
            __syncthreads();
            // pass 2: pack.  symbols are written last-to-first: bit position of symbol i = sum of lengths of later symbols
            for (u32 st = 0; st < nstreams; st++) {
                u32 const a = st * seg, b = st == nstreams - 1 ? nlit : a + seg;
                u32 const total_bits = S.stream_bits[st];
                u32 run = 0;                                    // bits of symbols before the current chunk (from the stream start)
                // word-aligned base for atomics: stream starts at an arbitrary byte -> offset in bits from an aligned word
                u32 const base_bit = sbyte[st] * 8;
                for (u32 c0 = a; c0 < b; c0 += ZE_THREADS) {
                    u32 const i = c0 + tid; bool const v = i < b;
                    u32 const sym = v ? G.lit[i] : 0; u32 const nb = v ? S.huf.nb[sym] : 0;
                    u32 tot; u32 const before = ze_block_scan(nb, S.s_warp, tot) + run;
                    if (v) ze_put_bits(G.tmp_lit, base_bit + (total_bits - before - nb), S.huf.code[sym], nb);
                    run += tot;
                }
                if (tid == 0) ze_put_bits(G.tmp_lit, base_bit + total_bits, 1, 1);   // end mark
            }
            __syncthreads();
        }

        ZE_MARK(5);
        // ---------------- E: sequences -> tmp_seq (PREFIX: seqbits)
        u32* const tseq = PREFIX ? GP.seqbits : G.tmp_seq;
        u32 seq_payload = 0;
        if (nseq) {
            // three state chains, last sequence to first (warps 0..2, lane 0)
            if (warp == 0 && lane < 3) {                                  // lanes 0,1,2 of one warp: LL, OF, ML
                ZeCTable const& ct = S.ct[lane];
                const u8* const codes = lane == 0 ? G.llc : (lane == 1 ? G.ofc : G.mlc);
                u16* const sb = G.sbits[lane];
                if (ct.mode == 1) { for (u32 i = 0; i < nseq; i++) sb[i] = 0; sb[nseq] = 0; }
                else {
                    u32 s = codes[nseq - 1];
                    u32 const nbo = (u32)(ct.dnb[s] + (1 << 15)) >> 16; u32 const v0 = (nbo << 16) - (u32)ct.dnb[s];
                    u32 st = ct.state[(v0 >> nbo) + ct.dfs[s]];
                    sb[nseq - 1] = 0;
                    // The chain st -> st' is serial; everything that does not depend on st (the symbol codes and
                    // their deltaNbBits / deltaFindState) is fetched a group of four ahead of it.
                    int i = (int)nseq - 2;
                    for (; i >= 0 && ((i & 3) != 3); i--) {
                        s = codes[i];
                        u32 const nb = (st + (u32)ct.dnb[s]) >> 16;
                        sb[i] = (u16)((st & ((1u << nb) - 1)) | (nb << 12));
                        st = ct.state[(st >> nb) + ct.dfs[s]];
                    }
                    if (i >= 3) {
                        u32 grp = *(const u32*)(codes + i - 3);                 // codes[i-3..i], 4-byte aligned
                        for (; i >= 3; i -= 4) {
                            u32 const g = grp;
                            if (i >= 7) grp = *(const u32*)(codes + i - 7);     // next group, needed four steps from now
                            u32 const s3 = g >> 24, s2 = (g >> 16) & 255, s1 = (g >> 8) & 255, s0 = g & 255;
                            int const n3 = ct.dnb[s3], f3 = ct.dfs[s3], n2 = ct.dnb[s2], f2 = ct.dfs[s2];
                            int const n1 = ct.dnb[s1], f1 = ct.dfs[s1], n0 = ct.dnb[s0], f0 = ct.dfs[s0];
                            u32 nb;
                            nb = (st + (u32)n3) >> 16; sb[i]     = (u16)((st & ((1u << nb) - 1)) | (nb << 12)); st = ct.state[(st >> nb) + f3];
                            nb = (st + (u32)n2) >> 16; sb[i - 1] = (u16)((st & ((1u << nb) - 1)) | (nb << 12)); st = ct.state[(st >> nb) + f2];
                            nb = (st + (u32)n1) >> 16; sb[i - 2] = (u16)((st & ((1u << nb) - 1)) | (nb << 12)); st = ct.state[(st >> nb) + f1];
                            nb = (st + (u32)n0) >> 16; sb[i - 3] = (u16)((st & ((1u << nb) - 1)) | (nb << 12)); st = ct.state[(st >> nb) + f0];
                        }
                    }
                    sb[nseq] = (u16)((st & ((1u << ct.log) - 1)));      // final state (flushed with `log` bits)
                }
            }
            __syncthreads();
            ZE_MARK(6);
            // bit count per sequence; chunks are written last sequence first
            u32 const logLL = S.ct[0].mode == 1 ? 0 : S.ct[0].log, logOF = S.ct[1].mode == 1 ? 0 : S.ct[1].log, logML = S.ct[2].mode == 1 ? 0 : S.ct[2].log;
            u32 run = 0;
            for (u32 base = 0; base < nseq; base += ZE_THREADS) {
                u32 const k = base + tid; bool const v = k < nseq;          // k-th chunk in write order = sequence nseq-1-k
                u32 const i = v ? nseq - 1 - k : 0;
                u32 nb = 0;
                if (v) nb = (G.sbits[0][i] >> 12) + (G.sbits[1][i] >> 12) + (G.sbits[2][i] >> 12) + e_LL_bits[G.llc[i]] + e_ML_bits[G.mlc[i]] + G.ofc[i];
                u32 tot; u32 const before = ze_block_scan(nb, S.s_warp, tot) + run;
                if (v) G.bitpos[i] = before;
                run += tot;
            }
            u32 const total_bits = run + logML + logOF + logLL;
            seq_payload = (total_bits + 1 + 7) / 8;
            for (u32 i = tid; i < seq_payload / 4 + 2; i += ZE_THREADS) tseq[i] = 0;
            __syncthreads();
            for (u32 i = tid; i < nseq; i += ZE_THREADS) {
                uint2 const r = G.seq[i];
                u32 const ll = r.x, ml = (PREFIX ? GP.seqml[i] : r.y >> 20) - 3, ob = PREFIX ? r.y : r.y & 0xFFFFFu;
                u32 bp = G.bitpos[i];
                u32 const so = G.sbits[1][i], sm = G.sbits[2][i], sl = G.sbits[0][i];
                ze_put_bits(tseq, bp, so & 0xFFF, so >> 12); bp += so >> 12;     // OF, ML, LL state bits
                ze_put_bits(tseq, bp, sm & 0xFFF, sm >> 12); bp += sm >> 12;
                ze_put_bits(tseq, bp, sl & 0xFFF, sl >> 12); bp += sl >> 12;
                u32 const lb = e_LL_bits[G.llc[i]], mb = e_ML_bits[G.mlc[i]], obits = G.ofc[i];
                ze_put_bits(tseq, bp, ll, lb); bp += lb;                          // LL, ML, OF additional bits
                ze_put_bits(tseq, bp, ml, mb); bp += mb;
                ze_put_bits(tseq, bp, ob, obits);
            }
            if (tid == 0) {
                u32 bp = run;
                ze_put_bits(tseq, bp, G.sbits[2][nseq], logML); bp += logML;      // flush ML, OF, LL states
                ze_put_bits(tseq, bp, G.sbits[1][nseq], logOF); bp += logOF;
                ze_put_bits(tseq, bp, G.sbits[0][nseq], logLL); bp += logLL;
                ze_put_bits(tseq, bp, 1, 1);
            }
            __syncthreads();
        }

        ZE_MARK(7);
        // ---------------- F: assemble the block in its slot
        if (tid == 0) {
            u8* o = S.lit_hdr_buf; u32 p = 0;
            // literals section header (ZSTD_compressLiterals / ZSTD_noCompressLiterals, zstd/zstd.c:20851-21038)
            if (S.lit_mode == 2) {
                u32 const lh = 3 + (nlit >= 1024) + (nlit >= 16384);
                u32 const ty = S.lit_treeless ? 3u : 2u;       // compressed / treeless (the dictionary's table)
                if (lh == 3) { u32 const v = ty | ((four ? 1u : 0u) << 2) | (nlit << 4) | (lit_payload << 14); o[0] = (u8)v; o[1] = (u8)(v >> 8); o[2] = (u8)(v >> 16); }
                else if (lh == 4) { u32 const v = ty | (2u << 2) | (nlit << 4) | (lit_payload << 18); o[0] = (u8)v; o[1] = (u8)(v >> 8); o[2] = (u8)(v >> 16); o[3] = (u8)(v >> 24); }
                else { u32 const v = ty | (3u << 2) | (nlit << 4) | (lit_payload << 22); o[0] = (u8)v; o[1] = (u8)(v >> 8); o[2] = (u8)(v >> 16); o[3] = (u8)(v >> 24); o[4] = (u8)(lit_payload >> 10); }
                p = lh;
            } else {
                u32 const t = S.lit_mode;      // 0 raw, 1 RLE
                u32 const lh = 1 + (nlit > 31) + (nlit > 4095);
                if (lh == 1) o[0] = (u8)(t | (nlit << 3));
                else if (lh == 2) { u32 const v = t | (1u << 2) | (nlit << 4); o[0] = (u8)v; o[1] = (u8)(v >> 8); }
                else { u32 const v = t | (3u << 2) | (nlit << 4); o[0] = (u8)v; o[1] = (u8)(v >> 8); o[2] = (u8)(v >> 16); }
                p = lh;
                if (t == 1) { o[p++] = G.lit[0]; }
            }
            S.lit_hdr = p;
            // sequences section header (ZSTD_entropyCompressSeqStore_internal, zstd/zstd.c:25893-25926)
            u8* q = S.seq_hdr_buf; u32 k = 0;
            if (nseq < 128) q[k++] = (u8)nseq;
            else if (nseq < 0x7F00) { q[k++] = (u8)((nseq >> 8) + 0x80); q[k++] = (u8)nseq; }
            else { q[k++] = 0xFF; q[k++] = (u8)(nseq - 0x7F00); q[k++] = (u8)((nseq - 0x7F00) >> 8); }
            if (nseq) {
                q[k++] = (u8)((S.ct[0].mode << 6) | (S.ct[1].mode << 4) | (S.ct[2].mode << 2));
                for (int t = 0; t < 3; t++) for (u32 i = 0; i < S.ct[t].hdr_bytes; i++) q[k++] = S.ct[t].hdr[i];
            }
            S.seq_hdr_bytes = k;
            u32 const lit_body = S.lit_mode == 2 ? lit_payload : (S.lit_mode == 0 ? nlit : 0);
            u32 const body = p + lit_body + k + seq_payload;
            // raw fallback when nothing was gained (cSize >= srcSize - minGain, zstd/zstd.c:25987); compressed blocks stay < 128 KiB
            S.use_raw = (body + (n >> 7) + 2 >= n || body >= ZE_BLOCK) ? 1u : 0u;
            S.body = S.use_raw ? n : body;
            u32 const bh = job.last | ((S.use_raw ? 0u : 2u) << 1) | (S.body << 3);
            out[0] = (u8)bh; out[1] = (u8)(bh >> 8); out[2] = (u8)(bh >> 16);
            outs[j].csize = 3 + S.body;
        }
        __syncthreads();
        if constexpr (STATS) {
            if (!S.use_raw) {
                for (u32 i = tid; i < 256; i += ZE_THREADS) if (S.hist[i]) atomicAdd(&stats[i], S.hist[i]);
                for (u32 i = tid; i < 36; i += ZE_THREADS) if (S.hLL[i]) atomicAdd(&stats[256 + i], S.hLL[i]);
                for (u32 i = tid; i < 53; i += ZE_THREADS) if (S.hML[i]) atomicAdd(&stats[292 + i], S.hML[i]);
                for (u32 i = tid; i < 32; i += ZE_THREADS) if (S.hOF[i]) atomicAdd(&stats[345 + i], S.hOF[i]);
            }
        }
        {
            u8* const o = out + 3;
            if (S.use_raw) { for (u32 i = tid; i < n; i += ZE_THREADS) o[i] = in[i]; }
            else {
                u32 p = S.lit_hdr;
                if (tid < p) o[tid] = S.lit_hdr_buf[tid];
                if (S.lit_mode == 2) { const u8* pl = (const u8*)G.tmp_lit; for (u32 i = tid; i < lit_payload; i += ZE_THREADS) o[p + i] = pl[i]; p += lit_payload; }
                else if (S.lit_mode == 0) { for (u32 i = tid; i < nlit; i += ZE_THREADS) o[p + i] = G.lit[i]; p += nlit; }
                for (u32 i = tid; i < S.seq_hdr_bytes; i += ZE_THREADS) o[p + i] = S.seq_hdr_buf[i];
                p += S.seq_hdr_bytes;
                if (nseq) { const u8* ps = (const u8*)tseq; for (u32 i = tid; i < seq_payload; i += ZE_THREADS) o[p + i] = ps[i]; }
            }
        }
        ZE_MARK(8);
        __syncthreads();
    }
}

#include "zb_encode2.cuh"
#include "zb_encode3.cuh"

// ===========================================================================
// dictionary hash table: the block compressor's table state after "having seen" the dictionary tail
// (restates what ZSTD_loadDictionaryContent leaves in the match-state tables, zstd/zstd.c:27900-27990)
// ===========================================================================
// the dictionary's three sequence CTables, built once (ZSTD_loadCEntropy builds the same at dictionary load, zstd/zstd.c:28015)
__global__ void zb_dict_ctables(const ZbDictDigest* __restrict__ ent, ZeCTable* __restrict__ out3)
{
    u32 const k = threadIdx.x >> 5;
    if ((threadIdx.x & 31) || k > 2) return;
    const short* const src = k == 0 ? ent->c_norm_ll : (k == 1 ? ent->c_norm_of : ent->c_norm_ml);
    u32 const mx = k == 0 ? ent->c_max_ll : (k == 1 ? ent->c_max_of : ent->c_max_ml), lg = k == 0 ? ent->ll_log : (k == 1 ? ent->of_log : ent->ml_log);
    u32 const cap = k == 0 ? 35u : (k == 1 ? 31u : 52u), maxlog = k == 1 ? 8u : 9u;
    ZeCTable& ct = out3[k];
    ct.mode = 0xFF; ct.hdr_bytes = 0; ct.rle_sym = 0; ct.log = 0;
    if (!ent->has_entropy || mx > cap || lg > maxlog || lg < 5) return;
    short dn[56]; u32 sum = 0;
    for (u32 s = 0; s < 56; s++) { dn[s] = s <= mx ? src[s] : 0; sum += dn[s] == -1 ? 1u : (dn[s] > 0 ? (u32)dn[s] : 0u); }
    if (sum != (1u << lg)) return;
    u8 tmp[512];
    ze_build_ctable(ct, dn, mx, lg, tmp);
    for (u32 s = mx + 1; s < 56; s++) { ct.dnb[s] = 0; ct.dfs[s] = 0; }
    ct.mode = 3;
}

__global__ void zb_dict_table(const u8* __restrict__ tail, u32 D, u16* __restrict__ table)
{
    u32 const lane = threadIdx.x;
    for (u32 i = lane; i < (1u << ZE_HLOG); i += 32) table[i] = 0xFFFFu;
    __syncwarp();
    for (u32 base = 0; base + 4 <= D; base += 32) {
        u32 const p = base + lane; bool const valid = p + 4 <= D;
        u32 const h = valid ? ze_hash4((u32)tail[p] | ((u32)tail[p + 1] << 8) | ((u32)tail[p + 2] << 16) | ((u32)tail[p + 3] << 24)) : 0;
        u32 const m = __match_any_sync(0xFFFFFFFFu, valid ? h : (0x10000u + lane));
        if (valid && (m >> lane) == 1u && (p & 0xFFFFu) != 0xFFFFu) table[h] = (u16)p;
        __syncwarp();
    }
}

// ===========================================================================
// content-dictionary chains: one index per chunk of a run (a thread per sampled position, grid-stride).  Position p of chunk
// s (every ZE_CHAIN_STEP-th position with 8 bytes behind it) goes to slot ze_chain_slot(8 bytes, p) of the chunk's table, and
// with ZE_CHAIN_FAR bytes behind it also to slot ze_chain_far_slot, by
// atomicMin: the earliest position wins whatever the order the threads run in, so the table -- and with it every frame --
// is the same on every run and on the CPU build.  pos_off[s] = sampled positions of the chunks before s (host prefix sum).
// ===========================================================================
__global__ void __launch_bounds__(256)
zb_chain_index(const u8* __restrict__ src, const ZeChainSeg* __restrict__ segs, const u64* __restrict__ pos_off, u32 n_segs)
{
    u64 const total = pos_off[n_segs];
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (u64)gridDim.x * blockDim.x) {
        u32 lo = 0, hi = n_segs;                     // the chunk: last s with pos_off[s] <= g
        while (hi - lo > 1) { u32 const mid = (lo + hi) >> 1; if (pos_off[mid] <= g) lo = mid; else hi = mid; }
        ZeChainSeg const& c = segs[lo];
        u32 const p = (u32)(g - pos_off[lo]) * ZE_CHAIN_STEP;
        atomicMin((u32*)&c.tab[ze_chain_slot(ze_ld64(src + c.start + p), p, c.log)], p);
        if (p + ZE_CHAIN_FAR <= c.len) atomicMin((u32*)&c.tab[ze_chain_far_slot(src + c.start + p, c.log)], p);
    }
}

// ===========================================================================
// frame layout
// ===========================================================================
struct ZeSegInfo { u64 first_job; u32 n_jobs; u32 pad; };

// frame header bytes for a segment of `size` bytes (restates ZSTD_writeFrameHeader, zstd/zstd.c:27649-27697)
__device__ __forceinline__ u32 ze_frame_header(u8* o, u64 size, ZeParams P)
{
    u32 p = 0;
    o[p++] = 0x28; o[p++] = 0xB5; o[p++] = 0x2F; o[p++] = 0xFD;
    u32 const did = P.dict_id ? (P.dict_id < 256 ? 1 : (P.dict_id < 65536 ? 2 : 3)) : 0;
    if (P.content_size) {
        u32 const fcs = (size >= 256) + (size >= 65536 + 256) + (size >= 0xFFFFFFFFull);
        // like the reference at level 3 (window log 21): a frame is "single segment" (window = content) only up to 2 MiB;
        // bigger frames declare a 2 MiB window, so that streaming decoders with a window limit still take them
        // (our matches never reach further back than 64 KiB + the dictionary tail)
        // ZstdCompressionParameters(window_log=W) moves that threshold: single segment up to 2^W, a 2^W window beyond
        u32 const wl = P.window_log ? P.window_log : 21u;
        bool const single = size <= (1ull << wl);
        o[p++] = (u8)((fcs << 6) | ((single ? 1u : 0u) << 5) | (P.checksum << 2) | did);
        if (!single) o[p++] = (u8)((wl - 10) << 3);
        if (did == 1) o[p++] = (u8)P.dict_id; else if (did == 2) { o[p++] = (u8)P.dict_id; o[p++] = (u8)(P.dict_id >> 8); }
        else if (did == 3) for (int k = 0; k < 4; k++) o[p++] = (u8)(P.dict_id >> (8 * k));
        if (fcs == 0) { if (single) o[p++] = (u8)size; }
        else if (fcs == 1) { u32 const v = (u32)size - 256; o[p++] = (u8)v; o[p++] = (u8)(v >> 8); }
        else if (fcs == 2) for (int k = 0; k < 4; k++) o[p++] = (u8)(size >> (8 * k));
        else for (int k = 0; k < 8; k++) o[p++] = (u8)(size >> (8 * k));
    } else {
        o[p++] = (u8)((P.checksum << 2) | did);
        u32 wlog = 10; while (wlog < 17 && (1ull << wlog) < size) wlog++;        // our matches never reach beyond a block
        if (P.window_log && wlog > P.window_log) wlog = P.window_log;            // (blocks are cut to the window, zb_api.cu)
        o[p++] = (u8)((wlog - 10) << 3);
        if (did == 1) o[p++] = (u8)P.dict_id; else if (did == 2) { o[p++] = (u8)P.dict_id; o[p++] = (u8)(P.dict_id >> 8); }
        else if (did == 3) for (int k = 0; k < 4; k++) o[p++] = (u8)(P.dict_id >> (8 * k));
    }
    return p;
}

__global__ void zb_frame_sizes(const ZbSegment* __restrict__ segs, const ZeSegInfo* __restrict__ info, const ZeBlockOut* __restrict__ outs,
                               u32 n_segs, ZeParams P, u64* __restrict__ sizes)
{
    u32 const f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_segs) return;
    u8 tmp[20]; u64 sz = ze_frame_header(tmp, segs[f].length, P);
    ZeSegInfo const si = info[f];
    for (u32 k = 0; k < si.n_jobs; k++) sz += outs[si.first_job + k].csize;
    if (si.n_jobs == 0) sz += 3;                        // empty input: one empty raw block
    if (P.checksum) sz += 4;
    sizes[f] = sz;
}

// exclusive scan of u64 sizes by one CTA -> segment table of the output; total in *total
__global__ void __launch_bounds__(1024) zb_scan_sizes(const u64* __restrict__ sizes, u32 n, ZbSegment* __restrict__ out_segs, u64* __restrict__ total)
{
    __shared__ u64 s_part[32]; __shared__ u64 s_run;
    u32 const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_run = 0;
    __syncthreads();
    for (u32 base = 0; base < n; base += 1024) {
        u32 const i = base + tid; u64 const v = i < n ? sizes[i] : 0; u64 x = v;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { u64 y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= (u32)d) x += y; }
        if (lane == 31) s_part[warp] = x;
        __syncthreads();
        if (warp == 0) { u64 y = s_part[lane];
            #pragma unroll
            for (int d = 1; d < 32; d <<= 1) { u64 z = __shfl_up_sync(0xFFFFFFFFu, y, d); if (lane >= (u32)d) y += z; }
            s_part[lane] = y; }
        __syncthreads();
        u64 const off = s_run + (warp ? s_part[warp - 1] : 0) + x - v;
        if (i < n) { ZbSegment s; s.offset = off; s.length = v; out_segs[i] = s; }
        __syncthreads();
        if (tid == 0) s_run += s_part[31];
        __syncthreads();
    }
    if (tid == 0) *total = s_run;
}

// XXH64 of one buffer by one thread (restates XXH64 as zstd uses it for the content checksum, zstd/zstd.c:27562)
__device__ static u64 ze_xxh64(const u8* p, u64 len)
{
    u64 const P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull, P4 = 0x85EBCA77C2B2AE63ull, P5 = 0x27D4EB2F165667C5ull;
    auto rotl = [](u64 x, int r) { return (x << r) | (x >> (64 - r)); };
    auto rd64 = [](const u8* q) { u64 v = 0; for (int k = 0; k < 8; k++) v |= (u64)q[k] << (8 * k); return v; };
    auto round = [&](u64 acc, u64 in) { return rotl(acc + in * P2, 31) * P1; };
    const u8* const end = p + len; u64 h;
    if (len >= 32) {
        u64 v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0 - P1;
        do { v1 = round(v1, rd64(p)); v2 = round(v2, rd64(p + 8)); v3 = round(v3, rd64(p + 16)); v4 = round(v4, rd64(p + 24)); p += 32; } while (p + 32 <= end);
        h = rotl(v1, 1) + rotl(v2, 7) + rotl(v3, 12) + rotl(v4, 18);
        h = (h ^ round(0, v1)) * P1 + P4; h = (h ^ round(0, v2)) * P1 + P4; h = (h ^ round(0, v3)) * P1 + P4; h = (h ^ round(0, v4)) * P1 + P4;
    } else h = P5;
    h += len;
    while (p + 8 <= end) { h ^= round(0, rd64(p)); h = rotl(h, 27) * P1 + P4; p += 8; }
    if (p + 4 <= end) { u64 v = 0; for (int k = 0; k < 4; k++) v |= (u64)p[k] << (8 * k); h ^= v * P1; h = rotl(h, 23) * P2 + P3; p += 4; }
    while (p < end) { h ^= (*p++) * P5; h = rotl(h, 11) * P1; }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

// one warp per segment: header, blocks copied from their slots, optional checksum
__global__ void __launch_bounds__(256)
zb_write_frames(const u8* __restrict__ src, const ZbSegment* __restrict__ segs, const ZeSegInfo* __restrict__ info,
                const ZeBlockOut* __restrict__ outs, const u8* __restrict__ slots, u64 slot_bytes, u32 n_segs, ZeParams P,
                const ZbSegment* __restrict__ out_segs, u8* __restrict__ dst)
{
    u32 const lane = threadIdx.x & 31;
    u32 const f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (f >= n_segs) return;
    u8* const o = dst + out_segs[f].offset;
    ZeSegInfo const si = info[f];
    u32 hdr = 0;
    if (lane == 0) {
        hdr = ze_frame_header(o, segs[f].length, P);
        if (si.n_jobs == 0) { o[hdr] = 1; o[hdr + 1] = 0; o[hdr + 2] = 0; }      // last raw block of size 0
    }
    hdr = __shfl_sync(0xFFFFFFFFu, hdr, 0);
    u64 p = hdr + (si.n_jobs == 0 ? 3 : 0);
    for (u32 k = 0; k < si.n_jobs; k++) {
        u32 const cs = outs[si.first_job + k].csize;
        const u8* const s = slots + (si.first_job + k) * slot_bytes;
        for (u32 i = lane; i < cs; i += 32) o[p + i] = s[i];
        p += cs;
    }
    if (P.checksum && lane == 0) {
        u64 const h = ze_xxh64(src + segs[f].offset, segs[f].length);
        for (int k = 0; k < 4; k++) o[p + k] = (u8)(h >> (8 * k));
    }
}

// ===========================================================================
// launchers
// ===========================================================================
extern "C" {

size_t zb_encode_scratch_bytes() { return sizeof(ZeScratch); }

void zb_launch_dict_table(const u8* tail, u32 D, u16* table, cudaStream_t st) { ZB_LAUNCH(zb_dict_table, 1, 32, 0, st, tail, D, table); }

void zb_launch_compress_blocks(const u8* src, const void* jobs, u32 n_jobs, void* scratch, u32 n_ctas, u8* slots, u64 slot_bytes,
                               void* outs, u32* work_counter, const u8* dict_tail, u32 dict_D, const u16* dict_table, const void* dict_digest, const void* dict_cct,
                               const unsigned long long* upload_progress, unsigned long long upload_total, u32* upload_status, int dual, int small_blocks, cudaStream_t st,
                               u32* stats)
{
    ZeDict dict; dict.tail = dict_tail; dict.D = dict_D; dict.pad = 0; dict.table = dict_table; dict.ent = (const ZbDictDigest*)dict_digest; dict.cct = dict_digest ? dict_cct : nullptr;
    ZeUpload up; up.progress = upload_progress; up.total = upload_total; up.status = upload_status;
    // the instantiation: two hash tables from level 4 on, 256-byte parse units for small blocks, statistics for dictionary
    // training (ZDICT_countEStats)
    decltype(&zb_compress_blocks<false, ZE_UNIT, false>) k;
    if (stats) k = dual ? (small_blocks ? zb_compress_blocks<true, ZE_UNIT_SMALL, true> : zb_compress_blocks<true, ZE_UNIT, true>)
                        : (small_blocks ? zb_compress_blocks<false, ZE_UNIT_SMALL, true> : zb_compress_blocks<false, ZE_UNIT, true>);
    else k = dual ? (small_blocks ? zb_compress_blocks<true, ZE_UNIT_SMALL, false> : zb_compress_blocks<true, ZE_UNIT, false>)
                  : (small_blocks ? zb_compress_blocks<false, ZE_UNIT_SMALL, false> : zb_compress_blocks<false, ZE_UNIT, false>);
    ZB_LAUNCH(k, n_ctas, ZE_THREADS, sizeof(ZeShared), st, src, (const ZeBlockJob*)jobs, n_jobs, (ZeScratch*)scratch, slots, slot_bytes,
              (ZeBlockOut*)outs, work_counter, dict, up, stats);
}

// content-dictionary chains: the chunk indexes of a run, and its block jobs through the prefix mode
size_t zb_encode_pscratch_bytes() { return sizeof(ZePScratch); }
size_t zb_chain_seg_bytes() { return sizeof(ZeChainSeg); }
void zb_launch_chain_index(const u8* src, const void* segs, const u64* pos_off, u32 n_segs, u64 total_pos, u32 sms, cudaStream_t st)
{
    if (!total_pos) return;
    u64 const want = (total_pos + 255) / 256; u32 const grid = (u32)(want < (u64)sms * 16 ? want : (u64)sms * 16);
    ZB_LAUNCH(zb_chain_index, grid, 256, 0, st, src, (const ZeChainSeg*)segs, pos_off, n_segs);
}
void zb_launch_compress_chain_blocks(const u8* src, const void* jobs, u32 n_jobs, void* scratch, u32 n_ctas, u8* slots, u64 slot_bytes,
                                     void* outs, u32* work_counter, const void* segs, cudaStream_t st)
{
    ZeDict dict; memset(&dict, 0, sizeof dict); dict.cct = segs;
    ZeUpload up; up.progress = nullptr; up.total = 0; up.status = nullptr;
    ZB_LAUNCH((zb_compress_blocks<false, ZE_UNIT, false, true>), n_ctas, ZE_THREADS, sizeof(ZeShared), st, src, (const ZeBlockJob*)jobs, n_jobs,
              (ZeScratch*)scratch, slots, slot_bytes, (ZeBlockOut*)outs, work_counter, dict, up, nullptr);
}

void zb_launch_frame_layout(const ZbSegment* segs, const void* seginfo, const void* outs, u32 n_segs, u32 checksum, u32 content_size,
                            u32 dict_id, u32 window_log, u64* sizes, ZbSegment* out_segs, u64* total, cudaStream_t st)
{
    ZeParams P; P.checksum = checksum; P.content_size = content_size; P.dict_id = dict_id; P.level = 3; P.window_log = window_log;
    ZB_LAUNCH(zb_frame_sizes, (n_segs + 255) / 256, 256, 0, st, segs, (const ZeSegInfo*)seginfo, (const ZeBlockOut*)outs, n_segs, P, sizes);
    ZB_LAUNCH(zb_scan_sizes, 1, 1024, 0, st, sizes, n_segs, out_segs, total);
}

void zb_launch_write_frames(const u8* src, const ZbSegment* segs, const void* seginfo, const void* outs, const u8* slots, u64 slot_bytes,
                            u32 n_segs, u32 checksum, u32 content_size, u32 dict_id, u32 window_log, const ZbSegment* out_segs, u8* dst, cudaStream_t st)
{
    ZeParams P; P.checksum = checksum; P.content_size = content_size; P.dict_id = dict_id; P.level = 3; P.window_log = window_log;
    ZB_LAUNCH(zb_write_frames, (n_segs + 7) / 8, 256, 0, st, src, segs, (const ZeSegInfo*)seginfo, (const ZeBlockOut*)outs, slots, slot_bytes, n_segs, P,
              out_segs, dst);
}

u32 zb_encode_smem_bytes() { return (u32)sizeof(ZeShared); }

// round-2 kernel: one CTA per SM, block resident in shared memory (no dictionary, blocks compressed independently)
size_t zb_encode2_scratch_bytes() { return sizeof(Z2Scratch); }
u32 zb_encode2_smem_bytes() { return (u32)sizeof(Z2Shared); }
void zb_launch_compress_smem(const u8* src, const void* jobs, u32 n_jobs, void* scratch, u32 n_ctas, u8* slots, u64 slot_bytes, void* outs, u32* work_counter,
                             const unsigned long long* upload_progress, unsigned long long upload_total, u32* upload_status, cudaStream_t st)
{
    ZeUpload up; up.progress = upload_progress; up.total = upload_total; up.status = upload_status;
    ZB_LAUNCH(zb_compress_smem, n_ctas, Z2_NT, sizeof(Z2Shared), st, src, (const ZeBlockJob*)jobs, n_jobs, (Z2Scratch*)scratch, slots, slot_bytes,
              (ZeBlockOut*)outs, work_counter, up);
}
u32 zb_encode_small_max() { return ZE_SMALL_MAX; }

// small records with a full dictionary: a warp per record (zb_encode3.cuh)
u32 zb_encode3_record_max() { return Z3_RMAX; }
u32 zb_encode3_records_per_cta() { return Z3_WARPS; }
void zb_launch_compress_recs(const u8* src, const void* jobs, u32 n_jobs, u32 n_ctas, u8* slots, u64 slot_bytes, void* outs, u32* work_counter,
                             const u8* dict_tail, u32 dict_D, const u16* dict_table, const void* dict_digest, const void* dict_cct,
                             const unsigned long long* upload_progress, unsigned long long upload_total, u32* upload_status, cudaStream_t st)
{
    ZeDict dict; dict.tail = dict_tail; dict.D = dict_D; dict.pad = 0; dict.table = dict_table; dict.ent = (const ZbDictDigest*)dict_digest; dict.cct = dict_cct;
    ZeUpload up; up.progress = upload_progress; up.total = upload_total; up.status = upload_status;
    ZB_LAUNCH(zb_compress_recs, n_ctas, Z3_NT, sizeof(Z3Shared), st, src, (const ZeBlockJob*)jobs, n_jobs, slots, slot_bytes, (ZeBlockOut*)outs, work_counter,
              dict, up);
}
u32 zb_encode_ctable_bytes() { return (u32)sizeof(ZeCTable); }
void zb_launch_dict_ctables(const void* digest, void* out3, cudaStream_t st) { ZB_LAUNCH(zb_dict_ctables, 1, 96, 0, st, (const ZbDictDigest*)digest, (ZeCTable*)out3); }

void zb_encode_phase_read(unsigned long long* out16, int reset)
{
#ifdef ZB_PHASE_TIMERS
    cudaMemcpyFromSymbol(out16, g_ze_phase, sizeof(unsigned long long) * 16);
    if (reset) { unsigned long long z[16] = {0}; cudaMemcpyToSymbol(g_ze_phase, z, sizeof z); }
#else
    for (int i = 0; i < 16; i++) out16[i] = 0; (void)reset;
#endif
}
void zb_encode2_phase_read(unsigned long long* out16, int reset)
{
#ifdef ZB_PHASE_TIMERS
    cudaMemcpyFromSymbol(out16, g_z2_phase, sizeof(unsigned long long) * 16);
    if (reset) { unsigned long long z[16] = {0}; cudaMemcpyToSymbol(g_z2_phase, z, sizeof z); }
#else
    for (int i = 0; i < 16; i++) out16[i] = 0; (void)reset;
#endif
}

}  // extern "C"

// dictionary training: its kernels and launchers (they reuse the entropy helpers above)
#include "zb_train.cuh"
