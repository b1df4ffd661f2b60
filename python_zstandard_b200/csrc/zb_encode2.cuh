// zb_encode2.cuh -- the round-2 block compressor: ONE CTA of 1024 threads per SM, the <= 128 KiB block resident in
// shared memory (TMA bulk copy); every dependent access (hash table, candidate verification, parse, FSE states, Huffman
// codes) is served from shared memory; only streaming intermediates (match records, final sequences) pass through the
// L2-resident per-CTA scratch.  Included by zb_encode.cu (it reuses the serial table builders above).
//
// Stands in for ZSTD_compressBlock_doubleFast (zstd/zstd.c:31039) + ZSTD_entropyCompressSeqStore (:25842) per block:
//   load     cp.async.bulk global -> shared, mbarrier completion
//   match    passes of 8192 positions, software-pipelined: while warp 0 LINKS pass k+1, warps 1-29 VERIFY + PARSE pass k
//     hash   all threads: 14-bit hash of the 5 bytes at every position
//     link   warp 0, 32 positions per step in order through ONE 2^14-entry table: distance to the previous position with
//            the same hash (exact except inside a step); eight steps' table accesses in flight
//     v + p  a warp per 288-position region, 32 positions per step: every lane verifies its candidate (common prefix
//            4..15, 15 = "or more"), one ballot tells every match where the next one may start, the warp hops along that
//            chain (true greedy + one-step lazy inside the region), "15 or more" matches are extended 256 bytes per vote,
//            every selected lane extends its own match backwards and writes its record
//   stitch   fold of the regions' last match ends -> what each region must drop / front-trim; survivors are compacted;
//            repcode history is an MTF(3) list, so region summaries (3 most recent distinct offsets) scan exactly and
//            every lane codes its region's offsets with the true history (ZSTD_updateRep :19971)
//   entropy  FSE tables: a warp per table (LL, OF, ML), lanes = symbols (normalise, cost, spread by closed form, cells by
//            match.any ranks); Huffman code by warp 3 beside them.  The sequences are cut into <= 10 runs, each run becomes
//            a zstd block of its own ("repeat" tables / "treeless" literals after the first): the three FSE state chains
//            of every run are strictly serial, so 30 lanes walk them side by side (exact), leaving the state on entry
//            of every thread's range; all threads then re-run their ranges to count and to write the bits
//   write    bit counts are prefix-scanned; literal streams and sequence streams are OR-ed straight into the slot
//            (first/last word of a span atomically, the words between plainly); raw fallback for the whole chunk
#pragma once

#define Z2_NT       1024
#define Z2_REG      288                   // positions per parse region (a warp walks one per pass)
#define Z2_RPP      29                    // regions per pass
#define Z2_Q        8192                  // positions per pass
#define Z2_MAXU     512
#define Z2_RMAX     76                    // records per region (at most 72 matches start in one: they are >= 4 bytes and do not overlap)
#define Z2_FARLOG   14
#define Z2_MAXSEQ   33024
#define Z2_STAGE    57344                 // bytes of staging / literal buffer in shared memory
#define Z2_WARM     24                    // FSE warm-up symbols
#define Z2_SEQ_SMEM 16384                 // sequence records that fit the (by then dead) input buffer
#define Z2_MAXSUB   10                    // sub-blocks per chunk (3 chain lanes each: one warp)
#define Z2_SUBSEQ   1536                  // sequences per sub-block aimed at

struct Z2Scratch {
    u64 rec[Z2_MAXU * Z2_RMAX];           // unit records: start | len << 17 | dist << 35
    u64 fseq[Z2_MAXSEQ + 8];              // final sequences: ll | (ml - 3) << 17 | offBase << 34
    u8  lit[ZE_BLOCK + 64];               // gathered literals when they do not fit shared memory
};

static_assert(true, "");
struct Z2Mf { u16 far[1 << Z2_FARLOG]; __align__(16) u16 hd[2][Z2_Q]; };
struct Z2Ent {
    __align__(16) u32 stage[Z2_STAGE / 4];        // literals (gathered), later the sequence bitstream
    ZeCTable ct[4];                       // LL, OF, ML, Huffman-weight table
    ZeHuf huf;
    u32 wk[1600];
    u8 tmp_sym[4][512];
    u8 huf_tbl[160]; u8 seq_hdr_buf[256];
    u32 hist[8][256];
    u32 hLL[36], hOF[32], hML[56];
    short nrm[3][64]; u16 cum[3][64];
};
struct Z2Shared {
    __align__(16) u8 in[ZE_BLOCK + 48];   // the block, at in[skew ..]; after the literals section: the sequence records
    union { Z2Mf mf; Z2Ent en; };
    u32 x0[1024], x1[1024], x2[1024];     // per-unit exchange arrays (match ends, covers, repcode summaries, FSE states)
    u32 part[40];
    u8 llcode[64], mlcode[128];
    unsigned long long mbar;
    u32 job, tail_from, bad, lit_mode, huf_tbl_bytes, seq_hdr_bytes, all_same, carry;
    u32 mtmp[36];
    // sub-blocks and their literal streams
    u32 sub_seq[Z2_MAXSUB + 1], sub_lit[Z2_MAXSUB + 1], sub_st0[Z2_MAXSUB + 1], sub_spre[Z2_MAXSUB + 1], sub_off[Z2_MAXSUB + 1];
    u32 sub_mode[Z2_MAXSUB], sub_lh[Z2_MAXSUB], sub_pay[Z2_MAXSUB], sub_shb[Z2_MAXSUB], sub_spay[Z2_MAXSUB];
    u32 fin[Z2_MAXSUB][3];
    u32 st_start[4 * Z2_MAXSUB + 1], st_len[4 * Z2_MAXSUB + 1], st_cum[4 * Z2_MAXSUB + 1], st_pre[4 * Z2_MAXSUB + 1], st_byte[4 * Z2_MAXSUB + 1];
    u32 n_streams;
};

// ---- shared-memory byte window helpers (buffer is 4-byte aligned, 12 bytes of slack after the last position read)
__device__ __forceinline__ u32 z2_ld32(const u8* b, u32 pos)
{
    const u32* const w = (const u32*)b + (pos >> 2); u32 const sh = (pos & 3) * 8;
    return __funnelshift_r(w[0], w[1], sh);
}
__device__ __forceinline__ u64 z2_ld64(const u8* b, u32 pos)
{
    const u32* const w = (const u32*)b + (pos >> 2); u32 const sh = (pos & 3) * 8;
    u32 const w0 = w[0], w1 = w[1], w2 = w[2];
    return (u64)__funnelshift_r(w0, w1, sh) | ((u64)__funnelshift_r(w1, w2, sh) << 32);
}
__device__ __forceinline__ u32 z2_hash5(u64 v) { return (u32)(((v << 24) * 889523592379ull) >> (64 - Z2_FARLOG)); }

// common prefix of the bytes at a and at c (c < a), looking at most 16 bytes ahead and never past n; A = the 8 bytes at a
__device__ __forceinline__ u32 z2_match16(const u8* b, u32 skew, u64 A, u32 a, u32 c, u32 n)
{
    u64 const x = A ^ z2_ld64(b, skew + c);
    if (x) return ze_common8(0, x);
    if (a + 16 > n) return 8;
    return 8 + ze_common8(z2_ld64(b, skew + a + 8), z2_ld64(b, skew + c + 8));
}

// exclusive scan of one u32 per thread over the CTA (1024 threads); part: 33+ words of shared memory
__device__ __forceinline__ u32 z2_scan(u32 v, u32* part, u32& total)
{
    u32 const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 x = v;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { u32 const y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= (u32)d) x += y; }
    if (lane == 31) part[warp] = x;
    __syncthreads();
    if (warp == 0) {
        u32 y = part[lane];
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { u32 const z = __shfl_up_sync(0xFFFFFFFFu, y, d); if (lane >= (u32)d) y += z; }
        part[lane] = y;
    }
    __syncthreads();
    total = part[31];
    u32 const r = (warp ? part[warp - 1] : 0u) + x - v;
    __syncthreads();
    return r;
}

// repcode history as an MTF(3) list: apply the (<= 3, most recent first, 0 = none) distinct offsets of a unit
__device__ __forceinline__ void z2_rep_apply(u32& r0, u32& r1, u32& r2, u32 a, u32 b, u32 c)
{
    u32 o[6]; u32 k = 0;
    if (a) o[k++] = a;
    if (b) o[k++] = b;
    if (c) o[k++] = c;
    u32 const t = k;
    u32 const old[3] = {r0, r1, r2};
    #pragma unroll
    for (int i = 0; i < 3; i++) {
        u32 const v = old[i]; bool dup = false;
        for (u32 q = 0; q < t; q++) if (o[q] == v && v) dup = true;
        if (!dup) o[k++] = v;
    }
    r0 = o[0]; r1 = k > 1 ? o[1] : 0; r2 = k > 2 ? o[2] : 0;
}
// the unit's most recent distinct offsets, collected from its LAST sequence backwards
__device__ __forceinline__ void z2_recent_push_back(u32& a, u32& b, u32& c, u32 d)
{
    if (d == a || d == b || d == c) return;
    if (!a) a = d; else if (!b) b = d; else if (!c) c = d;
}

// LSB-first bit accumulator over a zeroed word array (shared or global): the first and the last word of a lane's span
// may be shared with its neighbours (atomicOr), the words in between are its own (plain stores)
struct Z2Bits {
    u32* words; u32 w; u64 acc; u32 nacc; bool first;
    __device__ __forceinline__ void init(u32* base, u32 bitpos) { words = base; w = bitpos >> 5; acc = 0; nacc = bitpos & 31; first = true; }
    __device__ __forceinline__ void put(u32 v, u32 nb) {          // nb <= 26
        acc |= (u64)(v & ((1u << nb) - 1)) << nacc; nacc += nb;
        if (nacc >= 32) { if (first) { atomicOr(&words[w], (u32)acc); first = false; } else words[w] = (u32)acc; w++; acc >>= 32; nacc -= 32; }
    }
    __device__ __forceinline__ void flush() { if (nacc) atomicOr(&words[w], (u32)acc); }
};
__device__ __forceinline__ void z2_or_byte(u32* words, u32 byte_off, u32 v) { atomicOr(&words[byte_off >> 2], (v & 255u) << ((byte_off & 3) * 8)); }

__device__ __forceinline__ u32 z2_fse_init(const ZeCTable& ct, u32 s)      // FSE_initCState2, zstd/zstd.c:2770
{
    u32 const nbo = (u32)(ct.dnb[s] + (1 << 15)) >> 16; u32 const v = (nbo << 16) - (u32)ct.dnb[s];
    return ct.state[(v >> nbo) + ct.dfs[s]];
}


// ---- FSE table of one symbol stream, built by a whole warp (lane l looks after symbols l and l + 32).  Same decisions as
// ze_make_table (mode by cost, normalisation, NCount header) except that the costs are summed in another order.
// nrm: 64 shorts, cum: 64 u16 of shared memory.
__device__ static void z2_build_ctable_warp(ZeCTable& ct, const short* nrm, u32 max_sym, u32 log, u8* tmp_sym, u16* cum, u32 lane)
{
    // restates FSE_buildCTable_wksp (zstd/zstd.c:16005-16155) for tables without "less than one" cells
    u32 const size = 1u << log, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
    u32 const n0 = lane <= max_sym ? (u32)nrm[lane] : 0u, n1 = lane + 32 <= max_sym ? (u32)nrm[lane + 32] : 0u;
    u32 x0 = n0, x1 = n1;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { u32 const y0 = __shfl_up_sync(0xFFFFFFFFu, x0, d), y1 = __shfl_up_sync(0xFFFFFFFFu, x1, d); if (lane >= (u32)d) { x0 += y0; x1 += y1; } }
    u32 const tot0 = __shfl_sync(0xFFFFFFFFu, x0, 31);
    u32 const pre0 = x0 - n0, pre1 = tot0 + x1 - n1;                  // cells in front of my symbols
    cum[lane] = (u16)pre0; cum[lane + 32] = (u16)pre1;
    __syncwarp();
    for (u32 s = 0; s <= max_sym; s++) {                              // spread: cell k of the cumulative order sits at (k * step) & mask
        u32 const c0 = cum[s], n = (u32)nrm[s];
        for (u32 i = lane; i < n; i += 32) tmp_sym[((c0 + i) * step) & mask] = (u8)s;
    }
    __syncwarp();
    for (u32 u0 = 0; u0 < size; u0 += 32) {                           // every symbol's cells in ascending table order
        u32 const u = u0 + lane, sy = tmp_sym[u];
        u32 const peers = __match_any_sync(0xFFFFFFFFu, sy);
        u32 const rank = (u32)__popc(peers & ((1u << lane) - 1u));
        u32 const base = cum[sy];
        ct.state[base + rank] = (u16)(size + u);
        __syncwarp();
        if (rank == 0) cum[sy] = (u16)(base + (u32)__popc(peers));
        __syncwarp();
    }
    #pragma unroll
    for (u32 h = 0; h < 2; h++) {
        u32 const sy = lane + 32 * h, c = h ? n1 : n0, pre = h ? pre1 : pre0;
        if (sy < 56) {
            int dnb = 0, dfs = 0;
            if (sy <= max_sym) {
                if (c == 0) { dnb = (int)(((log + 1) << 16) - size); dfs = 0; }
                else if (c == 1) { dnb = (int)((log << 16) - size); dfs = (int)pre - 1; }
                else { u32 const maxBitsOut = log - ze_hibit(c - 1), minStatePlus = c << maxBitsOut; dnb = (int)((maxBitsOut << 16) - minStatePlus); dfs = (int)pre - (int)c; }
            }
            ct.dnb[sy] = dnb; ct.dfs[sy] = dfs;
        }
    }
    if (lane == 0) ct.log = log;
    __syncwarp();
}

__device__ static float z2_cost_warp(u32 c0, u32 c1, int n0, int n1, u32 log, bool& bad)
{
    float bits = 0.f; bool b = false;
    if (c0) { int n = n0 == -1 ? 1 : n0; if (n <= 0) b = true; else bits += (float)c0 * ((float)log - __log2f((float)n)); }
    if (c1) { int n = n1 == -1 ? 1 : n1; if (n <= 0) b = true; else bits += (float)c1 * ((float)log - __log2f((float)n)); }
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1) bits += __shfl_xor_sync(0xFFFFFFFFu, bits, d);
    bad = __any_sync(0xFFFFFFFFu, b);
    return bits;
}

__device__ static void z2_make_table_warp(ZeCTable& ct, const u32* count, u32 kind_max, u32 nseq, u32 max_log, u32 def_log,
                                          const short* defnorm, u32 def_max, u8* tmp_sym, short* nrm, u16* cum, u32 lane)
{
    u32 const c0 = lane <= kind_max ? count[lane] : 0u, c1 = lane + 32 <= kind_max ? count[lane + 32] : 0u;
    u32 present = (c0 ? 1u : 0u) + (c1 ? 1u : 0u), most = max(c0, c1), max_sym = c1 ? lane + 32 : (c0 ? lane : 0u);
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        present += __shfl_xor_sync(0xFFFFFFFFu, present, d);
        most = max(most, __shfl_xor_sync(0xFFFFFFFFu, most, d)); max_sym = max(max_sym, __shfl_xor_sync(0xFFFFFFFFu, max_sym, d));
    }
    if (most == nseq && nseq > 2) {                       // one symbol only: RLE (ZSTD_selectEncodingType, zstd/zstd.c:21262)
        if (lane < 28) { ct.dnb[lane] = 0; ct.dfs[lane] = 0; ct.dnb[lane + 28] = 0; ct.dfs[lane + 28] = 0; }
        if (lane == 0) { ct.mode = 1; ct.rle_sym = max_sym; ct.hdr[0] = (u8)max_sym; ct.hdr_bytes = 1; ct.log = 0; ct.state[0] = 1; }
        __syncwarp();
        return;
    }
    // predefined table usable?  every present symbol must have a cell in it
    int const dn0 = lane <= def_max ? (int)defnorm[lane] : 0, dn1 = lane + 32 <= def_max ? (int)defnorm[lane + 32] : 0;
    bool const def_ok = !__any_sync(0xFFFFFFFFu, (c0 && dn0 == 0) || (c1 && dn1 == 0));
    u32 cost_def = 0xFFFFFFFFu;
    if (def_ok) { bool bad; float const f = z2_cost_warp(c0, c1, dn0, dn1, def_log, bad); if (!bad) cost_def = (u32)(f + 0.5f); }
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
    u32 cost_cmp = 0xFFFFFFFFu, nc_bytes = 0;
    bool ok = nseq >= 32 && (1u << log) >= present;
    if (ok) {        // normalise to 2^log, every present symbol >= 1, remainder to the most frequent symbol (ze_normalize)
        u32 const size = 1u << log;
        u64 const scale = ((u64)size << 20) / nseq;
        u32 p0 = 0, p1 = 0;
        if (c0) { p0 = (u32)(((u64)c0 * scale + (1u << 19)) >> 20); if (!p0) p0 = 1; }
        if (c1) { p1 = (u32)(((u64)c1 * scale + (1u << 19)) >> 20); if (!p1) p1 = 1; }
        u32 used = p0 + p1, key = max(c0 ? (c0 << 6) | (63u - lane) : 0u, c1 ? (c1 << 6) | (31u - lane) : 0u);
        #pragma unroll
        for (int d = 16; d > 0; d >>= 1) { used += __shfl_xor_sync(0xFFFFFFFFu, used, d); key = max(key, __shfl_xor_sync(0xFFFFFFFFu, key, d)); }
        u32 const largest = 63u - (key & 63u);
        int const diff = (int)size - (int)used;
        int const nl = (int)__shfl_sync(0xFFFFFFFFu, largest < 32 ? p0 : p1, (int)(largest & 31u));
        if (nl + diff < 1) {                              // rare: too many rare symbols rounded up -- the serial routine sorts it out
            u32 r = 0;
            if (lane == 0) r = ze_normalize(nrm, count, max_sym, nseq, log) ? 1u : 0u;
            ok = __shfl_sync(0xFFFFFFFFu, r, 0) != 0;
        } else {
            if (largest == lane) p0 = (u32)((int)p0 + diff);
            if (largest == lane + 32) p1 = (u32)((int)p1 + diff);
            nrm[lane] = (short)p0; nrm[lane + 32] = (short)p1;
        }
        __syncwarp();
        if (ok) {
            u32 nb = 0;
            if (lane == 0) nb = ze_write_ncount(ct.hdr, nrm, max_sym, log);
            nc_bytes = __shfl_sync(0xFFFFFFFFu, nb, 0);
            bool bad; float const f = z2_cost_warp(c0, c1, (int)nrm[lane], (int)nrm[lane + 32], log, bad);
            if (!bad) cost_cmp = (u32)(f + 0.5f) + nc_bytes * 8;
        }
    }
    if (ok && cost_cmp < cost_def) {
        z2_build_ctable_warp(ct, nrm, max_sym, log, tmp_sym, cum, lane);
        if (lane == 0) { ct.mode = 2; ct.hdr_bytes = nc_bytes; }
        __syncwarp();
        return;
    }
    if (lane == 0) {                                      // predefined table, or a flat one: the serial builders
        short norm[56];
        if (!def_ok) {     // neither fits (tiny block with a symbol outside the predefined alphabet): flat table over present symbols
            u32 lg = 5; while ((1u << lg) < present) lg++;
            u32 k = 0, per = (1u << lg) / present, extra = (1u << lg) - per * present;
            for (u32 s = 0; s <= max_sym; s++) { norm[s] = count[s] ? (short)(per + (k < extra ? 1 : 0)) : 0; if (count[s]) k++; }
            ct.mode = 2; ct.hdr_bytes = ze_write_ncount(ct.hdr, norm, max_sym, lg); ze_build_ctable(ct, norm, max_sym, lg, tmp_sym);
            for (u32 s = max_sym + 1; s < 56; s++) { ct.dnb[s] = 0; ct.dfs[s] = 0; }
        } else {
            ct.mode = 0; ct.hdr_bytes = 0;
            for (u32 s = 0; s <= def_max; s++) norm[s] = defnorm[s];
            ze_build_ctable(ct, norm, def_max, def_log, tmp_sym);
            for (u32 s = def_max + 1; s < 56; s++) { ct.dnb[s] = 0; ct.dfs[s] = 0; }
        }
    }
    __syncwarp();
}

// Huffman code lengths, warp-cooperative front end: rank the present symbols by (count, symbol) -- every lane ranks
// eight of them against all 256 -- then lane 0 runs the serial tree construction of ze_huf_from_sorted
__device__ static bool z2_huf_build(ZeHuf& H, const u32* count, u32* wk, u32 lane)
{
    u32* const sym = wk; u32* const key = wk + 1100;             // key[]: 256 words inside the (not yet used) tail of wk
    u32 present = 0, mxs = 0;
    for (u32 k = 0; k < 8; k++) { u32 const s = lane * 8 + k, c = count[s]; key[s] = c ? ((c << 8) | s) : 0xFFFFFFFFu; if (c) { present++; mxs = s; } }
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1) { present += __shfl_xor_sync(0xFFFFFFFFu, present, d); mxs = max(mxs, __shfl_xor_sync(0xFFFFFFFFu, mxs, d)); }
    __syncwarp();
    if (present < 2) return false;
    u32 mykey[8], rank[8];
    #pragma unroll
    for (int k = 0; k < 8; k++) { mykey[k] = key[lane * 8 + k]; rank[k] = 0; }
    for (u32 t = 0; t < 256; t++) {
        u32 const kt = key[t];
        #pragma unroll
        for (int k = 0; k < 8; k++) rank[k] += kt < mykey[k] ? 1u : 0u;
    }
    #pragma unroll
    for (int k = 0; k < 8; k++) if (mykey[k] != 0xFFFFFFFFu) sym[rank[k]] = lane * 8 + k;
    __syncwarp();
    u32 ok = 0;
    if (lane == 0) ok = ze_huf_from_sorted(H, count, wk, present, mxs) ? 1u : 0u;
    return __shfl_sync(0xFFFFFFFFu, ok, 0) != 0;
}

// barrier over a subset of the CTA's warps (bar.sync id, threads); the CPU build of the kernels has its own
#ifdef ZB_SIMT_EMULATION
#define Z2_BAR_SYNC(id_, n_) simt_named_bar_sync(id_, n_)
#elif defined(__CUDA_ARCH__)
#define Z2_BAR_SYNC(id_, n_) asm volatile("bar.sync %0, %1;" :: "r"(id_), "r"(n_) : "memory")
#else
#define Z2_BAR_SYNC(id_, n_) do { } while (0)
#endif

#ifdef __CUDA_ARCH__
#define Z2_OPAQUE8(a_) asm volatile("" : "+r"(a_[0]), "+r"(a_[1]), "+r"(a_[2]), "+r"(a_[3]), "+r"(a_[4]), "+r"(a_[5]), "+r"(a_[6]), "+r"(a_[7]) :: "memory")
#else
#define Z2_OPAQUE8(a_) do { } while (0)
#endif

#ifdef ZB_PHASE_TIMERS
__device__ unsigned long long g_z2_phase[16];
#define Z2_MARK(k) do { if (tid == 0) { long long const t_ = clock64(); atomicAdd(&g_z2_phase[k], (unsigned long long)(t_ - t_phase)); t_phase = t_; } } while (0)
#define Z2_T0() t_aux = clock64()
#define Z2_T1(k) atomicAdd(&g_z2_phase[k], (unsigned long long)(clock64() - t_aux))
#else
#define Z2_MARK(k) do { } while (0)
#define Z2_T0() do { } while (0)
#define Z2_T1(k) do { } while (0)
#endif

// records of one unit, four at a time (two 16-byte loads in flight) so that the L2 latency is paid once per four
#define Z2_FOR_RECS(k0_, k1_, r_, q_, ...) \
    for (u32 b_ = (k0_) & ~1u; b_ < (k1_); b_ += 4) { \
        ulonglong2 const v0_ = *(const ulonglong2*)(myrec + b_); \
        ulonglong2 const v1_ = b_ + 2 < (k1_) ? *(const ulonglong2*)(myrec + b_ + 2) : make_ulonglong2(0, 0); \
        u64 const rr_[4] = {v0_.x, v0_.y, v1_.x, v1_.y}; \
        _Pragma("unroll") for (u32 i_ = 0; i_ < 4; i_++) { u32 const q_ = b_ + i_; if (q_ >= (k0_) && q_ < (k1_)) { u64 const r_ = rr_[i_]; __VA_ARGS__ } } }

__global__ void __launch_bounds__(Z2_NT, 1)
zb_compress_smem(const u8* __restrict__ src, const ZeBlockJob* __restrict__ jobs, u32 n_jobs, Z2Scratch* __restrict__ scratch,
                 u8* __restrict__ slots, u64 slot_bytes, ZeBlockOut* __restrict__ outs, u32* __restrict__ work_counter, ZeUpload up)
{
    ZB_DYN_SMEM(z2_smem_raw);
    Z2Shared& S = *(Z2Shared*)z2_smem_raw;
    Z2Scratch& G = scratch[blockIdx.x];
    u32 const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#ifdef ZB_PHASE_TIMERS
    long long t_phase = clock64(), t_aux = 0;
#endif

    // symbol code look-up tables (ZSTD_LLcode / ZSTD_MLcode, zstd/zstd.c:19738,:19755), derived from the baselines
    if (tid < 64) { u32 c = tid < 16 ? tid : 16; if (tid >= 16) while (c < 35 && tid >= e_LL_base[c + 1]) c++; S.llcode[tid] = (u8)c; }
    if (tid < 128) { u32 c = tid < 32 ? tid : 32; if (tid >= 32) while (c < 52 && tid + 3 >= e_ML_base[c + 1]) c++; S.mlcode[tid] = (u8)c; }
#ifdef __CUDA_ARCH__
    u32 const mbar = (u32)__cvta_generic_to_shared(&S.mbar);
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(mbar));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    u32 parity = 0;
#endif
    __syncthreads();

    for (;;) {
        // ---------------- next block; its bytes go global -> shared memory in one bulk copy
        if (tid == 0) {
            u32 const jn = atomicAdd(work_counter, 1u);
            if (up.progress && jn < n_jobs) {       // host input still being uploaded: wait until this block (and a margin) has landed
                unsigned long long const want = jobs[jn].src_pos + jobs[jn].size + 256u;
                unsigned long long const need = want < up.total ? want : up.total;
                long long t0 = clock64(); unsigned long long seen = 0;
                for (;;) {
                    unsigned long long const now = *(volatile const unsigned long long*)up.progress;
                    if (now >= need) break;
                    if (now != seen) { seen = now; t0 = clock64(); }                  // the upload is making progress
                    __nanosleep(400);
                    if (clock64() - t0 > 6000000000ll) { atomicExch(up.status, 1u); break; }
                }
                __threadfence();
            }
            S.job = jn;
#ifdef __CUDA_ARCH__
            if (jn < n_jobs && jobs[jn].size) {
                const u8* const p = src + jobs[jn].src_pos;
                const u8* const pal = (const u8*)((uintptr_t)p & ~(uintptr_t)15);
                u32 const bytes = ((u32)(p - pal) + jobs[jn].size + 15u) & ~15u;
                u32 const dst = (u32)__cvta_generic_to_shared(S.in);
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mbar), "r"(bytes) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             :: "r"(dst), "l"(pal), "r"(bytes), "r"(mbar) : "memory");
            }
#endif
        }
        __syncthreads();
        u32 const j = S.job;
        if (j >= n_jobs) return;
        ZeBlockJob const job = jobs[j];
        u32 const n = job.size;
        const u8* const gsrc = src + job.src_pos;
        u32 const skew = (u32)((uintptr_t)gsrc & 15);
        u8* const out = slots + (u64)j * slot_bytes;
        u32* const ow = (u32*)out;                                    // slots are 16-byte aligned
        const u8* const in = S.in;                                    // block byte i is in[skew + i]
        // while the copy is in flight: clear the far table
        for (u32 i = tid; i < (1u << Z2_FARLOG) / 2; i += Z2_NT) ((u32*)S.mf.far)[i] = 0u;
        if (tid == 0) { S.bad = 0; S.all_same = 1; }
#ifdef __CUDA_ARCH__
        if (n) { u32 ok = 0;
          while (!ok) asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                                   : "=r"(ok) : "r"(mbar), "r"(parity) : "memory");
          parity ^= 1; }
#else
        for (u32 i = tid; i < n; i += Z2_NT) S.in[skew + i] = gsrc[i];
#endif
        __syncthreads();
        if (tid < 32) S.in[skew + n + tid] = 0;                       // slack after the block: defined bytes for window loads
        __syncthreads();

        // ---------------- trivial blocks: tiny -> raw, all bytes equal -> RLE (not as the first block of a frame: the
        // reference emits its first block compressed, zstd/zstd.c:27378)
        if (n >= 9) {
            u8 const b0 = in[skew]; bool same = true;
            for (u32 i = tid; i < n && same; i += Z2_NT) if (in[skew + i] != b0) same = false;
            if (!same) S.all_same = 0;
            __syncthreads();
            if (S.all_same && !job.first) {
                if (tid == 0) { u32 const bh = job.last | (1u << 1) | (n << 3); out[0] = (u8)bh; out[1] = (u8)(bh >> 8); out[2] = (u8)(bh >> 16); out[3] = b0; outs[j].csize = 4; }
                __syncthreads();
                continue;
            }
        } else {
            for (u32 i = tid; i < n; i += Z2_NT) out[3 + i] = in[skew + i];
            if (tid == 0) { u32 const bh = job.last | (n << 3); out[0] = (u8)bh; out[1] = (u8)(bh >> 8); out[2] = (u8)(bh >> 16); outs[j].csize = 3 + n; }
            __syncthreads();
            continue;
        }
        Z2_MARK(0);

        // ================================================================= match finding
        // Positions are offsets into the shared-memory buffer here (s = skew + block position), so that groups of four and
        // eight positions are word-aligned whatever the block's alignment in global memory.  A pass covers Z2_Q positions:
        //   H  all threads: 14-bit hash of the five bytes at every position -> hd[]
        //   L  warp 0, 32 positions per step, in order: hd[s] = distance to the previous position with the same hash
        //      (one table for the whole block: the positions of a step do not see each other, everything earlier is exact)
        //   V  warps 1-31, four positions per thread: common prefix with the candidate, 4..15 (15 = "15 or more") -> ml[]
        //   P  warps 1-2, a lane per 132-byte unit: lazy greedy walk over ml[]; long matches are extended by the whole warp
        // L of pass k+1 runs beside V and P of pass k (hd[] and ml[] are double-buffered).
        u32 const e_end = skew + n;
        u32 const npass = (e_end + Z2_Q - 1) / Z2_Q;
        if (tid == 0) S.carry = 0;
        #define Z2_HASH_PASS(k_) do { \
            u32 const s0_ = (k_) * Z2_Q + 8 * tid; \
            uint2 const w01_ = *(const uint2*)(in + s0_); u32 const w2_ = *(const u32*)(in + s0_ + 8); \
            u32 wj_[9]; \
            wj_[0] = w01_.x; wj_[1] = __funnelshift_r(w01_.x, w01_.y, 8); wj_[2] = __funnelshift_r(w01_.x, w01_.y, 16); wj_[3] = __funnelshift_r(w01_.x, w01_.y, 24); \
            wj_[4] = w01_.y; wj_[5] = __funnelshift_r(w01_.y, w2_, 8); wj_[6] = __funnelshift_r(w01_.y, w2_, 16); wj_[7] = __funnelshift_r(w01_.y, w2_, 24); wj_[8] = w2_; \
            u32 hh_[8]; \
            _Pragma("unroll") for (u32 q_ = 0; q_ < 8; q_++) hh_[q_] = ((wj_[q_] * 2654435761u) ^ ((wj_[q_ + 1] >> 24) * 0x9E3779B1u)) >> (32 - Z2_FARLOG); \
            *(uint4*)&S.mf.hd[(k_) & 1][8 * tid] = make_uint4(hh_[0] | (hh_[1] << 16), hh_[2] | (hh_[3] << 16), hh_[4] | (hh_[5] << 16), hh_[6] | (hh_[7] << 16)); \
        } while (0)
        // eight steps' table accesses are issued back to back (the stores do not need the loads' results); the distances are
        // worked out afterwards (the empty asm keeps the compiler from pulling that work up between the loads)
        #define Z2_LG 8
        #define Z2_LINK_PASS(k_) do { \
            u16* const hd_ = S.mf.hd[(k_) & 1]; \
            u32 hq_[Z2_LG]; \
            _Pragma("unroll") for (u32 u_ = 0; u_ < Z2_LG; u_++) hq_[u_] = hd_[u_ * 32 + lane]; \
            for (u32 st_ = 0; st_ < Z2_Q / 32; st_ += Z2_LG) { \
                u32 hn_[Z2_LG], cc_[Z2_LG]; \
                _Pragma("unroll") for (u32 u_ = 0; u_ < Z2_LG; u_++) hn_[u_] = st_ + Z2_LG < Z2_Q / 32 ? (u32)hd_[(st_ + Z2_LG + u_) * 32 + lane] : 0u; \
                _Pragma("unroll") for (u32 u_ = 0; u_ < Z2_LG; u_++) { \
                    u32 const s_ = (k_) * Z2_Q + (st_ + u_) * 32 + lane; \
                    cc_[u_] = S.mf.far[hq_[u_]]; \
                    ZB_SIMT_STEP(); \
                    if (s_ >= skew && s_ + 8 <= e_end) S.mf.far[hq_[u_]] = (u16)s_; \
                    ZB_SIMT_STEP(); \
                } \
                Z2_OPAQUE8(cc_); \
                _Pragma("unroll") for (u32 u_ = 0; u_ < Z2_LG; u_++) { \
                    u32 const s_ = (k_) * Z2_Q + (st_ + u_) * 32 + lane; \
                    u32 const d_ = (s_ - cc_[u_]) & 0xFFFFu; \
                    hd_[(st_ + u_) * 32 + lane] = (u16)(s_ >= skew && s_ + 8 <= e_end && d_ + skew <= s_ ? d_ : 0u); \
                    hq_[u_] = hn_[u_]; \
                } \
            } \
        } while (0)
        Z2_HASH_PASS(0);
        __syncthreads();
        if (warp == 0) Z2_LINK_PASS(0);
        __syncthreads();
        Z2_MARK(1);
        for (u32 ps = 0; ps < npass; ps++) {
            u32 const q0 = ps * Z2_Q;
            if (ps + 1 < npass) Z2_HASH_PASS(ps + 1);
            __syncthreads();
            if (warp == 0) { if (ps + 1 < npass) Z2_LINK_PASS(ps + 1); }
            else {
                // ---- V + P: warp w owns the w-th region of Z2_REG positions of the pass and walks it in steps of 32: every lane
                // verifies its position's candidate (common prefix 4..15, 15 = "15 or more"), then the warp takes the matches
                // of the step greedily from the left (one-step lazy), extending long ones 256 bytes per vote

                const u16* const hd = S.mf.hd[ps & 1];
                u32 const carry = S.carry;                                    // end of the longest match of the earlier passes (buffer offset)
                u32 const reg = warp - 1;
                u32 const r0 = q0 + reg * Z2_REG, r1 = min(min(r0 + (u32)Z2_REG, q0 + (u32)Z2_Q), e_end);
                if (reg < Z2_RPP && r0 < r1) {
                    u32 const unit = ps * Z2_RPP + reg;
                    u64* const rec = G.rec + (u64)unit * Z2_RMAX;
                    u32 cover = max(max(r0, skew), carry), cnt = 0, endm = 0;
                    // the candidate of position pos_ (0 = none) and the bytes it shares with it, 4..15
                    #define Z2_VERIFY(pos_, m_, d_) { \
                        m_ = 0; d_ = 0; \
                        if ((pos_) < r1 && (pos_) > skew && (pos_) >= cover && (pos_) + 8 <= e_end) { \
                            d_ = hd[(pos_) - q0]; \
                            if (d_) { \
                                u64 const x_ = z2_ld64(in, (pos_)) ^ z2_ld64(in, (pos_) - d_); \
                                if (x_) m_ = ze_common8(0, x_); \
                                else m_ = 8 + ze_common8(z2_ld64(in, (pos_) + 8), z2_ld64(in, (pos_) + 8 - d_)); \
                                m_ = min(m_, min(15u, e_end - (pos_))); \
                                if (m_ < 4) m_ = 0; \
                            } \
                        } }
                    u32 m, d;
                    Z2_VERIFY(r0 + lane, m, d)
                    for (u32 b = r0; b < r1 && cover < r1; b += 32) {
                        u32 const pos = b + lane;
                        u32 m_nx, d_nx;                                       // the next step's candidates: their loads overlap this step's matches
                        Z2_VERIFY(pos + 32, m_nx, d_nx)
                        u32 mn = __shfl_down_sync(0xFFFFFFFFu, m, 1); if (lane == 31) mn = 0;
                        bool const take = m >= 4 && !(m < 15 && mn > m + 1);                 // one-step lazy
                        // selection: every match knows the first one that starts at or after its end (one ballot, no loop); the
                        // warp then hops from match to match.  Only "15 or more" matches are extended on the way.
                        u32 const takemask = __ballot_sync(0xFFFFFFFFu, take);
                        u32 my_end = pos + m;
                        #define Z2_NEXT_FROM(e_) ((e_) >= b + 32 ? 32u : min(32u, (u32)__ffs((int)(takemask & (0xFFFFFFFFu << ((e_) > b ? (e_) - b : 0u)))) - 1u))   /* 32 = none */
                        u32 my_hop = take ? (Z2_NEXT_FROM(my_end) | (m == 15 ? 0x100u : 0u)) : 0u;      // bit 8: to be extended
                        u32 selmask = 0, lastL = 0;
                        u32 L = Z2_NEXT_FROM(cover);
                        while (L < 32) {
                            selmask |= 1u << L; lastL = L;
                            u32 const hop = __shfl_sync(0xFFFFFFFFu, my_hop, (int)L);
                            if (hop & 0x100u) {                 // bytes [p, p + 15) match: compare on from p + 8, eight bytes per lane
                                u32 const dL = __shfl_sync(0xFFFFFFFFu, d, (int)L);
                                u32 a = b + L + 8, endL;
                                for (;;) {
                                    u32 const my = a + 8 * lane;
                                    u32 cm = 8;                 // bytes of my window that match
                                    if (my + 8 <= e_end) { u64 const x = z2_ld64(in, my) ^ z2_ld64(in, my - dL); if (x) cm = ze_common8(0, x); }
                                    else { cm = 0; while (my + cm < e_end && in[my + cm] == in[my + cm - dL]) cm++; }
                                    u32 const stop = __ballot_sync(0xFFFFFFFFu, cm < 8);
                                    if (stop) { u32 const fl = (u32)__ffs((int)stop) - 1; endL = a + 8 * fl + __shfl_sync(0xFFFFFFFFu, cm, (int)fl); break; }
                                    a += 256;
                                }
                                if (lane == L) my_end = endL;
                                L = Z2_NEXT_FROM(endL);
                            } else L = hop & 0xFFu;
                        }
                        u32 my_prev = cover;                    // the end of the match selected before mine
                        if (selmask) {
                            u32 const below = selmask & ((1u << lane) - 1u);
                            u32 const pe = __shfl_sync(0xFFFFFFFFu, my_end, below ? 31 - __clz((int)below) : 0);
                            if (below) my_prev = pe;
                            cover = __shfl_sync(0xFFFFFFFFu, my_end, (int)lastL);
                        }
                        // ... then every selected lane finishes its own match: up to four bytes backwards (down to the end of
                        // the match before it), record
                        if ((selmask >> lane) & 1u) {
                            u32 start = pos;
                            if (start > my_prev) {
                                if (start >= d + 4 + skew) {
                                    u32 const x = z2_ld32(in, start - 4) ^ z2_ld32(in, start - 4 - d);
                                    u32 const same = x ? ((u32)__clz((int)x) >> 3) : 4u;
                                    start -= min(same, start - my_prev);
                                } else while (start > my_prev && start > d + skew && in[start - 1] == in[start - 1 - d]) start--;
                            }
                            rec[cnt + (u32)__popc(selmask & ((1u << lane) - 1u))] = (u64)(start - skew) | ((u64)(my_end - start) << 17) | ((u64)d << 35);
                        }
                        if (selmask) { cnt += (u32)__popc(selmask); endm = cover - skew; }
                        m = pos + 32 >= cover ? m_nx : 0u; d = d_nx;
                    }
                    if (lane == 0) { S.x0[unit] = endm; S.x1[unit] = cnt; if (endm) atomicMax(&S.carry, endm + skew); }
                }

            }
            __syncthreads();
            Z2_MARK(8);
        }
        u32 const nunits = (npass - 1) * Z2_RPP + ((e_end - (npass - 1) * Z2_Q) + Z2_REG - 1) / Z2_REG;
        u32 const my_cnt = tid < nunits ? S.x1[tid] : 0u;
        __syncthreads();

        // ================================================================= stitch: cover on entry of every unit
        if (tid == 0) {
            u32 c = 0;
            for (u32 u = 0; u < nunits; u++) { S.x1[u] = c; u32 const e = S.x0[u]; if (e >= c + 3) c = e; }
            S.tail_from = c;
        }
        __syncthreads();
        // survivors of this unit: drop what an earlier match covers, front-trim the first one that sticks out by >= 3
        u32 const cin = tid < nunits ? S.x1[tid] : 0u;
        u32 first_k = my_cnt, lits = 0, ra = 0, rb = 0, rc = 0;
        const u64* const myrec = G.rec + (u64)tid * Z2_RMAX;
        if (my_cnt) {
            u32 cover = cin;
            Z2_FOR_RECS(0u, my_cnt, r, q, {
                u32 s = (u32)r & 0x1FFFFu; u32 const e = s + ((u32)(r >> 17) & 0x3FFFFu);
                if (first_k == my_cnt && (s >= cover || e >= cover + 3)) first_k = q;
                if (q >= first_k) {
                    if (s < cover) s = cover;
                    lits += s - cover; cover = e;
                    u32 const d = (u32)(r >> 35);          // the unit's three most recent distinct offsets (move to front)
                    if (d == ra) { } else if (d == rb) { rb = ra; ra = d; } else { rc = rb; rb = ra; ra = d; }
                }
            })
        }
        u32 const nsv = my_cnt - first_k;
        __syncthreads();
        S.x0[tid] = ra; S.x1[tid] = rb; S.x2[tid] = rc;
        u32 nseq, nlit_seq;
        u32 const seq_base = z2_scan(nsv, S.part, nseq);
        u32 const lit_base = z2_scan(lits, S.part, nlit_seq);
        // repcode history on entry of every unit: warp 0, lane l folds units [32 l, 32 l + 32)
        if (warp == 0) {
            u32 r0 = 0, r1 = 0, r2 = 0;
            for (u32 u = lane * 32; u < lane * 32 + 32 && u < nunits; u++) z2_rep_apply(r0, r1, r2, S.x0[u], S.x1[u], S.x2[u]);
            u32 e0 = 0, e1 = 0, e2 = 0;
            u32 s0 = job.first ? 1u : 0u, s1 = job.first ? 4u : 0u, s2 = job.first ? 8u : 0u;      // a frame starts from {1, 4, 8}; later blocks: unknown
            for (u32 l = 0; l < 32; l++) {
                u32 const a = __shfl_sync(0xFFFFFFFFu, r0, l), b = __shfl_sync(0xFFFFFFFFu, r1, l), c = __shfl_sync(0xFFFFFFFFu, r2, l);
                if (lane == l) { e0 = s0; e1 = s1; e2 = s2; }
                z2_rep_apply(s0, s1, s2, a, b, c);
            }
            for (u32 u = lane * 32; u < lane * 32 + 32 && u < nunits; u++) {
                u32 const a = S.x0[u], b = S.x1[u], c = S.x2[u];
                S.x0[u] = e0; S.x1[u] = e1; S.x2[u] = e2;
                z2_rep_apply(e0, e1, e2, a, b, c);
            }
        }
        Z2_MARK(9);
        for (u32 i = tid; i < 8 * 256; i += Z2_NT) ((u32*)S.en.hist)[i] = 0;
        if (tid < 36) S.en.hLL[tid] = 0;
        if (tid < 32) S.en.hOF[tid] = 0;
        if (tid < 56) S.en.hML[tid] = 0;
        __syncthreads();
        u32 const tail_from = S.tail_from;
        u32 const nlit = nlit_seq + (n - tail_from);
        u8* const lit = nlit <= Z2_STAGE ? (u8*)S.en.stage : G.lit;
        // final sequences (offsets coded against the true history), code histograms, literal gather + histogram
        if (nsv) {
            u32 r0 = S.x0[tid], r1 = S.x1[tid], r2 = S.x2[tid];
            u32 cover = cin, lp = lit_base; u32* const hist = S.en.hist[warp & 7];
            Z2_FOR_RECS(first_k, my_cnt, r, q, {
                u32 s = (u32)r & 0x1FFFFu; u32 const e = s + ((u32)(r >> 17) & 0x3FFFFu), d = (u32)(r >> 35);
                if (s < cover) s = cover;
                u32 const ll = s - cover, ml = e - s;
                if (ll == 0 && d == r0) S.bad = 1;         // two adjacent matches with one offset: cannot be formed (see the notes); raw block if it ever is
                u32 const ob = ze_off_code(d, ll, r0, r1, r2);
                u32 const lc = ll < 64 ? S.llcode[ll] : ze_hibit(ll) + 19, mc = ml - 3 < 128 ? S.mlcode[ml - 3] : ze_hibit(ml - 3) + 36, oc = ze_hibit(ob);
                G.fseq[seq_base + (q - first_k)] = (u64)ll | ((u64)(ml - 3) << 17) | ((u64)ob << 34) | ((u64)lc << 52) | ((u64)mc << 58);
                atomicAdd(&S.en.hLL[lc], 1u); atomicAdd(&S.en.hML[mc], 1u); atomicAdd(&S.en.hOF[oc], 1u);
                for (u32 k = 0; k < ll; k++) { u8 const b = in[skew + cover + k]; lit[lp + k] = b; atomicAdd(&hist[b], 1u); }
                lp += ll; cover = e;
            })
        }
        {   // last literals of the block
            u32* const hist = S.en.hist[warp & 7];
            for (u32 k = tid; k < n - tail_from; k += Z2_NT) { u8 const b = in[skew + tail_from + k]; lit[nlit_seq + k] = b; atomicAdd(&hist[b], 1u); }
        }
        __syncthreads();
        for (u32 s = tid; s < 256; s += Z2_NT) { u32 t = 0; for (int k = 0; k < 8; k++) t += S.en.hist[k][s]; S.en.hist[0][s] = t; }
        __syncthreads();
        Z2_MARK(2);

        // ================================================================= sub-blocks
        // The chunk's sequences are cut into up to Z2_MAXSUB runs of equal length and every run becomes a zstd block of its
        // own (its literals are a contiguous range of the gathered literals).  The FSE state chains -- three strictly serial
        // recurrences per block -- then run side by side, one lane per (sub-block, table), each over ~nseq / nsub
        // sequences.  The first sub-block carries the tables; the others say "repeat" (sequences) / "treeless" (literals).
        // The input buffer is dead from here on (a raw block is copied from global memory): it takes the sequence records.
        u64* const sq = (u64*)S.in;
        for (u32 i = tid; i < nseq && i < Z2_SEQ_SMEM; i += Z2_NT) sq[i] = G.fseq[i];
        #define Z2_SEQ(i_) ((i_) < Z2_SEQ_SMEM ? sq[i_] : G.fseq[i_])
        u32 const K = nseq ? (nseq + Z2_NT - 1) / Z2_NT : 1u;
        u32 const nthr = (nseq + K - 1) / K;                                   // threads that own sequences
        u32 const want = nseq ? min((u32)Z2_MAXSUB, (nseq + Z2_SUBSEQ - 1) / Z2_SUBSEQ) : 1u;
        u32 const tps = nseq ? (nthr + want - 1) / want : 1u;                  // threads per sub-block
        u32 const nsub = nseq ? (nthr + tps - 1) / tps : 1u;
        u32 const lo = tid * K, hi = min(lo + K, nseq);
        bool const act = lo < nseq;
        u32 const mysub = act ? tid / tps : 0u;
        __syncthreads();
        {   // where every sub-block's literals start
            u32 lsum = 0;
            if (act) for (u32 i = lo; i < hi; i++) lsum += (u32)Z2_SEQ(i) & 0x1FFFFu;
            u32 tot; u32 const lpre = z2_scan(lsum, S.part, tot);
            if (act && tid % tps == 0) { S.sub_lit[mysub] = lpre; S.sub_seq[mysub] = lo; }
            if (tid == 0) { S.sub_lit[nsub] = nlit; S.sub_seq[nsub] = nseq; if (!nseq) { S.sub_lit[0] = 0; S.sub_seq[0] = 0; } }
        }
        __syncthreads();
        // ================================================================= entropy tables and FSE state chains, side by side
        //   warps 0-2: the LL / OF / ML tables (one lane each), then warp 0 runs the state chains
        //   warp 3   : the Huffman code of the literals and its description
        Z2_T0();
        if (warp < 3) {
            if (nseq) {
                if (warp == 0) z2_make_table_warp(S.en.ct[0], S.en.hLL, 35, nseq, 9, 6, e_LL_defnorm, 35, S.en.tmp_sym[0], S.en.nrm[0], S.en.cum[0], lane);
                if (warp == 1) z2_make_table_warp(S.en.ct[1], S.en.hOF, 31, nseq, 8, 5, e_OF_defnorm, 28, S.en.tmp_sym[1], S.en.nrm[1], S.en.cum[1], lane);
                if (warp == 2) z2_make_table_warp(S.en.ct[2], S.en.hML, 52, nseq, 9, 6, e_ML_defnorm, 52, S.en.tmp_sym[2], S.en.nrm[2], S.en.cum[2], lane);
            }
            if (tid == 0) Z2_T1(7);
            Z2_BAR_SYNC(2, 96);
            if (tid == 0) Z2_T0();
            // ---- FSE state chains: warp 0, lane 3 * sub-block + table (0 LL, 1 OF, 2 ML) walks its sub-block from the last
            // sequence to the first and leaves the state on entry of every thread's range in x0 / x1 / x2 (the ranges are then
            // re-run by their threads, all at once, to count and to write the bits)
            if (warp == 0 && nseq) {
                u32 const sb = lane / 3, t = lane - 3 * sb;
                if (sb < nsub) {
                    ZeCTable const& ct = S.en.ct[t];
                    if (ct.mode == 1) S.fin[sb][t] = 0;            // RLE: no state bits
                    else {
                        u32* const xb = t == 0 ? S.x0 : t == 1 ? S.x1 : S.x2;
                        u32 const s_lo = S.sub_seq[sb], s_hi = S.sub_seq[sb + 1];
                        u32 const sh = t == 0 ? 52u : 58u;
                        u32 const m_of = t == 1 ? 0xFFFFFFFFu : 0u;           // branch-free selection: the three lanes of a sub-block stay converged
                        #define Z2_CODE_OF(r_) ((ze_hibit(((u32)((r_) >> 34) & 0x3FFFFu) | 1u) & m_of) | ((u32)((r_) >> sh) & 63u & ~m_of))
                        u32 i = s_hi - 1;
                        u32 q = i / K, r = i - q * K;
                        u32 state = z2_fse_init(ct, Z2_CODE_OF(Z2_SEQ(i)));
                        int dnb = 0, dfs = 0;
                        if (i > s_lo) { u32 const sym = Z2_CODE_OF(Z2_SEQ(i - 1)); dnb = ct.dnb[sym]; dfs = ct.dfs[sym]; }
                        // two sequences ahead: the record; one ahead: its symbol's deltas; now: the state transition
                        #define Z2_CHAIN_LOOP(SEQ_) { \
                            u64 rr1_ = i > s_lo + 1 ? SEQ_(i - 2) : 0ull; \
                            while (i > s_lo) { \
                                i--; if (r == 0) { r = K - 1; q--; } else r--; \
                                u64 const rr2_ = i > s_lo + 1 ? SEQ_(i - 2) : 0ull; \
                                u32 const nsym_ = Z2_CODE_OF(rr1_); \
                                int const ndnb_ = ct.dnb[nsym_], ndfs_ = ct.dfs[nsym_]; \
                                if (r == K - 1) xb[q] = state; \
                                u32 const nb_ = (state + (u32)dnb) >> 16; \
                                state = ct.state[(state >> nb_) + dfs]; \
                                dnb = ndnb_; dfs = ndfs_; rr1_ = rr2_; \
                            } }
                        #define Z2_SEQ_S(i_) sq[i_]
                        if (s_hi <= Z2_SEQ_SMEM) Z2_CHAIN_LOOP(Z2_SEQ_S) else Z2_CHAIN_LOOP(Z2_SEQ)
                        S.fin[sb][t] = state;
                    }
                }
            }
            if (tid == 0) Z2_T1(13);
        } else if (warp == 3) {
            u32 mode = 0, tb = 0;
            u32 most = 0; for (u32 s = lane; s < 256; s += 32) most = max(most, S.en.hist[0][s]);
            #pragma unroll
            for (int d = 16; d > 0; d >>= 1) most = max(most, __shfl_xor_sync(0xFFFFFFFFu, most, d));
            if (nlit >= 8 && most == nlit) mode = 1;                                   // RLE literals
            else if (nlit >= 64) {                                                     // ZSTD_minLiteralsToCompress, zstd/zstd.c:20918
                bool const ok = z2_huf_build(S.en.huf, S.en.hist[0], S.en.wk, lane);
                if (lane == 0 && ok) { tb = ze_huf_write_table(S.en.huf_tbl, S.en.huf, S.en.ct[3], S.en.tmp_sym[3]); if (tb) mode = 2; }
            }
            if (lane == 0) { S.lit_mode = mode; S.huf_tbl_bytes = tb; }
            if (lane == 0) Z2_T1(15);
        }
        __syncthreads();
        Z2_MARK(3);
        u32 const chunk_lit_mode = S.lit_mode, tb = S.huf_tbl_bytes;
        // ---- Huffman streams: every sub-block with >= 64 literals gets one (< 256 literals) or four streams
        if (tid == 0) {
            u32 ns = 0, cum = 0;
            for (u32 sb = 0; sb < nsub; sb++) {
                u32 const l0 = S.sub_lit[sb], nl = S.sub_lit[sb + 1] - l0;
                S.sub_st0[sb] = ns;
                if (chunk_lit_mode == 2 && nl >= 64) {
                    u32 const nst = nl >= 256 ? 4u : 1u, seg = nst == 4 ? (nl + 3) / 4 : nl;
                    for (u32 k = 0; k < nst; k++) {
                        u32 const a0 = k * seg, a1 = k == nst - 1 ? nl : (k + 1) * seg;
                        S.st_start[ns] = l0 + a0; S.st_len[ns] = a1 - a0; S.st_cum[ns] = cum; cum += (a1 - a0 + 31) / 32; ns++;
                    }
                }
            }
            S.sub_st0[nsub] = ns; S.st_cum[ns] = cum; S.n_streams = ns;
        }
        __syncthreads();
        u32 const n_streams = S.n_streams, n_chunks = S.st_cum[n_streams];
        // a chunk = 32 literals of one stream; its bytes come as nine aligned words
        #define Z2_CHUNK_LOAD(g_, k_, c_, cnt_, cw_) \
            u32 k_ = 0, c_ = 0, cnt_ = 0; u32 cw_[8]; \
            if ((g_) < n_chunks) { \
                { u32 a_ = 0, b_ = n_streams; while (b_ - a_ > 1) { u32 const m_ = (a_ + b_) >> 1; if (S.st_cum[m_] <= (g_)) a_ = m_; else b_ = m_; } k_ = a_; } \
                c_ = (g_) - S.st_cum[k_]; cnt_ = min(32u, S.st_len[k_] - 32 * c_); \
                u32 const off_ = S.st_start[k_] + 32 * c_; const u32* const wp_ = (const u32*)lit + (off_ >> 2); u32 const sh_ = (off_ & 3) * 8; \
                u32 prev_ = wp_[0]; \
                _Pragma("unroll") for (u32 q_ = 0; q_ < 8; q_++) { u32 const nx_ = wp_[q_ + 1]; cw_[q_] = __funnelshift_r(prev_, nx_, sh_); prev_ = nx_; } \
            } else { _Pragma("unroll") for (u32 q_ = 0; q_ < 8; q_++) cw_[q_] = 0; }
        u32 const lrounds = (n_chunks + Z2_NT - 1) / Z2_NT;                     // <= 5
        u32 cbits[5] = {0, 0, 0, 0, 0}, cpre[5] = {0, 0, 0, 0, 0};
        {
            u32 running = 0;
            #pragma unroll
            for (u32 rd = 0; rd < 5; rd++) if (rd < lrounds) {
                u32 const g = rd * Z2_NT + tid;
                Z2_CHUNK_LOAD(g, k, c, cnt, cw)
                u32 bits = 0;
                #pragma unroll
                for (u32 q = 0; q < 32; q++) if (q < cnt) bits += S.en.huf.nb[(cw[q >> 2] >> ((q & 3) * 8)) & 255u];
                u32 tot; u32 const pre = z2_scan(bits, S.part, tot) + running;
                cbits[rd] = bits; cpre[rd] = pre;
                if (g < n_chunks && c == 0) S.st_pre[k] = pre;
                running += tot;
            }
            if (tid == 0) S.st_pre[n_streams] = running;
        }
        __syncthreads();
        Z2_MARK(11);
        Z2_MARK(10);
        // ---- every thread re-runs its range from the recorded states: bit count, then (below) the bits themselves
        ZeCTable const& cL = S.en.ct[0]; ZeCTable const& cO = S.en.ct[1]; ZeCTable const& cM = S.en.ct[2];
        bool const rL = cL.mode == 1, rO = cO.mode == 1, rM = cM.mode == 1;
        u32 const my_shi = act ? S.sub_seq[mysub + 1] : 0u;
        u32 inL = 0, inO = 0, inM = 0;
        if (act) {
            if (hi == my_shi) { u64 const r = Z2_SEQ(hi - 1); u32 const lc = (u32)(r >> 52) & 63u, mc = (u32)(r >> 58), oc = ze_hibit((u32)(r >> 34) & 0x3FFFFu);
                                inL = rL ? 0u : z2_fse_init(cL, lc); inO = rO ? 0u : z2_fse_init(cO, oc); inM = rM ? 0u : z2_fse_init(cM, mc); }
            else { inL = S.x0[tid]; inO = S.x1[tid]; inM = S.x2[tid]; }
        }
        u32 sbits = 0;
        if (act) {
            u32 sL = inL, sO = inO, sM = inM;
            for (u32 i = hi; i-- > lo;) {
                u64 const r = Z2_SEQ(i);
                u32 const lc = (u32)(r >> 52) & 63u, mc = (u32)(r >> 58), oc = ze_hibit((u32)(r >> 34) & 0x3FFFFu);
                sbits += e_LL_bits[lc] + e_ML_bits[mc] + oc;
                if (i == my_shi - 1) continue;                                       // the last sequence only initialises the states
                if (!rO) { u32 const nb = (sO + (u32)cO.dnb[oc]) >> 16; sbits += nb; sO = cO.state[(sO >> nb) + cO.dfs[oc]]; }
                if (!rM) { u32 const nb = (sM + (u32)cM.dnb[mc]) >> 16; sbits += nb; sM = cM.state[(sM >> nb) + cM.dfs[mc]]; }
                if (!rL) { u32 const nb = (sL + (u32)cL.dnb[lc]) >> 16; sbits += nb; sL = cL.state[(sL >> nb) + cL.dfs[lc]]; }
            }
        }
        u32 seq_tot; u32 const spre = z2_scan(sbits, S.part, seq_tot);
        if (act && tid % tps == 0) S.sub_spre[mysub] = spre;
        if (tid == 0) S.sub_spre[nsub] = seq_tot;
        __syncthreads();
        // ---- layout (thread 0): literal mode, header sizes and byte offset of every sub-block
        if (tid == 0) {
            bool have_tree = false; u32 off = 0;
            u32 const logsum = nseq ? (S.en.ct[0].mode == 1 ? 0u : S.en.ct[0].log) + (S.en.ct[1].mode == 1 ? 0u : S.en.ct[1].log) + (S.en.ct[2].mode == 1 ? 0u : S.en.ct[2].log) : 0u;
            u32 hdr_first = 0, hdr_next = 0;               // table descriptions in the first / the following sub-blocks
            if (nseq) for (int t = 0; t < 3; t++) { hdr_first += S.en.ct[t].hdr_bytes; if (S.en.ct[t].mode == 1) hdr_next += 1; }
            for (u32 sb = 0; sb < nsub; sb++) {
                u32 const nl = S.sub_lit[sb + 1] - S.sub_lit[sb];
                u32 mode = 0, pay = nl, lh;
                if (chunk_lit_mode == 1 && nl) { mode = 1; pay = 1; }
                else if (chunk_lit_mode == 2 && nl >= 64) {
                    u32 const k0 = S.sub_st0[sb], k1 = S.sub_st0[sb + 1];
                    u32 est = (have_tree ? 0u : tb) + (k1 - k0 == 4 ? 6u : 0u);
                    for (u32 k = k0; k < k1; k++) est += (S.st_pre[k + 1] - S.st_pre[k] + 1 + 7) / 8;
                    if (est < nl) { mode = have_tree ? 3u : 2u; have_tree = true; pay = est; }
                }
                if (mode >= 2) lh = 3 + (nl >= 1024) + (nl >= 16384); else lh = 1 + (nl > 31) + (nl > 4095);
                u32 const ns = S.sub_seq[sb + 1] - S.sub_seq[sb];
                u32 shb = ns < 128 ? 1u : (ns < 0x7F00 ? 2u : 3u);
                u32 spay = 0;
                if (ns) { shb += 1 + (sb == 0 ? hdr_first : hdr_next); spay = (S.sub_spre[sb + 1] - S.sub_spre[sb] + logsum + 1 + 7) / 8; }
                S.sub_mode[sb] = mode; S.sub_lh[sb] = lh; S.sub_pay[sb] = pay; S.sub_shb[sb] = shb; S.sub_spay[sb] = spay; S.sub_off[sb] = off;
                off += 3 + lh + pay + shb + spay;
            }
            S.sub_off[nsub] = off;
        }
        __syncthreads();
        Z2_MARK(12);
        u32 const body_total = S.sub_off[nsub];
        bool const use_raw = S.bad || body_total + (n >> 7) + 2 >= n + 3 * nsub || body_total >= slot_bytes;
        if (use_raw) {          // cSize >= srcSize - minGain (zstd/zstd.c:25987): one raw block
            for (u32 i = tid; i < n; i += Z2_NT) out[3 + i] = gsrc[i];
            if (tid == 0) { u32 const bh = job.last | (n << 3); out[0] = (u8)bh; out[1] = (u8)(bh >> 8); out[2] = (u8)(bh >> 16); outs[j].csize = 3 + n; }
            Z2_MARK(5);
            __syncthreads();
            continue;
        }
        for (u32 i = tid; i < body_total / 4 + 2; i += Z2_NT) ow[i] = 0;
        __syncthreads();
        // ---- headers: block, literals section, sequences section (OR-ed: their words also hold payload bits)
        if (tid < nsub) {
            u32 const sb = tid, o = S.sub_off[sb], mode = S.sub_mode[sb], lh = S.sub_lh[sb], pay = S.sub_pay[sb];
            u32 const nl = S.sub_lit[sb + 1] - S.sub_lit[sb], ns = S.sub_seq[sb + 1] - S.sub_seq[sb];
            u32 const bsz = S.sub_off[sb + 1] - o - 3;
            u32 const bh = ((job.last && sb == nsub - 1) ? 1u : 0u) | (2u << 1) | (bsz << 3);
            z2_or_byte(ow, o, bh); z2_or_byte(ow, o + 1, bh >> 8); z2_or_byte(ow, o + 2, bh >> 16);
            u32 hb[5] = {0, 0, 0, 0, 0};
            if (mode >= 2) {        // ZSTD_compressLiterals, zstd/zstd.c:20932-21038
                bool const four = S.sub_st0[sb + 1] - S.sub_st0[sb] == 4;
                if (lh == 3) { u32 const v = mode | ((four ? 1u : 0u) << 2) | (nl << 4) | (pay << 14); hb[0] = v; hb[1] = v >> 8; hb[2] = v >> 16; }
                else if (lh == 4) { u32 const v = mode | (2u << 2) | (nl << 4) | (pay << 18); hb[0] = v; hb[1] = v >> 8; hb[2] = v >> 16; hb[3] = v >> 24; }
                else { u32 const v = mode | (3u << 2) | (nl << 4) | (pay << 22); hb[0] = v; hb[1] = v >> 8; hb[2] = v >> 16; hb[3] = v >> 24; hb[4] = pay >> 10; }
            } else {                // ZSTD_noCompressLiterals / ZSTD_compressRleLiteralsBlock, zstd/zstd.c:20851-20930
                if (lh == 1) hb[0] = mode | (nl << 3);
                else if (lh == 2) { u32 const v = mode | (1u << 2) | (nl << 4); hb[0] = v; hb[1] = v >> 8; }
                else { u32 const v = mode | (3u << 2) | (nl << 4); hb[0] = v; hb[1] = v >> 8; hb[2] = v >> 16; }
            }
            for (u32 k = 0; k < lh; k++) z2_or_byte(ow, o + 3 + k, hb[k]);
            if (mode == 1) z2_or_byte(ow, o + 3 + lh, lit[S.sub_lit[sb]]);
            // sequences section header (ZSTD_entropyCompressSeqStore_internal, zstd/zstd.c:25893-25926)
            u32 q = o + 3 + lh + pay;
            if (ns < 128) z2_or_byte(ow, q++, ns);
            else if (ns < 0x7F00) { z2_or_byte(ow, q++, (ns >> 8) + 0x80); z2_or_byte(ow, q++, ns); }
            else { z2_or_byte(ow, q++, 0xFF); z2_or_byte(ow, q++, ns - 0x7F00); z2_or_byte(ow, q++, (ns - 0x7F00) >> 8); }
            if (ns) {
                u32 md = 0;
                for (int t = 0; t < 3; t++) { u32 const m = S.en.ct[t].mode; md |= (sb == 0 || m != 2 ? m : 3u) << (6 - 2 * t); }
                z2_or_byte(ow, q++, md);
                for (int t = 0; t < 3; t++) {
                    u32 const nb = sb == 0 ? S.en.ct[t].hdr_bytes : (S.en.ct[t].mode == 1 ? 1u : 0u);
                    for (u32 i = 0; i < nb; i++) z2_or_byte(ow, q++, S.en.ct[t].hdr[i]);
                }
            }
        }
        // ---- literal payloads
        for (u32 sb = 0; sb < nsub; sb++) {
            u32 const mode = S.sub_mode[sb], o_pl = S.sub_off[sb] + 3 + S.sub_lh[sb], l0 = S.sub_lit[sb], nl = S.sub_lit[sb + 1] - l0;
            if (mode == 0) { for (u32 i = tid; i < nl; i += Z2_NT) z2_or_byte(ow, o_pl + i, lit[l0 + i]); }
            else if (mode >= 2) {
                u32 const k0 = S.sub_st0[sb], k1 = S.sub_st0[sb + 1];
                u32 o = o_pl;
                if (mode == 2) { for (u32 i = tid; i < tb; i += Z2_NT) z2_or_byte(ow, o + i, S.en.huf_tbl[i]); o += tb; }
                if (tid == 0) {         // jump table, stream positions, end marks
                    u32 q = o + (k1 - k0 == 4 ? 6u : 0u);
                    for (u32 k = k0; k < k1; k++) {
                        u32 const bits = S.st_pre[k + 1] - S.st_pre[k], bytes = (bits + 1 + 7) / 8;
                        if (k1 - k0 == 4 && k < k1 - 1) { z2_or_byte(ow, o + 2 * (k - k0), bytes); z2_or_byte(ow, o + 2 * (k - k0) + 1, bytes >> 8); }
                        S.st_byte[k] = q;
                        atomicOr(&ow[(q * 8 + bits) >> 5], 1u << ((q * 8 + bits) & 31));
                        q += bytes;
                    }
                }
            }
        }
        __syncthreads();
        #pragma unroll
        for (u32 rd = 0; rd < 5; rd++) if (rd < lrounds) {
            u32 const g = rd * Z2_NT + tid;
            Z2_CHUNK_LOAD(g, k, c, cnt, cw)
            (void)c;
            if (g < n_chunks) {
                // the sub-block of stream k; symbols are written last to first: a chunk's span ends where the bits before it begin
                u32 sb = 0; while (S.sub_st0[sb + 1] <= k) sb++;
                if (S.sub_mode[sb] >= 2) {
                    u32 const tot = S.st_pre[k + 1] - S.st_pre[k];
                    Z2Bits w; w.init(ow, S.st_byte[k] * 8 + (tot - (cpre[rd] - S.st_pre[k]) - cbits[rd]));
                    #pragma unroll
                    for (u32 qq = 0; qq < 32; qq++) { u32 const q = 31 - qq; if (q < cnt) { u32 const sym = (cw[q >> 2] >> ((q & 3) * 8)) & 255u; w.put(S.en.huf.code[sym], S.en.huf.nb[sym]); } }
                    w.flush();
                }
            }
        }
        Z2_MARK(4);
        // ---- sequence streams: every thread packs its own span
        if (act) {
            u32 const sb = mysub;
            u32 const o_st = S.sub_off[sb] + 3 + S.sub_lh[sb] + S.sub_pay[sb] + S.sub_shb[sb];
            u32 const tot = S.sub_spre[sb + 1] - S.sub_spre[sb];
            Z2Bits w; w.init(ow, o_st * 8 + (tot - (spre - S.sub_spre[sb]) - sbits));
            u32 sL = inL, sO = inO, sM = inM;
            for (u32 i = hi; i-- > lo;) {
                u64 const r = Z2_SEQ(i);
                u32 const ll = (u32)r & 0x1FFFFu, mb = (u32)(r >> 17) & 0x1FFFFu, ob = (u32)(r >> 34) & 0x3FFFFu;
                u32 const lc = (u32)(r >> 52) & 63u, mc = (u32)(r >> 58), oc = ze_hibit(ob);
                if (i != my_shi - 1) {
                    if (!rO) { u32 const nb = (sO + (u32)cO.dnb[oc]) >> 16; w.put(sO, nb); sO = cO.state[(sO >> nb) + cO.dfs[oc]]; }
                    if (!rM) { u32 const nb = (sM + (u32)cM.dnb[mc]) >> 16; w.put(sM, nb); sM = cM.state[(sM >> nb) + cM.dfs[mc]]; }
                    if (!rL) { u32 const nb = (sL + (u32)cL.dnb[lc]) >> 16; w.put(sL, nb); sL = cL.state[(sL >> nb) + cL.dfs[lc]]; }
                }
                w.put(ll, e_LL_bits[lc]); w.put(mb, e_ML_bits[mc]); w.put(ob, oc);
            }
            if (tid % tps == 0) {       // flush ML, OF, LL states + end mark
                u32 const logL = rL ? 0u : cL.log, logO = rO ? 0u : cO.log, logM = rM ? 0u : cM.log;
                w.put(sM, logM); w.put(sO, logO); w.put(sL, logL); w.put(1, 1);
            }
            w.flush();
        }
        if (tid == 0) outs[j].csize = body_total;
        Z2_MARK(5);
        Z2_MARK(6);
        __syncthreads();
    }
}
static_assert(sizeof(Z2Shared) <= 227 * 1024, "Z2Shared exceeds the 227 KB a CTA may own");

