// zb_entropy.cuh -- K3, the entropy stage (included by zb_decode.cu).
//
// One LANE per frame: the bit-serial chains of a frame (Huffman literal streams, FSE table
// builds, the 3-state FSE sequence stream, repcode history) cannot be parallelised inside a
// block, so 32 independent frames advance in lock-step per warp and every issue slot carries
// 32 frames' worth of serial work.
//
// Every decode table lives in SHARED MEMORY: each warp owns a pool, lanes claim exactly the
// bytes their tables need (2^log cells) through a warp prefix-scan, and when a pool cannot hold
// all 32 claims the remaining lanes run in a second pass.  A frame's tables are rebuilt per block
// from the header that defined them ("repeat" modes re-read that header), so nothing but a few
// descriptors has to survive between blocks.
//
// Restates, per lane: ZSTD_decodeLiteralsBlock (zstd/zstd.c:45767), HUF_readStats (:3457),
// HUF_readDTableX1_wksp (:39651), HUF_decompress{1,4}X1_usingDTable_internal_body (:39845,:39868),
// ZSTD_decodeSeqHeaders (:46328), ZSTD_buildFSETable_body (:46118), ZSTD_decodeSequence (:46862).
#pragma once

// Warps per CTA (one CTA per SM) is a template parameter: each warp owns a shared-memory pool of
// (227 KB - head) / warps.  Level-3 frames of a few KiB carry three FSE tables of 64-128 cells (~500 B per lane in 16-bit
// cells, so that all 32 lanes of a warp fit in one pass) and a ~600 B Huffman table: 8 warps (28.9 KB pools) serve them
// best; frames of 16 KiB and more have larger tables and run faster with 7 warps and 33 KB pools (measured 7.2 vs 8.8 ms on 65536 x 16 KiB), since a lane whose tables do not fit waits
// for a second pass.
//
// In front of the pools sits a CTA-wide head: the LL / ML baseline LUTs, the three predefined FSE tables and, when the
// dictionary carries entropy tables, the dictionary's three FSE tables (at most 2.5 KB, taken from the pools of that call),
// all in 16-bit cells (ZB_CELL16).  So every table the sequence loop reads is in shared memory and is addressed by a
// 32-bit offset: its cell loads are LDS.
#define ZB_ENT_WS_BYTES   256                     // per-lane workspace (weights / normalized counts)
// Lanes' workspaces lie 16 bytes further apart than their size.  The lanes of a warp touch the same workspace offset at the
// same moment (norm[s] while the FSE tables are built, the nibble of weight i), and at a 256-byte stride all 32 of those
// addresses fall in one bank; at 272 bytes they spread over 8 banks (shared memory is 32 banks of 4 bytes, and the bit
// readers' rings need 16-byte alignment, so 8 is the most a 16-byte skew gives).  The claim of the three FSE tables and the
// weight stream's rings are odd multiples of 16 bytes for the same reason; the Huffman table's claim is not skewed (its
// size varies from lane to lane, and its pool space is the tighter one).
#define ZB_ENT_WS_STRIDE  (ZB_ENT_WS_BYTES + 16)
#define ZB_ENT_SKEW(b)    ((((b) + 15u) & ~15u) | 16u)    // a claim of b bytes, rounded up to an odd multiple of 16
#define ZB_ENT_DEF_LL     512                     // after the baselines (LL_base, ML_base): predefined LL, OF, ML cells
#define ZB_ENT_DEF_OF     (ZB_ENT_DEF_LL + 2 * 64)
#define ZB_ENT_DEF_ML     (ZB_ENT_DEF_OF + 2 * 32)
#define ZB_ENT_HEAD_BYTES (ZB_ENT_DEF_ML + 2 * 64)  // the dictionary's tables follow, when there are any
#define ZB_ENT_POOL_BYTES(W) ((((227 * 1024 - ZB_ENT_HEAD_BYTES) / (W))) & ~15)
#define ZB_ENT_SMEM(W)    ((W) * ZB_ENT_POOL_BYTES(W) + ZB_ENT_HEAD_BYTES)

// where a table comes from; enough to rebuild it for a later block
enum : u32 { ZB_SRC_NONE = 0, ZB_SRC_PREDEF = 1, ZB_SRC_RLE = 2, ZB_SRC_NCOUNT = 3, ZB_SRC_DICT = 4 };
struct ZbTabSrc { u32 kind; u32 sym; const u8* p; u32 n; };

// ---- block-parallel decoding of frames with several blocks (zb_entropy_blocks below): what a lane needs to decode ONE block
// without having decoded the blocks before it.  Written per block by zb_scan_blocks (header parsing only).
enum : u32 { ZB_BD_FIRST = 1, ZB_BD_FSE_VALID = 2, ZB_BD_SKIP = 4 };
struct ZbBlkDesc {
    u64 hdr_off;                          // the block's 3-byte header, relative to src
    u64 seq_off, lit_off;                 // its sequence records / literal scratch
    u32 span;                             // header + payload bytes
    u32 frame;
    u32 flags;                            // ZB_BD_*
    u32 block_max;
    ZbTabSrc dHuf, dLL, dOF, dML;         // where the tables came from ON ENTRY ("treeless" / "repeat" re-read those headers)
};
struct ZbBlkExit { u32 rep[3]; u32 err; };   // repcode history on exit: concrete, or symbolic in the entry history (0x80000000 | k << 29 | d)

__device__ __forceinline__ u32 zb_warp_incl_scan(u32 v, u32 lane)
{
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { u32 y = __shfl_up_sync(0xFFFFFFFFu, v, d); if (lane >= (u32)d) v += y; }
    return v;
}

// Small counters packed into registers: field i (BITS wide) sits in word i / (32 / BITS).  Every access selects among the
// words with constant indices, so the lane's per-weight counts and cursors need no local memory.
template <int WORDS, int BITS>
struct ZbPacked {
    static constexpr u32 PER = 32 / BITS, MASK = (1u << BITS) - 1;
    u32 w[WORDS];
    __device__ __forceinline__ void clear() {
        #pragma unroll
        for (int j = 0; j < WORDS; j++) w[j] = 0;
    }
    __device__ __forceinline__ u32 get(u32 i) const {
        u32 const q = i / PER; u32 v = w[0];
        #pragma unroll
        for (int j = 1; j < WORDS; j++) v = q == (u32)j ? w[j] : v;
        return (v >> (BITS * (i - q * PER))) & MASK;
    }
    __device__ __forceinline__ void add(u32 i, u32 v) {
        u32 const q = i / PER, d = v << (BITS * (i - q * PER));
        #pragma unroll
        for (int j = 0; j < WORDS; j++) w[j] += q == (u32)j ? d : 0u;
    }
};
// the count of every Huffman weight 1..12 (at most 255 each), field wt - 1
struct ZbRank : ZbPacked<4, 10> {
    __device__ __forceinline__ u32 operator[](u32 wt) const { return get(wt - 1); }
    __device__ __forceinline__ void count(u32 wt) { if (wt) add(wt - 1, 1); }
};

// --- Huffman weights (HUF_readStats_body).  Weights go to ws as nibbles; the weight-FSE table
// --- (<= 64 cells, u16: sym | nb << 4 | next << 8) sits in ws + 128.
// returns header bytes consumed (0 = error); out: log, rank (count of every weight)
// `ring`: 64 bytes of the lane's shared memory for the bit reader (ws is full here)
__device__ static u32 zb_huf_weights(u8* ws, const u8* s, u32 n, u32& out_log, u32& out_nsym, ZbRank& rank, ZB_RING_ARG(ring))
{
    u8* const wn = ws;                       // 128 bytes: 256 nibbles
    u16* const wt = (u16*)(ws + 128);        // 64 cells
    u32 nsym, hdr;
    if (n == 0) return 0;
    rank.clear();
    u32 total = 0;
    auto put = [&](u32 i, u32 w) { wn[i >> 1] |= (u8)(w << ((i & 1) * 4)); };
    auto clear_nibbles = [&] { for (int i = 0; i < 32; i++) ((u32*)wn)[i] = 0; };
    if (s[0] >= 128) {
        nsym = (u32)s[0] - 127; hdr = (nsym + 1) / 2;
        if (hdr + 1 > n) return 0;
        clear_nibbles();
        for (u32 i = 0; i < nsym; i++) {
            u32 b = s[1 + i / 2], w = (i & 1) ? (b & 15) : (b >> 4);
            if (w > 12) return 0;
            put(i, w); rank.count(w); total += (1u << w) >> 1;
        }
    } else {
        hdr = s[0];
        if (hdr + 1 > n) return 0;
        // normalized counts of the weight alphabet, in the nibbles' bytes until the table is built.  A count above symbol 15
        // could never give a valid weight, so the read stops at symbol 15 and fails when the counts go on.
        short* const norm = (short*)wn; u32 max_sym = 15, log;
        u32 const used = zb_read_ncount(norm, max_sym, log, s + 1, hdr);
        if (used == 0 || log > 6) return 0;
        zb_fse_spread(wt, norm, max_sym, log);                       // norm: now each symbol's next-state counter
        u32 const size = 1u << log;
        for (u32 u = 0; u < size; u++) {
            u32 const sy = wt[u], x = (u32)(u16)norm[sy]; norm[sy] = (short)(x + 1);
            u32 const nb = log - (u32)zb_hibit(x);
            wt[u] = (u16)(sy | (nb << 4) | (((x << nb) - size) << 8));
        }
        clear_nibbles();
        ZbBitR<4> b;
        if (!b.init(s + 1 + used, hdr - used, ring)) return 0;
        u32 s1 = b.read(log), s2 = b.read(log); b.refill();
        if (b.left() < 0) return 0;
        nsym = 0;
        for (;;) {     // two interleaved states (FSE_decompress_usingDTable_generic, zstd/zstd.c:3840-3856)
            if (nsym + 2 > 255) return 0;
            { u32 c = wt[s1], w = c & 15; if (w > 12) return 0; put(nsym, w); rank.count(w); total += (1u << w) >> 1; nsym++;
              s1 = (c >> 8) + b.read((c >> 4) & 15); b.refill(); }
            if (b.left() < 0) { u32 w = wt[s2] & 15; if (w > 12) return 0; put(nsym, w); rank.count(w); total += (1u << w) >> 1; nsym++; break; }
            if (nsym + 2 > 255) return 0;
            { u32 c = wt[s2], w = c & 15; if (w > 12) return 0; put(nsym, w); rank.count(w); total += (1u << w) >> 1; nsym++;
              s2 = (c >> 8) + b.read((c >> 4) & 15); b.refill(); }
            if (b.left() < 0) { u32 w = wt[s1] & 15; if (w > 12) return 0; put(nsym, w); rank.count(w); total += (1u << w) >> 1; nsym++; break; }
        }
    }
    if (total == 0) return 0;
    u32 const log = (u32)zb_hibit(total) + 1;
    if (log > 12) return 0;
    u32 const rest = (1u << log) - total, hb = (u32)zb_hibit(rest);
    if ((1u << hb) != rest) return 0;
    put(nsym, hb + 1); rank.count(hb + 1); nsym++;
    if (rank[1] < 2 || (rank[1] & 1)) return 0;
    out_log = log; out_nsym = nsym;
    return hdr + 1;
}

// Split Huffman decode table.  The reference's table (HUF_readDTableX1_wksp, zstd/zstd.c:39651) has 2^log cells; at one
// frame per lane that is the shared-memory hog (2 KB at log 10: 13 of 32 lanes fit a warp's pool).  Cells are laid out by
// ascending weight, i.e. longest codes first, and every weight's range starts at a multiple of its cell run (Kraft
// equality), so above the codes longer than ZB_HUF_COARSE bits a cell depends only on the top ZB_HUF_COARSE bits of
// the index.  Only the first T cells (codes longer than 8 bits: the rare symbols) are kept at full resolution; the
// rest is one cell per 2^shift indices:   cell(v) = v < T ? fine[v] : coarse[v >> shift].
// A 4 KiB text frame needs ~600 bytes instead of 2 KB, so all 32 lanes of a warp decode in one pass.
#define ZB_HUF_COARSE 8u
struct ZbHufTab { const u16* cells; u32 log, shift, T, base; };       // base = index of coarse[0] in cells
__device__ __forceinline__ void zb_huf_shape(u32 log, ZbRank const& rank, u32& shift, u32& T, u32& base, u32& bytes)
{
    shift = log > ZB_HUF_COARSE ? log - ZB_HUF_COARSE : 0u;
    T = 0;
    #pragma unroll
    for (u32 wt = 1; wt <= 12 - ZB_HUF_COARSE; wt++) T += wt <= shift ? rank[wt] << (wt - 1) : 0u;
    base = (T + 3u) & ~3u;
    bytes = 2u * (base + (1u << (log - shift)));
}
__device__ __forceinline__ ZbHufTab zb_huf_full(const u16* cells, u32 log) { ZbHufTab t; t.cells = cells; t.log = log; t.shift = 0; t.T = 0; t.base = 0; return t; }
#define ZB_HCELL(t, v) ((t).cells[(v) < (t).T ? (v) : (t).base + ((v) >> (t).shift)])

// fill the decode cells (u16: symbol | nbBits << 8) from the nibble weights.  Every weight's cells start where the runs of
// the lighter weights end (a prefix over rank); a 16-bit cursor per weight, packed in registers, advances by one run per symbol.
__device__ static void zb_huf_fill(u16* cells, const u8* ws, u32 log, u32 nsym, ZbRank const& rank, u32 shift, u32 base)
{
    ZbPacked<6, 16> next; next.clear();
    {
        u32 p = 0;
        #pragma unroll
        for (u32 wt = 1; wt <= 12; wt++) { next.add(wt - 1, p); p += wt <= log ? (rank[wt] << (wt - 1)) : 0; }
    }
    for (u32 i = 0; i < nsym; i++) {
        u32 const wt = (ws[i >> 1] >> ((i & 1) * 4)) & 15; if (!wt) continue;
        u32 len = 1u << (wt - 1), p = next.get(wt - 1); next.add(wt - 1, len);
        if (wt > shift) { len >>= shift; p = base + (p >> shift); }       // coarse part: one cell per 2^shift indices
        u32 const cell = i | ((log + 1 - wt) << 8);
        if (len >= 4) { u64 const v = cell * 0x0001000100010001ull; u64* q = (u64*)(cells + p); for (u32 k = 0; k < len / 4; k++) q[k] = v; }
        else if (len == 2) *(u32*)(cells + p) = cell * 0x00010001u;
        else cells[p] = (u16)cell;
    }
}

#ifdef ZB_SIMT_EMULATION
// The CPU build's tests call the Huffman helpers with the weights' counts as u32 rank[0..12] (rank[0]: weight 0); the
// kernels pass ZbRank.  These adapters exist in that build only.
__device__ __forceinline__ ZbRank zb_rank_pack(const u32* rank) { ZbRank r; r.clear(); for (u32 wt = 1; wt <= 12; wt++) r.add(wt - 1, rank[wt]); return r; }
__device__ static u32 zb_huf_weights(u8* ws, const u8* s, u32 n, u32& out_log, u32& out_nsym, u32* rank, ZB_RING_ARG(ring))
{
    ZbRank r; u32 const used = zb_huf_weights(ws, s, n, out_log, out_nsym, r, ring);
    rank[0] = used ? out_nsym : 0;
    for (u32 w = 1; w <= 12; w++) { rank[w] = used ? r[w] : 0; rank[0] -= rank[w]; }
    return used;
}
__device__ __forceinline__ void zb_huf_shape(u32 log, const u32* rank, u32& shift, u32& T, u32& base, u32& bytes)
{
    zb_huf_shape(log, zb_rank_pack(rank), shift, T, base, bytes);
}
__device__ static void zb_huf_fill(u16* cells, const u8* ws, u32 log, u32 nsym, const u32* rank, u32 shift, u32 base)
{
    zb_huf_fill(cells, ws, log, nsym, zb_rank_pack(rank), shift, base);
}
#endif

// one Huffman stream -> n_out bytes at out (global scratch), 4 symbols per 32-bit store where aligned
__device__ static bool zb_huf_stream2(u8* out, u32 n_out, const u8* s, u32 n, ZbHufTab const t, u8* ring)
{
    ZbBitR<4> b;
    if (!b.init(s, n, ring)) return false;
    u32 const log = t.log;
    u32 i = 0;
    while (i < n_out && ((uintptr_t)(out + i) & 3)) { u32 v = b.peek(log); u32 c = ZB_HCELL(t, v); out[i++] = (u8)c; b.skip(c >> 8); b.refill(); }
    for (; i + 4 <= n_out; i += 4) {
        u32 v0 = b.peek(log); u32 c0 = ZB_HCELL(t, v0); b.skip(c0 >> 8);
        u32 v1 = b.peek(log); u32 c1 = ZB_HCELL(t, v1); b.skip(c1 >> 8); b.refill();
        u32 v2 = b.peek(log); u32 c2 = ZB_HCELL(t, v2); b.skip(c2 >> 8);
        u32 v3 = b.peek(log); u32 c3 = ZB_HCELL(t, v3); b.skip(c3 >> 8); b.refill();
        *(u32*)(out + i) = (c0 & 255) | ((c1 & 255) << 8) | ((c2 & 255) << 16) | (c3 << 24);
    }
    for (; i < n_out; i++) { u32 v = b.peek(log); u32 c = ZB_HCELL(t, v); out[i] = (u8)c; b.skip(c >> 8); b.refill(); }
    return b.left() == 0;
}

// The four literal streams of a block, interleaved in ONE lane: four independent bit readers advance side by
// side, so the dependent chain of one stream (table lookup -> bit count -> shift) fills the latency slots of the
// other three (what HUF_decompress4X1_usingDTable_internal_body does with its four BIT_DStream_t, zstd/zstd.c:39868-39964).
struct ZbHufLane { ZbBitR<4> b; u8* out; u32 left; };

__device__ __forceinline__ void zb_huf_one(ZbHufLane& h, ZbHufTab const& t)
{
    u32 const v = h.b.peek(t.log); u32 const c = ZB_HCELL(t, v); *h.out++ = (u8)c; h.b.skip(c >> 8); h.b.refill(); h.left--;
}
// four symbols of one stream -> one aligned 32-bit store
#define ZB_HUF4(h) do { \
        u32 const v0_ = h.b.peek(t.log); u32 const c0_ = ZB_HCELL(t, v0_); h.b.skip(c0_ >> 8); \
        u32 const v1_ = h.b.peek(t.log); u32 const c1_ = ZB_HCELL(t, v1_); h.b.skip(c1_ >> 8); h.b.refill(); \
        u32 const v2_ = h.b.peek(t.log); u32 const c2_ = ZB_HCELL(t, v2_); h.b.skip(c2_ >> 8); \
        u32 const v3_ = h.b.peek(t.log); u32 const c3_ = ZB_HCELL(t, v3_); h.b.skip(c3_ >> 8); h.b.refill(); \
        *(u32*)h.out = (c0_ & 255) | ((c1_ & 255) << 8) | ((c2_ & 255) << 16) | (c3_ << 24); h.out += 4; h.left -= 4; } while (0)

// `ring`: 256 bytes of the lane's shared memory, 64 per stream for its bit reader
__device__ static bool zb_huf_block(u8* dstl, u32 regen, const u8* p, u32 left, bool single, ZbHufTab const t, ZB_RING_ARG(ring))
{
    if (single) return zb_huf_stream2(dstl, regen, p, left, t, ring);
    if (left < 10) return false;
    u32 const l1 = zb_rd16(p), l2 = zb_rd16(p + 2), l3 = zb_rd16(p + 4), seg = (regen + 3) / 4;
    if (6 + l1 + l2 + l3 > left || seg * 3 > regen) return false;
    u32 const l4 = left - 6 - l1 - l2 - l3;
    ZbHufLane h0, h1, h2, h3;
    u8* const r1 = ring ? ring + 64 : nullptr; u8* const r2 = ring ? ring + 128 : nullptr; u8* const r3 = ring ? ring + 192 : nullptr;
    if (!h0.b.start(p + 6, l1, ring) || !h1.b.start(p + 6 + l1, l2, r1) || !h2.b.start(p + 6 + l1 + l2, l3, r2) || !h3.b.start(p + 6 + l1 + l2 + l3, l4, r3)) return false;
    if (!h0.b.finish() || !h1.b.finish() || !h2.b.finish() || !h3.b.finish()) return false;
    h0.out = dstl; h1.out = dstl + seg; h2.out = dstl + 2 * seg; h3.out = dstl + 3 * seg;
    h0.left = h1.left = h2.left = seg; h3.left = regen - 3 * seg;
    // bring every stream's output pointer to a 4-byte boundary
    while (h0.left && ((uintptr_t)h0.out & 3)) zb_huf_one(h0, t);
    while (h1.left && ((uintptr_t)h1.out & 3)) zb_huf_one(h1, t);
    while (h2.left && ((uintptr_t)h2.out & 3)) zb_huf_one(h2, t);
    while (h3.left && ((uintptr_t)h3.out & 3)) zb_huf_one(h3, t);
    // main loop: 4 symbols of each of the 4 streams per iteration
    while (h0.left >= 4 && h1.left >= 4 && h2.left >= 4 && h3.left >= 4) { ZB_HUF4(h0); ZB_HUF4(h1); ZB_HUF4(h2); ZB_HUF4(h3); }
    while (h0.left >= 4) ZB_HUF4(h0);
    while (h1.left >= 4) ZB_HUF4(h1);
    while (h2.left >= 4) ZB_HUF4(h2);
    while (h3.left >= 4) ZB_HUF4(h3);
    while (h0.left) zb_huf_one(h0, t);
    while (h1.left) zb_huf_one(h1, t);
    while (h2.left) zb_huf_one(h2, t);
    while (h3.left) zb_huf_one(h3, t);
    return h0.b.left() == 0 && h1.b.left() == 0 && h2.b.left() == 0 && h3.b.left() == 0;
}

// Resolve one sequence-table descriptor for this block.  For ZB_SRC_NCOUNT the normalized counts
// are parsed into `norm` (lane workspace) and the table log returned; bytes of smem needed -> need.
// returns consumed header bytes, or -1
__device__ static int zb_seq_desc(ZbTabSrc& d, u32 mode, u32 max_sym_kind, u32 max_log, const u8* ip, u32 avail,
                                  bool repeat_ok, short* norm, u32& log, u32& max_sym, u32& need)
{
    int used = 0;
    if (mode == 0) { d.kind = ZB_SRC_PREDEF; }
    else if (mode == 1) { if (avail == 0 || ip[0] > max_sym_kind) return -1; d.kind = ZB_SRC_RLE; d.sym = ip[0]; used = 1; }
    else if (mode == 2) { d.kind = ZB_SRC_NCOUNT; d.p = ip; d.n = avail; }
    else if (!repeat_ok || d.kind == ZB_SRC_NONE) return -1;
    need = 0; log = 0; max_sym = max_sym_kind;
    if (d.kind == ZB_SRC_NCOUNT) {
        u32 const u = zb_read_ncount(norm, max_sym, log, d.p, d.n);
        if (u == 0 || log > max_log) return -1;
        if (mode == 2) { used = (int)u; d.n = u; }
        need = 2u << log;                                   // 16-bit cells
    } else if (d.kind == ZB_SRC_RLE) need = 2;
    return used;
}

// i = 0 .. n-1 spread over the CTA's threads
template <class F> __device__ __forceinline__ void zb_cta_for(u32 n, F f)
{
#ifdef __CUDA_ARCH__
    for (u32 i = threadIdx.x; i < n; i += blockDim.x) f(i);
#else
    if (threadIdx.x == 0) for (u32 i = 0; i < n; i++) f(i);       // a CPU build may run thread 0 alone
#endif
}

// 32-bit cells of a table of 2^log -> ZB_CELL16 cells
__device__ __forceinline__ void zb_cta_cells16(u8* dst, const ZbFseCell* src, u32 log)
{
    zb_cta_for(1u << log, [&](u32 i) { u32 const c = src[i]; ((u16*)dst)[i] = ZB_CELL16(ZB_CELL_SYM(c), (ZB_CELL_NEXT(c) + (1u << log)) >> ZB_CELL_NB(c)); });
}

// Fill the CTA-wide head of the entropy kernels' shared memory (see ZB_ENT_HEAD_BYTES); returns the bytes of each warp's pool.
// The baseline LUTs carry the symbol's extra-bit count in bits 24-31.
template <int W>
__device__ __forceinline__ u32 zb_ent_head(u8* smem, ZbDictDev const& dict)
{
    u32* const lutLL = (u32*)smem; u32* const lutML = lutLL + 36;      // indexed by symbol code
    zb_cta_for(36, [&](u32 i) { lutLL[i] = c_LL_base[i] | ((u32)c_LL_bits[i] << 24); });
    zb_cta_for(53, [&](u32 i) { lutML[i] = c_ML_base[i] | ((u32)c_ML_bits[i] << 24); });
    zb_cta_cells16(smem + ZB_ENT_DEF_LL, g_defLL, 6);
    zb_cta_cells16(smem + ZB_ENT_DEF_OF, g_defOF, 5);
    zb_cta_cells16(smem + ZB_ENT_DEF_ML, g_defML, 6);
    u32 head = ZB_ENT_HEAD_BYTES;
    if (dict.has_entropy) {                                            // logs <= 9, 8, 9 (zb_digest_dict)
        zb_cta_cells16(smem + head, dict.ll, dict.ll_log); head += 2u << dict.ll_log;
        zb_cta_cells16(smem + head, dict.of, dict.of_log); head += 2u << dict.of_log;
        zb_cta_cells16(smem + head, dict.ml, dict.ml_log); head += 2u << dict.ml_log;
    }
    __syncthreads();
    return ((ZB_ENT_SMEM(W) - head) / W) & ~15u;
}

// per-phase cycle counters (lane 0 of every warp) exist only in tuning builds (-DZB_PHASE_TIMERS)
#ifdef ZB_PHASE_TIMERS
__device__ unsigned long long g_zb_ent_phase[8];
#define ZB_EMARK(k) do { if (lane == 0) { long long const t_ = clock64(); atomicAdd(&g_zb_ent_phase[k], (unsigned long long)(t_ - t_ph)); t_ph = t_; } } while (0)
#elif defined(ZB_DEBUG_BLOCKS)
#define ZB_EMARK(k) do { if (err && !(t_ph & 1)) { printf("[emark %d] lane %u err %u\n", k, lane, err); t_ph |= 1; } } while (0)
#else
#define ZB_EMARK(k) do { (void)t_ph; } while (0)
#endif

// -- D of one block in one lane: place the three FSE tables (built at q in the lane's pool claim, or the predefined or the
// dictionary's ones in the head), then run the 3-state sequence stream (restates ZSTD_decodeSequence, zstd/zstd.c:46862-46986)
// into sq[0, nseq).  Returns the error code; lit_used / produced / rep0..2 carry the block's totals and repcode history out.
// SYMREP: the history may be symbolic (zb_entropy_blocks: 0x80000000 | k << 29 | d stands for "entry repcode k, minus d").
//
// The bit window holds 32..64 bits after a refill, while a sequence takes ~16 on 4 KiB level-3 frames.  So the sequence refills
// once, after its cell loads, and reads its offset, ML + LL and state bits without refilling in between when they all fit in
// the window; otherwise it refills before each of the last two reads as well.  Either way every read sees the same bits as
// with a refill before each read, and left() and its checks are unchanged.
//
// Every lane of the warp calls this; the lanes with `go` decode a block, the others only join the warp's stores.  The records
// are not stored one per lane and sequence: a warp-wide store of 32 lanes' records touches 32 lines.  Each lane stages 8
// records in ws + 128 (the ring takes ws[0, 128) and nothing else of the workspace is live), and every 8 sequences the warp
// writes them out together: each 16-byte store instruction carries 4 lanes' runs of 8 consecutive records, 4 to 8 lines.
// Lanes whose block has ended or failed join those stores with nothing to write.  `ws_stride`: the distance between lanes'
// workspaces.
template <bool SYMREP>
__device__ __forceinline__ u32 zb_seq_block(bool go, const u8* smem, u8* q, u8* ws, u32 ws_stride, ZbDictDev const& dict,
                                            ZbTabSrc const& dLL, ZbTabSrc const& dOF, ZbTabSrc const& dML,
                                            u32 msLL, u32 msOF, u32 msML, u32 logLL, u32 logOF, u32 logML,
                                            const u8* ip, const u8* bend, u32 nseq, ZbSeq* sq, u32 n_lit, u64 room, u64 hist,
                                            u32& rep0, u32& rep1, u32& rep2, u32& lit_used, u32& produced, long long& t_ph)
{
    u32 const lane = threadIdx.x & 31;
    const u32* const lutLL = (const u32*)smem; const u32* const lutML = lutLL + 36;
    short* const normLL = (short*)ws; short* const normOF = normLL + 36; short* const normML = normOF + 32;
    u32 const dct_ll = ZB_ENT_HEAD_BYTES, dct_of = dct_ll + (2u << dict.ll_log), dct_ml = dct_of + (2u << dict.of_log);
    ZbTab tLL = {0, 0}, tOF = tLL, tML = tLL;
    auto setup = [&](const ZbTabSrc& d, short* norm, u32 ms, u32 lg, int kind, u32 dct, u32 dlog, u32 def, u32 deflog, ZbTab& t) {
        if (d.kind == ZB_SRC_NCOUNT) { zb_build_fse((u16*)q, norm, ms, lg, kind); t.off = (u32)(q - smem); t.log = lg; q += 2u << lg; }
        else if (d.kind == ZB_SRC_RLE) { *(u16*)q = ZB_CELL16(d.sym, 1u); t.off = (u32)(q - smem); t.log = 0; q += 2; }
        else if (d.kind == ZB_SRC_DICT) { t.off = dct; t.log = dlog; }
        else { t.off = def; t.log = deflog; }
    };
    u32 err = ZB_OK;
    ZbBitR<8> b;                        // ring: the lane workspace (the normalized counts are consumed)
    u32 sLL = 0, sOF = 0, sML = 0;
    if (go) {
        setup(dLL, normLL, msLL, logLL, K_LL, dct_ll, dict.ll_log, ZB_ENT_DEF_LL, 6, tLL);
        setup(dOF, normOF, msOF, logOF, K_OF, dct_of, dict.of_log, ZB_ENT_DEF_OF, 5, tOF);
        setup(dML, normML, msML, logML, K_ML, dct_ml, dict.ml_log, ZB_ENT_DEF_ML, 6, tML);
#ifdef ZB_PHASE_TIMERS
        ZB_EMARK(7);                                                  // the table builds of phase D
#endif
        if (!b.init(ip, (u32)(bend - ip), ws)) err = ZB_E_CORRUPTION;
        else { sLL = b.read(tLL.log); sOF = b.read(tOF.log); b.refill(); sML = b.read(tML.log); }
    }
    const u8* const TL = smem + tLL.off; const u8* const TO = smem + tOF.off; const u8* const TM = smem + tML.off;
    u32 const kL = 31 - tLL.log, kO = 31 - tOF.log, kM = 31 - tML.log;                 // nbBits = clz(x) - k
    u8* const stage = ws + 128;
    bool run = go && !err;
    u32 i = 0;                                                        // the next sequence
    for (u32 i0 = 0; __any_sync(0xFFFFFFFFu, run && i0 < nseq); i0 += 8) {
        bool const ran = run && i0 < nseq;                            // then sq[i0, i) are staged, in slots 0 .. i - i0 - 1
        if (ran) {
            while (i < nseq) {
                u32 const cl = *(const u16*)(TL + 2 * sLL), co = *(const u16*)(TO + 2 * sOF), cm = *(const u16*)(TM + 2 * sML);
                b.refill();
                u32 const llc = cl & 63, ofc = co & 63, xl = cl >> 6, xo = co >> 6, xm = cm >> 6;
                u32 const nl = __clz(xl) - kL, nm = __clz(xm) - kM, no = __clz(xo) - kO;
                u32 const eL = lutLL[llc], eM = lutML[cm & 63];            // baseline | extra bits << 24: off the state chain
                u32 const llb = eL >> 24, ab = (eM >> 24) + llb;                                 // ML then LL additional bits (<= 32)
                u32 const sb = i + 1 < nseq ? nl + nm + no : 0;                                  // the three state updates (<= 26)
                bool const slow = (int)(ofc + ab + sb) > b.avail;                                 // ofc: the offset's extra bits
                u32 const ob = b.read(ofc);
                u32 ll = eL & 0xFFFFFFu, ml = eM & 0xFFFFFFu, off;
                // (a branch-free select chain over {rep0, rep1, rep2, rep0 - 1, new} was measured 3-5 % slower than this branch)
                if (ofc > 1) {
                    off = (1u << ofc) - 3 + ob;
                    // SYMREP: bit 31 tags a symbolic history entry, so a concrete offset must stay below 2^31.  The launcher keeps
                    // frames whose window (plus the dictionary) reaches that far off the block path; here such an offset is corrupt.
                    if (SYMREP && (off & 0x80000000u)) { err = ZB_E_CORRUPTION; break; }
                    rep2 = rep1; rep1 = rep0; rep0 = off;
                } else {
                    u32 const ll0 = (llc == 0);
                    if (ofc == 0) {
                        if (ll0) { off = rep1; rep1 = rep0; rep0 = off; } else off = rep0;
                    } else {
                        u32 const idx = 1 + ll0 + ob;
                        u32 const r0m = SYMREP && (rep0 & 0x80000000u) ? rep0 + 1 : rep0 - 1;   // symbolic: one more off
                        u32 tmp = idx == 1 ? rep1 : (idx == 2 ? rep2 : r0m);
                        // rep0 - 1 == 0 is corrupt (zstd/zstd.c:46905).  SYMREP rejects it here: 0xFFFFFFFF would read as symbolic.
                        if (SYMREP && tmp == 0) { err = ZB_E_CORRUPTION; break; }
                        if (tmp == 0) tmp = 0xFFFFFFFFu;
                        if (idx != 1) rep2 = rep1;
                        rep1 = rep0; rep0 = off = tmp;
                    }
                }
                if (slow) b.refill();
                {
                    u32 const both = b.read(ab);
                    ml += both >> llb; ll += both & ((1u << llb) - 1);
                }
                if (slow) b.refill();
                {   // LL, ML, OF in one read
                    u32 const v = b.read(sb);
                    sLL = (xl << nl) - (1u << tLL.log) + (v >> (nm + no));
                    sML = (xm << nm) - (1u << tML.log) + ((v >> no) & ((1u << nm) - 1));
                    sOF = (xo << no) - (1u << tOF.log) + (v & ((1u << no) - 1));
                }
                *(ZbSeq*)(stage + 16 * (i & 7)) = make_uint4(lit_used, produced, ml, off);
                i++;
                // the checks of ZSTD_execSequence / ZSTD_execSequenceEnd (zstd/zstd.c:46540-46728)
                if ((u64)produced + ll + ml > room) { err = ZB_E_DSTSIZE_TOO_SMALL; break; }
                if (ll > n_lit - lit_used) { err = ZB_E_CORRUPTION; break; }
                lit_used += ll; produced += ll;
                if ((u64)off > hist + produced) { err = ZB_E_CORRUPTION; break; }
                produced += ml;
                if (!(i & 7)) break;
            }
            run = !err;
        }
        // the warp's stores: in step j, the 8 lanes of quarter k store record (lane & 7) of lane 4j + k's run.  A run's start
        // and length travel in one shuffle (ZbSeq is 16-byte aligned, so the pointer's low 4 bits are free for a length <= 8).
        __syncwarp();
        u64 const mine = (u64)(uintptr_t)(sq + i0) | (ran ? i - i0 : 0u);
        u8* const stage0 = stage - lane * ws_stride;
        u32 const r = lane & 7;
        #pragma unroll 1
        for (u32 j = 0; j < 8; j++) {
            u32 const o = 4 * j + (lane >> 3);
            u64 const p = __shfl_sync(0xFFFFFFFFu, mine, o);
            if (r < (u32)(p & 15)) ((ZbSeq*)(uintptr_t)(p & ~15ull))[r] = *(const ZbSeq*)(stage0 + o * ws_stride + 16 * r);
        }
        __syncwarp();
    }
    if (go && !err && b.left() != 0) err = ZB_E_CORRUPTION;
    return err;
}

template <int ZB_ENT_WARPS>
__global__ void __launch_bounds__(ZB_ENT_WARPS * 32)
zb_entropy_decode(const u8* __restrict__ src, const ZbSegment* __restrict__ segs, u32 n_frames,
                  const ZbFramePlace* __restrict__ place, const u64* __restrict__ dst_sizes,
                  ZbBlock* __restrict__ blocks, ZbSeq* __restrict__ seqs, u8* __restrict__ lits,
                  u32* __restrict__ work_counter, ZbDictDev dict, u32* status, u64* __restrict__ out_sizes,
                  u32* __restrict__ ck_expect, u32 take)
{
    ZB_DYN_SMEM(zb_smem);
    u32 const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 const pool_bytes = zb_ent_head<ZB_ENT_WARPS>(zb_smem, dict);
    u8* const pool = zb_smem + ZB_ENT_SMEM(ZB_ENT_WARPS) - (ZB_ENT_WARPS - warp) * pool_bytes;      // pools: behind the head
    u8* const ws = pool + lane * ZB_ENT_WS_STRIDE;                       // lane workspace
    u8* const tabs = pool + 32 * ZB_ENT_WS_STRIDE;                       // claimable table space
    u32 const TAB_BYTES = pool_bytes - 32 * ZB_ENT_WS_STRIDE;

    for (;;) {
        u32 base = 0;
        // `take` frames per warp and grab: 32 for small frames; fewer when frames (hence their tables) are large,
        // so that a warp holds only as many frames as its table pool serves in one pass and the batch spreads over
        // more warps and SMs
        if (lane == 0) base = atomicAdd(work_counter, take);
        base = __shfl_sync(0xFFFFFFFFu, base, 0);
        if (base >= n_frames) return;
        u32 const f = base + lane;
        bool done = lane >= take || !(f < n_frames) || status[f] != ZB_OK;

        // ---- per-frame lane state
        const u8* s = src; u64 n = 0; ZbHdr h; ZbFramePlace pl; u32 err = ZB_OK;
        u64 cap = 0, out_pos = 0, blk_i = 0, seq_i = 0, lit_i = 0, pos = 0; u32 block_max = 0;
        u32 rep0 = 1, rep1 = 4, rep2 = 8;
        ZbTabSrc dHuf = {ZB_SRC_NONE, 0, nullptr, 0}, dLL = dHuf, dOF = dHuf, dML = dHuf;
        bool fse_valid = false;
        if (!done) {
            s = src + segs[f].offset; n = segs[f].length;
            zb_skip_skippable(s, n);
            zb_parse_header(s, n, h);
            pl = place[f]; cap = pl.dst_cap; blk_i = pl.blk_off; seq_i = pl.seq_off; lit_i = pl.lit_off; pos = h.hdr_size;
            block_max = h.window < ZB_BLOCK_MAX ? (u32)h.window : ZB_BLOCK_MAX;
            if (dict.has_entropy) {
                dHuf.kind = dLL.kind = dOF.kind = dML.kind = ZB_SRC_DICT; fse_valid = true;
                rep0 = dict.rep[0]; rep1 = dict.rep[1]; rep2 = dict.rep[2];
            }
            if (h.dict_id && dict.dict_id && h.dict_id != dict.dict_id) { err = ZB_E_DICT_WRONG; done = true; }
        }
        u64 const hist_extra = dict.content_size;

        long long t_ph = clock64() & ~1ll;
        // ---- one block per lane per round
        while (__any_sync(0xFFFFFFFFu, !done)) {
            ZB_EMARK(0);
            ZbBlock B; B.kind = 0; B.regen = 0; B.n_seq = 0; B.n_lit = 0; B.lit_kind = 0; B.lit_byte = 0; B.src_pos = 0; B.seq_pos = seq_i; B.out_pos = out_pos;
            bool comp = false, last = false;
            u32 bsize = 0; const u8* bs = nullptr; const u8* bend = nullptr; const u8* ip = nullptr;
            ZbLitHdr L; L.type = 0; L.regen = 0; L.hdr = 0; L.csize = 0; L.single = 0;
            // -- A: block header
            if (!done) {
                do {
                    if (pos + 3 > n) { err = ZB_E_SRCSIZE_WRONG; break; }
                    u32 const bh = zb_rd24(s + pos); pos += 3;
                    last = bh & 1; u32 const type = (bh >> 1) & 3; bsize = bh >> 3; B.kind = type;
                    if (type == 3) { err = ZB_E_CORRUPTION; break; }
                    if (type == ZB_BLK_RLE) {
                        if (pos + 1 > n) { err = ZB_E_SRCSIZE_WRONG; break; }
                        if (bsize > block_max) { err = ZB_E_CORRUPTION; break; }
                        if (bsize > cap - out_pos) { err = ZB_E_DSTSIZE_TOO_SMALL; break; }
                        B.src_pos = (u64)(s + pos - src); B.regen = bsize; B.lit_byte = s[pos]; pos += 1;
                    } else if (type == ZB_BLK_RAW) {
                        if (pos + bsize > n) { err = ZB_E_SRCSIZE_WRONG; break; }
                        if (bsize > block_max) { err = ZB_E_CORRUPTION; break; }
                        if (bsize > cap - out_pos) { err = ZB_E_DSTSIZE_TOO_SMALL; break; }
                        B.src_pos = (u64)(s + pos - src); B.regen = bsize; pos += bsize;
                    } else {
                        if (pos + bsize > n || bsize > block_max) { err = ZB_E_SRCSIZE_WRONG; break; }
                        bs = s + pos; bend = bs + bsize;
                        err = zb_parse_lit_header(bs, bsize, L);
                        if (err) break;
                        if (L.regen > block_max) { err = ZB_E_CORRUPTION; break; }
                        B.n_lit = L.regen; comp = true;
                    }
                } while (0);
                if (err) { done = true; comp = false; }
            }
            ZB_EMARK(1);
            // -- B: literals
            bool wantH = false; u32 hlog = 0, hns = 0; ZbRank rank; const u8* hp = nullptr; u32 hleft = 0;
            if (comp) {
                do {
                    if (L.type == 0) {
                        if (L.hdr + L.regen > bsize) { err = ZB_E_CORRUPTION; break; }
                        B.lit_kind = ZB_LIT_RAW; B.src_pos = (u64)(bs + L.hdr - src); ip = bs + L.hdr + L.regen;
                    } else if (L.type == 1) {
                        if (L.hdr + 1 > bsize) { err = ZB_E_CORRUPTION; break; }
                        B.lit_kind = ZB_LIT_RLE; B.lit_byte = bs[L.hdr]; ip = bs + L.hdr + 1;
                    } else {
                        if (L.type == 3 && dHuf.kind == ZB_SRC_NONE) { err = ZB_E_DICT_CORRUPTED; break; }
                        if (!L.single && L.regen < 6) { err = ZB_E_LITERALS_HEADER_WRONG; break; }
                        if (L.csize + L.hdr > bsize || L.regen == 0) { err = ZB_E_CORRUPTION; break; }
                        hp = bs + L.hdr; hleft = L.csize;
                        if (L.type == 2) { dHuf.kind = ZB_SRC_NCOUNT; dHuf.p = hp; dHuf.n = hleft; }
                        if (dHuf.kind == ZB_SRC_NCOUNT) {
                            u32 const used = zb_huf_weights(ws, dHuf.p, dHuf.n, hlog, hns, rank, tabs + lane * 80);   // no table lives in the pool during B
                            if (used == 0 || (L.type == 2 && used >= hleft)) { err = ZB_E_CORRUPTION; break; }
                            if (L.type == 2) { hp += used; hleft -= used; dHuf.n = used; }
                            wantH = true;
                        }
                        B.lit_kind = ZB_LIT_SCRATCH; B.src_pos = lit_i; ip = bs + L.hdr + L.csize;
                    }
                } while (0);
                if (err) { done = true; comp = false; wantH = false; }
            }
            // dictionary Huffman table: read in place from the digest (shared by every lane, cache resident)
            if (comp && B.lit_kind == ZB_LIT_SCRATCH && dHuf.kind == ZB_SRC_DICT) {
                if (!zb_huf_block(lits + lit_i, L.regen, hp, hleft, L.single, zb_huf_full(dict.huf, dict.huf_log), ws)) { err = ZB_E_CORRUPTION; done = true; comp = false; }
            }
            ZB_EMARK(2);
            {   // claim pool space for the Huffman cells, decode; lanes that do not fit wait for the next pass
                bool pending = wantH;
                u32 hshift = 0, hT = 0, hbase = 0, hbytes = 0;
                if (wantH) zb_huf_shape(hlog, rank, hshift, hT, hbase, hbytes);
                while (__any_sync(0xFFFFFFFFu, pending)) {
                    u32 const need = pending ? hbytes : 0;
                    u32 const incl = zb_warp_incl_scan((need + 15) & ~15u, lane);
                    if (pending && incl <= TAB_BYTES) {
                        u16* cells = (u16*)(tabs + incl - ((need + 15) & ~15u));
                        zb_huf_fill(cells, ws, hlog, hns, rank, hshift, hbase);
                        ZB_EMARK(6);                                   // the Huffman table of phase B; its streams follow
                        ZbHufTab t; t.cells = cells; t.log = hlog; t.shift = hshift; t.T = hT; t.base = hbase;
                        if (!zb_huf_block(lits + lit_i, L.regen, hp, hleft, L.single, t, ws)) { err = ZB_E_CORRUPTION; done = true; comp = false; }
                        pending = false;
                    }
                    __syncwarp();
                }
            }
            ZB_EMARK(3);
            if (comp && B.lit_kind == ZB_LIT_SCRATCH) lit_i += (L.regen + 15) & ~15u;
            // -- C: sequences section header
            u32 nseq = 0, logLL = 0, logOF = 0, logML = 0, msLL = 0, msOF = 0, msML = 0, needS = 0;
            short* const normLL = (short*)ws; short* const normOF = normLL + 36; short* const normML = normOF + 32;
            if (comp) {
                do {
                    if (ip >= bend) { err = ZB_E_SRCSIZE_WRONG; break; }
                    nseq = *ip++;
                    if (nseq > 0x7F) {
                        if (nseq == 0xFF) { if (ip + 2 > bend) { err = ZB_E_SRCSIZE_WRONG; break; } nseq = zb_rd16(ip) + 0x7F00; ip += 2; }
                        else { if (ip >= bend) { err = ZB_E_SRCSIZE_WRONG; break; } nseq = ((nseq - 0x80) << 8) + *ip++; }
                    }
                    B.n_seq = nseq;
                    if (nseq == 0) { if (ip != bend) err = ZB_E_CORRUPTION; break; }
                    if (ip + 1 > bend) { err = ZB_E_SRCSIZE_WRONG; break; }
                    u32 const modes = *ip++;
                    if (modes & 3) { err = ZB_E_CORRUPTION; break; }
                    u32 nd; int r;
                    r = zb_seq_desc(dLL, modes >> 6, 35, 9, ip, (u32)(bend - ip), fse_valid, normLL, logLL, msLL, nd);
                    if (r < 0) { err = ZB_E_CORRUPTION; break; } ip += r; needS += nd;
                    r = zb_seq_desc(dOF, (modes >> 4) & 3, 31, 8, ip, (u32)(bend - ip), fse_valid, normOF, logOF, msOF, nd);
                    if (r < 0) { err = ZB_E_CORRUPTION; break; } ip += r; needS += nd;
                    r = zb_seq_desc(dML, (modes >> 2) & 3, 52, 9, ip, (u32)(bend - ip), fse_valid, normML, logML, msML, nd);
                    if (r < 0) { err = ZB_E_CORRUPTION; break; } ip += r; needS += nd;
                    fse_valid = true;
                } while (0);
                if (err) { done = true; comp = false; nseq = 0; }
            }
            ZB_EMARK(4);
            // -- D: build the three tables in the pool and run the sequence stream
            u32 lit_used = 0, produced = 0;
            {
                bool pending = comp && nseq > 0;
                while (__any_sync(0xFFFFFFFFu, pending)) {
                    u32 const need = pending ? ZB_ENT_SKEW(needS) : 0;
                    u32 const incl = zb_warp_incl_scan(need, lane);
                    bool const go = pending && incl <= TAB_BYTES;
                    u32 const e = zb_seq_block<false>(go, zb_smem, tabs + incl - need, ws, ZB_ENT_WS_STRIDE, dict, dLL, dOF, dML,
                                                      msLL, msOF, msML, logLL, logOF, logML, ip, bend, nseq, seqs + seq_i, L.regen,
                                                      cap - out_pos, out_pos + hist_extra, rep0, rep1, rep2, lit_used, produced, t_ph);
                    if (go) {
                        err = e;
                        if (err) { done = true; comp = false; }
                        pending = false;
                    }
                }
            }
            ZB_EMARK(5);
            // -- E: close the block
            if (!done) {
                if (comp) {
                    seqs[seq_i + nseq] = make_uint4(lit_used, produced, 0, 0);
                    seq_i += nseq + 1;
                    u32 const tail = L.regen - lit_used;
                    if ((u64)produced + tail > cap - out_pos) err = ZB_E_DSTSIZE_TOO_SMALL;
                    B.regen = produced + tail;
                    if (!err && B.regen > block_max) err = ZB_E_CORRUPTION;
                    pos += bsize;
                }
                if (!err) {
                    blocks[blk_i++] = B;
                    out_pos += B.regen;
                    if (last) {
                        if (h.content_size != ZB_CONTENT_UNKNOWN && out_pos != h.content_size) err = ZB_E_CORRUPTION;
                        else if (h.checksum && pos + 4 > n) err = ZB_E_CHECKSUM_WRONG;
                        else {
                            if (h.checksum) ck_expect[f] = zb_rd32(s + pos);      // compared with XXH64 of the output by zb_verify_checksums
                            if (dst_sizes && out_pos != cap) err = ZB_E_SIZE_MISMATCH;    // every frame, checksummed or not: c-ext/decompressor.c:1151-1162
                        }
                        done = true;
                    }
                }
                if (err) done = true;
            }
        }
        if (lane < take && f < n_frames && status[f] == ZB_OK) {
            if (err) { status[f] = err; out_sizes[f] = err == ZB_E_SIZE_MISMATCH ? out_pos : 0; } else out_sizes[f] = out_pos;     // (the mismatch message names the size)
        } else if (lane < take && f < n_frames) out_sizes[f] = 0;
    }
}

// ===========================================================================
// The same per-block work with a lane per BLOCK instead of a lane per frame: frames of many blocks (one huge frame at the
// limit: BASELINE config 5) are a single lane's serial chain above -- 4 ms per 128 KiB block.  Here every block of the call
// is an item of its own.  What a block inherits from its predecessors is made explicit: the tables' sources (zb_scan_blocks
// resolves "repeat" / "treeless" to the header that defined them), the repcode history (symbolic, resolved by
// zb_resolve_blocks) and the output position (prefix sum of the regenerated sizes, same kernel).
// ===========================================================================
template <int ZB_ENT_WARPS>
__global__ void __launch_bounds__(ZB_ENT_WARPS * 32)
zb_entropy_blocks(const u8* __restrict__ src, const ZbBlkDesc* __restrict__ bdesc, u32 n_blocks,
                  ZbBlock* __restrict__ blocks, ZbSeq* __restrict__ seqs, u8* __restrict__ lits,
                  u32* __restrict__ work_counter, ZbDictDev dict, u32* status, ZbBlkExit* __restrict__ bexit, u32 take)
{
    ZB_DYN_SMEM(zb_smem);
    u32 const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 const pool_bytes = zb_ent_head<ZB_ENT_WARPS>(zb_smem, dict);
    u8* const pool = zb_smem + ZB_ENT_SMEM(ZB_ENT_WARPS) - (ZB_ENT_WARPS - warp) * pool_bytes;      // pools: behind the head
    // a few lanes per warp (ZB_BLOCKS_TAKE): no lock-step bank conflicts to spread, so the workspaces are not skewed
    u8* const ws = pool + lane * ZB_ENT_WS_BYTES;                       // lane workspace
    u8* const tabs = pool + 32 * ZB_ENT_WS_BYTES;                       // claimable table space
    u32 const TAB_BYTES = pool_bytes - 32 * ZB_ENT_WS_BYTES;

    for (;;) {
        u32 base = 0;
        // `take` frames per warp and grab: 32 for small frames; fewer when frames (hence their tables) are large,
        // so that a warp holds only as many frames as its table pool serves in one pass and the batch spreads over
        // more warps and SMs
        if (lane == 0) base = atomicAdd(work_counter, take);
        base = __shfl_sync(0xFFFFFFFFu, base, 0);
        if (base >= n_blocks) return;
        u32 const bi = base + lane;                                   // this lane's BLOCK
        ZbBlkDesc D; D.frame = 0; D.flags = 0;
        if (lane < take && bi < n_blocks) D = bdesc[bi];
        bool done = lane >= take || !(bi < n_blocks) || (D.flags & ZB_BD_SKIP) || status[D.frame] != ZB_OK;

        // ---- per-frame lane state
        // The block is decoded on its own: tables as they stood on entry (zb_scan_blocks), output positions relative to the
        // block (the frame-relative start, the capacity and the offset-range checks follow in zb_resolve_blocks /
        // zb_patch_blocks), and -- unless it is the frame's first block -- a SYMBOLIC repcode history: 0x80000000 | k << 29 | d
        // stands for "entry repcode k, minus d".
        const u8* s = src; u64 n = 0; u32 err = ZB_OK;
        u64 const cap = ~0ull >> 1; u64 out_pos = 0, blk_i = bi, seq_i = 0, lit_i = 0, pos = 0; u32 block_max = 0;
        u32 rep0 = 1, rep1 = 4, rep2 = 8;
        ZbTabSrc dHuf = {ZB_SRC_NONE, 0, nullptr, 0}, dLL = dHuf, dOF = dHuf, dML = dHuf;
        bool fse_valid = false;
        if (!done) {
            s = src + D.hdr_off; n = D.span; seq_i = D.seq_off; lit_i = D.lit_off; block_max = D.block_max;
            dHuf = D.dHuf; dLL = D.dLL; dOF = D.dOF; dML = D.dML; fse_valid = (D.flags & ZB_BD_FSE_VALID) != 0;
            if (D.flags & ZB_BD_FIRST) { if (dict.has_entropy) { rep0 = dict.rep[0]; rep1 = dict.rep[1]; rep2 = dict.rep[2]; } }
            else { rep0 = 0x80000000u; rep1 = 0xA0000000u; rep2 = 0xC0000000u; }
        }
        u64 const hist_extra = 1ull << 40;                            // (no offset can fail the range check here)

        long long t_ph = clock64() & ~1ll;
        // ---- one block per lane per round
        while (__any_sync(0xFFFFFFFFu, !done)) {
            ZB_EMARK(0);
            ZbBlock B; B.kind = 0; B.regen = 0; B.n_seq = 0; B.n_lit = 0; B.lit_kind = 0; B.lit_byte = 0; B.src_pos = 0; B.seq_pos = seq_i; B.out_pos = out_pos;
            bool comp = false, last = false;
            u32 bsize = 0; const u8* bs = nullptr; const u8* bend = nullptr; const u8* ip = nullptr;
            ZbLitHdr L; L.type = 0; L.regen = 0; L.hdr = 0; L.csize = 0; L.single = 0;
            // -- A: block header
            if (!done) {
                do {
                    if (pos + 3 > n) { err = ZB_E_SRCSIZE_WRONG; break; }
                    u32 const bh = zb_rd24(s + pos); pos += 3;
                    last = bh & 1; u32 const type = (bh >> 1) & 3; bsize = bh >> 3; B.kind = type;
                    if (type == 3) { err = ZB_E_CORRUPTION; break; }
                    if (type == ZB_BLK_RLE) {
                        if (pos + 1 > n) { err = ZB_E_SRCSIZE_WRONG; break; }
                        if (bsize > block_max) { err = ZB_E_CORRUPTION; break; }
                        if (bsize > cap - out_pos) { err = ZB_E_DSTSIZE_TOO_SMALL; break; }
                        B.src_pos = (u64)(s + pos - src); B.regen = bsize; B.lit_byte = s[pos]; pos += 1;
                    } else if (type == ZB_BLK_RAW) {
                        if (pos + bsize > n) { err = ZB_E_SRCSIZE_WRONG; break; }
                        if (bsize > block_max) { err = ZB_E_CORRUPTION; break; }
                        if (bsize > cap - out_pos) { err = ZB_E_DSTSIZE_TOO_SMALL; break; }
                        B.src_pos = (u64)(s + pos - src); B.regen = bsize; pos += bsize;
                    } else {
                        if (pos + bsize > n || bsize > block_max) { err = ZB_E_SRCSIZE_WRONG; break; }
                        bs = s + pos; bend = bs + bsize;
                        err = zb_parse_lit_header(bs, bsize, L);
                        if (err) break;
                        if (L.regen > block_max) { err = ZB_E_CORRUPTION; break; }
                        B.n_lit = L.regen; comp = true;
                    }
                } while (0);
                if (err) { done = true; comp = false; }
            }
            ZB_EMARK(1);
            // -- B: literals
            bool wantH = false; u32 hlog = 0, hns = 0; ZbRank rank; const u8* hp = nullptr; u32 hleft = 0;
            if (comp) {
                do {
                    if (L.type == 0) {
                        if (L.hdr + L.regen > bsize) { err = ZB_E_CORRUPTION; break; }
                        B.lit_kind = ZB_LIT_RAW; B.src_pos = (u64)(bs + L.hdr - src); ip = bs + L.hdr + L.regen;
                    } else if (L.type == 1) {
                        if (L.hdr + 1 > bsize) { err = ZB_E_CORRUPTION; break; }
                        B.lit_kind = ZB_LIT_RLE; B.lit_byte = bs[L.hdr]; ip = bs + L.hdr + 1;
                    } else {
                        if (L.type == 3 && dHuf.kind == ZB_SRC_NONE) { err = ZB_E_DICT_CORRUPTED; break; }
                        if (!L.single && L.regen < 6) { err = ZB_E_LITERALS_HEADER_WRONG; break; }
                        if (L.csize + L.hdr > bsize || L.regen == 0) { err = ZB_E_CORRUPTION; break; }
                        hp = bs + L.hdr; hleft = L.csize;
                        if (L.type == 2) { dHuf.kind = ZB_SRC_NCOUNT; dHuf.p = hp; dHuf.n = hleft; }
                        if (dHuf.kind == ZB_SRC_NCOUNT) {
                            u32 const used = zb_huf_weights(ws, dHuf.p, dHuf.n, hlog, hns, rank, tabs + lane * 64);   // no table lives in the pool during B
                            if (used == 0 || (L.type == 2 && used >= hleft)) { err = ZB_E_CORRUPTION; break; }
                            if (L.type == 2) { hp += used; hleft -= used; dHuf.n = used; }
                            wantH = true;
                        }
                        B.lit_kind = ZB_LIT_SCRATCH; B.src_pos = lit_i; ip = bs + L.hdr + L.csize;
                    }
                } while (0);
                if (err) { done = true; comp = false; wantH = false; }
            }
            // dictionary Huffman table: read in place from the digest (shared by every lane, cache resident)
            if (comp && B.lit_kind == ZB_LIT_SCRATCH && dHuf.kind == ZB_SRC_DICT) {
                if (!zb_huf_block(lits + lit_i, L.regen, hp, hleft, L.single, zb_huf_full(dict.huf, dict.huf_log), ws)) { err = ZB_E_CORRUPTION; done = true; comp = false; }
            }
            ZB_EMARK(2);
            {   // claim pool space for the Huffman cells, decode; lanes that do not fit wait for the next pass
                bool pending = wantH;
                u32 hshift = 0, hT = 0, hbase = 0, hbytes = 0;
                if (wantH) zb_huf_shape(hlog, rank, hshift, hT, hbase, hbytes);
                while (__any_sync(0xFFFFFFFFu, pending)) {
                    u32 const need = pending ? hbytes : 0;
                    u32 const incl = zb_warp_incl_scan((need + 15) & ~15u, lane);
                    if (pending && incl <= TAB_BYTES) {
                        u16* cells = (u16*)(tabs + incl - ((need + 15) & ~15u));
                        zb_huf_fill(cells, ws, hlog, hns, rank, hshift, hbase);
                        ZB_EMARK(6);                                   // the Huffman table of phase B; its streams follow
                        ZbHufTab t; t.cells = cells; t.log = hlog; t.shift = hshift; t.T = hT; t.base = hbase;
                        if (!zb_huf_block(lits + lit_i, L.regen, hp, hleft, L.single, t, ws)) { err = ZB_E_CORRUPTION; done = true; comp = false; }
                        pending = false;
                    }
                    __syncwarp();
                }
            }
            ZB_EMARK(3);
            if (comp && B.lit_kind == ZB_LIT_SCRATCH) lit_i += (L.regen + 15) & ~15u;
            // -- C: sequences section header
            u32 nseq = 0, logLL = 0, logOF = 0, logML = 0, msLL = 0, msOF = 0, msML = 0, needS = 0;
            short* const normLL = (short*)ws; short* const normOF = normLL + 36; short* const normML = normOF + 32;
            if (comp) {
                do {
                    if (ip >= bend) { err = ZB_E_SRCSIZE_WRONG; break; }
                    nseq = *ip++;
                    if (nseq > 0x7F) {
                        if (nseq == 0xFF) { if (ip + 2 > bend) { err = ZB_E_SRCSIZE_WRONG; break; } nseq = zb_rd16(ip) + 0x7F00; ip += 2; }
                        else { if (ip >= bend) { err = ZB_E_SRCSIZE_WRONG; break; } nseq = ((nseq - 0x80) << 8) + *ip++; }
                    }
                    B.n_seq = nseq;
                    if (nseq == 0) { if (ip != bend) err = ZB_E_CORRUPTION; break; }
                    if (ip + 1 > bend) { err = ZB_E_SRCSIZE_WRONG; break; }
                    u32 const modes = *ip++;
                    if (modes & 3) { err = ZB_E_CORRUPTION; break; }
                    u32 nd; int r;
                    r = zb_seq_desc(dLL, modes >> 6, 35, 9, ip, (u32)(bend - ip), fse_valid, normLL, logLL, msLL, nd);
                    if (r < 0) { err = ZB_E_CORRUPTION; break; } ip += r; needS += nd;
                    r = zb_seq_desc(dOF, (modes >> 4) & 3, 31, 8, ip, (u32)(bend - ip), fse_valid, normOF, logOF, msOF, nd);
                    if (r < 0) { err = ZB_E_CORRUPTION; break; } ip += r; needS += nd;
                    r = zb_seq_desc(dML, (modes >> 2) & 3, 52, 9, ip, (u32)(bend - ip), fse_valid, normML, logML, msML, nd);
                    if (r < 0) { err = ZB_E_CORRUPTION; break; } ip += r; needS += nd;
                    fse_valid = true;
                } while (0);
                if (err) { done = true; comp = false; nseq = 0; }
            }
            ZB_EMARK(4);
            // -- D: build the three tables in the pool and run the sequence stream
            u32 lit_used = 0, produced = 0;
            {
                bool pending = comp && nseq > 0;
                while (__any_sync(0xFFFFFFFFu, pending)) {
                    u32 const need = pending ? ((needS + 15) & ~15u) : 0;
                    u32 const incl = zb_warp_incl_scan(need, lane);
                    bool const go = pending && incl <= TAB_BYTES;
                    u32 const e = zb_seq_block<true>(go, zb_smem, tabs + incl - need, ws, ZB_ENT_WS_BYTES, dict, dLL, dOF, dML,
                                                     msLL, msOF, msML, logLL, logOF, logML, ip, bend, nseq, seqs + seq_i, L.regen,
                                                     cap - out_pos, out_pos + hist_extra, rep0, rep1, rep2, lit_used, produced, t_ph);
                    if (go) {
                        err = e;
                        if (err) { done = true; comp = false; }
                        pending = false;
                    }
                }
            }
            ZB_EMARK(5);
            // -- E: close the block
            if (!done) {
                if (comp) {
                    seqs[seq_i + nseq] = make_uint4(lit_used, produced, 0, 0);
                    seq_i += nseq + 1;
                    u32 const tail = L.regen - lit_used;
                    if ((u64)produced + tail > cap - out_pos) err = ZB_E_DSTSIZE_TOO_SMALL;
                    B.regen = produced + tail;
                    if (!err && B.regen > block_max) err = ZB_E_CORRUPTION;
                    pos += bsize;
                }
                if (!err) blocks[blk_i] = B;
                done = true;                                          // one block per lane
            }
        }
        if (lane < take && bi < n_blocks && !(D.flags & ZB_BD_SKIP)) {
            ZbBlkExit X; X.rep[0] = rep0; X.rep[1] = rep1; X.rep[2] = rep2; X.err = err;
            bexit[bi] = X;
#ifdef ZB_DEBUG_BLOCKS
            if (err) printf("[entropy_blocks] block %u frame %u err %u flags %u span %u | huf k%u n%u | LL k%u n%u s%u | OF k%u n%u s%u | ML k%u n%u s%u | hdr %02x %02x %02x | LLp-src %lld\n", bi, D.frame, err, D.flags, D.span,
                            D.dHuf.kind, D.dHuf.n, D.dLL.kind, D.dLL.n, D.dLL.sym, D.dOF.kind, D.dOF.n, D.dOF.sym, D.dML.kind, D.dML.n, D.dML.sym,
                            src[D.hdr_off], src[D.hdr_off + 1], src[D.hdr_off + 2], D.dLL.p ? (long long)(D.dLL.p - src) : -1ll);
#endif
            if (err) atomicCAS(&status[D.frame], (u32)ZB_OK, err);
        }
    }
}
