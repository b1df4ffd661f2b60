// zb_common.cuh -- shared device-side definitions of the H100 zstd batch codec.
//
// Format constants are RFC 8878's (the reference holds them at zstd/zstd.c:15596-15662
// and :41266-41290); everything else here is this project's own design.
#pragma once
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

typedef uint8_t  u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

// ---- status codes: numeric values follow zstd_errors.h so host code can print
// ---- the reference's own error strings (c-ext/decompressor.c:1328-1371)
enum : u32 {
    ZB_OK = 0,
    ZB_E_GENERIC = 1,
    ZB_E_PREFIX_UNKNOWN = 10,
    ZB_E_FRAMEPARAM_UNSUPPORTED = 14,
    ZB_E_WINDOW_TOO_LARGE = 16,
    ZB_E_CORRUPTION = 20,
    ZB_E_CHECKSUM_WRONG = 22,
    ZB_E_LITERALS_HEADER_WRONG = 24,
    ZB_E_DICT_CORRUPTED = 30,
    ZB_E_DICT_WRONG = 32,
    ZB_E_TABLELOG_TOO_LARGE = 44,
    ZB_E_MAXSYMBOL_TOO_SMALL = 48,
    ZB_E_MEMORY = 64,
    ZB_E_DSTSIZE_TOO_SMALL = 70,
    ZB_E_SRCSIZE_WRONG = 72,
    // ours (python-zstandard worker errors, c-ext/decompressor.c:911-917)
    ZB_E_UNKNOWN_SIZE = 200,
    ZB_E_SIZE_MISMATCH = 201,
};

#define ZB_MAGIC       0xFD2FB528u
#define ZB_MAGIC_DICT  0xEC30A437u
#define ZB_MAGIC_SKIP  0x184D2A50u
#define ZB_BLOCK_MAX   (128u << 10)
#define ZB_CONTENT_UNKNOWN 0xFFFFFFFFFFFFFFFFull

struct ZbSegment { u64 offset, length; };       // == BufferSegment, c-ext/python-zstandard.h:307-313

// ---- kernel launches.  The launchers launch through ZB_LAUNCH, and the kernels name their dynamic shared memory with
// ZB_DYN_SMEM (zb_decode.cu, zb_encode.cu), so that the CPU build of these sources (ZB_SIMT_EMULATION, tests/simt.h) runs
// the very launches the device runs.  Pass a template kernel parenthesised: (k<a, b>).  On the device every launch with
// dynamic shared memory first raises the kernel's limit to it (per device: cheap, so set on every launch).
#ifdef ZB_SIMT_EMULATION
#define ZB_LAUNCH(kernel, grid, block, smem, stream, ...) simt::launch((grid), (block), [&] { kernel(__VA_ARGS__); })
#else
#define ZB_LAUNCH(kernel, grid, block, smem, stream, ...) do { \
        if (smem) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(smem)); \
        kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__); } while (0)
#endif

// Block_Maximum_Size = min(window, 128 KiB) (ZSTD_getBlockSize, zstd/zstd.c:27478): a window_log below 17 cuts blocks of
// 2^window_log bytes, and with them the reach of every match; 0 = the default window
static inline u32 zb_block_max(u32 window_log) { return window_log && window_log < 17 ? (1u << window_log) : ZB_BLOCK_MAX; }

// The block jobs of a compression call: every <= block_max slice of every segment (ZSTD_compress_frameChunk's block loop,
// zstd/zstd.c:27545), in segment order, so a job that is not the first of its frame comes right after the one in front of
// it.  Host code; the launcher and the CPU build of the kernels both cut their jobs here, each with its own structs of the
// same fields.  Returns the largest block.
template <class Seg, class JobVec, class InfoVec>
static inline u32 zb_cut_blocks(const Seg* segs, size_t n, u32 block_max, JobVec& jobs, InfoVec& info)
{
    u32 max_block = 0;
    for (size_t i = 0; i < n; i++) {
        u64 const len = segs[i].length; u64 pos = 0;
        info[i].first_job = jobs.size(); info[i].n_jobs = 0; info[i].pad = 0;
        while (pos < len) {
            u32 const sz = (u32)(len - pos < block_max ? len - pos : block_max);
            typename JobVec::value_type j;
            j.src_pos = segs[i].offset + pos; j.size = sz; j.seg = (u32)i; j.first = pos == 0; j.last = pos + sz == len;
            jobs.push_back(j); info[i].n_jobs++; pos += sz;
            if (sz > max_block) max_block = sz;
        }
    }
    return max_block;
}

// The output slot of one block job: a block of up to max_block bytes compresses to at most this many (raw block fallback,
// headers, the entropy coders' slack), rounded up to 16 bytes.
static inline u64 zb_slot_bytes(u32 max_block) { return ((u64)max_block + (max_block >> 7) + 64 + 15) & ~15ull; }

// The compression view of a dictionary: the last <= 32 KiB of its content act as history in front of every frame
// (zb200_ddict_create).  Fewer than 8 bytes are not used: D = 0.
struct ZbDictView { const u8* tail; u32 D; };
static inline ZbDictView zb_dict_view(const u8* content, u32 content_size)
{
    u32 const D = content_size < 32768u ? content_size : 32768u;
    ZbDictView v; v.tail = content + (content_size - D); v.D = D >= 8 ? D : 0;
    return v;
}

// Content-dictionary chains (zb200_compress_chain).  A chunk's index samples every ZE_CHAIN_STEP-th position with 8 bytes
// behind it and holds 2^log slots for the two keys of each, at a load of at most 1/2 and at least 16 slots.
#define ZE_CHAIN_STEP 4u                // backward extension finds the true match starts
static inline u64 zb_chain_positions(u64 len) { return len >= 8 ? (len - 8) / ZE_CHAIN_STEP + 1 : 0; }
static inline u32 zb_chain_log(u64 len)
{
    u64 const npos = zb_chain_positions(len);
    u32 L = 4; while ((1ull << L) < 4 * npos) L++;
    return L;
}
// The plan of one run of a chain: chunks[0] is the prefix of chunks[1] only, chunks 1..m-1 become frames, and chunks[1..m)
// are the frames' segments.  Fills each chunk's index descriptor except its device pointers (tab, prev_tab), the offsets of
// the chunks' indexes in the run's slot array (tab_off, m + 1 entries) and of their sampled positions (pos_off, m + 1), and
// the block jobs of the frames (ZB_BLOCK_MAX blocks, job.seg = the chunk's descriptor) with their layout info (m - 1 entries).
template <class Seg, class Desc, class JobVec, class InfoVec>
static inline void zb_chain_plan(const Seg* chunks, size_t m, Desc* cs, u64* tab_off, u64* pos_off, JobVec& jobs, InfoVec& info)
{
    tab_off[0] = pos_off[0] = 0;
    for (size_t i = 0; i < m; i++) {
        u64 const len = chunks[i].length;
        cs[i].start = chunks[i].offset; cs[i].len = (u32)len; cs[i].log = zb_chain_log(len);
        cs[i].prev_len = i ? cs[i - 1].len : 0; cs[i].prev_log = i ? cs[i - 1].log : 0;
        tab_off[i + 1] = tab_off[i] + (1ull << cs[i].log);
        pos_off[i + 1] = pos_off[i] + zb_chain_positions(len);
    }
    zb_cut_blocks(chunks + 1, m - 1, ZB_BLOCK_MAX, jobs, info);
    for (auto& j : jobs) j.seg++;
}

// The CTA count of the lane-per-block entropy launch (zb_entropy_blocks: 7 warps, ZB_BLOCKS_TAKE blocks per lane): one CTA
// per SM, fewer when the blocks do not fill them.
#define ZB_BLOCKS_TAKE 3u
static inline u32 zb_entropy_blocks_ctas(u64 n_blocks, u32 sm_count)
{
    u64 const need = (n_blocks + 7 * ZB_BLOCKS_TAKE - 1) / (7 * ZB_BLOCKS_TAKE);
    u32 const c = sm_count < need ? sm_count : (u32)need;
    return c ? c : 1;
}

// The output chunks of a batch decode (run_decompress, zb_api.cu): a call whose output is copied back to the host is cut
// into chunks of frames, and the copy of chunk k overlaps the kernels of chunk k + 1.  One chunk per `chunk_bytes` of
// output, at most 32 and never more than there are frames; the cuts are by frame count (cut k = n_frames * k / n_chunks),
// not by bytes, so every chunk holds at least one frame.  Host code; the launcher and the CPU build of the kernels both
// plan their chunks here.
#define ZB_OUT_CHUNK_BYTES (48ull << 20)
#define ZB_OUT_CHUNKS_MAX  32u
static inline u32 zb_chunk_count(u64 total_out, u32 n_frames, bool copy_back, u64 chunk_bytes)
{
    if (!copy_back || n_frames == 0) return 1;
    u64 const c = total_out / (chunk_bytes ? chunk_bytes : ZB_OUT_CHUNK_BYTES);
    u32 const k = (u32)(c < 1 ? 1 : (c > ZB_OUT_CHUNKS_MAX ? ZB_OUT_CHUNKS_MAX : c));
    return k > n_frames ? n_frames : k;
}
static inline u32 zb_chunk_cut(u32 n_frames, u32 k, u32 n_chunks) { return (u32)((u64)n_frames * k / n_chunks); }

// The lane-per-frame entropy launch of one chunk, from its output bytes, its frame count and the SM count: warps per CTA,
// frames per warp and CTAs of the persistent grid.  Large frames carry large decode tables (a 128 KiB block: ~4 KB Huffman
// + ~5 KB FSE cells per lane), so fewer of them share a warp (zb_entropy.cuh); small chunks spread their frames over all
// resident warps rather than filling few warps' lanes.
struct ZbChunkShape { u32 warps, take, ctas; };
static inline ZbChunkShape zb_chunk_shape(u64 out_bytes, u32 n_frames, u32 sm_count)
{
    u64 const avg_out = out_bytes / (n_frames ? n_frames : 1);
    ZbChunkShape s;
    s.warps = avg_out <= (8u << 10) ? 8u : 7u;
    s.take = avg_out <= (8u << 10) ? 32u : (avg_out <= (16u << 10) ? 16u : (avg_out <= (32u << 10) ? 8u : (avg_out <= (64u << 10) ? 4u : 3u)));
    { u32 const spread = (n_frames + sm_count * s.warps - 1) / (sm_count * s.warps); if (s.take > spread) s.take = spread ? spread : 1; }
    s.ctas = sm_count; { u32 const need = (n_frames + s.warps * s.take - 1) / (s.warps * s.take); if (s.ctas > need) s.ctas = need; if (s.ctas == 0) s.ctas = 1; }
    return s;
}

// result of the frame scan (one per frame)
struct ZbFrameInfo {
    u64 content_size;     // from the header, ZB_CONTENT_UNKNOWN if absent
    u64 n_seq_rec;        // sequence records needed: sum(nbSeq + 1) over compressed blocks
    u64 n_lit;            // literal bytes that must be regenerated into scratch (Huffman coded); 64-bit: an 8 GiB frame can
                          //   hold more than 4 GiB of them
    u32 n_blocks;
    u32 status;
    u32 dict_id;
    u32 flags;            // bit0: checksum present; bit1: window >= ZB_FAR_WINDOW
};

// The block-parallel entropy path tags symbolic repcodes with bit 31, so it needs every offset below 2^31.  A frame's offsets
// stay below its window plus the dictionary content; frames with a window of at least ZB_FAR_WINDOW, and dictionaries of
// ZB_FAR_DICT bytes or more, keep the batch on the lane-per-frame path.
#define ZB_FAR_WINDOW  ((1ull << 31) - (1ull << 27))
#define ZB_FAR_DICT    (1ull << 27)

// per-frame placement, produced by the offsets scan
struct ZbFramePlace {
    u64 dst_off;          // byte offset of the frame's output in dst
    u64 dst_cap;          // bytes the frame may write
    u64 blk_off;          // first ZbBlock of the frame
    u64 seq_off;          // first sequence record
    u64 lit_off;          // first literal scratch byte
};

enum : u32 { ZB_BLK_RAW = 0, ZB_BLK_RLE = 1, ZB_BLK_COMPRESSED = 2 };
enum : u32 { ZB_LIT_RAW = 0, ZB_LIT_RLE = 1, ZB_LIT_SCRATCH = 2 };

// one block of a frame, written by the entropy stage for the execute stage
struct ZbBlock {
    u64 out_pos;          // frame-relative start of the block's output
    u64 src_pos;          // raw/rle block: payload position in src.  compressed: literal position
                          //   (in src for ZB_LIT_RAW, in the literal scratch for ZB_LIT_SCRATCH)
    u64 seq_pos;          // first sequence record (absolute index)
    u32 kind;             // ZB_BLK_*
    u32 regen;            // regenerated size of the block
    u32 lit_kind;         // ZB_LIT_*  (ZB_LIT_RLE: byte value in lit_byte)
    u32 n_lit;
    u32 n_seq;
    u32 lit_byte;
};

// sequence record: .x = literal start (block-relative index into the block's literals)
//                  .y = output start of the sequence's literals (block-relative)
//                  .z = match length, .w = match offset (real distance, repcodes resolved)
// A sentinel record {.x = literals consumed, .y = output produced} ends every block.
typedef uint4 ZbSeq;

// FSE decode cell, 32 bits: the information of ZSTD_seqSymbol (zstd/zstd.c:41301-41306) minus the
// baseline, which is looked up from the symbol (off the state chain):
//   bits 0-9 nextState base, 10-13 nbBits, 14-18 nbAdditionalBits, 19-24 symbol code
typedef u32 ZbFseCell;
#define ZB_CELL(next, nb, add, sym) ((u32)(next) | ((u32)(nb) << 10) | ((u32)(add) << 14) | ((u32)(sym) << 19))
#define ZB_CELL_NEXT(c) ((c) & 1023u)
#define ZB_CELL_NB(c)   (((c) >> 10) & 15u)
#define ZB_CELL_ADD(c)  (((c) >> 14) & 31u)
#define ZB_CELL_SYM(c)  ((c) >> 19)
// The entropy kernels' sequence loop reads 16-bit cells instead, so that a lane's three tables take half the shared
// memory: symbol | x << 6, with x the state's occurrence count (< 2^(log + 1)).  nbBits = log - hibit(x), next state
// base = (x << nbBits) - 2^log, the extra-bit count comes from the symbol.  From a 32-bit cell: x = (next + 2^log) >> nb.
#define ZB_CELL16(sym, x) ((u16)((sym) | ((x) << 6)))

// digested dictionary, device resident (restates what ZSTD_loadDEntropy keeps, zstd/zstd.c:44673-44757)
struct ZbDictDev {
    const u8* content; u32 content_size; u32 dict_id;
    const u16* huf; u32 huf_log; u32 has_entropy;
    const ZbFseCell* ll; const ZbFseCell* of; const ZbFseCell* ml;
    u32 ll_log, of_log, ml_log;
    u32 rep[3];
};

// dictionary digest as the device kernel writes it
struct ZbDictDigest {
    u16 huf[4096]; ZbFseCell ll[512]; ZbFseCell ml[512]; ZbFseCell of[256];
    u32 huf_log, ll_log, of_log, ml_log; u32 rep[3]; u32 dict_id; u32 content_off; u32 status; u32 has_entropy; u32 pad;
    // encoder view of the same entropy tables (ZSTD_loadCEntropy, zstd/zstd.c:28015): normalized counts and code lengths
    short c_norm_ll[36], c_norm_of[32], c_norm_ml[54]; u32 c_max_ll, c_max_of, c_max_ml;
    u8 c_huf_nb[256]; u32 c_huf_max;
};

__device__ __forceinline__ u32 zb_rd16(const u8* p) { return (u32)p[0] | ((u32)p[1] << 8); }
__device__ __forceinline__ u32 zb_rd24(const u8* p) { return zb_rd16(p) | ((u32)p[2] << 16); }
__device__ __forceinline__ u32 zb_rd32(const u8* p) { return zb_rd16(p) | (zb_rd16(p + 2) << 16); }
__device__ __forceinline__ u64 zb_rd64(const u8* p) { return (u64)zb_rd32(p) | ((u64)zb_rd32(p + 4) << 32); }
__device__ __forceinline__ int zb_hibit(u32 v) { return 31 - __clz(v); }

// ---------------------------------------------------------------------------
// Asynchronous 16-byte global -> shared copies (cp.async.cg: cached in L2 only, never in L1).  The
// CPU build of these sources copies at once.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void zb_cp16(u8* sdst, const u8* gsrc)     // both 16-byte aligned
{
#ifdef __CUDA_ARCH__
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"((u32)__cvta_generic_to_shared(sdst)), "l"(gsrc) : "memory");
#else
    memcpy(sdst, gsrc, 16);
#endif
}
__device__ __forceinline__ void zb_cp_commit()
{
#ifdef __CUDA_ARCH__
    asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
template <int N> __device__ __forceinline__ void zb_cp_wait()         // all but the N most recent groups have landed
{
#ifdef __CUDA_ARCH__
    asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory");
#endif
}

// ---------------------------------------------------------------------------
// Backward bit reader over an arbitrary byte range, built on 32-bit words and 32-bit funnel shifts.
// (hi:lo) holds the next unread bits top-aligned; `avail` counts them; nx0, nx1 are the two words
// below the window.  left() is the number of unread stream bits; it goes negative when the stream is
// over-read (the reference's BIT_DStream_overflow, zstd/zstd.c:2517-2556).  Reads below the stream
// start return the neighbouring bytes (not zeros): harmless, because left() < 0 fails the block.
//
// The words come from a RING of D 16-byte chunks in the lane's shared memory (chunk k -- bytes
// [16k, 16k + 16) above the 16-byte aligned base -- in slot k mod D), which asynchronous copies keep
// filled ahead of the decode: a refill that moves into chunk k requests chunk k + 1 - D, whose first
// word is needed 4D - 7 refills later at the earliest (4D - 4 in steady state, less right after
// init): a refill moves at most one word into the window, however many bits were read since the
// last one.  Every refill commits one copy group and, before it reads the ring, waits for all but the
// 4D - 8 most recent groups of the thread; other readers' refills in between only add groups.  So a
// copy has 4(D - 1) refills of decode to land in -- in the sequence decoder, which refills once per
// sequence in the common case, that many sequences at least -- where a 4-byte load issued one word ahead
// could not hide its latency: lanes of a warp refill at different moments and the warp's
// load scoreboard made nearly every refill wait for the latest lane's load.  The cp.async groups
// are ordered, so the wait is for copies that are old.
//
// Memory: the copies read only the 16-byte aligned cover of [s, s + n), which never leaves a device
// allocation (those are 256-byte aligned).  The ring must stay untouched while the reader lives;
// the destructor waits for the copies still in flight.  The CPU build may pass no ring: the reader
// then uses storage of its own.
// ---------------------------------------------------------------------------
#ifdef __CUDA_ARCH__
#define ZB_RING_ARG(name) u8* name
#else
#define ZB_RING_ARG(name) u8* name = nullptr
#endif
template <int D>
struct ZbBitR {
    static_assert(D >= 2 && (D & (D - 1)) == 0, "ring depth: a power of two");
    const u8* c; u8* ring; int widx; u32 hi, lo; int avail; u32 nx0, nx1; int skew_bits; int lo_c; u32 n_;
#ifndef __CUDA_ARCH__
    alignas(16) u8 own[16 * D];
#endif

    __device__ __forceinline__ u32 word(int j) const { return *(const u32*)(ring + ((u32)j & (4u * D - 1)) * 4u); }
    __device__ __forceinline__ void fetch(int k) { zb_cp16(ring + ((u32)k & (D - 1)) * 16u, c + 16 * k); }
    __device__ __forceinline__ ~ZbBitR() { zb_cp_wait<0>(); }

    // start() requests the top D chunks; finish() waits for them and positions the reader at the end mark.
    // Several readers start() before the first finish() so that their first copies overlap.
    __device__ __forceinline__ bool start(const u8* s, u32 n, u8* ring_) {
        if (n == 0) return false;
#ifdef __CUDA_ARCH__
        ring = ring_;
#else
        ring = ring_ ? ring_ : own;
#endif
        c = (const u8*)((uintptr_t)s & ~(uintptr_t)15);
        int const skew = (int)(s - c);
        skew_bits = skew * 8; n_ = n;
        int const top = (skew + (int)n - 1) >> 4;                 // chunk of the last byte
        #pragma unroll
        for (int q = 0; q < D; q++) if (top - q >= 0) fetch(top - q);
        zb_cp_commit();
        lo_c = top - D + 1 > 0 ? top - D + 1 : 0;                 // lowest chunk requested
        return true;
    }
    __device__ __forceinline__ bool finish() {
        zb_cp_wait<0>();
        int const e = skew_bits / 8 + (int)n_ - 1;               // the last byte, relative to the aligned base
        u32 const last = ring[(u32)e & (16u * D - 1)];
        if (last == 0) return false;
        int const P = e * 8 + zb_hibit(last);                     // bits from the aligned base up to the end mark
        nx0 = nx1 = 0; lo = 0;
        if (P == 0) { hi = 0; avail = 0; widx = -1; return true; }
        int const wi = (P - 1) >> 5, k = P - wi * 32;              // k in 1..32 valid bits in the top word
        hi = word(wi) << (32 - k); avail = k; widx = wi - 1;
        if (widx >= 0) nx0 = word(widx);
        if (widx >= 1) nx1 = word(widx - 1);
        refill();
        return true;
    }
    __device__ __forceinline__ bool init(const u8* s, u32 n, u8* ring_) { return start(s, n, ring_) && finish(); }
    // branch-free: lanes of a warp refill at different moments, so the body is predicated, not branched
    __device__ __forceinline__ void refill() {
        zb_cp_wait<4 * D - 8>();
        bool const r = (avail <= 32) & (widx >= 0);                // lo is empty when r holds
        u32 const a = (u32)avail;
        u32 const add_hi = __funnelshift_rc(nx0, 0u, a);           // nx0 >> avail        (0 when avail == 32)
        u32 const new_lo = __funnelshift_lc(0u, nx0, 32u - a);     // nx0 << (32 - avail) (0 when avail == 0)
        hi |= r ? add_hi : 0u;
        lo = r ? new_lo : lo;
        avail += r ? 32 : 0;
        widx -= r ? 1 : 0;
        nx0 = r ? nx1 : nx0;
        if (r && widx >= 1) nx1 = word(widx - 1);
        int const t = ((widx - 1) >> 2) + 1 - D;                   // nx1's chunk + 1 - D: its slot has been read out
        if (t >= 0 && t < lo_c) { fetch(t); lo_c = t; }
        zb_cp_commit();
    }
    __device__ __forceinline__ u32 peek(u32 nb) const { return __funnelshift_rc(hi, 0u, 32u - nb); }   // nb in 0..32
    __device__ __forceinline__ void skip(u32 nb) {                                                      // nb in 0..32
        hi = __funnelshift_lc(lo, hi, nb); lo = __funnelshift_lc(0u, lo, nb); avail -= (int)nb;
    }
    __device__ __forceinline__ u32 read(u32 nb) { u32 const v = peek(nb); skip(nb); return v; }
    __device__ __forceinline__ int left() const { return avail + 32 * (widx + 1) - skew_bits; }
};
