// zb_decode.cu -- batch zstd decompression for sm_90a (H100).
//
// Replaces the per-segment ZSTD_decompressStream call of the reference batch path
// (c-ext/decompressor.c:1150 -> zstd/zstd.c:45307 -> ZSTD_decompressFrame :44174).
//
// Design (see DESIGN.md): the work of a frame is split by the KIND of parallelism it has.
//   K1 zb_scan_frames     one LANE per frame : header + block-chain walk -> sizes for placement
//   K2 zb_place_frames    one CTA             : exclusive scans -> per-frame offsets
//   K3 zb_entropy_decode  one LANE per frame : the bit-serial chains (Huffman literal streams,
//                          FSE table builds, the 3-state FSE sequence stream, repcode history).
//                          32 independent frames advance in lock-step per warp, so every issue
//                          slot does 32 frames' worth of serial work.
//   K4 zb_execute         one WARP per frame : the LZ copy-execute, lane per sequence with a
//                          frontier test for match dependencies, coalesced copies for long runs.
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

#ifdef ZB_DEBUG_BLOCKS
#include <cstdio>
#endif

// ---------------------------------------------------------------------------
// format constants (RFC 8878 3.1.1.3.2.1; reference zstd/zstd.c:15615-15659, :41266-41290)
// ---------------------------------------------------------------------------
__constant__ u8 c_LL_bits[36] = {0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,1,1,1,1,2,2,3,3,4,6,7,8,9,10,11,12,13,14,15,16};
__constant__ u8 c_ML_bits[53] = {0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,
                                 1,1,1,1,2,2,3,3,4,4,5,7,8,9,10,11,12,13,14,15,16};
__constant__ u32 c_LL_base[36] = {0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,16,18,20,22,24,28,32,40,48,64,
                                  0x80,0x100,0x200,0x400,0x800,0x1000,0x2000,0x4000,0x8000,0x10000};
__constant__ u32 c_ML_base[53] = {3,4,5,6,7,8,9,10,11,12,13,14,15,16,17,18,19,20,21,22,23,24,25,26,27,28,29,30,31,32,33,34,
                                  35,37,39,41,43,47,51,59,67,83,99,0x83,0x103,0x203,0x403,0x803,0x1003,0x2003,0x4003,0x8003,0x10003};
__constant__ short c_LL_defnorm[36] = {4,3,2,2,2,2,2,2,2,2,2,2,2,1,1,1,2,2,2,2,2,2,2,2,2,3,2,1,1,1,1,1,-1,-1,-1,-1};
__constant__ short c_ML_defnorm[53] = {1,4,3,2,2,2,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,
                                       1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1,-1,-1};
__constant__ short c_OF_defnorm[29] = {1,1,1,1,1,1,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1};

enum { K_LL = 0, K_OF = 1, K_ML = 2 };

// default tables, built once per context by zb_build_default_tables
__device__ ZbFseCell g_defLL[64];
__device__ ZbFseCell g_defOF[32];
__device__ ZbFseCell g_defML[64];

// ---------------------------------------------------------------------------
// frame header (restates ZSTD_getFrameHeader_advanced, zstd/zstd.c:43668-43778)
// ---------------------------------------------------------------------------
struct ZbHdr { u64 content_size; u64 window; u32 dict_id; u32 hdr_size; u32 checksum; u32 status; };

__device__ static void zb_parse_header(const u8* s, u64 n, ZbHdr& h)
{
    h.status = ZB_OK; h.content_size = ZB_CONTENT_UNKNOWN; h.window = 0; h.dict_id = 0; h.checksum = 0; h.hdr_size = 0;
    if (n < 5) {
        // too short for a header: still report a wrong magic as such (:43680-43697)
        bool zstd_ok = true, skip_ok = true;
        const u8 zm[4] = {0x28, 0xB5, 0x2F, 0xFD}, sm[4] = {0x50, 0x2A, 0x4D, 0x18};
        for (u32 k = 0; k < n && k < 4; k++) {
            if (s[k] != zm[k]) zstd_ok = false;
            if (k == 0 ? ((s[0] & 0xF0) != sm[0]) : (s[k] != sm[k])) skip_ok = false;
        }
        h.status = (n && !zstd_ok && !skip_ok) ? ZB_E_PREFIX_UNKNOWN : ZB_E_SRCSIZE_WRONG;
        return;
    }
    u32 magic = zb_rd32(s);
    if (magic != ZB_MAGIC) { h.status = ZB_E_PREFIX_UNKNOWN; return; }
    u32 fhd = s[4];
    u32 single = (fhd >> 5) & 1, did = fhd & 3, fcs = fhd >> 6;
    u32 need = 5 + (single ? 0 : 1) + (did == 3 ? 4 : did) + (fcs == 0 ? (single ? 1 : 0) : (1u << fcs));
    if (n < need) { h.status = ZB_E_SRCSIZE_WRONG; return; }
    h.hdr_size = need;
    if (fhd & 8) { h.status = ZB_E_FRAMEPARAM_UNSUPPORTED; return; }
    h.checksum = (fhd >> 2) & 1;
    u32 pos = 5;
    if (!single) {
        u32 wl = s[pos++], wlog = (wl >> 3) + 10;
        if (wlog > 31) { h.status = ZB_E_WINDOW_TOO_LARGE; return; }
        h.window = 1ull << wlog; h.window += (h.window >> 3) * (wl & 7);
    }
    if (did == 1) { h.dict_id = s[pos]; pos += 1; }
    else if (did == 2) { h.dict_id = zb_rd16(s + pos); pos += 2; }
    else if (did == 3) { h.dict_id = zb_rd32(s + pos); pos += 4; }
    if (fcs == 0) { if (single) h.content_size = s[pos]; }
    else if (fcs == 1) h.content_size = zb_rd16(s + pos) + 256;
    else if (fcs == 2) h.content_size = zb_rd32(s + pos);
    else h.content_size = zb_rd64(s + pos);
    if (single) h.window = h.content_size;
}

// skip leading skippable frames (ZSTD_decompressMultiFrame, zstd/zstd.c:44318-44330)
__device__ static bool zb_skip_skippable(const u8*& s, u64& n)
{
    while (n >= 8 && (zb_rd32(s) & 0xFFFFFFF0u) == ZB_MAGIC_SKIP) {
        u64 sz = (u64)zb_rd32(s + 4) + 8;
        if (sz > n) return false;
        s += sz; n -= sz;
    }
    return true;
}

// literal-section header.  returns false on a malformed header.
struct ZbLitHdr { u32 type, hdr, regen, csize, single; };
__device__ static u32 zb_parse_lit_header(const u8* s, u32 n, ZbLitHdr& L)
{
    if (n < 2) return ZB_E_CORRUPTION;                     // MIN_CBLOCK_SIZE
    L.type = s[0] & 3; u32 sf = (s[0] >> 2) & 3; L.single = 0; L.csize = 0;
    if (L.type < 2) {
        if (sf == 1) { L.hdr = 2; L.regen = zb_rd16(s) >> 4; }
        else if (sf == 3) { if (n < 3) return ZB_E_CORRUPTION; L.hdr = 3; L.regen = zb_rd24(s) >> 4; }
        else { L.hdr = 1; L.regen = s[0] >> 3; }
        return ZB_OK;
    }
    if (n < 5) return ZB_E_CORRUPTION;
    u32 lhc = zb_rd32(s);
    if (sf < 2) { L.single = (sf == 0); L.hdr = 3; L.regen = (lhc >> 4) & 0x3FF; L.csize = (lhc >> 14) & 0x3FF; }
    else if (sf == 2) { L.hdr = 4; L.regen = (lhc >> 4) & 0x3FFF; L.csize = lhc >> 18; }
    else { L.hdr = 5; L.regen = (lhc >> 4) & 0x3FFFF; L.csize = (lhc >> 22) + ((u32)s[4] << 10); }
    return ZB_OK;
}

// ===========================================================================
// K1: frame scan -- one lane per frame
// ===========================================================================
// Frames above ZB_SCAN_BIG compressed bytes are not walked by a single lane (every block costs it a chain of dependent global
// loads: ~7 us): they go onto big_list (big_list[0] = count) and a WARP walks each of them (zb_scan_frames_big below).
#ifndef ZB_SCAN_BIG
#define ZB_SCAN_BIG (512u << 10)
#endif

// the part of a compressed block the scan needs: literal scratch bytes and sequence records it will produce
__device__ static u32 zb_scan_block_counts(const u8* bs, u32 bsize, u64& n_lit, u64& n_seq_rec)
{
    ZbLitHdr L; u32 e = zb_parse_lit_header(bs, bsize, L);
    if (e) return e;
    u32 lsec = L.type == 0 ? L.hdr + L.regen : (L.type == 1 ? L.hdr + 1 : L.hdr + L.csize);
    if (L.regen > ZB_BLOCK_MAX || lsec > bsize) return ZB_E_CORRUPTION;
    if (L.type >= 2) n_lit += (L.regen + 15) & ~15u;             // 16-byte aligned scratch slices
    if (lsec >= bsize) return ZB_E_SRCSIZE_WRONG;
    const u8* q = bs + lsec; u32 left = bsize - lsec;
    u32 nseq = q[0];
    if (nseq > 0x7F) {
        if (nseq == 0xFF) { if (left < 3) return ZB_E_SRCSIZE_WRONG; nseq = zb_rd16(q + 1) + 0x7F00; }
        else { if (left < 2) return ZB_E_SRCSIZE_WRONG; nseq = ((nseq - 0x80) << 8) + q[1]; }
    }
    n_seq_rec += nseq + 1;
    return ZB_OK;
}

// ZbFrameInfo.flags of a parsed header (both frame scans write it)
__device__ __forceinline__ u32 zb_info_flags(ZbHdr const& h) { return h.checksum | (h.window >= ZB_FAR_WINDOW ? 2u : 0u); }

// K1 for one big frame per warp: lane 0 walks the block-header chain 32 blocks ahead (one dependent load per block), then
// every lane parses the sections of its block.
__global__ void __launch_bounds__(128)
zb_scan_frames_big(const u8* __restrict__ src, const ZbSegment* __restrict__ segs, const u32* __restrict__ big_list,
                   ZbFrameInfo* __restrict__ info)
{
    __shared__ u64 sh_pos[4][32]; __shared__ u32 sh_bh[4][32];
    u32 const lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    u32 const n_big = big_list[0];
    for (u32 w = blockIdx.x * 4 + wib; w < n_big; w += gridDim.x * 4) {
        u32 const f = big_list[1 + w];
        const u8* s = src + segs[f].offset; u64 n = segs[f].length;
        zb_skip_skippable(s, n);
        ZbHdr h; zb_parse_header(s, n, h);
        ZbFrameInfo fi; fi.content_size = h.content_size; fi.dict_id = h.dict_id; fi.flags = zb_info_flags(h); fi.status = ZB_OK;
        u64 pos = h.hdr_size, n_lit = 0, n_seq_rec = 0, n_blocks = 0;
        u32 err = ZB_OK; bool last = false;
        while (!last && !err) {
            u32 cnt = 0, cerr = ZB_OK;
            if (lane == 0) {
                while (cnt < 32) {
                    if (pos + 3 > n) { cerr = ZB_E_SRCSIZE_WRONG; break; }
                    u32 const bh = zb_rd24(s + pos); u32 const type = (bh >> 1) & 3; u32 bsize = bh >> 3;
                    if (type == 3) { cerr = ZB_E_CORRUPTION; break; }
                    if (type == 1) bsize = 1;
                    if (pos + 3 + bsize > n) { cerr = ZB_E_SRCSIZE_WRONG; break; }
                    sh_pos[wib][cnt] = pos + 3; sh_bh[wib][cnt] = bh; cnt++;
                    pos += 3 + bsize;
                    if (bh & 1) { last = true; break; }
                }
            }
            __syncwarp();
            cnt = __shfl_sync(0xFFFFFFFFu, cnt, 0); cerr = __shfl_sync(0xFFFFFFFFu, cerr, 0);
            last = __shfl_sync(0xFFFFFFFFu, (int)last, 0) != 0;
            u32 e = ZB_OK;
            if (lane < cnt) {
                u32 const bh = sh_bh[wib][lane];
                if (((bh >> 1) & 3) == 2) e = zb_scan_block_counts(s + sh_pos[wib][lane], bh >> 3, n_lit, n_seq_rec);
            }
            u32 const bad = __ballot_sync(0xFFFFFFFFu, e != ZB_OK);
            if (bad) err = __shfl_sync(0xFFFFFFFFu, e, __ffs((int)bad) - 1);
            else err = cerr;
            n_blocks += cnt;
            __syncwarp();
        }
        #pragma unroll
        for (int d = 16; d > 0; d >>= 1) { n_lit += __shfl_xor_sync(0xFFFFFFFFu, n_lit, d); n_seq_rec += __shfl_xor_sync(0xFFFFFFFFu, n_seq_rec, d); }
        if (!err && n_blocks > 0xFFFFFFFFull) err = ZB_E_MEMORY;
        fi.status = err; fi.n_lit = n_lit; fi.n_seq_rec = n_seq_rec; fi.n_blocks = (u32)n_blocks;
        if (lane == 0) info[f] = fi;
    }
}

__global__ void zb_scan_frames(const u8* __restrict__ src, const ZbSegment* __restrict__ segs, u32 n_frames,
                               ZbFrameInfo* __restrict__ info, u64 window_limit, u32* __restrict__ big_list)
{
    u32 f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    const u8* s = src + segs[f].offset; u64 n = segs[f].length;
    u64 n_lit = 0, n_seq_rec = 0, n_blocks = 0;
    ZbFrameInfo fi; fi.content_size = ZB_CONTENT_UNKNOWN; fi.n_blocks = 0; fi.n_seq_rec = 0; fi.n_lit = 0;
    fi.status = ZB_OK; fi.dict_id = 0; fi.flags = 0;
    if (!zb_skip_skippable(s, n)) { fi.status = ZB_E_SRCSIZE_WRONG; info[f] = fi; return; }
    ZbHdr h; zb_parse_header(s, n, h);
    if (h.status == ZB_OK && n < 9) h.status = ZB_E_SRCSIZE_WRONG;       // zstd/zstd.c:44188
    // the window limit binds where the reference's streaming decoder cannot take its single-pass shortcut, i.e. for frames
    // whose header has no content size (zstd/zstd.c:45406-45453, ZSTD_d_windowLogMax / ZSTD_DCtx_setMaxWindowSize :45025)
    if (h.status == ZB_OK && h.content_size == ZB_CONTENT_UNKNOWN && h.window > window_limit) h.status = ZB_E_WINDOW_TOO_LARGE;
    if (h.status != ZB_OK) { fi.status = h.status; info[f] = fi; return; }
    fi.content_size = h.content_size; fi.dict_id = h.dict_id; fi.flags = zb_info_flags(h);
    if (big_list && n > ZB_SCAN_BIG) { big_list[1 + atomicAdd(big_list, 1u)] = f; return; }      // a warp's work: zb_scan_frames_big
    u64 pos = h.hdr_size;
    for (;;) {
        if (pos + 3 > n) { fi.status = ZB_E_SRCSIZE_WRONG; break; }
        u32 bh = zb_rd24(s + pos); pos += 3;
        u32 type = (bh >> 1) & 3, bsize = bh >> 3;
        n_blocks++;
        if (type == 3) { fi.status = ZB_E_CORRUPTION; break; }
        if (type == 1) bsize = 1;
        if (pos + bsize > n) { fi.status = ZB_E_SRCSIZE_WRONG; break; }
        if (type == 2) {
            u32 const e = zb_scan_block_counts(s + pos, bsize, n_lit, n_seq_rec);
            if (e) { fi.status = e; break; }
        }
        pos += bsize;
        if (bh & 1) break;
    }
    if (fi.status == ZB_OK && n_blocks > 0xFFFFFFFFull) fi.status = ZB_E_MEMORY;
    fi.n_lit = n_lit; fi.n_seq_rec = n_seq_rec; fi.n_blocks = (u32)n_blocks;
    info[f] = fi;
}

// ===========================================================================
// K2: placement -- exclusive scans of the per-frame sizes (dst bytes, blocks, sequence records,
// literal scratch).  Two launches: zb_place_reduce sums each CTA's 1024 frames, zb_place_scan lets
// every CTA add up the partials before it and scan its own frames.
// totals[0..3] = the four grand totals
// ===========================================================================
#define ZB_PLACE_CTA 1024

__device__ __forceinline__ void zb_place_values(const ZbFrameInfo& fi, const u64* dst_sizes, u32 f, u64 v[4], u64& cap, u32& st)
{
    st = fi.status; cap = 0;
    if (dst_sizes) cap = dst_sizes[f];
    else if (fi.content_size != ZB_CONTENT_UNKNOWN) cap = fi.content_size;
    else st = ZB_E_UNKNOWN_SIZE;                 // ZSTD_getFrameContentSize UNKNOWN/ERROR, c-ext/decompressor.c:981-1014
    v[0] = cap;                                  // outputs are packed tightly, like the reference's
    v[1] = v[2] = v[3] = 0;
    if (st == ZB_OK) { v[1] = fi.n_blocks; v[2] = fi.n_seq_rec; v[3] = fi.n_lit; }
}

__global__ void __launch_bounds__(ZB_PLACE_CTA)
zb_place_reduce(const ZbFrameInfo* __restrict__ info, const u64* __restrict__ dst_sizes, u32 n_frames, u64* __restrict__ partial)
{
    __shared__ u64 s_part[4][32];
    u32 const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    u32 const f = blockIdx.x * ZB_PLACE_CTA + tid;
    u64 v[4] = {0, 0, 0, 0};
    if (f < n_frames) { u64 cap; u32 st; zb_place_values(info[f], dst_sizes, f, v, cap, st); }
    #pragma unroll
    for (int k = 0; k < 4; k++) {
        u64 x = v[k];
        #pragma unroll
        for (int d = 16; d > 0; d >>= 1) x += __shfl_xor_sync(0xFFFFFFFFu, x, d);
        if (lane == 0) s_part[k][warp] = x;
    }
    __syncthreads();
    if (warp == 0) {
        #pragma unroll
        for (int k = 0; k < 4; k++) {
            u64 x = s_part[k][lane];
            #pragma unroll
            for (int d = 16; d > 0; d >>= 1) x += __shfl_xor_sync(0xFFFFFFFFu, x, d);
            if (lane == 0) partial[blockIdx.x * 4 + k] = x;
        }
    }
}

__global__ void __launch_bounds__(ZB_PLACE_CTA)
zb_place_scan(const ZbFrameInfo* __restrict__ info, const u64* __restrict__ dst_sizes, u32 n_frames,
              const u64* __restrict__ partial, ZbFramePlace* __restrict__ place, u64* __restrict__ totals,
              u32* __restrict__ status)
{
    __shared__ u64 s_part[4][32];
    __shared__ u64 s_base[4];
    u32 const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // base of this CTA = sum of the partials of all CTAs before it
    {
        u64 acc[4] = {0, 0, 0, 0};
        for (u32 c = tid; c < blockIdx.x; c += ZB_PLACE_CTA) { for (int k = 0; k < 4; k++) acc[k] += partial[c * 4 + k]; }
        #pragma unroll
        for (int k = 0; k < 4; k++) {
            u64 x = acc[k];
            #pragma unroll
            for (int d = 16; d > 0; d >>= 1) x += __shfl_xor_sync(0xFFFFFFFFu, x, d);
            if (lane == 0) s_part[k][warp] = x;
        }
        __syncthreads();
        if (warp == 0) {
            #pragma unroll
            for (int k = 0; k < 4; k++) {
                u64 x = s_part[k][lane];
                #pragma unroll
                for (int d = 16; d > 0; d >>= 1) x += __shfl_xor_sync(0xFFFFFFFFu, x, d);
                if (lane == 0) s_base[k] = x;
            }
        }
        __syncthreads();
    }
    u32 const f = blockIdx.x * ZB_PLACE_CTA + tid;
    u64 v[4] = {0, 0, 0, 0}; u64 cap = 0; u32 st = ZB_OK;
    if (f < n_frames) { ZbFrameInfo const fi = info[f]; zb_place_values(fi, dst_sizes, f, v, cap, st); status[f] = st; if ((fi.flags & 1) && st == ZB_OK) totals[4] = 1; if ((fi.flags & 2) && st == ZB_OK) totals[5] = 1; }
    u64 incl[4];
    #pragma unroll
    for (int k = 0; k < 4; k++) {
        u64 x = v[k];
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { u64 y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= (u32)d) x += y; }
        incl[k] = x;
        if (lane == 31) s_part[k][warp] = x;
    }
    __syncthreads();
    if (warp == 0) {
        #pragma unroll
        for (int k = 0; k < 4; k++) {
            u64 x = s_part[k][lane];
            #pragma unroll
            for (int d = 1; d < 32; d <<= 1) { u64 y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= (u32)d) x += y; }
            s_part[k][lane] = x;
        }
    }
    __syncthreads();
    u64 off[4];
    #pragma unroll
    for (int k = 0; k < 4; k++) off[k] = s_base[k] + (warp ? s_part[k][warp - 1] : 0) + incl[k] - v[k];
    if (f < n_frames) {
        ZbFramePlace p; p.dst_off = off[0]; p.dst_cap = cap; p.blk_off = off[1]; p.seq_off = off[2]; p.lit_off = off[3];
        place[f] = p;
    }
    if (f == n_frames - 1) {                      // grand totals + the sentinel that bounds the last frame's slices
        ZbFramePlace p; p.dst_off = off[0] + v[0]; p.dst_cap = 0; p.blk_off = off[1] + v[1]; p.seq_off = off[2] + v[2]; p.lit_off = off[3] + v[3];
        place[n_frames] = p;
        totals[0] = p.dst_off; totals[1] = p.blk_off; totals[2] = p.seq_off; totals[3] = p.lit_off;
    }
}

// ===========================================================================
// K3: entropy decode -- one lane per frame
// ===========================================================================

// forward (LSB-first) bit reader for the small table headers: a 64-bit window refilled 4 bytes at
// a time, so a header costs a handful of memory round trips instead of one per field
struct ZbFwdR {
    const u8* s; u32 n; u32 next_byte; u64 win; u32 have; u32 bp;
    __device__ __forceinline__ void init(const u8* s_, u32 n_) { s = s_; n = n_; next_byte = 0; win = 0; have = 0; bp = 0; fill(); fill(); }
    __device__ __forceinline__ void fill() {
        if (have <= 32) {
            u32 v = 0;
            #pragma unroll
            for (u32 k = 0; k < 4; k++) if (next_byte + k < n) v |= (u32)s[next_byte + k] << (8 * k);
            win |= (u64)v << have; have += 32; next_byte += 4;
        }
    }
    __device__ __forceinline__ u32 peek(u32 nb) const { return (u32)win & ((1u << nb) - 1); }
    __device__ __forceinline__ void skip(u32 nb) { win >>= nb; have -= nb; bp += nb; fill(); }
};

// normalized-count header (restates FSE_readNCount_body, zstd/zstd.c:3256-3413).
// returns bytes consumed, 0 on error
__device__ static u32 zb_read_ncount(short* norm, u32& max_sym, u32& table_log, const u8* s, u32 n)
{
    u32 const max_sv1 = max_sym + 1;
    if (n == 0) return 0;
    for (u32 i = 0; i < max_sv1; i++) norm[i] = 0;
    ZbFwdR r; r.init(s, n);
    u32 sym = 0; int prev0 = 0;
    int nbits = (int)r.peek(4) + 5; r.skip(4);
    if (nbits > 15) return 0;
    table_log = (u32)nbits;
    int remaining = (1 << nbits) + 1, threshold = 1 << nbits; nbits++;
    for (;;) {
        if (prev0) {
            for (;;) {
                u32 rp = r.peek(2); r.skip(2); sym += rp;
                if (rp != 3) break;
                if (r.bp > 8 * n + 64) return 0;
            }
            if (sym >= max_sv1) break;
        }
        int const mx = (2 * threshold - 1) - remaining;
        int count; int low = (int)r.peek((u32)(nbits - 1));
        if (low < mx) { count = low; r.skip((u32)(nbits - 1)); }
        else { count = (int)r.peek((u32)nbits); if (count >= threshold) count -= mx; r.skip((u32)nbits); }
        count--;
        remaining -= count < 0 ? -count : count;
        norm[sym++] = (short)count;
        prev0 = !count;
        if (remaining < threshold) {
            if (remaining <= 1) break;
            nbits = zb_hibit((u32)remaining) + 1; threshold = 1 << (nbits - 1);
        }
        if (sym >= max_sv1) break;
    }
    if (remaining != 1 || sym > max_sv1 || r.bp > 8 * n) return 0;
    max_sym = sym - 1;
    return (r.bp + 7) >> 3;
}

// additional-bit count of a symbol code (LL_bits / ML_bits / OF_bits, zstd/zstd.c:15615-15659, :41279)
__device__ __forceinline__ u32 zb_code_add_bits(u32 sym, int kind)
{
    return kind == K_LL ? c_LL_bits[sym] : (kind == K_ML ? c_ML_bits[sym] : sym);
}

// Symbol spread of a tANS decode table (ZSTD_buildFSETable_body, zstd/zstd.c:46118-46233): t[u] = the symbol of cell u.
// `norm` (max_sym + 1 shorts) becomes each symbol's first next-state counter: its count, or 1 for a -1 ("less than one")
// symbol, which takes one cell at the top.  The placement steps past those top cells; without -1 symbols it steps once per
// cell.  (A copy of the placement loop for that case, without the walk, made the lane-per-block entropy kernel 3 % slower
// on 128 KiB blocks and saved nothing measurable, so there is one loop.)
template <typename Cell>
__device__ __forceinline__ void zb_fse_spread(Cell* t, short* norm, u32 max_sym, u32 log)
{
    u32 const size = 1u << log, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
    u32 high = size - 1;
    for (u32 s = 0; s <= max_sym; s++) if (norm[s] == -1) { t[high--] = (Cell)s; norm[s] = 0x4001; }
    u32 pos = 0;
    for (u32 s = 0; s <= max_sym; s++) {
        int const c = norm[s];
        if (c & 0x4000) { norm[s] = 1; continue; }
        for (int i = 0; i < c; i++) { t[pos] = (Cell)s; do pos = (pos + step) & mask; while (pos > high); }
    }
}

// tANS decode table (restates ZSTD_buildFSETable_body, zstd/zstd.c:46118-46233), serial: the spread, then every cell's
// state from its symbol's counter in index order.  `norm` (max_sym + 1 shorts) is consumed: it becomes those counters.
// Cells: 32-bit ZbFseCell, or the entropy kernels' 16-bit ZB_CELL16.
template <typename Cell = ZbFseCell>
__device__ static void zb_build_fse(Cell* t, short* norm, u32 max_sym, u32 log, int kind)
{
    zb_fse_spread(t, norm, max_sym, log);
    u32 const size = 1u << log;
    for (u32 u = 0; u < size; u++) {
        u32 const s = t[u], x = (u32)(u16)norm[s]; norm[s] = (short)(x + 1);
        u32 const nb = log - (u32)zb_hibit(x);
        if constexpr (sizeof(Cell) == 4) t[u] = ZB_CELL((x << nb) - size, nb, zb_code_add_bits(s, kind), s);
        else t[u] = ZB_CELL16(s, x);
    }
}

__global__ void zb_build_default_tables()
{
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        short norm[64];
        for (int i = 0; i < 36; i++) norm[i] = c_LL_defnorm[i];
        zb_build_fse(g_defLL, norm, 35, 6, K_LL);
        for (int i = 0; i < 29; i++) norm[i] = c_OF_defnorm[i];
        zb_build_fse(g_defOF, norm, 28, 5, K_OF);
        for (int i = 0; i < 53; i++) norm[i] = c_ML_defnorm[i];
        zb_build_fse(g_defML, norm, 52, 6, K_ML);
    }
}

struct ZbTab { u32 off; u32 log; };         // off: byte offset of the cells in the entropy kernels' shared memory

#include "zb_entropy.cuh"

// one sequence table's source after this block's mode: the rules of zb_seq_desc, without building anything
__device__ static u32 zb_scan_seq_table(ZbTabSrc& d, u32 mode, u32 kmax, u32 lmax, const u8*& ip, const u8* bend, bool fse_valid)
{
    if (mode == 0) d.kind = ZB_SRC_PREDEF;
    else if (mode == 1) { if (ip >= bend || ip[0] > kmax) return ZB_E_CORRUPTION; d.kind = ZB_SRC_RLE; d.sym = ip[0]; ip++; }
    else if (mode == 2) {
        short nn[64]; u32 lg = 0, ms = kmax;
        u32 const u = zb_read_ncount(nn, ms, lg, ip, (u32)(bend - ip));
        if (u == 0 || lg > lmax) return ZB_E_CORRUPTION;
        d.kind = ZB_SRC_NCOUNT; d.p = ip; d.n = u; ip += u;
    } else if (!fse_valid || d.kind == ZB_SRC_NONE) return ZB_E_CORRUPTION;
    return ZB_OK;
}

// ===========================================================================
// Block-parallel path, K1b: zb_scan_blocks -- one thread per frame walks the block chain once more and writes, for every
// block, what zb_entropy_blocks needs on entry: where the block sits, where its records go, and where the Huffman tree and
// the three FSE tables valid ON ENTRY were defined (restates the bookkeeping of ZSTD_decodeLiteralsBlock's HUFptr /
// litEntropy, zstd/zstd.c:45840-45870, and ZSTD_decodeSeqHeaders' LLTptr / OFTptr / MLTptr + fseEntropy, :46328-46400).
// Header parsing only; a frame whose headers do not parse is failed here.
// ===========================================================================
#define ZB_SRC_INHERIT 0xFFFFFFFFu            // (zb_scan_blocks_big: "this block does not redefine the table")

__device__ __forceinline__ ZbTabSrc zb_shfl_tab(ZbTabSrc const& t, int j)
{
    ZbTabSrc r;
    r.kind = __shfl_sync(0xFFFFFFFFu, t.kind, j); r.sym = __shfl_sync(0xFFFFFFFFu, t.sym, j); r.n = __shfl_sync(0xFFFFFFFFu, t.n, j);
    r.p = (const u8*)__shfl_sync(0xFFFFFFFFu, (unsigned long long)t.p, j);
    return r;
}

// K1b for one big frame per warp (the frames zb_scan_frames left on big_list): lane 0 walks the block-header chain 32 blocks
// ahead, every lane parses the sections of its block into "what this block redefines", then the 32 blocks' entry states are
// chained through the warp with shuffles.  Same records, same errors as the one-lane walk below.
__global__ void __launch_bounds__(128)
zb_scan_blocks_big(const u8* __restrict__ src, const ZbSegment* __restrict__ segs, const u32* __restrict__ big_list,
                   const ZbFramePlace* __restrict__ place, ZbDictDev dict, u32* __restrict__ status,
                   ZbBlkDesc* __restrict__ bdesc, u64* __restrict__ frame_end)
{
    __shared__ u64 sh_pos[4][32]; __shared__ u32 sh_bh[4][32];
    u32 const lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    u32 const n_big = big_list[0];
    for (u32 w = blockIdx.x * 4 + wib; w < n_big; w += gridDim.x * 4) {
        u32 const f = big_list[1 + w];
        u64 const b0 = place[f].blk_off, b1 = place[f + 1].blk_off;
        if (status[f] != ZB_OK) { for (u64 b = b0 + lane; b < b1; b += 32) { bdesc[b].flags = ZB_BD_SKIP; bdesc[b].frame = f; } continue; }
        const u8* s = src + segs[f].offset; u64 n = segs[f].length;
        zb_skip_skippable(s, n);
        ZbHdr h; zb_parse_header(s, n, h);
        u32 err = ZB_OK;
        if (h.dict_id && dict.dict_id && h.dict_id != dict.dict_id) err = ZB_E_DICT_WRONG;
        u32 const block_max = h.window < ZB_BLOCK_MAX ? (u32)h.window : ZB_BLOCK_MAX;
        ZbTabSrc dHuf = {ZB_SRC_NONE, 0, nullptr, 0}, dLL = dHuf, dOF = dHuf, dML = dHuf;       // the state after the blocks so far (warp-uniform)
        bool fse_valid = false;
        if (dict.has_entropy) { dHuf.kind = dLL.kind = dOF.kind = dML.kind = ZB_SRC_DICT; fse_valid = true; }
        u64 pos = h.hdr_size, seq_i = place[f].seq_off, lit_i = place[f].lit_off, b = b0;
        bool last = false;
        while (b < b1 && !err && !last) {
            u32 cnt = 0, cerr = ZB_OK;
            if (lane == 0) {
                u32 const want = b1 - b < 32 ? (u32)(b1 - b) : 32u;
                while (cnt < want) {
                    if (pos + 3 > n) { cerr = ZB_E_SRCSIZE_WRONG; break; }
                    u32 const bh = zb_rd24(s + pos); u32 const type = (bh >> 1) & 3; u32 bsize = bh >> 3;
                    if (type == 3) { cerr = ZB_E_CORRUPTION; break; }
                    if (type == 1) bsize = 1;
                    if (pos + 3 + bsize > n) { cerr = ZB_E_SRCSIZE_WRONG; break; }
                    sh_pos[wib][cnt] = pos; sh_bh[wib][cnt] = bh; cnt++;
                    pos += 3 + bsize;
                    if (bh & 1) { last = true; break; }
                }
            }
            __syncwarp();
            cnt = __shfl_sync(0xFFFFFFFFu, cnt, 0); cerr = __shfl_sync(0xFFFFFFFFu, cerr, 0);
            last = __shfl_sync(0xFFFFFFFFu, (int)last, 0) != 0;
            pos = __shfl_sync(0xFFFFFFFFu, pos, 0);
            // ---- my block: what it redefines
            u32 e = ZB_OK, lit_add = 0, seq_add = 0, rep_mask = 0, bsize = 0; bool new_huf = false, has_seq = false;
            u64 my_pos = 0;
            ZbTabSrc tHuf = {ZB_SRC_INHERIT, 0, nullptr, 0}, tLL = tHuf, tOF = tHuf, tML = tHuf;
            if (lane < cnt) {
                u32 const bh = sh_bh[wib][lane]; u32 const type = (bh >> 1) & 3;
                my_pos = sh_pos[wib][lane]; bsize = type == 1 ? 1u : bh >> 3;
                if (type == 2) do {
                    const u8* const bs = s + my_pos + 3;
                    ZbLitHdr L; e = zb_parse_lit_header(bs, bsize, L);
                    if (e) break;
                    u32 const lsec = L.type == 0 ? L.hdr + L.regen : (L.type == 1 ? L.hdr + 1 : L.hdr + L.csize);
                    if (L.regen > ZB_BLOCK_MAX || lsec >= bsize) { e = ZB_E_CORRUPTION; break; }
                    if (L.type == 2) { new_huf = true; tHuf.kind = ZB_SRC_NCOUNT; tHuf.p = bs + L.hdr; tHuf.n = L.csize; }
                    if (L.type >= 2) lit_add = (L.regen + 15) & ~15u;
                    const u8* ip = bs + lsec; const u8* const bend = bs + bsize;
                    u32 nseq = *ip++;
                    if (nseq > 0x7F) {
                        if (nseq == 0xFF) { if (ip + 2 > bend) { e = ZB_E_SRCSIZE_WRONG; break; } nseq = zb_rd16(ip) + 0x7F00; ip += 2; }
                        else { if (ip >= bend) { e = ZB_E_SRCSIZE_WRONG; break; } nseq = ((nseq - 0x80) << 8) + *ip++; }
                    }
                    seq_add = nseq + 1;
                    if (nseq) {
                        if (ip + 1 > bend) { e = ZB_E_SRCSIZE_WRONG; break; }
                        u32 const modes = *ip++;
                        if ((modes >> 6) == 3) rep_mask |= 1; if (((modes >> 4) & 3) == 3) rep_mask |= 2; if (((modes >> 2) & 3) == 3) rep_mask |= 4;
                        e = zb_scan_seq_table(tLL, modes >> 6, 35, 9, ip, bend, true);
                        if (!e) e = zb_scan_seq_table(tOF, (modes >> 4) & 3, 31, 8, ip, bend, true);
                        if (!e) e = zb_scan_seq_table(tML, (modes >> 2) & 3, 52, 9, ip, bend, true);
                        if (e) break;
                        has_seq = true;
                    }
                } while (0);
            }
            // ---- where my block's records go: exclusive sums over the lanes before me
            u32 sx = seq_add, lx = lit_add;
            #pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                u32 const ys = __shfl_up_sync(0xFFFFFFFFu, sx, d), yl = __shfl_up_sync(0xFFFFFFFFu, lx, d);
                if (lane >= (u32)d) { sx += ys; lx += yl; }
            }
            u64 const my_seq = seq_i + (sx - seq_add), my_lit = lit_i + (lx - lit_add);
            seq_i += __shfl_sync(0xFFFFFFFFu, sx, 31); lit_i += __shfl_sync(0xFFFFFFFFu, lx, 31);
            // ---- the state on entry of every block: chained through the lanes
            ZbTabSrc eHuf = dHuf, eLL = dLL, eOF = dOF, eML = dML; bool e_valid = fse_valid;
            for (u32 j = 0; j < cnt; j++) {
                if (lane == j) {
                    eHuf = dHuf; eLL = dLL; eOF = dOF; eML = dML; e_valid = fse_valid;
                    if (!e && rep_mask && (!fse_valid || ((rep_mask & 1) && dLL.kind == ZB_SRC_NONE) || ((rep_mask & 2) && dOF.kind == ZB_SRC_NONE)
                                           || ((rep_mask & 4) && dML.kind == ZB_SRC_NONE))) e = ZB_E_CORRUPTION;
                }
                ZbTabSrc const jH = zb_shfl_tab(tHuf, (int)j), jL = zb_shfl_tab(tLL, (int)j), jO = zb_shfl_tab(tOF, (int)j), jM = zb_shfl_tab(tML, (int)j);
                bool const jseq = __shfl_sync(0xFFFFFFFFu, (int)has_seq, (int)j) != 0;
                if (jH.kind != ZB_SRC_INHERIT) dHuf = jH;
                if (jL.kind != ZB_SRC_INHERIT) dLL = jL;
                if (jO.kind != ZB_SRC_INHERIT) dOF = jO;
                if (jM.kind != ZB_SRC_INHERIT) dML = jM;
                fse_valid = fse_valid || jseq;
            }
            (void)new_huf;
            u32 const bad = __ballot_sync(0xFFFFFFFFu, lane < cnt && e != ZB_OK);
            u32 nvalid = cnt;
            if (bad) { nvalid = (u32)__ffs((int)bad) - 1; err = __shfl_sync(0xFFFFFFFFu, e, (int)nvalid); }
            else err = cerr;
            if (lane < cnt && (!bad || lane <= nvalid)) {
                ZbBlkDesc D;
                D.hdr_off = (u64)(s + my_pos - src); D.seq_off = my_seq; D.lit_off = my_lit; D.frame = f; D.block_max = block_max;
                D.flags = (b + lane == b0 ? ZB_BD_FIRST : 0u) | (e_valid ? ZB_BD_FSE_VALID : 0u);
                D.dHuf = eHuf; D.dLL = eLL; D.dOF = eOF; D.dML = eML;
                D.span = 3 + bsize;
                bdesc[b + lane] = D;
            }
            b += nvalid;
            __syncwarp();
        }
        for (u64 k = b + lane; k < b1; k += 32) { bdesc[k].flags = ZB_BD_SKIP; bdesc[k].frame = f; }      // (after an error; a healthy frame has none left)
        if (lane == 0) { frame_end[f] = pos; if (err) status[f] = err; }
    }
}

__global__ void zb_scan_blocks(const u8* __restrict__ src, const ZbSegment* __restrict__ segs, u32 n_frames,
                               const ZbFramePlace* __restrict__ place, ZbDictDev dict, u32* __restrict__ status,
                               ZbBlkDesc* __restrict__ bdesc, u64* __restrict__ frame_end, const u32* __restrict__ big_list)
{
    u32 const f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    if (big_list && big_list[0] && segs[f].length > ZB_SCAN_BIG) {          // zb_scan_blocks_big's, if zb_scan_frames listed it
        const u8* s0 = src + segs[f].offset; u64 n0 = segs[f].length;
        zb_skip_skippable(s0, n0);
        if (n0 > ZB_SCAN_BIG) return;
    }
    u64 const b0 = place[f].blk_off, b1 = place[f + 1].blk_off;
    if (status[f] != ZB_OK) { for (u64 b = b0; b < b1; b++) { bdesc[b].flags = ZB_BD_SKIP; bdesc[b].frame = f; } return; }
    const u8* s = src + segs[f].offset; u64 n = segs[f].length;
    zb_skip_skippable(s, n);
    ZbHdr h; zb_parse_header(s, n, h);
    u32 err = ZB_OK;
    if (h.dict_id && dict.dict_id && h.dict_id != dict.dict_id) err = ZB_E_DICT_WRONG;
    u32 const block_max = h.window < ZB_BLOCK_MAX ? (u32)h.window : ZB_BLOCK_MAX;
    ZbTabSrc dHuf = {ZB_SRC_NONE, 0, nullptr, 0}, dLL = dHuf, dOF = dHuf, dML = dHuf;
    bool fse_valid = false;
    if (dict.has_entropy) { dHuf.kind = dLL.kind = dOF.kind = dML.kind = ZB_SRC_DICT; fse_valid = true; }
    u64 pos = h.hdr_size, seq_i = place[f].seq_off, lit_i = place[f].lit_off, b = b0;
    for (; b < b1 && !err; b++) {
        ZbBlkDesc D;
        D.hdr_off = (u64)(s + pos - src); D.seq_off = seq_i; D.lit_off = lit_i; D.frame = f; D.block_max = block_max;
        D.flags = (b == b0 ? ZB_BD_FIRST : 0u) | (fse_valid ? ZB_BD_FSE_VALID : 0u);
        D.dHuf = dHuf; D.dLL = dLL; D.dOF = dOF; D.dML = dML;
        if (pos + 3 > n) { err = ZB_E_SRCSIZE_WRONG; break; }
        u32 const bh = zb_rd24(s + pos), type = (bh >> 1) & 3; u32 bsize = bh >> 3;
        if (type == 3) { err = ZB_E_CORRUPTION; break; }
        if (type == 1) bsize = 1;
        if (pos + 3 + bsize > n) { err = ZB_E_SRCSIZE_WRONG; break; }
        D.span = 3 + bsize;
        bdesc[b] = D;
        if (type == 2) {            // what this block leaves behind for the next one
            const u8* const bs = s + pos + 3;
            ZbLitHdr L; u32 const e = zb_parse_lit_header(bs, bsize, L);
            if (e) { err = e; break; }
            u32 const lsec = L.type == 0 ? L.hdr + L.regen : (L.type == 1 ? L.hdr + 1 : L.hdr + L.csize);
            if (L.regen > ZB_BLOCK_MAX || lsec >= bsize) { err = ZB_E_CORRUPTION; break; }
            if (L.type == 2) { dHuf.kind = ZB_SRC_NCOUNT; dHuf.p = bs + L.hdr; dHuf.n = L.csize; }
            if (L.type >= 2) lit_i += (L.regen + 15) & ~15u;
            const u8* ip = bs + lsec; const u8* const bend = bs + bsize;
            u32 nseq = *ip++;
            if (nseq > 0x7F) {
                if (nseq == 0xFF) { if (ip + 2 > bend) { err = ZB_E_SRCSIZE_WRONG; break; } nseq = zb_rd16(ip) + 0x7F00; ip += 2; }
                else { if (ip >= bend) { err = ZB_E_SRCSIZE_WRONG; break; } nseq = ((nseq - 0x80) << 8) + *ip++; }
            }
            seq_i += nseq + 1;
            if (nseq) {
                if (ip + 1 > bend) { err = ZB_E_SRCSIZE_WRONG; break; }
                u32 const modes = *ip++;
                err = zb_scan_seq_table(dLL, modes >> 6, 35, 9, ip, bend, fse_valid);
                if (!err) err = zb_scan_seq_table(dOF, (modes >> 4) & 3, 31, 8, ip, bend, fse_valid);
                if (!err) err = zb_scan_seq_table(dML, (modes >> 2) & 3, 52, 9, ip, bend, fse_valid);
                if (err) break;
                fse_valid = true;
            }
        }
        pos += 3 + bsize;
        if (bh & 1) { b++; break; }
    }
    for (; b < b1; b++) { bdesc[b].flags = ZB_BD_SKIP; bdesc[b].frame = f; }      // (after an error; a healthy frame has none left)
    frame_end[f] = pos;
#ifdef ZB_DEBUG_BLOCKS
    if (err) printf("[scan_blocks] frame %u err %u at block %llu pos %llu\n", f, err, (unsigned long long)(b - b0), (unsigned long long)pos);
#endif
    if (err) status[f] = err;
}

// K3b: zb_resolve_blocks -- one thread per frame, after zb_entropy_blocks: frame-relative output position of every block,
// the repcode history on entry of every block (the exit histories are symbolic in it), and the checks on the frame as a
// whole that the lane-per-frame kernel makes after its last block (zstd/zstd.c:44260-44277, c-ext/decompressor.c:1151-1162).
__global__ void zb_resolve_blocks(const u8* __restrict__ src, const ZbSegment* __restrict__ segs, u32 n_frames,
                                  const ZbFramePlace* __restrict__ place, const ZbFrameInfo* __restrict__ info, const u64* __restrict__ dst_sizes,
                                  ZbBlock* __restrict__ blocks, const ZbBlkDesc* __restrict__ bdesc, const ZbBlkExit* __restrict__ bexit,
                                  const u64* __restrict__ frame_end, ZbDictDev dict, u32* __restrict__ status, u64* __restrict__ out_sizes,
                                  u32* __restrict__ ck_expect, u32* __restrict__ entry_rep /* [n_blocks][3] */)
{
    u32 const f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    out_sizes[f] = 0;
    if (status[f] != ZB_OK) return;
    u64 const b0 = place[f].blk_off, b1 = place[f + 1].blk_off, cap = place[f].dst_cap;
    u32 r[3] = {1, 4, 8};
    if (dict.has_entropy) { r[0] = dict.rep[0]; r[1] = dict.rep[1]; r[2] = dict.rep[2]; }
    u64 out_pos = 0; u32 err = ZB_OK;
    for (u64 b = b0; b < b1; b++) {
        if (bdesc[b].flags & ZB_BD_SKIP) break;
        ZbBlkExit const X = bexit[b];
        if (X.err) { err = X.err; break; }
        entry_rep[3 * b] = r[0]; entry_rep[3 * b + 1] = r[1]; entry_rep[3 * b + 2] = r[2];
        u32 const regen = blocks[b].regen;
        if (regen > cap - out_pos) { err = ZB_E_DSTSIZE_TOO_SMALL; break; }
        blocks[b].out_pos = out_pos; out_pos += regen;
        u32 nr[3];
        for (int k = 0; k < 3; k++) {
            u32 const x = X.rep[k];
            if (x & 0x80000000u) { u32 const e = r[(x >> 29) & 3], d = x & 0x1FFFFFFFu; nr[k] = e > d ? e - d : 0xFFFFFFFFu; }   // (0: "offset 0" is corrupt, zstd/zstd.c:46905)
            else nr[k] = x;
        }
        r[0] = nr[0]; r[1] = nr[1]; r[2] = nr[2];
    }
    if (!err) {
        ZbFrameInfo const fi = info[f];
        const u8* s = src + segs[f].offset; u64 n = segs[f].length;
        zb_skip_skippable(s, n);
        u64 const pos = frame_end[f];
        if (fi.content_size != ZB_CONTENT_UNKNOWN && out_pos != fi.content_size) err = ZB_E_CORRUPTION;
        else if ((fi.flags & 1) && pos + 4 > n) err = ZB_E_CHECKSUM_WRONG;
        else {
            if (fi.flags & 1) ck_expect[f] = zb_rd32(s + pos);
            if (dst_sizes && out_pos != cap) err = ZB_E_SIZE_MISMATCH;
        }
    }
#ifdef ZB_DEBUG_BLOCKS
    if (err) printf("[resolve] frame %u err %u out_pos %llu content %llu cap %llu blocks %llu..%llu\n", f, err, (unsigned long long)out_pos,
                    (unsigned long long)info[f].content_size, (unsigned long long)cap, (unsigned long long)b0, (unsigned long long)b1);
#endif
    if (err) { status[f] = err; out_sizes[f] = err == ZB_E_SIZE_MISMATCH ? out_pos : 0; } else out_sizes[f] = out_pos;
}

// K3c: zb_patch_blocks -- a warp per block: symbolic offsets become distances, and every offset is checked against what
// has been regenerated in front of it (the check of ZSTD_execSequence, zstd/zstd.c:46666, that zb_entropy_blocks postponed).
// Chain mode (decompress_content_dict_chain): no dictionary; frame f may reach the bytes between its predecessor's start and
// its own, place[f].dst_off - place[f - 1].dst_off (frame 0: the carried prefix, which the launcher put in front of it).
__global__ void __launch_bounds__(256)
zb_patch_blocks(const ZbBlock* __restrict__ blocks, const ZbBlkDesc* __restrict__ bdesc, u64 n_blocks, ZbSeq* __restrict__ seqs,
                const u32* __restrict__ entry_rep, ZbDictDev dict, u32* __restrict__ status,
                const ZbFramePlace* __restrict__ chain_place = nullptr)
{
    u32 const lane = threadIdx.x & 31;
    u64 const b = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= n_blocks) return;
    ZbBlkDesc const D = bdesc[b];
    if ((D.flags & ZB_BD_SKIP) || status[D.frame] != ZB_OK) return;
    ZbBlock const B = blocks[b];
    if (B.kind != ZB_BLK_COMPRESSED || B.n_seq == 0) return;
    u64 const reach = chain_place ? chain_place[D.frame].dst_off - (D.frame ? chain_place[D.frame - 1].dst_off : 0) : dict.content_size;
    u32 const e0 = entry_rep[3 * b], e1 = entry_rep[3 * b + 1], e2 = entry_rep[3 * b + 2];
    ZbSeq* const sq = seqs + B.seq_pos;
    bool bad = false;
    for (u32 i = lane; i < B.n_seq; i += 32) {
        ZbSeq r = sq[i];
        u32 const lit_next = sq[i + 1].x;
        if (r.w & 0x80000000u) {
            u32 const k = (r.w >> 29) & 3, d = r.w & 0x1FFFFFFFu, e = k == 0 ? e0 : (k == 1 ? e1 : e2);
            r.w = e > d ? e - d : 0xFFFFFFFFu;
            sq[i].w = r.w;
        }
        u64 const mstart = B.out_pos + r.y + (lit_next - r.x);            // frame-relative start of the match
        if ((u64)r.w > mstart + reach) {
            bad = true;
#ifdef ZB_DEBUG_BLOCKS
            printf("[patch] block %llu seq %u off %u (raw %u) mstart %llu out_pos %llu e %u %u %u\n", (unsigned long long)b, i, r.w, sq[i].w, (unsigned long long)mstart,
                   (unsigned long long)B.out_pos, e0, e1, e2);
#endif
        }
    }
    if (__any_sync(0xFFFFFFFFu, bad) && lane == 0) atomicCAS(&status[D.frame], (u32)ZB_OK, (u32)ZB_E_CORRUPTION);
}

// ===========================================================================
// K4: LZ copy-execute -- one warp per frame
// ===========================================================================

// per-lane forward copy in chunks of 8 bytes: the 8 loads of a chunk are independent (issued back to
// back) and precede its 8 stores, so a copy costs one memory latency per 8 bytes instead of per byte.
// Safe for overlapping ranges whenever dst - src >= 8.
__device__ __forceinline__ void zb_copy_fwd8(u8* d, const u8* s, u32 n)
{
    u32 k = 0;
    for (; k + 8 <= n; k += 8) {
        u8 t0 = s[k], t1 = s[k + 1], t2 = s[k + 2], t3 = s[k + 3], t4 = s[k + 4], t5 = s[k + 5], t6 = s[k + 6], t7 = s[k + 7];
        d[k] = t0; d[k + 1] = t1; d[k + 2] = t2; d[k + 3] = t3; d[k + 4] = t4; d[k + 5] = t5; d[k + 6] = t6; d[k + 7] = t7;
    }
    if (k + 4 <= n) {
        u8 t0 = s[k], t1 = s[k + 1], t2 = s[k + 2], t3 = s[k + 3];
        d[k] = t0; d[k + 1] = t1; d[k + 2] = t2; d[k + 3] = t3; k += 4;
    }
    for (; k < n; k++) d[k] = s[k];
}

// warp-cooperative byte copy (no overlap between src and dst)
__device__ __forceinline__ void zb_warp_copy(u8* dst, const u8* src, u32 n, u32 lane)
{
    if (n >= 64 && ((((uintptr_t)dst) ^ ((uintptr_t)src)) & 15) == 0) {
        u32 head = (u32)((16 - ((uintptr_t)dst & 15)) & 15);
        if (lane < head) dst[lane] = src[lane];
        dst += head; src += head; n -= head;
        u32 nv = n >> 4;
        const uint4* s4 = (const uint4*)src; uint4* d4 = (uint4*)dst;
        for (u32 i = lane; i < nv; i += 32) d4[i] = s4[i];
        u32 done = nv << 4;
        if (done + lane < n) dst[done + lane] = src[done + lane];
        return;
    }
    for (u32 i = lane; i < n; i += 32) dst[i] = src[i];
}

__global__ void __launch_bounds__(256)
zb_execute(const u8* __restrict__ src, const ZbFramePlace* __restrict__ place, const u32* __restrict__ status,
           const ZbBlock* __restrict__ blocks, const ZbSeq* __restrict__ seqs, const u8* __restrict__ lits,
           u8* dst, u32 first, u32 n_frames, ZbDictDev dict, u64 min_cap)
{
    u32 const lane = threadIdx.x & 31;
    u32 const f = first + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5);      // frames [first, n_frames)
    if (f >= n_frames) return;
    if (status[f] != ZB_OK) return;
    ZbFramePlace const pl = place[f];
    if (pl.dst_cap < min_cap) return;                    // staged in shared memory by zb_execute_tile
    u8* const out = dst + pl.dst_off;
    u64 const blk_end = place[f + 1].blk_off;            // place[] has n_frames + 1 entries
    const u8* const dict_end = dict.content + dict.content_size;

    for (u64 bi = pl.blk_off; bi < blk_end; bi++) {
        ZbBlock const B = blocks[bi];
        u8* const bout = out + B.out_pos;
        if (B.kind == ZB_BLK_RAW) { zb_warp_copy(bout, src + B.src_pos, B.regen, lane); continue; }
        if (B.kind == ZB_BLK_RLE) { for (u32 i = lane; i < B.regen; i += 32) bout[i] = (u8)B.lit_byte; continue; }
        if (B.kind != ZB_BLK_COMPRESSED) return;
        const u8* const lit = B.lit_kind == ZB_LIT_RAW ? src + B.src_pos : lits + B.src_pos;
        bool const lit_rle = B.lit_kind == ZB_LIT_RLE; u8 const lit_byte = (u8)B.lit_byte;
        const ZbSeq* const sq = seqs + B.seq_pos;
        u32 const nseq = B.n_seq;
        for (u32 g = 0; g < nseq; g += 32) {
            u32 const i = g + lane; bool const valid = i < nseq;
            ZbSeq r = valid ? sq[i] : make_uint4(0, 0, 0, 0);
            ZbSeq r2 = valid ? sq[i + 1] : make_uint4(0, 0, 0, 0);
            u32 const ll = r2.x - r.x, ml = r.z, off = r.w;
            u32 const ostart = r.y, mstart = r.y + ll;
            // literals: independent of everything else
            if (valid) {
                if (lit_rle) for (u32 k = 0; k < ll; k++) bout[ostart + k] = lit_byte;
                else zb_copy_fwd8(bout + ostart, lit + r.x, ll);
            }
            __syncwarp();
            // matches: a lane may run when every byte it reads that other sequences produce lies
            // below the frontier F (= match start of the first unfinished sequence)
            bool pending = valid;
            long long const abs_m = (long long)B.out_pos + mstart;       // frame-relative match start
            long long const srcp = abs_m - (long long)off;               // may be negative: dictionary
            long long const need = min(srcp + (long long)ml, (long long)B.out_pos + ostart);
            for (;;) {
                u32 const pm = __ballot_sync(0xFFFFFFFFu, pending);
                if (!pm) break;
                int const fu = __ffs(pm) - 1;
                long long const F = __shfl_sync(0xFFFFFFFFu, abs_m, fu);
                bool const ready = pending && need <= F;
                // long matches of ready lanes: the whole warp copies them, one at a time
                u32 big = __ballot_sync(0xFFFFFFFFu, ready && ml >= 48);
                while (big) {
                    int const l = __ffs(big) - 1; big &= big - 1;
                    long long const m0 = __shfl_sync(0xFFFFFFFFu, abs_m, l);
                    u32 const o = __shfl_sync(0xFFFFFFFFu, off, l), len = __shfl_sync(0xFFFFFFFFu, ml, l);
                    u8* d = out + m0;
                    if ((long long)o > m0) {
                        // starts in the dictionary: byte-wise with the source select
                        for (u32 j = lane; j < len; j += 32) {
                            long long sp = m0 - (long long)o + (long long)(j % o);
                            d[j] = sp < 0 ? dict_end[sp] : out[sp];
                        }
                    } else if (o >= 32) {
                        // chunks of 32 bytes never read bytes of their own chunk
                        const u8* sp = d - o;
                        for (u32 j = 0; j < len; j += 32) { if (j + lane < len) d[j + lane] = sp[j + lane]; __syncwarp(); }
                    } else {
                        const u8* sp = d - o;                            // periodic pattern of period o
                        for (u32 j = lane; j < len; j += 32) d[j] = sp[j % o];
                    }
                    __syncwarp();
                }
                if (ready) {
                    if (ml < 48) {
                        u8* d = out + abs_m;
                        if (srcp >= 0) {
                            const u8* sp = out + srcp;
                            if (off >= 8) zb_copy_fwd8(d, sp, ml);
                            else { u32 q = 0; for (u32 k = 0; k < ml; k++) { d[k] = sp[q]; if (++q == off) q = 0; } }
                        } else {
                            for (u32 k = 0; k < ml; k++) { long long p = srcp + (long long)(k % off); d[k] = p < 0 ? dict_end[p] : out[p]; }
                        }
                    }
                    pending = false;
                }
                __syncwarp();
            }
        }
        // last literals of the block
        {
            ZbSeq const e = sq[nseq];
            u32 const tail = B.n_lit - e.x;
            if (lit_rle) { for (u32 k = lane; k < tail; k += 32) bout[e.y + k] = lit_byte; }
            else zb_warp_copy(bout + e.y, lit + e.x, tail, lane);
        }
        __syncwarp();
    }
}




// ---------------------------------------------------------------------------
// K4 (tile variant): frames whose whole output fits a shared-memory tile.  The warp regenerates the
// frame in shared memory -- literal runs and match copies become LDS/STS with no global-memory
// sector scatter -- and writes the finished frame to HBM with 128-bit coalesced stores.
// ---------------------------------------------------------------------------
#define ZB_TILE_CAP    4096
#define ZB_TILE_WARPS  8
#define ZB_TILE_WARP_BYTES (ZB_TILE_CAP + 64)     // output tile at the frame's 16-byte phase; its literals are staged inside it
#define ZB_TILE_SMEM   (ZB_TILE_WARPS * ZB_TILE_WARP_BYTES)

// per-phase cycle counters of zb_execute_tile (lane 0 of every warp) exist only in tuning builds (-DZB_PHASE_TIMERS):
// 0 frame start and literal staging, 1 literal copies, 2 frontier passes, 3 write-out
#ifdef ZB_PHASE_TIMERS
__device__ unsigned long long g_zb_exe_phase[4];
#define ZB_XSTART() long long t_x = clock64(), x_acc[4] = {0, 0, 0, 0}
#define ZB_XMARK(k) do { long long const t_ = clock64(); x_acc[k] += t_ - t_x; t_x = t_; } while (0)
#define ZB_XFLUSH() do { if (lane == 0) for (int k_ = 0; k_ < 4; k_++) atomicAdd(&g_zb_exe_phase[k_], (unsigned long long)x_acc[k_]); } while (0)
#else
#define ZB_XSTART() do { } while (0)
#define ZB_XMARK(k) do { } while (0)
#define ZB_XFLUSH() do { } while (0)
#endif

// 5 CTAs per SM (40 warps; shared memory would allow 6): 48 registers.  Left to itself ptxas takes 62 and fits 4 CTAs,
// which measured slower (DESIGN §4, K4).
__global__ void __launch_bounds__(ZB_TILE_WARPS * 32, 5)
zb_execute_tile(const u8* __restrict__ src, const ZbFramePlace* __restrict__ place, const u32* __restrict__ status,
                const ZbBlock* __restrict__ blocks, const ZbSeq* __restrict__ seqs, const u8* __restrict__ lits,
                u8* __restrict__ dst, u32 first, u32 n_frames, ZbDictDev dict)
{
    ZB_DYN_SMEM(zb_tile);
    u32 const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 const f = first + blockIdx.x * ZB_TILE_WARPS + warp;                    // frames [first, n_frames)
    if (f >= n_frames) return;
    if (status[f] != ZB_OK) return;
    ZbFramePlace const pl = place[f];
    if (pl.dst_cap > ZB_TILE_CAP) return;                // handled by zb_execute
    ZB_XSTART();
    u64 const blk_end = place[f + 1].blk_off;
    u32 const skew = (u32)(pl.dst_off & 15);             // same 16-byte phase in smem as in dst
    u8* const so = zb_tile + warp * ZB_TILE_WARP_BYTES + skew;          // output tile
    const u8* const dict_end = dict.content + dict.content_size;
    u32 total = 0;

    // Literals are staged IN PLACE, at sl = align16(so + dst_cap - n_lit) inside the output tile.  Literal j of a block goes
    // to out_pos + j + M(j), M(j) = the block's match bytes in front of it, and out_pos + regen <= dst_cap with regen =
    // n_lit + all the block's match bytes, so every literal's output lies at or below its staged copy: P(j) <= sl + j.
    // Hence nothing written for literals up to j reaches a staged literal after j: match copies of a group end below the
    // next group's literals, literal runs and the block's last literals are copied forward with loads ahead of stores
    // (destination <= source), and the next block stages its literals above everything written so far.  The one hazard
    // is INSIDE a group's literal copies, which run side by side: a later lane's run may land on an earlier lane's
    // staged literals before that lane has read them.  A group whose runs all end at or below its lowest staged literal
    // copies lane by lane as usual; any other group copies its literals as one stream, in warp-wide steps that load
    // before they store, so each step writes only below what later steps read.  Rounding sl up only adds margin; the
    // 16-byte staging over-read ends at most 30 bytes past dst_cap, inside the warp's slice.
    for (u64 bi = pl.blk_off; bi < blk_end; bi++) {
        ZbBlock const B = blocks[bi];
        u8* const bout = so + B.out_pos;
        total = (u32)B.out_pos + B.regen;
        if (B.kind == ZB_BLK_RAW) { const u8* p = src + B.src_pos; for (u32 i = lane; i < B.regen; i += 32) bout[i] = p[i]; __syncwarp(); ZB_XMARK(0); continue; }
        if (B.kind == ZB_BLK_RLE) { for (u32 i = lane; i < B.regen; i += 32) bout[i] = (u8)B.lit_byte; __syncwarp(); ZB_XMARK(0); continue; }
        if (B.kind != ZB_BLK_COMPRESSED) return;
        bool const lit_rle = B.lit_kind == ZB_LIT_RLE; u8 const lit_byte = (u8)B.lit_byte;
        u32 const lrel = (((u32)(uintptr_t)(so + pl.dst_cap - B.n_lit) + 15) & ~15u) - (u32)(uintptr_t)so;
        u8* const sl = so + lrel;
        if (B.lit_kind == ZB_LIT_SCRATCH) {               // 16-byte aligned slice of the literal scratch
            const uint4* g = (const uint4*)(lits + B.src_pos); uint4* d4 = (uint4*)sl;
            for (u32 i = lane; i < (B.n_lit + 15) / 16; i += 32) d4[i] = g[i];
        } else if (B.lit_kind == ZB_LIT_RAW) {
            const u8* g = src + B.src_pos; for (u32 i = lane; i < B.n_lit; i += 32) sl[i] = g[i];
        }
        __syncwarp();
        ZB_XMARK(0);
        const ZbSeq* const sq = seqs + B.seq_pos;
        u32 const nseq = B.n_seq;
        for (u32 g = 0; g < nseq; g += 32) {
            u32 const i = g + lane; bool const valid = i < nseq;
            ZbSeq const r = valid ? sq[i] : make_uint4(0, 0, 0, 0);
            u32 nx = __shfl_down_sync(0xFFFFFFFFu, r.x, 1);
            if (lane == 31 || i + 1 >= nseq) nx = valid ? sq[i + 1].x : 0;
            u32 const ll = nx - r.x, ml = r.z, off = r.w;
            u32 const ostart = r.y, mstart = r.y + ll;
            u32 const x0 = __shfl_sync(0xFFFFFFFFu, r.x, 0);
            if (lit_rle || !__any_sync(0xFFFFFFFFu, valid && (u32)B.out_pos + mstart > lrel + x0)) {
                if (valid) {
                    u8* o = bout + ostart;
                    if (lit_rle) for (u32 k = 0; k < ll; k++) o[k] = lit_byte;
                    else zb_copy_fwd8(o, sl + r.x, ll);         // destination <= source: each 8-byte chunk loads first
                }
            } else {
                // literal j of the group goes to bout + ostart_s + j - x_s for the last lane s with x_s <= j
                u32 const xe = __shfl_sync(0xFFFFFFFFu, nx, min(31u, nseq - 1 - g));
                u32 const key = valid ? r.x : 0xFFFFFFFFu;
                int const delta = (int)ostart - (int)r.x;
                for (u32 j0 = x0; j0 < xe; j0 += 32) {
                    u32 const j = j0 + lane;
                    u32 s = 0;                                   // lane 0 (key x0 <= j) qualifies
                    for (u32 b = 16; b; b >>= 1) if (__shfl_sync(0xFFFFFFFFu, key, s + b) <= j) s += b;
                    int const dj = __shfl_sync(0xFFFFFFFFu, delta, (int)s);
                    u8 const v = j < xe ? sl[j] : 0;
                    __syncwarp();
                    if (j < xe) bout[(int)j + dj] = v;
                    __syncwarp();
                }
            }
            __syncwarp();
            ZB_XMARK(1);
            bool pending = valid;
            int const abs_m = (int)B.out_pos + (int)mstart;             // frame-relative match start
            int const srcp = abs_m - (int)off;                          // negative: reaches into the dictionary
            int const need = min(srcp + (int)ml, abs_m);                // bytes [srcp, need) come from other sequences
            // the group's sequences whose matches start below `need`: lanes [0, t) (match starts ascend with the lane)
            int const key = valid ? abs_m : 0x7FFFFFFF, mend = abs_m + (int)ml;
            u32 t = 0;
            for (u32 b = 16; b; b >>= 1) if (__shfl_sync(0xFFFFFFFFu, key, t + b - 1) < need) t += b;
            u32 const below = t ? 0xFFFFFFFFu >> (32 - t) : 0u;
            for (;;) {
                u32 const pm = __ballot_sync(0xFFFFFFFFu, pending);
                if (!pm) break;
                // a lane may run when no unfinished match overlaps its source: the last unfinished one starting below
                // `need` (it ends last: matches are disjoint and in order) ends at or before srcp
                u32 const cand = pm & below;
                int const e = __shfl_sync(0xFFFFFFFFu, mend, cand ? 31 - __clz((int)cand) : (int)lane);
                bool const ready = pending && (!cand || e <= srcp);
                u32 big = __ballot_sync(0xFFFFFFFFu, ready && ml >= 32);
                while (big) {
                    int const l = __ffs(big) - 1; big &= big - 1;
                    int const m0 = __shfl_sync(0xFFFFFFFFu, abs_m, l);
                    u32 const o = __shfl_sync(0xFFFFFFFFu, off, l), len = __shfl_sync(0xFFFFFFFFu, ml, l);
                    u8* d = so + m0;
                    if ((int)o > m0) {
                        for (u32 j = lane; j < len; j += 32) { int sp = m0 - (int)o + (int)(j % o); d[j] = sp < 0 ? dict_end[sp] : so[sp]; }
                    } else if (o >= 32) {
                        const u8* sp = d - o;
                        for (u32 j = 0; j < len; j += 32) { if (j + lane < len) d[j + lane] = sp[j + lane]; __syncwarp(); }
                    } else {
                        const u8* sp = d - o;
                        for (u32 j = lane; j < len; j += 32) d[j] = sp[j % o];
                    }
                    __syncwarp();
                }
                if (ready) {
                    if (ml < 32) {
                        u8* d = so + abs_m;
                        if (srcp >= 0) {
                            const u8* sp = so + srcp;
                            if (off >= 8) zb_copy_fwd8(d, sp, ml);      // 8-byte chunks never read their own output
                            else { u32 q = 0; for (u32 k = 0; k < ml; k++) { d[k] = sp[q]; if (++q == off) q = 0; } }
                        } else {
                            for (u32 k = 0; k < ml; k++) { int p = srcp + (int)(k % off); d[k] = p < 0 ? dict_end[p] : so[p]; }
                        }
                    }
                    pending = false;
                }
                __syncwarp();
            }
            ZB_XMARK(2);
        }
        {
            ZbSeq const e = sq[nseq];
            u32 const tail = B.n_lit - e.x;
            if (lit_rle) { for (u32 k = lane; k < tail; k += 32) bout[e.y + k] = lit_byte; }
            else
                for (u32 k0 = 0; k0 < tail; k0 += 32) {           // in place (destination <= source): load, then store
                    u32 const k = k0 + lane;
                    u8 const v = k < tail ? sl[e.x + k] : 0;
                    __syncwarp();
                    if (k < tail) bout[e.y + k] = v;
                    __syncwarp();
                }
        }
        __syncwarp();
        ZB_XMARK(1);
    }
    // finished frame -> HBM, 128-bit stores (so and dst share the same 16-byte phase)
    {
        u8* const out = dst + pl.dst_off;
        u32 head = (16 - skew) & 15; if (head > total) head = total;
        if (lane < head) out[lane] = so[lane];
        u32 const nv = (total - head) >> 4;
        const uint4* s4 = (const uint4*)(so + head); uint4* d4 = (uint4*)(out + head);
        for (u32 i = lane; i < nv; i += 32) d4[i] = s4[i];
        u32 const done = head + (nv << 4);
        if (done + lane < total) out[done + lane] = so[done + lane];
    }
    ZB_XMARK(3);
    ZB_XFLUSH();
}


// ===========================================================================
// content checksum: low 32 bits of XXH64(seed 0) over the regenerated frame (zstd/zstd.c:44260-44277).
// One lane per checksummed frame (the four accumulators are a serial chain over 32-byte stripes).
// ===========================================================================
// K4 (block-tile variant): frames of many blocks when few frames are in flight (the block-parallel path: one huge frame at
// the limit).  zb_execute walks such a frame with one warp straight in HBM/L2 -- every batch of 32 sequences pays global
// round trips: 1.5 ms per 128 KiB block.  Here the frame's CTA regenerates block after block in SHARED MEMORY (output tile
// 128 KiB + the block's literals) and writes each finished block with 128-bit stores; only matches that reach in front of
// the block read global memory (the frame's own earlier output, or the dictionary).
// ===========================================================================
#define ZB_BIG_NT       512
#define ZB_BIG_SEQCAP   6144u                      // sequences in flight at once (a block with more runs in chunks)
#define ZB_BIG_PER      (ZB_BIG_SEQCAP / ZB_BIG_NT)
#define ZB_BIG_SMEM     (ZB_BLOCK_MAX + 64 + (4 * ZB_BIG_SEQCAP + 4 + ZB_BIG_SEQCAP / 32) * 4)

// A persistent grid of CTAs (16 warps each) takes the BLOCKS of all frames in order from a ticket counter -- the blocks of one
// frame run on many SMs at once, each in its own 128 KiB shared-memory tile.  Inside a block up to 6144 sequences are IN
// FLIGHT together, 12 per thread: all literal runs are copied first (independent, straight from the literal buffer), then
// every warp sweeps over its pending matches without CTA barriers.  A match runs when
//   * the matches of the block that OVERLAP ITS SOURCE are finished: their index range [ja, jb) comes from two binary
//     searches over the sorted sequence starts / match starts, a done-bitmap in shared memory tells the rest -- so the
//     number of sweeps is the depth of the dependency chains, not their count;
//   * the part of its source in front of the block is final in global memory: the frame's FINISHED PREFIX (wave.done_pos:
//     every block below it is stored and fenced) covers it.
// Matches of 64 bytes and more are copied by their whole warp.  Matches only point backwards and tickets are handed out in
// order, so the lowest unfinished block never waits: no deadlock for any grid size.
__device__ __forceinline__ u32 zb_warp_or(u32 v)
{
    #pragma unroll
    for (int d = 16; d; d >>= 1) v |= __shfl_xor_sync(0xFFFFFFFFu, v, d);
    return v;
}

#ifdef ZB_DEBUG_BLOCKS
__device__ __forceinline__ unsigned long long zb_gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define ZB_BIGT(...) __VA_ARGS__
#else
#define ZB_BIGT(...)
#endif

struct ZbWave {                     // zeroed before every launch
    unsigned long long* done_pos;   // per frame: output bytes [0, done_pos) are final in global memory
    u32* pre_blk;                   // per frame: blocks [0, pre_blk) of the frame are finished
    u32* blk_flag;                  // per block (absolute index): finished
    u32* ticket;                    // next block to hand out, relative to blk_first
};

__global__ void __launch_bounds__(ZB_BIG_NT)
zb_execute_big(const u8* __restrict__ src, const ZbFramePlace* __restrict__ place, const u32* __restrict__ status,
               const ZbBlock* __restrict__ blocks, const ZbBlkDesc* __restrict__ bdesc, const ZbSeq* __restrict__ seqs,
               const u8* __restrict__ lits, u8* dst, u64 blk_first, u64 blk_last, ZbDictDev dict, u64 min_cap, ZbWave wave)
{
    ZB_DYN_SMEM(zb_big);
    __shared__ u32 s_ticket;
    u32 const tid = threadIdx.x, lane = tid & 31;
    const u8* const dict_end = dict.content + dict.content_size;
    u32* const sO = (u32*)(zb_big + ZB_BLOCK_MAX + 64);  // [SEQCAP + 1] output start of every sequence of the chunk (block-relative)
    u32* const sM = sO + ZB_BIG_SEQCAP + 4;              // [SEQCAP] its match start
    u32* const sF = sM + ZB_BIG_SEQCAP;                  // [SEQCAP] its offset
    u32* const sD = sF + ZB_BIG_SEQCAP;                  // [SEQCAP] ja | jb << 14 | (source in front of the block) << 31
    u32* const sB = sD + ZB_BIG_SEQCAP;                  // [SEQCAP / 32] done bitmap

    for (;;) {
        __syncthreads();                                  // (s_ticket and the tile are free again)
        if (tid == 0) s_ticket = atomicAdd(wave.ticket, 1u);
        __syncthreads();
        u64 const bi = blk_first + s_ticket;
        if (bi >= blk_last) return;
        ZB_BIGT(unsigned long long const tg0 = zb_gtime(); unsigned long long tg1 = 0, tg_seen = 0, tg2 = 0, tg3 = 0; u32 n_sweeps = 0; u32 n_ext = 0;)
        u32 const f = bdesc[bi].frame;
        if (status[f] != ZB_OK) continue;
        ZbFramePlace const pl = place[f];
        if (pl.dst_cap < min_cap) continue;              // staged whole by zb_execute_tile
        u8* const out = dst + pl.dst_off;
        ZbBlock const B = blocks[bi];
        u8* const gout = out + B.out_pos;
        if (B.kind == ZB_BLK_RAW) { const u8* p = src + B.src_pos; for (u32 i = tid; i < B.regen; i += ZB_BIG_NT) gout[i] = p[i]; }
        else if (B.kind == ZB_BLK_RLE) { for (u32 i = tid; i < B.regen; i += ZB_BIG_NT) gout[i] = (u8)B.lit_byte; }
        else if (B.kind == ZB_BLK_COMPRESSED) {
        u32 const skew = (u32)((uintptr_t)gout & 15);    // same 16-byte phase in the tile as in dst
        u8* const so = zb_big + skew;                    // so[i] = byte i of the block
        long long const base = (long long)B.out_pos;     // frame-relative position of so[0]
        bool const lit_rle = B.lit_kind == ZB_LIT_RLE; u8 const lit_byte = (u8)B.lit_byte;
        const u8* const lit = B.lit_kind == ZB_LIT_RAW ? src + B.src_pos : lits + B.src_pos;
        const ZbSeq* const sq = seqs + B.seq_pos;
        u32 const nseq = B.n_seq;
        long long seen = 0;                               // the frame's finished prefix as last polled (warp-uniform)
        for (u32 c0 = 0; c0 < nseq; c0 += ZB_BIG_SEQCAP) {
            u32 const cn = nseq - c0 < ZB_BIG_SEQCAP ? nseq - c0 : ZB_BIG_SEQCAP;
            __syncthreads();                              // (the previous chunk is over: its arrays are free, its bytes final)
            // ---- all literal runs of the chunk, and its sequences into shared memory
            for (u32 w = tid; w < ZB_BIG_SEQCAP / 32; w += ZB_BIG_NT) sB[w] = 0;
            for (u32 k = 0; k < ZB_BIG_PER; k++) {
                u32 const il = tid + k * ZB_BIG_NT;
                if (il < cn) {
                    ZbSeq const r = sq[c0 + il]; u32 const nx = sq[c0 + il + 1].x;
                    u32 const ll = nx - r.x;
                    sO[il] = r.y; sM[il] = r.y + ll; sF[il] = r.w;
                    u8* o = so + r.y;
                    if (lit_rle) for (u32 q = 0; q < ll; q++) o[q] = lit_byte;
                    else zb_copy_fwd8(o, lit + r.x, ll);
                }
            }
            if (tid == 0) sO[cn] = sq[c0 + cn].y;
            __syncthreads();
            // ---- the matches of this chunk my sources overlap: [ja, jb) -- spans that end above my source start, matches that
            //      start below my source end
            for (u32 k = 0; k < ZB_BIG_PER; k++) {
                u32 const il = tid + k * ZB_BIG_NT;
                if (il >= cn) break;
                long long const m = (long long)sM[il], ml = (long long)sO[il + 1] - m, srcp = m - (long long)sF[il];
                long long const s_lo = srcp, s_hi = min(srcp + ml, m);
                u32 ja, jb;
                { u32 lo = 0, hi = il; while (lo < hi) { u32 const md = (lo + hi) >> 1; if ((long long)sO[md + 1] > s_lo) hi = md; else lo = md + 1; } ja = lo; }
                { u32 lo = ja, hi = il; while (lo < hi) { u32 const md = (lo + hi) >> 1; if ((long long)sM[md] >= s_hi) hi = md; else lo = md + 1; } jb = lo; }
                bool const ext = srcp < 0 && base + min(srcp + ml, 0ll) > 0;
                sD[il] = ja | (jb << 14) | (ext ? 0x80000000u : 0u);
            }
            __syncthreads();
            // ---- who copies what: warps 0-7 the matches whose source lies in the block (shared memory only: a hop of a
            //      dependency chain costs a few hundred cycles), warps 8-15 the ones that read in front of the block (global
            //      memory: ~1 us per hop) -- thread t of a group has the sequences t + 256 k of its kind
            u32 const grp = tid >> 8, t8 = tid & 255u;
            u32 pend = 0;
            for (u32 k = 0; k < ZB_BIG_SEQCAP / 256; k++) {
                u32 const il = t8 + k * 256;
                if (il < cn && (sD[il] >> 31) == grp) pend |= 1u << k;
            }
            // ---- sweeps over the pending matches; no CTA barrier until the warp's matches are all done
            bool poll = true;
            ZB_BIGT(if (tid == 0 && c0 == 0) tg1 = zb_gtime(); n_ext += grp ? __popc(pend) : 0;)
            for (;;) {
                ZB_BIGT(n_sweeps++;)
                if (grp && seen < base && __any_sync(0xFFFFFFFFu, poll)) {
                    unsigned long long v = 0;
                    if (lane == 0) { v = *(volatile unsigned long long*)(wave.done_pos + f); __threadfence(); }
                    seen = (long long)__shfl_sync(0xFFFFFFFFu, v, 0);
                    ZB_BIGT(if (seen >= base && tid == 256) tg_seen = zb_gtime();)
                }
                poll = false;
                for (u32 un = zb_warp_or(pend); un; un &= un - 1) {
                    u32 const k = (u32)__ffs((int)un) - 1u;
                    bool const mine = (pend >> k) & 1u;
                    u32 const il = t8 + k * 256;
                    bool ready = mine;
                    int m = 0; u32 ml = 0, off = 0;
                    if (mine) {
                        u32 const d = sD[il]; u32 const ja = d & 0x3FFFu, jb = (d >> 14) & 0x7FFFu;
                        if (jb > ja) {
                            for (u32 w = ja >> 5; w <= (jb - 1) >> 5; w++) {
                                u32 const lo_b = w == (ja >> 5) ? (ja & 31) : 0u, hi_b = w == ((jb - 1) >> 5) ? ((jb - 1) & 31) : 31u;
                                u32 const mask = (0xFFFFFFFFu << lo_b) & (0xFFFFFFFFu >> (31 - hi_b));
                                if ((((volatile u32*)sB)[w] & mask) != mask) { ready = false; break; }
                            }
                        }
                        m = (int)sM[il]; ml = sO[il + 1] - (u32)m; off = sF[il];
                        if (ready && (d >> 31) && seen < base) {
                            long long const need = min(base, base + (long long)m - (long long)off + (long long)ml);
                            if (seen < need) { ready = false; poll = true; }
                        }
                        __threadfence_block();            // (the bitmap was read before the bytes are)
                    }
                    long long const srcp = (long long)m - (long long)off;       // block-relative source: negative = in front of the block
                    u32 big = __ballot_sync(0xFFFFFFFFu, ready && ml >= 64);
                    while (big) {          // long matches: the whole warp copies
                        int const l = __ffs(big) - 1; big &= big - 1;
                        int const m0 = __shfl_sync(0xFFFFFFFFu, m, l);
                        u32 const o = __shfl_sync(0xFFFFFFFFu, off, l), len = __shfl_sync(0xFFFFFFFFu, ml, l);
                        u8* d = so + m0;
                        if ((long long)o > (long long)m0) {                 // starts in front of the block: byte-wise with the source select
                            for (u32 j = lane; j < len; j += 32) {
                                long long const sp = (long long)m0 - (long long)o + (long long)(j % o);
                                u8 v;
                                if (sp >= 0) v = so[sp];
                                else { long long const fp = base + sp; v = fp >= 0 ? __ldcg(out + fp) : dict_end[fp]; }
                                d[j] = v;
                            }
                        } else if (o >= 32) {
                            const u8* sp = d - o;
                            for (u32 j = 0; j < len; j += 32) { if (j + lane < len) d[j + lane] = sp[j + lane]; __syncwarp(); }
                        } else {
                            const u8* sp = d - o;
                            for (u32 j = lane; j < len; j += 32) d[j] = sp[j % o];
                        }
                        __threadfence_block();
                        __syncwarp();
                    }
                    if (ready) {
                        if (ml < 64) {
                            u8* d = so + m;
                            if (srcp >= 0) {
                                const u8* sp = so + srcp;
                                if (off >= 8) zb_copy_fwd8(d, sp, ml);      // 8-byte chunks never read their own output
                                else { u32 q = 0; for (u32 j = 0; j < ml; j++) { d[j] = sp[q]; if (++q == off) q = 0; } }
                            } else if (off >= ml && srcp + (long long)ml <= 0 && base + srcp >= 0) {
                                // the whole source is earlier output of the frame: up to nine aligned 8-byte words, all loads in
                                // flight together (one trip to L2 instead of one per byte)
                                const u8* const gp = out + (base + srcp);
                                u32 const mis = (u32)((uintptr_t)gp & 7u);
                                const unsigned long long* const ga = (const unsigned long long*)(gp - mis);
                                unsigned long long w[9];
                                #pragma unroll
                                for (u32 q = 0; q < 9; q++) w[q] = q * 8 < mis + ml ? __ldcg(ga + q) : 0ull;
                                #pragma unroll
                                for (u32 q = 0; q < 9; q++) {
                                    #pragma unroll
                                    for (u32 bq = 0; bq < 8; bq++) {
                                        int const idx = (int)(q * 8 + bq) - (int)mis;
                                        if (idx >= 0 && idx < (int)ml) d[idx] = (u8)(w[q] >> (8 * bq));
                                    }
                                }
                            } else if (off >= ml) {
                                // the source starts in front of the block (dictionary, or straddling the block start) and does not
                                // overlap the match: eight loads, then eight stores
                                for (u32 k0 = 0; k0 < ml; k0 += 8) {
                                    u8 t[8];
                                    #pragma unroll
                                    for (u32 q = 0; q < 8; q++) {
                                        long long const sp = srcp + (long long)(k0 + q);
                                        u8 v = 0;
                                        if (k0 + q < ml) {
                                            if (sp >= 0) v = so[sp];
                                            else { long long const fp = base + sp; v = fp >= 0 ? __ldcg(out + fp) : dict_end[fp]; }
                                        }
                                        t[q] = v;
                                    }
                                    #pragma unroll
                                    for (u32 q = 0; q < 8; q++) if (k0 + q < ml) d[k0 + q] = t[q];
                                }
                            } else {
                                for (u32 j = 0; j < ml; j++) {
                                    long long const sp = srcp + (long long)(j % off);
                                    u8 v;
                                    if (sp >= 0) v = so[sp];
                                    else { long long const fp = base + sp; v = fp >= 0 ? __ldcg(out + fp) : dict_end[fp]; }
                                    d[j] = v;
                                }
                            }
                        }
                        __threadfence_block();            // the bytes before the bit
                        atomicOr(&sB[il >> 5], 1u << (il & 31));
                        pend &= ~(1u << k);
                    }
                }
                if (!__any_sync(0xFFFFFFFFu, pend != 0)) break;
            }
        }
        ZB_BIGT(u32 const my_sweeps = n_sweeps; if (tid == 256 && bi >= 2000 && bi < 2024) printf("  [blk %llu] ext warp 8: sweeps %u, seen at %llu, ext seqs of thread %u\n", bi, my_sweeps, tg_seen - tg0, n_ext);)
        __syncthreads();
        ZB_BIGT(tg2 = zb_gtime();)
        {   // last literals of the block
            ZbSeq const e = sq[nseq];
            u32 const tail = B.n_lit - e.x;
            if (lit_rle) { for (u32 k = tid; k < tail; k += ZB_BIG_NT) so[e.y + k] = lit_byte; }
            else for (u32 k = tid; k < tail; k += ZB_BIG_NT) so[e.y + k] = lit[e.x + k];
        }
        __syncthreads();
        {   // finished block -> HBM, 128-bit stores (so and gout share the same 16-byte phase)
            u32 const total = B.regen;
            u32 head = (16 - skew) & 15; if (head > total) head = total;
            if (tid < head) gout[tid] = so[tid];
            u32 const nv = (total - head) >> 4;
            const uint4* s4 = (const uint4*)(so + head); uint4* d4 = (uint4*)(gout + head);
            for (u32 i = tid; i < nv; i += ZB_BIG_NT) d4[i] = s4[i];
            u32 const done = head + (nv << 4);
            if (done + tid < total) gout[done + tid] = so[done + tid];
        }
        }
        // the block is in global memory: publish it and move the frame's finished prefix over every finished block behind it
        __threadfence();          // later blocks of this frame read these bytes through L2 (__ldcg)
        __syncthreads();
        if (tid == 0) {
            u32 const nblk = (u32)(place[f + 1].blk_off - pl.blk_off);
            atomicExch(wave.blk_flag + bi, 1u);
            __threadfence();
            for (;;) {
                u32 const cur = *(volatile u32*)(wave.pre_blk + f);
                if (cur >= nblk) break;
                if (*(volatile u32*)(wave.blk_flag + pl.blk_off + cur) == 0) break;
                __threadfence();
                if (atomicCAS(wave.pre_blk + f, cur, cur + 1) == cur) {
                    ZbBlock const Bc = blocks[pl.blk_off + cur];
                    __threadfence();
                    atomicMax(wave.done_pos + f, (unsigned long long)(Bc.out_pos + Bc.regen));
                }
            }
            ZB_BIGT(tg3 = zb_gtime(); if (bi >= 2000 && bi < 2024) printf("[blk %llu] start %llu  setup %llu  matches done +%llu  published +%llu  (abs publish %llu) nseq %u sweeps(warp0) %u\n", bi, tg0 % 100000000ull, tg1 - tg0, tg2 - tg0, tg3 - tg0, tg3 % 100000000ull, blocks[bi].n_seq, n_sweeps);)
        }
    }
}

// ===========================================================================
// K4 (pointer-jumping variant): FEW frames of very many blocks -- one huge frame at the limit (BASELINE config 5).  Copy-
// execute is a dependency chain: a match copies bytes that earlier matches produced (on text ~60 dependent hops inside a
// 128 KiB block, and the chains run on through the whole frame), so executing the blocks of one frame in order -- however
// many threads work on a block -- is bound by that chain (measured: 0.3-0.4 ms per block whatever the mapping).  Here the
// chain is not followed, it is SHORTENED: every output byte gets a source pointer, pointer doubling makes every byte point
// at the byte that first held its value (a literal, or a dictionary byte), one gather finishes the frame:
//   zb_chase_init    a thread per sequence: literal bytes are written to dst and point at themselves (DONE); match byte p
//                    points at p - offset (bytes that come from the dictionary are written at once and are DONE)
//   zb_chase_round   ptr[p] = ptr[ptr[p]] for every byte that is not DONE; DONE propagates; the host stops when a round
//                    changes nothing: ceil(log2(longest chain)) rounds, each a streaming pass plus one gather per open byte
//   zb_chase_gather  dst[p] = dst[ptr[p]]
// All three are embarrassingly parallel over the whole frame.  The price is a pointer per output byte (4 bytes below
// 2 GiB of output, 8 beyond) and ~10 passes over it.
// ===========================================================================
template <typename P> __device__ __forceinline__ P zb_chase_done() { return (P)1 << (sizeof(P) * 8 - 1); }

template <typename P>
__global__ void __launch_bounds__(256)
zb_chase_init(const u8* __restrict__ src, const ZbFramePlace* __restrict__ place, const u32* __restrict__ status,
              const ZbBlock* __restrict__ blocks, const ZbBlkDesc* __restrict__ bdesc, const ZbSeq* __restrict__ seqs,
              const u8* __restrict__ lits, u8* __restrict__ dst, P* __restrict__ ptr, u64 blk_first, u64 blk_last, ZbDictDev dict,
              bool chain = false)
{
    P const DONE = zb_chase_done<P>();
    u32 const tid = threadIdx.x, lane = tid & 31;
    const u8* const dict_end = dict.content + dict.content_size;
    for (u64 bi = blk_first + blockIdx.x; bi < blk_last; bi += gridDim.x) {
        u32 const f = bdesc[bi].frame;
        if (status[f] != ZB_OK) continue;
        ZbFramePlace const pl = place[f];
        ZbBlock const B = blocks[bi];
        u64 const gbase = pl.dst_off + B.out_pos;           // position of the block's first byte in dst
        u8* const gout = dst + gbase; P* const gp = ptr + gbase;
        if (B.kind == ZB_BLK_RAW) { const u8* q = src + B.src_pos; for (u32 i = tid; i < B.regen; i += 256) { gout[i] = q[i]; gp[i] = (P)(gbase + i) | DONE; } continue; }
        if (B.kind == ZB_BLK_RLE) { for (u32 i = tid; i < B.regen; i += 256) { gout[i] = (u8)B.lit_byte; gp[i] = (P)(gbase + i) | DONE; } continue; }
        if (B.kind != ZB_BLK_COMPRESSED) continue;
        bool const lit_rle = B.lit_kind == ZB_LIT_RLE; u8 const lit_byte = (u8)B.lit_byte;
        const u8* const lit = B.lit_kind == ZB_LIT_RAW ? src + B.src_pos : lits + B.src_pos;
        const ZbSeq* const sq = seqs + B.seq_pos;
        u32 const nseq = B.n_seq;
        // sources below fstart come from the dictionary; in chain mode the previous frame's output (the carried prefix in
        // front of frame 0) is part of dst, so they are pointed at like any other byte
        long long const fstart = chain ? (f ? (long long)place[f - 1].dst_off : 0ll) : (long long)pl.dst_off;
        for (u32 g = 0; g < nseq; g += 256) {
            u32 const i = g + tid; bool const valid = i < nseq;
            ZbSeq r = make_uint4(0, 0, 0, 0); u32 nx = 0;
            if (valid) { r = sq[i]; nx = sq[i + 1].x; }
            u32 const ll = nx - r.x, ml = r.z, off = r.w, m = r.y + ll;
            for (u32 k = 0; k < ll; k++) { gout[r.y + k] = lit_rle ? lit_byte : lit[r.x + k]; gp[r.y + k] = (P)(gbase + r.y + k) | DONE; }
            u32 big = __ballot_sync(0xFFFFFFFFu, valid && ml >= 128);
            if (valid && ml < 128) {
                for (u32 k = 0; k < ml; k++) {
                    long long const pos = (long long)(gbase + m + k), sp = pos - (long long)off;
                    if (sp >= fstart) gp[m + k] = (P)sp;
                    else { gout[m + k] = dict_end[sp - fstart]; gp[m + k] = (P)pos | DONE; }
                }
            }
            while (big) {          // long matches: the whole warp writes the pointers
                int const l = __ffs((int)big) - 1; big &= big - 1;
                u32 const m0 = __shfl_sync(0xFFFFFFFFu, m, l), len = __shfl_sync(0xFFFFFFFFu, ml, l), o = __shfl_sync(0xFFFFFFFFu, off, l);
                for (u32 k = lane; k < len; k += 32) {
                    long long const pos = (long long)(gbase + m0 + k), sp = pos - (long long)o;
                    if (sp >= fstart) gp[m0 + k] = (P)sp;
                    else { gout[m0 + k] = dict_end[sp - fstart]; gp[m0 + k] = (P)pos | DONE; }
                }
            }
        }
        {   // last literals of the block
            ZbSeq const e = sq[nseq];
            u32 const tail = B.n_lit - e.x;
            for (u32 k = tid; k < tail; k += 256) { gout[e.y + k] = lit_rle ? lit_byte : lit[e.x + k]; gp[e.y + k] = (P)(gbase + e.y + k) | DONE; }
        }
    }
}

// chain mode: the carried prefix in front of frame 0 (place[0].dst_off bytes) is final; its bytes are their own sources
template <typename P>
__global__ void __launch_bounds__(256)
zb_chase_prefix(const ZbFramePlace* __restrict__ place, P* __restrict__ ptr)
{
    u64 const carry = place[0].dst_off, stride = (u64)gridDim.x * 256;
    for (u64 p = (u64)blockIdx.x * 256 + threadIdx.x; p < carry; p += stride) ptr[p] = (P)p | zb_chase_done<P>();
}

// one round of pointer doubling over [lo, hi).  Racing updates are harmless: whatever a thread reads from ptr[q] is an ancestor
// of q (or q's final source), so it is one of p, too.
template <typename P>
__global__ void __launch_bounds__(256)
zb_chase_round(P* __restrict__ ptr, u64 lo, u64 hi, u32* __restrict__ changed)
{
    P const DONE = zb_chase_done<P>();
    bool ch = false;
    u64 const stride = (u64)gridDim.x * 256;
    for (u64 p = lo + (u64)blockIdx.x * 256 + threadIdx.x; p < hi; p += stride) {
        P const v = ptr[p];
        if (v & DONE) continue;
        P const w = __ldcg(ptr + v);
        ptr[p] = w;
        if (!(w & DONE)) ch = true;
    }
    if (__syncthreads_or(ch ? 1 : 0) && threadIdx.x == 0) *changed = 1;
}

template <typename P>
__global__ void __launch_bounds__(256)
zb_chase_gather(const P* __restrict__ ptr, u8* dst, u64 lo, u64 hi, u64 n_total)
{
    P const DONE = zb_chase_done<P>();
    u64 const stride = (u64)gridDim.x * 256;
    for (u64 p = lo + (u64)blockIdx.x * 256 + threadIdx.x; p < hi; p += stride) {
        P const t = ptr[p] & ~DONE;
        if ((u64)t != p && (u64)t < n_total) dst[p] = __ldcg(dst + t);
    }
}

// ===========================================================================
__device__ static u64 zb_xxh64(const u8* p, u64 len)
{
    u64 const P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull, P4 = 0x85EBCA77C2B2AE63ull, P5 = 0x27D4EB2F165667C5ull;
    auto rotl = [](u64 x, int r) { return (x << r) | (x >> (64 - r)); };
    auto round = [&](u64 acc, u64 in) { return rotl(acc + in * P2, 31) * P1; };
    const u8* const end = p + len; u64 h;
    if (len >= 32) {
        u64 v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0 - P1;
        do { v1 = round(v1, zb_rd64(p)); v2 = round(v2, zb_rd64(p + 8)); v3 = round(v3, zb_rd64(p + 16)); v4 = round(v4, zb_rd64(p + 24)); p += 32; } while (p + 32 <= end);
        h = rotl(v1, 1) + rotl(v2, 7) + rotl(v3, 12) + rotl(v4, 18);
        h = (h ^ round(0, v1)) * P1 + P4; h = (h ^ round(0, v2)) * P1 + P4; h = (h ^ round(0, v3)) * P1 + P4; h = (h ^ round(0, v4)) * P1 + P4;
    } else h = P5;
    h += len;
    while (p + 8 <= end) { h ^= round(0, zb_rd64(p)); h = rotl(h, 27) * P1 + P4; p += 8; }
    if (p + 4 <= end) { h ^= (u64)zb_rd32(p) * P1; h = rotl(h, 23) * P2 + P3; p += 4; }
    while (p < end) { h ^= (*p++) * P5; h = rotl(h, 11) * P1; }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

// Frames of ZB_XXH_BIG bytes and more are not hashed by a single lane (byte loads from global memory, one frame = one chain):
// zb_verify_checksums_big gives each a CTA.
#ifndef ZB_XXH_BIG
#define ZB_XXH_BIG (256u << 10)
#endif
#define ZB_XXH_TILE 16384u               // bytes per shared-memory tile (two tiles)

__global__ void zb_verify_checksums(const u8* __restrict__ dst, const ZbFramePlace* __restrict__ place, const u64* __restrict__ out_sizes,
                                    const ZbFrameInfo* __restrict__ info, const u32* __restrict__ ck_expect, u32 first, u32 n_frames,
                                    u32* __restrict__ status)
{
    u32 const f = first + blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    if (status[f] != ZB_OK || !(info[f].flags & 1)) return;
    if (out_sizes[f] >= ZB_XXH_BIG) return;                            // zb_verify_checksums_big's
    u64 const h = zb_xxh64(dst + place[f].dst_off, out_sizes[f]);
    if ((u32)h != ck_expect[f]) status[f] = ZB_E_CHECKSUM_WRONG;
}

// XXH64 of one large frame per CTA (zstd/zstd.c:44260-44277 over XXH64_update's stripe loop).  The four accumulators are
// four serial chains -- 64-bit add, rotate, 64-bit multiply per 32-byte stripe, ~27 cycles of dependent latency, no algebra
// gets around the rotate -- so a frame hashes at ~2 GB/s however many threads there are; the kernel only makes sure NOTHING
// ELSE sits on those chains: threads 32-255 stage the next 16 KiB tile in shared memory, realigned to the frame's start
// (two 32-bit loads and a funnel shift per word), while lanes 0-3 of warp 0 consume the current one with one aligned
// 64-bit read per stripe, the products in * P2 of the next four stripes computed in the shadow of the current four rounds.
__global__ void __launch_bounds__(256)
zb_verify_checksums_big(const u8* __restrict__ dst, const ZbFramePlace* __restrict__ place, const u64* __restrict__ out_sizes,
                        const ZbFrameInfo* __restrict__ info, const u32* __restrict__ ck_expect, u32 first, u32 n_frames,
                        u32* __restrict__ status)
{
    __shared__ __align__(16) u32 s_tile[2][ZB_XXH_TILE / 4];
    __shared__ u64 s_v[4];
    u64 const P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull, P4 = 0x85EBCA77C2B2AE63ull;
    u32 const tid = threadIdx.x;
    #define ZB_XXH_ROUND(v, c) do { u64 const s_ = (v) + (c); (v) = ((s_ << 31) | (s_ >> 33)) * P1; } while (0)
    for (u32 f = first + blockIdx.x; f < n_frames; f += gridDim.x) {
        if (status[f] != ZB_OK || !(info[f].flags & 1)) continue;
        u64 const len = out_sizes[f];
        if (len < ZB_XXH_BIG) continue;
        const u8* const p0 = dst + place[f].dst_off;
        u64 const n_words = (len >> 5) * 8;                            // 32-bit words inside whole stripes
        u32 const sh = (u32)((uintptr_t)p0 & 3) * 8;
        const u32* const g32 = (const u32*)(p0 - (sh >> 3));           // aligned words; word j of the frame = funnel(g32[j], g32[j + 1])
        u64 const n_tiles = (n_words + ZB_XXH_TILE / 4 - 1) / (ZB_XXH_TILE / 4);
        u64 v = tid == 0 ? P1 + P2 : (tid == 1 ? P2 : (tid == 2 ? 0ull : 0ull - P1));
        __syncthreads();                                               // (the tiles are free)
        for (u64 t = 0; t <= n_tiles; t++) {
            if (tid >= 32 && t < n_tiles) {                            // stage tile t
                u64 const w0 = t * (ZB_XXH_TILE / 4);
                u32 const nw = (u32)(n_words - w0 < ZB_XXH_TILE / 4 ? n_words - w0 : ZB_XXH_TILE / 4);
                u32* const d = s_tile[t & 1];
                if (sh == 0) for (u32 i = tid - 32; i < nw; i += 224) d[i] = __ldcg(g32 + w0 + i);
                else for (u32 i = tid - 32; i < nw; i += 224) d[i] = __funnelshift_r(__ldcg(g32 + w0 + i), __ldcg(g32 + w0 + i + 1), sh);
            }
            if (tid < 4 && t > 0) {                                    // consume tile t - 1: stripe k of my accumulator = q[4 k]
                u64 const w0 = (t - 1) * (ZB_XXH_TILE / 4);
                u32 const ns = (u32)(n_words - w0 < ZB_XXH_TILE / 4 ? n_words - w0 : ZB_XXH_TILE / 4) >> 3;
                const u64* const q = (const u64*)s_tile[(t - 1) & 1] + tid;
                u32 k = 0;
                if (ns >= 4) {
                    u64 c0 = q[0] * P2, c1 = q[4] * P2, c2 = q[8] * P2, c3 = q[12] * P2;
                    for (; k + 8 <= ns; k += 4) {
                        u64 const n0 = q[(k + 4) * 4] * P2, n1 = q[(k + 5) * 4] * P2, n2 = q[(k + 6) * 4] * P2, n3 = q[(k + 7) * 4] * P2;
                        ZB_XXH_ROUND(v, c0); ZB_XXH_ROUND(v, c1); ZB_XXH_ROUND(v, c2); ZB_XXH_ROUND(v, c3);
                        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
                    }
                    ZB_XXH_ROUND(v, c0); ZB_XXH_ROUND(v, c1); ZB_XXH_ROUND(v, c2); ZB_XXH_ROUND(v, c3);
                    k += 4;
                }
                for (; k < ns; k++) { u64 const c = q[k * 4] * P2; ZB_XXH_ROUND(v, c); }
            }
            __syncthreads();
        }
        #undef ZB_XXH_ROUND
        u64 const n_stripes = len >> 5;
        // the four accumulators -> lane 0; the tail (< 32 bytes) and the avalanche as in zb_xxh64
        if (tid < 4) s_v[tid] = v;
        __syncthreads();
        if (tid == 0) {
            auto rotl = [](u64 x, int r) { return (x << r) | (x >> (64 - r)); };
            auto round = [&](u64 acc, u64 in) { return rotl(acc + in * P2, 31) * P1; };
            u64 const P5 = 0x27D4EB2F165667C5ull;
            u64 h = rotl(s_v[0], 1) + rotl(s_v[1], 7) + rotl(s_v[2], 12) + rotl(s_v[3], 18);
            h = (h ^ round(0, s_v[0])) * P1 + P4; h = (h ^ round(0, s_v[1])) * P1 + P4; h = (h ^ round(0, s_v[2])) * P1 + P4; h = (h ^ round(0, s_v[3])) * P1 + P4;
            h += len;
            const u8* p = p0 + n_stripes * 32; const u8* const end = p0 + len;
            while (p + 8 <= end) { h ^= round(0, zb_rd64(p)); h = rotl(h, 27) * P1 + P4; p += 8; }
            if (p + 4 <= end) { h ^= (u64)zb_rd32(p) * P1; h = rotl(h, 23) * P2 + P3; p += 4; }
            while (p < end) { h ^= (*p++) * P5; h = rotl(h, 11) * P1; }
            h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
            if ((u32)h != ck_expect[f]) status[f] = ZB_E_CHECKSUM_WRONG;
        }
        __syncthreads();
    }
}

// ===========================================================================
// K5: finish -- output segment table + lowest failing frame
// ===========================================================================
__global__ void zb_finish(const ZbFramePlace* __restrict__ place, const u64* __restrict__ out_sizes,
                          const u32* __restrict__ status, u32 n_frames, ZbSegment* __restrict__ out_segs,
                          u32* __restrict__ first_error)
{
    u32 f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    ZbSegment s; s.offset = place[f].dst_off; s.length = out_sizes[f];
    out_segs[f] = s;
    if (status[f] != ZB_OK) atomicMin(first_error, f);
}

// chain mode: the run's frames are placed behind the `carry` bytes of the prefix carried in from the previous run
__global__ void zb_chain_shift(ZbFramePlace* __restrict__ place, u32 n_entries, u64 carry)
{
    u32 const i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_entries) place[i].dst_off += carry;
}

// ===========================================================================
// dictionary digest -- one thread, once per dictionary
// (restates ZSTD_loadDEntropy zstd/zstd.c:44673-44757 and ZSTD_decompress_insertDictionary :44760)
// ===========================================================================
__global__ void zb_digest_dict(const u8* __restrict__ dict, u32 n, ZbDictDigest* __restrict__ out)
{
    if (threadIdx.x || blockIdx.x) return;
    out->status = ZB_OK; out->has_entropy = 0; out->dict_id = 0; out->content_off = 0;
    if (n < 8 || zb_rd32(dict) != ZB_MAGIC_DICT) return;            // raw-content dictionary
    out->dict_id = zb_rd32(dict + 4);
    const u8* p = dict + 8; const u8* const end = dict + n;
    {
        __align__(16) u8 ws[256]; ZbRank rank; u32 log, nsym;
#ifdef __CUDA_ARCH__
        __shared__ __align__(16) u8 ring[64];
#else
        u8* const ring = nullptr;
#endif
        u32 const used = zb_huf_weights(ws, p, (u32)(end - p), log, nsym, rank, ring);
        if (!used) { out->status = ZB_E_DICT_CORRUPTED; return; }
        zb_huf_fill(out->huf, ws, log, nsym, rank, 0, 0);          // the digest keeps the full table (read in place from global memory)
        out->huf_log = log; p += used;
        u32 mxs = 0;
        for (u32 i = 0; i < 256; i++) {
            u32 const wt = i < nsym ? (ws[i >> 1] >> ((i & 1) * 4)) & 15 : 0;
            out->c_huf_nb[i] = wt ? (u8)(log + 1 - wt) : 0; if (wt) mxs = i;
        }
        out->c_huf_max = mxs;
    }
    short norm[64]; u32 mx, log, used;
    mx = 31; used = zb_read_ncount(norm, mx, log, p, (u32)(end - p));
    if (!used || log > 8) { out->status = ZB_E_DICT_CORRUPTED; return; }
    for (u32 i = 0; i < 32; i++) out->c_norm_of[i] = i <= mx ? norm[i] : 0; out->c_max_of = mx;      // before zb_build_fse: it consumes norm
    zb_build_fse(out->of, norm, mx, log, K_OF); out->of_log = log; p += used;
    mx = 52; used = zb_read_ncount(norm, mx, log, p, (u32)(end - p));
    if (!used || log > 9) { out->status = ZB_E_DICT_CORRUPTED; return; }
    for (u32 i = 0; i < 54; i++) out->c_norm_ml[i] = i <= mx ? norm[i] : 0; out->c_max_ml = mx;      // before zb_build_fse: it consumes norm
    zb_build_fse(out->ml, norm, mx, log, K_ML); out->ml_log = log; p += used;
    mx = 35; used = zb_read_ncount(norm, mx, log, p, (u32)(end - p));
    if (!used || log > 9) { out->status = ZB_E_DICT_CORRUPTED; return; }
    for (u32 i = 0; i < 36; i++) out->c_norm_ll[i] = i <= mx ? norm[i] : 0; out->c_max_ll = mx;      // before zb_build_fse: it consumes norm
    zb_build_fse(out->ll, norm, mx, log, K_LL); out->ll_log = log; p += used;
    if (p + 12 > end) { out->status = ZB_E_DICT_CORRUPTED; return; }
    u32 const content = (u32)(end - (p + 12));
    for (int i = 0; i < 3; i++) {
        u32 r = zb_rd32(p + 4 * i);
        if (r == 0 || r > content) { out->status = ZB_E_DICT_CORRUPTED; return; }
        out->rep[i] = r;
    }
    out->content_off = (u32)(p + 12 - dict);
    out->has_entropy = 1;
}

// ===========================================================================
// host-side launchers (called from zb_api.cu)
// ===========================================================================
extern "C" {

void zb_launch_default_tables(cudaStream_t st) { ZB_LAUNCH(zb_build_default_tables, 1, 32, 0, st); }

void zb_launch_scan(const u8* src, const ZbSegment* segs, u32 n, ZbFrameInfo* info, u64 window_limit, u32* big_list, cudaStream_t st)
{
    // big_list: n + 1 words; [0] = number of frames left to zb_scan_frames_big
    cudaMemsetAsync(big_list, 0, sizeof(u32), st);
    ZB_LAUNCH(zb_scan_frames, (n + 127) / 128, 128, 0, st, src, segs, n, info, window_limit, big_list);
    ZB_LAUNCH(zb_scan_frames_big, n < 128 ? (n + 3) / 4 : 32, 128, 0, st, src, segs, big_list, info);
}

void zb_launch_scan_blocks(const u8* src, const ZbSegment* segs, u32 n, const ZbFramePlace* place, ZbDictDev dict, u32* status,
                           void* bdesc, u64* frame_end, const u32* big_list, cudaStream_t st)
{
    ZB_LAUNCH(zb_scan_blocks, (n + 63) / 64, 64, 0, st, src, segs, n, place, dict, status, (ZbBlkDesc*)bdesc, frame_end, big_list);
    ZB_LAUNCH(zb_scan_blocks_big, n < 128 ? (n + 3) / 4 : 32, 128, 0, st, src, segs, big_list, place, dict, status, (ZbBlkDesc*)bdesc, frame_end);
}
void zb_launch_entropy_blocks(const u8* src, const void* bdesc, u32 n_blocks, ZbBlock* blocks, ZbSeq* seqs, u8* lits, u32 n_ctas, u32* work_counter,
                              ZbDictDev dict, u32* status, void* bexit, u32 take, cudaStream_t st)
{
    ZB_LAUNCH(zb_entropy_blocks<7>, n_ctas, 7 * 32, ZB_ENT_SMEM(7), st, src, (const ZbBlkDesc*)bdesc, n_blocks, blocks, seqs, lits, work_counter, dict,
              status, (ZbBlkExit*)bexit, take);
}
void zb_launch_resolve_blocks(const u8* src, const ZbSegment* segs, u32 n, const ZbFramePlace* place, const ZbFrameInfo* info, const u64* dst_sizes,
                              ZbBlock* blocks, const void* bdesc, const void* bexit, const u64* frame_end, u64 n_blocks, ZbSeq* seqs, ZbDictDev dict,
                              u32* status, u64* out_sizes, u32* ck_expect, u32* entry_rep, cudaStream_t st, int chain)
{
    ZB_LAUNCH(zb_resolve_blocks, (n + 63) / 64, 64, 0, st, src, segs, n, place, info, dst_sizes, blocks, (const ZbBlkDesc*)bdesc, (const ZbBlkExit*)bexit,
              frame_end, dict, status, out_sizes, ck_expect, entry_rep);
    if (n_blocks) ZB_LAUNCH(zb_patch_blocks, (unsigned)((n_blocks + 7) / 8), 256, 0, st, blocks, (const ZbBlkDesc*)bdesc, n_blocks, seqs, entry_rep, dict,
                            status, chain ? place : nullptr);
}
size_t zb_blkdesc_bytes() { return sizeof(ZbBlkDesc); }
size_t zb_blkexit_bytes() { return sizeof(ZbBlkExit); }

void zb_launch_place(const ZbFrameInfo* info, const u64* dst_sizes, u32 n, ZbFramePlace* place, u64* totals,
                     u32* status, u64* partial, cudaStream_t st)
{
    u32 const ctas = (n + ZB_PLACE_CTA - 1) / ZB_PLACE_CTA;
    ZB_LAUNCH(zb_place_reduce, ctas, ZB_PLACE_CTA, 0, st, info, dst_sizes, n, partial);
    ZB_LAUNCH(zb_place_scan, ctas, ZB_PLACE_CTA, 0, st, info, dst_sizes, n, partial, place, totals, status);
}

void zb_launch_entropy(const u8* src, const ZbSegment* segs, u32 n, const ZbFramePlace* place, const u64* dst_sizes,
                       ZbBlock* blocks, ZbSeq* seqs, u8* lits, u32 n_ctas, u32* work_counter,
                       ZbDictDev dict, u32* status, u64* out_sizes, u32* ck_expect, u32 take, u32 warps, cudaStream_t st)
{
    // persistent grid: one CTA of `warps` (7 or 8) warps per SM, each warp with its own shared-memory table pool
    if (warps == 8) ZB_LAUNCH(zb_entropy_decode<8>, n_ctas, 8 * 32, ZB_ENT_SMEM(8), st, src, segs, n, place, dst_sizes, blocks, seqs, lits,
                              work_counter, dict, status, out_sizes, ck_expect, take);
    else ZB_LAUNCH(zb_entropy_decode<7>, n_ctas, 7 * 32, ZB_ENT_SMEM(7), st, src, segs, n, place, dst_sizes, blocks, seqs, lits,
                   work_counter, dict, status, out_sizes, ck_expect, take);
}

// the pointer-jumping execute stage over the blocks [blk_first, blk_last) whose output is dst[lo, hi).  ptr_mem: (n_total + 16)
// pointers of 4 bytes (n_total < 2^31) or 8.  Returns the number of doubling rounds, or -1 on a CUDA error.
size_t zb_chase_bytes(u64 n_total) { return (size_t)((n_total + 16) * (n_total < (1ull << 31) ? 4 : 8)); }

extern "C++" {
template <typename P>
static int zb_chase_run(const u8* src, const ZbFramePlace* place, const u32* status, const ZbBlock* blocks, const void* bdesc,
                        const ZbSeq* seqs, const u8* lits, u8* dst, u64 lo, u64 hi, u64 n_total, u64 blk_first, u64 blk_last,
                        void* ptr_mem, u32* d_changed, u32 n_ctas, ZbDictDev dict, cudaStream_t st, bool chain)
{
    P* const ptr = (P*)ptr_mem;
    if (hi <= lo || blk_last <= blk_first) return 0;
    if (cudaMemsetAsync(ptr + lo, 0xFF, (hi - lo) * sizeof(P), st) != cudaSuccess) return -1;      // frames that failed stay "done, no source"
    u64 const nb = blk_last - blk_first;
    if (chain) ZB_LAUNCH(zb_chase_prefix<P>, n_ctas * 4, 256, 0, st, place, ptr);
    ZB_LAUNCH(zb_chase_init<P>, (unsigned)(nb < n_ctas * 8ull ? nb : n_ctas * 8ull), 256, 0, st, src, place, status, blocks, (const ZbBlkDesc*)bdesc, seqs,
              lits, dst, ptr, blk_first, blk_last, dict, chain);
    u64 const want = (hi - lo + 255) / 256;
    unsigned const grid = (unsigned)(want < n_ctas * 16ull ? want : n_ctas * 16ull);
    int rounds = 0;
    for (; rounds < 72; rounds++) {
        u32 h = 0;
        if (cudaMemsetAsync(d_changed, 0, sizeof(u32), st) != cudaSuccess) return -1;
        ZB_LAUNCH(zb_chase_round<P>, grid, 256, 0, st, ptr, lo, hi, d_changed);
        if (cudaMemcpyAsync(&h, d_changed, sizeof(u32), cudaMemcpyDeviceToHost, st) != cudaSuccess) return -1;
        if (cudaStreamSynchronize(st) != cudaSuccess) return -1;
        if (!h) { rounds++; break; }
    }
    ZB_LAUNCH(zb_chase_gather<P>, grid, 256, 0, st, ptr, dst, lo, hi, n_total);
    return rounds;
}
}

int zb_launch_execute_chase(const u8* src, const ZbFramePlace* place, const u32* status, const ZbBlock* blocks, const void* bdesc,
                            const ZbSeq* seqs, const u8* lits, u8* dst, u64 lo, u64 hi, u64 n_total, u64 blk_first, u64 blk_last,
                            void* ptr_mem, u32* d_changed, u32 n_ctas, ZbDictDev dict, cudaStream_t st, int chain)
{
    if (n_total < (1ull << 31)) return zb_chase_run<u32>(src, place, status, blocks, bdesc, seqs, lits, dst, lo, hi, n_total, blk_first, blk_last, ptr_mem, d_changed, n_ctas, dict, st, chain != 0);
    return zb_chase_run<u64>(src, place, status, blocks, bdesc, seqs, lits, dst, lo, hi, n_total, blk_first, blk_last, ptr_mem, d_changed, n_ctas, dict, st, chain != 0);
}

size_t zb_wave_bytes(u64 n_frames, u64 n_blocks) { return (size_t)(n_frames * 12 + n_blocks * 4 + 64); }

void zb_launch_execute_big(const u8* src, const ZbFramePlace* place, const u32* status, const ZbBlock* blocks, const void* bdesc,
                           const ZbSeq* seqs, const u8* lits, u8* dst, u32 first, u32 end, u64 blk_first, u64 blk_last,
                           u64 n_frames, u64 n_blocks, void* wave_mem, u32 n_ctas, ZbDictDev dict, cudaStream_t st)
{
    // the block-parallel path: few frames of many blocks.  Small frames as always; the blocks of the others are taken in
    // order by a persistent grid (16 warps and 219 KB of shared memory per CTA, one CTA per SM)
    u32 const n = end - first;
    ZB_LAUNCH(zb_execute_tile, (n + ZB_TILE_WARPS - 1) / ZB_TILE_WARPS, ZB_TILE_WARPS * 32, ZB_TILE_SMEM, st, src, place, status, blocks,
              seqs, lits, dst, first, end, dict);
    if (blk_last <= blk_first) return;
    cudaMemsetAsync(wave_mem, 0, zb_wave_bytes(n_frames, n_blocks), st);
    ZbWave w;
    w.done_pos = (unsigned long long*)wave_mem;
    w.pre_blk = (u32*)(w.done_pos + n_frames);
    w.blk_flag = w.pre_blk + n_frames;
    w.ticket = w.blk_flag + n_blocks;
    u64 grid = blk_last - blk_first; if (grid > n_ctas) grid = n_ctas;
    ZB_LAUNCH(zb_execute_big, (unsigned)grid, ZB_BIG_NT, ZB_BIG_SMEM, st, src, place, status, blocks, (const ZbBlkDesc*)bdesc, seqs, lits, dst,
              blk_first, blk_last, dict, (u64)ZB_TILE_CAP + 1, w);
}

void zb_launch_execute(const u8* src, const ZbFramePlace* place, const u32* status, const ZbBlock* blocks,
                       const ZbSeq* seqs, const u8* lits, u8* dst, u32 first, u32 end, ZbDictDev dict, cudaStream_t st)
{
    // frames [first, end).  Frames <= ZB_TILE_CAP bytes are regenerated in shared memory, larger ones straight in HBM/L2
    u32 const n = end - first;
    ZB_LAUNCH(zb_execute_tile, (n + ZB_TILE_WARPS - 1) / ZB_TILE_WARPS, ZB_TILE_WARPS * 32, ZB_TILE_SMEM, st, src, place, status, blocks,
              seqs, lits, dst, first, end, dict);
    u32 const warps_per_cta = 8;
    ZB_LAUNCH(zb_execute, (n + warps_per_cta - 1) / warps_per_cta, warps_per_cta * 32, 0, st, src, place, status, blocks, seqs,
              lits, dst, first, end, dict, (u64)ZB_TILE_CAP + 1);
}

void zb_launch_verify(const u8* dst, const ZbFramePlace* place, const u64* out_sizes, const ZbFrameInfo* info, const u32* ck_expect,
                      u32 first, u32 end, u32* status, cudaStream_t st)
{
    u32 const n = end - first;
    ZB_LAUNCH(zb_verify_checksums, (n + 127) / 128, 128, 0, st, dst, place, out_sizes, info, ck_expect, first, end, status);
    ZB_LAUNCH(zb_verify_checksums_big, n < 592 ? n : 592, 256, 0, st, dst, place, out_sizes, info, ck_expect, first, end, status);
}

void zb_launch_finish(const ZbFramePlace* place, const u64* out_sizes, const u32* status, u32 n, ZbSegment* out_segs,
                      u32* first_error, cudaStream_t st)
{
    ZB_LAUNCH(zb_finish, (n + 255) / 256, 256, 0, st, place, out_sizes, status, n, out_segs, first_error);
}

void zb_launch_chain_shift(ZbFramePlace* place, u32 n, u64 carry, cudaStream_t st)
{
    ZB_LAUNCH(zb_chain_shift, (n + 1 + 255) / 256, 256, 0, st, place, n + 1, carry);
}

void zb_entropy_phase_read(unsigned long long* out8, int reset)
{
#ifdef ZB_PHASE_TIMERS
    cudaMemcpyFromSymbol(out8, g_zb_ent_phase, sizeof(unsigned long long) * 8);
    if (reset) { unsigned long long z[8] = {0}; cudaMemcpyToSymbol(g_zb_ent_phase, z, sizeof z); }
#else
    for (int i = 0; i < 8; i++) out8[i] = 0; (void)reset;
#endif
}

void zb_execute_phase_read(unsigned long long* out4, int reset)
{
#ifdef ZB_PHASE_TIMERS
    cudaMemcpyFromSymbol(out4, g_zb_exe_phase, sizeof(unsigned long long) * 4);
    if (reset) { unsigned long long z[4] = {0}; cudaMemcpyToSymbol(g_zb_exe_phase, z, sizeof z); }
#else
    for (int i = 0; i < 4; i++) out4[i] = 0; (void)reset;
#endif
}

void zb_launch_digest_dict(const u8* dict, u32 n, ZbDictDigest* out, cudaStream_t st)
{
    ZB_LAUNCH(zb_digest_dict, 1, 32, 0, st, dict, n, out);
}

}  // extern "C"
