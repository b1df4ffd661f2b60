// simt_kernels.cpp -- the CPU build of the whole kernel source (test infrastructure, not product code).
//
// zb_decode.cu and zb_encode.cu (with zb_encode2.cuh, zb_encode3.cuh and zb_train.cuh) compile here as they are, launchers
// included, on the SIMT runtime of simt.h; tests/host_encoder.py builds this file with ZB_SIMT_EMULATION.  The wrappers
// below call the kernels' serial helpers by name, and call the launchers in the order zb_api.cu calls them and plan with the
// host functions of zb_common.cuh, on the SM counts, warps and frames per warp that the tests choose.  The CPU suite loads
// them over ctypes; it has no other build of the kernel source.
#include "simt.h"
#include "zb_decode.cu"
#include "zb_encode.cu"
#include <vector>

namespace {
std::vector<ZbSegment> t_segments(const u64* off, const u64* len, u32 n)
{
    std::vector<ZbSegment> segs(n);
    for (u32 i = 0; i < n; i++) { segs[i].offset = off[i]; segs[i].length = len[i]; }
    return segs;
}
struct TBuf {            // 64-byte aligned scratch
    void* p;
    explicit TBuf(size_t n) : p(aligned_alloc(64, (n + 63) & ~(size_t)63)) {}
    ~TBuf() { free(p); }
};

// zb_launch_frame_layout + zb_launch_write_frames over the segments' block outputs: the frames' total bytes, -1 when they do
// not fit out_cap
long long t_layout(const u8* src, const std::vector<ZbSegment>& segs, const std::vector<ZeSegInfo>& info, const ZeBlockOut* outs,
                   const u8* slots, u64 slot_bytes, u32 checksum, u32 content_size, u32 dict_id, u32 window_log,
                   u8* out, u64 out_cap, u64* out_off, u64* out_len)
{
    u32 const n = (u32)segs.size();
    std::vector<u64> sizes(n); std::vector<ZbSegment> out_segs(n); u64 total = 0;
    zb_launch_frame_layout(segs.data(), info.data(), outs, n, checksum, content_size, dict_id, window_log, sizes.data(), out_segs.data(), &total, 0);
    if (total > out_cap) return -1;
    zb_launch_write_frames(src, segs.data(), info.data(), outs, slots, slot_bytes, n, checksum, content_size, dict_id, window_log, out_segs.data(), out, 0);
    for (u32 i = 0; i < n; i++) { out_off[i] = out_segs[i].offset; out_len[i] = out_segs[i].length; }
    return (long long)total;
}

// the frame scans and the placement that start every batch decode (run_decompress)
struct TScan {
    std::vector<ZbSegment> segs; std::vector<ZbFrameInfo> info; std::vector<ZbFramePlace> place;
    std::vector<u32> status, big; std::vector<u64> partial; u64 totals[8] = {0};
    TScan(const u8* src, const u64* off, const u64* len, u32 n, const u64* dst_sizes)
        : segs(t_segments(off, len, n)), info(n), place(n + 1), status(n, 0), big(n + 1, 0),
          partial(((n + ZB_PLACE_CTA - 1) / ZB_PLACE_CTA) * 4 + 4)
    {
        // big: frames above ZB_SCAN_BIG (24 KB in this build) are scanned by a warp each
        zb_launch_scan(src, segs.data(), n, info.data(), (1ull << 27) + 1, big.data(), 0);
        zb_launch_place(info.data(), dst_sizes, n, place.data(), totals, status.data(), partial.data(), 0);
    }
};

// the decode kernels' view of a dictionary: zb_launch_digest_dict into dg, and dict pointing into it (empty without a
// dictionary).  Returns the digest's status.
u32 t_dict_dev(const u8* dict_raw, u32 dict_n, ZbDictDigest& dg, ZbDictDev& dict)
{
    memset(&dict, 0, sizeof dict);
    if (!dict_raw || !dict_n) return ZB_OK;
    zb_launch_digest_dict(dict_raw, dict_n, &dg, 0);
    if (dg.status != ZB_OK) return dg.status;
    if (dg.has_entropy) {
        dict.content = dict_raw + dg.content_off; dict.content_size = dict_n - dg.content_off; dict.dict_id = dg.dict_id; dict.has_entropy = 1;
        dict.huf = dg.huf; dict.huf_log = dg.huf_log; dict.ll = dg.ll; dict.of = dg.of; dict.ml = dg.ml;
        dict.ll_log = dg.ll_log; dict.of_log = dg.of_log; dict.ml_log = dg.ml_log;
        dict.rep[0] = dg.rep[0]; dict.rep[1] = dg.rep[1]; dict.rep[2] = dg.rep[2];
    } else { dict.content = dict_raw; dict.content_size = dict_n; }
    return ZB_OK;
}
}  // namespace

extern "C" unsigned long long t_any_calls(int reset) { unsigned long long v = simt_any_calls; if (reset) simt_any_calls = 0; return v; }

// ---- the serial helpers of the kernels: entropy tables, headers, literals.  None of them reaches a warp collective, a
// barrier or shared state, so they are called directly, outside any launch.
extern "C" {
// encoder (zb_encode.cu)
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
u32 t_frame_header(u8* o, u64 size, u32 checksum, u32 content_size, u32 dict_id)
{
    ZeParams P; P.checksum = checksum; P.content_size = content_size; P.dict_id = dict_id; P.level = 3;
    return ze_frame_header(o, size, P);
}

// decoder (zb_decode.cu, zb_entropy.cuh)
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
// out[6] = {content_size, window, dict_id, hdr_size, checksum, status}
void t_parse_header(const u8* s, u64 n, u64* out)
{
    ZbHdr h; zb_parse_header(s, n, h);
    out[0] = h.content_size; out[1] = h.window; out[2] = h.dict_id; out[3] = h.hdr_size; out[4] = h.checksum; out[5] = h.status;
}
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

// ---- compression
// The whole compression path of the library: block jobs cut as zb_api.cu cuts them (zb_cut_blocks, blocks of
// min(2^window_log, 128 KiB)), zb_launch_compress_blocks on `n_ctas` CTAs -- or zb_launch_compress_recs when `recs` is set --
// then the frame layout with the level and window_log of the call.  Input resident.  Returns total bytes.
extern "C" long long t_compress_batch(const u8* src, const u64* seg_off, const u64* seg_len, u32 n_segs, u32 checksum, u32 content_size,
                                      u32 n_ctas, u8* out, u64 out_cap, u64* out_off, u64* out_len, u32 recs, const u8* dict_raw, u32 dict_n,
                                      int level, u32 window_log)
{
    std::vector<ZbSegment> segs = t_segments(seg_off, seg_len, n_segs); std::vector<ZeBlockJob> jobs; std::vector<ZeSegInfo> info(n_segs);
    u32 const max_block = zb_cut_blocks(segs.data(), n_segs, zb_block_max(window_log), jobs, info);
    u32 const nj = (u32)jobs.size();
    u64 const slot_bytes = zb_slot_bytes(max_block);
    std::vector<u8> slots((size_t)(nj + 1) * slot_bytes); std::vector<ZeBlockOut> outs(nj + 1);
    if (n_ctas > nj) n_ctas = nj ? nj : 1;
    // what zb200_ddict_create does: digest, compression view, its hash table, the CTables of its entropy tables
    static ZbDictDigest dg; static u16 dtable[1 << ZE_HLOG]; static ZeCTable cct[3];
    ZbDictView view = {nullptr, 0};
    u32 dict_id = 0;
    if (dict_raw && dict_n) {
        zb_launch_digest_dict(dict_raw, dict_n, &dg, 0);
        if (dg.status != ZB_OK) return -2;
        view = dg.has_entropy ? zb_dict_view(dict_raw + dg.content_off, dict_n - dg.content_off) : zb_dict_view(dict_raw, dict_n);
        if (view.D) {
            dict_id = dg.dict_id;
            zb_launch_dict_table(view.tail, view.D, dtable, 0);
            if (dg.has_entropy) zb_launch_dict_ctables(&dg, cct, 0);
        }
    }
    const u16* const table = view.D ? dtable : nullptr;
    const void* const digest = view.D && dg.has_entropy ? &dg : nullptr;
    const void* const ccts = digest ? cct : nullptr;
    TBuf scratch(zb_encode_scratch_bytes() * n_ctas);
    u32 counter = 0;
    if (nj && recs) {
        u32 const need = (nj + zb_encode3_records_per_cta() - 1) / zb_encode3_records_per_cta();
        zb_launch_compress_recs(src, jobs.data(), nj, need < n_ctas ? need : n_ctas, slots.data(), slot_bytes, outs.data(), &counter,
                                view.tail, view.D, table, digest, ccts, nullptr, 0, nullptr, 0);
    }
    else if (nj) zb_launch_compress_blocks(src, jobs.data(), nj, scratch.p, n_ctas, slots.data(), slot_bytes, outs.data(), &counter,
                                           view.tail, view.D, table, digest, ccts, nullptr, 0, nullptr, level >= 4,
                                           max_block <= zb_encode_small_max(), 0, nullptr);
    return t_layout(src, segs, info, outs.data(), slots.data(), slot_bytes, checksum, content_size, dict_id, window_log, out, out_cap, out_off, out_len);
}

// The round-2 kernel (zb_compress_smem: one CTA of 1024 threads per block, block resident in "shared memory") with the
// jobs and frame headers of a call with this level and window_log.
extern "C" long long t_compress_batch2(const u8* src, const u64* seg_off, const u64* seg_len, u32 n_segs, u32 checksum, u32 content_size,
                                       u32 n_ctas, u8* out, u64 out_cap, u64* out_off, u64* out_len, int level, u32 window_log)
{
    (void)level;         // the frame layout does not depend on it
    std::vector<ZbSegment> segs = t_segments(seg_off, seg_len, n_segs); std::vector<ZeBlockJob> jobs; std::vector<ZeSegInfo> info(n_segs);
    u32 const max_block = zb_cut_blocks(segs.data(), n_segs, zb_block_max(window_log), jobs, info);
    u32 const nj = (u32)jobs.size();
    u64 const slot_bytes = zb_slot_bytes(max_block);
    TBuf slots((size_t)(nj + 1) * slot_bytes + 64); std::vector<ZeBlockOut> outs(nj + 1);
    if (n_ctas > nj) n_ctas = nj ? nj : 1;
    TBuf scratch(zb_encode2_scratch_bytes() * n_ctas);
    u32 counter = 0;
    if (nj) zb_launch_compress_smem(src, jobs.data(), nj, scratch.p, n_ctas, (u8*)slots.p, slot_bytes, outs.data(), &counter, nullptr, 0, nullptr, 0);
    return t_layout(src, segs, info, outs.data(), (const u8*)slots.p, slot_bytes, checksum, content_size, 0, window_log, out, out_cap, out_off, out_len);
}

// One run of a content-dictionary chain (zb200_compress_chain): chunk 0 of the run is the prefix of chunk 1 only; chunks
// 1..m-1 become frames.  src holds the run's chunks back to back (slack in front and behind), seg_off / seg_len locate them.
// The chunk indexes are built as on a device of one SM.  Returns the frames' total bytes.
extern "C" long long t_compress_chain_run(const u8* src, const u64* seg_off, const u64* seg_len, u32 m, u32 checksum, u32 n_ctas,
                                          u8* out, u64 out_cap, u64* out_off, u64* out_len)
{
    std::vector<ZbSegment> chunks = t_segments(seg_off, seg_len, m);
    std::vector<ZeChainSeg> cs(m); std::vector<u64> tab_off(m + 1), pos_off(m + 1);
    std::vector<ZeBlockJob> jobs; std::vector<ZeSegInfo> info(m - 1);
    zb_chain_plan(chunks.data(), m, cs.data(), tab_off.data(), pos_off.data(), jobs, info);
    std::vector<u32> tabs(tab_off[m], 0xFFFFFFFFu);
    for (u32 s = 0; s < m; s++) { cs[s].tab = tabs.data() + tab_off[s]; cs[s].prev_tab = s ? tabs.data() + tab_off[s - 1] : nullptr; }
    zb_launch_chain_index(src, cs.data(), pos_off.data(), m, pos_off[m], 1, 0);
    u32 const nj = (u32)jobs.size();
    u64 const slot_bytes = zb_slot_bytes(ZB_BLOCK_MAX);
    std::vector<u8> slots((size_t)(nj + 1) * slot_bytes); std::vector<ZeBlockOut> outs(nj + 1);
    if (n_ctas > nj) n_ctas = nj ? nj : 1;
    TBuf scratch(zb_encode_pscratch_bytes() * n_ctas);
    u32 counter = 0;
    if (nj) zb_launch_compress_chain_blocks(src, jobs.data(), nj, scratch.p, n_ctas, slots.data(), slot_bytes, outs.data(), &counter, cs.data(), 0);
    std::vector<ZbSegment> const fsegs(chunks.begin() + 1, chunks.end());
    return t_layout(src, fsegs, info, outs.data(), slots.data(), slot_bytes, checksum, 1, 0, 31, out, out_cap, out_off, out_len);
}

// ---- decompression
static int g_block_path = 0;
extern "C" void t_set_block_path(int on) { g_block_path = on; }
// The frame scans and the placement, as run_decompress runs them before it chooses a path: totals_out[0..5] = output,
// blocks, sequences, literals, any checksum, any window >= ZB_FAR_WINDOW.
extern "C" void t_scan_totals(const u8* src, const u64* seg_off, const u64* seg_len, u32 n, u64* totals_out)
{
    TScan S(src, seg_off, seg_len, n, nullptr);
    for (int k = 0; k < 6; k++) totals_out[k] = S.totals[k];
}

// Decode ONE frame through the launchers, as the library runs a batch of one: default tables, dictionary digest, scan,
// placement, then the lane-per-frame entropy kernel on one CTA of 7 warps with one frame per warp.  The output capacity is
// the frame's content size, or `cap` when the header does not state one.  The bytes are then regenerated from the kernel's
// block / sequence / literal records by a serial replay that shares no code with the execute kernels.  Returns the status
// code; *out_n = bytes produced.
extern "C" int t_decode_frame(const u8* src, u64 n, const u8* dict_raw, u32 dict_n, u8* out, u64 cap, u64* out_n, u32* n_blocks, u32* n_seq)
{
    static bool tables = false;
    if (!tables) { zb_launch_default_tables(0); tables = true; }
    static ZbDictDigest dg; ZbDictDev dict;
    if (u32 const st = t_dict_dev(dict_raw, dict_n, dg, dict)) return (int)st;
    ZbSegment seg; seg.offset = 0; seg.length = n;
    ZbFrameInfo fi; u32 big[2];
    zb_launch_scan(src, &seg, 1, &fi, (1ull << 27) + 1, big, 0);
    if (fi.status != ZB_OK) return (int)fi.status;
    u64 const want = fi.content_size != ZB_CONTENT_UNKNOWN ? fi.content_size : cap;
    if (want > cap) return (int)ZB_E_DSTSIZE_TOO_SMALL;
    ZbFramePlace place[2]; u64 totals[8] = {0}, partial[8]; u32 status = ZB_OK;
    zb_launch_place(&fi, &want, 1, place, totals, &status, partial, 0);
    std::vector<ZbBlock> vblocks(fi.n_blocks + 1); std::vector<ZbSeq> vseqs(fi.n_seq_rec + 2); std::vector<u8> vlits(fi.n_lit + 64);
    ZbBlock* const blocks = vblocks.data(); ZbSeq* const seqs = vseqs.data(); u8* const lits = vlits.data();
    u32 counter = 0, ck = 0; u64 out_size = 0;
    zb_launch_entropy(src, &seg, 1, place, fi.content_size != ZB_CONTENT_UNKNOWN ? &want : nullptr, blocks, seqs, lits, 1, &counter, dict, &status,
                      &out_size, &ck, 1, 7, 0);
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
    return rc;
}

// The whole decompression path (run_decompress): scan, placement, the entropy stage -- a lane per frame on `n_ctas` CTAs of
// `warps` warps with `take` frames per warp, or a lane per block (t_set_block_path 1: execute by zb_execute_big, 2: by
// pointer jumping) -- execute, checksums, finish.  Output: tightly packed bytes + per-frame {offset, length}, status[] per
// frame.
// `chunk_bytes` 0: one chunk of all frames with that launch shape.  Otherwise the call is cut as run_decompress cuts a call
// whose output is copied back (zb_chunk_count with this chunk size, zb_chunk_cut), and every chunk runs what the launcher
// runs for it: the lane-per-frame entropy launch over frames [0, cut[k + 1]) from a counter of its own that starts at cut[k],
// shaped by zb_chunk_shape from the chunk's output bytes with `n_ctas` as the SM count (the block path keeps its one
// entropy launch for all blocks, zb_entropy_blocks_ctas); then the chunk's execute stage and its checksums.
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
    if (!tables) { zb_launch_default_tables(0); tables = true; }
    static ZbDictDigest dg; ZbDictDev dict;
    if (u32 const st = t_dict_dev(dict_raw, dict_n, dg, dict)) return -(long long)st;
    TScan S(src, seg_off, seg_len, n, dst_sizes);
    ZbFramePlace* const place = S.place.data(); u32* const status = S.status.data(); u64 const* const totals = S.totals;
    if (totals[0] > out_cap) return -1000;
    std::vector<ZbBlock> blocks(totals[1] + 1); std::vector<ZbSeq> seqs(totals[2] + 2); std::vector<u8> lits(totals[3] + 64);
    std::vector<u64> out_sizes(n, 0); std::vector<u32> ck(n, 0);
    std::vector<u8> dev(totals[0] + 64, 0); u8* const d_out = dev.data();       // the device's output buffer
    u32 const n_chunks = chunk_bytes ? zb_chunk_count(totals[0], n, true, chunk_bytes) : 1;
    std::vector<u32> cut(n_chunks + 1); for (u32 k = 0; k <= n_chunks; k++) cut[k] = zb_chunk_cut(n, k, n_chunks);
    std::vector<ZbBlkDesc> bdesc;
    if (g_block_path) {          // a lane per BLOCK: zb_scan_blocks -> zb_entropy_blocks -> zb_resolve_blocks -> zb_patch_blocks
        u64 const nb = totals[1];
        u32 const btake = chunk_bytes ? ZB_BLOCKS_TAKE : (take > ZB_BLOCKS_TAKE ? ZB_BLOCKS_TAKE : take);
        u32 const bctas = chunk_bytes ? zb_entropy_blocks_ctas(nb, n_ctas) : n_ctas;
        u32 counter = 0;
        bdesc.resize(nb + 1); std::vector<ZbBlkExit> bexit(nb + 1); std::vector<u32> erep(3 * (nb + 1)); std::vector<u64> fend(n);
        zb_launch_scan_blocks(src, S.segs.data(), n, place, dict, status, bdesc.data(), fend.data(), S.big.data(), 0);
        zb_launch_entropy_blocks(src, bdesc.data(), (u32)nb, blocks.data(), seqs.data(), lits.data(), bctas, &counter, dict, status, bexit.data(), btake, 0);
        zb_launch_resolve_blocks(src, S.segs.data(), n, place, S.info.data(), dst_sizes, blocks.data(), bdesc.data(), bexit.data(), fend.data(), nb,
                                 seqs.data(), dict, status, out_sizes.data(), ck.data(), erep.data(), 0, 0);
    }
    std::vector<u64> chase(g_block_path == 2 ? (zb_chase_bytes(totals[0]) + 7) / 8 : 0);
    std::vector<u64> wave(g_block_path == 1 ? (zb_wave_bytes(n, totals[1]) + 7) / 8 : 0);
    u32 changed = 0;
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
            zb_launch_entropy(src, S.segs.data(), f1, place, dst_sizes, blocks.data(), seqs.data(), lits.data(), sh.ctas, &counter, dict, status,
                              out_sizes.data(), ck.data(), sh.take, sh.warps, 0);
        }
        if (g_block_path == 2)
            zb_launch_execute_chase(src, place, status, blocks.data(), bdesc.data(), seqs.data(), lits.data(), d_out, lo, hi, totals[0], blo, bhi,
                                    chase.data(), &changed, n_ctas, dict, 0, 0);
        else if (g_block_path)
            zb_launch_execute_big(src, place, status, blocks.data(), bdesc.data(), seqs.data(), lits.data(), d_out, f0, f1, blo, bhi, n, totals[1],
                                  wave.data(), n_ctas, dict, 0);
        else zb_launch_execute(src, place, status, blocks.data(), seqs.data(), lits.data(), d_out, f0, f1, dict, 0);
        if (totals[4]) zb_launch_verify(d_out, place, out_sizes.data(), S.info.data(), ck.data(), f0, f1, status, 0);
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
    zb_launch_finish(place, out_sizes.data(), status, n, out_segs.data(), &first_error, 0);
    for (u32 i = 0; i < n; i++) { out_off[i] = out_segs[i].offset; out_len[i] = out_segs[i].length; status_out[i] = status[i]; }
    return (long long)totals[0];
}

// One run in chain mode (zb200_decompress_chain), as run_decompress runs it with a ChainRun on a device of one SM: scan,
// placement, the shift behind the carried prefix, the block path, pointer jumping, checksums, finish.  out: the run's
// arena, carry[0, carry_n) first.
extern "C" long long t_decompress_chain_run(const u8* src, const u64* seg_off, const u64* seg_len, u32 n, const u8* carry, u64 carry_n,
                                            u8* out, u64 out_cap, u64* out_off, u64* out_len, u32* status_out, int* rounds_out)
{
    static bool tables = false;
    if (!tables) { zb_launch_default_tables(0); tables = true; }
    u32 const sms = 1;
    ZbDictDev dict; memset(&dict, 0, sizeof dict);
    TScan S(src, seg_off, seg_len, n, nullptr);
    ZbFramePlace* const place = S.place.data(); u32* const status = S.status.data(); u64 const* const totals = S.totals;
    if (carry_n) zb_launch_chain_shift(place, n, carry_n, 0);
    if (totals[5]) return -1001;
    u64 const total = totals[0] + carry_n;
    if (total > out_cap) return -1000;
    memcpy(out, carry, carry_n);
    u64 const nb = totals[1];
    std::vector<ZbBlock> blocks(nb + 1); std::vector<ZbSeq> seqs(totals[2] + 2); std::vector<u8> lits(totals[3] + 64);
    std::vector<u64> out_sizes(n, 0); std::vector<u32> ck(n, 0); u32 counter = 0;
    std::vector<ZbBlkDesc> bdesc(nb + 1); std::vector<ZbBlkExit> bexit(nb + 1); std::vector<u32> erep(3 * (nb + 1)); std::vector<u64> fend(n);
    zb_launch_scan_blocks(src, S.segs.data(), n, place, dict, status, bdesc.data(), fend.data(), S.big.data(), 0);
    zb_launch_entropy_blocks(src, bdesc.data(), (u32)nb, blocks.data(), seqs.data(), lits.data(), zb_entropy_blocks_ctas(nb, sms), &counter, dict,
                             status, bexit.data(), ZB_BLOCKS_TAKE, 0);
    zb_launch_resolve_blocks(src, S.segs.data(), n, place, S.info.data(), nullptr, blocks.data(), bdesc.data(), bexit.data(), fend.data(), nb,
                             seqs.data(), dict, status, out_sizes.data(), ck.data(), erep.data(), 0, 1);
    std::vector<u64> chase((zb_chase_bytes(total) + 7) / 8); u32 changed = 0;
    *rounds_out = zb_launch_execute_chase(src, place, status, blocks.data(), bdesc.data(), seqs.data(), lits.data(), out, 0, total, total, 0, nb,
                                          chase.data(), &changed, sms, dict, 0, 1);
    if (totals[4]) zb_launch_verify(out, place, out_sizes.data(), S.info.data(), ck.data(), 0, n, status, 0);
    std::vector<ZbSegment> out_segs(n); u32 first_error = 0xFFFFFFFFu;
    zb_launch_finish(place, out_sizes.data(), status, n, out_segs.data(), &first_error, 0);
    for (u32 i = 0; i < n; i++) { out_off[i] = out_segs[i].offset; out_len[i] = out_segs[i].length; status_out[i] = status[i]; }
    return (long long)total;
}

// ---- dictionary training: the kernels of zb_train.cuh on CTAs sized for the CPU (its header says why they may be)
// hash + count of one d (zt_hash_all, zt_count)
static void t_tables(const u8* s, const u64* offs, u32 n_train, u32 f, u32 d, u32 step, std::vector<u32>& hash, std::vector<u32>& freqs)
{
    u32 const n_dmers = (u32)(offs[n_train] - 8 + 1);
    hash.assign(n_dmers, 0); freqs.assign((size_t)1 << f, 0);
    simt::launch(4, 64, [&] { zt_hash_all(s, n_dmers, f, d, hash.data()); });
    simt::launch(4, 64, [&] { zt_count(hash.data(), offs, n_train, step, freqs.data()); });
}
extern "C" void t_freqs(const u8* s, const u64* offs, u32 n_train, u32 f, u32 d, u32 step, u32* out)
{
    std::vector<u32> hash, freqs; t_tables(s, offs, n_train, f, d, step, hash, freqs);
    memcpy(out, freqs.data(), freqs.size() * 4);
}
// prev[] of every position (zt_prev_local + zt_prev_link)
extern "C" void t_prev(const u32* hash, u32 n, u32 f, u32* prev)
{
    std::vector<u8> last(n); std::vector<u32> table((size_t)1 << f, 0xFFFFFFFFu);
    simt::launch((n + ZT_CHUNK - 1) / ZT_CHUNK, 128, [&] { zt_prev_local(hash, n, prev, last.data()); });
    simt::launch(1, 128, [&] { zt_prev_link(hash, n, prev, last.data(), table.data()); });
}
// one candidate (k, d) through zt_select: the content lands in dict[*tail .. cap)
extern "C" void t_select(const u8* s, const u64* offs, u32 n_train, u32 f, u32 d, u32 step, u32 k, u32 cap, u8* dict, u32* tail)
{
    std::vector<u32> hash, freqs; t_tables(s, offs, n_train, f, d, step, hash, freqs);
    u32 const n = (u32)hash.size();
    std::vector<u32> prev(n); t_prev(hash.data(), n, f, prev.data());
    u32 num, esz; zt_epochs(cap, n, k, num, esz);
    std::vector<u32> diff(esz + 2);
    ZtCand cand{k, d, 0, 0};
    ZtSelect A; memset(&A, 0, sizeof A);
    A.samples = s; A.n_dmers[0] = n; A.hash[0] = hash.data(); A.prev[0] = prev.data();
    A.freqs = freqs.data(); A.freqs_stride = 0; A.diff = diff.data(); A.diff_stride = 0; A.dict = dict; A.cap = cap;
    A.tail = tail; A.cand = &cand; A.first = 0;
    simt::launch(1, 128, [&] { zt_select(A); });
}
// zt_entropy + zt_finalize of one content with given statistics (u32[377])
extern "C" long long t_finalize(const u8* dict, u32 cap, u32 tail, const u32* stats, u32 dict_id, u8* out)
{
    u8 ent[512]; u32 ent_len = 0; long long res = 0;
    simt::launch(1, 32, [&] { zt_entropy(stats, cap - tail, ent, &ent_len); });
    simt::launch(1, 64, [&] { zt_finalize(dict, cap, &tail, ent, &ent_len, dict_id, out, &res); });
    return res;
}
