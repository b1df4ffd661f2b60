// simt_lazy.cpp -- the CPU build of the kernel source with a wrapper for the lazy mode of the block kernel (test
// infrastructure, not product code).
//
// The whole of simt_kernels.cpp -- zb_decode.cu and zb_encode.cu on the SIMT runtime of simt.h, and its wrappers -- plus
// t_compress_batch_lazy below; tests/test_compress_lazy_host.py builds this file with the flags of tests/host_encoder.py.
#include "simt_kernels.cpp"

// The lazy mode (an explicit greedy / lazy / lazy2 strategy: depth 0 / 1 / 2) through zb_launch_compress_lazy, with the jobs,
// the dictionary and the frame window of a call with this window_log and content-size flag.  Returns total bytes.
extern "C" long long t_compress_batch_lazy(const u8* src, const u64* seg_off, const u64* seg_len, u32 n_segs, u32 checksum, u32 content_size,
                                           u32 n_ctas, u8* out, u64 out_cap, u64* out_off, u64* out_len, const u8* dict_raw, u32 dict_n,
                                           u32 window_log, u32 depth, u32 search_log, u32 min_match)
{
    std::vector<ZbSegment> segs = t_segments(seg_off, seg_len, n_segs); std::vector<ZeBlockJob> jobs; std::vector<ZeSegInfo> info(n_segs);
    u32 const max_block = zb_cut_blocks(segs.data(), n_segs, zb_block_max(window_log), jobs, info);
    u32 const nj = (u32)jobs.size();
    u64 const slot_bytes = zb_slot_bytes(max_block);
    std::vector<u8> slots((size_t)(nj + 1) * slot_bytes); std::vector<ZeBlockOut> outs(nj + 1);
    if (n_ctas > nj) n_ctas = nj ? nj : 1;
    static ZbDictDigest dg; static ZeCTable cct[3];
    ZbDictView view = {nullptr, 0};
    u32 dict_id = 0;
    if (dict_raw && dict_n) {
        zb_launch_digest_dict(dict_raw, dict_n, &dg, 0);
        if (dg.status != ZB_OK) return -2;
        view = dg.has_entropy ? zb_dict_view(dict_raw + dg.content_off, dict_n - dg.content_off) : zb_dict_view(dict_raw, dict_n);
        if (view.D) { dict_id = dg.dict_id; if (dg.has_entropy) zb_launch_dict_ctables(&dg, cct, 0); }
    }
    const void* const digest = view.D && dg.has_entropy ? &dg : nullptr;
    TBuf scratch(zb_encode_lscratch_bytes() * n_ctas);
    u32 counter = 0;
    if (nj) zb_launch_compress_lazy(src, jobs.data(), nj, scratch.p, n_ctas, slots.data(), slot_bytes, outs.data(), &counter,
                                    view.tail, view.D, digest, digest ? cct : nullptr, nullptr, 0, nullptr, depth, search_log, min_match,
                                    zb_frame_window(window_log, content_size), 0);
    return t_layout(src, segs, info, outs.data(), slots.data(), slot_bytes, checksum, content_size, dict_id, window_log, out, out_cap, out_off, out_len);
}
