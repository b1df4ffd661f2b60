// zb_api.cu -- the C ABI of libzb200.so (include/zb200.h): contexts, memory pools, the host
// orchestration that replaces decompress_from_framesources (c-ext/decompressor.c:1186-1455).
//
// The reference partitions the batch over a pthread pool (POOL_add, c-ext/decompressor.c:1290-1320);
// here the partition is the CUDA grid and the "workers" are warps.  What stays on the host is only
// what the reference also does on its calling thread: argument marshalling, output ownership and
// first-error selection.
#include "zb_common.cuh"
#include "../../include/zb200.h"
#define ZT_TYPES_ONLY
#include "zb_train.cuh"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <chrono>
#include <cstdlib>
#include <string>
#include <vector>
#include <thread>
#include <map>
#include <algorithm>

extern "C" {
void zb_launch_default_tables(cudaStream_t st);
void zb_launch_scan(const u8* src, const ZbSegment* segs, u32 n, ZbFrameInfo* info, u64 window_limit, u32* big_list, cudaStream_t st);
void zb_launch_scan_blocks(const u8* src, const ZbSegment* segs, u32 n, const ZbFramePlace* place, ZbDictDev dict, u32* status,
                           void* bdesc, u64* frame_end, const u32* big_list, cudaStream_t st);
void zb_launch_entropy_blocks(const u8* src, const void* bdesc, u32 n_blocks, ZbBlock* blocks, ZbSeq* seqs, u8* lits, u32 n_ctas, u32* work_counter,
                              ZbDictDev dict, u32* status, void* bexit, u32 take, cudaStream_t st);
void zb_launch_resolve_blocks(const u8* src, const ZbSegment* segs, u32 n, const ZbFramePlace* place, const ZbFrameInfo* info, const u64* dst_sizes,
                              ZbBlock* blocks, const void* bdesc, const void* bexit, const u64* frame_end, u64 n_blocks, ZbSeq* seqs, ZbDictDev dict,
                              u32* status, u64* out_sizes, u32* ck_expect, u32* entry_rep, cudaStream_t st, int chain);
size_t zb_blkdesc_bytes();
size_t zb_blkexit_bytes();
void zb_launch_place(const ZbFrameInfo* info, const u64* dst_sizes, u32 n, ZbFramePlace* place, u64* totals,
                     u32* status, u64* partial, cudaStream_t st);
void zb_launch_entropy(const u8* src, const ZbSegment* segs, u32 n, const ZbFramePlace* place, const u64* dst_sizes,
                       ZbBlock* blocks, ZbSeq* seqs, u8* lits, u32 n_ctas, u32* work_counter,
                       ZbDictDev dict, u32* status, u64* out_sizes, u32* ck_expect, u32 take, u32 warps, cudaStream_t st);
size_t zb_wave_bytes(u64 n_frames, u64 n_blocks);
size_t zb_chase_bytes(u64 n_total);
int zb_launch_execute_chase(const u8* src, const ZbFramePlace* place, const u32* status, const ZbBlock* blocks, const void* bdesc,
                            const ZbSeq* seqs, const u8* lits, u8* dst, u64 lo, u64 hi, u64 n_total, u64 blk_first, u64 blk_last,
                            void* ptr_mem, u32* d_changed, u32 n_ctas, ZbDictDev dict, cudaStream_t st, int chain);
void zb_launch_execute_big(const u8* src, const ZbFramePlace* place, const u32* status, const ZbBlock* blocks, const void* bdesc,
                           const ZbSeq* seqs, const u8* lits, u8* dst, u32 first, u32 end, u64 blk_first, u64 blk_last,
                           u64 n_frames, u64 n_blocks, void* wave_mem, u32 n_ctas, ZbDictDev dict, cudaStream_t st);
void zb_launch_verify(const u8* dst, const ZbFramePlace* place, const u64* out_sizes, const ZbFrameInfo* info, const u32* ck_expect,
                      u32 first, u32 end, u32* status, cudaStream_t st);
void zb_launch_execute(const u8* src, const ZbFramePlace* place, const u32* status, const ZbBlock* blocks,
                       const ZbSeq* seqs, const u8* lits, u8* dst, u32 first, u32 end, ZbDictDev dict, cudaStream_t st);
void zb_launch_finish(const ZbFramePlace* place, const u64* out_sizes, const u32* status, u32 n, ZbSegment* out_segs,
                      u32* first_error, cudaStream_t st);
void zb_launch_chain_shift(ZbFramePlace* place, u32 n, u64 carry, cudaStream_t st);
void zb_launch_digest_dict(const u8* dict, u32 n, ZbDictDigest* out, cudaStream_t st);
size_t zb_encode_scratch_bytes();
void zb_launch_compress_blocks(const u8* src, const ZeBlockJob* jobs, u32 n_jobs, void* scratch, u32 n_ctas, u8* slots, u64 slot_bytes,
                               ZeBlockOut* outs, u32* work_counter, const u8* dict_tail, u32 dict_D, const u16* dict_table, const void* dict_digest, const void* dict_cct,
                               const unsigned long long* upload_progress, unsigned long long upload_total, u32* upload_status, int dual, int small_blocks, cudaStream_t st,
                               u32* stats = nullptr);
u32 zb_encode_small_max();
void zb_launch_dict_table(const u8* tail, u32 D, u16* table, cudaStream_t st);
size_t zb_encode_pscratch_bytes();
void zb_launch_chain_index(const u8* src, const ZeChainSeg* segs, const u64* pos_off, u32 n_segs, u64 total_pos, u32 sms, cudaStream_t st);
void zb_launch_compress_chain_blocks(const u8* src, const ZeBlockJob* jobs, u32 n_jobs, void* scratch, u32 n_ctas, u8* slots, u64 slot_bytes,
                                     ZeBlockOut* outs, u32* work_counter, const ZeChainSeg* segs, cudaStream_t st);
u32 zb_encode_ctable_bytes();
void zb_launch_dict_ctables(const void* digest, void* out3, cudaStream_t st);
void zb_launch_frame_layout(const ZbSegment* segs, const ZeSegInfo* seginfo, const ZeBlockOut* outs, u32 n_segs, u32 checksum, u32 content_size,
                            u32 dict_id, u32 window_log, u64* sizes, ZbSegment* out_segs, u64* total, cudaStream_t st);
void zb_launch_write_frames(const u8* src, const ZbSegment* segs, const ZeSegInfo* seginfo, const ZeBlockOut* outs, const u8* slots, u64 slot_bytes,
                            u32 n_segs, u32 checksum, u32 content_size, u32 dict_id, u32 window_log, const ZbSegment* out_segs, u8* dst, cudaStream_t st);
u32 zb_encode_smem_bytes();
u32 zb_encode3_record_max();
u32 zb_encode3_records_per_cta();
void zb_launch_compress_recs(const u8* src, const ZeBlockJob* jobs, u32 n_jobs, u32 n_ctas, u8* slots, u64 slot_bytes, ZeBlockOut* outs, u32* work_counter,
                             const u8* dict_tail, u32 dict_D, const u16* dict_table, const void* dict_digest, const void* dict_cct,
                             const unsigned long long* upload_progress, unsigned long long upload_total, u32* upload_status, cudaStream_t st);
size_t zb_encode2_scratch_bytes();
void zb_launch_compress_smem(const u8* src, const ZeBlockJob* jobs, u32 n_jobs, void* scratch, u32 n_ctas, u8* slots, u64 slot_bytes, ZeBlockOut* outs, u32* work_counter,
                             const unsigned long long* upload_progress, unsigned long long upload_total, u32* upload_status, cudaStream_t st);
// dictionary training (zb_train.cuh)
void zt_launch_hash(const u8* s, u32 n_dmers, u32 f, u32 d, u32* hash, u32 sms, cudaStream_t st);
void zt_launch_count(const u32* hash, const u64* offs, u32 n_train, u32 step, u32* freqs, u32 sms, cudaStream_t st);
void zt_launch_prev(const u32* hash, u32 n, u32* prev, u8* last, u32* table, cudaStream_t st);
void zt_launch_select(const void* args, u32 n_ctas, cudaStream_t st);
void zt_launch_entropy(const u32* stats, u32 content_size, u8* ent, u32* ent_len, cudaStream_t st);
void zt_launch_finalize(const u8* dict, u32 cap, const u32* tail, const u8* ent, const u32* ent_len, u32 dict_id, u8* out, long long* res,
                        cudaStream_t st);
}

namespace {

struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes + bytes / 8 + 4096;          // grow-only with slack
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T* as() const { return (T*)p; }
};

struct PinnedBlock { void* p; size_t cap; bool busy; };

}  // namespace

struct zb200_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;          // device->host copies of finished chunks, overlapping later chunks' kernels
    cudaEvent_t chunk_ev[64] = {nullptr};
    unsigned long long* h_progress = nullptr;    // pinned: the byte counts the chunked upload publishes to the compress kernel
    std::string last_error;
    int sm_count = 132;
    // device arenas (grow-only)
    DevBuf src, segs, dst_sizes, info, place, status, out_sizes, blocks, seqs, lits, dst, lane, small, out_segs, partial;
    DevBuf jobs, seginfo, slots, bouts, escratch, fsizes, ck;
    DevBuf bdesc, bexit, erep, fend, wave;    // block-parallel decode path
    DevBuf biglist;                           // frames whose scans are a warp's work (zb_scan_frames_big)
    DevBuf chase;                             // its pointer-jumping execute stage: a source pointer per output byte
    DevBuf carry;                             // content-dictionary chains: the last fulltext of a run, the prefix of the next
    DevBuf chain_tab, chain_seg, chain_pos;   // chain compression: the chunk indexes of a run, their descriptors, sampled positions
    int last_chase_rounds = 0;
    const char* last_compress_kernel = "";    // which of the three block kernels the last compress call ran (profile slot zb_compress_blocks)
    u32 entropy_warps = 0;
    // pinned pool
    std::mutex mu;
    std::vector<PinnedBlock> pinned;
    // profiling
    bool prof = false;
    std::vector<cudaEvent_t> ev_pool; size_t ev_used = 0;
    struct Span { int k; cudaEvent_t a, b; };
    std::vector<Span> spans;
    float k_ms[ZB200_K_COUNT] = {0}; u32 k_launch[ZB200_K_COUNT] = {0};
    u64 last_scratch = 0;
    int live_results = 0;
};

struct zb200_ddict {
    zb200_ctx* ctx; void* d_raw = nullptr; ZbDictDigest* d_digest = nullptr; ZbDictDev dev; size_t size = 0;
    u16* d_ctable = nullptr; const u8* c_tail = nullptr; u32 c_D = 0; void* d_cct = nullptr;      // compression view: last <= 32 KiB of the content + its hash table
};

struct zb200_result {
    zb200_ctx* ctx; void* data = nullptr; bool data_on_device = false; bool data_pinned_pool = false;
    bool data_owned_device = false;        // ZB200_DST_DEVICE: the result owns its device allocation (stream-ordered pool)
    std::vector<u8> host_data;             // zb200_compress_chain: the frames, in pageable memory the result owns
    u64 size = 0; size_t n = 0;
    std::vector<zb200_segment> segs;       // compress and chain results: the table in pageable memory the result owns
    // batch decode: the table in a block of the context's pinned pool.  A device-resident result (ZB200_DST_DEVICE) keeps
    // its table in a device allocation of its own (stream-ordered pool) and copies it here on the first
    // zb200_result_segments: a caller that never reads it pays no device->host copy
    mutable zb200_segment* segs_pinned = nullptr;
    ZbSegment* segs_device = nullptr;
    mutable std::mutex segs_mu;
    bool has_error = false; size_t err_item = 0; int err_code = 0; u64 err_got = 0, err_expected = 0;
};

namespace {

int fail(zb200_ctx* c, const char* what, cudaError_t e)
{
    char buf[512];
    snprintf(buf, sizeof buf, "%s: %s", what, e == cudaSuccess ? "invalid argument" : cudaGetErrorString(e));
    if (c) c->last_error = buf;
    return -1;
}
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(ctx, #call, e_); } while (0)

cudaEvent_t get_event(zb200_ctx* c)
{
    if (c->ev_used == c->ev_pool.size()) { cudaEvent_t e; cudaEventCreate(&e); c->ev_pool.push_back(e); }
    return c->ev_pool[c->ev_used++];
}
struct KSpan {
    zb200_ctx* c; int k; cudaEvent_t a = nullptr;
    KSpan(zb200_ctx* c_, int k_) : c(c_), k(k_) { if (c->prof) { a = get_event(c); cudaEventRecord(a, c->stream); } c->k_launch[k]++; }
    ~KSpan() { if (c->prof) { cudaEvent_t b = get_event(c); cudaEventRecord(b, c->stream); c->spans.push_back({k, a, b}); } }
};
void fold_spans(zb200_ctx* c)
{
    for (auto& s : c->spans) { float ms = 0; if (cudaEventElapsedTime(&ms, s.a, s.b) == cudaSuccess) c->k_ms[s.k] += ms; }
    c->spans.clear(); c->ev_used = 0;
}

void* pinned_get(zb200_ctx* c, size_t bytes)
{
    // size classes (powers of two up to 64 MiB, then multiples of 64 MiB) so that batches of slightly different
    // sizes reuse the same blocks; blocks are kept for the life of the context (page-locking is slow)
    size_t cls = 1 << 16;
    while (cls < bytes && cls < ((size_t)64 << 20)) cls <<= 1;
    if (cls < bytes) cls = (bytes + ((size_t)64 << 20) - 1) & ~(((size_t)64 << 20) - 1);
    std::lock_guard<std::mutex> g(c->mu);
    PinnedBlock* best = nullptr;
    for (auto& b : c->pinned) if (!b.busy && b.cap >= cls && (!best || b.cap < best->cap)) best = &b;
    if (best) { best->busy = true; return best->p; }
    void* p = nullptr;
    if (cudaHostAlloc(&p, cls, cudaHostAllocPortable) != cudaSuccess) {
        // out of pinned memory: release idle blocks and retry once
        for (size_t i = 0; i < c->pinned.size();) {
            if (!c->pinned[i].busy) { cudaFreeHost(c->pinned[i].p); c->pinned.erase(c->pinned.begin() + (long)i); } else i++;
        }
        if (cudaHostAlloc(&p, cls, cudaHostAllocPortable) != cudaSuccess) return nullptr;
    }
    c->pinned.push_back({p, cls, true});
    return p;
}
void pinned_put(zb200_ctx* c, void* p)
{
    std::lock_guard<std::mutex> g(c->mu);
    for (auto& b : c->pinned) if (b.p == p) { b.busy = false; return; }
}
bool zb_trace_on() { static int v = -1; if (v < 0) { const char* e = getenv("ZB200_TRACE"); v = (e && *e && *e != '0') ? 1 : 0; } return v == 1; }
double zb_now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

ZbDictDev no_dict() { ZbDictDev d; memset(&d, 0, sizeof d); return d; }

// One upload at a time per device: when several contexts work on sub-batches of one call, this staggers
// them (A computes and downloads while B uploads) instead of letting them share every stage in lock-step.
std::mutex g_upload_mu[16];

}  // namespace

extern "C" {

int zb200_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) return 0; return n; }

int zb200_ctx_create(int device, zb200_ctx** out)
{
    *out = nullptr;
    int n = zb200_device_count();
    if (n <= 0 || device < 0 || device >= n) return -2;          // no CUDA device: there is no CPU path
    zb200_ctx* ctx = new zb200_ctx();
    ctx->device = device;
    if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete ctx; return -1;
    }
    cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device);
    {   // device-resident results come from the stream-ordered pool: keep what it has freed (no cudaMalloc per call)
        cudaMemPool_t pool; unsigned long long keep = ~0ull;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking);
    for (auto& e : ctx->chunk_ev) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    cudaHostAlloc((void**)&ctx->h_progress, 64 * sizeof(unsigned long long), cudaHostAllocPortable);
    zb_launch_default_tables(ctx->stream);
    if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) { cudaStreamDestroy(ctx->stream); delete ctx; return -1; }
    *out = ctx;
    return 0;
}

void zb200_ctx_destroy(zb200_ctx* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    ctx->bdesc.release(); ctx->bexit.release(); ctx->erep.release(); ctx->fend.release(); ctx->wave.release(); ctx->chase.release(); ctx->biglist.release(); ctx->carry.release();
    ctx->chain_tab.release(); ctx->chain_seg.release(); ctx->chain_pos.release();
    DevBuf* all[] = {&ctx->src, &ctx->segs, &ctx->dst_sizes, &ctx->info, &ctx->place, &ctx->status, &ctx->out_sizes,
                     &ctx->blocks, &ctx->seqs, &ctx->lits, &ctx->dst, &ctx->lane, &ctx->small, &ctx->out_segs, &ctx->partial,
                     &ctx->jobs, &ctx->seginfo, &ctx->slots, &ctx->bouts, &ctx->escratch, &ctx->fsizes, &ctx->ck};
    for (auto* b : all) b->release();
    for (auto& b : ctx->pinned) cudaFreeHost(b.p);
    for (auto e : ctx->ev_pool) cudaEventDestroy(e);
    for (auto e : ctx->chunk_ev) if (e) cudaEventDestroy(e);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->h_progress) cudaFreeHost(ctx->h_progress);
    cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char* zb200_ctx_last_error(const zb200_ctx* ctx) { return ctx ? ctx->last_error.c_str() : "no context"; }
void* zb200_ctx_stream(zb200_ctx* ctx) { return (void*)ctx->stream; }
int zb200_ctx_synchronize(zb200_ctx* ctx) { cudaSetDevice(ctx->device); CK(cudaStreamSynchronize(ctx->stream)); return 0; }

const char* zb200_error_string(int code)
{
    // strings of ERR_getErrorString (zstd/zstd.c, error_private.c) so messages match the reference's
    switch (code) {
    case 0: return "No error detected";
    case 1: return "Error (generic)";
    case 10: return "Unknown frame descriptor";
    case 12: return "Version not supported";
    case 14: return "Unsupported frame parameter";
    case 16: return "Frame requires too much memory for decoding";
    case 20: return "Data corruption detected";
    case 22: return "Restored data doesn't match checksum";
    case 24: return "Header of Literals' block doesn't respect format specification";
    case 30: return "Dictionary is corrupted";
    case 32: return "Dictionary mismatch";
    case 40: return "Unsupported parameter";
    case 42: return "Parameter is out of bound";
    case 44: return "tableLog requires too much memory : unsupported";
    case 46: return "Unsupported max Symbol Value : too large";
    case 48: return "Specified maxSymbolValue is too small";
    case 64: return "Allocation error : not enough memory";      /* also: a frame whose literal / sequence counts do not fit 32 bits */
    case 70: return "Destination buffer is too small";
    case 72: return "Src size is incorrect";
    case 74: return "Operation on NULL destination buffer";
    case ZB200_E_UNKNOWN_SIZE: return "could not determine decompressed size";
    case ZB200_E_SIZE_MISMATCH: return "decompressed size mismatch";
    default: return "Unspecified error code";
    }
}

void* zb200_host_alloc(zb200_ctx* ctx, size_t bytes) { cudaSetDevice(ctx->device); return pinned_get(ctx, bytes ? bytes : 1); }
void  zb200_host_free(zb200_ctx* ctx, void* p) { pinned_put(ctx, p); }
void* zb200_device_alloc(zb200_ctx* ctx, size_t bytes)
{
    cudaSetDevice(ctx->device); void* p = nullptr;
    if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess) return nullptr;
    return p;
}
void zb200_device_free(zb200_ctx* ctx, void* p) { cudaSetDevice(ctx->device); cudaFree(p); }
int zb200_memcpy_h2d(zb200_ctx* ctx, void* dst, const void* src, size_t bytes)
{
    cudaSetDevice(ctx->device);
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream)); CK(cudaStreamSynchronize(ctx->stream)); return 0;
}
int zb200_memcpy_d2h(zb200_ctx* ctx, void* dst, const void* src, size_t bytes)
{
    cudaSetDevice(ctx->device);
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream)); CK(cudaStreamSynchronize(ctx->stream)); return 0;
}

void zb200_host_copy(void* dst, const void* src, size_t bytes)
{
    size_t const piece = 1u << 20;
    unsigned hw = std::thread::hardware_concurrency(); if (hw == 0) hw = 4;
    size_t nt = bytes / piece; if (nt > 16) nt = 16; if (nt > hw) nt = hw;
    if (nt < 2) { memcpy(dst, src, bytes); return; }
    size_t const n_pieces = (bytes + piece - 1) / piece;
    std::vector<std::thread> th;
    for (size_t t = 0; t < nt; t++)
        th.emplace_back([=] {
            for (size_t k = t; k < n_pieces; k += nt) {
                size_t const o = k * piece, len = o + piece <= bytes ? piece : bytes - o;
                memcpy((char*)dst + o, (const char*)src + o, len);
            }
        });
    for (auto& x : th) x.join();
}

int zb200_pointer_device(const void* p)
{
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return -1; }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged ? a.device : -1;
}

// ---------------------------------------------------------------- dictionaries
int zb200_ddict_create(zb200_ctx* ctx, const void* dict, size_t size, zb200_ddict** out)
{
    *out = nullptr;
    if (!ctx || !dict || size == 0 || size > 0x7FFFFFFFu) return fail(ctx, "zb200_ddict_create", cudaSuccess);
    cudaSetDevice(ctx->device);
    zb200_ddict* d = new zb200_ddict(); d->ctx = ctx; d->size = size;
    cudaError_t e = cudaMalloc(&d->d_raw, size + 16);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d->d_digest, sizeof(ZbDictDigest));
    if (e == cudaSuccess) e = cudaMemcpyAsync(d->d_raw, dict, size, cudaMemcpyHostToDevice, ctx->stream);
    ZbDictDigest* h = nullptr;
    if (e == cudaSuccess) {
        zb_launch_digest_dict((const u8*)d->d_raw, (u32)size, d->d_digest, ctx->stream);
        h = (ZbDictDigest*)malloc(sizeof(ZbDictDigest));
        e = cudaMemcpyAsync(h, d->d_digest, sizeof(ZbDictDigest), cudaMemcpyDeviceToHost, ctx->stream);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { free(h); zb200_ddict_free(d); return fail(ctx, "zb200_ddict_create", e); }
    if (h->status != ZB_OK) { int code = (int)h->status; free(h); zb200_ddict_free(d); ctx->last_error = zb200_error_string(code); return -code; }
    ZbDictDev& v = d->dev; memset(&v, 0, sizeof v);
    v.content = (const u8*)d->d_raw + h->content_off; v.content_size = (u32)size - h->content_off;
    v.dict_id = h->dict_id; v.has_entropy = h->has_entropy;
    v.huf = d->d_digest->huf; v.huf_log = h->huf_log;
    v.ll = d->d_digest->ll; v.of = d->d_digest->of; v.ml = d->d_digest->ml;
    v.ll_log = h->ll_log; v.of_log = h->of_log; v.ml_log = h->ml_log;
    v.rep[0] = h->rep[0]; v.rep[1] = h->rep[1]; v.rep[2] = h->rep[2];
    free(h);
    // compression view (built now, it is one tiny launch)
    ZbDictView const cv = zb_dict_view(v.content, v.content_size);
    d->c_tail = cv.tail; d->c_D = cv.D;
    if (d->c_D && cudaMalloc((void**)&d->d_ctable, 16384 * sizeof(u16)) == cudaSuccess) {
        zb_launch_dict_table(d->c_tail, d->c_D, d->d_ctable, ctx->stream);
        if (v.has_entropy && cudaMalloc(&d->d_cct, 3 * (size_t)zb_encode_ctable_bytes()) == cudaSuccess)
            zb_launch_dict_ctables(d->d_digest, d->d_cct, ctx->stream);
        cudaStreamSynchronize(ctx->stream);
    } else d->c_D = 0;
    *out = d;
    return 0;
}
void zb200_ddict_free(zb200_ddict* d)
{
    if (!d) return;
    cudaSetDevice(d->ctx->device);
    if (d->d_raw) cudaFree(d->d_raw);
    if (d->d_digest) cudaFree(d->d_digest);
    if (d->d_ctable) cudaFree(d->d_ctable);
    if (d->d_cct) cudaFree(d->d_cct);
    delete d;
}
uint32_t zb200_ddict_id(const zb200_ddict* d) { return d ? d->dev.dict_id : 0; }

// ---------------------------------------------------------------- batch decompression
// Device-side pipeline shared by the host and device entry points.  d_src/d_segs/d_dst_sizes are device
// pointers.  On return the output is in ctx->dst (or caller_dst), segment table + status on the host.
// chain: content-dictionary chain mode (zb200_decompress_chain).  The frames are revisions, each one's prefix is the previous
// one's output; the carried prefix -- ctx->carry, chain->carry bytes -- goes in front of frame 0.  The output stays in ctx->dst
// (nothing is copied back) and the path is always the block path with the pointer-jumping execute stage.
struct ChainRun { u64 carry; };
static int run_decompress(zb200_ctx* ctx, const u8* d_src, const ZbSegment* d_segs, size_t n, const u64* d_dst_sizes,
                          const zb200_ddict* dict, zb200_result* res, bool copy_back, bool exact_sizes, u64 window_limit,
                          const ChainRun* chain = nullptr)
{
    u32 const nf = (u32)n;
    ZbDictDev dd = dict ? dict->dev : no_dict();
    CK(ctx->info.ensure(n * sizeof(ZbFrameInfo)));
    CK(ctx->place.ensure((n + 1) * sizeof(ZbFramePlace)));
    CK(ctx->status.ensure(n * sizeof(u32)));
    CK(ctx->out_sizes.ensure(n * sizeof(u64)));
    CK(ctx->out_segs.ensure(n * sizeof(ZbSegment)));
    CK(ctx->small.ensure(512));
    CK(ctx->partial.ensure(((n + 1023) / 1024 + 1) * 4 * sizeof(u64)));
    u64* d_totals = ctx->small.as<u64>();                 // [0..3] totals
    u32* d_counter = (u32*)(d_totals + 8);                // work counter
    u32* d_first_err = d_counter + 1;
    u32 init[2] = {0, 0xFFFFFFFFu};
    CK(cudaMemcpyAsync(d_counter, init, sizeof init, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(d_totals, 0, 8 * sizeof(u64), ctx->stream));
    CK(ctx->ck.ensure(n * sizeof(u32)));

    CK(ctx->biglist.ensure(((size_t)n + 1) * sizeof(u32)));
    { KSpan s(ctx, ZB200_K_SCAN); zb_launch_scan(d_src, d_segs, nf, ctx->info.as<ZbFrameInfo>(), window_limit, ctx->biglist.as<u32>(), ctx->stream); }
    { KSpan s(ctx, ZB200_K_PLACE);
      zb_launch_place(ctx->info.as<ZbFrameInfo>(), d_dst_sizes, nf, ctx->place.as<ZbFramePlace>(), d_totals,
                      ctx->status.as<u32>(), ctx->partial.as<u64>(), ctx->stream); }
    u64 totals[6];          // output, blocks, sequences, literals, any checksum, any window >= ZB_FAR_WINDOW
    CK(cudaMemcpyAsync(totals, d_totals, sizeof totals, cudaMemcpyDeviceToHost, ctx->stream));
    if (chain && chain->carry) zb_launch_chain_shift(ctx->place.as<ZbFramePlace>(), nf, chain->carry, ctx->stream);
    CK(cudaStreamSynchronize(ctx->stream));
    if (chain) {
        if (totals[5]) return fail(ctx, "zb200_decompress_chain: a window of ZB_FAR_WINDOW or more", cudaSuccess);
        totals[0] += chain->carry;
    }

    // persistent entropy grid: one CTA per SM (its shared memory holds the decode tables); trimmed per chunk below
    u32 const ctas = (u32)ctx->sm_count;
    CK(ctx->blocks.ensure((totals[1] + 1) * sizeof(ZbBlock)));
    CK(ctx->seqs.ensure((totals[2] + 1) * sizeof(ZbSeq)));
    CK(ctx->lits.ensure(totals[3] + 64));
    // the output: the context's arena when it is copied back to the host, an allocation of its own (stream-ordered pool)
    // when the caller keeps it on the device -- the next call on this context must not touch a live result
    u8* d_out;
    if (copy_back || chain) {
        CK(ctx->dst.ensure(totals[0] + 64)); d_out = ctx->dst.as<u8>();
        if (chain && chain->carry) CK(cudaMemcpyAsync(d_out, ctx->carry.p, chain->carry, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    else { void* p = nullptr; CK(cudaMallocAsync(&p, totals[0] + 64, ctx->stream)); d_out = (u8*)p; res->data = p; res->data_on_device = true; res->data_owned_device = true; }
    ctx->last_scratch = (totals[1] + 1) * sizeof(ZbBlock) + (totals[2] + 1) * sizeof(ZbSeq) + totals[3];

    // ---- chunks of frames: the device->host copy of chunk k overlaps the kernels of chunk k+1 (zb_chunk_count)
    u64 const chunk_bytes = getenv("ZB200_OUT_CHUNK_BYTES") ? strtoull(getenv("ZB200_OUT_CHUNK_BYTES"), nullptr, 10) : 0;   // (read per call: tests switch it)
    u32 const n_chunks = zb_chunk_count(totals[0], nf, copy_back, chunk_bytes);
    std::vector<u32> cut(n_chunks + 1); for (u32 k = 0; k <= n_chunks; k++) cut[k] = zb_chunk_cut(nf, k, n_chunks);
    std::vector<ZbFramePlace> cpl(n_chunks + 1);
    if (n_chunks > 1) {
        for (u32 k = 0; k <= n_chunks; k++)
            CK(cudaMemcpyAsync(&cpl[k], ctx->place.as<ZbFramePlace>() + cut[k], sizeof(ZbFramePlace), cudaMemcpyDeviceToHost, ctx->stream));
        std::vector<u32> cinit(n_chunks); for (u32 k = 0; k < n_chunks; k++) cinit[k] = cut[k];
        CK(cudaMemcpyAsync(d_counter + 8, cinit.data(), n_chunks * sizeof(u32), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    // Frames of several blocks when the batch alone does not fill the machine (one huge frame at the limit): a lane per BLOCK
    // instead of a lane per frame for the entropy stage (zb_scan_blocks -> zb_entropy_blocks -> zb_resolve_blocks / zb_patch_blocks)
    // Measured (tools/gpu_c3_decode.py, tools/gpu_c5_frame.py): frames of one 128 KiB chunk -- the reference's single block or
    // our ten sub-blocks -- are faster a lane per frame at any batch size (2048 of ours: 18.4 vs 6.6 GB/s); from a few full
    // blocks per frame on the lane's serial chain (4-5 ms per 128 KiB) is what the block path removes.
    // The block path tags symbolic repcodes with bit 31 and rejects larger offsets, so it never takes a batch in which an
    // offset can reach 2^31: a frame with a window of ZB_FAR_WINDOW or more, or a dictionary of ZB_FAR_DICT bytes or more.
    int const force_blocks = getenv("ZB200_BLOCK_PATH") ? atoi(getenv("ZB200_BLOCK_PATH")) : -1;      // (read per call: tests switch it)
    bool const far = totals[5] != 0 || dd.content_size >= ZB_FAR_DICT;
    bool const block_path = chain || (!far && (force_blocks >= 0 ? force_blocks != 0 : (totals[1] > n && n < 3000 && totals[0] >= (u64)n * (512u << 10))));
    bool chase_path = false;
    ctx->last_chase_rounds = 0;
    if (block_path) {
        u64 const nb = totals[1];
        CK(ctx->bdesc.ensure((nb + 1) * zb_blkdesc_bytes()));
        CK(ctx->bexit.ensure((nb + 1) * zb_blkexit_bytes()));
        CK(ctx->erep.ensure((nb + 1) * 3 * sizeof(u32)));
        CK(ctx->fend.ensure(n * sizeof(u64)));
        CK(ctx->wave.ensure(zb_wave_bytes(nf, nb)));
        // FEW frames of many blocks (one huge frame at the limit): the copy-execute chain of a frame is serial however it is
        // mapped, so it is shortened by pointer doubling instead (zb_chase_*); many frames keep the machine busy frame-parallel
        int const force_chase = getenv("ZB200_CHASE") ? atoi(getenv("ZB200_CHASE")) : -1;
        chase_path = chain || (force_chase >= 0 ? force_chase != 0 : (nf < 64 && nb >= 8ull * nf));
        if (chain) CK(ctx->chase.ensure(zb_chase_bytes(totals[0])));      // frames of a chain are not independent: no other execute
        else if (chase_path && ctx->chase.ensure(zb_chase_bytes(totals[0])) != cudaSuccess) { cudaGetLastError(); chase_path = false; }
        { KSpan s(ctx, ZB200_K_SCAN);
          zb_launch_scan_blocks(d_src, d_segs, nf, ctx->place.as<ZbFramePlace>(), dd, ctx->status.as<u32>(), ctx->bdesc.p, ctx->fend.as<u64>(), ctx->biglist.as<u32>(), ctx->stream); }
        { KSpan s(ctx, ZB200_K_ENTROPY);
          zb_launch_entropy_blocks(d_src, ctx->bdesc.p, (u32)nb, ctx->blocks.as<ZbBlock>(), ctx->seqs.as<ZbSeq>(), ctx->lits.as<u8>(),
                                   zb_entropy_blocks_ctas(nb, ctas), d_counter, dd, ctx->status.as<u32>(), ctx->bexit.p, ZB_BLOCKS_TAKE, ctx->stream); }
        { KSpan s(ctx, ZB200_K_PLACE);
          zb_launch_resolve_blocks(d_src, d_segs, nf, ctx->place.as<ZbFramePlace>(), ctx->info.as<ZbFrameInfo>(), exact_sizes ? d_dst_sizes : nullptr,
                                   ctx->blocks.as<ZbBlock>(), ctx->bdesc.p, ctx->bexit.p, ctx->fend.as<u64>(), nb, ctx->seqs.as<ZbSeq>(), dd,
                                   ctx->status.as<u32>(), ctx->out_sizes.as<u64>(), ctx->ck.as<u32>(), ctx->erep.as<u32>(), ctx->stream, chain != nullptr); }
    }
    res->n = n; res->size = totals[0];
    if (copy_back) {
        res->data = pinned_get(ctx, totals[0] ? totals[0] : 1);
        if (!res->data) return fail(ctx, "pinned output allocation", cudaErrorMemoryAllocation);
        res->data_pinned_pool = true;
    }
    for (u32 k = 0; k < n_chunks; k++) {
        u32 const f0 = cut[k], f1 = cut[k + 1];
        u32* const counter = n_chunks > 1 ? d_counter + 8 + k : d_counter;
        if (!block_path) { KSpan s(ctx, ZB200_K_ENTROPY);
          ZbChunkShape const sh = zb_chunk_shape(n_chunks > 1 ? cpl[k + 1].dst_off - cpl[k].dst_off : totals[0], f1 - f0, ctas);
          zb_launch_entropy(d_src, d_segs, f1, ctx->place.as<ZbFramePlace>(), exact_sizes ? d_dst_sizes : nullptr, ctx->blocks.as<ZbBlock>(),
                            ctx->seqs.as<ZbSeq>(), ctx->lits.as<u8>(), sh.ctas, counter, dd,
                            ctx->status.as<u32>(), ctx->out_sizes.as<u64>(), ctx->ck.as<u32>(), sh.take, sh.warps, ctx->stream); }
        { KSpan s(ctx, ZB200_K_EXECUTE);
          if (chase_path) {
              int const r = zb_launch_execute_chase(d_src, ctx->place.as<ZbFramePlace>(), ctx->status.as<u32>(), ctx->blocks.as<ZbBlock>(), ctx->bdesc.p,
                                                    ctx->seqs.as<ZbSeq>(), ctx->lits.as<u8>(), d_out,
                                                    n_chunks > 1 ? cpl[k].dst_off : 0, n_chunks > 1 ? cpl[k + 1].dst_off : totals[0], totals[0],
                                                    n_chunks > 1 ? cpl[k].blk_off : 0, n_chunks > 1 ? cpl[k + 1].blk_off : totals[1],
                                                    ctx->chase.p, d_counter + 48, ctas, dd, ctx->stream, chain != nullptr);
              if (r < 0) return fail(ctx, "pointer-jumping execute", cudaGetLastError());
              ctx->last_chase_rounds = r;
          }
          else if (block_path) zb_launch_execute_big(d_src, ctx->place.as<ZbFramePlace>(), ctx->status.as<u32>(), ctx->blocks.as<ZbBlock>(), ctx->bdesc.p,
                                                ctx->seqs.as<ZbSeq>(), ctx->lits.as<u8>(), d_out, f0, f1,
                                                n_chunks > 1 ? cpl[k].blk_off : 0, n_chunks > 1 ? cpl[k + 1].blk_off : totals[1],
                                                nf, totals[1], ctx->wave.p, ctas, dd, ctx->stream);
          else zb_launch_execute(d_src, ctx->place.as<ZbFramePlace>(), ctx->status.as<u32>(), ctx->blocks.as<ZbBlock>(),
                                 ctx->seqs.as<ZbSeq>(), ctx->lits.as<u8>(), d_out, f0, f1, dd, ctx->stream); }
        if (totals[4]) { KSpan s(ctx, ZB200_K_VERIFY);
          zb_launch_verify(d_out, ctx->place.as<ZbFramePlace>(), ctx->out_sizes.as<u64>(), ctx->info.as<ZbFrameInfo>(),
                           ctx->ck.as<u32>(), f0, f1, ctx->status.as<u32>(), ctx->stream); }
        if (copy_back && n_chunks > 1) {
            CK(cudaEventRecord(ctx->chunk_ev[k], ctx->stream));
            CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->chunk_ev[k], 0));
            u64 const o0 = cpl[k].dst_off, o1 = cpl[k + 1].dst_off;
            if (o1 > o0) CK(cudaMemcpyAsync((u8*)res->data + o0, d_out + o0, o1 - o0, cudaMemcpyDeviceToHost, ctx->copy_stream));
        }
    }
    // The segment table.  Its memory is taken only now, with the decode kernels queued: nothing they do not need runs while
    // the device waits.  A result that stays on the device keeps its table in an allocation of its own (stream-ordered
    // pool) until the caller asks for it (zb200_result_segments); the others copy it into a block of the pinned pool.
    ZbSegment* d_table = ctx->out_segs.as<ZbSegment>();
    if (res->data_owned_device) {
        void* p = nullptr; CK(cudaMallocAsync(&p, n * sizeof(ZbSegment), ctx->stream));
        d_table = (ZbSegment*)p; res->segs_device = d_table;
    }
    { KSpan s(ctx, ZB200_K_FINISH);
      zb_launch_finish(ctx->place.as<ZbFramePlace>(), ctx->out_sizes.as<u64>(), ctx->status.as<u32>(), nf,
                       d_table, d_first_err, ctx->stream); }
    if (!res->segs_device) {
        res->segs_pinned = (zb200_segment*)pinned_get(ctx, n * sizeof(ZbSegment));
        if (!res->segs_pinned) return fail(ctx, "pinned segment table", cudaErrorMemoryAllocation);
        CK(cudaMemcpyAsync(res->segs_pinned, d_table, n * sizeof(ZbSegment), cudaMemcpyDeviceToHost, ctx->stream));
    }
    u32 first_err = 0xFFFFFFFFu;
    CK(cudaMemcpyAsync(&first_err, d_first_err, sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
    if (copy_back && n_chunks == 1) CK(cudaMemcpyAsync(res->data, d_out, totals[0], cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (copy_back && n_chunks > 1) CK(cudaStreamSynchronize(ctx->copy_stream));
    if (ctx->prof) fold_spans(ctx);
    if (first_err != 0xFFFFFFFFu) {
        u32 code = 0; u64 got = 0; ZbFramePlace pl;
        cudaMemcpy(&code, ctx->status.as<u32>() + first_err, sizeof code, cudaMemcpyDeviceToHost);
        cudaMemcpy(&pl, ctx->place.as<ZbFramePlace>() + first_err, sizeof pl, cudaMemcpyDeviceToHost);
        cudaMemcpy(&got, ctx->out_sizes.as<u64>() + first_err, sizeof got, cudaMemcpyDeviceToHost);     // what the frame regenerated (size mismatch)
        res->has_error = true; res->err_item = first_err; res->err_code = (int)code; res->err_got = got; res->err_expected = pl.dst_cap;
    }
    return 0;
}

static u64 window_limit_of(const zb200_dparams* p)
{
    // ZSTD_MAXWINDOWSIZE_DEFAULT = (1 << ZSTD_WINDOWLOG_LIMIT_DEFAULT) + 1 (zstd/zstd.c:43465, :5585)
    return p && p->max_window_size ? p->max_window_size : ((1ull << 27) + 1);
}

static int decompress_common(zb200_ctx* ctx, const void* src_base, const zb200_segment* segs, size_t n,
                             const uint64_t* dst_sizes, const zb200_ddict* dict, uint32_t flags, zb200_result** out,
                             const zb200_dparams* dparams = nullptr)
{
    *out = nullptr;
    if (!ctx || !segs || n == 0 || n > 0x7FFFFFF0u) return fail(ctx, "zb200_decompress_batch: bad arguments", cudaSuccess);
    cudaSetDevice(ctx->device);
    const u8* d_src; const ZbSegment* d_segs; const u64* d_dst_sizes = nullptr;
    if ((flags & ZB200_SRC_DEVICE) && (flags & ZB200_SEGS_HOST)) {
        // the frames are on the device, their table (and the sizes) on the host: only those are uploaded
        CK(ctx->segs.ensure(n * sizeof(ZbSegment)));
        if (dst_sizes) CK(ctx->dst_sizes.ensure(n * sizeof(u64)));
        CK(cudaMemcpyAsync(ctx->segs.p, segs, n * sizeof(ZbSegment), cudaMemcpyHostToDevice, ctx->stream));
        if (dst_sizes) CK(cudaMemcpyAsync(ctx->dst_sizes.p, dst_sizes, n * sizeof(u64), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));          // (the caller's tables may go away)
        d_src = (const u8*)src_base; d_segs = ctx->segs.as<ZbSegment>();
        if (dst_sizes) d_dst_sizes = ctx->dst_sizes.as<u64>();
    } else if (flags & ZB200_SRC_DEVICE) {
        d_src = (const u8*)src_base; d_segs = (const ZbSegment*)segs; d_dst_sizes = dst_sizes;
    } else {
        // host input: one contiguous copy of the referenced span (the data a BufferWithSegments holds)
        u64 lo = ~0ull, hi = 0;
        for (size_t i = 0; i < n; i++) { if (segs[i].offset < lo) lo = segs[i].offset; if (segs[i].offset + segs[i].length > hi) hi = segs[i].offset + segs[i].length; }
        if (hi < lo) { lo = hi = 0; }
        CK(ctx->src.ensure(hi - lo + 64));
        CK(ctx->segs.ensure(n * sizeof(ZbSegment)));
        if (dst_sizes) CK(ctx->dst_sizes.ensure(n * sizeof(u64)));
        std::vector<zb200_segment> tmp;
        {
            std::lock_guard<std::mutex> up(g_upload_mu[ctx->device & 15]);
            CK(cudaMemcpyAsync(ctx->src.p, (const u8*)src_base + lo, hi - lo, cudaMemcpyHostToDevice, ctx->stream));
            if (lo == 0) CK(cudaMemcpyAsync(ctx->segs.p, segs, n * sizeof(ZbSegment), cudaMemcpyHostToDevice, ctx->stream));
            else {
                tmp.assign(segs, segs + n);
                for (auto& s : tmp) s.offset -= lo;
                CK(cudaMemcpyAsync(ctx->segs.p, tmp.data(), n * sizeof(ZbSegment), cudaMemcpyHostToDevice, ctx->stream));
            }
            if (dst_sizes) CK(cudaMemcpyAsync(ctx->dst_sizes.p, dst_sizes, n * sizeof(u64), cudaMemcpyHostToDevice, ctx->stream));
            CK(cudaStreamSynchronize(ctx->stream));
        }
        d_src = ctx->src.as<u8>(); d_segs = ctx->segs.as<ZbSegment>();
        if (dst_sizes) d_dst_sizes = ctx->dst_sizes.as<u64>();
    }
    zb200_result* res = new zb200_result(); res->ctx = ctx;
    int rc = run_decompress(ctx, d_src, d_segs, n, d_dst_sizes, dict, res, !(flags & ZB200_DST_DEVICE),
                            !(flags & ZB200_SIZES_ARE_CAPACITY), window_limit_of(dparams));
    if (rc) { zb200_result_free(res); return rc; }
    *out = res;
    return 0;
}

int zb200_decompress_batch(zb200_ctx* ctx, const void* src_base, const zb200_segment* segs, size_t n,
                           const uint64_t* dst_sizes, const zb200_ddict* dict, uint32_t flags, zb200_result** out)
{
    return decompress_common(ctx, src_base, segs, n, dst_sizes, dict, flags, out);
}

int zb200_decompress_batch_ex(zb200_ctx* ctx, const void* src_base, const zb200_segment* segs, size_t n,
                              const uint64_t* dst_sizes, const zb200_ddict* dict, const zb200_dparams* params, uint32_t flags, zb200_result** out)
{
    return decompress_common(ctx, src_base, segs, n, dst_sizes, dict, flags, out, params);
}

int zb200_decompress_batch_ptrs(zb200_ctx* ctx, const void* const* srcs, const size_t* sizes, size_t n,
                                const uint64_t* dst_sizes, const zb200_ddict* dict, uint32_t flags, zb200_result** out)
{
    return zb200_decompress_batch_ptrs_ex(ctx, srcs, sizes, n, dst_sizes, dict, nullptr, flags, out);
}

int zb200_decompress_batch_ptrs_ex(zb200_ctx* ctx, const void* const* srcs, const size_t* sizes, size_t n,
                                   const uint64_t* dst_sizes, const zb200_ddict* dict, const zb200_dparams* params, uint32_t flags, zb200_result** out)
{
    *out = nullptr;
    if (!ctx || !srcs || !sizes || n == 0) return fail(ctx, "zb200_decompress_batch_ptrs: bad arguments", cudaSuccess);
    cudaSetDevice(ctx->device);
    // gather the independent buffers into pinned staging (this is the copy a list-of-bytes input costs anyway)
    u64 total = 0; for (size_t i = 0; i < n; i++) total += sizes[i];
    u8* stage = (u8*)pinned_get(ctx, total ? total : 1);
    if (!stage) return fail(ctx, "pinned staging allocation", cudaErrorMemoryAllocation);
    std::vector<zb200_segment> segs(n); u64 pos = 0;
    for (size_t i = 0; i < n; i++) { memcpy(stage + pos, srcs[i], sizes[i]); segs[i].offset = pos; segs[i].length = sizes[i]; pos += sizes[i]; }
    int rc = decompress_common(ctx, stage, segs.data(), n, dst_sizes, dict, flags & ~ZB200_SRC_DEVICE, out, params);
    pinned_put(ctx, stage);
    return rc;
}

// ---------------------------------------------------------------- content-dictionary chains
// decompress_content_dict_chain (c-ext/decompressor.c:620-890): frame k is decoded with frame k-1's fulltext as a raw-content
// prefix, and only the last fulltext is returned.  The entropy stage of every frame is independent (a raw-content prefix
// brings no tables and no repcodes), so all frames of a run go through the block path side by side; only the LZ execute is
// chained, and the pointer-jumping stage shortens those chains across frame borders instead of following them.
// A run is as many consecutive frames as fit the memory budget; the next run starts from its last fulltext.
int zb200_decompress_chain(zb200_ctx* ctx, const void* const* srcs, const size_t* sizes, size_t n,
                           const zb200_ddict* first_dict, const zb200_dparams* params, zb200_result** out)
{
    *out = nullptr;
    if (!ctx || !srcs || !sizes || n == 0 || n > 0x7FFFFFF0u) return fail(ctx, "zb200_decompress_chain: bad arguments", cudaSuccess);
    cudaSetDevice(ctx->device);
    // ---- the header checks, chunk by chunk; the first chunk that fails one ends the chain (h): chunks [0, h) are decoded,
    // and a decode error among them wins, as when the reference decodes chunk k before it looks at chunk k + 1
    std::vector<u64> csize(n, 0);
    std::vector<char> skip(n, 0);
    size_t h = n; int h_code = 0;
    for (size_t k = 0; k < n && h == n; k++) {
        const u8* s = (const u8*)srcs[k];
        int code = 0;
        if (sizes[k] >= 4 && (zb_rd32(s) & 0xFFFFFFF0u) == ZB_MAGIC_SKIP) {
            // a skippable frame first: the reference's stream decoder stops behind it, so the fulltext is empty
            u64 const len = sizes[k] >= 8 ? zb_rd32(s + 4) : 0;
            if (sizes[k] < 8 + len) code = ZB_E_SRCSIZE_WRONG;
            skip[k] = 1;
        } else {
            zb200_frame_info_t fi; zb200_frame_info(s, sizes[k], &fi);
            if (fi.status) code = (int)fi.status;
            else if (fi.content_size == ~0ull) code = ZB200_E_UNKNOWN_SIZE;
            // the block path reads offsets of 2^31 and more as symbolic repcodes (DESIGN.md section 6); a match may reach
            // back over the whole prefix, so the prefix counts too
            else if (fi.content_size >= ZB_FAR_WINDOW || fi.window_size >= ZB_FAR_WINDOW
                     || (k && csize[k - 1] + fi.content_size >= ZB_FAR_WINDOW)) code = ZB_E_WINDOW_TOO_LARGE;
            // a raw-content prefix has dictionary ID 0, and zstd checks the header's ID against it (zstd/zstd.c:43938)
            else if (fi.dict_id && !(k == 0 && first_dict)) code = ZB_E_DICT_WRONG;
            else csize[k] = fi.content_size;
        }
        if (code) { h = k; h_code = code; }
    }
    zb200_result* res = new zb200_result(); res->ctx = ctx;
    auto finish = [&](int rc) { if (rc) zb200_result_free(res); else *out = res; return rc; };
    auto chunk_error = [&](size_t k, int code) { res->has_error = true; res->err_item = k; res->err_code = code; };
    // ---- every chunk before h goes to the device once
    u64 total = 0; for (size_t k = 0; k < h; k++) total += sizes[k];
    std::vector<zb200_segment> segs(h);
    if (h) {
        u8* stage = (u8*)pinned_get(ctx, total ? total : 1);
        if (!stage) return finish(fail(ctx, "pinned staging allocation", cudaErrorMemoryAllocation));
        u64 pos = 0;
        for (size_t k = 0; k < h; k++) { memcpy(stage + pos, srcs[k], sizes[k]); segs[k].offset = pos; segs[k].length = sizes[k]; pos += sizes[k]; }
        cudaError_t e = ctx->src.ensure(total + 64);
        if (e == cudaSuccess) e = ctx->segs.ensure(h * sizeof(ZbSegment));
        if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->src.p, stage, total, cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->segs.p, segs.data(), h * sizeof(ZbSegment), cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        pinned_put(ctx, stage);
        if (e != cudaSuccess) return finish(fail(ctx, "zb200_decompress_chain upload", e));
    }
    const u8* const d_src = ctx->src.as<u8>(); const ZbSegment* const d_segs = ctx->segs.as<ZbSegment>();
    u64 const wl = window_limit_of(params);
    u64 carry = 0;              // bytes of the last fulltext in ctx->carry
    size_t k = 0;
    // ---- chunk 0 with the decompressor's dictionary: on its own through the batch path; its output is the first carry
    if (h && first_dict && !skip[0]) {
        zb200_result* r0 = new zb200_result(); r0->ctx = ctx;
        int rc = run_decompress(ctx, d_src, d_segs, 1, nullptr, first_dict, r0, false, true, wl);
        cudaError_t e = cudaSuccess;
        if (!rc && !r0->has_error && csize[0]) {
            e = ctx->carry.ensure(csize[0]);
            if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->carry.p, r0->data, csize[0], cudaMemcpyDeviceToDevice, ctx->stream);
        }
        if (!rc && r0->has_error) chunk_error(0, r0->err_code);
        zb200_result_free(r0);
        if (rc) return finish(rc);
        if (e != cudaSuccess) return finish(fail(ctx, "zb200_decompress_chain carry", e));
        if (res->has_error) return finish(0);
        carry = csize[0]; k = 1;
    }
    // ---- runs: device bytes per chunk of output ~ 1 (fulltext) + 8 (pointer) + 5.3 (sequence records of >= 3-byte matches)
    // + 1 (literals); the budget is most of the free device memory, or ZB200_CHAIN_RUN_BYTES (read per call: tests force runs)
    u64 budget;
    {
        const char* env = getenv("ZB200_CHAIN_RUN_BYTES");
        size_t fr = 0, tot = 0; cudaMemGetInfo(&fr, &tot);
        budget = env && *env ? strtoull(env, nullptr, 10) : (u64)fr / 10 * 6;
    }
    auto cost = [&](size_t j) { return 16 * csize[j] + sizes[j] + 4096; };
    int rounds = 0;
    while (k < h) {
        if (skip[k]) { carry = 0; k++; continue; }
        size_t b = k + 1; u64 use = 16 * carry + cost(k);
        while (b < h && !skip[b] && use + cost(b) <= budget) use += cost(b++);
        zb200_result* rr = new zb200_result(); rr->ctx = ctx;
        ChainRun cr; cr.carry = carry;
        int rc = run_decompress(ctx, d_src, d_segs + k, b - k, nullptr, nullptr, rr, false, true, wl, &cr);
        rounds += ctx->last_chase_rounds;
        cudaError_t e = cudaSuccess;
        if (!rc && rr->has_error) chunk_error(k + rr->err_item, rr->err_code);
        else if (!rc) {         // the run's last fulltext becomes the next prefix
            zb200_segment const last = rr->segs_pinned[b - k - 1];
            carry = last.length;
            if (carry) e = ctx->carry.ensure(carry);
            if (carry && e == cudaSuccess) e = cudaMemcpyAsync(ctx->carry.p, ctx->dst.as<u8>() + last.offset, carry, cudaMemcpyDeviceToDevice, ctx->stream);
        }
        zb200_result_free(rr);
        if (rc) return finish(rc);
        if (e != cudaSuccess) return finish(fail(ctx, "zb200_decompress_chain carry", e));
        if (res->has_error) { ctx->last_chase_rounds = rounds; return finish(0); }
        k = b;
    }
    ctx->last_chase_rounds = rounds;
    if (h < n) { chunk_error(h, h_code); return finish(0); }
    // ---- the last fulltext, copied back alone
    res->data = pinned_get(ctx, carry ? carry : 1);
    if (!res->data) return finish(fail(ctx, "pinned output allocation", cudaErrorMemoryAllocation));
    res->data_pinned_pool = true;
    if (carry) {
        cudaError_t e = cudaMemcpyAsync(res->data, ctx->carry.p, carry, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) return finish(fail(ctx, "zb200_decompress_chain copy-back", e));
    }
    res->n = 1; res->size = carry; res->segs.assign(1, zb200_segment{0, carry});
    return finish(0);
}


// ---------------------------------------------------------------- batch compression
// d_stats (dictionary training): u32[377] on the device that the block kernel's STATS instantiation adds its literal and
// LL / ML / OF code counts to; only zb_compress_blocks has it, so such a call always runs that kernel
static int compress_common(zb200_ctx* ctx, const void* src_base, const zb200_segment* segs, size_t n,
                           const zb200_cparams* params, const zb200_ddict* dict, uint32_t flags, zb200_result** out, u32* d_stats = nullptr)
{
    *out = nullptr;
    if (!ctx || !segs || n == 0 || n > 0x7FFFFFF0u) return fail(ctx, "zb200_compress_batch: bad arguments", cudaSuccess);
    cudaSetDevice(ctx->device);
    double const tr0 = zb_trace_on() ? zb_now_ms() : 0; double tr1 = 0, tr2 = 0;
    zb200_cparams P; if (params) P = *params; else { memset(&P, 0, sizeof P); P.level = 3; P.write_content_size = 1; }
    if (P.window_log && (P.window_log < 10 || P.window_log > 31)) return fail(ctx, "zb200_compress_batch: window_log out of range [10, 31]", cudaSuccess);
    u32 const block_max = zb_block_max(P.window_log);
    std::vector<zb200_segment> hsegs;
    const u8* d_src; const ZbSegment* d_segs;
    const u8* up_src = nullptr; u64 up_bytes = 0;          // host input to upload while the kernel runs
    if ((flags & ZB200_SRC_DEVICE) && (flags & ZB200_SEGS_HOST)) {
        hsegs.assign(segs, segs + n);
        CK(ctx->segs.ensure(n * sizeof(ZbSegment)));
        CK(cudaMemcpyAsync(ctx->segs.p, segs, n * sizeof(ZbSegment), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));          // (the caller's table may go away)
        d_src = (const u8*)src_base; d_segs = ctx->segs.as<ZbSegment>();
    } else if (flags & ZB200_SRC_DEVICE) {
        hsegs.resize(n);
        CK(cudaMemcpyAsync(hsegs.data(), segs, n * sizeof(ZbSegment), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        d_src = (const u8*)src_base; d_segs = (const ZbSegment*)segs;
    } else {
        hsegs.assign(segs, segs + n);
        u64 lo = ~0ull, hi = 0;
        for (size_t i = 0; i < n; i++) { if (segs[i].offset < lo) lo = segs[i].offset; if (segs[i].offset + segs[i].length > hi) hi = segs[i].offset + segs[i].length; }
        if (hi < lo) { lo = hi = 0; }
        for (auto& s : hsegs) s.offset -= lo;
        CK(ctx->src.ensure(hi - lo + 512));
        CK(ctx->segs.ensure(n * sizeof(ZbSegment)));
        CK(cudaMemcpyAsync(ctx->segs.p, hsegs.data(), n * sizeof(ZbSegment), cudaMemcpyHostToDevice, ctx->stream));
        // the input itself is uploaded in chunks on the copy stream AFTER the block kernel has been launched: the kernel
        // waits per block for the bytes it needs (ZeUpload), so the upload hides behind the compression of earlier blocks
        up_src = (const u8*)src_base + lo; up_bytes = hi - lo;
        d_src = ctx->src.as<u8>(); d_segs = ctx->segs.as<ZbSegment>();
    }
    if (zb_trace_on()) tr1 = zb_now_ms();
    std::vector<ZeBlockJob> jobs; std::vector<ZeSegInfo> sinfo(n);
    jobs.reserve(n);
    u32 const max_block = zb_cut_blocks(hsegs.data(), n, block_max, jobs, sinfo);
    size_t const nj = jobs.size();
    u64 const slot_bytes = zb_slot_bytes(max_block);
    // Blocks of 8 KiB and more (no dictionary, level-3 class) take the round-2 kernel: one CTA per SM with the block resident in
    // shared memory.  Small blocks, dictionaries and the level >= 4 mode stay on the CTA-per-block kernel (6 CTAs per SM).
    static int const force_v1 = getenv("ZB200_ENCODER_V1") ? atoi(getenv("ZB200_ENCODER_V1")) : 0;
    bool const smem_kernel = !dict && P.level < 4 && max_block >= 8192 && !force_v1 && !d_stats;
    // Small records with a full dictionary (config 4): a warp per record, 22 records per SM (zb_encode3.cuh).
    bool const recs_kernel = dict && dict->c_D >= 8 && dict->dev.has_entropy && dict->d_cct && P.level < 4 && nj != 0 &&
                             max_block <= zb_encode3_record_max() && !force_v1 && !d_stats;
    u32 ctas = smem_kernel ? (u32)ctx->sm_count : (u32)ctx->sm_count * (227u * 1024u / zb_encode_smem_bytes());
    if (recs_kernel) { ctas = (u32)ctx->sm_count; u32 const need = ((u32)nj + zb_encode3_records_per_cta() - 1) / zb_encode3_records_per_cta(); if (ctas > need) ctas = need; }
    if (ctas > nj) ctas = (u32)nj;
    if (ctas == 0) ctas = 1;
    CK(ctx->jobs.ensure((nj + 1) * sizeof(ZeBlockJob)));
    CK(ctx->seginfo.ensure(n * sizeof(ZeSegInfo)));
    CK(ctx->slots.ensure((nj + 1) * slot_bytes));
    CK(ctx->bouts.ensure((nj + 1) * sizeof(ZeBlockOut)));
    if (!recs_kernel) CK(ctx->escratch.ensure((size_t)ctas * (smem_kernel ? zb_encode2_scratch_bytes() : zb_encode_scratch_bytes())));
    CK(ctx->fsizes.ensure(n * sizeof(u64)));
    CK(ctx->out_segs.ensure(n * sizeof(ZbSegment)));
    CK(ctx->small.ensure(256));
    u64* d_total = ctx->small.as<u64>();
    u32* d_counter = (u32*)(d_total + 8);
    if (nj) CK(cudaMemcpyAsync(ctx->jobs.p, jobs.data(), nj * sizeof(ZeBlockJob), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->seginfo.p, sinfo.data(), n * sizeof(ZeSegInfo), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(d_counter, 0, 64, ctx->stream));                       // work counter, upload status, upload progress
    u32* const d_upstatus = d_counter + 1;
    unsigned long long* const d_progress = (unsigned long long*)(d_counter + 4);
    bool const overlap_upload = up_bytes != 0 && nj != 0 && ctx->h_progress != nullptr;
    if (up_bytes && !overlap_upload) CK(cudaMemcpyAsync(ctx->src.p, up_src, up_bytes, cudaMemcpyHostToDevice, ctx->stream));
    if (overlap_upload) {
        CK(cudaEventRecord(ctx->chunk_ev[0], ctx->stream)); CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->chunk_ev[0], 0));
        // The whole upload is queued BEFORE the block kernel is launched: the kernel spins until its bytes have landed, so
        // every copy it waits for must already be in the device's queues.  Queued after the launch, the copies depend on
        // this thread reaching them, and a device-synchronising call of another thread (cudaFree in DevBuf::ensure, with
        // a second context's kernel in flight) can hold it back until the kernel gives up.
        // <= 48 chunks of >= 4 MiB; after each chunk the copy engine also writes the new byte count next to the work counter
        u64 chunk = (up_bytes + 47) / 48; if (chunk < ((u64)4 << 20)) chunk = (u64)4 << 20; chunk = (chunk + 255) & ~(u64)255;
        u32 k = 0;
        for (u64 pos = 0; pos < up_bytes; pos += chunk, k++) {
            u64 const len = up_bytes - pos < chunk ? up_bytes - pos : chunk;
            CK(cudaMemcpyAsync((u8*)ctx->src.p + pos, up_src + pos, len, cudaMemcpyHostToDevice, ctx->copy_stream));
            ctx->h_progress[k] = pos + len;
            CK(cudaMemcpyAsync(d_progress, &ctx->h_progress[k], sizeof(unsigned long long), cudaMemcpyHostToDevice, ctx->copy_stream));
        }
        CK(cudaEventRecord(ctx->chunk_ev[1], ctx->copy_stream));
    }
    ctx->last_compress_kernel = recs_kernel ? "zb_compress_recs" : (smem_kernel ? "zb_compress_smem" : "zb_compress_blocks");
    if (recs_kernel) { KSpan s(ctx, ZB200_K_COMPRESS);
      zb_launch_compress_recs(d_src, ctx->jobs.as<ZeBlockJob>(), (u32)nj, ctas, ctx->slots.as<u8>(), slot_bytes, ctx->bouts.as<ZeBlockOut>(), d_counter,
                              dict->c_tail, dict->c_D, dict->d_ctable, (const void*)dict->d_digest, dict->d_cct,
                              overlap_upload ? d_progress : nullptr, up_bytes, d_upstatus, ctx->stream); }
    else if (nj && smem_kernel) { KSpan s(ctx, ZB200_K_COMPRESS);
      zb_launch_compress_smem(d_src, ctx->jobs.as<ZeBlockJob>(), (u32)nj, ctx->escratch.p, ctas, ctx->slots.as<u8>(), slot_bytes, ctx->bouts.as<ZeBlockOut>(), d_counter,
                              overlap_upload ? d_progress : nullptr, up_bytes, d_upstatus, ctx->stream); }
    else if (nj) { KSpan s(ctx, ZB200_K_COMPRESS);
      zb_launch_compress_blocks(d_src, ctx->jobs.as<ZeBlockJob>(), (u32)nj, ctx->escratch.p, ctas, ctx->slots.as<u8>(), slot_bytes, ctx->bouts.as<ZeBlockOut>(), d_counter,
                                dict ? dict->c_tail : nullptr, dict ? dict->c_D : 0, dict ? dict->d_ctable : nullptr,
                                (dict && dict->c_D && dict->dev.has_entropy) ? (const void*)dict->d_digest : nullptr, dict ? dict->d_cct : nullptr,
                                overlap_upload ? d_progress : nullptr, up_bytes, d_upstatus, P.level >= 4 ? 1 : 0, max_block <= zb_encode_small_max() ? 1 : 0, ctx->stream, d_stats); }
    // the layout kernels read the input again (raw blocks): they wait for the whole upload, whatever order the segments came in
    if (overlap_upload) CK(cudaStreamWaitEvent(ctx->stream, ctx->chunk_ev[1], 0));
    { KSpan s(ctx, ZB200_K_LAYOUT);
      zb_launch_frame_layout(d_segs, ctx->seginfo.as<ZeSegInfo>(), ctx->bouts.as<ZeBlockOut>(), (u32)n, P.write_checksum ? 1 : 0, P.write_content_size ? 1 : 0, P.dict_id, P.window_log,
                             ctx->fsizes.as<u64>(), ctx->out_segs.as<ZbSegment>(), d_total, ctx->stream); }
    u64 total = 0; u32 upstatus = 0;
    CK(cudaMemcpyAsync(&total, d_total, sizeof total, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(&upstatus, d_upstatus, sizeof upstatus, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (overlap_upload) CK(cudaStreamSynchronize(ctx->copy_stream));
    if (upstatus) return fail(ctx, "zb200_compress_batch: the input upload did not complete", cudaErrorUnknown);
    if (zb_trace_on()) tr2 = zb_now_ms();
    // the result is held by a unique_ptr until it is handed out: every early return below frees it (and its buffers)
    std::unique_ptr<zb200_result, void (*)(zb200_result*)> res(new zb200_result(), zb200_result_free);
    res->ctx = ctx; res->n = n; res->size = total; res->segs.resize(n);
    u8* d_out;
    if (!(flags & ZB200_DST_DEVICE)) { CK(ctx->dst.ensure(total + 64)); d_out = ctx->dst.as<u8>(); }
    else {      // a device-resident result owns its allocation: later calls on this context leave it alone
        void* p = nullptr; CK(cudaMallocAsync(&p, total + 64, ctx->stream));
        d_out = (u8*)p; res->data = p; res->data_on_device = true; res->data_owned_device = true;
    }
    { KSpan s(ctx, ZB200_K_FRAMES);
      zb_launch_write_frames(d_src, d_segs, ctx->seginfo.as<ZeSegInfo>(), ctx->bouts.as<ZeBlockOut>(), ctx->slots.as<u8>(), slot_bytes, (u32)n, P.write_checksum ? 1 : 0,
                             P.write_content_size ? 1 : 0, P.dict_id, P.window_log, ctx->out_segs.as<ZbSegment>(), d_out, ctx->stream); }
    CK(cudaMemcpyAsync(res->segs.data(), ctx->out_segs.p, n * sizeof(ZbSegment), cudaMemcpyDeviceToHost, ctx->stream));
    if (!(flags & ZB200_DST_DEVICE)) {
        res->data = pinned_get(ctx, total ? total : 1);
        if (!res->data) return fail(ctx, "pinned output allocation", cudaErrorMemoryAllocation);
        res->data_pinned_pool = true;
        CK(cudaMemcpyAsync(res->data, d_out, total, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CK(cudaStreamSynchronize(ctx->stream));
    if (ctx->prof) fold_spans(ctx);
    ctx->last_scratch = (recs_kernel ? 0ull : (u64)ctas * (smem_kernel ? zb_encode2_scratch_bytes() : zb_encode_scratch_bytes())) + nj * slot_bytes;
    if (zb_trace_on()) { double const tr3 = zb_now_ms();
        fprintf(stderr, "[zb200] compress ctx %p n=%zu blocks=%zu: start %.3f upload %.2f kernels %.2f frames+download %.2f ms\n",
                (void*)ctx, n, nj, tr0, tr1 - tr0, tr2 - tr1, tr3 - tr2); }
    *out = res.release();
    return 0;
}

int zb200_compress_batch(zb200_ctx* ctx, const void* src_base, const zb200_segment* segs, size_t n,
                         const zb200_cparams* params, const zb200_ddict* dict, uint32_t flags, zb200_result** out)
{
    return compress_common(ctx, src_base, segs, n, params, dict, flags, out);
}

int zb200_compress_batch_ptrs(zb200_ctx* ctx, const void* const* srcs, const size_t* sizes, size_t n,
                              const zb200_cparams* params, const zb200_ddict* dict, uint32_t flags, zb200_result** out)
{
    *out = nullptr;
    if (!ctx || !srcs || !sizes || n == 0) return fail(ctx, "zb200_compress_batch_ptrs: bad arguments", cudaSuccess);
    cudaSetDevice(ctx->device);
    u64 total = 0; for (size_t i = 0; i < n; i++) total += sizes[i];
    u8* stage = (u8*)pinned_get(ctx, total ? total : 1);
    if (!stage) return fail(ctx, "pinned staging allocation", cudaErrorMemoryAllocation);
    std::vector<zb200_segment> segs(n); u64 pos = 0;
    for (size_t i = 0; i < n; i++) { if (sizes[i]) memcpy(stage + pos, srcs[i], sizes[i]); segs[i].offset = pos; segs[i].length = sizes[i]; pos += sizes[i]; }
    int rc = compress_common(ctx, stage, segs.data(), n, params, dict, flags & ~ZB200_SRC_DEVICE, out);
    pinned_put(ctx, stage);
    return rc;
}

// ---------------------------------------------------------------- content-dictionary chains, compression
// The inverse of zb200_decompress_chain: frame k is chunk k compressed with chunk k-1 as a raw-content prefix.  Chunk 0 goes
// through the batch path with the dictionary; every later chunk is independent work once all chunks are known, so a run of
// them is one batch: the chunks back to back on the device (chunk k-1 directly in front of chunk k), an index per chunk
// (zb_chain_index), every block through the prefix mode of zb_compress_blocks, the frames laid out by the batch kernels with
// window_log 31 (single segment: the window is the content size, so offsets may reach the whole prefix, RFC 8878 section 3.1.1.1.2).
int zb200_compress_chain(zb200_ctx* ctx, const void* const* srcs, const size_t* sizes, size_t n,
                         const zb200_cparams* params, const zb200_ddict* dict, zb200_result** out)
{
    *out = nullptr;
    if (!ctx || !srcs || !sizes || n == 0 || n > 0x7FFFFFF0u) return fail(ctx, "zb200_compress_chain: bad arguments", cudaSuccess);
    for (size_t k = 0; k < n; k++)       // the chain decoder's limit (ZB_FAR_WINDOW); the Python layer checks it first
        if (sizes[k] >= ZB_FAR_WINDOW || (k && sizes[k - 1] + sizes[k] >= ZB_FAR_WINDOW)) return fail(ctx, "zb200_compress_chain: chunk of ZB_FAR_WINDOW or more", cudaSuccess);
    cudaSetDevice(ctx->device);
    zb200_cparams P; if (params) P = *params; else { memset(&P, 0, sizeof P); P.level = 3; }
    P.write_content_size = 1;
    std::vector<u8> host;                       // the frames, back to back (becomes the result's buffer)
    std::vector<zb200_segment> fsegs(n);
    // ---- chunk 0: the batch path, exactly as compress() with content size on
    {
        zb200_result* r0 = nullptr;
        int rc = zb200_compress_batch_ptrs(ctx, srcs, sizes, 1, &P, dict, 0, &r0);
        if (rc) return rc;
        host.assign((const u8*)r0->data, (const u8*)r0->data + r0->size);
        fsegs[0].offset = 0; fsegs[0].length = r0->size;
        zb200_result_free(r0);
    }
    // ---- runs of chunks 1..n-1.  Device bytes per input byte: 1 (input) + <= 8 (index, two keys per 4 bytes) + ~1 (block slots); the budget is most
    // of the free device memory, or ZB200_CHAIN_RUN_BYTES (read per call: tests force runs)
    u64 budget;
    {
        const char* env = getenv("ZB200_CHAIN_RUN_BYTES");
        size_t fr = 0, tot = 0; cudaMemGetInfo(&fr, &tot);
        budget = env && *env ? strtoull(env, nullptr, 10) : (u64)fr / 10 * 6;
    }
    auto cost = [&](size_t j) { return (u64)sizes[j] + (4ull << zb_chain_log(sizes[j])) + sizes[j] + (sizes[j] >> 7) + 4096 + 200 * (sizes[j] / ZB_BLOCK_MAX + 1); };
    u64 const slot_bytes = zb_slot_bytes(ZB_BLOCK_MAX);
    u32 const ctas_max = (u32)ctx->sm_count * (227u * 1024u / zb_encode_smem_bytes());
    size_t k = 1;
    while (k < n) {
        size_t b = k + 1; u64 use = cost(k - 1) + cost(k);
        while (b < n && use + cost(b) <= budget) use += cost(b++);
        size_t const m = b - (k - 1);            // staged chunks: k-1 (the prefix) .. b-1
        // pinned staging: 64 bytes of slack on both sides (the kernels read a few bytes around what they compare)
        u64 total = 0; for (size_t j = k - 1; j < b; j++) total += sizes[j];
        u8* stage = (u8*)pinned_get(ctx, total + 128);
        if (!stage) return fail(ctx, "pinned staging allocation", cudaErrorMemoryAllocation);
        memset(stage, 0, 64); memset(stage + 64 + total, 0, 64);
        // the chunks in the staging buffer; chunks 1..m-1 are the frames' segments
        std::vector<zb200_segment> rsegs(m);
        for (size_t i = 0, pos = 64; i < m; pos += sizes[k - 1 + i], i++) {
            if (sizes[k - 1 + i]) memcpy(stage + pos, srcs[k - 1 + i], sizes[k - 1 + i]);
            rsegs[i].offset = pos; rsegs[i].length = sizes[k - 1 + i];
        }
        std::vector<ZeChainSeg> cs(m); std::vector<u64> tab_off(m + 1), pos_off(m + 1);
        std::vector<ZeBlockJob> jobs; std::vector<ZeSegInfo> sinfo(m - 1);
        zb_chain_plan(rsegs.data(), m, cs.data(), tab_off.data(), pos_off.data(), jobs, sinfo);
        size_t const nj = jobs.size(), nf = m - 1;
        u32 ctas = ctas_max; if (ctas > nj) ctas = (u32)nj; if (ctas == 0) ctas = 1;
        cudaError_t e = ctx->src.ensure(total + 128);
        if (e == cudaSuccess) e = ctx->chain_tab.ensure(tab_off[m] * 4);
        if (e == cudaSuccess) e = ctx->chain_seg.ensure(m * sizeof(ZeChainSeg));
        if (e == cudaSuccess) e = ctx->chain_pos.ensure((m + 1) * sizeof(u64));
        if (e == cudaSuccess) e = ctx->segs.ensure(nf * sizeof(ZbSegment));
        if (e == cudaSuccess) e = ctx->jobs.ensure((nj + 1) * sizeof(ZeBlockJob));
        if (e == cudaSuccess) e = ctx->seginfo.ensure(nf * sizeof(ZeSegInfo));
        if (e == cudaSuccess) e = ctx->slots.ensure((nj + 1) * slot_bytes);
        if (e == cudaSuccess) e = ctx->bouts.ensure((nj + 1) * sizeof(ZeBlockOut));
        if (e == cudaSuccess) e = ctx->escratch.ensure((size_t)ctas * zb_encode_pscratch_bytes());
        if (e == cudaSuccess) e = ctx->fsizes.ensure(nf * sizeof(u64));
        if (e == cudaSuccess) e = ctx->out_segs.ensure(nf * sizeof(ZbSegment));
        if (e == cudaSuccess) e = ctx->small.ensure(256);
        if (e != cudaSuccess) { pinned_put(ctx, stage); return fail(ctx, "zb200_compress_chain allocation", e); }
        u8* const d_src = ctx->src.as<u8>(); u32* const d_tab = ctx->chain_tab.as<u32>();
        for (size_t i = 0; i < m; i++) { cs[i].tab = d_tab + tab_off[i]; cs[i].prev_tab = i ? d_tab + tab_off[i - 1] : nullptr; }
        u64* d_total = ctx->small.as<u64>(); u32* d_counter = (u32*)(d_total + 8);
        e = cudaMemcpyAsync(d_src, stage, total + 128, cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_tab, 0xFF, tab_off[m] * 4, ctx->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->chain_seg.p, cs.data(), m * sizeof(ZeChainSeg), cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->chain_pos.p, pos_off.data(), (m + 1) * sizeof(u64), cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->segs.p, rsegs.data() + 1, nf * sizeof(ZbSegment), cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess && nj) e = cudaMemcpyAsync(ctx->jobs.p, jobs.data(), nj * sizeof(ZeBlockJob), cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->seginfo.p, sinfo.data(), nf * sizeof(ZeSegInfo), cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_counter, 0, 64, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);          // (the staging block goes back to the pool)
        pinned_put(ctx, stage);
        if (e != cudaSuccess) return fail(ctx, "zb200_compress_chain upload", e);
        { KSpan s(ctx, ZB200_K_CHAIN_INDEX);
          zb_launch_chain_index(d_src, ctx->chain_seg.as<ZeChainSeg>(), ctx->chain_pos.as<u64>(), (u32)m, pos_off[m], (u32)ctx->sm_count, ctx->stream); }
        if (nj) { KSpan s(ctx, ZB200_K_COMPRESS);
          zb_launch_compress_chain_blocks(d_src, ctx->jobs.as<ZeBlockJob>(), (u32)nj, ctx->escratch.p, ctas, ctx->slots.as<u8>(), slot_bytes, ctx->bouts.as<ZeBlockOut>(), d_counter,
                                          ctx->chain_seg.as<ZeChainSeg>(), ctx->stream); }
        { KSpan s(ctx, ZB200_K_LAYOUT);
          zb_launch_frame_layout(ctx->segs.as<ZbSegment>(), ctx->seginfo.as<ZeSegInfo>(), ctx->bouts.as<ZeBlockOut>(), (u32)nf, P.write_checksum ? 1 : 0, 1, 0, 31,
                                 ctx->fsizes.as<u64>(), ctx->out_segs.as<ZbSegment>(), d_total, ctx->stream); }
        u64 ftotal = 0;
        CK(cudaMemcpyAsync(&ftotal, d_total, sizeof ftotal, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        CK(ctx->dst.ensure(ftotal + 64));
        { KSpan s(ctx, ZB200_K_FRAMES);
          zb_launch_write_frames(d_src, ctx->segs.as<ZbSegment>(), ctx->seginfo.as<ZeSegInfo>(), ctx->bouts.as<ZeBlockOut>(), ctx->slots.as<u8>(), slot_bytes, (u32)nf,
                                 P.write_checksum ? 1 : 0, 1, 0, 31, ctx->out_segs.as<ZbSegment>(), ctx->dst.as<u8>(), ctx->stream); }
        std::vector<ZbSegment> osegs(nf);
        size_t const base = host.size();
        host.resize(base + ftotal);
        CK(cudaMemcpyAsync(osegs.data(), ctx->out_segs.p, nf * sizeof(ZbSegment), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaMemcpyAsync(host.data() + base, ctx->dst.p, ftotal, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        if (ctx->prof) fold_spans(ctx);
        for (size_t f = 0; f < nf; f++) { fsegs[k + f].offset = base + osegs[f].offset; fsegs[k + f].length = osegs[f].length; }
        k = b;
    }
    // ---- the result owns the buffer the runs were copied into (no second host copy)
    zb200_result* res = new zb200_result();
    res->ctx = ctx; res->n = n; res->size = host.size(); res->segs = fsegs;
    res->host_data = std::move(host); res->data = res->host_data.data();
    *out = res;
    return 0;
}

uint64_t zb200_compress_bound(uint64_t n) { return n + (n >> 8) + (n < (128u << 10) ? (((128u << 10) - n) >> 11) : 0); }

const void* zb200_result_data(const zb200_result* r) { return r->data; }
uint64_t zb200_result_size(const zb200_result* r) { return r->size; }
size_t zb200_result_count(const zb200_result* r) { return r->n; }
const zb200_segment* zb200_result_segments(const zb200_result* r)
{
    if (!r->segs_device) return r->segs_pinned ? r->segs_pinned : r->segs.data();
    // a device-resident decode result: its table comes to the host on the first read.  The call that made the result
    // synchronised its stream, so the table is complete; the copy goes on the copy stream, not behind later calls' kernels
    std::lock_guard<std::mutex> g(r->segs_mu);
    if (!r->segs_pinned) {
        zb200_ctx* const ctx = r->ctx;
        cudaSetDevice(ctx->device);
        size_t const bytes = r->n * sizeof(zb200_segment);
        auto* h = (zb200_segment*)pinned_get(ctx, bytes);
        if (!h) { fail(ctx, "pinned segment table", cudaErrorMemoryAllocation); return nullptr; }
        cudaError_t e = cudaMemcpyAsync(h, r->segs_device, bytes, cudaMemcpyDeviceToHost, ctx->copy_stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->copy_stream);
        if (e != cudaSuccess) { pinned_put(ctx, h); fail(ctx, "zb200_result_segments", e); return nullptr; }
        r->segs_pinned = h;
    }
    return r->segs_pinned;
}
int zb200_result_first_error(const zb200_result* r, size_t* item, int* code, uint64_t* got, uint64_t* expected)
{
    if (!r->has_error) return 0;
    if (item) *item = r->err_item; if (code) *code = r->err_code; if (got) *got = r->err_got; if (expected) *expected = r->err_expected;
    return 1;
}
void zb200_result_free(zb200_result* r)
{
    if (!r) return;
    if (r->data && r->data_pinned_pool) pinned_put(r->ctx, r->data);
    if (r->segs_pinned) pinned_put(r->ctx, r->segs_pinned);
    if (r->data && r->data_owned_device) { cudaSetDevice(r->ctx->device); cudaFreeAsync(r->data, r->ctx->stream); }
    if (r->segs_device) { cudaSetDevice(r->ctx->device); cudaFreeAsync(r->segs_device, r->ctx->stream); }
    delete r;
}

// ---------------------------------------------------------------- frame inspection (host, header only)
int zb200_frame_info(const void* src, size_t n, zb200_frame_info_t* o)
{
    ZbHdr h; zb_parse_header((const u8*)src, n, h);
    o->content_size = h.content_size; o->window_size = h.window; o->dict_id = h.dict_id; o->header_size = h.hdr_size;
    o->has_checksum = h.checksum; o->status = h.status;
    return 0;
}

// ---------------------------------------------------------------- profiling
void zb200_profile_enable(zb200_ctx* ctx, int on) { ctx->prof = on != 0; }
void zb200_profile_reset(zb200_ctx* ctx) { memset(ctx->k_ms, 0, sizeof ctx->k_ms); memset(ctx->k_launch, 0, sizeof ctx->k_launch); }
int zb200_profile_read(zb200_ctx* ctx, float ms[ZB200_K_COUNT], uint32_t launches[ZB200_K_COUNT])
{
    memcpy(ms, ctx->k_ms, sizeof ctx->k_ms); memcpy(launches, ctx->k_launch, sizeof ctx->k_launch); return 0;
}
const char* zb200_kernel_name(int k)
{
    static const char* names[ZB200_K_COUNT] = {"zb_scan_frames", "zb_place_frames", "zb_entropy_decode", "zb_execute", "zb_finish",
                                                "zb_compress_blocks", "zb_frame_layout", "zb_write_frames", "zb_verify_checksums",
                                                "zb_chain_index"};
    return (k >= 0 && k < ZB200_K_COUNT && names[k]) ? names[k] : "";
}
// ---------------------------------------------------------------- one batch over several devices
}  // extern "C"
namespace {
struct MultiSlot { zb200_ctx* ctx = nullptr; std::mutex mu; };
std::mutex g_multi_mu;
std::map<std::pair<int, int>, MultiSlot*> g_multi;      // (device, k-th mention of it in a call) -> its context, kept for the process
thread_local std::string g_multi_err;

MultiSlot* multi_slot(int device, int rep)
{
    std::lock_guard<std::mutex> g(g_multi_mu);
    auto& s = g_multi[std::make_pair(device, rep)];
    if (!s) s = new MultiSlot();
    return s;
}

// contiguous, non-empty ranges balanced by input bytes (the rule of python_zstandard_b200/sharding.py::split_ranges, which
// restates the reference's worker partition, c-ext/compressor.c:1183-1200)
std::vector<size_t> multi_cuts(const zb200_segment* segs, size_t n, size_t parts)
{
    std::vector<size_t> cuts{0};
    if (parts > n) parts = n;
    if (parts > 1 && n >= 2) {
        std::vector<u64> cum(n); u64 acc = 0;
        for (size_t i = 0; i < n; i++) { acc += segs[i].length; cum[i] = acc; }
        for (size_t p = 1; p < parts; p++) {
            u64 const target = (u64)((unsigned __int128)acc * p / parts);
            size_t k = (size_t)(std::lower_bound(cum.begin(), cum.end(), target) - cum.begin()) + 1;
            if (k < cuts.back() + 1) k = cuts.back() + 1;
            if (k > n - (parts - p)) k = n - (parts - p);
            cuts.push_back(k);
        }
    }
    cuts.push_back(n);
    return cuts;
}

template <class Call>
int multi_run(const int* devices, int n_devices, const zb200_segment* segs, size_t n, const void* dict, size_t dict_size,
              zb200_result** results, size_t* first_item, Call call)
{
    g_multi_err.clear();
    if (!devices || n_devices <= 0 || !segs || n == 0 || !results) { g_multi_err = "bad arguments"; return -3; }
    for (int k = 0; k < n_devices; k++) { results[k] = nullptr; if (first_item) first_item[k] = n; }
    std::vector<size_t> const cuts = multi_cuts(segs, n, (size_t)n_devices);
    size_t const nr = cuts.size() - 1;
    std::vector<int> rc(nr, 0); std::vector<std::string> msg(nr);
    std::vector<std::thread> th;
    std::map<int, int> seen;
    for (size_t k = 0; k < nr; k++) {
        MultiSlot* const slot = multi_slot(devices[k], seen[devices[k]]++);
        size_t const lo = cuts[k], hi = cuts[k + 1];
        if (first_item) first_item[k] = lo;
        th.emplace_back([=, &rc, &msg] {
            std::lock_guard<std::mutex> g(slot->mu);
            if (!slot->ctx && zb200_ctx_create(devices[k], &slot->ctx) != 0) { rc[k] = -2; msg[k] = "cannot create a context on device " + std::to_string(devices[k]); return; }
            zb200_ddict* dd = nullptr;
            if (dict && dict_size && zb200_ddict_create(slot->ctx, dict, dict_size, &dd) != 0) { rc[k] = -1; msg[k] = zb200_ctx_last_error(slot->ctx); return; }
            rc[k] = call(slot->ctx, lo, hi, dd, &results[k]);
            if (rc[k]) msg[k] = zb200_ctx_last_error(slot->ctx);
            if (dd) zb200_ddict_free(dd);
        });
    }
    for (auto& t : th) t.join();
    for (size_t k = 0; k < nr; k++) if (rc[k]) { g_multi_err = "range " + std::to_string(k) + " (device " + std::to_string(devices[k]) + "): " + msg[k]; return rc[k]; }
    return 0;
}
}  // namespace
extern "C" {

const char* zb200_multi_last_error(void) { return g_multi_err.c_str(); }

int zb200_decompress_batch_multi(const int* devices, int n_devices, const void* src_base, const zb200_segment* segs, size_t n,
                                 const uint64_t* dst_sizes, const void* dict, size_t dict_size, const zb200_dparams* params,
                                 uint32_t flags, zb200_result** results, size_t* first_item)
{
    if (flags & (ZB200_SRC_DEVICE | ZB200_DST_DEVICE | ZB200_SEGS_HOST)) { g_multi_err = "host buffers only"; return -3; }
    return multi_run(devices, n_devices, segs, n, dict, dict_size, results, first_item,
                     [=](zb200_ctx* ctx, size_t lo, size_t hi, zb200_ddict* dd, zb200_result** out) {
                         return zb200_decompress_batch_ex(ctx, src_base, segs + lo, hi - lo, dst_sizes ? dst_sizes + lo : nullptr, dd, params, flags, out);
                     });
}

int zb200_compress_batch_multi(const int* devices, int n_devices, const void* src_base, const zb200_segment* segs, size_t n,
                               const zb200_cparams* params, const void* dict, size_t dict_size, uint32_t flags,
                               zb200_result** results, size_t* first_item)
{
    if (flags & (ZB200_SRC_DEVICE | ZB200_DST_DEVICE | ZB200_SEGS_HOST)) { g_multi_err = "host buffers only"; return -3; }
    return multi_run(devices, n_devices, segs, n, dict, dict_size, results, first_item,
                     [=](zb200_ctx* ctx, size_t lo, size_t hi, zb200_ddict* dd, zb200_result** out) {
                         return zb200_compress_batch(ctx, src_base, segs + lo, hi - lo, params, dd, flags, out);
                     });
}

uint64_t zb200_last_scratch_bytes(const zb200_ctx* ctx) { return ctx->last_scratch; }
int zb200_last_chase_rounds(const zb200_ctx* ctx) { return ctx->last_chase_rounds; }
const char* zb200_last_compress_kernel(const zb200_ctx* ctx) { return ctx->last_compress_kernel; }

}  // extern "C"

// ---------------------------------------------------------------- dictionary training
// zstandard.train_dictionary (c-ext/compressiondict.c:13-146) runs ZDICT_optimizeTrainFromBuffer_fastCover
// (zstd/zstd.c:52408).  The samples go to the device once; hashing, counting, the previous-occurrence table, segment
// selection and finalisation of every candidate run there (zb_train.cuh).  Each finished candidate comes back (at most
// `capacity` bytes) to become a dictionary handle, and is scored by compressing the test samples -- still on the device --
// with it: score = dictionary size + summed frame sizes (COVER_checkTotalCompressedSize, zstd/zstd.c:49352).  The smallest
// score wins, ties go to the first candidate in ZDICT's loop order (d ascending, then k ascending).
namespace {
int train_fail(zb200_ctx* ctx, int code) { ctx->last_error = zb200_error_string(code); return code; }
struct DevAllocs {
    std::vector<void*> p;
    ~DevAllocs() { for (void* q : p) cudaFree(q); }
    template <class T> cudaError_t get(T** out, size_t bytes) { void* q = nullptr; cudaError_t e = cudaMalloc(&q, bytes ? bytes : 1); if (e == cudaSuccess) p.push_back(q); *out = (T*)q; return e; }
};
}  // namespace

extern "C" int zb200_train_dictionary(zb200_ctx* ctx, const void* samples, const size_t* sizes, size_t n, const zb200_train_params* params,
                                      void* out, size_t capacity, size_t* out_size, uint32_t* chosen_k, uint32_t* chosen_d)
{
    if (!ctx || !params || !out || !out_size || (n && (!samples || !sizes))) return fail(ctx, "zb200_train_dictionary: bad arguments", cudaSuccess);
    cudaSetDevice(ctx->device);
    zb200_train_params const P = *params;
    // the parameter checks and the search range of ZDICT_optimizeTrainFromBuffer_fastCover, in its order
    double const split = P.split_point <= 0.0 ? 0.75 : P.split_point;
    u32 const min_d = P.d ? P.d : 6, max_d = P.d ? P.d : 8, min_k = P.k ? P.k : 50, max_k = P.k ? P.k : 2000;
    u32 const steps = P.steps ? P.steps : 40, kstep = std::max((max_k - min_k) / steps, 1u);
    u32 const f = P.f ? P.f : 20, accel = P.accel ? P.accel : 1;
    if (split <= 0 || split > 1) return train_fail(ctx, 42);
    if (accel == 0 || accel > 10) return train_fail(ctx, 42);
    if (min_k < max_d || max_k < min_k) return train_fail(ctx, 42);
    if (n == 0) return train_fail(ctx, 72);
    if (capacity < 256) return train_fail(ctx, 70);
    // FASTCOVER_ctx_init's checks (zstd/zstd.c:52103)
    u32 const nb = (u32)n;
    u32 const n_train = split < 1.0 ? (u32)((double)nb * split) : nb, n_test = split < 1.0 ? nb - n_train : nb;
    std::vector<u64> offs(n + 1, 0);
    for (size_t i = 0; i < n; i++) offs[i + 1] = offs[i] + sizes[i];
    u64 const total = offs[n], train_size = offs[n_train];
    if (total < std::max(min_d, 8u) || total >= 0xFFFFFFFFull || n_train < 5 || n_test < 1 || train_size < 8) return train_fail(ctx, 72);
    u32 const n_dmers = (u32)(train_size - 8 + 1);
    static const u32 fin_pct[11] = {100, 100, 50, 34, 25, 20, 17, 14, 13, 11, 10};      // FASTCOVER_defaultAccelParameters
    u32 const step = accel, n_fin = (u32)((u64)n_train * fin_pct[accel] / 100);       // skip = accel - 1
    // candidates; those FASTCOVER_checkParameters refuses are skipped, as there
    std::vector<ZtCand> cands; u32 max_esz = 1;
    for (u32 d = min_d; d <= max_d; d += 2)
        for (u32 k = min_k; k <= max_k; k += kstep) {
            if ((d == 6 || d == 8) && k <= capacity && d <= k && f >= 1 && f <= 31) {
                cands.push_back(ZtCand{k, d, (d - min_d) / 2, 0});
                u32 num, esz; zt_epochs((u32)capacity, n_dmers, k, num, esz); max_esz = std::max(max_esz, esz);
            }
            if (k > 0xFFFFFFFFu - kstep) break;
        }
    if (cands.empty()) return train_fail(ctx, 1);        // no candidate ran: COVER_best_t's initial (size_t)-1
    u32 const cap = (u32)capacity;
    size_t const tbl = (size_t)4 << f;
    DevAllocs A;
    u8* d_s; u64* d_offs; ZtCand* d_cand; u32 *d_tail, *d_stats, *d_entlen; u8* d_ent; long long* d_res;
    CK(A.get(&d_s, total + 16)); CK(A.get(&d_offs, (n + 1) * 8)); CK(A.get(&d_cand, cands.size() * sizeof(ZtCand)));
    CK(A.get(&d_tail, cands.size() * 4)); CK(A.get(&d_res, cands.size() * 8)); CK(A.get(&d_stats, 512 * 4)); CK(A.get(&d_ent, 512)); CK(A.get(&d_entlen, 4));
    CK(cudaMemcpyAsync(d_s, samples, total, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(d_s + total, 0, 16, ctx->stream));
    CK(cudaMemcpyAsync(d_offs, offs.data(), (n + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_cand, cands.data(), cands.size() * sizeof(ZtCand), cudaMemcpyHostToDevice, ctx->stream));
    ZtSelect S; memset(&S, 0, sizeof S);
    S.samples = d_s; S.cap = cap; S.tail = d_tail; S.cand = d_cand;
    u32* d_freqs[2] = {nullptr, nullptr};
    {   u8* d_last; u32* d_table;
        CK(A.get(&d_last, n_dmers)); CK(A.get(&d_table, tbl));
        for (u32 di = 0; di <= (max_d - min_d) / 2; di++) {
            u32 const d = min_d + 2 * di;
            if (d != 6 && d != 8) continue;
            u32 *h, *pv;
            CK(A.get(&h, (size_t)n_dmers * 4)); CK(A.get(&pv, (size_t)n_dmers * 4)); CK(A.get(&d_freqs[di], tbl));
            zt_launch_hash(d_s, n_dmers, f, d, h, (u32)ctx->sm_count, ctx->stream); CK(cudaGetLastError());
            CK(cudaMemsetAsync(d_freqs[di], 0, tbl, ctx->stream));
            zt_launch_count(h, d_offs, n_train, step, d_freqs[di], (u32)ctx->sm_count, ctx->stream); CK(cudaGetLastError());
            CK(cudaMemsetAsync(d_table, 0xFF, tbl, ctx->stream));
            zt_launch_prev(h, n_dmers, pv, d_last, d_table, ctx->stream); CK(cudaGetLastError());
            S.n_dmers[di] = n_dmers; S.hash[di] = h; S.prev[di] = pv;
        }
    }
    CK(cudaStreamSynchronize(ctx->stream));
    // candidates side by side, in waves that fit the free device memory
    size_t const per = tbl + (size_t)4 * (max_esz + 2) + 2 * (size_t)cap;
    size_t free_b = 0, total_b = 0; CK(cudaMemGetInfo(&free_b, &total_b));
    size_t wave = std::min(cands.size(), std::max((size_t)1, free_b / 2 / per));
    wave = std::min(wave, (size_t)ctx->sm_count * 2);
    u32 *d_wfreqs, *d_diff; u8 *d_dict, *d_out;
    CK(A.get(&d_wfreqs, wave * tbl)); CK(A.get(&d_diff, wave * 4 * (size_t)(max_esz + 2)));
    CK(A.get(&d_dict, wave * (size_t)cap)); CK(A.get(&d_out, wave * (size_t)cap));
    S.freqs = d_wfreqs; S.freqs_stride = tbl / 4; S.diff = d_diff; S.diff_stride = max_esz + 2; S.dict = d_dict;
    // test samples: compressed where they lie, in the uploaded buffer
    std::vector<zb200_segment> tsegs, fsegs;
    for (u32 i = split < 1.0 ? n_train : 0; i < nb; i++) tsegs.push_back(zb200_segment{offs[i], sizes[i]});
    // finalisation samples (ZDICT_countEStats): the first n_fin training samples, each cut to one 128 KiB block
    for (u32 i = 0; i < n_fin; i++) fsegs.push_back(zb200_segment{offs[i], std::min<u64>(sizes[i], 128u << 10)});
    int const level = P.level ? P.level : 3;
    std::vector<u32> tails(cands.size());
    std::vector<u8> host(wave * (size_t)cap), best;
    std::vector<long long> res(cands.size());
    u64 best_score = ~0ull; size_t best_c = 0;
    for (size_t w0 = 0; w0 < cands.size(); w0 += wave) {
        u32 const nw = (u32)std::min(wave, cands.size() - w0);
        for (u32 i = 0; i < nw; i++)
            CK(cudaMemcpyAsync(d_wfreqs + i * (tbl / 4), d_freqs[cands[w0 + i].di], tbl, cudaMemcpyDeviceToDevice, ctx->stream));
        S.first = (u32)w0;
        zt_launch_select(&S, nw, ctx->stream); CK(cudaGetLastError());
        CK(cudaMemcpyAsync(tails.data() + w0, d_tail + w0, nw * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaMemcpyAsync(host.data(), d_dict, (size_t)nw * cap, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        for (u32 i = 0; i < nw; i++) {
            size_t const c = w0 + i;
            // entropy statistics: the finalisation samples compressed with the candidate's content as a raw dictionary
            u32 const csize = cap - tails[c];
            zb200_ddict* raw = nullptr;
            if (csize) { int rc = zb200_ddict_create(ctx, host.data() + (size_t)i * cap + tails[c], csize, &raw); if (rc) return rc < 0 ? rc : -1; }
            CK(cudaMemsetAsync(d_stats, 0, 512 * 4, ctx->stream));
            if (!fsegs.empty()) {
                zb200_cparams cp; memset(&cp, 0, sizeof cp); cp.level = level; cp.write_content_size = 1;
                zb200_result* r = nullptr;
                int const rc = compress_common(ctx, d_s, fsegs.data(), fsegs.size(), &cp, raw, ZB200_SRC_DEVICE | ZB200_SEGS_HOST | ZB200_DST_DEVICE, &r, d_stats);
                zb200_result_free(r);
                if (rc) { zb200_ddict_free(raw); return rc; }
            }
            zb200_ddict_free(raw);
            zt_launch_entropy(d_stats, csize, d_ent, d_entlen, ctx->stream); CK(cudaGetLastError());
            zt_launch_finalize(d_dict + (size_t)i * cap, cap, d_tail + c, d_ent, d_entlen, P.dict_id, d_out + (size_t)i * cap, d_res + c, ctx->stream);
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(res.data() + c, d_res + c, 8, cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaMemcpyAsync(host.data() + (size_t)i * cap, d_out + (size_t)i * cap, cap, cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaStreamSynchronize(ctx->stream));
            u64 score;
            if (res[c] < 0) score = (u64)res[c];                       // (size_t)-code, as ZSTD errors compare in COVER_best_finish
            else {
                const u8* const dict = host.data() + (size_t)i * cap;
                zb200_ddict* dd = nullptr;
                int rc = zb200_ddict_create(ctx, dict, (size_t)res[c], &dd);
                if (rc > 0 || rc == -1) return rc ? rc : -1;
                if (rc < 0) score = (u64)(long long)rc;                // the digest refused the dictionary: its zstd code
                else {
                    zb200_cparams cp; memset(&cp, 0, sizeof cp);
                    cp.level = P.level ? P.level : 3; cp.write_content_size = 1; cp.dict_id = zb200_ddict_id(dd);
                    zb200_result* r = nullptr;
                    rc = compress_common(ctx, d_s, tsegs.data(), tsegs.size(), &cp, dd, ZB200_SRC_DEVICE | ZB200_SEGS_HOST | ZB200_DST_DEVICE, &r);
                    zb200_ddict_free(dd);
                    if (rc) return rc;
                    int code = 0;
                    score = zb200_result_first_error(r, nullptr, &code, nullptr, nullptr) ? (u64)-(long long)code : (u64)res[c] + zb200_result_size(r);
                    zb200_result_free(r);
                }
            }
            if (score < best_score) { best_score = score; best_c = c; best.assign(host.data() + (size_t)i * cap, host.data() + (size_t)i * cap + (res[c] > 0 ? res[c] : 0)); }
        }
    }
    if (best_score > ~0ull - 120) return train_fail(ctx, (int)(0 - best_score));      // ZSTD_isError: every candidate failed
    memcpy(out, best.data(), best.size());
    *out_size = best.size();
    if (chosen_k) *chosen_k = cands[best_c].k;
    if (chosen_d) *chosen_d = cands[best_c].d;
    return 0;
}
