/*
 * zb200.h -- C ABI of libzb200.so, the H100-native zstd batch codec.
 *
 * This is the drop-in boundary for python-zstandard's batch path.  Every entry
 * point replaces one piece of the reference's C extension (paths relative to
 * /root/reference):
 *
 *   zb200_decompress_batch      decompress_from_framesources   c-ext/decompressor.c:1186-1455
 *                               (decompress_worker :944-1181, ZSTD_decompressStream call :1150)
 *   zb200_compress_batch        compress_from_datasources      c-ext/compressor.c:1084-1336
 *                               (compress_worker :856-1076, ZSTD_compressStream2 call :1035-1044)
 *   zb200_segment               BufferSegment                  c-ext/python-zstandard.h:307-313
 *   zb200_result                DecompressorDestBuffer / CompressorDestBuffer (+ BufferWithSegments_FromMemory,
 *                               c-ext/bufferutil.c:107-148): one owned buffer + its segment table
 *   zb200_ddict_create / _free  ensure_ddict / ZSTD_createDDict_advanced   c-ext/compressiondict.c:148-162
 *   zb200_frame_info            ZSTD_getFrameHeader_advanced   zstd/zstd.c:43668 (c-ext/frameparams.c)
 *   zb200_error_string          ZSTD_getErrorName              zstd/zstd.c (error_private.c)
 *   zb200_*_batch_multi         the worker partition and pool of both functions above: `threads` workers over contiguous
 *                               ranges balanced by bytes   c-ext/compressor.c:1127,1183-1200; c-ext/decompressor.c:1237,1290-1305
 *   zb200_dparams               ZstdDecompressor(max_window_size=) -> ZSTD_DCtx_setMaxWindowSize   c-ext/decompressor.c:17-60
 *   zb200_decompress_chain      ZstdDecompressor.decompress_content_dict_chain   c-ext/decompressor.c:620-890
 *   zb200_compress_chain        the per-revision ZSTD_CCtx_refPrefix + ZSTD_compress2 loop that writes such a chain (no entry
 *                               point of the reference; tests/chain_ref.py:compress_chain restates the loop)
 *   zb200_cparams.window_log    ZSTD_c_windowLog of ZstdCompressionParameters   c-ext/compressionparams.c:46
 *   zb200_cparams.strategy,     ZSTD_c_strategy / _searchLog / _minMatch of ZstdCompressionParameters, greedy to lazy2 only
 *     .search_log, .min_match   (c-ext/compressionparams.c:198-206)
 *   zb200_host_copy             the write into the result PyBytes   c-ext/decompressor.c:283-352
 *   ZB200_SRC/DST_DEVICE, ZB200_SEGS_HOST, zb200_pointer_device: no counterpart (device-resident callers, SURVEY.md 8(f)-2)
 *
 * Plain pointers and sizes only; no torch / Python types.  All functions return 0 on
 * success or a negative value for an infrastructure failure (CUDA, allocation, bad
 * argument; text via zb200_ctx_last_error).  Codec failures of individual segments are
 * reported per item through zb200_result_first_error, with zstd's own error codes.
 *
 * There is no CPU fallback: every codec entry point runs CUDA kernels on the
 * context's device and fails if no device is present.
 */
#ifndef ZB200_H
#define ZB200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct zb200_ctx zb200_ctx;
typedef struct zb200_result zb200_result;
typedef struct zb200_ddict zb200_ddict;

/* == BufferSegment: native-endian {u64 offset; u64 length} */
typedef struct { uint64_t offset, length; } zb200_segment;

/* per-item codec status: zstd_errors.h values, plus two worker errors of the reference */
#define ZB200_E_UNKNOWN_SIZE   200   /* DecompressorWorkerError_unknownSize  c-ext/decompressor.c:914 */
#define ZB200_E_SIZE_MISMATCH  201   /* DecompressorWorkerError_sizeMismatch c-ext/decompressor.c:913 */

/* flags for the batch calls */
#define ZB200_SRC_DEVICE   1u   /* src_base and segs are device pointers                         */
#define ZB200_DST_DEVICE   2u   /* keep the output on the device (result_data is a device ptr)  */
#define ZB200_SIZES_ARE_CAPACITY 4u /* dst_sizes are upper bounds (decompress(max_output_size=)), not exact sizes */
#define ZB200_SEGS_HOST    8u   /* with ZB200_SRC_DEVICE: segs (and dst_sizes) are HOST arrays -- the data is on the device, its
                                   table where the reference's callers keep it (BufferWithSegments.segments)           */

typedef struct {
    uint64_t content_size;   /* UINT64_MAX when the header has none */
    uint64_t window_size;
    uint32_t dict_id;
    uint32_t header_size;
    uint32_t has_checksum;
    uint32_t status;         /* 0 or a zstd error code */
} zb200_frame_info_t;

/* ---- context: one per (process, device).  Owns a stream, scratch arenas, pinned staging. */
int  zb200_device_count(void);
int  zb200_ctx_create(int device, zb200_ctx** out);
void zb200_ctx_destroy(zb200_ctx* ctx);
const char* zb200_ctx_last_error(const zb200_ctx* ctx);
const char* zb200_error_string(int zstd_code);
int  zb200_ctx_synchronize(zb200_ctx* ctx);
void* zb200_ctx_stream(zb200_ctx* ctx);                 /* cudaStream_t the kernels are launched on */

/* pinned host memory from the context's pool (inputs staged here copy at full PCIe rate) */
void* zb200_host_alloc(zb200_ctx* ctx, size_t bytes);
void  zb200_host_free(zb200_ctx* ctx, void* p);
/* plain device memory helpers for device-resident callers (bench, GPU-native users) */
void* zb200_device_alloc(zb200_ctx* ctx, size_t bytes);
void  zb200_device_free(zb200_ctx* ctx, void* p);
int   zb200_memcpy_h2d(zb200_ctx* ctx, void* dst, const void* src, size_t bytes);
int   zb200_memcpy_d2h(zb200_ctx* ctx, void* dst, const void* src, size_t bytes);
/* host-to-host copy on several threads: moving a large result out of the pinned pool into a caller's (not yet touched)
   buffer is bound by page faults on one thread (~3 GB/s); the reference writes into its PyBytes in place
   (c-ext/decompressor.c:283-352), this is the equivalent step after the device-to-host copy */
void  zb200_host_copy(void* dst, const void* src, size_t bytes);
/* the device a pointer belongs to (cudaPointerGetAttributes), -1 for host memory: device-resident callers hand in
   buffers they did not get from zb200_device_alloc (a torch tensor, a __cuda_array_interface__ object) */
int   zb200_pointer_device(const void* p);

/* ---- dictionaries (device-resident digest) */
int  zb200_ddict_create(zb200_ctx* ctx, const void* dict, size_t size, zb200_ddict** out);
void zb200_ddict_free(zb200_ddict* d);
uint32_t zb200_ddict_id(const zb200_ddict* d);

/* ---- batch decompression.
 * src_base + segs[i].offset .. +length is the i-th compressed frame (FramePointer, c-ext/decompressor.c:892-897).
 * dst_sizes: optional u64[n] of expected decompressed sizes (`decompressed_sizes`), NULL = use the
 * frame headers' content size.  On success *out owns the output buffer and its segment table. */
int zb200_decompress_batch(zb200_ctx* ctx, const void* src_base, const zb200_segment* segs, size_t n,
                           const uint64_t* dst_sizes, const zb200_ddict* dict, uint32_t flags,
                           zb200_result** out);
/* same, from an array of independent host buffers (list-of-bytes input, c-ext/decompressor.c:1601-1685) */
int zb200_decompress_batch_ptrs(zb200_ctx* ctx, const void* const* srcs, const size_t* sizes, size_t n,
                                const uint64_t* dst_sizes, const zb200_ddict* dict, uint32_t flags,
                                zb200_result** out);

/* ---- decompression parameters: what ZstdDecompressor(max_window_size=...) configures (c-ext/decompressor.c:17-60,
 * ZSTD_DCtx_setMaxWindowSize zstd/zstd.c:45025).  As in the reference's streaming decoder (zstd/zstd.c:45406-45453) the
 * limit binds for frames whose header carries no content size -- the others take the single-pass path that needs no
 * window buffer.  A frame over the limit fails with code 16, "Frame requires too much memory for decoding". */
typedef struct {
    uint64_t max_window_size;     /* 0 = the reference's default, (1 << 27) + 1 (ZSTD_MAXWINDOWSIZE_DEFAULT, zstd/zstd.c:43465) */
    uint32_t reserved[2];
} zb200_dparams;
int zb200_decompress_batch_ex(zb200_ctx* ctx, const void* src_base, const zb200_segment* segs, size_t n,
                              const uint64_t* dst_sizes, const zb200_ddict* dict, const zb200_dparams* params,
                              uint32_t flags, zb200_result** out);
int zb200_decompress_batch_ptrs_ex(zb200_ctx* ctx, const void* const* srcs, const size_t* sizes, size_t n,
                                   const uint64_t* dst_sizes, const zb200_ddict* dict, const zb200_dparams* params,
                                   uint32_t flags, zb200_result** out);

/* ---- content-dictionary chains: decompress_content_dict_chain.  srcs[k] (sizes[k] bytes, host memory) is chunk k, one zstd
 * frame with its content size in the header; chunk k >= 1 is decoded with chunk k-1's fulltext as a raw-content prefix
 * (ZSTD_DCtx_refPrefix_advanced(..., ZSTD_dct_rawContent)), chunk 0 with first_dict (or none).  On success *out holds one
 * segment, the last fulltext.  A chunk that fails -- a header check (bad frame, no content size, a dictionary ID on a
 * prefixed chunk, a content size, window or prefix + content size of 2 GiB - 128 MiB or more: code 16) or its decoding --
 * is reported through zb200_result_first_error as (chunk, zstd code); the lowest failing chunk wins, and chunks behind the
 * first header failure are not looked at.  A chunk that starts with a skippable frame has an empty fulltext.
 * params: accepted for API parity; a chain frame always has a content size, and then the reference does not apply the limit.
 * The chain is decoded in runs of consecutive chunks sized to free device memory (ZB200_CHAIN_RUN_BYTES overrides the
 * budget, for tests); each run starts from the previous run's last fulltext. */
int zb200_decompress_chain(zb200_ctx* ctx, const void* const* srcs, const size_t* sizes, size_t n,
                           const zb200_ddict* first_dict, const zb200_dparams* params, zb200_result** out);

/* ---- one batch over several devices: the `threads` argument of the reference's batch calls as a C entry point.
 * The items are cut into contiguous ranges balanced by input bytes -- the reference's static worker partition
 * (c-ext/compressor.c:1127,1183-1200; c-ext/decompressor.c:1237,1290-1305) --, range k runs on devices[k] in its own context
 * (created on first use and kept by the library; a device may be named more than once and then gets a context per mention),
 * all ranges concurrently, and comes back as results[k]: what the reference returns per worker, in item order.
 * results[k] is NULL and first_item[k] = n where the partition has fewer than n_devices ranges.  Host buffers only
 * (no ZB200_SRC_DEVICE / ZB200_DST_DEVICE).  dict / dict_size: the raw dictionary or NULL; digested per device.
 * Returns 0, or the first failing range's code with its text in zb200_multi_last_error() (per-item codec errors are in
 * the results, as always). */
int zb200_decompress_batch_multi(const int* devices, int n_devices, const void* src_base, const zb200_segment* segs, size_t n,
                                 const uint64_t* dst_sizes, const void* dict, size_t dict_size, const zb200_dparams* params,
                                 uint32_t flags, zb200_result** results, size_t* first_item);
const char* zb200_multi_last_error(void);

/* ---- batch compression.
 * src_base + segs[i].offset .. +length is the i-th input (DataSource, c-ext/compressor.c:805-808).
 * Every input becomes one zstd frame (RFC 8878) of independent <=128 KiB blocks. */
typedef struct {
    int32_t  level;               /* accepted for API parity; the GPU parse is one strategy (level-3 class) */
    uint32_t write_checksum;      /* append XXH64 content checksum  (ZSTD_c_checksumFlag)    */
    uint32_t write_content_size;  /* frame content size in header   (ZSTD_c_contentSizeFlag) */
    uint32_t dict_id;             /* dictionary id to record, 0 = none (ZSTD_c_dictIDFlag)   */
    uint32_t window_log;          /* 0 = default (21); 10..31: ZSTD_c_windowLog (c-ext/compressionparams.c:46): frames up to 2^W are
                                     single-segment, larger ones declare a 2^W window; blocks are cut to min(2^W, 128 KiB) */
    uint32_t strategy;            /* 0 = the level's own parse; 3 greedy, 4 lazy, 5 lazy2: ZSTD_c_strategy (c-ext/compressionparams.c:206),
                                     the hash-chain lazy parse of zb_compress_blocks for every block whatever the level, dictionary
                                     or block size; the other strategies fail the call */
    uint32_t search_log;          /* with a strategy: 2^min(search_log, 6) chain candidates per position (ZSTD_c_searchLog); 0 = 1,
                                     level 3's; at most 30 */
    uint32_t min_match;           /* with a strategy: bytes hashed and shortest match, clamp(min_match, 4, 6) (ZSTD_c_minMatch);
                                     0 = 5, level 3's; 3..7 */
} zb200_cparams;
/* dict: optional dictionary (the same handle decompression uses; compression sees its last <= 32 KiB of
 * content as history before every frame, ZSTD_CCtx_refCDict / loadDictionary_byReference, c-ext/compressor.c:1146-1168) */
int zb200_compress_batch(zb200_ctx* ctx, const void* src_base, const zb200_segment* segs, size_t n,
                         const zb200_cparams* params, const zb200_ddict* dict, uint32_t flags, zb200_result** out);
/* one batch over several devices, as zb200_decompress_batch_multi */
int zb200_compress_batch_multi(const int* devices, int n_devices, const void* src_base, const zb200_segment* segs, size_t n,
                               const zb200_cparams* params, const void* dict, size_t dict_size, uint32_t flags,
                               zb200_result** results, size_t* first_item);
/* same, from an array of independent host buffers (list input, c-ext/compressor.c:1434-1466) */
int zb200_compress_batch_ptrs(zb200_ctx* ctx, const void* const* srcs, const size_t* sizes, size_t n,
                              const zb200_cparams* params, const zb200_ddict* dict, uint32_t flags, zb200_result** out);
/* ---- content-dictionary chains, compression: the inverse of zb200_decompress_chain.  srcs[k] (sizes[k] bytes, host memory) is
 * revision k; *out holds n segments, frame k for chunk k.  Frame 0 is what zb200_compress_batch_ptrs writes for chunk 0 with
 * `dict` and `params`, except that its content size is always written.  Every frame k >= 1 is chunk k compressed with chunk
 * k-1 as a raw-content prefix: single segment (window = content size), content size, dictionary ID 0, a checksum when
 * params->write_checksum is set; its match sources may lie anywhere in chunk k-1 (DESIGN.md section 4).  The chunks are cut into runs sized to free device
 * memory (ZB200_CHAIN_RUN_BYTES overrides the budget, for tests); each run carries the previous run's last chunk as its
 * prefix, and the frames do not depend on where the runs are cut.  A chunk of ZB_FAR_WINDOW (2 GiB - 128 MiB) bytes or more,
 * or with its predecessor that many, fails the call: the chain decoder refuses such chunks. */
int zb200_compress_chain(zb200_ctx* ctx, const void* const* srcs, const size_t* sizes, size_t n,
                         const zb200_cparams* params, const zb200_ddict* dict, zb200_result** out);
/* ZSTD_compressBound (zstd/zstd.c:4547) */
uint64_t zb200_compress_bound(uint64_t src_size);

/* ---- dictionary training: zstandard.train_dictionary (c-ext/compressiondict.c:13-146), which runs
 * ZDICT_optimizeTrainFromBuffer_fastCover (zstd/zstd.c:52408).  Fields left at 0 take ZDICT's defaults or search ranges:
 * d in {6, 8}, k in 50..2000 over `steps` (40) steps, f 20, accel 1, split_point 0.75, level 3, an ID derived from the
 * content.  The caller applies train_dictionary's own defaulting (d 8, steps 4, level 3 when steps and threads are 0).
 * The samples (host memory, packed back to back, sizes[i] bytes each) are uploaded once; hashing, counting, segment
 * selection and finalisation of every candidate run on the device, each candidate is scored by compressing the test
 * samples with it (zb200_compress_batch on the uploaded buffer), and the winner is copied to `out` (capacity bytes).
 * Returns 0, a positive zstd error code when training fails as the reference's would (its name through
 * zb200_ctx_last_error), or a negative value for an infrastructure failure. */
typedef struct {
    uint32_t k, d, f, steps, accel;
    int32_t  level;               /* level of the candidate score's compression, 0 = 3 */
    uint32_t dict_id;             /* 0 = XXH64 of the content, as ZDICT_finalizeDictionary */
    uint32_t reserved;
    double   split_point;         /* fraction of the samples trained on; the rest score the candidates. 0 = 0.75, 1 = all both */
} zb200_train_params;
int zb200_train_dictionary(zb200_ctx* ctx, const void* samples, const size_t* sizes, size_t n, const zb200_train_params* params,
                           void* out, size_t capacity, size_t* out_size, uint32_t* chosen_k, uint32_t* chosen_d);

/* ---- result accessors */
const void*          zb200_result_data(const zb200_result* r);       /* host (pinned; pageable for zb200_compress_chain) or device pointer */
uint64_t             zb200_result_size(const zb200_result* r);       /* bytes in data */
size_t               zb200_result_count(const zb200_result* r);
/* host array, count entries, valid until zb200_result_free.  A decode result copies its table into pinned memory of the
 * context's pool; one that stays on the device (ZB200_DST_DEVICE) keeps the table on the device until the first call of
 * this function, which copies it and waits for the copy (later calls return the same array).  NULL if that copy fails
 * (zb200_ctx_last_error says why). */
const zb200_segment* zb200_result_segments(const zb200_result* r);
/* first failing item (lowest index wins, like the reference's worker error scan):
 * returns 0 if every item succeeded, else 1 and fills item/code/got/expected */
int  zb200_result_first_error(const zb200_result* r, size_t* item, int* code, uint64_t* got, uint64_t* expected);
void zb200_result_free(zb200_result* r);

/* ---- frame inspection on the host (no GPU work; header parse only) */
int zb200_frame_info(const void* src, size_t size, zb200_frame_info_t* out);

/* ---- profiling: with profiling on, every kernel launch is bracketed by CUDA events on the
 * context's stream; times accumulate per kernel until reset. */
#define ZB200_K_SCAN     0
#define ZB200_K_PLACE    1
#define ZB200_K_ENTROPY  2
#define ZB200_K_EXECUTE  3
#define ZB200_K_FINISH   4
#define ZB200_K_COMPRESS 5
#define ZB200_K_LAYOUT   6
#define ZB200_K_FRAMES   7
#define ZB200_K_VERIFY   8
#define ZB200_K_CHAIN_INDEX 9   /* zb_chain_index (zb200_compress_chain) */
#define ZB200_K_COUNT    16
void zb200_profile_enable(zb200_ctx* ctx, int on);
void zb200_profile_reset(zb200_ctx* ctx);
/* ms[k] = summed device time of kernel k, launches[k] = its launch count */
int  zb200_profile_read(zb200_ctx* ctx, float ms[ZB200_K_COUNT], uint32_t launches[ZB200_K_COUNT]);
const char* zb200_kernel_name(int k);
/* bytes of intermediate state the last batch call allocated (sequence records, literals, tables) */
uint64_t zb200_last_scratch_bytes(const zb200_ctx* ctx);
/* pointer-doubling rounds of the last decompress call that took the pointer-jumping execute stage (0: it did not) */
int      zb200_last_chase_rounds(const zb200_ctx* ctx);
/* the block kernel the last compress call ran: "zb_compress_smem", "zb_compress_recs", "zb_compress_blocks" or, with a
   strategy, "zb_compress_lazy" (the lazy mode of zb_compress_blocks; they all share the profile slot named zb_compress_blocks) */
const char* zb200_last_compress_kernel(const zb200_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif
