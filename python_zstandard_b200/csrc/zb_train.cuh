// zb_train.cuh -- dictionary training on the device: the fastCover trainer that zstandard.train_dictionary runs
// (ZDICT_optimizeTrainFromBuffer_fastCover, zstd/zstd.c:52408), restated for sm_90a.
//
// Included at the end of zb_encode.cu, so that finalisation reuses the encoder's Huffman, NCount and XXH64 helpers.
// Every kernel sizes its loops from blockDim, so the CPU build of tests/simt.h can run it with small CTAs.
//
//   zt_hash_all     hash of every d-mer of the training buffer (ZSTD_hash6Ptr / ZSTD_hash8Ptr into f bits)
//   zt_count        FASTCOVER_computeFrequency (:52074): training samples only, every (skip + 1)-th position, global atomics
//   zt_prev_local   previous position with the same hash, inside a chunk of ZT_CHUNK positions (bitonic sort in shared memory)
//   zt_prev_link    the same across chunks: one CTA walks the chunks in order with a last-position table of 2^f entries
//   zt_select       FASTCOVER_buildDictionary (:52190), one CTA per candidate (k, d).  Every window score of an epoch at once:
//                   d-mer j counts towards the window [a, e) iff a <= j < e and prev[j] < a, so it adds freq[h_j] to the ends
//                   e in [max(j + 1, prev[j] + W + 1), j + W] (the prev bound only when prev[j] is inside the epoch), a
//                   difference array and a prefix sum give every score, the first strict maximum is the segment
//   zt_entropy      entropy section of the dictionary header (Huffman table, OF / ML / LL NCounts, repcodes) from the
//                   literal and code counts zb_compress_blocks<.., STATS = true> gathers over the finalisation samples
//   zt_finalize     ZDICT_finalizeDictionary (:53416): ID from XXH64 of the content, shrink to capacity, zero padding
#pragma once

#define ZT_CHUNK 4096u
#define ZT_NONE  0xFFFFFFFFu
#define ZT_DICT_MAGIC 0xEC30A437u

struct ZtCand { u32 k, d, di, pad; };       // di: index of d's tables (0: the first d of the search, 1: the second)

struct ZtSelect {
    const u8* samples;
    u32 n_dmers[2];
    const u32* hash[2];
    const u32* prev[2];
    u32* freqs; u64 freqs_stride;           // per CTA: a private copy of the frequency table of its d
    u32* diff; u64 diff_stride;             // per CTA: the epoch's difference array
    u8* dict; u32 cap;                      // per CTA: cap bytes, filled from the back
    u32* tail;                              // per candidate: first used byte of its dict buffer
    const ZtCand* cand; u32 first;          // CTA b runs candidate first + b
};

// COVER_computeEpochs (:49220) with passes = 1, in the reference's u32 arithmetic
__device__ __host__ inline void zt_epochs(u32 cap, u32 n_dmers, u32 k, u32& num, u32& size)
{
    u32 const min_size = k * 10;
    num = cap / k; if (num < 1) num = 1;
    size = n_dmers / num;
    if (size >= min_size) return;
    size = min_size < n_dmers ? min_size : n_dmers;
    num = n_dmers / size;
}

#ifndef ZT_TYPES_ONLY          // zb_api.cu takes the argument types only

__device__ __forceinline__ u64 zt_ld64(const u8* p)
{
    u64 v = 0;
    for (int i = 7; i >= 0; i--) v = (v << 8) | p[i];
    return v;
}
// FASTCOVER_hashPtrToIndex (:51882): ZSTD_hash6Ptr for d = 6, ZSTD_hash8Ptr otherwise; both read 8 bytes
__device__ __forceinline__ u32 zt_hash(const u8* p, u32 f, u32 d)
{
    u64 const v = zt_ld64(p);
    if (d == 6) return (u32)(((v << 16) * 227718039650203ull) >> (64 - f));
    return (u32)((v * 0xCF1BBCDCB7A56463ull) >> (64 - f));
}

__global__ void zt_hash_all(const u8* __restrict__ s, u32 n_dmers, u32 f, u32 d, u32* __restrict__ hash)
{
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < n_dmers; j += (u64)gridDim.x * blockDim.x)
        hash[j] = zt_hash(s + j, f, d);
}

// offs[0..n_train]: sample starts in the training buffer.  A position counts when it is a multiple of `step` into its
// sample and the 8 bytes the hash reads end inside the sample.
__global__ void zt_count(const u32* __restrict__ hash, const u64* __restrict__ offs, u32 n_train, u32 step, u32* __restrict__ freqs)
{
    u64 const total = offs[n_train];
    for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (u64)gridDim.x * blockDim.x) {
        u32 lo = 0, hi = n_train - 1;             // the last sample starting at or before p
        while (lo < hi) { u32 const mid = (lo + hi + 1) >> 1; if (offs[mid] <= p) lo = mid; else hi = mid - 1; }
        if ((p - offs[lo]) % step == 0 && p + 8 <= offs[lo + 1]) atomicAdd(&freqs[hash[p]], 1u);
    }
}

// prev[j] for the positions of one chunk: the previous position of the chunk with the same hash, ZT_NONE for the first
// one (zt_prev_link fills those in); last[j] = 1 for the last position of the chunk with its hash
__global__ void zt_prev_local(const u32* __restrict__ hash, u32 n, u32* __restrict__ prev, u8* __restrict__ last)
{
    __shared__ u64 key[ZT_CHUNK];
    u32 const c0 = blockIdx.x * ZT_CHUNK, m = min(ZT_CHUNK, n - c0);
    for (u32 i = threadIdx.x; i < ZT_CHUNK; i += blockDim.x) key[i] = i < m ? ((u64)hash[c0 + i] << 32) | (c0 + i) : ~0ull;
    __syncthreads();
    for (u32 size = 2; size <= ZT_CHUNK; size <<= 1)
        for (u32 stride = size >> 1; stride > 0; stride >>= 1) {
            for (u32 t = threadIdx.x; t < ZT_CHUNK / 2; t += blockDim.x) {
                u32 const i = 2 * t - (t & (stride - 1)), j = i + stride;
                u64 const a = key[i], b = key[j];
                if ((a > b) == ((i & size) == 0)) { key[i] = b; key[j] = a; }
            }
            __syncthreads();
        }
    for (u32 i = threadIdx.x; i < m; i += blockDim.x) {
        u64 const kv = key[i]; u32 const h = (u32)(kv >> 32), pos = (u32)kv;
        prev[pos] = i > 0 && (u32)(key[i - 1] >> 32) == h ? (u32)key[i - 1] : ZT_NONE;
        last[pos] = i + 1 == m || (u32)(key[i + 1] >> 32) != h;
    }
}

// one CTA; table: 2^f entries set to ZT_NONE
__global__ void zt_prev_link(const u32* __restrict__ hash, u32 n, u32* __restrict__ prev, const u8* __restrict__ last, u32* __restrict__ table)
{
    for (u32 c0 = 0; c0 < n; c0 += ZT_CHUNK) {
        u32 const m = min(ZT_CHUNK, n - c0);
        for (u32 i = threadIdx.x; i < m; i += blockDim.x) if (prev[c0 + i] == ZT_NONE) prev[c0 + i] = table[hash[c0 + i]];
        __syncthreads();
        for (u32 i = threadIdx.x; i < m; i += blockDim.x) if (last[c0 + i]) table[hash[c0 + i]] = c0 + i;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(1024) zt_select(ZtSelect A)
{
    __shared__ u32 s_sum[32], s_max[32], s_at[32];
    ZtCand const C = A.cand[A.first + blockIdx.x];
    u32 const tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = (nt + 31) >> 5;
    u32 const n = A.n_dmers[C.di];
    const u32* const hash = A.hash[C.di];
    const u32* const prev = A.prev[C.di];
    u32* const fr = A.freqs + blockIdx.x * A.freqs_stride;
    u32* const diff = A.diff + blockIdx.x * A.diff_stride;
    u8* const dict = A.dict + (u64)blockIdx.x * A.cap;
    u32 const k = C.k, d = C.d, W = k - d + 1;
    u32 num, esz; zt_epochs(A.cap, n, k, num, esz);
    u32 tail = A.cap, epoch = 0, zero_run = 0;        // the same in every thread
    while (tail > 0) {
        u32 const eb = epoch * esz, ee = eb + esz;
        epoch = (epoch + 1) % num;
        for (u32 i = tid; i <= esz + 1; i += nt) diff[i] = 0;
        __syncthreads();
        for (u32 j = eb + tid; j < ee; j += nt) {
            u32 const fq = fr[hash[j]];
            if (!fq) continue;
            u64 lo = (u64)j + 1; u32 const p = prev[j];
            if (p != ZT_NONE && p >= eb && (u64)p + W + 1 > lo) lo = (u64)p + W + 1;
            u64 const hi = min((u64)j + W, (u64)ee);
            if (lo <= hi) { atomicAdd(&diff[lo - eb], fq); atomicAdd(&diff[hi + 1 - eb], 0u - fq); }
        }
        __syncthreads();
        // score of the window ending at e = eb + i is diff[1] + .. + diff[i] (mod 2^32, as the reference's running score)
        u32 carry = 0, best = 0, best_i = 0;
        for (u32 t0 = 1; t0 <= esz; t0 += 4 * nt) {
            u32 const b = t0 + 4 * tid;
            u32 v[4], run = 0;
            for (int q = 0; q < 4; q++) { v[q] = b + q <= esz ? diff[b + q] : 0u; run += v[q]; }
            u32 x = run;
            for (int o = 1; o < 32; o <<= 1) { u32 const y = __shfl_up_sync(0xFFFFFFFFu, x, o); if (lane >= (u32)o) x += y; }
            if (lane == 31 || tid == nt - 1) s_sum[warp] = x;
            __syncthreads();
            u32 base = carry, total = 0;
            for (u32 w = 0; w < nw; w++) { if (w < warp) base += s_sum[w]; total += s_sum[w]; }
            u32 acc = base + x - run, m = 0, at = 0;
            for (int q = 0; q < 4; q++) { acc += v[q]; if (b + q <= esz && acc > m) { m = acc; at = b + q; } }
            for (int o = 16; o > 0; o >>= 1) {
                u32 const om = __shfl_down_sync(0xFFFFFFFFu, m, o), oa = __shfl_down_sync(0xFFFFFFFFu, at, o);
                if (lane + o < 32 && (om > m || (om == m && oa < at))) { m = om; at = oa; }
            }
            if (lane == 0) { s_max[warp] = m; s_at[warp] = at; }
            __syncthreads();
            for (u32 w = 0; w < nw; w++) if (s_max[w] > best) { best = s_max[w]; best_i = s_at[w]; }
            carry += total;
            __syncthreads();
        }
        if (best == 0) {                              // nothing new in this epoch
            if (++zero_run >= 10) break;
            continue;
        }
        zero_run = 0;
        u32 const e = eb + best_i, a = e >= eb + W ? e - W : eb;
        u32 const seg = min(e - a + d - 1, tail);
        if (seg < d) break;
        tail -= seg;
        for (u32 i = tid; i < seg; i += nt) dict[tail + i] = A.samples[a + i];
        for (u32 p = a + tid; p < e; p += nt) fr[hash[p]] = 0;
        __syncthreads();
    }
    if (tid == 0) A.tail[A.first + blockIdx.x] = tail;
}

// ZDICT_analyzeEntropy (:53217) from the counts ZDICT_countEStats gathers (stats: the STATS output of zb_compress_blocks over
// the finalisation samples, compressed with the candidate's content as a raw dictionary).  Every count starts at 1 -- OF
// codes up to highbit(content + 128 KiB) --; the Huffman code is limited to 11 bits (ZDICT_flatLit's counts when it comes
// out flat at 8 bits); the OF / ML / LL tables are normalised at logs 8 / 9 / 9; repcodes 1 4 8.  One thread.
// out: >= 256 bytes; *out_len = bytes written, 0 if a table cannot be built.
__global__ void zt_entropy(const u32* __restrict__ stats, u32 content_size, u8* __restrict__ out, u32* __restrict__ out_len)
{
    if (threadIdx.x || blockIdx.x) return;
    u32 lit[256], ll[36], ml[53], of[32];
    ZeHuf H; u32 wk[1600]; ZeCTable ct; u8 tmp[512]; short norm[56];
    u32 const of_max = ze_hibit(content_size + (128u << 10));
    u32 n_ll = 0, n_ml = 0, n_of = 0;
    for (u32 s = 0; s < 256; s++) lit[s] = 1 + stats[s];
    for (u32 s = 0; s < 36; s++) { ll[s] = 1 + stats[256 + s]; n_ll += ll[s]; }
    for (u32 s = 0; s < 53; s++) { ml[s] = 1 + stats[292 + s]; n_ml += ml[s]; }
    for (u32 s = 0; s <= of_max; s++) { of[s] = 1 + stats[345 + s]; n_of += of[s]; }
    *out_len = 0;
    bool ok = ze_huf_build(H, lit, wk);
    if (ok && H.log == 8) {
        for (u32 s = 1; s < 256; s++) lit[s] = 2;
        lit[0] = 4; lit[253] = 1; lit[254] = 1;
        ok = ze_huf_build(H, lit, wk);
    }
    u32 o = ok ? ze_huf_write_table(out, H, ct, tmp) : 0;
    if (!o) return;
    if (!ze_normalize(norm, of, of_max, n_of, 8)) return;
    o += ze_write_ncount(out + o, norm, of_max, 8);
    if (!ze_normalize(norm, ml, 52, n_ml, 9)) return;
    o += ze_write_ncount(out + o, norm, 52, 9);
    if (!ze_normalize(norm, ll, 35, n_ll, 9)) return;
    o += ze_write_ncount(out + o, norm, 35, 9);
    u32 const rep[3] = {1, 4, 8};
    for (u32 r = 0; r < 3; r++) for (u32 b = 0; b < 4; b++) out[o++] = (u8)(rep[r] >> (8 * b));
    *out_len = o;
}

// ZDICT_finalizeDictionary (:53416) for one candidate: header + padding + content into out (cap bytes), the size or a zstd
// error code as a negative number into *res.  content = dict + *tail, cap - *tail bytes.
__global__ void zt_finalize(const u8* __restrict__ dict, u32 cap, const u32* __restrict__ tail, const u8* __restrict__ ent,
                            const u32* __restrict__ ent_len, u32 dict_id, u8* __restrict__ o, long long* __restrict__ res)
{
    __shared__ u32 s_id;
    u32 const t = *tail;
    const u8* const content = dict + t;
    u32 const csize = cap - t, el = *ent_len, hsize = 8 + el;
    if (threadIdx.x == 0) {
        u64 const r = ze_xxh64(content, csize);
        s_id = dict_id ? dict_id : (u32)(r % ((1u << 31) - 32768u)) + 32768u;
    }
    __syncthreads();
    if (el == 0) { if (threadIdx.x == 0) *res = -1; return; }                      // GENERIC
    if (hsize + 8 > cap) { if (threadIdx.x == 0) *res = -70; return; }             // dstSize_tooSmall
    u32 const cs = hsize + csize > cap ? cap - hsize : csize;                       // the content's first bytes stay
    u32 const pad = cs < 8 ? 8 - cs : 0;
    for (u32 i = threadIdx.x; i < cs; i += blockDim.x) o[hsize + pad + i] = content[i];
    for (u32 i = threadIdx.x; i < pad; i += blockDim.x) o[hsize + i] = 0;
    for (u32 i = threadIdx.x; i < el; i += blockDim.x) o[8 + i] = ent[i];
    if (threadIdx.x == 0) {
        for (u32 b = 0; b < 4; b++) { o[b] = (u8)(ZT_DICT_MAGIC >> (8 * b)); o[4 + b] = (u8)(s_id >> (8 * b)); }
        *res = (long long)(hsize + pad + cs);
    }
}

extern "C" {

void zt_launch_hash(const u8* s, u32 n_dmers, u32 f, u32 d, u32* hash, u32 sms, cudaStream_t st)
{
    zt_hash_all<<<sms * 8, 256, 0, st>>>(s, n_dmers, f, d, hash);
}
void zt_launch_count(const u32* hash, const u64* offs, u32 n_train, u32 step, u32* freqs, u32 sms, cudaStream_t st)
{
    zt_count<<<sms * 8, 256, 0, st>>>(hash, offs, n_train, step, freqs);
}
void zt_launch_prev(const u32* hash, u32 n, u32* prev, u8* last, u32* table, cudaStream_t st)
{
    zt_prev_local<<<(n + ZT_CHUNK - 1) / ZT_CHUNK, 1024, 0, st>>>(hash, n, prev, last);
    zt_prev_link<<<1, 1024, 0, st>>>(hash, n, prev, last, table);
}
void zt_launch_select(const void* a, u32 n_ctas, cudaStream_t st) { zt_select<<<n_ctas, 1024, 0, st>>>(*(const ZtSelect*)a); }
void zt_launch_entropy(const u32* stats, u32 content_size, u8* ent, u32* ent_len, cudaStream_t st)
{
    zt_entropy<<<1, 32, 0, st>>>(stats, content_size, ent, ent_len);
}
void zt_launch_finalize(const u8* dict, u32 cap, const u32* tail, const u8* ent, const u32* ent_len, u32 dict_id, u8* out, long long* res,
                        cudaStream_t st)
{
    zt_finalize<<<1, 256, 0, st>>>(dict, cap, tail, ent, ent_len, dict_id, out, res);
}

}  // extern "C"

#endif  // ZT_TYPES_ONLY
