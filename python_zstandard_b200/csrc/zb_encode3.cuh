// zb_encode3.cuh -- small records with a full dictionary (BASELINE config 4: ~1 KiB records, one frame each): a WARP per
// record, 22 records in flight per SM, everything a record needs in the warp's own slice of shared memory; the dictionary
// (its last <= 32 KiB of content, the hash table built over it, its FSE tables and Huffman code) is staged once per CTA
// and shared read-only.  Included by zb_encode.cu after zb_encode2.cuh (it reuses the helpers of both).
//
// Stands in, per record, for ZSTD_compressBlock_doubleFast_dictMatchState (zstd/zstd.c:31262) + ZSTD_entropyCompressSeqStore:
//   match    32 positions per step, in order: every lane looks its position up in the record's own 1024-entry table
//            (and enters it) and in the dictionary's table, verifies both candidates (common prefix 4..15, 15 = "or more"),
//            keeps the longer; one ballot tells every match where the next one may start and the warp hops along that
//            chain (true greedy + one-step lazy over the whole record: no units, no stitching); long matches are extended
//            256 bytes per vote; every selected lane extends its match backwards and writes {ll, ml, distance}
//   codes    lane 0 walks the sequences forwards: repcodes against the running history (which starts from the
//            dictionary's, ZSTD_loadCEntropy), symbol codes, histograms
//   tables   per stream the cheaper of the dictionary's table ("repeat") and the predefined one (both prebuilt, by cost in
//            1/256 bit); literals: the dictionary's Huffman code ("treeless") when that beats raw
//   write    literals: lanes split the streams, bit counts by prefix scan, every lane packs its own span;
//            sequences: lane 0 runs the three FSE states backwards and writes the bitstream
// Records that do not fit this scheme (more than Z3_SEQ sequences, no gain) are written as raw blocks.
#pragma once

#define Z3_WARPS  22
#define Z3_NT     (Z3_WARPS * 32)
#define Z3_RMAX   2048                    // bytes per record
#define Z3_SEQ    256                     // sequences per record
#define Z3_PLOG   10
#define Z3_MINM   5                       // shortest match with a new offset (a repeated offset: 4): a 4-byte match with ~20 bits of offset does not pay
#define Z3_DMAX   32768                   // dictionary content bytes kept as history

struct Z3Warp {
    __align__(16) u8 rec[Z3_RMAX + 48];   // the record at rec[sk ..], later its literals (compacted in place)
    u16 ptab[1 << Z3_PLOG];
    u64 seq[Z3_SEQ];                      // ll | ml << 12 | distance << 24; later ll | (ml - 3) << 12 | offBase << 24 | lc << 42 | mc << 48
    u16 hist[3][64];
};
struct Z3Shared {
    __align__(16) u8 dtail[Z3_DMAX + 32];
    u16 dtab[1 << ZE_HLOG];
    ZeCTable ct[2][3];                    // [0]: the dictionary's LL, OF, ML tables, [1]: the predefined ones
    u16 cost[2][3][64];                   // bits x 256 per symbol, 0xFFFF = not in the table
    u16 hcode[256]; u8 hnb[256];
    u8 llcode[64], mlcode[128];
    u32 huf_ok;
    Z3Warp w[Z3_WARPS];
};
static_assert(sizeof(Z3Shared) <= 227 * 1024, "Z3Shared exceeds the 227 KB a CTA may own");

__global__ void __launch_bounds__(Z3_NT, 1)
zb_compress_recs(const u8* __restrict__ src, const ZeBlockJob* __restrict__ jobs, u32 n_jobs, u8* __restrict__ slots, u64 slot_bytes,
                 ZeBlockOut* __restrict__ outs, u32* __restrict__ work_counter, ZeDict dict, ZeUpload up)
{
    ZB_DYN_SMEM(z3_smem_raw);
    Z3Shared& S = *(Z3Shared*)z3_smem_raw;
    u32 const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const ZbDictDigest* const de = dict.ent;
    u32 const D = dict.D;

    // ---------------- once per CTA: the dictionary's view
    for (u32 i = tid; i < D; i += Z3_NT) S.dtail[i] = dict.tail[i];
    for (u32 i = tid; i < 32; i += Z3_NT) S.dtail[D + i] = 0;
    for (u32 i = tid; i < (1u << ZE_HLOG) / 2; i += Z3_NT) ((u32*)S.dtab)[i] = ((const u32*)dict.table)[i];
    for (u32 i = tid; i < 3 * sizeof(ZeCTable) / 4; i += Z3_NT) ((u32*)S.ct[0])[i] = ((const u32*)dict.cct)[i];
    if (tid < 64) { u32 c = tid < 16 ? tid : 16; if (tid >= 16) while (c < 35 && tid >= e_LL_base[c + 1]) c++; S.llcode[tid] = (u8)c; }
    if (tid < 128) { u32 c = tid < 32 ? tid : 32; if (tid >= 32) while (c < 52 && tid + 3 >= e_ML_base[c + 1]) c++; S.mlcode[tid] = (u8)c; }
    if (tid < 3) {          // predefined tables (ZSTD_buildCTable set_basic, zstd/zstd.c:21353)
        short nm[56]; u32 const mx = tid == 0 ? 35u : tid == 1 ? 28u : 52u, lg = tid == 1 ? 5u : 6u;
        const short* const dn = tid == 0 ? e_LL_defnorm : tid == 1 ? e_OF_defnorm : e_ML_defnorm;
        for (u32 s = 0; s <= mx; s++) nm[s] = dn[s];
        ze_build_ctable(S.ct[1][tid], nm, mx, lg, S.w[tid].rec);        // (scratch: a record buffer, not yet in use)
        for (u32 s = mx + 1; s < 56; s++) { S.ct[1][tid].dnb[s] = 0; S.ct[1][tid].dfs[s] = 0; }
    }
    if (tid >= 32 && tid < 32 + 6 * 64) {        // cost of every symbol in both table sets
        u32 const k = tid - 32, set = k / 192, t = (k / 64) % 3, s = k & 63;
        u32 const mx = set ? (t == 0 ? 35u : t == 1 ? 28u : 52u) : (t == 0 ? de->c_max_ll : t == 1 ? de->c_max_of : de->c_max_ml);
        u32 const lg = set ? (t == 1 ? 5u : 6u) : (t == 0 ? de->ll_log : t == 1 ? de->of_log : de->ml_log);
        int nrm = 0;
        if (s <= mx) nrm = set ? (int)(t == 0 ? e_LL_defnorm[s] : t == 1 ? e_OF_defnorm[s] : e_ML_defnorm[s])
                               : (int)(t == 0 ? de->c_norm_ll[s] : t == 1 ? de->c_norm_of[s] : de->c_norm_ml[s]);
        if (nrm == -1) nrm = 1;
        S.cost[set][t][s] = nrm > 0 ? (u16)(256.f * ((float)lg - __log2f((float)nrm)) + 0.5f) : (u16)0xFFFF;
    }
    if (tid == 1023 % Z3_NT) {          // the dictionary's Huffman code
        bool ok = de->huf_log != 0 && de->huf_log <= 11;
        ZeHuf* const H = (ZeHuf*)S.w[Z3_WARPS - 1].rec;                 // scratch: 776 bytes of the last warp's record buffer
        for (u32 s = 0; s < 256; s++) H->nb[s] = s <= de->c_huf_max ? de->c_huf_nb[s] : 0;
        if (ok) ze_huf_assign(*H, de->c_huf_max, de->huf_log);
        for (u32 s = 0; s < 256; s++) { S.hcode[s] = ok ? H->code[s] : 0; S.hnb[s] = ok ? H->nb[s] : 0; }
        S.huf_ok = ok ? 1u : 0u;
    }
    __syncthreads();

    Z3Warp& W = S.w[warp];
    const u8* const Dt = S.dtail;
    for (;;) {
        // ---------------- next record
        u32 jn = 0;
        if (lane == 0) {
            jn = atomicAdd(work_counter, 1u);
            if (up.progress && jn < n_jobs) {       // host input still being uploaded: wait until this record (and a margin) has landed
                unsigned long long const want = jobs[jn].src_pos + jobs[jn].size + 256u;
                unsigned long long const need = want < up.total ? want : up.total;
                long long t0 = clock64(); unsigned long long seen = 0;
                for (;;) {
                    unsigned long long const now = *(volatile const unsigned long long*)up.progress;
                    if (now >= need) break;
                    if (now != seen) { seen = now; t0 = clock64(); }
                    __nanosleep(400);
                    if (clock64() - t0 > 6000000000ll) { atomicExch(up.status, 1u); break; }
                }
                __threadfence();
            }
        }
        u32 const j = __shfl_sync(0xFFFFFFFFu, jn, 0);
        if (j >= n_jobs) return;
        ZeBlockJob const job = jobs[j];
        u32 const n = job.size;
        const u8* const gsrc = src + job.src_pos;
        u32 const sk = (u32)((uintptr_t)gsrc & 3);
        u8* const out = slots + (u64)j * slot_bytes;
        u32* const ow = (u32*)out;
        u8* const R = W.rec;                                               // record byte i is R[sk + i]
        u32 const e_end = sk + n;
        {   // load (aligned words), slack, tables, slot
            const u32* const gw = (const u32*)(gsrc - sk);
            for (u32 i = lane; i < (e_end + 3) / 4; i += 32) ((u32*)R)[i] = gw[i];
            __syncwarp();
            for (u32 i = lane; i < 32; i += 32) R[e_end + i] = 0;
            for (u32 i = lane; i < (1u << Z3_PLOG) / 2; i += 32) ((u32*)W.ptab)[i] = 0xFFFFFFFFu;
            for (u32 i = lane; i < 3 * 64 / 2; i += 32) ((u32*)W.hist)[i] = 0;
            for (u32 i = lane; i < (n + 3 + 64) / 4 && i < slot_bytes / 4; i += 32) ow[i] = 0;
            __syncwarp();
        }
        // ================================================================= matches
        u32 nseq = 0, cover = sk; bool overflow = false;
        u32 rep_d = de->rep[0];                                            // the offset of the last match taken: tried at every position (a repcode is cheap to code)
        for (u32 b = 0; b < e_end && cover < e_end; b += 32) {
            u32 const pos = b + lane;
            bool const inr = pos >= sk && pos + 8 <= e_end, valid = inr && pos >= cover;     // every position enters the table, covered or not
            u64 const A = inr ? z2_ld64(R, pos) : 0ull;
            u32 const h = ze_hash4((u32)A);
            u32 c_own = valid ? (u32)W.ptab[h >> (ZE_HLOG - Z3_PLOG)] : 0xFFFFu;
            {   // positions of this very step with my hash: the nearest one below me beats the table (records are short: 32
                // blind positions would be 3 % of one)
                u32 const peers = __match_any_sync(0xFFFFFFFFu, inr ? h : 0x80000000u + lane) & ((1u << lane) - 1u);
                if (valid && peers) c_own = b + (31u - (u32)__clz((int)peers));
            }
            ZB_SIMT_STEP();
            if (inr) W.ptab[h >> (ZE_HLOG - Z3_PLOG)] = (u16)pos;
            ZB_SIMT_STEP();
            u32 const c_dic = valid ? (u32)S.dtab[h] : 0xFFFFu;
            u32 m = 0, d = 0, csrc = 0; bool isd = false;
            if (c_own != 0xFFFFu && c_own < pos) {
                u64 const x = A ^ z2_ld64(R, c_own);
                u32 mo = x ? ze_common8(0, x) : 8 + ze_common8(z2_ld64(R, pos + 8), z2_ld64(R, c_own + 8));
                mo = min(mo, min(15u, e_end - pos));
                if (mo >= Z3_MINM) { m = mo; d = pos - c_own; csrc = c_own; }
            }
            if (c_dic != 0xFFFFu && c_dic + 4 <= D) {
                u64 const x = A ^ z2_ld64(Dt, c_dic);
                u32 md = x ? ze_common8(0, x) : 8 + ze_common8(z2_ld64(R, pos + 8), z2_ld64(Dt, c_dic + 8));
                md = min(md, min(min(15u, e_end - pos), D - c_dic));         // a dictionary match stops at the dictionary's end
                if (md >= Z3_MINM && md > m) { m = md; d = (pos - sk) + (D - c_dic); csrc = c_dic; isd = true; }
            }
            if (valid && rep_d && rep_d != d) {                                   // the same offset as the match before
                u32 const back = pos - sk;                                        // bytes of the record in front of pos
                bool const rd = rep_d > back;                                     // the source lies in the dictionary
                u32 const cs = rd ? D - (rep_d - back) : pos - rep_d;
                if (!rd || rep_d - back <= D) {
                    const u8* const sb = rd ? Dt : (const u8*)R;
                    u64 const x = A ^ z2_ld64(sb, cs);
                    u32 mr = x ? ze_common8(0, x) : 8 + ze_common8(z2_ld64(R, pos + 8), z2_ld64(sb, cs + 8));
                    mr = min(mr, min(15u, e_end - pos));
                    if (rd) mr = min(mr, D - cs);
                    if (mr >= 4 && mr + 1 >= m) { m = mr; d = rep_d; csrc = cs; isd = rd; }
                }
            }
            u32 mn = __shfl_down_sync(0xFFFFFFFFu, m, 1); if (lane == 31) mn = 0;
            bool const take = m >= 4 && !(m < 15 && mn > m + 1);                     // one-step lazy
            u32 const takemask = __ballot_sync(0xFFFFFFFFu, take);
            u32 my_end = pos + m;
            #define Z3_NEXT_FROM(e_) ((e_) >= b + 32 ? 32u : min(32u, (u32)__ffs((int)(takemask & (0xFFFFFFFFu << ((e_) > b ? (e_) - b : 0u)))) - 1u))
            bool const lng = m == 15 && (!isd || csrc + 15 < D);
            u32 my_hop = take ? (Z3_NEXT_FROM(my_end) | (lng ? 0x100u : 0u)) : 0u;
            u32 selmask = 0, lastL = 0;
            u32 L = Z3_NEXT_FROM(cover);
            while (L < 32) {
                selmask |= 1u << L; lastL = L;
                u32 const hop = __shfl_sync(0xFFFFFFFFu, my_hop, (int)L);
                if (hop & 0x100u) {                     // "15 or more": compare on from byte 8, eight bytes per lane and vote
                    u32 const cL = __shfl_sync(0xFFFFFFFFu, csrc, (int)L);
                    bool const dL = __shfl_sync(0xFFFFFFFFu, isd ? 1u : 0u, (int)L) != 0;
                    const u8* const sb = dL ? Dt : (const u8*)R;
                    u32 const s_end = dL ? D : e_end;                                 // where the source side ends
                    u32 a = b + L + 8, c = cL + 8, endL;
                    for (;;) {
                        u32 const my = a + 8 * lane, mc = c + 8 * lane;
                        u32 cm = 8;
                        if (my + 8 <= e_end && mc + 8 <= s_end) { u64 const x = z2_ld64(R, my) ^ z2_ld64(sb, mc); if (x) cm = ze_common8(0, x); }
                        else { cm = 0; while (my + cm < e_end && mc + cm < s_end && R[my + cm] == sb[mc + cm]) cm++; }
                        u32 const stop = __ballot_sync(0xFFFFFFFFu, cm < 8);
                        if (stop) { u32 const fl = (u32)__ffs((int)stop) - 1; endL = a + 8 * fl + __shfl_sync(0xFFFFFFFFu, cm, (int)fl); break; }
                        a += 256; c += 256;
                    }
                    if (lane == L) my_end = endL;
                    L = Z3_NEXT_FROM(endL);
                } else L = hop & 0xFFu;
            }
            u32 my_prev = cover;
            if (selmask) {
                u32 const below = selmask & ((1u << lane) - 1u);
                u32 const pe = __shfl_sync(0xFFFFFFFFu, my_end, below ? 31 - __clz((int)below) : 0);
                if (below) my_prev = pe;
                cover = __shfl_sync(0xFFFFFFFFu, my_end, (int)lastL);
                rep_d = __shfl_sync(0xFFFFFFFFu, d, (int)lastL);
            }
            if ((selmask >> lane) & 1u) {
                u32 start = pos, c = csrc;
                const u8* const sb = isd ? Dt : (const u8*)R;
                while (start > my_prev && c > (isd ? 0u : sk) && R[start - 1] == sb[c - 1] && pos - start < 8) { start--; c--; }
                u32 const idx = nseq + (u32)__popc(selmask & ((1u << lane) - 1u));
                if (idx < Z3_SEQ) W.seq[idx] = (u64)(start - my_prev) | ((u64)(my_end - start) << 12) | ((u64)d << 24);
            }
            nseq += (u32)__popc(selmask);
            if (nseq > Z3_SEQ) { overflow = true; break; }
        }
        __syncwarp();
        u32 const tail_lits = e_end - cover;
        // ================================================================= literals: compact in place, in order
        u32 nlit = 0;
        if (!overflow) {
            u32 srcp = sk, dstp = sk;
            for (u32 i = 0; i < nseq; i++) {
                u64 const r = W.seq[i];
                u32 const ll = (u32)r & 0xFFFu, ml = (u32)(r >> 12) & 0xFFFu;
                for (u32 k0 = 0; k0 < ll; k0 += 32) {
                    u8 v = 0; if (k0 + lane < ll) v = R[srcp + k0 + lane];
                    __syncwarp();
                    if (k0 + lane < ll) R[dstp + k0 + lane] = v;
                    __syncwarp();
                }
                srcp += ll + ml; dstp += ll;
            }
            for (u32 k0 = 0; k0 < tail_lits; k0 += 32) {
                u8 v = 0; if (k0 + lane < tail_lits) v = R[srcp + k0 + lane];
                __syncwarp();
                if (k0 + lane < tail_lits) R[dstp + k0 + lane] = v;
                __syncwarp();
            }
            nlit = dstp + tail_lits - sk;
        }
        const u8* const lit = R + sk;
        // ---- literal section: the dictionary's Huffman code ("treeless") or raw
        bool const four = nlit >= 256;
        u32 const nst = four ? 4u : 1u, seg = four ? (nlit + 3) / 4 : nlit;
        u32 const lps = 32 / nst;                                        // lanes per stream
        u32 const st = lane / lps, li = lane % lps;
        u32 const s0 = st * seg, s1 = four ? (st == 3 ? nlit : s0 + seg) : nlit;
        u32 const part = (s1 - s0 + lps - 1) / lps;
        u32 const p0 = min(s0 + li * part, s1), p1 = min(p0 + part, s1);     // my literals
        u32 mybits = 0; bool badsym = false;
        for (u32 i = p0; i < p1; i++) { u32 const nb = S.hnb[lit[i]]; if (!nb) badsym = true; mybits += nb; }
        bool const huf_usable = S.huf_ok && nlit >= 32 && !overflow && !__any_sync(0xFFFFFFFFu, badsym);
        u32 incl = mybits;                                                // inclusive prefix inside my stream's lane group
        #pragma unroll
        for (int dd = 1; dd < 32; dd <<= 1) { u32 const y = __shfl_up_sync(0xFFFFFFFFu, incl, dd); if (li >= (u32)dd) incl += y; }
        u32 const st_bits = __shfl_sync(0xFFFFFFFFu, incl, (int)(st * lps + lps - 1));
        u32 sb_bytes[4];
        #pragma unroll
        for (u32 k = 0; k < 4; k++) sb_bytes[k] = k < nst ? (__shfl_sync(0xFFFFFFFFu, st_bits, (int)(k * lps)) + 1 + 7) / 8 : 0u;
        u32 const huf_pay = (four ? 6u : 0u) + sb_bytes[0] + sb_bytes[1] + sb_bytes[2] + sb_bytes[3];
        u32 const lh_h = 3 + (nlit >= 1024), lh_r = 1 + (nlit > 31);
        bool const use_huf = huf_usable && huf_pay + lh_h < nlit + lh_r;
        u32 const lh = use_huf ? lh_h : lh_r, lit_pay = use_huf ? huf_pay : nlit;
        u32 const o_lit = 3;                                              // after the block header
        if (!overflow) {
            if (use_huf) {
                if (lane == 0) {
                    u32 hb[4] = {0, 0, 0, 0};
                    if (lh == 3) { u32 const v = 3u | ((four ? 1u : 0u) << 2) | (nlit << 4) | (lit_pay << 14); hb[0] = v; hb[1] = v >> 8; hb[2] = v >> 16; }
                    else { u32 const v = 3u | (2u << 2) | (nlit << 4) | (lit_pay << 18); hb[0] = v; hb[1] = v >> 8; hb[2] = v >> 16; hb[3] = v >> 24; }
                    for (u32 k = 0; k < lh; k++) z2_or_byte(ow, o_lit + k, hb[k]);
                    if (four) for (u32 k = 0; k < 3; k++) { z2_or_byte(ow, o_lit + lh + 2 * k, sb_bytes[k]); z2_or_byte(ow, o_lit + lh + 2 * k + 1, sb_bytes[k] >> 8); }
                }
                u32 sbyte = o_lit + lh + (four ? 6u : 0u);
                #pragma unroll
                for (u32 k = 0; k < 3; k++) if (k < st) sbyte += sb_bytes[k];
                if (li == 0) { u32 const q = sbyte * 8 + st_bits; atomicOr(&ow[q >> 5], 1u << (q & 31)); }       // end mark
                if (p1 > p0) {          // symbols are written last to first: my span ends where the bits before it begin
                    Z2Bits w; w.init(ow, sbyte * 8 + (st_bits - incl));
                    for (u32 i = p1; i-- > p0;) { u32 const sy = lit[i]; w.put(S.hcode[sy], S.hnb[sy]); }
                    w.flush();
                }
            } else {
                if (lane == 0) {
                    if (lh == 1) z2_or_byte(ow, o_lit, nlit << 3);
                    else { u32 const v = (1u << 2) | (nlit << 4); z2_or_byte(ow, o_lit, v); z2_or_byte(ow, o_lit + 1, v >> 8); }
                }
                for (u32 i = lane; i < nlit; i += 32) z2_or_byte(ow, o_lit + lh + i, lit[i]);
            }
        }
        __syncwarp();
        // ================================================================= sequences: lane 0
        u32 total = 0;
        if (lane == 0 && !overflow) {
            u32 r0 = de->rep[0], r1 = de->rep[1], r2 = de->rep[2];
            for (u32 i = 0; i < nseq; i++) {          // forwards: offset codes against the running history, symbol codes, histograms
                u64 const r = W.seq[i];
                u32 const ll = (u32)r & 0xFFFu, ml = (u32)(r >> 12) & 0xFFFu, dist = (u32)(r >> 24);
                u32 const ob = ze_off_code(dist, ll, r0, r1, r2);
                u32 const lc = ll < 64 ? S.llcode[ll] : ze_hibit(ll) + 19, mc = ml - 3 < 128 ? S.mlcode[ml - 3] : ze_hibit(ml - 3) + 36, oc = ze_hibit(ob);
                W.seq[i] = (u64)ll | ((u64)(ml - 3) << 12) | ((u64)ob << 24) | ((u64)lc << 42) | ((u64)mc << 48);
                W.hist[0][lc]++; W.hist[1][oc]++; W.hist[2][mc]++;
            }
            u32 q = o_lit + lh + lit_pay;             // sequences section (ZSTD_entropyCompressSeqStore_internal, zstd/zstd.c:25893-25926)
            if (nseq < 128) z2_or_byte(ow, q++, nseq); else { z2_or_byte(ow, q++, (nseq >> 8) + 0x80); z2_or_byte(ow, q++, nseq); }
            if (nseq) {
                u32 set[3];
                for (u32 t = 0; t < 3; t++) {         // the dictionary's table ("repeat") or the predefined one, by cost
                    u32 c0 = 0, c1 = 0; bool ok0 = true, ok1 = true;
                    for (u32 s = 0; s < 64; s++) { u32 const cnt = W.hist[t][s]; if (!cnt) continue;
                        u32 const a0 = S.cost[0][t][s], a1 = S.cost[1][t][s];
                        if (a0 == 0xFFFFu) ok0 = false; else c0 += cnt * a0;
                        if (a1 == 0xFFFFu) ok1 = false; else c1 += cnt * a1; }
                    set[t] = (ok0 && (!ok1 || c0 <= c1)) ? 0u : 1u;
                    if (!ok0 && !ok1) overflow = true;                    // (cannot happen: the predefined tables cover every code we emit)
                }
                z2_or_byte(ow, q++, ((set[0] ? 0u : 3u) << 6) | ((set[1] ? 0u : 3u) << 4) | ((set[2] ? 0u : 3u) << 2));
                ZeCTable const& cL = S.ct[set[0]][0]; ZeCTable const& cO = S.ct[set[1]][1]; ZeCTable const& cM = S.ct[set[2]][2];
                Z2Bits w; w.init(ow, q * 8);
                u32 i = nseq - 1;
                u64 r = W.seq[i];
                u32 sL = z2_fse_init(cL, (u32)(r >> 42) & 63u), sO = z2_fse_init(cO, ze_hibit((u32)(r >> 24) & 0x3FFFFu)), sM = z2_fse_init(cM, (u32)(r >> 48) & 63u);
                for (;;) {
                    u32 const ll = (u32)r & 0xFFFu, mb = (u32)(r >> 12) & 0xFFFu, ob = (u32)(r >> 24) & 0x3FFFFu;
                    u32 const lc = (u32)(r >> 42) & 63u, mc = (u32)(r >> 48) & 63u, oc = ze_hibit(ob);
                    if (i != nseq - 1) {
                        { u32 const nb = (sO + (u32)cO.dnb[oc]) >> 16; w.put(sO, nb); sO = cO.state[(sO >> nb) + cO.dfs[oc]]; }
                        { u32 const nb = (sM + (u32)cM.dnb[mc]) >> 16; w.put(sM, nb); sM = cM.state[(sM >> nb) + cM.dfs[mc]]; }
                        { u32 const nb = (sL + (u32)cL.dnb[lc]) >> 16; w.put(sL, nb); sL = cL.state[(sL >> nb) + cL.dfs[lc]]; }
                    }
                    w.put(ll, e_LL_bits[lc]); w.put(mb, e_ML_bits[mc]); w.put(ob, oc);
                    if (i == 0) break;
                    r = W.seq[--i];
                }
                w.put(sM, cM.log); w.put(sO, cO.log); w.put(sL, cL.log); w.put(1, 1);
                u32 const endbit = w.w * 32 + w.nacc;
                w.flush();
                q = (endbit + 7) / 8;
            }
            total = q;                                                    // block bytes, header included
        }
        total = __shfl_sync(0xFFFFFFFFu, total, 0);
        bool const raw = overflow || __shfl_sync(0xFFFFFFFFu, overflow ? 1u : 0u, 0) != 0 || total >= n + 3;
        __syncwarp();
        if (raw) {                                  // ZSTD_noCompressBlock, zstd/zstd.c:27337
            for (u32 i = lane; i < (n + 3 + 3) / 4; i += 32) ow[i] = 0;
            __syncwarp();
            for (u32 i = lane; i < n; i += 32) out[3 + i] = gsrc[i];
            if (lane == 0) { u32 const bh = job.last | (n << 3); out[0] = (u8)bh; out[1] = (u8)(bh >> 8); out[2] = (u8)(bh >> 16); outs[j].csize = 3 + n; }
        } else if (lane == 0) {
            u32 const bh = job.last | (2u << 1) | ((total - 3) << 3);
            z2_or_byte(ow, 0, bh); z2_or_byte(ow, 1, bh >> 8); z2_or_byte(ow, 2, bh >> 16);
            outs[j].csize = total;
        }
        __syncwarp();
    }
}
