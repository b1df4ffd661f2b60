// simt_tables.cpp -- the entropy decoder's table builders on the CPU build of zb_decode.cu (test infrastructure).
//
// tests/test_entropy_tables_host.py builds this file with the flags of tests/host_encoder.py and checks every cell these
// wrappers return against a fixture.  They call the kernels' own builders: nothing here restates them.
#include "simt.h"
#include "zb_decode.cu"

extern "C" {
// the tANS decode table of one sequence stream (kind 0 LL, 1 OF, 2 ML) in both cell formats: the entropy kernels' 16-bit
// ZB_CELL16 and the 32-bit ZbFseCell of the predefined and dictionary tables.  norm is read, not consumed.
void tt_build_fse(const short* norm, u32 max_sym, u32 log, int kind, u16* cells16, u32* cells32)
{
    short nn[64];
    for (u32 s = 0; s <= max_sym; s++) nn[s] = norm[s];
    zb_build_fse(cells16, nn, max_sym, log, kind);
    for (u32 s = 0; s <= max_sym; s++) nn[s] = norm[s];
    zb_build_fse((ZbFseCell*)cells32, nn, max_sym, log, kind);
}
// a Huffman tree description -> the lane workspace as the entropy kernels leave it (256 nibble weights, then the weight
// stream's 64-cell FSE table when the weights are FSE-coded), the weights' counts, log, symbol count; returns bytes used
u32 tt_huf_weights(const u8* s, u32 n, u8* ws, u32* rank, u32* log, u32* nsym)
{
    memset(ws, 0, 256);
    u32 lg = 0, ns = 0;
    u32 const used = zb_huf_weights(ws, s, n, lg, ns, rank);
    *log = lg; *nsym = ns;
    return used;
}
// the split Huffman decode table of those weights (cells: 4096 entries); returns its bytes
u32 tt_huf_fill(const u8* ws, u32 log, u32 nsym, const u32* rank, u16* cells)
{
    u32 shift, T, base, bytes;
    zb_huf_shape(log, rank, shift, T, base, bytes);
    zb_huf_fill(cells, ws, log, nsym, rank, shift, base);
    return bytes;
}
u32 tt_read_ncount(short* norm, u32* max_sym, u32* log, const u8* s, u32 n)
{
    u32 ms = *max_sym, lg = 0; u32 const r = zb_read_ncount(norm, ms, lg, s, n); *max_sym = ms; *log = lg; return r;
}
}
