// simt.h -- a minimal SIMT runtime for running CUDA kernels' source on the CPU (test infrastructure only).
//
// Every thread of a CTA is a fiber (ucontext); CTAs run one after another.  Fibers run until they reach a
// synchronisation point -- __syncthreads, __syncwarp or a warp collective (__shfl*_sync, __ballot_sync, __any_sync,
// __all_sync, __match_any_sync) -- where they deposit their operand and yield until every live lane named by the mask
// has arrived.  Between such points a fiber runs alone, so unsynchronised shared-memory traffic of a warp is NOT
// interleaved instruction by instruction as on the device: code whose RESULT depends on that interleaving (the hash
// heads of the compressor's link phase: hints that the parse verifies) may produce different but equally valid output.
// Atomics are plain read-modify-writes (one OS thread).  Exited threads count as arrived, as on the device.
//
// The launchers of the kernel sources compile here as they are: ZB_LAUNCH (zb_common.cuh) becomes simt::launch, and the
// few runtime calls they make are the synchronous definitions at the end of this file.
#pragma once
#include <cuda_runtime.h>
#include <ucontext.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <type_traits>
#include <cmath>
#include <vector>

namespace simt {

struct Dim3 { unsigned x = 1, y = 1, z = 1; };
static Dim3 g_threadIdx, g_blockIdx, g_blockDim, g_gridDim;

struct Thread { ucontext_t ctx; char* stack = nullptr; bool done = false; unsigned warp_gen = 0, cta_gen = 0;
                unsigned wait = 0, wait_mask = 0, nb_gen = 0; };      // wait 4: named barrier wait_mask (id)      // wait: 0 runnable, 1 CTA barrier, 2 previous collective being read, 3 collective arrivals
struct Warp {
    unsigned gen = 0, arrived = 0, read = 0;
    unsigned long long val[32];                 // operands of the collective in flight
};
static std::vector<Thread> g_threads;
static std::vector<Warp> g_warps;
static unsigned g_cta_gen = 0, g_cta_arrived = 0;
static unsigned g_nb_gen[16], g_nb_arrived[16];             // named barriers (bar.sync id, count)
static int g_cur = 0;
static ucontext_t g_sched;
static std::function<void()> g_body;
static unsigned long long g_switches = 0, g_progress = 0;     // g_progress: rendezvous completed / thread finished

static inline unsigned tid() { return g_threadIdx.x; }
static inline void yield() { g_switches++; swapcontext(&g_threads[g_cur].ctx, &g_sched); }
static inline unsigned alive_mask(unsigned warp)
{
    unsigned m = 0, n = (unsigned)g_threads.size();
    for (unsigned l = 0; l < 32 && warp * 32 + l < n; l++) if (!g_threads[warp * 32 + l].done) m |= 1u << l;
    return m;
}

// rendezvous of the live lanes of `mask`; f(values, need) computes this lane's result from the deposited operands
template <class F>
static inline unsigned long long collective(unsigned mask, unsigned long long mine, F f)
{
    unsigned const t = tid(), w = t >> 5, lane = t & 31;
    Warp& W = g_warps[w]; Thread& T = g_threads[t];
    while (W.gen != T.warp_gen) { T.wait = 2; yield(); }       // the previous collective is still being read
    W.val[lane] = mine; W.arrived |= 1u << lane;
    for (;;) { unsigned const need = mask & alive_mask(w); if ((W.arrived & need) == need) break; T.wait = 3; T.wait_mask = mask; yield(); }
    T.wait = 0;
    unsigned const part = W.arrived;                          // the participants: everybody who deposited (a lane may
    unsigned long long const r = f(W.val, part, lane);        //   finish the kernel before the others have read its value)
    W.read |= 1u << lane; T.warp_gen++;
    if ((W.read & part) == part) { W.arrived = 0; W.read = 0; W.gen++; g_progress++; }
    return r;
}

static void trampoline() { g_body(); g_threads[g_cur].done = true; swapcontext(&g_threads[g_cur].ctx, &g_sched); }

// run body() once per thread of every CTA of the grid
static void launch(unsigned grid, unsigned block, std::function<void()> body)
{
    size_t const STACK = 256 << 10;
    static std::vector<char*> stacks;                           // fiber stacks, reused by every CTA of every launch
    while (stacks.size() < block) stacks.push_back((char*)malloc(STACK));
    static ucontext_t proto; static bool have_proto = false;     // every fiber starts from the same saved context
    if (!have_proto) { getcontext(&proto); have_proto = true; }
    g_body = body; g_gridDim.x = grid; g_blockDim.x = block;
    for (unsigned b = 0; b < grid; b++) {
        g_blockIdx.x = b;
        g_threads.assign(block, Thread()); g_warps.assign((block + 31) / 32, Warp());
        g_cta_gen = 0; g_cta_arrived = 0;
        for (int q = 0; q < 16; q++) { g_nb_gen[q] = 0; g_nb_arrived[q] = 0; }
        for (unsigned t = 0; t < block; t++) {
            Thread& T = g_threads[t]; T.stack = stacks[t];
            T.ctx = proto; T.ctx.uc_stack.ss_sp = T.stack; T.ctx.uc_stack.ss_size = STACK; T.ctx.uc_link = &g_sched;
            makecontext(&T.ctx, trampoline, 0);
        }
        unsigned live = block;
        unsigned long long idle_rounds = 0;
        while (live) {
            unsigned long long const before = g_progress;
            unsigned done_now = 0;
            // the CTA barrier is released here as well (threads that exit shrink the quorum), so that waiting fibers need
            // not be resumed just to look at it
            if (g_cta_arrived) { unsigned lv = 0; for (auto& q : g_threads) lv += !q.done; if (g_cta_arrived >= lv) { g_cta_arrived = 0; g_cta_gen++; g_progress++; } }
            for (unsigned t = 0; t < block; t++) {
                Thread& Q = g_threads[t];
                if (Q.done) continue;
                if (Q.wait == 1 && g_cta_gen == Q.cta_gen) continue;                     // still at the barrier
                if (Q.wait == 2 && g_warps[t >> 5].gen != Q.warp_gen) continue;
                if (Q.wait == 4 && g_nb_gen[Q.wait_mask] == Q.nb_gen) continue;
                if (Q.wait == 3) { Warp& W = g_warps[t >> 5]; unsigned const need = Q.wait_mask & alive_mask(t >> 5); if ((W.arrived & need) != need) continue; }
                g_cur = (int)t; g_threadIdx.x = t;
                swapcontext(&g_sched, &g_threads[t].ctx);
                if (g_threads[t].done) done_now++;
            }
            live -= done_now;
            // a round ends when every live fiber waits at a rendezvous; many rounds in a row without any rendezvous
            // completing and without any thread finishing is a deadlock (a lane that never joins a collective)
            if (g_progress == before && !done_now) { if (++idle_rounds > 100000) { fprintf(stderr, "simt: deadlock in CTA %u (grid %u, block %u); waiting threads:", b, grid, block);
                for (unsigned t = 0; t < block; t++) if (!g_threads[t].done) fprintf(stderr, " %u(w%u c%u)", t, g_threads[t].warp_gen, g_threads[t].cta_gen);
                for (size_t w = 0; w < g_warps.size(); w++) fprintf(stderr, " | warp %zu gen %u arrived %08x read %08x", w, g_warps[w].gen, g_warps[w].arrived, g_warps[w].read);
                fprintf(stderr, " | cta gen %u arrived %u\n", g_cta_gen, g_cta_arrived); abort(); } } else idle_rounds = 0;
        }
    }
}

}  // namespace simt

// ---- the CUDA surface the kernels use ----------------------------------------------------------------------------
#define threadIdx simt::g_threadIdx
#define blockIdx simt::g_blockIdx
#define blockDim simt::g_blockDim
#define gridDim simt::g_gridDim
#undef __shared__
#define __shared__ static                      /* one CTA at a time: a function-level static is CTA-shared storage */
#undef __launch_bounds__
#define __launch_bounds__(...)

static inline void __syncthreads()
{
    using namespace simt;
    Thread& T = g_threads[tid()];
    unsigned const my = T.cta_gen;
    auto live = [] { unsigned n = 0; for (auto& t : g_threads) n += !t.done; return n; };
    g_cta_arrived++;
    // the last live thread to arrive releases the generation; threads that exit meanwhile shrink the quorum
    for (;;) {
        if (g_cta_gen != my) break;
        if (g_cta_arrived >= live()) { g_cta_arrived = 0; g_cta_gen++; g_progress++; break; }
        T.wait = 1; yield();
    }
    T.wait = 0; T.cta_gen = my + 1;
}
static inline void simt_named_bar_sync(unsigned id, unsigned count)
{
    using namespace simt;
    Thread& T = g_threads[tid()];
    unsigned const my = g_nb_gen[id];
    if (++g_nb_arrived[id] >= count) { g_nb_arrived[id] = 0; g_nb_gen[id]++; g_progress++; return; }
    T.wait = 4; T.wait_mask = id; T.nb_gen = my;
    while (g_nb_gen[id] == my) yield();
    T.wait = 0;
}
static inline int __syncthreads_or(int p)
{
    static int acc = 0;                    // one CTA at a time
    if (p) acc = 1;
    __syncthreads();
    int const r = acc;
    __syncthreads();
    if (simt::tid() == 0 || simt::g_threads[0].done) acc = 0;
    __syncthreads();
    return r;
}
static inline void __syncwarp(unsigned mask = 0xFFFFFFFFu)
{
    simt::collective(mask, 0, [](const unsigned long long*, unsigned, unsigned) { return 0ull; });
}
template <class T> static inline T simt_bits_to(unsigned long long v) { T r; memcpy(&r, &v, sizeof r); return r; }
template <class T> static inline unsigned long long simt_to_bits(T v) { static_assert(sizeof(T) <= 8, "operand too wide"); unsigned long long r = 0; memcpy(&r, &v, sizeof v); return r; }
template <class T> static inline T __shfl_sync(unsigned mask, T v, int src)
{
    return simt_bits_to<T>(simt::collective(mask, simt_to_bits(v), [src](const unsigned long long* a, unsigned need, unsigned lane) {
        unsigned const s = (unsigned)src & 31; return (need >> s) & 1 ? a[s] : a[lane]; }));
}
template <class T> static inline T __shfl_up_sync(unsigned mask, T v, int d)
{
    return simt_bits_to<T>(simt::collective(mask, simt_to_bits(v), [d](const unsigned long long* a, unsigned need, unsigned lane) {
        return (int)lane - d >= 0 && ((need >> (lane - d)) & 1) ? a[lane - d] : a[lane]; }));
}
template <class T> static inline T __shfl_down_sync(unsigned mask, T v, int d)
{
    return simt_bits_to<T>(simt::collective(mask, simt_to_bits(v), [d](const unsigned long long* a, unsigned need, unsigned lane) {
        return lane + d < 32 && ((need >> (lane + d)) & 1) ? a[lane + d] : a[lane]; }));
}
template <class T> static inline T __shfl_xor_sync(unsigned mask, T v, int x)
{
    return simt_bits_to<T>(simt::collective(mask, simt_to_bits(v), [x](const unsigned long long* a, unsigned need, unsigned lane) {
        unsigned const s = lane ^ (unsigned)x; return s < 32 && ((need >> s) & 1) ? a[s] : a[lane]; }));
}
static inline unsigned __ballot_sync(unsigned mask, int p)
{
    return (unsigned)simt::collective(mask, p ? 1 : 0, [](const unsigned long long* a, unsigned need, unsigned) {
        unsigned r = 0; for (unsigned l = 0; l < 32; l++) if (((need >> l) & 1) && a[l]) r |= 1u << l; return (unsigned long long)r; });
}
static unsigned long long simt_any_calls = 0;      // __any_sync calls by thread 0: the iteration count of vote-driven loops
static inline int __any_sync(unsigned mask, int p) { if (simt::tid() == 0) simt_any_calls++; return __ballot_sync(mask, p) != 0; }
static inline int __all_sync(unsigned mask, int p)
{
    return (int)simt::collective(mask, p ? 1 : 0, [](const unsigned long long* a, unsigned need, unsigned) {
        for (unsigned l = 0; l < 32; l++) if (((need >> l) & 1) && !a[l]) return 0ull; return 1ull; });
}
static inline unsigned __match_any_sync(unsigned mask, unsigned v)
{
    return (unsigned)simt::collective(mask, v, [](const unsigned long long* a, unsigned need, unsigned lane) {
        unsigned r = 0; for (unsigned l = 0; l < 32; l++) if (((need >> l) & 1) && a[l] == a[lane]) r |= 1u << l; return (unsigned long long)r; });
}

template <class T, class U> static inline T atomicAdd(T* p, U v) { T o = *p; *p = (T)(o + (T)v); return o; }
template <class T, class U> static inline T atomicOr(T* p, U v) { T o = *p; *p = (T)(o | (T)v); return o; }
template <class T, class U> static inline T atomicExch(T* p, U v) { T o = *p; *p = (T)v; return o; }
template <class T, class U, class V> static inline T atomicCAS(T* p, U cmp, V v) { T o = *p; if (o == (T)cmp) *p = (T)v; return o; }
template <class T, class U> static inline T atomicMin(T* p, U v) { T o = *p; if ((T)v < o) *p = (T)v; return o; }
template <class T, class U> static inline T atomicMax(T* p, U v) { T o = *p; if ((T)v > o) *p = (T)v; return o; }
static inline void __nanosleep(unsigned) { simt::yield(); }
static inline void __threadfence() {}
static inline void __threadfence_block() {}
static inline long long clock64() { return 0; }
#define __log2f log2f
// the bit reader's funnel shifts (PTX shf.{l,r}.{wrap,clamp}) and the other integer intrinsics
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned s) { unsigned long long v = ((unsigned long long)hi << 32) | lo; return (unsigned)(v >> (s & 31)); }
static inline unsigned __funnelshift_rc(unsigned lo, unsigned hi, unsigned s) { unsigned long long v = ((unsigned long long)hi << 32) | lo; s = s > 32 ? 32 : s; return (unsigned)(s == 32 ? v >> 32 : v >> s); }
static inline unsigned __funnelshift_lc(unsigned lo, unsigned hi, unsigned s) { unsigned long long v = ((unsigned long long)hi << 32) | lo; s = s > 32 ? 32 : s; return (unsigned)((s == 32 ? (v << 31) << 1 : v << s) >> 32); }
static inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
template <class T> static inline T __ldcg(const T* p) { return *p; }

// min / max over mixed integer types, as the CUDA headers provide
template <class A, class B> static inline typename std::common_type<A, B>::type min(A a, B b) { typedef typename std::common_type<A, B>::type T; return (T)a < (T)b ? (T)a : (T)b; }
template <class A, class B> static inline typename std::common_type<A, B>::type max(A a, B b) { typedef typename std::common_type<A, B>::type T; return (T)a > (T)b ? (T)a : (T)b; }

// a CTA's dynamic shared memory (ZB_DYN_SMEM): one CTA runs at a time
alignas(16) static unsigned char simt_dyn_smem[256 << 10];

// the runtime calls of the launchers: the CPU build does not link libcudart, and every launch has finished when it returns
extern "C" cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }
extern "C" cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return cudaSuccess; }
extern "C" cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
