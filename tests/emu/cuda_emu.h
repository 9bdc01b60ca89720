// tests/emu/cuda_emu.h -- TEST INFRASTRUCTURE: runs the product's CUDA device code on the CPU, unchanged, so that the kernels' logic
// (warp-synchronous traversal, index mapping of the launchers, interleaved layouts) is checked against the oracle WITHOUT a GPU.
//
// The emulation TU defines DG_EMU, includes this header and then the .cu file itself.  A kernel "launch" runs the blocks one after the
// other; the 32 lanes of a warp are fibers on one OS thread, resumed round-robin, and a warp collective (__ballot_sync,
// __reduce_add_sync) parks a lane until all live lanes of its warp have arrived -- i.e. the code sees exactly the values it would see
// on the device.  fp64 arithmetic is the host's IEEE arithmetic (the TU is built with -ffp-contract=off, like -fmad=false).
// fp32 arithmetic only feeds the traversal FILTERS, whose decisions must be valid, not bit-identical to the device's -- but a filter whose
// error budget does not cover the device's arithmetic changes results, so what the device does differently from IEEE fp32 is modelled where
// that is cheap: plain fp32 operations are IEEE with subnormals on both sides (no -ftz); sqrt.approx.ftz.f32 flushes subnormal inputs and
// results to zero (dg_emu_ftz; k1_sdf.cu's sqrt_approx); __fdividef returns 0 for 2^126 < |b| (NaN for an infinite numerator, since
// it multiplies by an approximate reciprocal that is 0 there).  The directed-rounding intrinsics are exact for products and within a
// double rounding elsewhere.  NOT modelled, and therefore carried by the error budgets in k1_sdf.cu rather than checked here: the 2-ulp
// error of sqrt.approx and the 2-ulp error of __fdividef on normal operands, and __fdividef on subnormal denominators.
// Not emulated: block-level barriers and shared-memory exchange between warps (K1 has none), inline PTX (guarded in the sources).
#pragma once
#include <cuda_runtime.h>          // vector types, cudaError_t ... (declarations only; nothing of the runtime is called)
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

namespace dg_emu {

struct Idx { unsigned x = 0, y = 0, z = 0; };
inline Idx g_threadIdx, g_blockIdx, g_blockDim, g_gridDim;
inline unsigned long long g_counters[32];        // DG_EMU_COUNT(i) in the kernel sources
inline std::vector<unsigned> g_block_trace;      // DG_EMU_TRACE_BLOCK: block ids in the order the sampling kernel ran them

// Fiber switch: callee-saved registers + stack pointer, no system call (glibc's swapcontext does a sigprocmask per switch, which made a
// warp vote cost ~60 us).  x86-64 System V only -- what the build container and the GPU boxes are.
#if !defined(__x86_64__)
#error "tests/emu needs x86-64 (hand-written fiber switch)"
#endif
extern "C" void dg_emu_switch(void** save_sp, void* load_sp);
__asm__(R"(
    .text
    .weak dg_emu_switch
    .type dg_emu_switch,@function
dg_emu_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
    .size dg_emu_switch, .-dg_emu_switch
)");

struct WarpRun {
    static constexpr int N = 32;
    void* sched_sp = nullptr;
    void* lane_sp[N];
    std::vector<unsigned char> stacks;
    bool finished[N];
    bool waiting[N];
    unsigned contrib[N];           // predicate (ballot) or addend (reduce)
    unsigned result_ballot = 0, result_sum = 0;
    int n_lanes = 0, cur = -1;
    const std::function<void()>* body = nullptr;
};
inline WarpRun* g_warp = nullptr;

extern "C" inline void dg_emu_lane_entry()
{
    WarpRun* w = g_warp;
    const int lane = w->cur;
    (*w->body)();
    w->finished[lane] = true;
    dg_emu_switch(&w->lane_sp[lane], w->sched_sp);        // never resumed
    std::abort();
}

// park the calling lane at a warp collective; returns when every live lane has arrived and the result is available
inline void collective_wait(unsigned value)
{
    WarpRun* w = g_warp;
    const int lane = w->cur;
    w->contrib[lane] = value;
    w->waiting[lane] = true;
    dg_emu_switch(&w->lane_sp[lane], w->sched_sp);
}

inline void run_warp(unsigned first_thread, int n_lanes, const std::function<void()>& body)
{
    static WarpRun w;
    const size_t STACK = 256 * 1024;
    if (w.stacks.empty()) w.stacks.resize(STACK * WarpRun::N + 64);
    w.n_lanes = n_lanes; w.body = &body;
    g_warp = &w;
    for (int l = 0; l < n_lanes; l++) {
        w.finished[l] = false; w.waiting[l] = false;
        uintptr_t top = (uintptr_t)(w.stacks.data() + STACK * (l + 1));
        top &= ~(uintptr_t)15;
        void** sp = (void**)top;
        *--sp = nullptr;                                   // padding: the entry function sees the stack as after a call
        *--sp = (void*)&dg_emu_lane_entry;                 // popped by `ret`
        for (int r = 0; r < 6; r++) *--sp = nullptr;       // rbp rbx r12 r13 r14 r15
        w.lane_sp[l] = sp;
    }
    for (;;) {
        bool any_live = false;
        for (int l = 0; l < n_lanes; l++) {
            if (w.finished[l] || w.waiting[l]) continue;
            any_live = true;
            w.cur = l;
            g_threadIdx.x = first_thread + (unsigned)l;
            dg_emu_switch(&w.sched_sp, w.lane_sp[l]);         // runs until the lane parks at a collective or returns
        }
        bool all_done = true, any_waiting = false;
        for (int l = 0; l < n_lanes; l++) { if (!w.finished[l]) all_done = false; if (w.waiting[l]) any_waiting = true; }
        if (all_done) break;
        if (any_waiting) {                                    // every live lane is parked: resolve the collective
            unsigned mask = 0, sum = 0;
            for (int l = 0; l < n_lanes; l++) if (w.waiting[l]) { if (w.contrib[l]) mask |= 1u << l; sum += w.contrib[l]; }
            w.result_ballot = mask; w.result_sum = sum;
            for (int l = 0; l < n_lanes; l++) w.waiting[l] = false;
        } else if (!any_live) {
            std::fprintf(stderr, "dg_emu: warp made no progress\n"); std::abort();
        }
    }
    g_warp = nullptr;
}

// kernel<<<grid, block, smem>>>(args) : `body` invokes the kernel function for the current thread
inline void launch(unsigned grid, unsigned block, size_t /*smem*/, const std::function<void()>& body)
{
    g_gridDim.x = grid; g_blockDim.x = block;
    for (unsigned b = 0; b < grid; b++) {
        g_blockIdx.x = b;
        for (unsigned t0 = 0; t0 < block; t0 += 32) run_warp(t0, (int)std::min(32u, block - t0), body);
    }
}

}  // namespace dg_emu

// ---- names the device code uses ------------------------------------------------------------------------------------------------
#define threadIdx dg_emu::g_threadIdx
#define blockIdx dg_emu::g_blockIdx
#define blockDim dg_emu::g_blockDim
#define gridDim dg_emu::g_gridDim

inline unsigned __ballot_sync(unsigned, int pred) { dg_emu::collective_wait(pred ? 1u : 0u); return dg_emu::g_warp->result_ballot; }
inline int __any_sync(unsigned m, int pred) { return __ballot_sync(m, pred) != 0u; }
inline unsigned __reduce_add_sync(unsigned, unsigned v) { dg_emu::collective_wait(v); return dg_emu::g_warp->result_sum; }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __ffs(int v) { return __builtin_ffs(v); }
template <class T> inline T __ldg(const T* p) { return *p; }
inline float __int_as_float(int v) { float f; std::memcpy(&f, &v, 4); return f; }
inline double __longlong_as_double(long long v) { double r; std::memcpy(&r, &v, 8); return r; }
// atomics: lanes run one at a time, so plain read-modify-write is atomic here
inline unsigned atomicAdd(unsigned* p, unsigned v) { const unsigned o = *p; *p = o + v; return o; }
inline unsigned long long atomicMax(unsigned long long* p, unsigned long long v) { const unsigned long long o = *p; if (v > o) *p = v; return o; }
inline long long __double_as_longlong(double v) { long long r; std::memcpy(&r, &v, 8); return r; }

// directed rounding to fp32 of a value held exactly (or nearly) in a double
inline float dg_emu_round_dn(double v) { float f = (float)v; return ((double)f > v) ? std::nextafterf(f, -INFINITY) : f; }
inline float dg_emu_round_up(double v) { float f = (float)v; return ((double)f < v) ? std::nextafterf(f, INFINITY) : f; }
inline float __double2float_rd(double v) { return dg_emu_round_dn(v); }
inline float __double2float_ru(double v) { return dg_emu_round_up(v); }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
inline float __fmul_rd(float a, float b) { return dg_emu_round_dn((double)a * (double)b); }      // the product of two floats is exact in a double
inline float __fmul_ru(float a, float b) { return dg_emu_round_up((double)a * (double)b); }
inline float __fadd_ru(float a, float b) { return dg_emu_round_up((double)a + (double)b); }      // exact unless the exponents differ by > 29
inline float __fmaf_rd(float a, float b, float c) { return dg_emu_round_dn(std::fma((double)a, (double)b, (double)c)); }
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __fma_rn(double a, double b, double c) { return std::fma(a, b, c); }
// a * approximate reciprocal of b: for 2^126 < |b| (and b = inf) the reciprocal is 0, so the result is 0 -- or NaN when a is infinite
inline float __fdividef(float a, float b) { return (std::fabs(b) > 0x1p126f) ? a * std::copysign(0.f, b) : a / b; }
// flush-to-zero of the .ftz instructions: a subnormal reads / is written as a zero of the same sign
inline float dg_emu_ftz(float x) { return (std::fabs(x) < 0x1p-126f) ? std::copysign(0.f, x) : x; }
using std::max;
using std::min;
#ifdef __launch_bounds__
#undef __launch_bounds__
#endif
#define __launch_bounds__(...)
