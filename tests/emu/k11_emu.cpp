// tests/emu/k11_emu.cpp -- TEST INFRASTRUCTURE: the product's field-gradient translation unit (discregrid_b200/csrc/k11_field_grad.cu)
// compiled for the CPU through tests/emu/cuda_emu.h; part of build/bin/libdgemu.so (the radix sort it calls is k10_emu.cpp's).
#define DG_EMU 1
#include "cuda_emu.h"

// The warp shuffles of K11's first level on the emulation's collective: every live lane publishes its value, waits until all have, reads
// its source lane's, and waits again so that no lane overwrites its value before every lane has read.  Every lane of K11's warps is live.
namespace dg_emu {
inline double shfl_exchange(double v, unsigned src)
{
    static double slot[32];
    slot[g_warp->cur] = v;
    collective_wait(0u);
    const double r = slot[src];
    collective_wait(0u);
    return r;
}
}  // namespace dg_emu
inline double __shfl_sync(unsigned, double v, int src) { return dg_emu::shfl_exchange(v, (unsigned)src & 31u); }
inline double __shfl_down_sync(unsigned, double v, unsigned d)
{
    const unsigned lane = (unsigned)dg_emu::g_warp->cur;
    return dg_emu::shfl_exchange(v, lane + d < 32u ? lane + d : lane);
}

#include "../../discregrid_b200/csrc/k11_field_grad.cu"
