// tests/emu/k10_emu.cpp -- TEST INFRASTRUCTURE: the product's distance-gradient and radix-sort translation units
// (discregrid_b200/csrc/k10_distance_grad.cu, radix_sort.cu) compiled for the CPU through tests/emu/cuda_emu.h.  Part of build/bin/libdgemu.so
// as it is; with K10_EMU_SURFACE it also exports a small extern "C" surface for tests/test_mesh_distance_grad_emulated.py (build/bin/libk10emu.so).
#define DG_EMU 1
#include "cuda_emu.h"

// __syncwarp on the emulation's collective: every live lane arrives before any lane goes on, so what one lane wrote before it is visible to
// the others after it (the scatter pass of radix_sort.cu reads its cursors, syncs, and then the lowest lane of each digit advances them)
inline void __syncwarp(unsigned = 0xffffffffu) { dg_emu::collective_wait(0u); }

#include "../../discregrid_b200/csrc/radix_sort.cu"
#include "../../discregrid_b200/csrc/k10_distance_grad.cu"

#if K10_EMU_SURFACE
#include <vector>
using namespace dgb;

extern "C" {

int emu_k10_sort_passes(int key_bits) { return radix_sort_passes(key_bits); }

// radix_sort_pairs on host arrays ("device" memory is host memory here); vals NULL: the values 0 .. n - 1
int emu_k10_sort(const uint32_t* keys, const uint32_t* vals, uint64_t n, int key_bits, uint32_t* keys_out, uint32_t* vals_out)
{
    std::vector<unsigned char> scratch(radix_sort_scratch_bytes(n) + 256);
    void* s = reinterpret_cast<void*>(((uintptr_t)scratch.data() + 255) & ~(uintptr_t)255);
    return (int)radix_sort_pairs(keys, vals, n, key_bits, keys_out, vals_out, s, nullptr);
}

// k10_launch_check + k10_launch_vjp over F [nT][3] (the incidence table built here as K8's k8_build_topology builds it: vertex-major,
// ascending 3 * triangle + slot).  Returns the number of refused triangle ids (nothing is computed then), or -1 on a launch error.
int emu_k10_vjp(uint64_t n, const double* x, const double* dist, const double* near, const int32_t* tri, const double* bary, const double* g,
                const uint32_t* F, uint64_t nT, uint64_t nV, double* grad_points, double* grad_vertices)
{
    std::vector<uint32_t> inc_begin(nV + 1, 0), inc(3 * nT);
    for (uint64_t i = 0; i < 3 * nT; i++) inc_begin[F[i] + 1]++;
    for (uint64_t v = 0; v < nV; v++) inc_begin[v + 1] += inc_begin[v];
    std::vector<uint32_t> cursor(inc_begin.begin(), inc_begin.end() - 1);
    for (uint64_t i = 0; i < 3 * nT; i++) inc[cursor[F[i]]++] = (uint32_t)i;
    unsigned bad = 0;
    if (k10_launch_check(tri, n, (int)nT, &bad, nullptr) != cudaSuccess) return -1;
    if (bad) return (int)bad;
    K10Topo topo;
    topo.F = F; topo.inc_begin = inc_begin.data(); topo.inc = inc.data(); topo.n_vertices = nV; topo.n_tri = (int)nT;
    K10Query q;
    q.x = x; q.dist = dist; q.near = near; q.tri = tri; q.bary = bary; q.g = g; q.n = n;
    std::vector<unsigned char> scratch(k10_scratch_bytes(n, (int)nT, grad_points != nullptr, grad_vertices != nullptr) + 256);
    void* s = reinterpret_cast<void*>(((uintptr_t)scratch.data() + 255) & ~(uintptr_t)255);
    return k10_launch_vjp(topo, q, grad_points, grad_vertices, s, nullptr) == cudaSuccess ? 0 : -1;
}

}  // extern "C"
#endif
