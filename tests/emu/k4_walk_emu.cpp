// tests/emu/k4_walk_emu.cpp -- TEST INFRASTRUCTURE: the product's device swap walk (k4_swap_walk in discregrid_b200/csrc/k4_reduce.cu)
// compiled for the CPU through tests/emu/cuda_emu.h, next to the serial host walk it replaces (reduce_swap_walk, reduce_field.cpp), in
// build/bin/libk4emu.so.  Both return m and write the first m positions to perm; emu_k4_swap_walk also reports the pointer-jumping rounds.
#define DG_EMU 1
#include "cuda_emu.h"
#include "../../discregrid_b200/csrc/k4_reduce.cu"
#include "../../discregrid_b200/csrc/reduce_field.h"

extern "C" uint64_t emu_k4_swap_walk(const uint8_t* used, uint64_t n, uint32_t* perm, unsigned* rounds)
{
    const uint64_t tiles = (n + dgb::k4_tile() - 1) / dgb::k4_tile();
    std::vector<unsigned char> d_used(used, used + n);
    std::vector<unsigned> d_tile(tiles + 1), d_flag(1), d_walk(n + 1);
    uint64_t m = 0;
    if (dgb::k4_swap_walk(d_used.data(), n, d_tile.data(), d_flag.data(), d_walk.data(), m, *rounds, nullptr) != cudaSuccess) return ~0ull;
    std::copy(d_walk.begin(), d_walk.begin() + m, perm);
    return m;
}

extern "C" uint64_t emu_reduce_swap_walk(const uint8_t* used, uint64_t n, uint32_t* perm)
{
    std::vector<uint32_t> p;
    const uint64_t m = dgb::reduce_swap_walk(used, n, p);
    std::copy(p.begin(), p.begin() + m, perm);
    return m;
}
