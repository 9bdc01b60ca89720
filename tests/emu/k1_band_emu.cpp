// tests/emu/k1_band_emu.cpp -- TEST INFRASTRUCTURE: tests/emu/k1_emu.cpp (the K1 translation unit compiled for the CPU) plus the
// narrow-band launcher (classifier passes + band form of the node loop, k1_launch_sample_nodes_band) for tests/test_k1_band_emulated.py
// and tools/k1_fuzz.py's band option.
#include "k1_emu.cpp"

#include <cstdlib>

extern "C" {

// nodes [l_begin, l_end) of addFunction with pred(x) = |distance| <= band into out[0 .. l_end - l_begin); scratch from the host heap
int emu_sample_sdf_band(void* h, const double* gd, const uint32_t* res, double sign, double band, uint64_t l_begin, uint64_t l_end, double* out)
{
    GridDev g; if (!to_grid(gd, res, g)) return -1;
    const size_t bytes = k1_band_scratch_bytes(g, l_begin, l_end - l_begin);
    void* scratch = bytes ? std::malloc(bytes) : nullptr;
    const int rc = (int)k1_launch_sample_nodes_band(((EmuMesh*)h)->dev, g, sign, band, l_begin, l_end - l_begin, out, scratch, nullptr);
    std::free(scratch);
    return rc;
}

}  // extern "C"
