// tests/emu/k3_volume_emu.cpp -- TEST INFRASTRUCTURE: the K3 emulation surface of k3_emu.cpp (included unchanged: the product's
// k3_density.cu compiled for the CPU, emu_field_create & co.) plus the volume-map entry point, in the form K3's density map has there, for
// tests/test_volume_map_emulated.py.  Built with k2_emu.cpp into build/bin/libk3vemu.so; the product never loads it.
#include "k3_emu.cpp"

extern "C" {

int emu_volume_map(void* h, double hh, double scale, int no_reduction, uint64_t l_begin, uint64_t l_end, double* out)
{
    const EmuField* f = (EmuField*)h;
    return (int)k3_launch_volume(f->dev, hh, scale, no_reduction, l_begin, l_end - l_begin, out, nullptr);
}

}  // extern "C"
