// tests/emu/k2_hessian_emu.cpp -- TEST INFRASTRUCTURE: the emulated field / interpolate surface of k3_emu.cpp (the product's K3 translation
// unit compiled for the CPU, with emu_field_create / emu_interpolate) plus K2's Hessian mode, for tests/test_k2_hessian_emulated.py.
// Linked with tests/emu/k2_emu.cpp (the product's K2 translation unit) into build/bin/libk2hemu.so.
#include "k3_emu.cpp"

extern "C" {

// K2's Hessian mode on a field of emu_field_create: phi[n], grad[n][3], hess[n][3][3]
int emu_interpolate_hessian(void* h, const double* x, uint64_t n, double* phi, double* grad, double* hess)
{
    return (int)k2_launch_interpolate(((EmuField*)h)->dev, x, n, phi, grad, nullptr, hess);
}

}  // extern "C"
