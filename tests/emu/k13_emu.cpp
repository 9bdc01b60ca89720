// tests/emu/k13_emu.cpp -- TEST INFRASTRUCTURE: the product's level-set gradient translation unit (discregrid_b200/csrc/k13_isosurface_grad.cu)
// compiled for the CPU through tests/emu/cuda_emu.h; part of build/bin/libdgemu.so (the K2 and K11 passes it calls are k2_emu.cpp's and
// k11_emu.cpp's).
#define DG_EMU 1
#include "cuda_emu.h"

#include "../../discregrid_b200/csrc/k13_isosurface_grad.cu"
