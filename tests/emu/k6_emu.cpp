// tests/emu/k6_emu.cpp -- TEST INFRASTRUCTURE: the product's level-set kernels (discregrid_b200/csrc/k6_isosurface.cu) compiled for the CPU
// through tests/emu/cuda_emu.h (part of build/bin/libdgemu.so).
#define DG_EMU 1
#include "cuda_emu.h"
#include "../../discregrid_b200/csrc/k6_isosurface.cu"
