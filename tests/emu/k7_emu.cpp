// tests/emu/k7_emu.cpp -- TEST INFRASTRUCTURE: the product's ray-cast kernel (discregrid_b200/csrc/k7_raycast.cu) compiled for the CPU
// through tests/emu/cuda_emu.h (part of build/bin/libdgemu.so).
#define DG_EMU 1
#include "cuda_emu.h"
#include "../../discregrid_b200/csrc/k7_raycast.cu"
