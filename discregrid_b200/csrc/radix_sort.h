// Launch interface of the device radix sort (radix_sort.cu): a stable LSD sort of (uint32 key, uint32 value) pairs.  Host-callable, no
// kernel code here.  Used by K10 (k10_distance_grad.cu) to group queries by triangle and by K11 (k11_field_grad.cu) to group them by cell; written to be reused (DESIGN §7: reduceField).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace dgb {

constexpr int RS_DIGIT_BITS = 8;                      // one pass per 8 key bits
constexpr unsigned RS_RADIX = 1u << RS_DIGIT_BITS;
constexpr unsigned RS_TILE = 1024;                    // pairs per warp in the histogram and scatter passes
constexpr unsigned RS_SCAN_CHUNK = 1024;              // histogram entries per warp in the scan
constexpr int RS_THREADS = 128;

// digit passes for keys below 2^key_bits: ceil(key_bits / 8), at least 1
int radix_sort_passes(int key_bits);
// bytes of device scratch radix_sort_pairs needs for n pairs
uint64_t radix_sort_scratch_bytes(uint64_t n);

// Sorts n pairs by key, stably (equal keys keep their input order), into keys_out / vals_out.  Every key must be below 2^key_bits
// (1 <= key_bits <= 32); only the digit passes those bits need run.  vals_in NULL stands for the values 0, 1, ..., n - 1.  The inputs
// are not modified and must not overlap the outputs or the scratch (radix_sort_scratch_bytes(n) bytes, 256-byte aligned).  Queued on
// `stream`; no host synchronisation.  n < 2^32; n == 0 launches nothing.
cudaError_t radix_sort_pairs(const uint32_t* keys_in, const uint32_t* vals_in, uint64_t n, int key_bits, uint32_t* keys_out,
                             uint32_t* vals_out, void* scratch, cudaStream_t stream);

// bytes of device scratch exclusive_scan_u32 needs for len entries
uint64_t exclusive_scan_scratch_bytes(uint64_t len);
// In place: a[i] = a[0] + ... + a[i - 1] (a[0] = 0), the sort's own scan.  The total must be below 2^32.  Queued on `stream`.
cudaError_t exclusive_scan_u32(unsigned* a, uint64_t len, void* scratch, cudaStream_t stream);

}  // namespace dgb
