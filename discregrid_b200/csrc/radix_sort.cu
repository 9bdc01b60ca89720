// Stable LSD radix sort of (uint32 key, uint32 value) pairs on the device (radix_sort.h), 8 bits per pass.
//
// A pass is three steps, all warp-synchronous (ballot / popc / redux / __syncwarp; no block barrier, no shared memory, no atomics), so that
// tests/emu runs every one of them unchanged:
//   histogram : one warp per tile of RS_TILE pairs.  Per group of 32 pairs, 8 ballots give each digit bit of the 32 keys; the lanes whose
//               digit is d are then the AND of those ballots (or their complements) -- every lane can form that mask for any d.  Lane j
//               counts the digits j, j + 32, ..., j + 224 and writes hist[d][tile] (digit-major).
//   scan      : exclusive prefix sums of hist in that order, so that hist[d][tile] becomes where the pairs of digit d in that tile start in
//               the output: one warp per RS_SCAN_CHUNK entries sums its chunk, one warp scans the chunk sums, one warp per chunk adds.
//               Within 32 lanes the prefix is bit-sliced: sum over bits b of popc(ballot(bit b of v) & lanes below) << b.
//   scatter   : the same tiles in the same order.  A pair goes to hist[d][tile] + (pairs of digit d in earlier groups of the tile) + (lanes
//               below it with digit d in its group); the lowest such lane then advances hist[d][tile] for the next group.  The order of the
//               input among equal digits is therefore kept: the sort is stable.
// Only ceil(key_bits / 8) passes run.  Integer work only: the result does not depend on the launch geometry, the stream or the run.
#include "radix_sort.h"
#include "dg_launch.h"

namespace dgb {
namespace {

constexpr unsigned RS_FULL = 0xffffffffu;

// the lanes of the group (live) whose digit is d, from the ballots of the digit bits
__device__ __forceinline__ unsigned rs_digit_lanes(const unsigned* bits, unsigned live, unsigned d)
{
    unsigned m = live;
#pragma unroll
    for (int b = 0; b < RS_DIGIT_BITS; b++) m &= ((d >> b) & 1u) ? bits[b] : ~bits[b];
    return m;
}

// exclusive prefix sum of v over the lanes of the warp; total = the sum over all lanes (< 2^32)
__device__ __forceinline__ unsigned rs_warp_exclusive(unsigned v, unsigned lane, unsigned& total)
{
    total = __reduce_add_sync(RS_FULL, v);
    const unsigned lt = (1u << lane) - 1u;
    unsigned p = 0;
    for (int b = 0; b < 32 && (total >> b) != 0u; b++) p += (unsigned)__popc(__ballot_sync(RS_FULL, (v >> b) & 1u) & lt) << b;
    return p;
}

__global__ void __launch_bounds__(RS_THREADS)
rs_hist_kernel(const uint32_t* __restrict__ keys, unsigned long long n, int shift, unsigned long long n_tiles, unsigned* __restrict__ hist)
{
    const unsigned long long tile = ((unsigned long long)blockIdx.x * RS_THREADS + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    if (tile >= n_tiles) return;                                   // whole warps
    unsigned cnt[RS_RADIX / 32];
#pragma unroll
    for (unsigned j = 0; j < RS_RADIX / 32; j++) cnt[j] = 0;
    const unsigned long long base = tile * RS_TILE;
    for (unsigned k = 0; k < RS_TILE && base + k < n; k += 32) {
        const unsigned long long i = base + k + lane;
        const bool live = i < n;
        const unsigned dig = live ? (keys[i] >> shift) & (RS_RADIX - 1u) : 0u;
        unsigned bits[RS_DIGIT_BITS];
#pragma unroll
        for (int b = 0; b < RS_DIGIT_BITS; b++) bits[b] = __ballot_sync(RS_FULL, live && ((dig >> b) & 1u));
        const unsigned lv = __ballot_sync(RS_FULL, live);
#pragma unroll
        for (unsigned j = 0; j < RS_RADIX / 32; j++) cnt[j] += (unsigned)__popc(rs_digit_lanes(bits, lv, lane + 32u * j));
    }
#pragma unroll
    for (unsigned j = 0; j < RS_RADIX / 32; j++) hist[(unsigned long long)(lane + 32u * j) * n_tiles + tile] = cnt[j];
}

__global__ void __launch_bounds__(RS_THREADS)
rs_chunk_sum_kernel(const unsigned* __restrict__ a, unsigned long long len, unsigned long long n_chunks, unsigned* __restrict__ sums)
{
    const unsigned long long c = ((unsigned long long)blockIdx.x * RS_THREADS + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    if (c >= n_chunks) return;
    unsigned s = 0;
    for (unsigned k = 0; k < RS_SCAN_CHUNK; k += 32) {
        const unsigned long long i = c * RS_SCAN_CHUNK + k + lane;
        s += __reduce_add_sync(RS_FULL, i < len ? a[i] : 0u);
    }
    if (lane == 0) sums[c] = s;
}

// one warp: lane j scans a contiguous run of the chunk sums in place
__global__ void rs_chunk_offsets_kernel(unsigned* __restrict__ sums, unsigned long long n_chunks)
{
    const unsigned lane = threadIdx.x & 31u;
    const unsigned long long per = (n_chunks + 31) / 32, b = lane * per, e = (b + per < n_chunks) ? b + per : n_chunks;
    unsigned s = 0;
    for (unsigned long long i = b; i < e; i++) s += sums[i];
    unsigned total;
    unsigned run = rs_warp_exclusive(s, lane, total);
    for (unsigned long long i = b; i < e; i++) { const unsigned v = sums[i]; sums[i] = run; run += v; }
}

__global__ void __launch_bounds__(RS_THREADS)
rs_scan_apply_kernel(unsigned* __restrict__ a, unsigned long long len, unsigned long long n_chunks, const unsigned* __restrict__ sums)
{
    const unsigned long long c = ((unsigned long long)blockIdx.x * RS_THREADS + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    if (c >= n_chunks) return;
    unsigned run = sums[c];
    for (unsigned k = 0; k < RS_SCAN_CHUNK; k += 32) {
        const unsigned long long i = c * RS_SCAN_CHUNK + k + lane;
        const unsigned v = i < len ? a[i] : 0u;
        unsigned total;
        const unsigned p = rs_warp_exclusive(v, lane, total);
        if (i < len) a[i] = run + p;
        run += total;
    }
}

__global__ void __launch_bounds__(RS_THREADS)
rs_scatter_kernel(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in, unsigned long long n, int shift,
                  unsigned long long n_tiles, unsigned* cursor, uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out)
{
    const unsigned long long tile = ((unsigned long long)blockIdx.x * RS_THREADS + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    if (tile >= n_tiles) return;
    const unsigned lt = (1u << lane) - 1u;
    const unsigned long long base = tile * RS_TILE;
    for (unsigned k = 0; k < RS_TILE && base + k < n; k += 32) {
        const unsigned long long i = base + k + lane;
        const bool live = i < n;
        const uint32_t key = live ? keys_in[i] : 0u;
        const uint32_t val = live ? (vals_in ? vals_in[i] : (uint32_t)i) : 0u;
        const unsigned dig = (key >> shift) & (RS_RADIX - 1u);
        unsigned bits[RS_DIGIT_BITS];
#pragma unroll
        for (int b = 0; b < RS_DIGIT_BITS; b++) bits[b] = __ballot_sync(RS_FULL, live && ((dig >> b) & 1u));
        const unsigned same = rs_digit_lanes(bits, __ballot_sync(RS_FULL, live), dig);
        unsigned* cur = cursor + (unsigned long long)dig * n_tiles + tile;
        const unsigned at = live ? *cur : 0u;
        __syncwarp();                                              // every lane has read its cursor before the leaders advance them
        if (live) {
            const unsigned rank = (unsigned)__popc(same & lt);
            keys_out[at + rank] = key;
            vals_out[at + rank] = val;
            if (rank == 0) *cur = at + (unsigned)__popc(same);
        }
        __syncwarp();                                              // the next group reads the advanced cursors
    }
}

uint64_t rs_align(uint64_t b) { return (b + 255) & ~(uint64_t)255; }
uint64_t rs_tiles(uint64_t n) { return (n + RS_TILE - 1) / RS_TILE; }
unsigned rs_blocks_for_warps(uint64_t warps) { return (unsigned)((warps * 32 + RS_THREADS - 1) / RS_THREADS); }

}  // namespace

int radix_sort_passes(int key_bits) { return key_bits <= RS_DIGIT_BITS ? 1 : (key_bits + RS_DIGIT_BITS - 1) / RS_DIGIT_BITS; }

uint64_t exclusive_scan_scratch_bytes(uint64_t len) { return rs_align(4 * ((len + RS_SCAN_CHUNK - 1) / RS_SCAN_CHUNK)); }

uint64_t radix_sort_scratch_bytes(uint64_t n)
{
    const uint64_t len = (uint64_t)RS_RADIX * rs_tiles(n);
    return 2 * rs_align(4 * n) + rs_align(4 * len) + exclusive_scan_scratch_bytes(len);
}

cudaError_t exclusive_scan_u32(unsigned* a, uint64_t len, void* scratch, cudaStream_t stream)
{
    if (len == 0) return cudaSuccess;
    const uint64_t chunks = (len + RS_SCAN_CHUNK - 1) / RS_SCAN_CHUNK;
    unsigned* sums = static_cast<unsigned*>(scratch);
    cudaError_t e;
    DG_KERNEL_LAUNCH(rs_chunk_sum_kernel, rs_blocks_for_warps(chunks), RS_THREADS, 0, stream, a, (unsigned long long)len,
                     (unsigned long long)chunks, sums);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    DG_KERNEL_LAUNCH(rs_chunk_offsets_kernel, 1, 32, 0, stream, sums, (unsigned long long)chunks);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    DG_KERNEL_LAUNCH(rs_scan_apply_kernel, rs_blocks_for_warps(chunks), RS_THREADS, 0, stream, a, (unsigned long long)len,
                     (unsigned long long)chunks, sums);
    return DG_AFTER_LAUNCH();
}

cudaError_t radix_sort_pairs(const uint32_t* keys_in, const uint32_t* vals_in, uint64_t n, int key_bits, uint32_t* keys_out,
                             uint32_t* vals_out, void* scratch, cudaStream_t stream)
{
    if (key_bits < 1 || key_bits > 32 || n >= (1ull << 32)) return cudaErrorInvalidValue;
    if (n == 0) return cudaSuccess;
    const uint64_t tiles = rs_tiles(n), len = (uint64_t)RS_RADIX * tiles;
    char* s = static_cast<char*>(scratch);
    uint32_t* alt_keys = reinterpret_cast<uint32_t*>(s); s += rs_align(4 * n);
    uint32_t* alt_vals = reinterpret_cast<uint32_t*>(s); s += rs_align(4 * n);
    unsigned* hist = reinterpret_cast<unsigned*>(s); s += rs_align(4 * len);
    unsigned* sums = reinterpret_cast<unsigned*>(s);
    const int passes = radix_sort_passes(key_bits);
    const uint32_t* src_k = keys_in;
    const uint32_t* src_v = vals_in;
    cudaError_t e;
    for (int p = 0; p < passes; p++) {
        const bool to_out = ((passes - 1 - p) % 2) == 0;           // the last pass writes keys_out / vals_out
        uint32_t* dk = to_out ? keys_out : alt_keys;
        uint32_t* dv = to_out ? vals_out : alt_vals;
        const int shift = p * RS_DIGIT_BITS;
        DG_KERNEL_LAUNCH(rs_hist_kernel, rs_blocks_for_warps(tiles), RS_THREADS, 0, stream, src_k, (unsigned long long)n, shift,
                         (unsigned long long)tiles, hist);
        if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
        if ((e = exclusive_scan_u32(hist, len, sums, stream)) != cudaSuccess) return e;
        DG_KERNEL_LAUNCH(rs_scatter_kernel, rs_blocks_for_warps(tiles), RS_THREADS, 0, stream, src_k, src_v, (unsigned long long)n, shift,
                         (unsigned long long)tiles, hist, dk, dv);
        if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
        src_k = dk; src_v = dv;
    }
    return cudaSuccess;
}

}  // namespace dgb
