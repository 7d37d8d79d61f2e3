// CUB-free LSD radix sort (onesweep: one read + one write of the data per digit pass, chained-scan
// with decoupled look-back between thread blocks) for 32-bit keys with 32-bit payloads, plus the
// single-pass prefix sum used by the binning stage. Stable, which the tile lists rely on
// (reference relies on the same property of cub::DeviceRadixSort, rasterizer_impl.cu:303-308).
#pragma once
#include "psb_common.cuh"

namespace psb {

constexpr int RS_THREADS = 256;
constexpr int RS_ITEMS = 16;
constexpr int RS_TILE = RS_THREADS * RS_ITEMS;  // 4096 keys per thread block
constexpr int RS_RADIX = 256;                   // status stride; a pass may use fewer bins
constexpr int RS_MAX_PASS = 4;

struct SortPlan {
	int npass;
	int shift[RS_MAX_PASS];
	int bits[RS_MAX_PASS];
	// the ping-pong buffer radix_sort_pairs leaves the sorted keys and values in
	int result() const { return npass & 1; }
};

// Digit plan covering key bits [0, nbits): ceil(nbits/8) passes of equal width.
SortPlan make_sort_plan(int nbits);

// Scratch layout (uint32 words): hist[RS_MAX_PASS][256] | tickets[16] | status[npass][ntiles][256]
size_t sort_scratch_bytes(size_t max_n, int npass);

// Sorts (keys, vals) of length n (n = *n_dev if n_dev != nullptr, else n_host; n_host must be an upper
// bound used to size grids). Buffers ping-pong: pass p reads buffer (p & 1) and writes buffer ((p+1) & 1);
// the result is in buffer plan.result(). If vals[0] == nullptr is passed with iota_vals = true the
// first pass uses the element index as payload.
int radix_sort_pairs(uint32_t* keys[2], uint32_t* vals[2], bool iota_vals, const uint32_t* n_dev, size_t n_host,
                     const SortPlan& plan, void* scratch, size_t scratch_bytes, cudaStream_t stream);

}  // namespace psb
