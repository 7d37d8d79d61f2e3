// Scratch layout of one rasterization (forward -> backward). Like the reference's
// GeometryState / BinningState / ImageState (reference cuda_rasterizer/rasterizer_impl.h:30-64) each
// block is carved out of ONE caller-owned byte chunk and its layout is a pure function of a single
// size (P, num_rendered R, or W*H), so backward can re-derive every pointer from (P, R, W*H) alone
// (the contract at reference rasterizer_impl.cu:370-372). The contents are private to this library.
#pragma once
#include "psb_common.cuh"
#include "psb_sort.cuh"

namespace psb {

template <typename T>
static inline T* carve(char*& chunk, size_t count, size_t alignment = 128)
{
	const uintptr_t p = (reinterpret_cast<uintptr_t>(chunk) + alignment - 1) & ~(uintptr_t)(alignment - 1);
	T* ptr = reinterpret_cast<T*>(p);
	chunk = reinterpret_cast<char*>(ptr + count);
	return ptr;
}

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;
// look-back status words for the scan over P Gaussians (sized for the smaller of the two scan tiles: 1024, emit_scan_kernel)
static inline size_t scan_status_words(size_t P) { return (P + 1023) / 1024 + 1; }

// Per-Gaussian state: function of P.
struct GeomState {
	GaussRec* rec;            // [P] packed screen-space record (see psb_common.cuh)
	// [P] {x0 | y0<<16, x1 | y1<<16, instance count, tile mask}: the tile rectangle, the number of (Gaussian, tile)
	// instances (0 when culled; tight lists: exact count | TT_VISIBLE) and, for tight lists over rectangles of <= 32 tiles,
	// bit k set = tile k (row-major) of the rectangle gets an instance. One 16-byte gather per Gaussian in depth order.
	uint4* tile_info;
	uint32_t* depth_key[2];   // [P] float bits of view-space depth (0xFFFFFFFF when culled), ping-pong
	uint32_t* order[2];       // [P] Gaussian indices, ping-pong; order[0] ends up depth-sorted (4 passes)
	uint32_t* offsets;        // [P] exclusive scan of the instance counts in depth-sorted order (B1/B2 path only)
	uint32_t* counters;       // [32] counters[0] = num_rendered, [1] = scan ticket
	uint32_t* scan_status;    // [scan_status_words(P)]
	char* sort_scratch;       // radix scratch for 4 passes over P
	size_t sort_scratch_bytes;

	static GeomState from_chunk(char*& chunk, size_t P)
	{
		GeomState g;
		g.rec = carve<GaussRec>(chunk, P);
		g.tile_info = carve<uint4>(chunk, P);
		g.depth_key[0] = carve<uint32_t>(chunk, P);
		g.depth_key[1] = carve<uint32_t>(chunk, P);
		g.order[0] = carve<uint32_t>(chunk, P);
		g.order[1] = carve<uint32_t>(chunk, P);
		g.offsets = carve<uint32_t>(chunk, P);
		g.counters = carve<uint32_t>(chunk, 32);
		g.scan_status = carve<uint32_t>(chunk, scan_status_words(P));
		g.sort_scratch_bytes = ::psb::sort_scratch_bytes(P, 4);
		g.sort_scratch = carve<char>(chunk, g.sort_scratch_bytes);
		return g;
	}
};

// Per-instance state: function of R = num_rendered (capacity).
struct BinState {
	uint32_t* tile_key[2];  // [R] tile id of each (Gaussian, tile) instance, ping-pong
	uint32_t* inst[2];      // [R] Gaussian index of each instance, ping-pong
	char* sort_scratch;
	size_t sort_scratch_bytes;

	static BinState from_chunk(char*& chunk, size_t R)
	{
		BinState b;
		b.tile_key[0] = carve<uint32_t>(chunk, R);
		b.tile_key[1] = carve<uint32_t>(chunk, R);
		b.inst[0] = carve<uint32_t>(chunk, R);
		b.inst[1] = carve<uint32_t>(chunk, R);
		b.sort_scratch_bytes = ::psb::sort_scratch_bytes(R, 3);  // tile ids up to 24 bits
		b.sort_scratch = carve<char>(chunk, b.sort_scratch_bytes);
		return b;
	}
};

// Per-pixel state: function of N = W*H (tile count <= N, so per-tile arrays are sized N like the reference).
struct ImgState {
	float* final_T;       // [N] transmittance after the last blended splat
	uint32_t* n_contrib;  // [N] 1-based list position of the last blended splat
	uint2* ranges;        // [N] (only #tiles used) [start, end) of each tile in the sorted instance list

	static ImgState from_chunk(char*& chunk, size_t N)
	{
		ImgState s;
		s.final_T = carve<float>(chunk, N);
		s.n_contrib = carve<uint32_t>(chunk, N);
		s.ranges = carve<uint2>(chunk, N);
		return s;
	}
};

// Scratch of the deterministic operator backward (psb_rasterize_backward_deterministic): function of (P, R). It is a separate,
// caller-allocated chunk, so the three chunks above and psb_*_bytes stay what the forward carved.
struct OpDetState {
	float4* slots;    // [R][3]: one packed sink row per instance (DetSlots::slots)
	uint32_t* base;   // [P] emission offset of each Gaussian with instances (DetSlots::base)

	static OpDetState from_chunk(char*& chunk, size_t P, size_t R)
	{
		OpDetState s;
		s.slots = carve<float4>(chunk, 3 * R);
		s.base = carve<uint32_t>(chunk, P);
		return s;
	}
	static size_t required_bytes(size_t P, size_t R)
	{
		char* p = nullptr;
		from_chunk(p, P, R);
		return reinterpret_cast<size_t>(p) + 128;
	}
};

// Scratch of the operator's normal plane (psb_rasterize_planes_bytes): n_i of every Gaussian, which the forward renders and the backward
// recomputes, the unpacked sink's dL/dn and, for the deterministic backward only (R > 0), the 64-byte slots of its normal variant.
struct OpPlaneState {
	float4* normals;  // [P]
	float* dn;        // [P][3]
	float4* slots;    // [R][4]: one 16-float sink row per instance (DetSlots::slots of a normal pass)

	static OpPlaneState from_chunk(char*& chunk, size_t P, size_t R)
	{
		OpPlaneState s;
		s.normals = carve<float4>(chunk, P);
		s.dn = carve<float>(chunk, 3 * P);
		s.slots = carve<float4>(chunk, 4 * R);
		return s;
	}
	static size_t required_bytes(size_t P, size_t R)
	{
		char* p = nullptr;
		from_chunk(p, P, R);
		return reinterpret_cast<size_t>(p) + 128;
	}
};

template <typename S>
static inline size_t required_bytes(size_t n)
{
	char* p = nullptr;
	S::from_chunk(p, n);
	return reinterpret_cast<size_t>(p) + 128;
}

// The bytes of a chunk that state S is carved from for `count` rows (P, R or W*H): a CudaBuffer<char, ..., StateBytes<S>> counts rows.
template <typename S>
struct StateBytes {
	static size_t of(size_t count) { return required_bytes<S>(count); }
};

static inline int tile_id_bits(int num_tiles)
{
	int b = 1;
	while ((1 << b) < num_tiles) b++;
	return b;
}

}  // namespace psb
